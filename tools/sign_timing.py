"""tools/sign_timing.py -- what the secret-key paths cost on the GPU: blsSignHash (H(m) cold / cached) and blsGetPublicKey latency, the
batch entries hbls_sign_hash_batch / hbls_get_public_key_batch at k = 1, 64, 1 024, 16 384, and the constant-time ladder kernels against
the variable-time ladders they replaced (tests/ct/ct_driver.cu, CUDA events, the two forms alternated in one process) on sparse and
dense keys.  Prints the card name and power limit first, then one JSON line per measurement.

    python tools/sign_timing.py [--driver libct_time.so] [--reps N]

--driver: a build of tests/ct/ct_driver.cu without probes (compiled here into a temporary directory when omitted).
"""
import argparse, ctypes, json, os, random, subprocess, statistics, sys, tempfile, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from harmony_b200 import bls, build, workload as wl          # noqa: E402

Z = 0xd201000000010000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def median_ms(fn, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def api(reps):
    sk = bls.SecretKey(); sk.Deserialize(wl.sk_bytes(wl.seeded_sk("timing", 0)))
    sk.SignHash(wl.commit_payload("timing-warm", 0)); sk.GetPublicKey()
    n = [0]
    def cold():
        n[0] += 1; assert sk.SignHash(wl.commit_payload("timing-cold", n[0])) is not None
    hot = wl.commit_payload("timing-hot", 0)
    emit(what="blsSignHash", hm="cold", ms=median_ms(cold, reps))
    emit(what="blsSignHash", hm="cached", ms=median_ms(lambda: sk.SignHash(hot), reps))
    emit(what="blsGetPublicKey", ms=median_ms(sk.GetPublicKey, reps))
    for k in (1, 64, 1024, 16384):
        sks = b"".join(wl.sk_bytes(wl.seeded_sk("timing-b", i)) for i in range(k))
        msgs = b"".join(wl.commit_payload("timing-b", i) for i in range(k))
        r = max(3, reps // (1 + k // 64))
        bls.SignHashBatch(sks, msgs, 48); bls.GetPublicKeyBatch(sks)
        emit(what="hbls_sign_hash_batch", k=k, ms=median_ms(lambda: bls.SignHashBatch(sks, msgs, 48), r))
        emit(what="hbls_get_public_key_batch", k=k, ms=median_ms(lambda: bls.GetPublicKeyBatch(sks), r))


def digits(k):
    d = []
    for _ in range(3):
        d.append(k % Z); k //= Z
    return d + [k]


def ladders(path, reps):
    L = ctypes.CDLL(path)
    L.ct_time.argtypes = [ctypes.c_int, ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_uint64), ctypes.c_char_p, ctypes.c_uint32,
                          ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    n = 16384
    rng = random.Random(7)
    # sparse: bits 250 and 0 only (the variable-time 256-bit ladders skip all but two windows) and, for the psi ladder, the digits
    # (1, 0, 0, 2^40) (all but two columns zero); dense: every 4-bit window non-zero, random base-|z| digits
    dense = [(int("f" * 62, 16) ^ rng.getrandbits(60)) | (1 << 252) | int("1" * 62, 16) for _ in range(n)]
    sets = {"sparse": [(1 << 250) | 1] * n, "dense": dense}
    psi_sets = {"sparse": [1 + Z ** 3 * 2 ** 40] * n, "dense": dense}
    msg = wl.commit_payload("timing-ladder", 0)
    names = {0: ("g1_generator", "variable"), 1: ("g1_generator", "constant"), 2: ("g2_256bit_pair", "variable"),
             3: ("g2_256bit_pair", "constant"), 4: ("g2_psi_pair", "variable"), 5: ("g2_psi_pair", "constant")}
    res = {}
    for rnd in range(3):                                    # alternate the forms and key sets; keep the best of three rounds
        for which in range(6):
            for kind, keys in (psi_sets if which >= 4 else sets).items():
                sk = b"".join(k.to_bytes(32, "little") for k in keys)
                dig = (ctypes.c_uint64 * (4 * n))(*[x for k in keys for x in digits(k)])
                ms = ctypes.c_float()
                assert L.ct_time(which, n, sk, dig, msg, len(msg), reps, ctypes.byref(ms)) == 0
                key = (which, kind)
                res[key] = min(res.get(key, 1e30), ms.value)
    for which in range(6):
        ladder, form = names[which]
        s, d = res[(which, "sparse")], res[(which, "dense")]
        emit(what="ladder_kernel", ladder=ladder, form=form, items=n, sparse_ms=s, dense_ms=d, dense_over_sparse=d / s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--driver"); ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    bls.Init(device=0)
    api(a.reps)
    path = a.driver
    if not path:
        path = os.path.join(tempfile.mkdtemp(prefix="hbls_sign_timing_"), "libct_time.so")
        subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + build.NVCC_FLAGS
                              + ["-o", path, os.path.join(ROOT, "tests", "ct", "ct_driver.cu")])
    ladders(path, max(3, a.reps // 10))


if __name__ == "__main__":
    main()
