"""tools/multikey_sign_time.py -- what a node with k BLS keys pays to sign one consensus message with all of them, at k = 1, 4, 10, 32, 100,
with H(m) cold (a message not seen before, as each new block hash / commit payload is) and cached (the same message again):

    (a) the reference's loop through the C ABI (consensus/construct.go:97-114): k blsSignHash + blsSignatureAdd, then blsSignatureSerialize
    (b) hbls_sign_hash_keys, aggregate only
    (c) hbls_sign_hash_keys, per-key signatures and aggregate
    (d) the view-change shape: hbls_sign_hash_keys with k keys x 2 messages, per-key signatures (view_change_construct.go:402-483), and
        (d_ref) its reference loop: 2 k blsSignHash + blsSignatureSerialize

Every call returns with its results on the host, so a host clock around each call is its latency.  Prints the card name and power limit
first, then one JSON line per (shape, k, H(m) state): median, 10th / 90th percentile, min and max in ms.  (a) and (b) are checked to
give the same bytes at each k before they are timed.

    python tools/multikey_sign_time.py [--reps N]
"""
import argparse, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from harmony_b200 import bls, workload as wl          # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(fn, reps):
    t = []
    for i in range(reps):
        t0 = time.perf_counter(); fn(i); t.append((time.perf_counter() - t0) * 1e3)
    t.sort()
    q = statistics.quantiles(t, n=10) if len(t) >= 2 else [t[0]] * 9
    return {"median_ms": round(statistics.median(t), 3), "p10_ms": round(q[0], 3), "p90_ms": round(q[-1], 3),
            "min_ms": round(t[0], 3), "max_ms": round(t[-1], 3), "reps": reps}


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    bls.Init(device=0)
    fresh = [0]
    def msg(state, tag):
        """cold: a message no call has hashed before; cached: one fixed message per tag, hashed by the warm-up"""
        if state == "cached": return wl.commit_payload(f"mk-hot-{tag}", 0)
        fresh[0] += 1
        return wl.commit_payload(f"mk-cold-{tag}", fresh[0])
    for k in (1, 4, 10, 32, 100):
        raw = [wl.sk_bytes(wl.seeded_sk("mk-time", i)) for i in range(k)]
        blob = b"".join(raw)
        keys = []
        for b in raw:
            s = bls.SecretKey(); s.Deserialize(b); keys.append(s)

        def ref_loop(m):                                    # (a)
            agg = bls.Sign()
            for s in keys:
                sig = s.SignHash(m)
                if sig is not None: agg.Add(sig)
            return agg.Serialize()

        def ref_view_change(m1, m2):                        # (d_ref)
            out = []
            for m in (m1, m2):
                for s in keys:
                    sig = s.SignHash(m)
                    out.append(sig.Serialize() if sig is not None else b"")
            return out

        check = wl.commit_payload("mk-check", k)
        assert bls.SignHashKeys(blob, check, 48, per_key=False)[1] == ref_loop(check), k
        m1, m2 = wl.commit_payload("mk-check-vc", k), wl.commit_payload("mk-check-vc", k + 1000)
        assert bls.SignHashKeys(blob, m1 + m2, 48, aggregate=False)[0] == b"".join(ref_view_change(m1, m2)), k
        # the reference loop runs k (2 k) device round trips per call: fewer repetitions at large k
        ref_reps = max(5, a.reps // (1 + k // 10))
        for state in ("cold", "cached"):
            for tag in ("a", "b", "c", "d0", "d1", "dref0", "dref1"):     # warm-up: modules loaded, the cached messages hashed
                m = msg("cached", tag) if state == "cached" else msg("cold", tag)
                bls.SignHashKeys(blob, m, 48)
            ref_loop(msg(state, "a"))
            emit(shape="a_ref_loop", k=k, hm=state, **stats(lambda i: ref_loop(msg(state, "a")), ref_reps))
            emit(shape="b_aggregate", k=k, hm=state, **stats(lambda i: bls.SignHashKeys(blob, msg(state, "b"), 48, per_key=False), a.reps))
            emit(shape="c_per_key_and_aggregate", k=k, hm=state, **stats(lambda i: bls.SignHashKeys(blob, msg(state, "c"), 48), a.reps))
            emit(shape="d_view_change_2msg", k=k, hm=state,
                 **stats(lambda i: bls.SignHashKeys(blob, msg(state, "d0") + msg(state, "d1"), 48, aggregate=False), a.reps))
            emit(shape="d_ref_view_change_2msg", k=k, hm=state,
                 **stats(lambda i: ref_view_change(msg(state, "dref0"), msg(state, "dref1")), max(3, ref_reps // 2)))


if __name__ == "__main__":
    main()
