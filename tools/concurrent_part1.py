"""tools/concurrent_part1.py -- herumi-API calls (include/hbls.h part 1) from many threads at once.

For 1, 8 and 64 threads, each thread loops for a fixed time over its own share of distinct struct triples and calls
blsVerifyHash (about 1 % of the triples carry a wrong message; every boolean is checked against the expected value), then
blsSignHash.  Reports calls per second and the turns the library combined the calls into (hbls_coalesce_stats: mean turn size,
time per turn; max_turn is the largest turn so far in the process), with the card name and power limit, as one JSON line.

  python tools/concurrent_part1.py [--seconds S] [--triples N] [--threads 1,8,64]
"""
import argparse, json, os, subprocess, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from harmony_b200 import bls, workload as wl

MSG_LEN = 48

def card(device=0):
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception:
        return None, None

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0, help="length of each timed leg")
    ap.add_argument("--triples", type=int, default=1024, help="distinct (key, message, signature) triples")
    ap.add_argument("--threads", default="1,8,64")
    args = ap.parse_args()
    n, threads = args.triples, [int(x) for x in args.threads.split(",")]
    bls.Init(device=0)
    keys = [wl.sk_bytes(wl.seeded_sk("part1", i)) for i in range(n)]
    msgs = [wl.seeded_bytes("part1/m", i, MSG_LEN) for i in range(n)]
    pk48 = bls.GetPublicKeyBatch(b"".join(keys))
    sig96, ok = bls.SignHashBatch(b"".join(keys), b"".join(msgs), MSG_LEN)
    assert ok == b"\x01" * n
    want = [i % 100 != 37 for i in range(n)]
    vmsgs = [m if w else bytes([m[0] ^ 1]) + m[1:] for m, w in zip(msgs, want)]
    sks, pks, sigs = [None] * n, [None] * n, [None] * n
    def load(t, T):
        for i in range(t, n, T):
            sks[i] = bls.SecretKey(); sks[i].Deserialize(keys[i])
            pks[i] = bls.PublicKey(); pks[i].Deserialize(pk48[48 * i:48 * i + 48])
            sigs[i] = bls.Sign(); sigs[i].Deserialize(sig96[96 * i:96 * i + 96])
    th = [threading.Thread(target=load, args=(t, 64)) for t in range(64)]
    for x in th: x.start()
    for x in th: x.join()

    def run(T, body):
        done, bad = [0] * T, [0] * T
        stop = time.perf_counter() + args.seconds
        def worker(t):
            k = 0
            while True:
                i = t + T * (k % (n // T)); k += 1
                if not body(i): bad[t] += 1
                done[t] += 1
                if time.perf_counter() >= stop: break
        s0 = bls.CoalesceStats(); t0 = time.perf_counter()
        ths = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
        for x in ths: x.start()
        for x in ths: x.join()
        el = time.perf_counter() - t0; s1 = bls.CoalesceStats()
        assert sum(bad) == 0, f"{sum(bad)} wrong results with {T} threads"
        turns, reqs = s1["turns"] - s0["turns"], s1["requests"] - s0["requests"]
        return {"per_s": sum(done) / el, "calls": sum(done), "turns": turns, "mean_turn": reqs / turns if turns else None,
                "max_turn_so_far": s1["max_turn"], "ms_per_turn": el * 1e3 / turns if turns else None}

    verify = lambda i: sigs[i].VerifyHash(pks[i], vmsgs[i]) == want[i]
    sign = lambda i: sks[i].SignHash(msgs[i]) is not None
    out = {"metric": "concurrent herumi-API calls", "api": "blsVerifyHash / blsSignHash on struct triples (ctypes, GIL released per call)",
           "distinct_triples": n, "invalid_triples": n - sum(want), "seconds_per_leg": args.seconds, "verify_hash": {}, "sign_hash": {}}
    for T in threads:
        out["verify_hash"][str(T)] = run(T, verify)
        out["sign_hash"][str(T)] = run(T, sign)
    if len(threads) > 1:
        lo, hi = str(min(threads)), str(max(threads))
        out[f"verify_speedup_{hi}_vs_{lo}"] = out["verify_hash"][hi]["per_s"] / out["verify_hash"][lo]["per_s"]
    out["card"], out["power_limit"] = card()
    print(json.dumps(out), flush=True)

if __name__ == "__main__":
    main()
