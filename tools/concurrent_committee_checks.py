"""tools/concurrent_committee_checks.py -- single committee checks from many threads at once.

hbls_aggregate_verify (Committee.AggregateVerify) and hbls_mask_verify (DeviceMask.VerifyHash) join the turns of the herumi-API
combiner (include/hbls.h: threading).  For 1, 8 and 64 threads, each thread loops for a fixed time over its share of distinct
250-key rounds (10 of them carry a wrong message; every boolean is checked against the expected value) and reports checks per
second and the turns the library combined them into (hbls_coalesce_stats: mean turn size, time per turn).  The mask leg checks the
same rounds against one resident mask per round.

--lone-lib PATH (repeatable, e.g. this build and the parent's libhbls.so): the latency of a lone hbls_aggregate_verify and
hbls_mask_verify with the H(m) cache off, median over --lone-calls calls per build, the builds alternating in blocks (each block a
fresh process with HBLS_LIB set).  The card name and power limit are read in the same run.  One JSON line.

  python tools/concurrent_committee_checks.py [--seconds S] [--rounds N] [--threads 1,8,64] [--lone-lib PATH ...]
"""
import argparse, json, os, statistics, subprocess, sys, threading, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_KEYS, MSG_LEN, N_BAD = 250, 48, 10


def card(device=0):
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip().split(", ")
        return q[0], q[1]
    except Exception:
        return None, None


def make_rounds(bls, wl, n):
    sks = [wl.seeded_sk("ccchk", i) for i in range(N_KEYS)]
    blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    com = bls.Committee([blob[48 * i:48 * i + 48] for i in range(N_KEYS)])
    bms = [wl.bitmap_with_k("ccchk", j, N_KEYS, wl.quorum_k(N_KEYS) + j % 40) for j in range(n)]
    msgs = [wl.seeded_bytes("ccchk/m", j, MSG_LEN) for j in range(n)]
    sig96, ok = bls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, bm)) for bm in bms), b"".join(msgs), MSG_LEN)
    assert ok == b"\x01" * n
    sigs = [sig96[96 * j:96 * j + 96] for j in range(n)]
    bad = set(range(37, n, max(1, n // N_BAD))[:N_BAD])
    vmsgs = [bytes([m[0] ^ 1]) + m[1:] if j in bad else m for j, m in enumerate(msgs)]
    return com, bms, sigs, vmsgs, [j not in bad for j in range(n)]


def lone_block(calls):
    """one block of lone calls in this process (the build HBLS_LIB names): per-call milliseconds of both entry points"""
    from harmony_b200 import bls, workload as wl
    bls.Init(device=0)
    com, bms, sigs, vmsgs, want = make_rounds(bls, wl, 8)
    mask = bls.DeviceMask(com); mask.SetMask(bms[0])
    bls.SetParam("hm_cache", 0)
    for _ in range(5): com.AggregateVerify(bms[0], sigs[0], vmsgs[0]); mask.VerifyHash(sigs[0], vmsgs[0])       # warm-up
    out = {"agg": [], "mask": []}
    for i in range(calls):
        t0 = time.perf_counter(); r = com.AggregateVerify(bms[0], sigs[0], vmsgs[0]); out["agg"].append((time.perf_counter() - t0) * 1e3)
        assert r is want[0]
        t0 = time.perf_counter(); r = mask.VerifyHash(sigs[0], vmsgs[0]); out["mask"].append((time.perf_counter() - t0) * 1e3)
        assert r is want[0]
    print("LONE " + json.dumps(out), flush=True)


def lone_latency(libs, calls, blocks=4):
    per = {p: {"agg": [], "mask": []} for p in libs}
    for b in range(blocks):
        for p in libs:
            env = {**os.environ, "HBLS_LIB": os.path.abspath(p)}
            r = subprocess.run([sys.executable, __file__, "--lone-block", str(max(1, calls // blocks))], capture_output=True, text=True,
                               timeout=600, env=env)
            line = [l for l in r.stdout.splitlines() if l.startswith("LONE ")]
            if r.returncode != 0 or not line: raise RuntimeError(f"lone block with {p} failed: {r.stderr[-2000:]}")
            got = json.loads(line[0][5:])
            for k in per[p]: per[p][k] += got[k]
    return {p: {k: {"median_ms": statistics.median(v), "p10_ms": sorted(v)[len(v) // 10], "p90_ms": sorted(v)[(9 * len(v)) // 10], "calls": len(v)}
                for k, v in d.items()} for p, d in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0, help="length of each timed leg")
    ap.add_argument("--rounds", type=int, default=1024, help="distinct 250-key rounds")
    ap.add_argument("--threads", default="1,8,64")
    ap.add_argument("--lone-lib", action="append", default=[], help="libhbls.so builds to time lone calls of (alternating)")
    ap.add_argument("--lone-calls", type=int, default=120)
    ap.add_argument("--lone-block", type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.lone_block:
        return lone_block(args.lone_block)
    from harmony_b200 import bls, workload as wl
    n, threads = args.rounds, [int(x) for x in args.threads.split(",")]
    bls.Init(device=0)
    com, bms, sigs, vmsgs, want = make_rounds(bls, wl, n)
    masks = []
    for j in range(n):
        m = bls.DeviceMask(com); m.SetMask(bms[j]); masks.append(m)

    def run(T, body):
        done, bad = [0] * T, [0] * T
        stop = time.perf_counter() + args.seconds
        def worker(t):
            k = 0
            while True:
                i = t + T * (k % (n // T)); k += 1
                if body(i) != want[i]: bad[t] += 1
                done[t] += 1
                if time.perf_counter() >= stop: break
        s0 = bls.CoalesceStats(); t0 = time.perf_counter()
        ths = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
        for x in ths: x.start()
        for x in ths: x.join()
        el = time.perf_counter() - t0; s1 = bls.CoalesceStats()
        assert sum(bad) == 0, f"{sum(bad)} wrong results with {T} threads"
        turns, reqs = s1["turns"] - s0["turns"], s1["requests"] - s0["requests"]
        return {"per_s": sum(done) / el, "checks": sum(done), "turns": turns, "mean_turn": reqs / turns if turns else None,
                "max_turn_so_far": s1["max_turn"], "ms_per_turn": el * 1e3 / turns if turns else None}

    agg = lambda i: com.AggregateVerify(bms[i], sigs[i], vmsgs[i])
    mask = lambda i: masks[i].VerifyHash(sigs[i], vmsgs[i])
    for i in range(min(n, 64)): agg(i); mask(i)                                              # warm-up
    out = {"metric": "concurrent committee checks", "api": "hbls_aggregate_verify / hbls_mask_verify (ctypes, GIL released per call)",
           "committee_keys": N_KEYS, "distinct_rounds": n, "invalid_rounds": n - sum(want), "seconds_per_leg": args.seconds,
           "hm_cache": bls.GetParam("hm_cache"), "aggregate_verify": {}, "mask_verify": {}}
    for T in threads:
        out["aggregate_verify"][str(T)] = run(T, agg)
        out["mask_verify"][str(T)] = run(T, mask)
    if len(threads) > 1:
        lo, hi = str(min(threads)), str(max(threads))
        out[f"aggregate_verify_speedup_{hi}_vs_{lo}"] = out["aggregate_verify"][hi]["per_s"] / out["aggregate_verify"][lo]["per_s"]
        out[f"mask_verify_speedup_{hi}_vs_{lo}"] = out["mask_verify"][hi]["per_s"] / out["mask_verify"][lo]["per_s"]
    if args.lone_lib:
        out["lone_latency_hm_cache_off"] = lone_latency(args.lone_lib, args.lone_calls)
    out["card"], out["power_limit"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
