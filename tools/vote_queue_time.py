"""tools/vote_queue_time.py -- one tick of a leader's vote collection on a 250-key committee: VoteCollector (device backend: key sums
through PublicKey.Add, hbls_verify_batch_status, hbls_aggregate_sigs) against BallotBoxCollector (one hbls_ballot_box_submit_votes,
then the box's aggregate), alternating in one process.

Timed: onVotes over the queue plus AggregateVotes, host clock around calls that end in a device synchronise.  Two queues: 250 one-key
votes, and 50 senders holding 4 keys each (+ 50 one-key votes); each with the H(m) cache cold (hm_cache off) and warm (the message
hashed before the tick, as a node that signed it has).  Prints one JSON line per case: median and spread (min, max) in ms of both,
their ratio, and the card's name and power limit.
Run:  python tools/vote_queue_time.py [--reps N]
"""
import argparse, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    a = ap.parse_args()
    from harmony_b200 import bls, consensus as cs, workload as wl
    bls.Init()
    n = 250
    sks = [wl.seeded_sk("vqt", i) for i in range(n)]
    blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    members = [blob[48 * i:48 * i + 48] for i in range(n)]
    message = wl.commit_payload("vqt", 0)
    groups = {"one_key_250": [[i] for i in range(n)],
              "multikey_50x4": [[4 * j + t for t in range(4)] for j in range(50)] + [[200 + i] for i in range(50)]}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    for name, idx in groups.items():
        sk_sum = [sum(sks[i] for i in g) % wl.R_ORDER for g in idx]
        sigs, ok = bls.SignHashBatch(b"".join(wl.sk_bytes(s) for s in sk_sum), message * len(idx), len(message))
        assert all(ok)
        votes = [cs.Vote([members[i] for i in g], sigs[96 * j:96 * j + 96]) for j, g in enumerate(idx)]
        for cache in ("cold", "warm"):
            bls.SetParam("hm_cache", 0 if cache == "cold" else 1)
            def tick(kind):
                col = (cs.VoteCollector if kind == "old" else cs.BallotBoxCollector)(members, message)
                if cache == "warm": bls.HashPrefetch(message)
                t0 = time.perf_counter()
                errs, _ = col.onVotes(votes)
                agg = col.AggregateVotes()
                dt = (time.perf_counter() - t0) * 1e3
                assert errs == [None] * len(votes)
                return dt, agg
            tick("old"); tick("new")                                      # warm-up: modules, scratch, committee paths
            t = {"old": [], "new": []}
            for _ in range(a.reps):
                for kind in ("old", "new"):
                    dt, agg = tick(kind); t[kind].append(dt); t[kind + "_agg"] = agg
            assert t["old_agg"] == t["new_agg"]
            med = {k: statistics.median(t[k]) for k in ("old", "new")}
            print(json.dumps({"case": name, "hm_cache": cache, "votes": len(votes), "reps": a.reps,
                              "vote_collector_ms": round(med["old"], 3), "vote_collector_range_ms": [round(min(t["old"]), 3), round(max(t["old"]), 3)],
                              "ballot_box_ms": round(med["new"], 3), "ballot_box_range_ms": [round(min(t["new"]), 3), round(max(t["new"]), 3)],
                              "ratio_old_over_new": round(med["old"] / med["new"], 2),
                              "gpu": smi[0] if smi else None, "power_limit_w": float(smi[1]) if len(smi) > 1 else None}), flush=True)
    bls.SetParam("hm_cache", 1)


if __name__ == "__main__":
    main()
