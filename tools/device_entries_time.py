"""tools/device_entries_time.py -- host forms of the batch verifiers against their device forms, alternating in one process.

Host form: host bytes in, statuses copied back to the host (hbls_verify_batch_status / hbls_aggregate_verify_items / hbls_verify_headers).
Device form: the same inputs already in HBM as uint8 CUDA tensors, statuses in HBM (the *_device entry points), timed up to a
torch.cuda.synchronize() after the call plus the copy of the statuses back for the comparison.  Host clock around each call; median and range of --reps calls after a warm-up call of
each.  The H(m) cache is off (hm_cache 0) for both, so the host forms do not reuse the previous repetition's H(m).
Cases: 10 000 triples with 1 % invalid (BASELINE configs[3]), 500 view-change-shaped triples over 3 messages, 4 x 250 items
(4 committees of 250, one message each), a 4 096-header range of one committee.  Prints one JSON line per case with the card's name,
power limit and maximum SM clock.
Run:  python tools/device_entries_time.py [--reps N]
"""
import argparse, json, os, random, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    a = ap.parse_args()
    import torch
    from harmony_b200 import bls, workload as wl
    bls.Init()
    dev = lambda b, w: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda().view(-1, w)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")

    def triples(tag, k, nmsg, nbad):
        sks = b"".join(wl.sk_bytes(wl.seeded_sk(tag, i)) for i in range(k))
        msgs = b"".join(wl.seeded_bytes(tag + "/m", i % nmsg, 32) for i in range(k))
        pks = bytearray(bls.GetPublicKeyBatch(sks)); sigs, _ = bls.SignHashBatch(sks, msgs, 32); sigs = bytearray(sigs)
        for t, i in enumerate(random.Random(tag).sample(range(k), nbad)):
            if t % 2: sigs[96 * i + 11] ^= 1
            else: pks[48 * i:48 * i + 48] = b"\xff" * 48
        return bytes(pks), bytes(sigs), msgs

    def committee(tag, n):
        sks = [wl.seeded_sk(tag, i) for i in range(n)]
        blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(s) for s in sks))
        return sks, bls.Committee([blob[48 * i:48 * i + 48] for i in range(n)])

    cases = []
    p, s, m = triples("det-c4", 10000, 10000, 100)
    tp, ts, tm = dev(p, 48), dev(s, 96), dev(m, 32)
    cases.append(("triples_10000_1pct_invalid", lambda: bls.VerifyBatchStatus(p, s, m, 32), lambda: bls.VerifyBatchStatusDevice(tp, ts, tm)))
    p2, s2, m2 = triples("det-vc", 500, 3, 5)
    tp2, ts2, tm2 = dev(p2, 48), dev(s2, 96), dev(m2, 32)
    cases.append(("view_change_500_over_3_messages", lambda: bls.VerifyBatchStatus(p2, s2, m2, 32), lambda: bls.VerifyBatchStatusDevice(tp2, ts2, tm2)))
    coms, bms, isigs, imsgs = [], [], [], []
    for sh in range(4):
        sks, com = committee(f"det-i{sh}", 250); coms.append(com)
        shard_bms = [wl.bitmap_with_k(f"det-i{sh}", j, 250, 167 + j % 80) for j in range(250)]
        msg = wl.commit_payload(f"det-i{sh}", 0)
        sg, _ = bls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, bm)) for bm in shard_bms), msg * 250, 48)
        bms += shard_bms; isigs.append(sg); imsgs.append(msg * 250)
    items = [coms[j // 250] for j in range(1000)]
    isig, imsg = b"".join(isigs), b"".join(imsgs)
    tb, tis, tim = dev(b"".join(bms), 32), dev(isig, 96), dev(imsg, 48)
    cases.append(("items_4x250", lambda: bls.AggregateVerifyItems(items, bms, isig, imsg, 48), lambda: bls.AggregateVerifyItemsDevice(items, tb, tis, tim)))
    sks, com = committee("det-h", 250)
    N = 4096
    hbms = [wl.bitmap_with_k("det-h", j, 250, [167, 200, 250][j % 3]) for j in range(N)]
    hpay = [wl.commit_payload("det-h", j) for j in range(N)]
    hsig, _ = bls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks, bm)) for bm in hbms), b"".join(hpay), 48)
    hb, hp = b"".join(hbms), b"".join(hpay)
    q = wl.quorum_k(250)
    thb, ths, thp = dev(hb, 32), dev(hsig, 96), dev(hp, 48)
    cases.append(("headers_4096", lambda: com.VerifyHeaders(hsig, hb, hp, 48, q), lambda: com.VerifyHeadersDevice(ths, thb, thp, q)))

    old_cache = bls.GetParam("hm_cache")
    bls.SetParam("hm_cache", 0)
    try:
        for name, host, device in cases:
            def run(kind):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if kind == "host": out = host()
                else: out = device(); torch.cuda.synchronize(); out = out.cpu().numpy().tobytes()
                return (time.perf_counter() - t0) * 1e3, out
            _, want = run("host"); _, got = run("device")
            assert got == want, name
            t = {"host": [], "device": []}
            for _ in range(a.reps):
                for kind in ("host", "device"):
                    dt, out = run(kind); t[kind].append(dt)
                    assert out == want, (name, kind)
            med = {k: statistics.median(v) for k, v in t.items()}
            print(json.dumps({"case": name, "items": len(want), "reps": a.reps,
                              "host_form_ms": round(med["host"], 3), "host_form_range_ms": [round(min(t["host"]), 3), round(max(t["host"]), 3)],
                              "device_form_ms": round(med["device"], 3), "device_form_range_ms": [round(min(t["device"]), 3), round(max(t["device"]), 3)],
                              "ratio_host_over_device": round(med["host"] / med["device"], 2),
                              "gpu": smi[0] if smi else None, "power_limit_w": float(smi[1]) if len(smi) > 1 else None,
                              "max_sm_clock_mhz": float(smi[2]) if len(smi) > 2 else None}), flush=True)
    finally:
        bls.SetParam("hm_cache", old_cache)


if __name__ == "__main__":
    main()
