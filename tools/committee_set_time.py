"""tools/committee_set_time.py -- the multi-committee batch from device memory in three forms, alternating in one process:
  items   hbls_aggregate_verify_items_device: a host list of k committee handles, descriptors built on the host and uploaded
  set     hbls_aggregate_verify_set_device called directly: an int32 index tensor, descriptors built on the device
  replay  the set call captured once into a CUDA graph (torch.cuda.CUDAGraph on the same static tensors), then g.replay()
Items: k = 4 (one item per shard of a 4-shard block seal), 1 024 and 16 384 over 4 committees of 250 slots, item j against committee
j mod 4, 167 / 200 / 250 signers, 4 payloads, the inputs already in HBM.  For each form: host enqueue time (the host clock around the
call / the replay, no synchronisation inside; for items it includes building the Python list of handles) and device time (CUDA
events recorded around it on the stream), median and range of --reps alternating repetitions after one warm-up of each; every output
is checked equal to the host form hbls_aggregate_verify_items.  Prints one JSON line per k with the card's name, power limit and
maximum SM clock read in the same run.
Run:  python tools/committee_set_time.py [--reps N] [--sizes 4,1024,16384]
"""
import argparse, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--sizes", default="4,1024,16384")
    a = ap.parse_args()
    import torch
    from harmony_b200 import bls, workload as wl
    bls.Init()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    dev = lambda b, w: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda().view(-1, w)
    n, m, pool = 250, 4, 64
    sks, coms = [], []
    for c in range(m):
        s = [wl.seeded_sk(f"cst-{c}", i) for i in range(n)]
        blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(x) for x in s))
        sks.append(s); coms.append(bls.Committee([blob[48 * i:48 * i + 48] for i in range(n)]))
    cset = bls.CommitteeSet(coms)
    bms = [wl.bitmap_with_k("cst", j, n, [167, 200, 250][j % 3]) for j in range(pool)]
    pays = [wl.commit_payload("cst", j % 4) for j in range(pool)]
    sigs, _ = bls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(sks[j % m], bms[j])) for j in range(pool)), b"".join(pays), 48)

    stream = torch.cuda.Stream()
    for k in [int(x) for x in a.sizes.split(",")]:
        src = [j % pool for j in range(k)]                     # pool is a multiple of m: item j's committee stays j mod m
        bm_blob = b"".join(bms[i] for i in src)
        sg_blob = b"".join(sigs[96 * i:96 * i + 96] for i in src)
        pay_blob = b"".join(pays[i] for i in src)
        want = bls.AggregateVerifyItems([coms[j % m] for j in range(k)], [bms[i] for i in src], sg_blob, pay_blob, 48)
        index = torch.tensor([j % m for j in range(k)], dtype=torch.int32, device="cuda")
        tbm, tsig, tpay = dev(bm_blob, 1).view(-1), dev(sg_blob, 96), dev(pay_blob, 48)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            graph_out = cset.AggregateVerifyDevice(index, tbm, tsig, tpay)
        calls = {"items": lambda: bls.AggregateVerifyItemsDevice([coms[j % m] for j in range(k)], tbm, tsig, tpay),
                 "set": lambda: cset.AggregateVerifyDevice(index, tbm, tsig, tpay),
                 "replay": lambda: (g.replay(), graph_out)[1]}

        def run(kind):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                e0.record(stream)
                t0 = time.perf_counter()
                out = calls[kind]()
                t1 = time.perf_counter()
                e1.record(stream)
            torch.cuda.synchronize()
            return (t1 - t0) * 1e3, e0.elapsed_time(e1), out.cpu().numpy().tobytes()

        for kind in calls:
            assert run(kind)[2] == want, (k, kind)
        t = {kind: ([], []) for kind in calls}
        for _ in range(a.reps):
            for kind in calls:
                host_ms, dev_ms, out = run(kind)
                assert out == want, (k, kind)
                t[kind][0].append(host_ms); t[kind][1].append(dev_ms)
        row = {"k": k, "committees": m, "slots": n, "reps": a.reps}
        for kind in calls:
            h, d = t[kind]
            row[kind + "_enqueue_ms"] = round(statistics.median(h), 4)
            row[kind + "_enqueue_range_ms"] = [round(min(h), 4), round(max(h), 4)]
            row[kind + "_device_ms"] = round(statistics.median(d), 4)
            row[kind + "_device_range_ms"] = [round(min(d), 4), round(max(d), 4)]
        row.update({"gpu": smi[0] if smi else None, "power_limit_w": float(smi[1]) if len(smi) > 1 else None,
                    "max_sm_clock_mhz": float(smi[2]) if len(smi) > 2 else None})
        print(json.dumps(row), flush=True)
        del g, graph_out


if __name__ == "__main__":
    main()
