"""tools/graph_replay_time.py -- a direct device-form call against a replay of the same call captured once into a CUDA graph,
alternating in one process.

Forms: triples (hbls_verify_batch_status_device, one message per 37 triples) and headers (hbls_verify_headers_device against one
250-slot committee, 5 payloads), at k = 1, 64, 500, 5 000 and 20 000 items, the inputs already in HBM.  Direct: the call on a torch
stream.  Replay: torch.cuda.CUDAGraph captured once on the same static tensors, then g.replay().  For each: host enqueue time (the
host clock around the call / the replay, no synchronisation inside) and device time (CUDA events recorded around it on the stream),
median and range of --reps alternating repetitions after one warm-up of each; both outputs are checked equal to the host form.
Prints one JSON line per (form, k) with the card's name, power limit and maximum SM clock read in the same run.
Run:  python tools/graph_replay_time.py [--reps N] [--sizes 1,64,...]
"""
import argparse, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--sizes", default="1,64,500,5000,20000")
    a = ap.parse_args()
    import torch
    from harmony_b200 import bls, workload as wl
    bls.Init()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    dev = lambda b, w: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda().view(-1, w)
    sizes = [int(x) for x in a.sizes.split(",")]
    kmax = max(sizes)

    pool = 256
    tsk = b"".join(wl.sk_bytes(wl.seeded_sk("grt", i % 64)) for i in range(pool))
    tmsg = b"".join(wl.seeded_bytes("grt/m", i % 37, 32) for i in range(pool))
    tpk = bls.GetPublicKeyBatch(tsk); tsig, _ = bls.SignHashBatch(tsk, tmsg, 32)
    n = 250
    csk = [wl.seeded_sk("grt-c", i) for i in range(n)]
    blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(s) for s in csk))
    com = bls.Committee([blob[48 * i:48 * i + 48] for i in range(n)])
    hbm = [wl.bitmap_with_k("grt-h", j, n, [167, 200, 250][j % 3]) for j in range(pool)]
    hpay = [wl.commit_payload("grt-h", j % 5) for j in range(pool)]
    hsig, _ = bls.SignHashBatch(b"".join(wl.sk_bytes(wl.round_signer_sum(csk, b)) for b in hbm), b"".join(hpay), 48)
    q = wl.quorum_k(n)
    rep = lambda blob_, w, k: b"".join(blob_[w * (i % pool):w * (i % pool) + w] for i in range(k))

    stream = torch.cuda.Stream()
    for form in ("triples", "headers"):
        for k in sizes:
            if form == "triples":
                arrays = (rep(tpk, 48, k), rep(tsig, 96, k), rep(tmsg, 32, k))
                static = [dev(arrays[0], 48), dev(arrays[1], 96), dev(arrays[2], 32)]
                call = lambda t: bls.VerifyBatchStatusDevice(t[0], t[1], t[2])
                want = bls.VerifyBatchStatus(arrays[0], arrays[1], arrays[2], 32)
            else:
                arrays = (rep(hsig, 96, k), rep(b"".join(hbm), 32, k), rep(b"".join(hpay), 48, k))
                static = [dev(arrays[0], 96), dev(arrays[1], 32), dev(arrays[2], 48)]
                call = lambda t: com.VerifyHeadersDevice(t[0], t[1], t[2], q)
                want = com.VerifyHeaders(arrays[0], arrays[1], arrays[2], 48, q)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                graph_out = call(static)

            def run(kind):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(stream):
                    e0.record(stream)
                    t0 = time.perf_counter()
                    out = call(static) if kind == "direct" else (g.replay(), graph_out)[1]
                    t1 = time.perf_counter()
                    e1.record(stream)
                torch.cuda.synchronize()
                return (t1 - t0) * 1e3, e0.elapsed_time(e1), out.cpu().numpy().tobytes()

            for kind in ("direct", "replay"):
                assert run(kind)[2] == want, (form, k, kind)
            t = {"direct": ([], []), "replay": ([], [])}
            for _ in range(a.reps):
                for kind in ("direct", "replay"):
                    host_ms, dev_ms, out = run(kind)
                    assert out == want, (form, k, kind)
                    t[kind][0].append(host_ms); t[kind][1].append(dev_ms)
            row = {"form": form, "k": k, "reps": a.reps}
            for kind in ("direct", "replay"):
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
