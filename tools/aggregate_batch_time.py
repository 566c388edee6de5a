"""tools/aggregate_batch_time.py -- B AggregateSig calls of 1 000 signatures each (BASELINE configs[4]: rounds of a 1 000-validator
committee) as one hbls_aggregate_sigs_batch call against B hbls_aggregate_sigs calls, alternating in one process.

Host forms: the host clock around the whole call(s), signatures and offsets staged in host memory beforehand (the batch: one call;
the singles: B calls, one per set).  Device form: hbls_aggregate_sigs_batch_device on a torch stream with the inputs already in HBM,
timed with CUDA events recorded around it.  Median and range of --reps alternating repetitions after one warm-up of each; every form's
bytes are checked against the singles.  Prints one JSON line per B with the card's name, power limit and maximum SM clock read in the
same run.
Run:  python tools/aggregate_batch_time.py [--reps N] [--sizes 64,256,1024] [--set 1000]
"""
import argparse, ctypes, json, os, statistics, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="64,256,1024")
    ap.add_argument("--set", type=int, default=1000)
    a = ap.parse_args()
    import torch
    from harmony_b200 import bls, workload as wl
    bls.Init()
    L = bls.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    m = a.set
    sks = b"".join(wl.sk_bytes(wl.seeded_sk("abt", i)) for i in range(m))
    pool, ok = bls.SignHashBatch(sks, wl.commit_payload("abt", 0) * m, 48)       # the committee's votes on one round's payload
    assert ok == b"\x01" * m
    stream = torch.cuda.Stream()
    for B in [int(x) for x in a.sizes.split(",")]:
        blobs = [pool[96 * (j % m):] + pool[:96 * (j % m)] for j in range(B)]      # round j: the votes rotated by j
        blob = b"".join(blobs)
        offsets = (ctypes.c_uint64 * (B + 1))(*[m * j for j in range(B + 1)])
        out_b = ctypes.create_string_buffer(96 * B); st_b = ctypes.create_string_buffer(B)
        out_s = ctypes.create_string_buffer(96 * B)
        d_off = torch.tensor([m * j for j in range(B + 1)], dtype=torch.int64, device="cuda")
        d_sig = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda().view(-1, 96)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def batch():
            t = time.perf_counter()
            assert L.hbls_aggregate_sigs_batch(B, offsets, blob, out_b, st_b) == 0
            return (time.perf_counter() - t) * 1e3

        def singles():
            t = time.perf_counter()
            for j in range(B):
                assert L.hbls_aggregate_sigs(blobs[j], m, ctypes.addressof(out_s) + 96 * j) == 0
            return (time.perf_counter() - t) * 1e3

        def device():
            with torch.cuda.stream(stream):
                e0.record(stream)
                res = bls.AggregateSigsBatchDevice(d_off, d_sig, stream=stream)
                e1.record(stream)
            e1.synchronize()
            device.res = res
            return e0.elapsed_time(e1)

        t = {"batch": [], "singles": [], "device": []}
        for r in range(a.reps + 1):
            for name, f in (("batch", batch), ("singles", singles), ("device", device)):
                v = f()
                if r: t[name].append(v)
        dev_out = device.res[0].cpu().numpy().tobytes(); dev_st = device.res[1].cpu().numpy().tobytes()
        assert out_b.raw == out_s.raw == dev_out and st_b.raw == dev_st == bytes([bls.AGG_OK]) * B
        med = {k: statistics.median(v) for k, v in t.items()}
        print(json.dumps({"B": B, "set": m, "gpu": smi[0], "power_limit_w": float(smi[1]), "max_sm_clock_mhz": float(smi[2]),
                          "reps": a.reps,
                          **{f"{k}_ms": round(med[k], 3) for k in t}, **{f"{k}_ms_range": [round(min(v), 3), round(max(v), 3)] for k, v in t.items()},
                          "singles_over_batch": round(med["singles"] / med["batch"], 2),
                          "signatures_per_s_device": round(B * m / (med["device"] * 1e-3))}), flush=True)


if __name__ == "__main__":
    main()
