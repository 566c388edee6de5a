"""tools/kernel_times.py -- device time of every kernel of one benchmark-size step, from torch.profiler's CUDA activities.

    python tools/kernel_times.py [--rounds 270336] [--steps 2] [--out DIR] [--label NAME]

Builds the benchmark's inputs (bench.make_rounds, seed 2024, the 250-key committee), runs one warm-up step, then profiles
`--steps` device-resident steps (hbls_aggregate_verify_batch_device, the call bench.py times) and writes DIR/kernel_times_<label>.json:
per kernel name the number of launches and the total / per-step device time in ms, with the card name, power limit and the SM
clock read at the end of the run.  The profiler slows the host side only; the per-kernel device times are what the kernels took.
"""
import argparse, json, os, subprocess, sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=270336)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default=".", help="directory for kernel_times_<label>.json (default: the current directory)")
    ap.add_argument("--label", default="current")
    args = ap.parse_args()

    import torch
    from torch.profiler import profile, ProfilerActivity
    if not torch.cuda.is_available():
        raise SystemExit("kernel_times.py: no CUDA device")
    import bench
    from harmony_b200 import bls, workload as wl

    bls.Init(device=0)
    L = bls.lib()
    B = args.rounds
    sks = bench.make_committee_sks()
    pks_blob = bls.GetPublicKeyBatch(b"".join(wl.sk_bytes(k) for k in sks))
    com = bls.Committee([pks_blob[48 * i:48 * i + 48] for i in range(bench.N_COMMITTEE)])
    bitmaps, agg_sk, msgs, nsig = bench.make_rounds(sks, B, seed=2024)
    sigs, ok = bls.SignHashBatch(agg_sk, msgs, bench.MSG_LEN)
    assert ok == b"\x01" * B
    dev = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
    d_bm, d_sig, d_msg = dev(bitmaps), dev(sigs), dev(msgs)
    d_res = torch.zeros(B, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    blen = (bench.N_COMMITTEE + 7) // 8

    def step():
        rc = L.hbls_aggregate_verify_batch_device(com.h, B, d_bm.data_ptr(), blen, d_sig.data_ptr(), d_msg.data_ptr(), bench.MSG_LEN,
                                                  d_res.data_ptr(), stream.cuda_stream)
        assert rc == 0, rc

    step(); torch.cuda.synchronize()
    assert int(d_res.sum().item()) == B
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    assert int(d_res.sum().item()) == B

    calls, us = defaultdict(int), defaultdict(float)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in ev.name.lower() and "memset" not in ev.name.lower():
            name = ev.name.split("(")[0].replace("void ", "").replace("hb::", "").replace("(anonymous namespace)::", "")
            calls[name] += 1; us[name] += ev.device_time_total
    total = sum(us.values())
    kernels = {n: {"launches_per_step": calls[n] / args.steps, "ms_per_step": us[n] / args.steps / 1e3, "share": us[n] / total}
               for n in sorted(us, key=lambda k: -us[k])}
    res = {"label": args.label, "rounds": B, "steps": args.steps, "sigs_per_step": nsig, "gpu": gpu_info(),
           "kernel_ms_per_step_total": total / args.steps / 1e3, "kernels": kernels}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"kernel_times_{args.label}.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    for n, k in kernels.items():
        print(f"{k['ms_per_step']:9.3f} ms  {k['launches_per_step']:5.1f}x  {n}")
    print(f"{res['kernel_ms_per_step_total']:9.3f} ms  total kernel time per step -> {path}")


if __name__ == "__main__":
    main()
