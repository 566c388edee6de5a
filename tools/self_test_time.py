"""tools/self_test_time.py -- what the built-in self-test (hbls_self_test) costs on this GPU.

Prints one JSON line: the first run in the process (after blsInit), the median of the later runs, the device memory the runs
leave allocated (free memory before the first run minus after the last), the kernels launched, and the card's name and power limit.
Run:  python tools/self_test_time.py [--runs N]
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    a = ap.parse_args()
    import torch
    from harmony_b200 import bls
    bls.Init()
    torch.cuda.init()
    free0, _ = torch.cuda.mem_get_info()
    first = bls.SelfTest()
    later = [bls.SelfTest() for _ in range(a.runs)]
    free1, _ = torch.cuda.mem_get_info()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    print(json.dumps({
        "first_ms": round(first["ms"], 2),
        "median_ms": round(statistics.median(r["ms"] for r in later), 2),
        "runs": a.runs, "legs": first["legs"], "kernels": first["kernels"],
        "failed": sorted(set(first["failed"]).union(*(r["failed"] for r in later))),
        "reserved_bytes": int(free0 - free1),
        "gpu": smi[0] if smi else None, "power_limit_w": float(smi[1]) if len(smi) > 1 else None}))


if __name__ == "__main__":
    main()
