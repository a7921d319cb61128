"""Host cost of one GeneratorDevice.forward call at B = 1, T = 1, two ways, each repeated R times after a warm-up:
  - host wall clock over N back-to-back calls, ending in a synchronise (when the device takes longer per forward than
    the host, this is device time);
  - the host time of each of N calls made on an idle device (a synchronise before each), median over the calls: the
    Python and C work one call adds, launches included.

    python scripts/forward_host_time.py [--calls N] [--repeats R] [--root DIR]

--root: the tree whose melgan_multi_b200 is imported (default: this one), so two trees can be compared in one session.
Prints one JSON line: the card and microseconds per call of every repeat, and their medians."""
import argparse
import json
import os
import statistics
import sys
import time


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--calls", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from melgan_multi_b200 import models

    torch.manual_seed(0)
    dev = models.Generator().cuda()._ensure_packed()
    mel = torch.randn(1, 80, 1, device="cuda")
    out = torch.empty(1, 1, 256, device="cuda")
    for _ in range(200):
        dev.forward(mel, out)
    torch.cuda.synchronize()
    total, idle = [], []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        for _ in range(args.calls):
            dev.forward(mel, out)
        torch.cuda.synchronize()
        total.append((time.perf_counter() - t0) / args.calls * 1e6)
        one = []
        for _ in range(args.calls):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dev.forward(mel, out)
            one.append(time.perf_counter() - t0)
        idle.append(statistics.median(one) * 1e6)
    dev.check_status(1, 1)
    print(json.dumps({"root": os.path.abspath(args.root), "gpu": torch.cuda.get_device_name(), "calls": args.calls,
                      "us_per_call": [round(v, 3) for v in total], "median_us": round(statistics.median(total), 3),
                      "idle_host_us_per_call": [round(v, 3) for v in idle], "median_idle_host_us": round(statistics.median(idle), 3)}))


if __name__ == "__main__":
    main()
