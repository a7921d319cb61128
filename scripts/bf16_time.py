"""fp32 against bf16 inference (Generator.generate(..., precision=...)) on the same weights and inputs, in one process:
  config2  B = 64, T = 32 (bench.py's workload)
  ragged   the 64 utterances of scripts/ragged_time.py (same seeds: lengths uniform in [86, 861] mel frames), one
           ragged forward
  config1  B = 1, T = 32
  config5  B = 1, T = 1000
Per workload, REPS rounds of one fp32 pass then one bf16 pass, each preceded by a write of 256 MB (L2 flushed) and
bracketed by CUDA events; median, min and max device time per precision.  Then one torch.profiler pass per precision at
config 2 for the per-kernel times, and the bf16 output's rel-L2 / SNR against the fp32 output of every workload.
Writes a JSON record with the card's name, power limit and SM clock cap (default profiles/h100_bf16.json)."""
import argparse
import json
import math
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth

REPS = 15
RAGGED_B, RAGGED_LO, RAGGED_HI, RAGGED_SEED = 64, 86, 861, 2024  # scripts/ragged_time.py


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def workloads():
    lens = [int(v) for v in np.random.default_rng(RAGGED_SEED).integers(RAGGED_LO, RAGGED_HI + 1, RAGGED_B)]
    mel = torch.zeros(RAGGED_B, 80, max(lens), device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, RAGGED_SEED + i)[0])
    return {
        "config2_B64_T32": (torch.from_numpy(synth.mel_input(64, 32, 0)).cuda(), None),
        "ragged_64_utterances": (mel, lens),
        "config1_B1_T32": (torch.from_numpy(synth.mel_input(1, 32, 0)).cuda(), None),
        "config5_B1_T1000": (torch.from_numpy(synth.mel_input(1, 1000, 0)).cuda(), None),
    }


def stats(v):
    return {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v)), "runs_ms": v}


def accuracy(y, ref, lens):
    """bf16 output against the fp32 output over the valid samples: rel-L2, SNR, max |d|."""
    if lens is not None:
        y = torch.cat([y[i, 0, :256 * L] for i, L in enumerate(lens)])
        ref = torch.cat([ref[i, 0, :256 * L] for i, L in enumerate(lens)])
    d = (y.double() - ref.double())
    rel = float(d.norm() / ref.double().norm())
    return {"rel_l2": rel, "snr_db": -20 * math.log10(rel), "max_abs": float(d.abs().max())}


def kernel_times(g, mel, precision):
    """{kernel name: device microseconds per forward} from one torch.profiler pass of 5 forwards."""
    from torch.profiler import ProfilerActivity, profile
    n = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            g.generate(mel, precision=precision)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0 and "memcpy" not in e.key.lower() and "memset" not in e.key.lower():
            out[e.key] = t / n
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_bf16.json")
    args = ap.parse_args()
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")  # 256 MB, five times the L2
    rec = {"card": card(), "reps": REPS, "workloads": {}}
    with torch.no_grad():
        for name, (mel, lens) in workloads().items():
            def run(p):
                return g.generate(mel, lens, precision=p)
            for p in ("fp32", "bf16"):  # warm the shapes and the workspace
                run(p)
            torch.cuda.synchronize()
            ms = {"fp32": [], "bf16": []}
            for _ in range(REPS):
                for p in ("fp32", "bf16"):
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    run(p)
                    b.record()
                    torch.cuda.synchronize()
                    ms[p].append(a.elapsed_time(b))
            y32, y16 = run("fp32"), run("bf16")
            g._dev.check_status(mel.shape[0], mel.shape[2])
            s32, s16 = stats(ms["fp32"]), stats(ms["bf16"])
            rec["workloads"][name] = {
                "shape": list(mel.shape), "frames": sum(lens) if lens else mel.shape[0] * mel.shape[2],
                "fp32": s32, "bf16": s16,
                "speedup": {"median": s32["median_ms"] / s16["median_ms"], "worst": s32["min_ms"] / s16["max_ms"],
                            "best": s32["max_ms"] / s16["min_ms"]},
                "bf16_vs_fp32": accuracy(y16, y32, lens),
            }
            print(name, json.dumps({k: v for k, v in rec["workloads"][name].items() if k not in ("fp32", "bf16")}), flush=True)
        mel = workloads()["config2_B64_T32"][0]
        rec["kernels_config2_us_per_forward"] = {p: kernel_times(g, mel, p) for p in ("fp32", "bf16")}
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
