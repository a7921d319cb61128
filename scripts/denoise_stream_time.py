"""Streaming denoising of 64 live sessions (the seeded utterance lengths of scripts/ragged_time.py and scripts/stream_time.py,
uniform in [86, 861] mel frames), every session pushing n = 4, 8 or 16 frames per step (the last push carries END), at
n_fft 1024, hop 256, win_length 1024, served three ways on the same weights:
  gen       Generator.stream alone (no denoiser)
  gen+dn    Generator.stream chained into Denoiser.stream: each step's audio and counts go straight to the denoiser step
  whole     one ragged generate of the whole utterances followed by one Denoiser.forward (the floor: no streaming)
Per arm and n: total device time of the schedule (CUDA events, no synchronisation inside), median (min - max) over REPS
alternated passes, and per-step latency from call to audio ready (host clock around step + synchronise), median and p95.
A separate torch.profiler run of gen+dn at each n splits the device time between the generator stream's kernels and the
denoiser stream's three kernels.  Every arm's audio is compared with the whole arm's (torch.equal on the float bits).
Writes a JSON record with the card's name, power limit and clock cap."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import denoiser, engine, models, synth

B, LO, HI, SEED, REPS = 64, 86, 861, 2024, 5
PUSH = (4, 8, 16)
N_FFT, HOP, WIN = 1024, 256, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def schedule(mel, lens, n):
    """Per step: (packed mel [S, 80, n], frames, flags) for sessions pushing n frames per step."""
    S = len(lens)
    steps = []
    for s in range((max(lens) + n - 1) // n):
        m = torch.zeros((S, 80, n), device="cuda")
        frames, flags = [], []
        for i, L in enumerate(lens):
            a, b = min(L, s * n), min(L, (s + 1) * n)
            m[i, :, :b - a] = mel[i, :, a:b]
            frames.append(b - a)
            flags.append(engine.STREAM_END if a < L and b == L else 0)
        steps.append((m, frames, flags))
    return steps


def run(gen, dn, steps, n, denoise, keep=False, lat=None):
    gs = gen.stream(B, n)
    ds = dn.stream(B, gs.max_out) if denoise else None
    outs = [[] for _ in range(B)] if keep else None
    for m, frames, flags in steps:
        if lat is not None:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        a, c = gs.step_packed(m, frames, flags)
        if denoise:
            a, c = ds.step_packed(a, c, flags)
        if lat is not None:
            torch.cuda.synchronize()
            lat.append(1e3 * (time.perf_counter() - t0))
        if keep:
            for i, k in enumerate(c):
                outs[i].append(a[i, :k])
    return outs


def whole(gen, dn, mel, lens, denoise=True):
    y = gen.generate(mel, lens)
    return dn(y, lengths=[256 * L for L in lens]) if denoise else y


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def summary(v):
    return {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)), "runs": [float(x) for x in v]}


def stats(v):
    return {"median_ms": float(np.median(v)), "p95_ms": float(np.percentile(v, 95)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_denoise_stream.json")
    args = ap.parse_args()
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    dn = denoiser.Denoiser(g, N_FFT, N_FFT // HOP, WIN)
    lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B)]
    T = max(lens)
    mel = torch.zeros(B, 80, T, device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    rec = {"card": card(), "analysis": {"n_fft": N_FFT, "hop": HOP, "win_length": WIN, "strength": 0.1},
           "workload": {"sessions": B, "frames": sum(lens), "lengths_uniform_in": [LO, HI], "seed": SEED,
                        "audio_seconds": sum(lens) * 256 / 22050.0}, "push": {}}
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        ref_gen = whole(g, dn, mel, lens, denoise=False)
        ref = whole(g, dn, mel, lens)
        bits = lambda x: x.contiguous().view(torch.int32)
        for n in PUSH:
            steps = schedule(mel, lens, n)
            for denoise, r in ((False, ref_gen), (True, ref)):
                outs = run(g, dn, steps, n, denoise, keep=True)
                for i, L in enumerate(lens):
                    assert torch.equal(bits(torch.cat(outs[i])), bits(r[i, 0, :256 * L])), (n, denoise, i)
            tot = {"gen": [], "gen+dn": [], "whole": []}
            for _ in range(REPS):  # alternated
                tot["gen"].append(timed(lambda: run(g, dn, steps, n, False)))
                tot["gen+dn"].append(timed(lambda: run(g, dn, steps, n, True)))
                tot["whole"].append(timed(lambda: whole(g, dn, mel, lens)))
            lat_g, lat_d = [], []
            run(g, dn, steps, n, False, lat=lat_g)
            run(g, dn, steps, n, True, lat=lat_d)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(g, dn, steps, n, True)
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                if t:
                    per[e.key] = per.get(e.key, 0.0) + t / 1e3
            dn_ms = sum(v for k, v in per.items() if "denoise_stream" in k)
            dn_calls = sum(e.count for e in prof.key_averages() if "denoise_stream" in e.key)
            rec["push"][str(n)] = {
                "steps": len(steps), "total": {k: summary(v) for k, v in tot.items()},
                "step_latency": {"gen": stats(lat_g), "gen+dn": stats(lat_d)},
                "profiler": {"denoise_stream_ms": dn_ms, "denoise_stream_ms_per_step": dn_ms / len(steps),
                             "denoise_stream_launches": int(dn_calls),
                             "kernels_ms": {k: v for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:16]}},
                "bit_identical_to_whole": True}
            print(n, json.dumps(rec["push"][str(n)]["total"]["gen+dn"]["median_ms"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps({k: v for k, v in rec.items() if k != "push"}))
    for n, r in rec["push"].items():
        print(n, {k: round(v["median_ms"], 3) for k, v in r["total"].items()}, "step", {k: round(v["median_ms"], 3) for k, v in
              r["step_latency"].items()}, "dn/step %.4f ms" % r["profiler"]["denoise_stream_ms_per_step"])


if __name__ == "__main__":
    main()
