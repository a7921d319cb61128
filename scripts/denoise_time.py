"""Denoising vocoded audio (denoiser.Denoiser, WaveGlow's analysis: n_fft 1024, hop 256, window 1024) on four workloads:
  config2   64 x 8192 samples (bench.py config 2's audio)
  ragged    the 64 seeded utterances of scripts/ragged_time.py, each with its own length
  voices    16 voices x 4 of those utterances (one bias row per voice)
  long      B = 1 x 10 s (220 500 samples)
and these arms, on the same inputs:
  kernels        Denoiser eager, fp32 out          kernels_pcm16  the same, int16 out
  graph          the fp32 call captured once in a CUDA graph and replayed
  torch          stock fp32 torch.stft / torch.istft on the same GPU (cuFFT; one call per item for ragged batches)
  generate       Generator.generate alone      generate+denoise  generate, then the denoiser (their difference is
                                                                   the denoiser's share of a vocoding call)
Device time per call (CUDA events, median and min / max of REPS alternated runs).  Also checks that each arm's output
agrees with the kernels' (max abs difference).  Writes a JSON record with the card's name and power limit
(default profiles/h100_denoise.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import denoiser, models, synth

N, H, W = 1024, 256, 1024
REPS, INNER = 5, 10
SEED, LO, HI = 2024, 86, 861  # scripts/ragged_time.py's utterances


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def torch_route(audio, bias, lens, voice, strength=0.1):
    win = torch.hann_window(W, device=audio.device)
    out = torch.zeros_like(audio)
    B, L = audio.shape
    if lens is None:
        S = torch.stft(audio, N, H, W, win, center=True, pad_mode="reflect", return_complex=True)
        M = S.abs()
        b = bias[torch.as_tensor(voice or [0] * B, device=audio.device)][:, :, None]
        Y = torch.clamp(M - strength * b, min=0) * torch.where(M > 0, S / M, torch.ones_like(S))
        return torch.istft(Y, N, H, W, win, center=True, length=L)
    for i, Li in enumerate(lens):
        S = torch.stft(audio[i, :Li], N, H, W, win, center=True, pad_mode="reflect", return_complex=True)
        M = S.abs()
        b = bias[voice[i] if voice else 0][:, None]
        Y = torch.clamp(M - strength * b, min=0) * torch.where(M > 0, S / M, torch.ones_like(S))
        out[i, :Li] = torch.istft(Y, N, H, W, win, center=True, length=Li)
    return out


def timed(f):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(INNER):
        f()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / INNER


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_denoise.json")
    args = ap.parse_args()
    gens = []
    for v in range(16):
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(x) for k, x in synth.generator_state(1234 + v).items()})
        gens.append(g.cuda().eval())
    rng = np.random.default_rng(SEED)
    lens_f = [int(v) for v in rng.integers(LO, HI + 1, 64)]
    T = max(lens_f)
    mel = torch.zeros(64, 80, T, device="cuda")
    for i, L in enumerate(lens_f):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    mel2 = torch.from_numpy(synth.mel_input(64, 32, 5)).cuda()
    with torch.no_grad():
        d1 = denoiser.Denoiser(gens[0])
        d16 = denoiser.Denoiser(gens)
        a_cfg2 = gens[0].generate(mel2)[:, 0].contiguous()
        a_rag = gens[0].generate(mel, lens_f)[:, 0].contiguous()
        voice = [v for v in range(16) for _ in range(4)]
        a_voi = models.generate_voices(gens, mel, voice, lens_f)[:, 0].contiguous()
        a_long = torch.from_numpy(np.random.default_rng(1).uniform(-0.5, 0.5, (1, 220500)).astype(np.float32)).cuda()
    work = {
        "config2": dict(audio=a_cfg2, d=d1, lens=None, voice=None, mel=mel2, mel_lens=None),
        "ragged": dict(audio=a_rag, d=d1, lens=[256 * v for v in lens_f], voice=None, mel=mel, mel_lens=lens_f),
        "voices": dict(audio=a_voi, d=d16, lens=[256 * v for v in lens_f], voice=voice, mel=mel, mel_lens=lens_f),
        "long": dict(audio=a_long, d=d1, lens=None, voice=None, mel=None, mel_lens=None),
    }
    rec = {"card": card(), "analysis": {"n_fft": N, "hop": H, "win_length": W, "strength": 0.1}, "reps": REPS,
           "calls_per_timing": INNER, "workloads": {}}
    with torch.no_grad():
        for name, w in work.items():
            a, d, lens, vo = w["audio"], w["d"], w["lens"], w["voice"]
            arms = {
                "kernels": lambda: d(a, 0.1, lens, vo),
                "kernels_pcm16": lambda: d(a, 0.1, lens, vo, dtype=torch.int16),
                "torch": lambda: torch_route(a, d.bias_spec, lens, vo),
            }
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                d(a, 0.1, lens, vo)
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                yg = d(a, 0.1, lens, vo)
            arms["graph"] = g.replay
            if w["mel"] is not None:
                gm, ml = w["mel"], w["mel_lens"]
                if name == "voices":
                    gen_only = lambda: models.generate_voices(gens, gm, vo, ml)
                    gen_den = lambda: d(models.generate_voices(gens, gm, vo, ml), 0.1, lens, vo)
                else:
                    gen_only = lambda: gens[0].generate(gm, ml)
                    gen_den = lambda: d(gens[0].generate(gm, ml), 0.1, lens, vo)
                arms["generate"] = gen_only
                arms["generate+denoise"] = gen_den
            for f in arms.values():
                f()
            torch.cuda.synchronize()
            ms = {k: [] for k in arms}
            for _ in range(REPS):
                for k, f in arms.items():
                    ms[k].append(timed(f))
            ref = d(a, 0.1, lens, vo)
            agree = {"torch_max_abs_diff": float((torch_route(a, d.bias_spec, lens, vo) - ref).abs().max()),
                     "graph_bit_identical": bool(torch.equal(yg, ref))}
            stat = {k: {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v)), "runs_ms": v}
                    for k, v in ms.items()}
            entry = {"shape": list(a.shape), "items": a.shape[0],
                     "samples": int(sum(lens)) if lens else int(a.numel()), "timing": stat, "agreement": agree,
                     "kernels_vs_torch_median": stat["torch"]["median_ms"] / stat["kernels"]["median_ms"]}
            if "generate" in stat:
                entry["denoise_share_of_vocoding"] = 1 - stat["generate"]["median_ms"] / stat["generate+denoise"]["median_ms"]
            rec["workloads"][name] = entry
            print(name, json.dumps({k: round(v["median_ms"], 4) for k, v in stat.items()}), flush=True)
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
