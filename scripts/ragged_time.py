"""Vocoding 64 utterances of different lengths (seeded, uniform in [86, 861] mel frames: 1 to 10 s at 22.05 kHz) three
ways, on the same weights and inputs:
  ragged  one Generator.generate(mel [64, 80, T_max], lengths) call
  loop    64 calls of Generator.forward(mel[i:i+1, :, :T_i]) (B = 1 each)
  padded  one Generator.forward on the batch zero-padded to T_max, then cropped
Device time per pass (CUDA events around the whole pass, median of REPS alternated passes, min / max for the spread).
The padded pass is not exact: it also reports, per item, the largest deviation from the item's own audio in its last
2048 samples.  Writes a JSON record with the card's name and power limit (default profiles/h100_ragged.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth

B, LO, HI, SEED, REPS = 64, 86, 861, 2024, 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_ragged.json")
    args = ap.parse_args()
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B)]
    T = max(lens)
    mel = torch.zeros(B, 80, T, device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    items = [mel[i:i + 1, :, :L].contiguous() for i, L in enumerate(lens)]

    def ragged():
        return g.generate(mel, lens)

    def loop():
        return [g(x) for x in items]

    def padded():
        return g(mel)

    passes = {"ragged": ragged, "loop": loop, "padded": padded}
    with torch.no_grad():
        for f in passes.values():  # warm every shape (and the workspace at its largest)
            f()
        torch.cuda.synchronize()
        ms = {k: [] for k in passes}
        for _ in range(REPS):
            for k, f in passes.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                torch.cuda.synchronize()
                ms[k].append(a.elapsed_time(b))
        exact = [y[0, 0] for y in loop()]
        yr, yp = ragged(), padded()
        g._dev.check_status(B, T)
    bit_identical = all(torch.equal(yr[i, 0, :256 * L], exact[i]) for i, L in enumerate(lens))
    pad_dev = [float((yp[i, 0, 256 * L - 2048:256 * L] - exact[i][-2048:]).abs().max()) for i, L in enumerate(lens)]
    stat = {k: {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v)), "runs_ms": v}
            for k, v in ms.items()}
    rec = {
        "card": card(),
        "workload": {"items": B, "frames": sum(lens), "T_max": T, "lengths_uniform_in": [LO, HI], "seed": SEED,
                     "audio_seconds": sum(lens) * 256 / 22050.0},
        "timing": stat,
        "speedup_ragged_vs_loop": {"median": stat["loop"]["median_ms"] / stat["ragged"]["median_ms"],
                                   "worst": stat["loop"]["min_ms"] / stat["ragged"]["max_ms"],
                                   "best": stat["loop"]["max_ms"] / stat["ragged"]["min_ms"]},
        "ragged_bit_identical_to_loop": bit_identical,
        "padded_last_2048_max_abs_dev": {"max": max(pad_dev), "median": float(np.median(pad_dev)),
                                         "items_exact": sum(d == 0.0 for d in pad_dev)},
    }
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
