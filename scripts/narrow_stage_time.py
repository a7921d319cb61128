"""The two narrow ResBlock kernels of the default chain at config 2 (B = 64, T = 32): res2 (64 channels) and
up3+res3+post (32 channels).
  kernel_ms   per-kernel CUDA-event times of every launch of the forward (mg_gen_forward_timed: one chain, every kernel
              bracketed), mean and median over REPS forwards, the L2 flushed before each
  trace       clock64 phases of one interior CTA (mg_gen_resblock_trace) of stage codes 2, 3 and 14: tile load / front
              section, per conv the MMA phase and the hand-off, the conv_post epilogue
Prints one JSON record with the card's name, power limit and SM clock cap, read in the same call; --out writes it too."""
import argparse
import ctypes
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import engine, synth

REPS = 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def trace(gd, code):
    """Cycle counts of one interior CTA of stage code 2, 3 or 14 at config 2's shapes."""
    L = engine.lib()
    L.mg_gen_resblock_trace.restype = ctypes.c_int
    L.mg_gen_resblock_trace.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_void_p]
    C, Lp = (64, 4096) if code == 2 else (32, 8192)
    x = torch.randn(64, 2 * C, Lp // 2, device="cuda") if code == 14 else torch.randn(64, C, Lp, device="cuda")
    y = torch.empty(64, 1, Lp, device="cuda") if code == 14 else torch.empty_like(x)
    tr = np.zeros(128, np.int64)
    for _ in range(2):
        engine.check(L.mg_gen_resblock_trace(gd.packed.data_ptr(), code, x.data_ptr(), y.data_ptr(), 64, Lp, tr.ctypes.data))
    d = lambda a, b: int(tr[a] - tr[b])
    out = {"total": d(20, 0), "before_first_conv": d(1, 0),
           "mma_phase_per_conv": [d(3 + 3 * c, 2 + 3 * c) for c in range(6)],
           "hand_off_per_conv": [d(4 + 3 * c, 3 + 3 * c) for c in range(5)]}
    if code == 14 and tr[21] > 0:  # (a build without the front-section stamps leaves the slots at zero)
        out["front"] = {"operand_load": d(21, 0), "convt_mmas": d(22, 21), "deinterleave": d(23, 22),
                        "slack_zero_and_first_hand_off": d(1, 23)}
        out["conv_post"] = {"per_tap_sums": d(26, 24), "barrier_taps_tanh_store": d(25, 26)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    args = ap.parse_args()
    state = synth.generator_state(1234)
    gd = engine.GeneratorDevice("cuda:0")
    order = [n for n, *_ in synth.GENERATOR_LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    gd.pack([to(state[n + ".weight_v"]) for n in order], [to(state[n + ".weight_g"]) for n in order],
            [to(state[n + ".bias"]) for n in order])
    mels = [to(synth.mel_input(64, 32, i)) for i in range(4)]
    out = torch.empty((64, 1, 8192), dtype=torch.float32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for i in range(5):
        gd.forward_timed(mels[i % 4], out)
    names, rows = None, []
    for k in range(REPS):
        flush.zero_()
        timed = gd.forward_timed(mels[k % 4], out)
        names = [n for n, _ in timed]
        rows.append([v for _, v in timed])
    gd.check_status(64, 32)
    rows = np.array(rows)
    rec = {"card": card(), "config": "config 2: B = 64, T = 32", "reps": REPS,
           "kernel_ms_mean": {n: float(rows[:, i].mean()) for i, n in enumerate(names)},
           "kernel_ms_median": {n: float(np.median(rows[:, i])) for i, n in enumerate(names)},
           "trace_cycles": {str(c): trace(gd, c) for c in (2, 3, 14)}}
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
