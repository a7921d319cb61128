"""Context numbers (NOT part of bench.py's contract): the same forwards run by stock PyTorch ops (cuDNN/ATen) on the same
GPU, TF32 (PyTorch default) and strict fp32, next to this engine.  Uses the torch restatements that the autograd path
keeps anyway (Generator._torch_forward / MultiScaleDiscriminator._torch_forward).  CUDA events, L2 flushed between steps."""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth


def timed(fn, steps=20, warmup=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for a, b in ev:
        flush.zero_()
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def main():
    out = {}
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    vs, gs, bs = g._param_triplets()
    leaves = [t for trip in zip(vs, gs, bs) for t in trip]
    x = torch.from_numpy(synth.mel_input(64, 32, 0)).cuda()
    with torch.no_grad():
        ours = g(x)
        for name, prec in (("tf32", "tf32"), ("ieee", "ieee")):
            torch.backends.cudnn.conv.fp32_precision = prec
            ref = g._torch_forward(x, leaves)
            err = float((ours - ref).abs().max() / ref.abs().max())
            out["gen_stock_%s_ms" % name] = timed(lambda: g._torch_forward(x, leaves))
            out["gen_ours_vs_stock_%s_maxrel" % name] = err
        out["gen_ours_ms"] = timed(lambda: g(x))
    d = models.MultiScaleDiscriminator()
    d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    d = d.cuda().eval()
    vs, gs, bs = d._param_triplets()
    dleaves = [t for trip in zip(vs, gs, bs) for t in trip]
    y = torch.from_numpy(synth.audio_input(16, 8192, 0)).cuda()
    yh = torch.from_numpy(synth.audio_input(16, 8192, 1)).cuda()
    y2 = torch.cat([y, yh])
    with torch.no_grad():
        for name, prec in (("tf32", "tf32"), ("ieee", "ieee")):
            torch.backends.cudnn.conv.fp32_precision = prec
            out["msd_stock_%s_ms" % name] = timed(lambda: d._torch_forward(y2, dleaves))
        out["msd_ours_ms"] = timed(lambda: d(y, yh))
    out["config"] = "generator: B=64, T=32 (config 2); MSD: B=16 real + 16 generated, L=8192 (config 3 shapes, forward only)"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
