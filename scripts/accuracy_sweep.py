"""Accuracy margin of the split-bf16 wgmma pipeline (context evidence; the parity tests proper are tests/ against the
oracle and the reference goldens): config 2 (B=64, T=32) generator forward and the MSD forward against the stock-PyTorch
restatement of the same modules in strict fp32 on the same GPU, over several weight seeds and input distributions
(standard normal, and log-mel-like U(-11.5, 2): meldataset.py:22).  Tolerance of BASELINE north_star: 1e-3."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth

torch.backends.cudnn.conv.fp32_precision = "ieee"


def rel(a, b):
    d = (a - b).double()
    return float(d.abs().max() / b.double().abs().max()), float(d.norm() / b.double().norm())


def main():
    out = {"generator": [], "msd": []}
    for seed in range(6):
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1000 + seed).items()})
        g = g.cuda().eval()
        vs, gs, bs = g._param_triplets()
        leaves = [t for trip in zip(vs, gs, bs) for t in trip]
        for realistic in (False, True):
            x = torch.from_numpy(synth.mel_input(64, 32, seed, realistic)).cuda()
            with torch.no_grad():
                m, l2 = rel(g(x), g._torch_forward(x, leaves))
            out["generator"].append({"weight_seed": 1000 + seed, "input": "log-mel-like" if realistic else "normal",
                                     "max_rel": m, "l2_rel": l2})
        d = models.MultiScaleDiscriminator()
        d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(2000 + seed).items()})
        d = d.cuda().eval()
        vs, gs, bs = d._param_triplets()
        dleaves = [t for trip in zip(vs, gs, bs) for t in trip]
        y = torch.from_numpy(synth.audio_input(8, 8192, seed)).cuda()
        yh = torch.from_numpy(synth.audio_input(8, 8192, 100 + seed)).cuda()
        with torch.no_grad():
            _, _, fr, fg = d(y, yh)
            ref = d._torch_forward(torch.cat([y, yh]), dleaves)
        worst = (0.0, 0.0)
        for s in range(3):
            for l in range(7):
                got = torch.cat([fr[s][l], fg[s][l]])
                m, l2 = rel(got, ref[7 * s + l])
                worst = (max(worst[0], m), max(worst[1], l2))
        out["msd"].append({"weight_seed": 2000 + seed, "worst_fmap_max_rel": worst[0], "worst_fmap_l2_rel": worst[1]})
    out["summary"] = {"generator_max_rel": max(r["max_rel"] for r in out["generator"]),
                      "msd_max_rel": max(r["worst_fmap_max_rel"] for r in out["msd"]), "tolerance": 1e-3}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
