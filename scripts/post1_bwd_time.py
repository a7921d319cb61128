"""conv_post1 (Conv1d 1024 -> 1024, k5) backward at the three training shapes (2 x 16 items of 8192 samples: 128 / 65 / 33 positions): the wgmma
data- and weight-gradient kernels (split-bf16, fp32-grade) against aten.convolution_backward (cuDNN, TF32 default)."""
import json
import sys

import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth

d = models.MultiScaleDiscriminator()
d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
d = d.cuda()
with torch.no_grad():
    d(torch.zeros(1, 1, 64).cuda(), torch.zeros(1, 1, 64).cuda())
dev = d._dev


def timed(fn, n=50):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


out = {}
for s, L in enumerate((128, 65, 33)):
    conv = d.discriminators[s].layers()[5]
    w = torch._weight_norm(conv.weight_v, conv.weight_g, 0).detach()
    x = torch.randn(32, 1024, L, device="cuda")
    dz = torch.randn(32, 1024, L, device="cuda")
    out[f"L{L}"] = {
        "wgrad_tc_us": timed(lambda: dev.post1_wgrad(x, dz)),
        "dgrad_tc_us": timed(lambda: dev.post1_dgrad(s, dz)),
        "aten_wgrad_us": timed(lambda: torch.ops.aten.convolution_backward(dz, x, w, [1024], [1], [2], [1], False, [0], 1, [False, True, True])),
        "aten_dgrad_us": timed(lambda: torch.ops.aten.convolution_backward(dz, x, w, [1024], [1], [2], [1], False, [0], 1, [True, False, False])),
        "wgrad_algorithmic_gflop": 2 * 1024 * 1024 * 5 * 32 * L / 1e9,
    }
print(json.dumps(out, indent=1))
