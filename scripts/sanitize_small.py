"""Tiny generator + discriminator forwards, a sliced generator forward, a ragged batch, one training step (fused losses, native
discriminator backward, multi-tensor Adam) for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os
import sys

import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth
from melgan_multi_b200.optim import Adam

g = models.Generator()
g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
g = g.cuda().eval()
d = models.MultiScaleDiscriminator()
d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
d = d.cuda().eval()
with torch.no_grad():
    y = g(torch.from_numpy(synth.mel_input(1, 3, 5)).cuda())
    g._dev.check_status(1, 3)
    out = d(y, torch.from_numpy(synth.audio_input(1, 768, 1)).cuda())
    d._dev.check_status()
    if os.environ.get("MG_GEN_SLICES"):  # two batch-slice chains on forked streams
        y2 = g(torch.from_numpy(synth.mel_input(2, 3, 6)).cuda())
        g._dev.check_status(2, 3)
    # T = 40: stage 0 is 320 positions -> several 64-position tiles per item, several tiles per item in the later stages,
    # stage 3's ConvT fused at the front of the last kernel
    y3 = g(torch.from_numpy(synth.mel_input(1, 40, 9)).cuda())
    g._dev.check_status(1, 40)
    # the chain with stage 1's and 3's ConvTs at the tail of the previous ResBlock (fp32 fix-up included) and the mel front end
    from melgan_multi_b200 import engine, meldataset
    engine.check(engine.lib().mg_gen_set_pipeline(0b1010))
    y4 = g(torch.from_numpy(synth.mel_input(1, 5, 10)).cuda())
    g._dev.check_status(1, 5)
    engine.check(engine.lib().mg_gen_set_pipeline(-1))
    # a ragged batch of three items (NaN past each length), cut into two slices when MG_GEN_SLICES=2
    mr = torch.from_numpy(synth.mel_input(3, 40, 11)).cuda()
    mr[0, :, 5:] = float("nan")
    mr[2, :, 17:] = float("nan")
    yr = g.generate(mr, [5, 40, 17])
    g._dev.check_status(3, 40)
    # the single-pass bf16 kernels (hi-only weight stream, multicast and halo exchange of the clustered stages): a uniform
    # batch with several tiles per item, and the ragged batch
    yb = g.generate(torch.from_numpy(synth.mel_input(1, 40, 9)).cuda(), precision="bf16")
    g._dev.check_status(1, 40)
    yrb = g.generate(mr, [5, 40, 17], precision="bf16")
    g._dev.check_status(3, 40)
    m = meldataset.mel_spectrogram(y3[0, 0].clamp(-1, 1), 1024, 80, 22050, 256, 1024, 55, 9000)
# one train.py:108-129 step on a 512-sample segment
g.train(); d.train()
og, od = Adam(g.parameters(), 1e-4, betas=(0.5, 0.9)), Adam(d.parameters(), 1e-4, betas=(0.5, 0.9))
x = torch.from_numpy(synth.mel_input(1, 2, 7)).cuda()
yr = torch.from_numpy(synth.audio_input(1, 512, 8)).cuda()
yh = g(x)
dr, dg, fr, fg = d(yr, yh)
loss = models.generator_loss(dg) + models.feature_loss(fr, fg)
loss.backward(); og.step()
od.zero_grad()
dr, dg, _, _ = d(yr, yh.detach())
ld, _, _ = models.discriminator_loss(dr, dg)
ld.backward(); od.step()
torch.cuda.synchronize()
print("ok", float(y.abs().sum()), float(out[0][0].abs().sum()), float(loss), float(ld))
