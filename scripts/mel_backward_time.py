"""The mel front end's forward + backward against a stock fp32 torch path, and what a mel-L1 term adds to a training step:
  config3   B = 16 segments of 8192 samples (BASELINE config 3's shape)
  long      B = 64 utterances of 10 s (220 500 samples at 22.05 kHz)
For each shape, one "fwd+bwd" is mel = mel_spectrogram(y) then mel.backward(g):
  kernels   meldataset.mel_spectrogram (mg_mel_spectrogram forward, mg_mel_spectrogram_backward backward)
  stock     torch.stft (center=False on the 384-padded signal, periodic Hann) -> |.| -> matmul with the fp32 filter bank ->
            clamp(min=1e-5) -> log, all in fp32 autograd
Both arms' gradients are compared against each other (max |d| over max |g|).  Then one config-3 training step
(generator forward, MSD, generator loss + feature loss, backward, Adam; the discriminator step) is timed without and with
`45 * l1_loss(mel_spectrogram(y_ghat.squeeze(1)), x)` in the generator loss.  Device time by CUDA events; arms alternate;
each reports the median of REPS runs of ITERS calls.  Writes a JSON record with the card's name and power limit (default
profiles/h100_mel_backward.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from melgan_multi_b200 import meldataset, models, synth
from melgan_multi_b200.optim import Adam
from oracle import mel_oracle as mo

REPS, ITERS = 5, 20
ARGS = (1024, 80, 22050, 256, 1024, 55.0, 9000.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "runs": [float(x) for x in v]}


def device_ms(f, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        f()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def stock_mel(fb, win):
    def f(y):
        spec = torch.stft(F.pad(y, (384, 384)), 1024, hop_length=256, win_length=1024, window=win, center=False,
                          return_complex=True).abs()
        return torch.log(torch.clamp(torch.matmul(fb, spec), min=1e-5))
    return f


def fwd_bwd_arms(B, L):
    rs = np.random.RandomState(B)
    y = torch.from_numpy((rs.uniform(-1, 1, (B, L)) * 0.5).astype(np.float32)).cuda().requires_grad_(True)
    g = torch.from_numpy(rs.standard_normal((B, 80, L // 256)).astype(np.float32)).cuda()
    fb = torch.from_numpy(mo.mel_filterbank64(22050, 1024, 80, 55.0, 9000.0, 1).astype(np.float32)).cuda()
    win = torch.hann_window(1024, periodic=True, device="cuda")
    stock = stock_mel(fb, win)

    def kernels():
        y.grad = None
        meldataset.mel_spectrogram(y, *ARGS, check_range=False).backward(g)

    def torch_arm():
        y.grad = None
        stock(y).backward(g)

    kernels()
    gk = y.grad.clone()
    torch_arm()
    gt = y.grad.clone()
    agree = float((gk - gt).abs().max() / gt.abs().max())
    runs = {"kernels": [], "stock": []}
    for f in (kernels, torch_arm):
        device_ms(f, 3)
    for _ in range(REPS):
        runs["kernels"].append(device_ms(kernels, ITERS))
        runs["stock"].append(device_ms(torch_arm, ITERS))
    fwd = []
    with torch.no_grad():
        for _ in range(REPS):
            fwd.append(device_ms(lambda: meldataset.mel_spectrogram(y, *ARGS, check_range=False), ITERS))
    return {"B": B, "L": L, "T": L // 256, "fwd_bwd_ms": {k: stats(v) for k, v in runs.items()},
            "kernel_forward_only_ms": stats(fwd), "grad_max_abs_diff_over_max": agree}


def train_steps():
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    msd = models.MultiScaleDiscriminator()
    msd.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    gen, msd = gen.cuda().train(), msd.cuda().train()
    g_opt, d_opt = Adam(gen.parameters(), 2e-4, betas=(0.5, 0.9)), Adam(msd.parameters(), 2e-4, betas=(0.5, 0.9))
    x = torch.from_numpy(synth.mel_input(16, 32, 100)).cuda()
    y = torch.from_numpy(synth.audio_input(16, 8192, 200)).cuda()

    def step(mel_term):
        g_opt.zero_grad()
        y_ghat = gen(x)
        dr, dg, fr, fg = msd(y, y_ghat)
        loss_gen = models.generator_loss(dg) + models.feature_loss(fr, fg)
        if mel_term:
            loss_gen = loss_gen + 45 * F.l1_loss(meldataset.mel_spectrogram(y_ghat.squeeze(1), *ARGS, check_range=False), x)
        loss_gen.backward()
        g_opt.step()
        d_opt.zero_grad()
        dr, dg, _, _ = msd(y, y_ghat.detach())
        loss_disc, _, _ = models.discriminator_loss(dr, dg)
        loss_disc.backward()
        d_opt.step()

    runs = {"without_mel_term": [], "with_mel_term": []}
    for m in (False, True):
        device_ms(lambda: step(m), 3)
    for _ in range(REPS):
        runs["without_mel_term"].append(device_ms(lambda: step(False), 10))
        runs["with_mel_term"].append(device_ms(lambda: step(True), 10))
    return {k: stats(v) for k, v in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_mel_backward.json")
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    rec = {"card": card(), "torch": torch.__version__,
           "config3": fwd_bwd_arms(16, 8192), "long": fwd_bwd_arms(64, 220500), "train_step_config3_ms": train_steps()}
    rec["card_after"] = card()
    print(json.dumps(rec, indent=1))
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
