"""The multi-resolution STFT loss's forward + backward against the same loss in stock fp32 torch, and what sc + mag adds
to a training step:
  config3   B = 16 segments of 8192 samples (BASELINE config 3's shape)
  long      B = 64 utterances of 10 s (220 500 samples at 22.05 kHz)
For each shape, one "fwd+bwd" is sc, mag = loss(x, y) then (sc + mag).backward(), at the default resolutions
(fft 1024/2048/512, hop 120/240/50, win 600/1200/240):
  kernels   stft_loss.MultiResolutionSTFTLoss (mg_stft_loss_forward, mg_stft_loss_backward)
  stock     Parallel WaveGAN's statement in fp32 autograd: torch.stft (center=True, reflect, periodic Hann) ->
            sqrt(clamp(re^2 + im^2, 1e-7)) -> Frobenius-norm ratio and L1 of the logs
Both arms' gradients are compared (max |d| over max |g|).  "kernel_forward_only_ms" is the forward alone under no_grad.
"kernels_graph_ms" replays the kernels' forward + backward from a CUDA graph: device time without the host's launch
cost, which at 16 x 8192 is most of the eager figure.  "per_kernel_ms" is each kernel's device time per fwd+bwd from
torch.profiler in a run of its own.  "save_arm_floor_ms" times a device-to-device copy of 12 bytes per bin (X of x as
complex64 and y_mag as fp32, every resolution): the least extra traffic a backward that reads saved spectra instead of
recomputing them would add (the forward writes those bytes, the backward reads them), to set against the recompute's
forward-kernel time.  Then one config-3 training step (generator forward, MSD,
generator loss + feature loss, backward, Adam; the discriminator step) is timed without and with sc + mag in the
generator loss.  Device time by CUDA events; arms alternate; each reports the median, min and max of REPS runs of ITERS
calls.  Writes a JSON record with the card's name and power limit (default profiles/h100_stft_loss.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from melgan_multi_b200 import models, stft_loss, synth
from melgan_multi_b200.optim import Adam

REPS, ITERS = 5, 20
RES = ((1024, 2048, 512), (120, 240, 50), (600, 1200, 240))


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


def stock_loss(x, y):
    sc = mag = 0.0
    for n, h, w in zip(*RES):
        win = torch.hann_window(w, device=x.device)

        def m(s):
            X = torch.stft(s, n, h, w, win, center=True, pad_mode="reflect", return_complex=True)
            return torch.sqrt(torch.clamp(X.real ** 2 + X.imag ** 2, min=1e-7)).transpose(2, 1)
        xm, ym = m(x), m(y)
        sc = sc + torch.norm(ym - xm, p="fro") / torch.norm(ym, p="fro")
        mag = mag + F.l1_loss(torch.log(ym), torch.log(xm))
    return sc / 3, mag / 3


def fwd_bwd_arms(B, L):
    rs = np.random.RandomState(B)
    x = torch.from_numpy((rs.uniform(-1, 1, (B, L)) * 0.5).astype(np.float32)).cuda().requires_grad_(True)
    y = torch.from_numpy((rs.uniform(-1, 1, (B, L)) * 0.5).astype(np.float32)).cuda()
    loss = stft_loss.MultiResolutionSTFTLoss(*RES)

    def kernels():
        x.grad = None
        sc, mag = loss(x, y)
        (sc + mag).backward()

    def torch_arm():
        x.grad = None
        sc, mag = stock_loss(x, y)
        (sc + mag).backward()

    kernels()
    gk = x.grad.clone()
    vk = [float(v) for v in loss(x.detach(), y)]
    torch_arm()
    gt = x.grad.clone()
    vt = [float(v) for v in stock_loss(x.detach(), y)]
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
            fwd.append(device_ms(lambda: loss(x, y), ITERS))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            kernels()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sc, mag = loss(x, y)
        torch.autograd.grad(sc + mag, x)
    graphed = []
    device_ms(graph.replay, 3)
    for _ in range(REPS):
        graphed.append(device_ms(graph.replay, ITERS))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(ITERS):
            kernels()
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        if "stft_loss_" in e.key:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            per_kernel[e.key] = t / 1000.0 / ITERS
    nbytes = sum(12 * B * (1 + L // h) * (n // 2 + 1) for n, h in zip(RES[0], RES[1]))
    src = torch.empty(nbytes // 4, device="cuda")
    dst = torch.empty_like(src)
    copies = []
    device_ms(lambda: dst.copy_(src), 3)
    for _ in range(REPS):
        copies.append(device_ms(lambda: dst.copy_(src), ITERS))
    del src, dst
    return {"B": B, "L": L, "fwd_bwd_ms": {k: stats(v) for k, v in runs.items()}, "kernel_forward_only_ms": stats(fwd),
            "kernels_graph_ms": stats(graphed), "per_kernel_ms": per_kernel,
            "save_arm_floor_ms": stats(copies), "save_arm_bytes": nbytes,
            "grad_max_abs_diff_over_max": agree, "sc_mag_kernels": vk, "sc_mag_stock": vt}


def train_steps():
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    msd = models.MultiScaleDiscriminator()
    msd.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    gen, msd = gen.cuda().train(), msd.cuda().train()
    g_opt, d_opt = Adam(gen.parameters(), 2e-4, betas=(0.5, 0.9)), Adam(msd.parameters(), 2e-4, betas=(0.5, 0.9))
    x = torch.from_numpy(synth.mel_input(16, 32, 100)).cuda()
    y = torch.from_numpy(synth.audio_input(16, 8192, 200)).cuda()
    loss = stft_loss.MultiResolutionSTFTLoss(*RES)

    def step(stft_term):
        g_opt.zero_grad()
        y_ghat = gen(x)
        dr, dg, fr, fg = msd(y, y_ghat)
        loss_gen = models.generator_loss(dg) + models.feature_loss(fr, fg)
        if stft_term:
            sc, mag = loss(y_ghat.squeeze(1), y.squeeze(1))
            loss_gen = loss_gen + sc + mag
        loss_gen.backward()
        g_opt.step()
        d_opt.zero_grad()
        dr, dg, _, _ = msd(y, y_ghat.detach())
        loss_disc, _, _ = models.discriminator_loss(dr, dg)
        loss_disc.backward()
        d_opt.step()

    runs = {"without_stft_term": [], "with_stft_term": []}
    for m in (False, True):
        device_ms(lambda: step(m), 3)
    for _ in range(REPS):
        runs["without_stft_term"].append(device_ms(lambda: step(False), 10))
        runs["with_stft_term"].append(device_ms(lambda: step(True), 10))
    return {k: stats(v) for k, v in runs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_stft_loss.json")
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
