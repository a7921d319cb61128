"""The multi-resolution mel loss's forward + backward against the same loss in stock fp32 torch, and what 45 * loss adds
to a training step:
  config3   B = 16 segments of 8192 samples (BASELINE config 3's shape)
  long      B = 64 utterances of 10 s (220 500 samples at 22.05 kHz)
For each shape and each analysis set, one "fwd+bwd" is loss = mel_loss(x, y) then loss.backward():
  reference  one resolution, the reference's config.json analysis (n_fft 1024, hop 256, win 1024, 80 mels, 55-9000 Hz)
  five       n_fft 128 / 256 / 512 / 1024 / 2048, hop n_fft / 4, win n_fft, 10 / 20 / 40 / 80 / 160 mels
Arms:
  kernels    mel_loss.MultiResolutionMelLoss (mg_mel_loss_forward, mg_mel_loss_backward), eager and replayed from a CUDA
             graph (device time without the host's launch cost)
  stock      the definition in fp32 autograd: zero pad, unfold, window, torch.fft.rfft, |.|, matmul with the filter bank,
             clamp / log, F.l1_loss
  front      (reference analysis only) today's route: two meldataset.mel_spectrogram calls and F.l1_loss
Each arm's gradient is compared with the kernels' (max |d| over max |g|).  Then one config-3 training step (generator
forward, MSD, generator loss + feature loss, backward, Adam; the discriminator step) is timed without and with
45 * loss (reference analysis) in the generator loss.  Device time by CUDA events; arms alternate; each reports the
median, min and max of REPS runs of ITERS calls.  Writes a JSON record with the card's name, power limit and SM clock
cap (default profiles/h100_mel_loss.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from melgan_multi_b200 import mel_loss, meldataset, models, synth
from melgan_multi_b200.optim import Adam
from oracle import mel_oracle

REPS, ITERS = 5, 20
ANALYSES = {"reference": ((1024,), (256,), (1024,), (80,)),
            "five": ((128, 256, 512, 1024, 2048), (32, 64, 128, 256, 512), (128, 256, 512, 1024, 2048), (10, 20, 40, 80, 160))}
SR, FMIN, FMAX = 22050, 55.0, 9000.0


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


def stock_loss_fn(res):
    """The definition in fp32 torch ops, with each resolution's window and filter bank on the device."""
    parts = []
    for n, h, w, m in zip(*res):
        win = F.pad(torch.hann_window(w), ((n - w) // 2, n - w - (n - w) // 2)).cuda()
        fb = torch.from_numpy(mel_oracle.mel_filterbank64(SR, n, m, FMIN, FMAX, norm=1)).float().cuda()
        parts.append((n, h, win, fb))

    def loss(x, y):
        total = 0.0
        for n, h, win, fb in parts:
            p = (n - h) // 2

            def mel(s):
                S = torch.fft.rfft(F.pad(s, (p, p)).unfold(-1, n, h) * win).abs() @ fb.T
                return torch.log(torch.clamp(S, min=1e-5))
            total = total + F.l1_loss(mel(x), mel(y))
        return total / len(parts)
    return loss


def front_loss(x, y):
    mx = meldataset.mel_spectrogram(x, 1024, 80, SR, 256, 1024, FMIN, FMAX, check_range=False)
    my = meldataset.mel_spectrogram(y, 1024, 80, SR, 256, 1024, FMIN, FMAX, check_range=False)
    return F.l1_loss(mx, my)


def fwd_bwd_arms(B, L, name):
    res = ANALYSES[name]
    rs = np.random.RandomState(B)
    x = torch.from_numpy((rs.uniform(-1, 1, (B, L)) * 0.5).astype(np.float32)).cuda().requires_grad_(True)
    y = torch.from_numpy((rs.uniform(-1, 1, (B, L)) * 0.5).astype(np.float32)).cuda()
    mod = mel_loss.MultiResolutionMelLoss(*res, sampling_rate=SR, fmin=FMIN, fmax=FMAX).cuda()
    arms = {"kernels": lambda a, b: mod(a, b), "stock": stock_loss_fn(res)}
    if name == "reference":
        arms["front"] = front_loss
    grads, values = {}, {}
    for k, f in arms.items():
        x.grad = None
        loss = f(x, y)
        loss.backward()
        grads[k], values[k] = x.grad.clone(), float(loss.detach())
    del loss                                    # frees the graph, so the capture below meets no stale AccumulateGrad node
    agree = {k: float((grads[k] - grads["kernels"]).abs().max() / grads["kernels"].abs().max()) for k in arms if k != "kernels"}

    def run(f):
        def g():
            x.grad = None
            f(x, y).backward()
        return g
    fns = {k: run(f) for k, f in arms.items()}
    for f in fns.values():
        device_ms(f, 3)
    runs = {k: [] for k in fns}
    for _ in range(REPS):
        for k, f in fns.items():
            runs[k].append(device_ms(f, ITERS))
    xg = x.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            torch.autograd.grad(mod(xg, y), xg)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        torch.autograd.grad(mod(xg, y), xg)
    graphed = []
    device_ms(graph.replay, 3)
    for _ in range(REPS):
        graphed.append(device_ms(graph.replay, ITERS))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(ITERS):
            fns["kernels"]()
        torch.cuda.synchronize()
    per_kernel = {}
    for e in prof.key_averages():
        if "mel_loss_" in e.key:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            per_kernel[e.key] = t / 1000.0 / ITERS
    return {"B": B, "L": L, "analysis": [list(v) for v in res], "fwd_bwd_ms": {k: stats(v) for k, v in runs.items()},
            "kernels_graph_ms": stats(graphed), "per_kernel_ms": per_kernel, "grad_max_abs_diff_over_max": agree,
            "loss_values": values}


def train_steps():
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    msd = models.MultiScaleDiscriminator()
    msd.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    gen, msd = gen.cuda().train(), msd.cuda().train()
    g_opt, d_opt = Adam(gen.parameters(), 2e-4, betas=(0.5, 0.9)), Adam(msd.parameters(), 2e-4, betas=(0.5, 0.9))
    x = torch.from_numpy(synth.mel_input(16, 32, 100)).cuda()
    y = torch.from_numpy(synth.audio_input(16, 8192, 200)).cuda()
    loss = mel_loss.MultiResolutionMelLoss().cuda()

    def step(mel_term):
        g_opt.zero_grad()
        y_ghat = gen(x)
        dr, dg, fr, fg = msd(y, y_ghat)
        loss_gen = models.generator_loss(dg) + models.feature_loss(fr, fg)
        if mel_term:
            loss_gen = loss_gen + 45 * loss(y_ghat, y)
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
    ap.add_argument("--out", default="profiles/h100_mel_loss.json")
    a = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    rec = {"card": card(), "torch": torch.__version__}
    for shape, (B, L) in (("config3", (16, 8192)), ("long", (64, 220500))):
        for name in ANALYSES:
            rec["%s_%s" % (shape, name)] = fwd_bwd_arms(B, L, name)
            torch.cuda.empty_cache()
    rec["train_step_config3_ms"] = train_steps()
    rec["card_after"] = card()
    print(json.dumps(rec, indent=1))
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
