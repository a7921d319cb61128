"""The multi-resolution mel loss (csrc/mg_mel_loss.cu through mel_loss.MultiResolutionMelLoss) against float64 autograd
of its definition, run on the CPU through torch.fft.rfft, at every supported n_fft, window and hop shape, and through
the generator; at the reference analysis against meldataset.mel_spectrogram's forward and backward; then determinism,
concurrency, CUDA-graph replay, no host sync, poisoned buffers and NaN / Inf.

Error model.  As in test_stft_loss_gpu.py, per frame f, E_f = TAU_F ||w . frame_f||_2 is taken as the error of each
bin the fp32 FFT computes, hence of each magnitude |X_k| (a per-bin RMS model; the propagation below is worst-case given
it).  Per band, with kc_m the filter's bins:
  dS_m = E_f sum_k F[m, k] + (kc_m + 3) u S_m               (the fp32 dot product, the fp32 weights, the sqrt)
  lo_m = max(S_m - dS_m, 1e-5),  dmel_m = dS_m / lo_m + 2 u |mel_m|
  loss          each resolution: mean(dmel_x + dmel_y) + (M / 256 + 16) u l_r (the per-CTA fp32 tree), plus 2 u of the loss
  gradient      c = grad / (R B M T);  where the band passes the clip,
                dgs_m = |c| (dS_m / (S_m lo_m) + 3 u / S_m) + 2 |c| / lo_m   if |mel_x - mel_y| <= dmel_x + dmel_y (sign unsure)
                                                            + |c| / lo_m     if |S_m - 1e-5| <= dS_m (clip unsure)
                ddm_k = sum_m F[m, k] dgs_m + 3 u sum_m F[m, k] |gs_m|,  dG_k = ddm_k + |dm_k| min(2, 2 E_f / |X_k|) + 2 u |dm_k|;
                per frame S_f = 2 sum_k dG_k + 2 TAU_F sqrt(N/2) ||G||_2 + 72 u sum_k |G_k| (test_stft_loss_gpu.py's
                propagation through the split's adjoint, the inverse FFT, the window and the gather), and
                bound_i = sum over resolutions and over the frame positions reading sample i of |w_n| S_f.
The module prints the worst ratio |got - ref| / bound seen for each case.
"""
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import meldataset, mel_loss, models, synth
from oracle import mel_oracle

U = 2.0 ** -24
TAU_F = 2.0 ** -17
CLIP = 1e-5
REF = dict(sampling_rate=22050, fmin=55.0, fmax=9000.0)
FIVE = ((128, 256, 512, 1024, 2048), (32, 64, 128, 256, 512), (128, 256, 512, 1024, 2048), (10, 20, 40, 80, 160))
WORST = {}


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst ratios to the bound: " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------------------------
# float64: the definition, and the bound's ingredients
# ------------------------------------------------------------------------------------------------------------------
def _window64(n, w):
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(w) / w) if w > 1 else np.ones(1)
    return torch.from_numpy(np.pad(win, ((n - w) // 2, n - w - (n - w) // 2)))


def _bank64(n, m, sr, fmin, fmax):
    return torch.from_numpy(mel_oracle.mel_filterbank64(sr, n, m, fmin, sr / 2.0 if fmax is None else fmax, norm=1))


def _frames64(x, n, h, w):
    p = (n - h) // 2
    win = _window64(n, w)
    return F.pad(x, (p, p)).unfold(-1, n, h) * win, win


def _res64(x, n, h, w, m, sr, fmin, fmax):
    """float64 S [B, T, M] and mel of x [B, L] at one resolution, and the pieces the bound uses."""
    fr, win = _frames64(x, n, h, w)
    X = torch.fft.rfft(fr)
    Fb = _bank64(n, m, sr, fmin, fmax)
    S = X.abs() @ Fb.T
    return dict(X=X, S=S, mel=torch.log(torch.clamp(S, min=CLIP)), fr=fr, win=win, Fb=Fb)


def loss64(x, y, res, sampling_rate=22050, fmin=55.0, fmax=9000.0):
    sr = sampling_rate
    total = 0.0
    for n, h, w, m in zip(*res):
        total = total + (_res64(x, n, h, w, m, sr, fmin, fmax)["mel"] - _res64(y, n, h, w, m, sr, fmin, fmax)["mel"]).abs().mean()
    return total / len(res[0])


def grad64(x, y, res, grad=1.0, **kw):
    xt = torch.from_numpy(x).double().requires_grad_(True)
    loss = loss64(xt, torch.from_numpy(y).double(), res, **kw)
    return torch.autograd.grad(loss, xt, torch.tensor(float(grad), dtype=torch.float64))[0].numpy()


def _terms(r):
    E = TAU_F * r["fr"].norm(dim=-1, keepdim=True)                      # [B, T, 1]
    kc = (r["Fb"] > 0).sum(1).double()                                   # [M]
    dS = E * r["Fb"].sum(1) + (kc + 3) * U * r["S"]
    lo = torch.clamp(r["S"] - dS, min=CLIP)
    dmel = dS / lo + 2 * U * r["mel"].abs()
    return E, dS, lo, dmel


def value_bound(x, y, res, sampling_rate=22050, fmin=55.0, fmax=9000.0):
    sr = sampling_rate
    R = len(res[0])
    b = 0.0
    for n, h, w, m in zip(*res):
        rx, ry = _res64(x, n, h, w, m, sr, fmin, fmax), _res64(y, n, h, w, m, sr, fmin, fmax)
        dx, dy = _terms(rx)[3], _terms(ry)[3]
        lr = (rx["mel"] - ry["mel"]).abs().mean()
        b += float((dx + dy).mean() + (m / 256 + 16) * U * lr)
    return b / R + 2 * U * abs(float(loss64(x, y, res, sr, fmin, fmax)))


def _fold(vals, B, L, n, h):
    """Sum of nonnegative per-frame-position values [B, T, n] onto the samples they read (padding dropped)."""
    z = torch.zeros(B, L, dtype=torch.float64, requires_grad=True)
    p = (n - h) // 2
    fr = F.pad(z, (p, p)).unfold(-1, n, h)
    return torch.autograd.grad(fr, z, vals)[0]


def grad_bound(x, y, res, grad=1.0, sampling_rate=22050, fmin=55.0, fmax=9000.0):
    sr = sampling_rate
    B, L = x.shape
    R = len(res[0])
    out = torch.zeros(B, L, dtype=torch.float64)
    for n, h, w, m in zip(*res):
        rx, ry = _res64(x, n, h, w, m, sr, fmin, fmax), _res64(y, n, h, w, m, sr, fmin, fmax)
        E, dS, lo, dmx = _terms(rx)
        dmy = _terms(ry)[3]
        S, T = rx["S"], rx["S"].shape[1]
        c = abs(grad) / (R * B * m * T)
        on = (S >= CLIP) | ((S - CLIP).abs() <= dS)
        gs = on * c / torch.clamp(S, min=CLIP)
        dgs = on * (c * (dS / (torch.clamp(S, min=CLIP) * lo) + 3 * U / torch.clamp(S, min=CLIP)))
        dgs = dgs + on * ((rx["mel"] - ry["mel"]).abs() <= dmx + dmy) * 2 * c / lo
        dgs = dgs + ((S - CLIP).abs() <= dS) * c / lo
        Fb = rx["Fb"]
        dm = gs @ Fb                                                   # [B, T, N/2 + 1], |dm_k| bound
        ddm = dgs @ Fb + 3 * U * dm
        ax = rx["X"].abs()
        ph = torch.where(ax > 0, torch.clamp(2 * E / torch.where(ax > 0, ax, 1.0), max=2.0), torch.full_like(ax, 2.0))
        dG = ddm + dm * ph + 2 * U * dm
        Sf = 2 * dG.sum(-1) + 2 * TAU_F * (n // 2) ** 0.5 * dm.norm(dim=-1) + 72 * U * dm.sum(-1)
        out += _fold(rx["win"].abs() * Sf[..., None], B, L, n, h)
    return out.numpy()


def _signals(B, L, seed):
    """Smooth seeded audio: a few partials with random phase plus a little noise, in [-1, 1]."""
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 22050.0
    out = np.zeros((B, L))
    for b in range(B):
        for _ in range(4):
            out[b] += rng.uniform(0.05, 0.25) * np.sin(2 * np.pi * rng.uniform(60, 6000) * t + rng.uniform(0, 2 * np.pi))
        out[b] += 0.01 * rng.standard_normal(L)
    return out.astype(np.float32)


def _module(res, **kw):
    n, h, w, m = res
    return mel_loss.MultiResolutionMelLoss(n, h, w, m, **{**REF, **kw})


def _run(x, y, res, grad=1.0, module=None, **kw):
    m = module or _module(res, **kw)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    loss = m(xt, torch.from_numpy(y).cuda())
    g, = torch.autograd.grad(loss, xt, torch.tensor(grad, device="cuda"))
    return float(loss), g.cpu().numpy()


def check(x, y, res, key, grads=(1.0, -2.5), **kw):
    args = {**REF, **kw}
    x64, y64 = torch.from_numpy(x).double(), torch.from_numpy(y).double()
    ref = float(loss64(x64, y64, res, **args))
    bv = value_bound(x64, y64, res, **args)
    m = _module(res, **kw)
    for grad in grads:
        loss, g = _run(x, y, res, grad, m)
        assert abs(loss - ref) <= bv, (loss, ref, bv)
        _note(key + " loss", abs(loss - ref) / bv)
        gref = grad64(x, y, res, grad, **args)
        bound = grad_bound(x64, y64, res, grad, **args)
        err = np.abs(g.astype(np.float64) - gref)
        bad = err > bound
        assert not bad.any(), (grad, np.argwhere(bad)[:5], err[bad][:5], bound[bad][:5])
        _note(key + " grad", (err / np.maximum(bound, 1e-300)).max())
    return g


# ------------------------------------------------------------------------------------------------------------------
# values and gradients against float64
# ------------------------------------------------------------------------------------------------------------------
MELS = {128: 20, 256: 40, 512: 64, 1024: 80, 2048: 128}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 256, 512, 1024, 2048])
def test_each_n_fft_alone(n):
    """win_length = n_fft and an odd win_length < n_fft; a hop that divides n_fft and ones that do not, with n_fft - hop
    even and odd; L at the one-frame minimum and long; B of 1 to 3."""
    m = MELS[n]
    cases = [(n, n // 4, 4 * n + 5, 3),
             (n - 3, n // 4 + 3, 8192 + 7, 2),
             (n - 1, n // 3, n - 2 * ((n - n // 3) // 2), 1),       # exactly one frame
             (n // 2 + 1, n // 2 + 1, 5000, 2)]
    for w, h, L, B in cases:
        check(_signals(B, L, 10 + w), _signals(B, L, 20 + h), ((n,), (h,), (w,), (m,)), "n_fft %d" % n)


MIXED8 = ((128, 256, 512, 1024, 2048, 512, 1024, 256), (32, 50, 120, 240, 480, 128, 256, 64),
          (128, 200, 512, 600, 1200, 300, 1024, 255), (16, 30, 64, 80, 128, 50, 100, 24))


@pytest.mark.gpu
def test_eight_mixed_resolutions():
    B, L = 3, 8192
    check(_signals(B, L, 30), _signals(B, L, 31), MIXED8, "8 resolutions")


@pytest.mark.gpu
def test_most_bands_and_empty_filters():
    """512 bands at n_fft 2048, and at n_fft 128 128 bands of which the low ones cover no bin (their band is log(1e-5)
    and gets no gradient)."""
    x, y = _signals(2, 8192, 32), _signals(2, 8192, 33)
    check(x, y, ((2048,), (512,), (2048,), (512,)), "512 bands", fmin=0.0, fmax=None)
    assert (_bank64(128, 128, 22050, 0.0, 11025.0).sum(1) == 0).sum() > 10
    check(x, y, ((128,), (32,), (128,), (128,)), "empty filters", fmin=0.0, fmax=None)


@pytest.mark.gpu
def test_fmax_none_is_half_the_sampling_rate():
    x, y = _signals(2, 8192, 34), _signals(2, 8192, 35)
    res = ((1024, 512), (256, 128), (1024, 512), (80, 40))
    assert _run(x, y, res, fmax=None)[0] == _run(x, y, res, fmax=11025.0)[0]
    check(x, y, res, "fmax None", fmax=None)


@pytest.mark.gpu
def test_bands_below_at_and_above_the_clip_and_silence():
    """Silent stretches, and tones whose bands sit below, around and above S = 1e-5, in x and in y."""
    B, L = 2, 8192
    x, y = _signals(B, L, 3), _signals(B, L, 4)
    t = np.arange(1500)
    for a, (lo, hi) in zip((0.0, 2e-7, 2e-6, 2e-5), ((1000, 2500), (3000, 4500), (5000, 6500), (6600, 8100))):
        x[0, lo:hi] = a * np.sin(0.3 * t)
        y[1, lo:hi] = a * np.cos(0.2 * t)
    y[0, 2000:3500] = 0.0
    check(x, y, ((1024,), (256,), (1024,), (80,)), "clip")
    check(x, y, FIVE, "clip")


@pytest.mark.gpu
def test_equal_signals_give_zero_loss_and_gradient():
    x = _signals(3, 8192, 5)
    for res in (((1024,), (256,), (1024,), (80,)), FIVE):
        loss, g = _run(x, x.copy(), res)
        assert loss == 0.0 and not g.any()
        assert not grad64(x, x.copy(), res, **REF).any()


@pytest.mark.gpu
def test_ten_seconds():
    L = 220500
    check(_signals(1, L, 36), _signals(1, L, 37), ((1024, 256), (256, 64), (1024, 256), (80, 20)), "L 220500", grads=(1.0,))


# ------------------------------------------------------------------------------------------------------------------
# the reference analysis against the front end
# ------------------------------------------------------------------------------------------------------------------
def _front(x):
    return meldataset.mel_spectrogram(x, 1024, 80, 22050, 256, 1024, 55.0, 9000.0, check_range=False)


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(16, 8192), (3, 66167)])
def test_reference_analysis_equals_the_front_end(B, L):
    """The loss is the float64 mean of |mel_spectrogram(x) - mel_spectrogram(y)| within the rounding of the fp32
    per-frame partials; the gradient is mel_spectrogram's own backward driven by the grad_mel the loss forms,
    sign(mel_x - mel_y) * fp32(grad / (B 80 T)), bit for bit: both run the same frame, band and band-adjoint code, the
    same Stockham passes and the same ascending-t gather."""
    x, y = (torch.from_numpy(_signals(B, L, s)).cuda() for s in (40, 41))
    m = mel_loss.MultiResolutionMelLoss()
    xl = x.clone().requires_grad_(True)
    loss = m(xl, y)
    grad = torch.tensor(0.75, device="cuda")
    g, = torch.autograd.grad(loss, xl, grad)
    mx, my = _front(x), _front(y)
    T = mx.shape[-1]
    d = (mx.double() - my.double()).abs()
    ref = float(d.mean())
    bound = (80 / 256 + 18) * U * ref          # each frame's fp32 tree over 80 bands, the float64 finish, the fp32 result
    assert abs(float(loss) - ref) <= bound, (float(loss), ref, bound)
    _note("reference analysis loss (of its rounding)", abs(float(loss) - ref) / bound)
    c = torch.tensor(0.75, dtype=torch.float32) * torch.tensor(1.0 / (1 * B * 80 * T), dtype=torch.float32)
    grad_mel = torch.sign(mx - my) * c.cuda()
    xr = x.clone().requires_grad_(True)
    gref, = torch.autograd.grad(_front(xr), xr, grad_mel)
    assert torch.equal(g, gref), float((g - gref).abs().max())


# ------------------------------------------------------------------------------------------------------------------
# through the generator
# ------------------------------------------------------------------------------------------------------------------
TAU_IEEE = (1e-4, 5e-5)   # test_generator_backward_gpu.py's (max-rel, l2-rel) per tensor under cuDNN "ieee"


@pytest.fixture
def ieee_deterministic():
    old = (torch.backends.cudnn.conv.fp32_precision, torch.backends.cudnn.deterministic)
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.conv.fp32_precision, torch.backends.cudnn.deterministic = old


@pytest.mark.gpu
def test_mel_loss_trains_the_generator(ieee_deterministic):
    """B x T = 2 x 16 mel frames (4096 samples): the parameter and mel gradients of 45 * loss(G(x), y) over the
    five-resolution set equal those of feeding the same generator backward the float64 reference's audio gradient
    (cast to fp32), within the generator backward's own tolerance."""
    from conftest import rel_errors
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    gen = gen.cuda().train()
    x = torch.from_numpy(synth.mel_input(2, 16, 5)).cuda().requires_grad_(True)
    target = torch.from_numpy(_signals(2, 4096, 8)).cuda()
    loss = _module(FIVE)
    y = gen(x)
    gen.zero_grad()
    (45 * loss(y, target[:, None])).backward()
    params = [p for p in gen.parameters()]
    got = [p.grad.clone() for p in params] + [x.grad.clone()]
    assert all(g is not None and g.abs().max() > 0 for g in got)
    g_audio = grad64(y.detach().squeeze(1).cpu().numpy(), target.cpu().numpy(), FIVE, 45.0, **REF)
    gen.zero_grad()
    x.grad = None
    y = gen(x)
    y.backward(torch.from_numpy(g_audio).float().cuda()[:, None, :])
    ref = [p.grad.clone() for p in params] + [x.grad.clone()]
    worst = 0.0
    for i, (a, r) in enumerate(zip(got, ref)):
        m, l2 = rel_errors(a.cpu().numpy(), r.cpu().numpy())
        worst = max(worst, m / TAU_IEEE[0], l2 / TAU_IEEE[1])
        assert m <= TAU_IEEE[0] and l2 <= TAU_IEEE[1], (i, m, l2)
    _note("generator (of its tolerance)", worst)


# ------------------------------------------------------------------------------------------------------------------
# properties
# ------------------------------------------------------------------------------------------------------------------
def _step(m, x, y):
    leaf = x.clone().requires_grad_(True)
    loss = m(leaf, y)
    loss.backward()
    return loss.detach(), leaf.grad


@pytest.mark.gpu
def test_repeated_calls_are_bit_identical_and_do_not_sync():
    m = _module(FIVE)
    x, y = (torch.from_numpy(_signals(4, 8192, s)).cuda() for s in (11, 12))
    first = _step(m, x, y)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        runs = [_step(m, x, y) for _ in range(3)]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for v, g in runs:
        assert torch.equal(v, first[0]) and torch.equal(g, first[1])


@pytest.mark.gpu
def test_two_streams_from_two_threads_match_serial():
    m = _module(FIVE)
    data = [tuple(torch.from_numpy(_signals(4, 22050, 40 + 2 * k + j)).cuda() for j in range(2)) for k in range(2)]
    serial = [_step(m, *data[k]) for k in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None, None]

    def worker(k):
        with torch.cuda.stream(streams[k]):
            for _ in range(5):
                out[k] = _step(m, *data[k])

    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    threads = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(out[k][0], serial[k][0]) and torch.equal(out[k][1], serial[k][1]), k


@pytest.mark.gpu
def test_captured_and_replayed_in_a_cuda_graph():
    m = _module(FIVE)
    x = torch.from_numpy(_signals(4, 8192, 13)).cuda().requires_grad_(True)
    y = torch.from_numpy(_signals(4, 8192, 14)).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            torch.autograd.grad(m(x, y), x)
    torch.cuda.current_stream().wait_stream(s)
    eager = _step(m, x.detach(), y)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = m(x, y)
        grad, = torch.autograd.grad(loss, x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, eager[0]) and torch.equal(grad, eager[1])
    with torch.no_grad():
        x.mul_(0.5)
        y.mul_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    again = _step(m, x.detach(), y)
    assert torch.equal(loss, again[0]) and torch.equal(grad, again[1])


@pytest.mark.gpu
def test_first_call_inside_a_capture_after_moving_the_module():
    """.cuda() uploads the tables, so a module whose first call is inside a CUDA graph capture works."""
    x = torch.from_numpy(_signals(2, 8192, 19)).cuda().requires_grad_(True)
    y = torch.from_numpy(_signals(2, 8192, 20)).cuda()
    eager = _step(_module(FIVE), x.detach(), y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                          # warm the allocator and autograd on the capture stream
        for _ in range(2):
            torch.autograd.grad(_module(FIVE)(x, y), x)
    torch.cuda.current_stream().wait_stream(s)
    m = _module(FIVE).cuda()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = m(x, y)
        grad, = torch.autograd.grad(loss, x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(loss, eager[0]) and torch.equal(grad, eager[1])


@pytest.mark.gpu
def test_nan_filled_outputs_and_workspaces_do_not_leak(monkeypatch):
    m = _module(FIVE)
    x, y = (torch.from_numpy(_signals(4, 8192, s)).cuda() for s in (15, 16))
    clean = _step(m, x, y)
    real = mel_loss._workspace

    def poisoned(nbytes, device):
        return real(nbytes, device).fill_(float("nan"))
    monkeypatch.setattr(mel_loss, "_workspace", poisoned)
    junk = [torch.full((1 << 22,), float("nan"), device="cuda") for _ in range(8)]   # freed blocks the outputs reuse
    del junk
    got = _step(m, x, y)
    assert torch.equal(got[0], clean[0]) and torch.equal(got[1], clean[1])


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["x", "y"])
@pytest.mark.parametrize("value", [float("nan"), float("inf"), -float("inf")])
def test_nan_and_inf_samples_follow_float64(where, value):
    """One NaN or Inf sample: the loss and the gradient are NaN / Inf exactly where float64 autograd's are."""
    B, L = 2, 4096
    x, y = _signals(B, L, 17), _signals(B, L, 18)
    (x if where == "x" else y)[1, 1777] = value
    for res in (((1024,), (256,), (1024,), (80,)), FIVE):
        loss, g = _run(x, y, res)
        ref = float(loss64(torch.from_numpy(x).double(), torch.from_numpy(y).double(), res, **REF))
        assert np.isnan(loss) == np.isnan(ref) and np.isinf(loss) == np.isinf(ref), (loss, ref)
        gref = grad64(x, y, res, **REF)
        assert np.array_equal(np.isnan(g), np.isnan(gref)), (np.isnan(g).sum(), np.isnan(gref).sum())
        assert np.array_equal(np.isposinf(g), np.isposinf(gref)) and np.array_equal(np.isneginf(g), np.isneginf(gref))
        assert np.isfinite(g[0]).all()
