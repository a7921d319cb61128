"""The multi-resolution STFT loss (csrc/mg_stft_loss.cu through stft_loss.MultiResolutionSTFTLoss) against float64
autograd of its definition, run on the CPU through torch.stft, at every supported n_fft, window and hop shape, and
through the generator; then determinism, concurrency, CUDA-graph replay, no host sync, poisoned buffers and NaN / Inf.

Error model.  Per frame f of a signal, E_f = TAU_F ||w . frame_f||_2 is taken as the error of each bin the fp32 FFT
computes, hence of each clamped magnitude (clamp and |.| are 1-Lipschitz).  This is a per-bin RMS model, not a rigorous
worst case: the radix-2 FFT's normwise bound ||dZ||_2 <= c log2(M) u ||Z||_2 = c log2(M) u sqrt(M) ||z||_2 spreads over
M bins, so TAU_F = 2^-17 = 128 u covers c log2(M) u per bin on average at M <= 1024, while a single bin's rigorous
bound carries a further factor of up to sqrt(M).  The error propagation below is worst-case given that model.  A float32
torch.stft implementation of the loss stays under 0.35 of the bound on this file's signals.  With
lo = max(m - E, sqrt(1e-7)) the smallest magnitude either side can hold:

  loss values   d||y_mag - x_mag|| <= sqrt(sum (E_x + E_y)^2) + 16 u ||.||,  d||y_mag|| <= sqrt(sum E_y^2) + 16 u ||.||,
                d sc_r <= (d num + sc_r d den) / (den - d den) + 4 u sc_r,
                d mag_r <= mean(E_x / lo_x + E_y / lo_y + 2 u (|log x_mag| + |log y_mag|)) + 16 u mag_r,
                and the bound of each loss is the mean over resolutions plus 2 u of the loss.
  gradient      with A = g_sc / (R num den), C = g_mag / (R B T (N/2 + 1)), per bin
                dG <= |A| ((E_x + E_y) + |y_mag - x_mag| (2 E_x / lo_x + dA)) + |C| (2 E_x / lo_x^2 + 8 u / x_mag)
                      + 2 |C| / lo_x                                  where |log y_mag - log x_mag| <= dlog (sign unsure)
                      + |A| (|y_mag - x_mag| + E_x + E_y) + |C| / lo_x  where | |X|^2 - 1e-7 | <= 2 |X| E_x + E_x^2
                (dA = d num / num + d den / den + 8 u); per frame S_f = 2 sum_k dG_k + 2 TAU_F sqrt(N/2) ||G||_2
                + 72 u sum_k |G_k| (the propagated error, at most 2 per unit input through the split's adjoint and the
                inverse FFT, the inverse FFT's own rounding, and the windowing, gather and resolution sums), and
                bound_i = sum over resolutions and over the frame positions reading sample i, reflected copies
                included, of |w_n| S_f.
The module prints the worst ratio |got - ref| / bound seen for each case.
"""
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import models, stft_loss, synth

U = 2.0 ** -24
TAU_F = 2.0 ** -17
FLOOR = 1e-7
DEFAULT = ((1024, 2048, 512), (120, 240, 50), (600, 1200, 240))
WORST = {}


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst ratios to the bound: " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))


# ------------------------------------------------------------------------------------------------------------------
# float64: the definition through torch.stft, and the bound's ingredients
# ------------------------------------------------------------------------------------------------------------------
def _mag64(x, n, h, w):
    X = torch.stft(x, n, h, w, torch.hann_window(w, dtype=torch.float64), center=True, pad_mode="reflect",
                   return_complex=True)
    return torch.sqrt(torch.clamp(X.real ** 2 + X.imag ** 2, min=FLOOR)).transpose(2, 1)


def loss64(x, y, res):
    """(sc, mag) of float64 tensors x, y [B, L] as Parallel WaveGAN states them."""
    sc = mag = 0.0
    for n, h, w in zip(*res):
        xm, ym = _mag64(x, n, h, w), _mag64(y, n, h, w)
        sc = sc + torch.norm(ym - xm, p="fro") / torch.norm(ym, p="fro")
        mag = mag + F.l1_loss(torch.log(ym), torch.log(xm))
    return sc / len(res[0]), mag / len(res[0])


def _frames64(x, n, h, w):
    """Windowed frames [B, T, n] of float64 x as torch.stft forms them, and the window."""
    win = F.pad(torch.hann_window(w, dtype=torch.float64), ((n - w) // 2, n - w - (n - w) // 2))
    fr = F.pad(x[:, None], (n // 2, n // 2), mode="reflect")[:, 0].unfold(-1, n, h)
    return fr * win, win


def _fold(vals, B, L, n, h):
    """Sum of nonnegative per-frame-position values [B, T, n] onto the samples they read, reflections included."""
    z = torch.zeros(B, L, dtype=torch.float64, requires_grad=True)
    fr = F.pad(z[:, None], (n // 2, n // 2), mode="reflect")[:, 0].unfold(-1, n, h)
    return torch.autograd.grad(fr, z, vals)[0]


def _res_terms(x, y, n, h, w):
    xw, win = _frames64(x, n, h, w)
    yw, _ = _frames64(y, n, h, w)
    X, Y = torch.fft.rfft(xw), torch.fft.rfft(yw)
    Ex = TAU_F * xw.norm(dim=-1, keepdim=True)
    Ey = TAU_F * yw.norm(dim=-1, keepdim=True)
    x2, y2 = X.abs() ** 2, Y.abs() ** 2
    xm, ym = torch.sqrt(torch.clamp(x2, min=FLOOR)), torch.sqrt(torch.clamp(y2, min=FLOOR))
    lo_x = torch.clamp(xm - Ex, min=FLOOR ** 0.5)
    lo_y = torch.clamp(ym - Ey, min=FLOOR ** 0.5)
    lx, ly = torch.log(xm), torch.log(ym)
    dlog = Ex / lo_x + Ey / lo_y + 2 * U * (lx.abs() + ly.abs())
    num, den = torch.norm(ym - xm), torch.norm(ym)
    dnum = torch.sqrt(((Ex + Ey) ** 2).expand_as(xm).sum()) + 16 * U * num
    dden = torch.sqrt((Ey ** 2).expand_as(ym).sum()) + 16 * U * den
    return dict(X=X, x2=x2, xm=xm, ym=ym, lx=lx, ly=ly, Ex=Ex, Ey=Ey, lo_x=lo_x, dlog=dlog, num=num, den=den, dnum=dnum,
                dden=dden, win=win)


def value_bounds(x, y, res):
    bsc = bmag = 0.0
    for n, h, w in zip(*res):
        t = _res_terms(x, y, n, h, w)
        sc = t["num"] / t["den"]
        bsc += (t["dnum"] + sc * t["dden"]) / (t["den"] - t["dden"]) + 4 * U * sc
        mag = (t["ly"] - t["lx"]).abs().mean()
        bmag += t["dlog"].mean() + 16 * U * mag
    sc, mag = loss64(x, y, res)
    R = len(res[0])
    return float(bsc / R + 2 * U * sc), float(bmag / R + 2 * U * mag)


def grad_bound(x, y, res, gsc, gmag):
    B, L = x.shape
    R = len(res[0])
    out = torch.zeros(B, L, dtype=torch.float64)
    for n, h, w in zip(*res):
        t = _res_terms(x, y, n, h, w)
        T = t["X"].shape[1]
        A = 0.0 if float(t["num"]) == 0.0 else gsc / (R * float(t["num"]) * float(t["den"]))
        C = gmag / (R * B * T * (n // 2 + 1))
        dA = (float(t["dnum"] / t["num"]) if A else 0.0) + float(t["dden"] / t["den"]) + 8 * U
        xm, ym, Ex, Ey, lo_x = t["xm"], t["ym"], t["Ex"], t["Ey"], t["lo_x"]
        diff = (ym - xm).abs()
        on = t["x2"] >= FLOOR
        sg = torch.sign(t["ly"] - t["lx"])
        G = on * (abs(A) * diff + abs(C) * sg.abs() / xm)
        dG = on * (abs(A) * ((Ex + Ey) + diff * (2 * Ex / lo_x + dA)) + abs(C) * (2 * Ex / lo_x ** 2 + 8 * U / xm))
        dG = dG + ((t["ly"] - t["lx"]).abs() <= t["dlog"]) * 2 * abs(C) / lo_x
        amb = (t["x2"] - FLOOR).abs() <= 2 * t["X"].abs() * Ex + Ex ** 2
        dG = dG + amb * (abs(A) * (diff + Ex + Ey) + abs(C) / lo_x)
        S = 2 * dG.sum(-1) + 2 * TAU_F * (n // 2) ** 0.5 * G.norm(dim=-1) + 72 * U * G.sum(-1)
        out += _fold(t["win"].abs() * S[..., None], B, L, n, h)
    return out.numpy()


def grad64(x, y, res, gsc, gmag):
    xt = torch.from_numpy(x).double().requires_grad_(True)
    sc, mag = loss64(xt, torch.from_numpy(y).double(), res)
    return torch.autograd.grad((sc, mag), xt, (torch.tensor(float(gsc), dtype=torch.float64),
                                               torch.tensor(float(gmag), dtype=torch.float64)))[0].numpy()


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


def _run(x, y, res, gsc=1.0, gmag=1.0, module=None):
    """The kernels' (sc, mag) and d(gsc sc + gmag mag) / dx for numpy x, y."""
    m = module or stft_loss.MultiResolutionSTFTLoss(*res)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    sc, mag = m(xt, torch.from_numpy(y).cuda())
    g, = torch.autograd.grad((sc, mag), xt, (torch.tensor(gsc, device="cuda"), torch.tensor(gmag, device="cuda")))
    return float(sc), float(mag), g.cpu().numpy()


def check(x, y, res, key, grads=((1.0, 1.0), (1.0, 0.0), (0.0, 1.0))):
    x64, y64 = torch.from_numpy(x).double(), torch.from_numpy(y).double()
    sc_ref, mag_ref = (float(v) for v in loss64(x64, y64, res))
    bsc, bmag = value_bounds(x64, y64, res)
    m = stft_loss.MultiResolutionSTFTLoss(*res)
    for gsc, gmag in grads:
        sc, mag, g = _run(x, y, res, gsc, gmag, m)
        assert abs(sc - sc_ref) <= bsc and abs(mag - mag_ref) <= bmag, (sc, sc_ref, bsc, mag, mag_ref, bmag)
        _note(key + " sc", abs(sc - sc_ref) / bsc)
        _note(key + " mag", abs(mag - mag_ref) / bmag)
        ref = grad64(x, y, res, gsc, gmag)
        bound = grad_bound(x64, y64, res, gsc, gmag)
        err = np.abs(g.astype(np.float64) - ref)
        bad = err > bound
        assert not bad.any(), (gsc, gmag, np.argwhere(bad)[:5], err[bad][:5], bound[bad][:5])
        _note(key + " grad", (err / np.maximum(bound, 1e-300)).max())
    return g


# ------------------------------------------------------------------------------------------------------------------
# values and gradients against float64
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_default_resolutions_at_the_config3_shape():
    B, L = 16, 8192
    check(_signals(B, L, 1), _signals(B, L, 2), DEFAULT, "default 16x8192")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 256, 512, 1024, 2048])
def test_each_n_fft_alone(n):
    """win_length = n_fft, and shorter with n_fft - win_length even and odd; hops that divide L and that do not; L from
    n_fft / 2 + 1 (both reflections reach across the whole signal) to long; B of 1 and 16."""
    cases = [(n, n // 4, n // 2 + 1, 1),               # hop does not divide L = n/2 + 1
             (n - 2, n // 8, 4 * n, 16),               # even padding; hop divides L
             (n - 3, n // 4 + 3, 8192 + 5, 3),         # odd padding; hop does not divide L
             (n // 2 + 1, 50, 22050, 1)]               # long L
    for w, h, L, B in cases:
        check(_signals(B, L, 10 + w), _signals(B, L, 20 + h), ((n,), (h,), (w,)), "n_fft %d" % n)


MIXED8 = ((128, 256, 512, 1024, 2048, 512, 1024, 256), (32, 50, 120, 240, 480, 128, 256, 64),
          (128, 200, 512, 600, 1200, 300, 1024, 255))


@pytest.mark.gpu
def test_eight_mixed_resolutions():
    """The most resolutions a call takes: the finish kernel's loop and the gradient's accumulation over resolutions."""
    B, L = 4, 8192
    check(_signals(B, L, 30), _signals(B, L, 31), MIXED8, "8 resolutions")


@pytest.mark.gpu
def test_bins_below_at_and_above_the_clamp_and_silence():
    """Silent stretches, and tones whose bins sit below, around and above |X|^2 = 1e-7, in x and in y."""
    B, L = 2, 8192
    x, y = _signals(B, L, 3), _signals(B, L, 4)
    t = np.arange(1500)
    for a, (lo, hi) in zip((0.0, 2e-7, 6e-7, 2e-6), ((1000, 2500), (3000, 4500), (5000, 6500), (6600, 8100))):
        x[0, lo:hi] = a * np.sin(0.3 * t)
        y[1, lo:hi] = a * np.cos(0.2 * t)
    y[0, 2000:3500] = 0.0
    check(x, y, DEFAULT, "clamp")
    check(x, y, ((512,), (128,), (512,)), "clamp")


@pytest.mark.gpu
def test_equal_signals_give_zero_gradient():
    """x == y: the sc numerator is 0, and float64 autograd gives both terms a gradient of exactly 0."""
    x = _signals(3, 8192, 5)
    sc, mag, g = _run(x, x.copy(), DEFAULT)
    assert sc == 0.0 and mag == 0.0
    assert not g.any()
    for gsc, gmag in ((1.0, 0.0), (0.0, 1.0)):
        assert not _run(x, x.copy(), DEFAULT, gsc, gmag)[2].any()
        assert not grad64(x, x.copy(), DEFAULT, gsc, gmag).any()


@pytest.mark.gpu
def test_reflected_copies_carry_gradient():
    """The first and last n_fft / 2 samples are read twice (directly and through the reflection); a loss that only sees
    the edge frames still meets float64 there."""
    n, h, L = 1024, 256, 1200
    x, y = _signals(2, L, 6), _signals(2, L, 7)
    g = check(x, y, ((n,), (h,), (n,)), "reflect")
    assert np.abs(g[:, 1:n // 2]).min() > 0 and np.abs(g[:, L - 1 - n // 2:L - 1]).min() > 0


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
def test_stft_loss_trains_the_generator(ieee_deterministic):
    """B x T = 2 x 16 mel frames (4096 samples): the parameter and mel gradients of sc + mag of G(x) against seeded target
    audio equal those of feeding the same generator backward the float64 reference's audio gradient (cast to fp32),
    within the generator backward's own tolerance."""
    from conftest import rel_errors
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    gen = gen.cuda().train()
    x = torch.from_numpy(synth.mel_input(2, 16, 5)).cuda().requires_grad_(True)
    target = torch.from_numpy(_signals(2, 4096, 8)).cuda()
    loss = stft_loss.MultiResolutionSTFTLoss()
    y = gen(x)
    sc, mag = loss(y.squeeze(1), target)
    gen.zero_grad()
    (sc + mag).backward()
    params = [p for p in gen.parameters()]
    got = [p.grad.clone() for p in params] + [x.grad.clone()]
    assert all(g is not None and g.abs().max() > 0 for g in got)
    g_audio = grad64(y.detach().squeeze(1).cpu().numpy(), target.cpu().numpy(), DEFAULT, 1.0, 1.0)
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
    sc, mag = m(leaf, y)
    (sc + mag).backward()
    return torch.stack([sc.detach(), mag.detach()]), leaf.grad


@pytest.mark.gpu
def test_repeated_calls_are_bit_identical_and_do_not_sync():
    m = stft_loss.MultiResolutionSTFTLoss()
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
    m = stft_loss.MultiResolutionSTFTLoss()
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
    m = stft_loss.MultiResolutionSTFTLoss()
    x = torch.from_numpy(_signals(4, 8192, 13)).cuda().requires_grad_(True)
    y = torch.from_numpy(_signals(4, 8192, 14)).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            sc, mag = m(x, y)
            torch.autograd.grad(sc + mag, x)
    torch.cuda.current_stream().wait_stream(s)
    eager = _step(m, x.detach(), y)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sc, mag = m(x, y)
        grad, = torch.autograd.grad(sc + mag, x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(torch.stack([sc, mag]), eager[0]) and torch.equal(grad, eager[1])
    with torch.no_grad():
        x.mul_(0.5)
        y.mul_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    again = _step(m, x.detach(), y)
    assert torch.equal(torch.stack([sc, mag]), again[0]) and torch.equal(grad, again[1])


@pytest.mark.gpu
def test_first_call_inside_a_capture_after_moving_the_module():
    """.cuda() uploads the tables, so a module whose first call is inside a CUDA graph capture works."""
    x = torch.from_numpy(_signals(2, 8192, 19)).cuda().requires_grad_(True)
    y = torch.from_numpy(_signals(2, 8192, 20)).cuda()
    eager = _step(stft_loss.MultiResolutionSTFTLoss(), x.detach(), y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                          # warm the allocator and autograd on the capture stream
        for _ in range(2):
            sc, mag = stft_loss.MultiResolutionSTFTLoss()(x, y)
            torch.autograd.grad(sc + mag, x)
    torch.cuda.current_stream().wait_stream(s)
    m = stft_loss.MultiResolutionSTFTLoss().cuda()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sc, mag = m(x, y)
        grad, = torch.autograd.grad(sc + mag, x)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(torch.stack([sc, mag]), eager[0]) and torch.equal(grad, eager[1])


@pytest.mark.gpu
def test_nan_filled_outputs_and_workspaces_do_not_leak(monkeypatch):
    m = stft_loss.MultiResolutionSTFTLoss()
    x, y = (torch.from_numpy(_signals(4, 8192, s)).cuda() for s in (15, 16))
    clean = _step(m, x, y)
    real = stft_loss._workspace

    def poisoned(nbytes, device):
        return real(nbytes, device).fill_(float("nan"))
    monkeypatch.setattr(stft_loss, "_workspace", poisoned)
    junk = [torch.full((1 << 22,), float("nan"), device="cuda") for _ in range(8)]   # freed blocks the outputs reuse
    del junk
    got = _step(m, x, y)
    assert torch.equal(got[0], clean[0]) and torch.equal(got[1], clean[1])


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["x", "y"])
@pytest.mark.parametrize("value", [float("nan"), float("inf")])
def test_nan_and_inf_samples_follow_float64(where, value):
    """One NaN or Inf sample: the losses and the gradient are NaN / Inf exactly where float64 autograd's are."""
    B, L = 2, 4096
    x, y = _signals(B, L, 17), _signals(B, L, 18)
    (x if where == "x" else y)[1, 1777] = value
    for gsc, gmag in ((1.0, 1.0), (1.0, 0.0), (0.0, 1.0)):
        sc, mag, g = _run(x, y, DEFAULT, gsc, gmag)
        x64, y64 = torch.from_numpy(x).double(), torch.from_numpy(y).double()
        sc_ref, mag_ref = (float(v) for v in loss64(x64, y64, DEFAULT))
        for got, ref in ((sc, sc_ref), (mag, mag_ref)):
            assert np.isnan(got) == np.isnan(ref) and np.isinf(got) == np.isinf(ref), (got, ref)
        ref = grad64(x, y, DEFAULT, gsc, gmag)
        assert np.array_equal(np.isnan(g), np.isnan(ref)), (gsc, gmag, np.isnan(g).sum(), np.isnan(ref).sum())
        assert np.array_equal(np.isposinf(g), np.isposinf(ref)) and np.array_equal(np.isneginf(g), np.isneginf(ref))
