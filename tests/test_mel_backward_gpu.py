"""The mel front end's gradient (csrc/mg_mel.cu mel_backward_*_kernel through meldataset.mel_spectrogram's autograd
Function) against float64 torch autograd of a restatement of the forward, at every option, frame-geometry length and
batch layout, and through the generator.

The float64 reference: zero pad by 384, frames [256 t, 256 t + 1024) of the padded signal, the periodic Hann window,
torch.fft.rfft, |.|, the float64 filter bank of oracle/mel_oracle.py, log(clamp(., 1e-5)); torch.autograd.grad of that
with the same grad_mel.  Each sample i of the kernel's gradient is held to

    |got_i - ref_i| <= sum over the frames t reading i of  w_n (sum_k dG_k + TAU_B ||dmag||_2)  +  5 u sum_t |dframe_t,n|

where, per frame, dG_k = sum_m M_mk dgs_m + 3 u sum_m M_mk |gs_m| + |dmag_k| min(2, TAU_F |x_w|_2 / |X_k| + 4 u) carries
the error of gs_m = g_m / s_m (s_m off by the forward's own bound TAU_F |x_w|_2 sum_k M_mk + (kc_m + 2) u s_m, so
dgs_m = |g_m| ds_m / (s_m (s_m - ds_m)); the whole |g_m| / 1e-5 where the clamp could fall either way) and of the phasor
X_k / |X_k| (the FFT's error over |X_k|), and TAU_B ||dmag||_2 is the inverse FFT's own rounding, the forward's TAU_F
on its input's norm.  Where the bound is 0 (no frame reading i has a nonzero grad_mel) got must be exactly 0.
test_bound_calibration_on_emulated_backward checks both sides on the CPU with a float32 emulation of the kernels,
operation for operation: the emulation stays below 0.5 of the bound, and each deliberately wrong variant (no window,
doubled interior bins, overlap-add one hop off, the clamp ignored, the first or the last frame dropped) exceeds it >= 8x.
"""
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import meldataset, models, synth
from oracle import mel_oracle as mo
from kernel_model import DEFAULT, NORMS, mel_option_cases

TAU_F = 2.0 ** -17
TAU_B = 2.0 ** -17
U = 2.0 ** -24
CLIP = 1e-5
NFFT, HOP, PAD = 1024, 256, 384
WIN64 = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / NFFT)   # periodic Hann
F32 = np.float32


# ------------------------------------------------------------------------------------------------------------------
# float64: torch autograd of the restated forward, and the bound's ingredients
# ------------------------------------------------------------------------------------------------------------------
def fbank(opts):
    sr, n_mels, fmin, fmax, norm = opts
    return mo.mel_filterbank64(sr, NFFT, n_mels, fmin, fmax, NORMS[norm])


def mel_graph64(y, fb):
    """log-mel [B, n_mels, T] of float64 y [B, L] through stock torch ops (autograd builds the reference's graph)."""
    T = y.shape[-1] // HOP
    frames = F.pad(y, (PAD, PAD)).unfold(-1, NFFT, HOP)[:, :T]
    mag = torch.fft.rfft(frames * torch.from_numpy(WIN64).to(y), dim=-1).abs()
    return torch.log(torch.clamp(torch.einsum("mk,btk->bmt", torch.from_numpy(fb).to(y), mag), min=CLIP))


def grad64(y, gmel, fb):
    """d loss / d y in float64 for y [B, L], gmel [B, n_mels, T] (numpy)."""
    yt = torch.from_numpy(np.asarray(y, np.float64)).requires_grad_(True)
    mel = mel_graph64(yt, fb)
    return torch.autograd.grad(mel, yt, torch.from_numpy(np.asarray(gmel, np.float64)))[0].numpy()


def frames_of(y):
    T = len(y) // HOP
    yp = np.pad(np.asarray(y, np.float64), (PAD, PAD))
    return yp[HOP * np.arange(T)[:, None] + np.arange(NFFT)[None, :]]


def overlap_add(dframe, L):
    """sum over frames of [T, 1024] per-frame gradients onto the unpadded signal (padding dropped)."""
    T = dframe.shape[0]
    out = np.zeros(L + 2 * PAD)
    for t in range(T):
        out[HOP * t:HOP * t + NFFT] += dframe[t]
    return out[PAD:PAD + L]


def adjoint64(y, gmel, fb):
    """The gradient by the adjoint written out in float64 (numpy), and the error bound of each sample."""
    xw = frames_of(y) * WIN64                        # [T, 1024]
    X = np.fft.rfft(xw, axis=1)                      # [T, 513]
    mag = np.abs(X)
    s = fb @ mag.T                                   # [n_mels, T]
    g = np.asarray(gmel, np.float64)
    live = s >= CLIP
    gs = np.where(live, g / np.where(live, s, 1.0), 0.0)
    dmag = fb.T @ gs                                 # [513, T]
    phase = np.where(mag > 0, X / np.where(mag > 0, mag, 1.0), 0.0)
    G = dmag.T * phase                               # [T, 513]
    full = np.zeros((G.shape[0], NFFT), complex)
    full[:, :513] = G
    dframe = WIN64 * (np.fft.ifft(full, axis=1).real * NFFT)
    # the bound
    xn = np.sqrt((xw * xw).sum(axis=1))              # [T]
    sw = fb.sum(axis=1)[:, None]
    kc = (fb > 0).sum(axis=1)[:, None]
    ds = TAU_F * xn[None, :] * sw + (kc + 2) * U * s
    ag = np.abs(g)
    above = s - ds >= CLIP
    below = s + ds < CLIP
    with np.errstate(divide="ignore", invalid="ignore"):
        dgs = np.where(above, ag * ds / (s * np.maximum(s - ds, CLIP)) + 2 * U * ag / np.maximum(s, CLIP), 0.0)
    dgs = np.where(~above & ~below, ag / CLIP, dgs)
    ddmag = fb.T @ dgs + 3 * U * (fb.T @ np.abs(gs))           # [513, T]
    with np.errstate(divide="ignore"):
        dph = np.minimum(2.0, np.where(mag > 0, TAU_F * xn[:, None] / mag, 2.0) + 4 * U)
    dG = ddmag.T + np.abs(dmag.T) * dph                        # [T, 513]
    per_frame = dG.sum(axis=1) + TAU_B * np.sqrt((dmag * dmag).sum(axis=0))
    dfr = WIN64[None, :] * per_frame[:, None] + 5 * U * np.abs(dframe)
    return overlap_add(dframe, len(y)), overlap_add(dfr, len(y))


def bound_ratio(got, ref, bound):
    """Worst |got - ref| / bound; where the bound is 0, got must be exactly 0."""
    got = np.asarray(got, np.float64)
    assert not np.isnan(got).any(), "NaN in the gradient"
    zero = bound == 0
    assert (got[zero] == 0).all(), "a sample no live frame reaches is not exactly 0"
    return float((np.abs(got - ref)[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0


def check_item(got, y, gmel, opts, fb=None):
    fb = fbank(opts) if fb is None else fb
    ref = grad64(y[None], gmel[None], fb)[0]
    man, bound = adjoint64(y, gmel, fb)
    assert np.abs(man - ref).max() <= 1e-7 * (np.abs(ref).max() + 1e-300), "the written-out adjoint left autograd"
    return bound_ratio(got, ref, bound)


# ------------------------------------------------------------------------------------------------------------------
# the bound, calibrated on the CPU against a float32 emulation of the kernels
# ------------------------------------------------------------------------------------------------------------------
def _f(x):
    return np.asarray(x, F32)


def _stockham(re, im, twr, twi):
    ns, j = 1, np.arange(256)
    while ns < 512:
        kk = j & (ns - 1)
        wr, wi = twr[kk * (512 // ns)], twi[kk * (512 // ns)]
        ar, ai = re[:, j + 256], im[:, j + 256]
        v1r, v1i = ar * wr - ai * wi, ar * wi + ai * wr
        j0 = ((j - kk) << 1) + kk
        nr, ni = np.empty_like(re), np.empty_like(im)
        nr[:, j0], ni[:, j0] = re[:, j] + v1r, im[:, j] + v1i
        nr[:, j0 + ns], ni[:, j0 + ns] = re[:, j] - v1r, im[:, j] - v1i
        re, im, ns = nr, ni, ns << 1
    return re, im


def _fma_acc(acc, w, v):
    return _f(np.asarray(w, np.float64) * np.asarray(v, np.float64) + acc.astype(np.float64))


def emulate_backward(y, gmel, fb32, window=True, double_interior=False, ola_shift=0, ignore_clamp=False, drop=None):
    """The two backward kernels' arithmetic in float32 for one waveform y [L] and gmel [n_mels, T]; the keyword
    arguments select the wrong variants."""
    k = np.arange(NFFT // 2)
    twr, twi = _f(np.cos(2 * np.pi * k / NFFT)), _f(-np.sin(2 * np.pi * k / NFFT))
    win = _f(WIN64)
    x = _f(frames_of(y))
    n_fr = x.shape[0]
    re, im = _stockham(x[:, 0::2] * win[0::2], x[:, 1::2] * win[1::2], twr, twi)
    kb = np.arange(513)
    zr, zi = re[:, kb & 511], im[:, kb & 511]
    cr, ci = re[:, (512 - kb) & 511], im[:, (512 - kb) & 511]
    h = F32(0.5)
    er, ei = h * (zr + cr), h * (zi - ci)
    orr, oi = h * (zi + ci), -h * (zr - cr)
    wr = np.where(kb < 512, twr[np.minimum(kb, 511)], F32(-1))
    wi = np.where(kb < 512, twi[np.minimum(kb, 511)], F32(0))
    xr, xi = er + wr * orr - wi * oi, ei + wr * oi + wi * orr
    mag = np.sqrt(xr * xr + xi * xi)                                   # [T, 513]
    n_mels = fb32.shape[0]
    s = np.zeros((n_mels, n_fr), F32)
    for kk in range(513):
        nz = fb32[:, kk] != 0
        if nz.any():
            s[nz] = _fma_acc(s[nz], fb32[nz, kk][:, None], mag[None, :, kk])
    g = _f(gmel)
    live = (s >= F32(CLIP)) | ignore_clamp
    gs = np.where(live, g / np.where(s != 0, s, F32(1)), F32(0)).astype(F32)
    dm = np.zeros((n_fr, 513), F32)
    for par in (0, 1):   # even filters, then odd ones; within a parity no bin is shared
        for kk in range(513):
            rows = [m for m in range(par, n_mels, 2) if fb32[m, kk] != 0]
            if rows:
                dm[:, kk] = _fma_acc(dm[:, kk], fb32[rows[0], kk], gs[rows[0]])
    r = np.where(mag > 0, dm / np.where(mag > 0, mag, F32(1)), F32(0)).astype(F32)
    gr, gi = r * xr, r * xi
    if double_interior:
        gr[:, 1:512] *= 2
        gi[:, 1:512] *= 2

    def conj_a(Gr, Gi, cw, sw):   # split_adjoint: conj(a) G
        return h * (Gr + sw * Gr - cw * Gi), h * (Gi + cw * Gr + sw * Gi)

    def b_conj(Gr, Gi, cw, sw):   # split_adjoint_conj: b conj(G)
        return h * (Gr - sw * Gr + cw * Gi), h * (-Gi + cw * Gr + sw * Gi)
    j = np.arange(512)
    jc = (512 - j) & 511
    pr, pi = conj_a(gr[:, j], gi[:, j], twr[j], twi[j])
    qr, qi = b_conj(gr[:, jc], gi[:, jc], twr[jc], twi[jc])
    dr, di = pr + qr, pi + qi
    p5r, p5i = conj_a(gr[:, 512], gi[:, 512], F32(-1), F32(0))
    q5r, q5i = b_conj(gr[:, 512], gi[:, 512], F32(-1), F32(0))
    dr[:, 0] += p5r + q5r
    di[:, 0] += p5i + q5i
    zr, zi = _stockham(dr, di, twr, -twi)
    dframe = np.empty((n_fr, NFFT), F32)
    w = win if window else np.ones(NFFT, F32)
    dframe[:, 0::2], dframe[:, 1::2] = w[0::2] * zr, w[1::2] * zi
    if drop is not None:
        dframe[drop] = 0
    L = len(y)
    out = np.zeros(L, F32)
    for i in range(L):
        p = i + PAD
        for t in range(max(0, (p - NFFT) // HOP + 1), min(p // HOP, n_fr - 1) + 1):
            tt = t + ola_shift
            if 0 <= tt < n_fr and 0 <= p - HOP * tt < NFFT:
                out[i] += dframe[tt, p - HOP * tt]
    return out


def _calibration_signals():
    """Noise, a tone mix, a quiet signal with a near-silent middle (bands below the clip) and a square wave."""
    rs = np.random.RandomState(11)
    L = 2600
    t = np.arange(L) / 22050.0
    quiet = rs.standard_normal(L) * 1e-3
    quiet[800:1900] *= 1e-5
    sig = [rs.uniform(-1, 1, L) * 0.9,
           0.4 * np.sin(2 * np.pi * 220 * t) + 0.3 * np.sin(2 * np.pi * 3000 * t + 1),
           quiet,
           np.sign(np.sin(2 * np.pi * 441 * t + 0.5))]
    return [_f(s) for s in sig]


def _wrong_variants():
    return {"no window": dict(window=False), "doubled interior bins": dict(double_interior=True),
            "overlap-add one hop late": dict(ola_shift=1), "clamp ignored": dict(ignore_clamp=True),
            "first frame dropped": dict(drop=0), "last frame dropped": dict(drop=-1)}


@pytest.mark.parametrize("opts", [DEFAULT, (44100, 128, 0.0, 22050.0, 0), (16000, 40, 0.0, 8000.0, 2)])
def test_bound_calibration_on_emulated_backward(opts):
    fb = fbank(opts)
    fb32 = fb.astype(F32)
    rs = np.random.RandomState(3)
    good, wrong = 0.0, {}
    for y in _calibration_signals():
        T = len(y) // HOP
        gmel = _f(rs.standard_normal((opts[1], T)))
        ref, bound = adjoint64(y, gmel, fb)
        good = max(good, bound_ratio(emulate_backward(y, gmel, fb32), ref, bound))
        for name, v in _wrong_variants().items():
            r = np.abs(emulate_backward(y, gmel, fb32, **v).astype(np.float64) - ref) / np.maximum(bound, 1e-300)
            wrong[name] = max(wrong.get(name, 0.0), float(r.max()))
    print("\n%s: emulation %.3f of the bound; wrong variants: %s" % (
        opts, good, ", ".join("%s %.1f" % kv for kv in wrong.items())))
    assert good < 0.5, good
    assert min(wrong.values()) >= 8, wrong


def test_written_out_adjoint_equals_float64_autograd():
    """The bound's float64 adjoint (split run backwards, inverse DFT) is torch autograd's gradient, not a second opinion."""
    for opts in (DEFAULT, (16000, 40, 0.0, 8000.0, 2)):
        fb = fbank(opts)
        for y in _calibration_signals():
            gmel = np.random.RandomState(1).standard_normal((opts[1], len(y) // HOP))
            ref = grad64(y[None], gmel[None], fb)[0]
            man, _ = adjoint64(y, gmel, fb)
            assert np.abs(man - ref).max() <= 1e-7 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _signals(L, seed, count=4):
    """Noise, a speech-like signal (a gliding harmonic voice under an envelope with pauses), a quiet signal and a
    full-scale square wave, fp32 in [-1, 1]."""
    rs = np.random.RandomState(seed)
    t = np.arange(L) / 22050.0
    f0 = 120 + 40 * np.sin(2 * np.pi * 3 * t)
    phase = 2 * np.pi * np.cumsum(f0) / 22050.0
    voice = sum(np.sin(h * phase) / h for h in range(1, 12)) * np.clip(np.sin(2 * np.pi * 4 * t), 0, None) * 0.5
    sig = [rs.uniform(-1, 1, L) * 0.9,
           voice + 0.003 * rs.standard_normal(L),
           rs.standard_normal(L) * 1e-4,
           np.sign(np.sin(2 * np.pi * 441 * t + 0.5))]
    return np.clip(np.stack(sig[:count]), -1, 1).astype(np.float32)


def gpu_grad(y, gmel, opts, dtype=torch.float32):
    """d loss / d y through mel_spectrogram's autograd Function: (grad [B, L] numpy, mel)."""
    sr, n_mels, fmin, fmax, norm = opts
    yt = torch.from_numpy(np.asarray(y)).to("cuda", dtype).requires_grad_(True)
    mel = meldataset.mel_spectrogram(yt, NFFT, n_mels, sr, HOP, NFFT, fmin, fmax, check_range=False, norm=norm)
    mel.backward(torch.from_numpy(np.asarray(gmel, np.float32)).cuda())
    return yt.grad, mel


def check_batch(y, gmel, opts):
    got = gpu_grad(y, gmel, opts)[0].cpu().numpy()
    fb = fbank(opts)
    return max(check_item(got[i], y[i], gmel[i], opts, fb) for i in range(y.shape[0]))


def abi_backward(tab, y, gmel, out, ws, nbytes=None, stream=None):
    lib = meldataset._lib()
    B, L = y.shape
    nbytes = lib.mg_mel_backward_workspace_bytes(B, L) if nbytes is None else nbytes
    s = (stream or torch.cuda.current_stream()).cuda_stream
    return lib.mg_mel_spectrogram_backward(tab.data_ptr(), y.data_ptr(), gmel.data_ptr(), out.data_ptr(), B, L,
                                           ws.data_ptr(), nbytes, s)


def workspace(B, L):
    return torch.empty(meldataset._lib().mg_mel_backward_workspace_bytes(B, L) // 4, device="cuda")


@pytest.mark.gpu
def test_option_sweep_against_float64():
    """Sampling rates, 1 - 128 mels, norm none / Slaney / L1, fmin 0 / 55, fmax 8000 / 9000 / sr/2; random grad_mel."""
    worst = 0.0
    for i, opts in enumerate(mel_option_cases()):
        L = 4096 + 77 * i
        y = _signals(L, 200 + i)
        gmel = np.random.RandomState(i).standard_normal((4, opts[1], L // HOP)).astype(np.float32)
        r = check_batch(y, gmel, opts)
        assert r <= 1, (opts, r)
        worst = max(worst, r)
    print("\noption sweep (%d settings): worst %.3f of the bound" % (len(mel_option_cases()), worst))


@pytest.mark.gpu
def test_one_hot_grad_mel_on_single_frames_and_bands():
    """grad_mel one-hot at the first, a middle and the last frame, on the first, a middle and the last band: within the
    bound, and exactly 0 on every sample the frame does not read."""
    L = 4096 + 100
    T = L // HOP
    y = _signals(L, 7)
    worst = 0.0
    for t in (0, T // 2, T - 1):
        for m in (0, 40, 79):
            gmel = np.zeros((4, 80, T), np.float32)
            gmel[:, m, t] = 1.0
            got = gpu_grad(y, gmel, DEFAULT)[0].cpu().numpy()
            lo, hi = max(0, HOP * t - PAD), min(L, HOP * t - PAD + NFFT)
            assert (got[:, :lo] == 0).all() and (got[:, hi:] == 0).all(), (t, m)
            worst = max(worst, max(check_item(got[i], y[i], gmel[i], DEFAULT) for i in range(4)))
    print("\none-hot: worst %.3f of the bound" % worst)
    assert worst <= 1, worst


def _geometry_lengths():
    """The first length with a frame and around it, lengths of 2, 4 and 32 frames -1 / 0 / +1 sample, a length
    whose frames all read both pads, and a long odd length."""
    return [256, 257, 511, 512, 513, 639, 767, 768, 1023, 1024, 1025, 8191, 8192, 8193, 23457]


def test_every_sample_is_read_by_a_frame():
    """With T = floor(L / 256) frames the last one ends 384 samples past 256 T > L - 1: no sample of the signal is left
    unread, so the trailing L mod 256 samples get the last frames' gradients, and a sample is exactly 0 only where
    every frame reading it has a zero grad_mel (test_one_hot_grad_mel_on_single_frames_and_bands)."""
    for L in _geometry_lengths():
        T = L // HOP
        assert HOP * (T - 1) + NFFT - PAD >= L


@pytest.mark.gpu
@pytest.mark.parametrize("L", _geometry_lengths())
def test_frame_geometry_lengths_against_float64(L):
    y = _signals(L, L)
    gmel = np.random.RandomState(L).standard_normal((4, 80, L // HOP)).astype(np.float32)
    r = check_batch(y, gmel, DEFAULT)
    print("L=%d (T=%d): %.3f of the bound" % (L, L // HOP, r))
    assert r <= 1, (L, r)


@pytest.mark.gpu
def test_clamp_floor_silence_and_bands_below_the_clip():
    """A silent item's gradient is exactly 0 (no NaN from 0 / 0); a faint low tone leaves its high bands below the clip
    next to live low bands: a grad_mel on the clipped bands alone gives exactly 0, and the mixed case meets float64."""
    L = 4096
    T = L // HOP
    t = np.arange(L) / 22050.0
    tone = (1e-3 * np.sin(2 * np.pi * 200 * t)).astype(np.float32)
    y = np.stack([np.zeros(L, np.float32), tone])
    gmel = np.random.RandomState(5).standard_normal((2, 80, T)).astype(np.float32)
    grad, mel = gpu_grad(y, gmel, DEFAULT)
    got = grad.cpu().numpy()
    assert (got[0] == 0).all()
    floor = mel.detach()[0, 0, 0]
    clipped = (mel.detach()[1] == floor).cpu().numpy()
    assert clipped.sum() >= 10 * T and (~clipped).sum() >= 5 * T, clipped.sum()
    assert check_item(got[1], y[1], gmel[1], DEFAULT) <= 1
    only = np.where(clipped, gmel[1], 0).astype(np.float32)
    got = gpu_grad(y[1:], only[None], DEFAULT)[0].cpu().numpy()
    assert (got == 0).all()


@pytest.mark.gpu
def test_calls_are_deterministic_and_items_equal_their_own_calls():
    """Two calls are bit-identical; each item of a B = 37 batch equals its own B = 1 call bit for bit; a grad_audio
    pre-filled with NaN (with a guard tail) is fully overwritten and nothing past it is touched."""
    B, L = 37, 8192 + 300
    rs = np.random.RandomState(37)
    y = np.concatenate([_signals(L, i) for i in range(10)])[:B]
    gmel = rs.standard_normal((B, 80, L // HOP)).astype(np.float32)
    a = gpu_grad(y, gmel, DEFAULT)[0]
    b = gpu_grad(y, gmel, DEFAULT)[0]
    assert torch.equal(a, b)
    for i in range(B):
        assert torch.equal(a[i], gpu_grad(y[i:i + 1], gmel[i:i + 1], DEFAULT)[0][0]), i
    tab = meldataset._tables(torch.device("cuda", torch.cuda.current_device()), *DEFAULT)
    yt, gt = torch.from_numpy(y).cuda(), torch.from_numpy(gmel).cuda()
    out = torch.full((B * L + 4096,), float("nan"), device="cuda")
    assert abi_backward(tab, yt, gt, out, workspace(B, L)) == 0
    assert not out[:B * L].isnan().any() and out[B * L:].isnan().all()
    assert torch.equal(out[:B * L].view(B, L), a)


@pytest.mark.gpu
def test_batch_beyond_65535_items():
    """70 000 one-frame items: equal to the same items in batches of at most 65 535; sampled items equal their own
    call and meet float64."""
    B, L = 70000, 300
    rs = np.random.RandomState(70000)
    y = (rs.uniform(-1, 1, (B, L)) * rs.uniform(0, 1, (B, 1))).astype(np.float32)
    gmel = rs.standard_normal((B, 80, 1)).astype(np.float32)
    got = gpu_grad(y, gmel, DEFAULT)[0]
    parts = torch.cat([gpu_grad(y[s:s + 65535], gmel[s:s + 65535], DEFAULT)[0] for s in range(0, B, 65535)])
    assert torch.equal(got, parts)
    sample = [0, 1, 65534, 65535, 65536, B - 2, B - 1] + list(rs.randint(0, B, 9))
    fb = fbank(DEFAULT)
    worst = 0.0
    for i in sample:
        own = gpu_grad(y[i:i + 1], gmel[i:i + 1], DEFAULT)[0][0]
        assert torch.equal(got[i], own), i
        worst = max(worst, check_item(own.cpu().numpy(), y[i], gmel[i], DEFAULT, fb))
    print("\nB=70000: sampled items %.3f of the bound" % worst)
    assert worst <= 1, worst


# ------------------------------------------------------------------------------------------------------------------
# autograd wiring
# ------------------------------------------------------------------------------------------------------------------
ARGS = (NFFT, 80, 22050, HOP, NFFT, 55.0, 9000.0)


@pytest.mark.gpu
def test_one_and_two_dimensional_inputs_and_float64_leaves():
    L = 8192
    y = _signals(L, 3)
    gmel = np.random.RandomState(3).standard_normal((4, 80, L // HOP)).astype(np.float32)
    batch = gpu_grad(y, gmel, DEFAULT)[0]
    for i in range(4):
        one = torch.from_numpy(y[i]).cuda().requires_grad_(True)
        mel = meldataset.mel_spectrogram(one, *ARGS, check_range=False)
        assert mel.shape == (80, L // HOP)
        mel.backward(torch.from_numpy(gmel[i]).cuda())
        assert one.grad.shape == (L,) and torch.equal(one.grad, batch[i])
    g64, _ = gpu_grad(y, gmel, DEFAULT, dtype=torch.float64)
    assert g64.dtype == torch.float64 and torch.equal(g64, batch.double())


@pytest.mark.gpu
def test_gradients_accumulate_and_forward_bits_do_not_depend_on_grad():
    L = 8192 + 55
    y = torch.from_numpy(_signals(L, 9)).cuda()
    off = meldataset.mel_spectrogram(y, *ARGS, check_range=False)
    leaf = y.clone().requires_grad_(True)
    on = meldataset.mel_spectrogram(leaf, *ARGS)
    assert on.grad_fn is not None and off.grad_fn is None
    assert torch.equal(on.detach(), off)
    with torch.no_grad():
        assert torch.equal(meldataset.mel_spectrogram(leaf, *ARGS, check_range=False), off)
    g = torch.randn(on.shape, generator=torch.Generator().manual_seed(1)).cuda()
    on.backward(g)
    first = leaf.grad.clone()
    meldataset.mel_spectrogram(leaf, *ARGS).backward(g)
    assert torch.equal(leaf.grad, 2 * first)
    # an L1 loss through squeeze and a dtype cast reaches the leaf
    leaf.grad = None
    F.l1_loss(meldataset.mel_spectrogram(leaf.double()[:1].squeeze(0), *ARGS), off[0].double() + 0.5).backward()
    assert leaf.grad is not None and (leaf.grad[1:] == 0).all() and leaf.grad[0].abs().max() > 0


@pytest.mark.gpu
def test_backward_is_captured_and_replayed_in_a_cuda_graph():
    L = 8192
    y = torch.from_numpy(_signals(L, 4)).cuda().requires_grad_(True)
    g = torch.randn((4, 80, L // HOP), generator=torch.Generator().manual_seed(2)).cuda()
    meldataset.mel_spectrogram(y, *ARGS)                 # tables uploaded, library loaded
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):                               # warm the allocator's pool on this stream
            y.grad = None
            meldataset.mel_spectrogram(y, *ARGS, check_range=False).backward(g)
    torch.cuda.current_stream().wait_stream(s)
    eager = y.grad.clone()
    graph = torch.cuda.CUDAGraph()
    y.grad = None
    with torch.cuda.graph(graph):
        mel = meldataset.mel_spectrogram(y, *ARGS, check_range=False)
        grad, = torch.autograd.grad(mel, y, g)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(grad, eager)
    with torch.no_grad():
        y.mul_(0.5)
        g.mul_(-1.0)
    graph.replay()
    torch.cuda.synchronize()
    y.grad = None
    meldataset.mel_spectrogram(y, *ARGS, check_range=False).backward(g)
    assert torch.equal(grad, y.grad)


@pytest.mark.gpu
def test_two_streams_run_backward_at_once_and_match_serial():
    L = 22050 * 2
    ys = [torch.from_numpy(_signals(L, 40 + k)).cuda() for k in range(2)]
    gs = [torch.randn((4, 80, L // HOP), generator=torch.Generator().manual_seed(k)).cuda() for k in range(2)]

    def run(k):
        leaf = ys[k].clone().requires_grad_(True)
        meldataset.mel_spectrogram(leaf, *ARGS, check_range=False).backward(gs[k])
        return leaf.grad

    serial = [run(k) for k in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    out = [None, None]

    def worker(k):
        with torch.cuda.stream(streams[k]):
            for _ in range(5):
                out[k] = run(k)

    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    threads = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(out[k], serial[k]), k


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


def _gen_params(gen):
    vs, gs, bs = gen._param_triplets()
    return [t for trip in zip(vs, gs, bs) for t in trip]


@pytest.mark.gpu
def test_mel_l1_loss_trains_the_generator(ieee_deterministic):
    """B x T = 2 x 16: the parameter gradients of L1(mel(G(x)), x) through the engine equal those of feeding the same
    generator backward the float64 reference's audio gradient (cast to fp32), within the generator backward's own
    tolerance.  The L1 term's sign is taken from the kernel's mel, as a float64 forward could disagree only where
    mel = x, which says nothing about the mel gradient."""
    from conftest import rel_errors
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    gen = gen.cuda().train()
    x = torch.from_numpy(synth.mel_input(2, 16, 5)).cuda()
    y = gen(x)
    mel = meldataset.mel_spectrogram(y.squeeze(1), *ARGS, check_range=False)
    assert mel.shape == x.shape
    gen.zero_grad()
    F.l1_loss(mel, x).backward()
    got = [p.grad.clone() for p in _gen_params(gen)]
    assert all(g is not None and g.abs().max() > 0 for g in got)
    # the float64 reference's audio gradient for the same upstream sign(mel - x) / N
    gmel = (torch.sign(mel.detach() - x) / x.numel()).cpu().numpy()
    audio = y.detach().squeeze(1).cpu().numpy()
    g_audio = grad64(audio, gmel, fbank(DEFAULT))
    gen.zero_grad()
    y = gen(x)
    y.backward(torch.from_numpy(g_audio).float().cuda()[:, None, :])
    ref = [p.grad.clone() for p in _gen_params(gen)]
    worst = 0.0
    for i, (a, r) in enumerate(zip(got, ref)):
        m, l2 = rel_errors(a.cpu().numpy(), r.cpu().numpy())
        worst = max(worst, m / TAU_IEEE[0], l2 / TAU_IEEE[1])
        assert m <= TAU_IEEE[0] and l2 <= TAU_IEEE[1], (i, m, l2)
    print("\nmel L1 through the generator: worst %.3f of the tolerance" % worst)
