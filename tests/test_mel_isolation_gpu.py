"""The mel front end (csrc/mg_mel.cu through meldataset.mel_spectrogram) against a float64 statement of its own
arithmetic, at every option, frame-geometry length and batch layout.

The float64 reference: frames of the zero-padded signal (frame t reads samples [256 t - 384, 256 t + 640)), the float64
periodic Hann window times the frame, np.fft.rfft in float64, |.|, the float64 filter bank of oracle/mel_oracle.py
(mel_filterbank64: Slaney, L1 or none), log(max(., 1e-5)).  For mel band m of frame t the kernel's linear value is held to

    |exp(got) - max(mel64, 1e-5)| <= TAU_F * |x_w|_2 * sum_k w_k  +  (kc_m + 2) 2^-24 mel64  +  (rounding of logf),

with x_w the windowed frame, w_k the band's float64 weights and kc_m its bin count.  The first term is the FFT's error
(fp32 radix-2 passes on table twiddles: a few ulps of the frame's energy in every bin, whatever the bin's own size), the
second the fp32 weights and the fma dot product.  Where mel64 plus the bound is still below the clip, got must be the clip
floor exactly.  test_tau_calibration_on_emulated_mel_kernel checks both sides of TAU_F on the CPU with a float32
emulation of the kernel, operation for operation (Stockham passes, real-transform split, fma dot product): the emulation
uses 0.10 of the bound; twiddles rounded to 11 bits, a symmetric Hann window, a frame shifted by one sample and
bf16 filter weights exceed it by >= 119x.

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s): worst |exp(got) - mel64| as a fraction
of the bound over the option sweep (34 settings) 0.22, over the frame-geometry lengths 0.16, over the sampled items of
the 70 000-item batch 0.04.

What this anchors is the kernel against its own restatement of librosa's algorithm; librosa itself is absent here, so
parity with it stays unpinned (DESIGN.md section 2).
"""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, meldataset
from oracle import mel_oracle as mo
from kernel_model import DEFAULT, NORMS, mel_option_cases

TAU_F = 2.0 ** -17
U = 2.0 ** -24
CLIP = 1e-5
NFFT, HOP, PAD = 1024, 256, 384
WIN64 = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / NFFT)   # periodic Hann


def frames_of(y, shift=0):
    """[T, 1024] frames of one waveform as the kernel reads them (zero outside [0, L))."""
    y = np.asarray(y)
    T = len(y) // HOP
    yp = np.pad(y, (PAD, PAD + 1))
    idx = HOP * np.arange(T)[:, None] + np.arange(NFFT)[None, :] + shift
    return yp[idx]


def mel64(y, sr, n_mels, fmin, fmax, norm):
    """float64 reference of one waveform: (mel64 [n_mels, T], |x_w|_2 [T], filter bank [n_mels, 513])."""
    fb = mo.mel_filterbank64(sr, NFFT, n_mels, fmin, fmax, NORMS[norm])
    xw = frames_of(np.asarray(y, np.float64)) * WIN64
    mag = np.abs(np.fft.rfft(xw, axis=1))
    return fb @ mag.T, np.sqrt((xw * xw).sum(axis=1)), fb


def bound_ratio(got, ref, xnorm, fb, floor, check_floor=True):
    """Worst |exp(got) - max(mel64, 1e-5)| / bound over a [n_mels, T] result; asserts the clip-floor values exactly."""
    got = np.asarray(got, np.float64)
    sw = fb.sum(axis=1)[:, None]
    kc = (fb > 0).sum(axis=1)[:, None]
    delta = TAU_F * xnorm[None, :] * sw + (kc + 2) * U * ref
    c = np.maximum(ref, CLIP)
    dlog = 2.0 ** -22 * (1.0 + np.abs(np.log(c))) * c   # logf's rounding, seen through exp
    both_clip = ref + delta < CLIP * (1 - 1e-6)
    if check_floor:
        assert (got[both_clip] == floor).all(), "a band below the clip is not the clip floor"
    return float((np.abs(np.exp(got) - c) / (delta + dlog)).max())


# ------------------------------------------------------------------------------------------------------------------
# the bound, calibrated on the CPU against a float32 emulation of the kernel
# ------------------------------------------------------------------------------------------------------------------
F32 = np.float32


def _f(x):
    return np.asarray(x, F32)


def emulate_kernel(frames, fb32, win=None, tw_bits=None):
    """mel_kernel's arithmetic in float32, operation for operation, on [F, 1024] fp32 frames: windowing into the complex
    512-point signal, nine radix-2 Stockham passes with table twiddles, the real-transform split, |X|, the fma dot
    product with the fp32 weights, logf(fmaxf(., 1e-5f)).  Returns [n_mels, F] float32."""
    k = np.arange(NFFT // 2)
    twr, twi = _f(np.cos(2 * np.pi * k / NFFT)), _f(-np.sin(2 * np.pi * k / NFFT))
    if tw_bits is not None:
        s = 2.0 ** tw_bits
        twr, twi = _f(np.round(twr * s) / s), _f(np.round(twi * s) / s)
    win = _f(0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / NFFT)) if win is None else _f(win)
    x = _f(frames)
    re, im = x[:, 0::2] * win[0::2], x[:, 1::2] * win[1::2]
    ns = 1
    j = np.arange(256)
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
    kb = np.arange(513)
    zr, zi = re[:, kb & 511], im[:, kb & 511]
    cr, ci = re[:, (512 - kb) & 511], im[:, (512 - kb) & 511]
    h = F32(0.5)
    er, ei = h * (zr + cr), h * (zi - ci)
    orr, oi = h * (zi + ci), -h * (zr - cr)
    wr = np.where(kb < 512, twr[np.minimum(kb, 511)], F32(-1))
    wi = np.where(kb < 512, twi[np.minimum(kb, 511)], F32(0))
    xr, xi = er + wr * orr - wi * oi, ei + wr * oi + wi * orr
    mag = np.sqrt(xr * xr + xi * xi)
    s = np.zeros((fb32.shape[0], x.shape[0]), F32)
    mag64, fb64 = mag.astype(np.float64), fb32.astype(np.float64)
    for kk in range(513):   # fmaf(w, mag, s) in bin order: exact product and sum in float64, one rounding
        nz = fb64[:, kk] != 0
        if nz.any():
            s[nz] = _f(fb64[nz, kk][:, None] * mag64[None, :, kk] + s[nz].astype(np.float64))
    return np.log(np.maximum(s, F32(CLIP)))


def _calibration_frames():
    rs = np.random.RandomState(5)
    n = np.arange(NFFT)
    out = []
    for i in range(200):
        if i % 3 == 0:
            x = 0.8 * np.sin(2 * np.pi * rs.uniform(50, 10000) * n / 22050 + rs.uniform(0, 6))
        elif i % 3 == 1:
            x = rs.uniform(-1, 1, NFFT) * rs.choice([1.0, 0.9, 1e-3])
        else:
            x = rs.standard_normal(NFFT) * 1e-4
        out.append(x)
    return _f(out)


def _wrong_variants():
    sym = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / (NFFT - 1))
    return {
        "twiddles rounded to 11 bits": dict(tw_bits=11),
        "symmetric Hann (N - 1)": dict(win=sym),
        "frame start shifted by one sample": dict(shift=1),
        "bf16 filter weights": dict(bf16=True),
    }


@pytest.mark.parametrize("sr,n_mels,fmin,fmax,norm", [DEFAULT, (44100, 128, 0.0, 22050.0, 0), (16000, 40, 0.0, 8000.0, 2)])
def test_tau_calibration_on_emulated_mel_kernel(sr, n_mels, fmin, fmax, norm):
    """The fp32 emulation of the kernel uses < 0.5 of the bound; every named wrong variant exceeds it by >= 8x."""
    frames = _calibration_frames()
    # frames_of pads; here the frames are given, so the float64 side is built directly
    fb = mo.mel_filterbank64(sr, NFFT, n_mels, fmin, fmax, NORMS[norm])
    fb32 = fb.astype(F32)
    xw = frames.astype(np.float64) * WIN64
    ref = fb @ np.abs(np.fft.rfft(xw, axis=1)).T
    xnorm = np.sqrt((xw * xw).sum(axis=1))
    floor = F32(np.log(F32(CLIP)))
    good = bound_ratio(emulate_kernel(frames, fb32), ref, xnorm, fb, floor)
    wrong = {}
    for name, v in _wrong_variants().items():
        fr = frames
        if "shift" in v:   # the same signals, each frame read one sample late
            long = np.concatenate([frames, _f(np.random.RandomState(9).uniform(-1, 1, (len(frames), 1)))], axis=1)
            fr = long[:, 1:]
        w32 = torch.from_numpy(fb32).to(torch.bfloat16).float().numpy() if v.get("bf16") else fb32
        got = emulate_kernel(fr, w32, win=v.get("win"), tw_bits=v.get("tw_bits"))
        wrong[name] = bound_ratio(got, ref, xnorm, fb, floor, check_floor=False)
    print("\n(sr=%d, %d mels, norm %d) emulation %.3f of the bound; wrong variants: %s" % (
        sr, n_mels, norm, good, ", ".join("%s %.1f" % kv for kv in wrong.items())))
    assert good < 0.5, good
    assert min(wrong.values()) >= 8, wrong


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernel against the float64 reference
# ------------------------------------------------------------------------------------------------------------------
def _signals(L, seed, count=4):
    """Noise, a tone mix, a quiet signal and a full-scale square wave, fp32 in [-1, 1]."""
    rs = np.random.RandomState(seed)
    t = np.arange(L) / 22050.0
    sig = [rs.uniform(-1, 1, L) * 0.9,
           0.4 * np.sin(2 * np.pi * 220 * t) + 0.3 * np.sin(2 * np.pi * rs.uniform(1000, 7000) * t + 1) + 0.01 * rs.standard_normal(L),
           rs.standard_normal(L) * 1e-4,
           np.sign(np.sin(2 * np.pi * 441 * t + 0.5))]
    return np.clip(np.stack(sig[:count]), -1, 1).astype(np.float32)


def _gpu_mel(y, sr, n_mels, fmin, fmax, norm):
    args = (NFFT, n_mels, sr, HOP, NFFT, fmin, fmax)
    return meldataset.mel_spectrogram(torch.from_numpy(y).cuda(), *args, norm=norm).cpu().numpy()


@pytest.fixture(scope="module")
def floor():
    """The value the kernel writes on the clip floor (a silent frame), within an ulp of log(1e-5)."""
    f = _gpu_mel(np.zeros(256, np.float32), *DEFAULT)
    assert (f == f.flat[0]).all()
    f = F32(f.flat[0])
    assert abs(float(f) - np.log(1e-5)) <= float(np.spacing(F32(11.5))), f
    return f


def _check(y, got, opts, floor):
    worst = 0.0
    for i in range(y.shape[0]):
        ref, xnorm, fb = mel64(y[i], *opts)
        assert got[i].shape == ref.shape
        worst = max(worst, bound_ratio(got[i], ref, xnorm, fb, floor))
    return worst


@pytest.mark.gpu
def test_option_sweep_against_float64(floor):
    """Sampling rates, 1 - 128 mels, norm none / Slaney / L1, fmin 0 / 55, fmax 8000 / 9000 / sr/2."""
    worst = 0.0
    for i, opts in enumerate(mel_option_cases()):
        y = _signals(8192 + 77 * i, 100 + i)
        r = _check(y, _gpu_mel(y, *opts), opts, floor)
        assert r <= 1, (opts, r)
        worst = max(worst, r)
    print("\noption sweep (%d settings): worst %.3f of the bound" % (len(mel_option_cases()), worst))


def test_empty_filters_sit_on_the_clip_floor():
    """At 44.1 kHz, 128 mels from 0 Hz to 4 kHz, some triangles fall between two bins (every filter covers a bin once fmax
    reaches 8 kHz): the tables give them no bins, and the GPU sweep checks their rows are the floor."""
    fb = mo.mel_filterbank64(44100, NFFT, 128, 0.0, 4000.0, 1)
    assert ((fb > 0).sum(axis=1) == 0).sum() >= 5
    assert (44100, 128, 0.0, 4000.0, 1) in mel_option_cases()


def _frames(L):
    lib = engine.lib()
    lib.mg_mel_frames.restype = ctypes.c_int
    lib.mg_mel_frames.argtypes = [ctypes.c_int]
    return lib.mg_mel_frames(L)


def _geometry_lengths():
    """The frame geometry's borders, from mg_mel_frames: the first length with a frame, the first lengths of 2, 4 and 32
    frames (each -1, 0, +1), the last length of 2 frames, the longest length whose every frame reads both zero pads (639:
    frame 0 reads [-384, 640)), and a long odd length."""
    firsts = {}
    for L in range(1, 8200):
        firsts.setdefault(_frames(L), L)
    out = [firsts[1], firsts[1] + 1, firsts[3] - 1]
    for T in (2, 4, 32):
        out += [firsts[T] - 1, firsts[T], firsts[T] + 1]
    both = [L for L in range(firsts[1], 4096)
            if all(HOP * t - PAD < 0 and HOP * t + NFFT - PAD > L for t in range(_frames(L)))]
    out += [max(both), 23457]
    return sorted(set(out))


def test_geometry_lengths_follow_the_frame_count():
    Ls = _geometry_lengths()
    assert Ls == [256, 257, 511, 512, 513, 639, 767, 1023, 1024, 1025, 8191, 8192, 8193, 23457], Ls
    assert all(_frames(L) == L // HOP for L in Ls)


@pytest.mark.gpu
@pytest.mark.parametrize("L", _geometry_lengths())
def test_frame_geometry_lengths_against_float64(floor, L):
    y = _signals(L, L)
    got = _gpu_mel(y, *DEFAULT)
    r = _check(y, got, DEFAULT, floor)
    print("L=%d (T=%d): %.3f of the bound" % (L, _frames(L), r))
    assert r <= 1, (L, r)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 5])
@pytest.mark.parametrize("L", [256, 767, 8193 - 256])   # T = 1, 2 (even: no dead frame) and 31
def test_dead_frame_of_the_last_cta_writes_nothing(floor, B, L):
    """Odd T: the last CTA's second frame is past the end.  Through the C ABI into a buffer with a guard tail, filled with
    NaN: every value is in the bound and the guard is untouched."""
    T = _frames(L)
    n_mels = 80
    y = torch.from_numpy(np.concatenate([_signals(L, B * L)] * 2)[:B]).cuda()
    tab = meldataset._tables(y.device, *DEFAULT[:1], n_mels, *DEFAULT[2:])
    out = torch.full((B * n_mels * T + 4096,), float("nan"), device="cuda")
    lib = engine.lib()
    lib.mg_mel_spectrogram.restype = ctypes.c_int
    lib.mg_mel_spectrogram.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    engine.check(lib.mg_mel_spectrogram(tab.data_ptr(), y.data_ptr(), out.data_ptr(), B, L, torch.cuda.current_stream().cuda_stream))
    out = out.cpu().numpy()
    assert np.isnan(out[B * n_mels * T:]).all(), "the dead frame wrote past the output"
    r = _check(y.cpu().numpy(), out[:B * n_mels * T].reshape(B, n_mels, T), DEFAULT, floor)
    assert r <= 1, r


@pytest.mark.gpu
def test_batch_items_equal_their_own_calls_and_layouts_agree():
    """Each item of a batch is bit-identical to its own B = 1 call (silence and full scale among them); non-contiguous,
    float64 and 1-D input give the same bits; two identical calls are identical."""
    L = 8192 + 300
    y = np.concatenate([_signals(L, 1), np.zeros((1, L), np.float32), np.ones((1, L), np.float32),
                        -np.ones((1, L), np.float32)])
    yt = torch.from_numpy(y).cuda()
    args = (NFFT, 80, 22050, HOP, NFFT, 55, 9000)
    got = meldataset.mel_spectrogram(yt, *args)
    assert torch.equal(got, meldataset.mel_spectrogram(yt, *args))
    for i in range(y.shape[0]):
        assert torch.equal(got[i], meldataset.mel_spectrogram(yt[i:i + 1], *args)[0]), i
        assert torch.equal(got[i], meldataset.mel_spectrogram(yt[i], *args)), i
    wide = torch.zeros((y.shape[0], 2 * L), device="cuda")
    wide[:, 1::2] = yt
    assert not wide[:, 1::2].is_contiguous()
    assert torch.equal(got, meldataset.mel_spectrogram(wide[:, 1::2], *args))
    assert torch.equal(got, meldataset.mel_spectrogram(yt.double(), *args))
    assert torch.equal(got[4], torch.full_like(got[4], float(got[4, 0, 0])))   # silence: the clip floor


@pytest.mark.gpu
def test_batch_beyond_65535_items(floor):
    """70 000 one-frame items (more than grid.y could hold): every item equals the same item in batches of at most
    65 535, a sample equals its own B = 1 call, and a sample is within the float64 bound."""
    B, L = 70000, 256
    rs = np.random.RandomState(70000)
    y = (rs.uniform(-1, 1, (B, L)) * rs.uniform(0, 1, (B, 1))).astype(np.float32)
    yt = torch.from_numpy(y).cuda()
    args = (NFFT, 80, 22050, HOP, NFFT, 55, 9000)
    got = meldataset.mel_spectrogram(yt, *args, check_range=False)
    parts = torch.cat([meldataset.mel_spectrogram(yt[s:s + 65535], *args, check_range=False) for s in range(0, B, 65535)])
    assert torch.equal(got, parts)
    sample = [0, 1, 65534, 65535, 65536, B - 2, B - 1] + list(rs.randint(0, B, 9))
    for i in sample:
        assert torch.equal(got[i], meldataset.mel_spectrogram(yt[i], *args)), i
    got = got.cpu().numpy()
    r = _check(y[sample], got[sample], DEFAULT, floor)
    print("\nB=70000: sampled items %.3f of the bound" % r)
    assert r <= 1, r
