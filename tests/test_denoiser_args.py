"""The denoiser without a GPU: every argument the C calls refuse is reported (an error code and a message naming it)
before anything touches CUDA, the NOLA refusal against torch.istft's own, the workspace at the frame-count borders, the
float64 definition (tests/denoise_model.py) against a numpy restatement of WaveGlow's conv-basis STFT, and the Python
module's argument checks.  Fake device addresses stand in for buffers: a call that reached CUDA would fail with
MG_ERR_CUDA instead."""
import ctypes

import numpy as np
import pytest
import torch

import denoise_model as dm
from melgan_multi_b200 import denoiser, engine

INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL


def _lib():
    return denoiser._lib()


def _ints(v):
    return None if v is None else (ctypes.c_int * len(v))(*v)


def _ws(n, h, B, L, lengths=None):
    b = ctypes.c_size_t()
    rc = _lib().mg_denoise_workspace_bytes(n, h, B, L, _ints(lengths), ctypes.byref(b))
    return rc, b.value


def _call(pcm=False, n=1024, h=256, w=1024, B=2, L=8192, lengths=None, n_voices=1, voice=None, strength=0.1, ws_bytes=None,
          **ptr):
    p = dict(tables=256, audio=512, bias=1024, out=2048, ws=4096)
    p.update(ptr)
    if ws_bytes is None:
        rc, ws_bytes = _ws(n, h, B, L, lengths)
        ws_bytes = ws_bytes if rc == 0 else 1 << 62
    fn = _lib().mg_denoise_forward_pcm16 if pcm else _lib().mg_denoise_forward
    rc = fn(p["tables"], n, h, w, p["audio"], B, L, _ints(lengths), p["bias"], n_voices, _ints(voice), strength, p["out"], p["ws"],
            ws_bytes, None)
    return rc, _lib().mg_last_error_string().decode()


@pytest.mark.parametrize("pcm", [False, True])
def test_refusals_before_any_launch(pcm):
    fn = "mg_denoise_forward_pcm16" if pcm else "mg_denoise_forward"
    for k in ("tables", "audio", "bias", "out", "ws"):
        rc, msg = _call(pcm, **{k: None})
        assert rc == INVALID and msg.startswith(fn) and "%s is NULL" % ("workspace" if k == "ws" else k) in msg, (k, msg)
    for k, align in (("tables", 16), ("audio", 4), ("bias", 4), ("out", 2 if pcm else 4), ("ws", 16)):
        rc, msg = _call(pcm, **{k: 256 + align // 2})
        assert rc == INVALID and "%s must be %d-byte aligned" % ("workspace" if k == "ws" else k, align) in msg, (k, msg)
    for n in (64, 100, 1000, 4096, 0, -1024):
        rc, msg = _call(pcm, n=n, w=min(max(n, 1), 64))
        assert rc == INVALID and "n_fft=%d is not a power of two in [128, 2048]" % n in msg, msg
    for h in (0, -3):
        rc, msg = _call(pcm, h=h)
        assert rc == INVALID and "hop=%d, at least 1 needed" % h in msg, msg
    for w in (0, -1, 1025):
        rc, msg = _call(pcm, w=w)
        assert rc == INVALID and "win_length=%d is outside [1, n_fft=1024]" % w in msg, msg
    rc, msg = _call(pcm, w=255)
    assert rc == INVALID and "hop=256 exceeds win_length=255" in msg, msg
    for B in (0, -1):
        rc, msg = _call(pcm, B=B)
        assert rc == INVALID and "B=%d, at least 1 item needed" % B in msg, msg
    rc, msg = _call(pcm, L=(1 << 30) + 1)
    assert rc == INVALID and "L_max=1073741825 samples, at most 2^30 supported" in msg, msg
    for L in (512, 100):
        rc, msg = _call(pcm, L=L)
        assert rc == INVALID and "L_max=%d samples, reflect padding by n_fft/2=512 needs more" % L in msg, msg
    for bad in (512, 8193, 0, -5):
        rc, msg = _call(pcm, lengths=[8192, bad])
        assert rc == INVALID and "lengths[1]=%d is outside (n_fft/2=512, L_max=8192]" % bad in msg, msg
    for nv in (0, -1):
        rc, msg = _call(pcm, n_voices=nv)
        assert rc == INVALID and "n_voices=%d, at least 1 needed" % nv in msg, msg
    for v in (-1, 3):
        rc, msg = _call(pcm, n_voices=3, voice=[0, v])
        assert rc == INVALID and "voice[1]=%d is outside [0, n_voices=3)" % v in msg, msg
    for s in (float("nan"), float("inf"), -float("inf")):
        rc, msg = _call(pcm, strength=s)
        assert rc == INVALID and "strength=" in msg and "is not finite" in msg, msg
    rc, need = _ws(1024, 256, 2, 8192)
    rc, msg = _call(pcm, ws_bytes=need - 1)
    assert rc == WS_SMALL and "workspace of %d bytes, %d needed" % (need - 1, need) in msg, msg
    rc, msg = _call(pcm, ws_bytes=0)
    assert rc == WS_SMALL
    # the NOLA condition: a window of 2 samples at hop 2 leaves samples with no envelope
    rc, msg = _call(pcm, h=2, w=2)
    assert rc == INVALID and "(n_fft=1024, hop=2, win_length=2) leaves the window-square envelope below 1e-11" in msg, msg
    # frames past 2^31 - 1 CTAs at hop 1 (uniform: no item limit)
    rc, msg = _call(pcm, n=128, h=1, w=128, B=1 << 16, L=1 << 15)
    assert rc == INVALID and "frames exceed 2^31 - 1 CTAs" in msg, msg


@pytest.mark.parametrize("pcm", [False, True])
def test_ragged_and_voiced_item_limit(pcm):
    lim = 256  # MG_GEN_RAGGED_MAX_B
    for B in (lim, lim + 1):
        for kw in (dict(lengths=[8192] * B), dict(voice=[0] * B, n_voices=1), dict(lengths=[8000] * B, voice=[0] * B)):
            rc, msg = _call(pcm, B=B, out=None, **kw)
            if B == lim:
                assert rc == INVALID and "out is NULL" in msg, msg
            else:
                assert rc == INVALID and "B=%d exceeds MG_GEN_RAGGED_MAX_B=256" % B in msg, msg
        rc, need = _ws(1024, 256, B, 8192, [8192] * B)
        assert (rc == 0) == (B == lim)
    # a uniform batch has no item limit
    rc, need = _ws(1024, 256, 1000, 8192)
    assert rc == 0 and need == 1000 * (1 + 8192 // 256) * 1024 * 4


def test_workspace_call_refusals():
    lib = _lib()
    assert lib.mg_denoise_workspace_bytes(1024, 256, 2, 8192, None, None) == INVALID
    assert b"bytes is NULL" in lib.mg_last_error_string()
    for args in ((1000, 256, 2, 8192), (1024, 0, 2, 8192), (1024, 256, 0, 8192), (1024, 256, 2, 512), (1024, 256, 2, (1 << 30) + 1)):
        assert _ws(*args)[0] == INVALID, args


@pytest.mark.parametrize("n,h", [(128, 1), (128, 32), (256, 67), (512, 128), (1024, 256), (1024, 1024), (2048, 512), (2048, 3000)])
def test_workspace_at_the_frame_count_borders(n, h):
    Ls = {n // 2 + 1, 8192}
    for k in range(max(1, (n // 2 + 1) // h), (n // 2 + 1) // h + 4):
        Ls |= {k * h - 1, k * h, k * h + 1}
    Ls = sorted(v for v in Ls if v > n // 2)
    for L in Ls:
        rc, b = _ws(n, h, 3, L)
        assert rc == 0 and b == 3 * (1 + L // h) * n * 4, (L, b)
    Lmax = max(Ls)
    rc, b = _ws(n, h, len(Ls), Lmax, Ls)
    assert rc == 0 and b == sum(1 + L // h for L in Ls) * n * 4


def test_bias_call_refusals():
    lib = _lib()
    for args, match in (((256, 1000, 512, 1, 2048, 1024), "n_fft=1000"), ((256, 1024, 512, 0, 2048, 1024), "n_rows=0"),
                        ((256, 1024, 512, 1, 512, 1024), "L=512 is outside"), ((None, 1024, 512, 1, 2048, 1024), "tables is NULL"),
                        ((264, 1024, 512, 1, 2048, 1024), "tables must be 16-byte aligned"),
                        ((256, 1024, None, 1, 2048, 1024), "audio is NULL"), ((256, 1024, 512, 1, 2048, None), "bias is NULL"),
                        ((256, 1024, 514, 1, 2048, 1024), "audio must be 4-byte aligned")):
        t, n, a, rows, L, b = args
        assert lib.mg_denoise_bias(t, n, a, rows, L, b, None) == INVALID, args
        msg = lib.mg_last_error_string().decode()
        assert msg.startswith("mg_denoise_bias") and match in msg, (args, msg)


def _torch_refuses(n, h, w, L):
    win = torch.hann_window(w, dtype=torch.float64)
    S = torch.zeros(n // 2 + 1, 1 + L // h, dtype=torch.complex128)
    try:
        torch.istft(S, n, h, w, win, center=True, length=L)
    except RuntimeError as e:
        assert "window overlap add min" in str(e) or "expected 0 < hop_length <= win_length" in str(e), str(e)
        return True
    return False


def test_nola_refusal_agrees_with_torch_istft():
    cases = []
    for n in (128, 256):
        for w in sorted({1, 2, 3, 31, 32, 33, 63, 64, 65, n // 2 - 1, n // 2 + 1, n - 1, n}):
            for h in sorted({1, 16, 31, w - 1 if w > 1 else 1, w, w + 1, n // 4, n // 2, n // 2 + 1, n - 1, n, n + 5}):
                if h < 1:
                    continue
                for L in sorted({n // 2 + 1, n - 1, n, 3 * h - 1, 3 * h, 3 * h + 1, 1000}):
                    if L > n // 2:
                        cases.append((n, h, w, L))
    refused = agreed = 0
    for n, h, w, L in cases:
        want = _torch_refuses(n, h, w, L)
        if h <= w:
            assert dm.nola_ok(n, h, w, L) == (not want), (n, h, w, L)
        rc, msg = _call(n=n, h=h, w=w, B=1, L=L, out=None)  # (an accepted call stops at the NULL out, before CUDA)
        ours = "NOLA" in msg or "exceeds win_length" in msg
        assert rc == INVALID and ours == want and (want or "out is NULL" in msg), (n, h, w, L, msg)
        refused += want
        agreed += 1
    assert refused > 50 and agreed - refused > 50, (refused, agreed)


# ------------------------------------------------------------------------------------------------------------------
# the float64 definition against WaveGlow's algorithm restated in numpy
# ------------------------------------------------------------------------------------------------------------------
def waveglow_denoise(a, n, h, w, bias, strength):
    """WaveGlow's STFT module and Denoiser (stft.py, denoiser.py) in float64 numpy: conv1d with the stacked real/imag
    Fourier basis times the window, magnitude and atan2 phase, conv_transpose1d with pinv(scale basis)^T times the
    window, division by the window-square sum where it exceeds float32 tiny, times n / h, N/2 trimmed at each end."""
    scale = n / h
    fb = np.fft.fft(np.eye(n))
    cutoff = n // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff]), np.imag(fb[:cutoff])])
    fwd = fb.copy()
    inv = np.linalg.pinv(scale * fb).T
    win = dm.hann64(w, n).numpy()
    fwd = fwd * win[None]
    inv = inv * win[None]
    x = np.pad(a, (n // 2, n // 2), mode="reflect")
    T = (len(x) - n) // h + 1
    frames = np.stack([x[t * h:t * h + n] for t in range(T)], 1)  # [n, T]
    ft = fwd @ frames
    re, im = ft[:cutoff], ft[cutoff:]
    mag = np.sqrt(re ** 2 + im ** 2)
    ph = np.arctan2(im, re)
    mag = np.clip(mag - bias[:, None] * strength, 0.0, None)
    rec = np.concatenate([mag * np.cos(ph), mag * np.sin(ph)], 0)
    ycols = inv.T @ rec  # [n, T]
    out = np.zeros(n + h * (T - 1))
    wsum = np.zeros_like(out)
    for t in range(T):
        out[t * h:t * h + n] += ycols[:, t]
        wsum[t * h:t * h + n] += win ** 2
    nz = wsum > np.finfo(np.float32).tiny
    out[nz] /= wsum[nz]
    out *= scale
    return out[n // 2:len(out) - n // 2]


@pytest.mark.parametrize("n,h,w", [(1024, 256, 1024), (1024, 256, 800), (512, 128, 512), (2048, 512, 2048)])
def test_definition_equals_waveglows_algorithm(n, h, w):
    rng = np.random.default_rng(n + w)
    bias = np.abs(rng.standard_normal(n // 2 + 1)) * 2
    for L in (8 * h, 8 * h + 1, 9 * h - 1, 12 * h + h // 2):
        a = rng.standard_normal(L)
        ref = dm.denoise64(torch.from_numpy(a), n, h, w, torch.from_numpy(bias), 0.3).numpy()
        wg = waveglow_denoise(a, n, h, w, bias, 0.3)
        k = h * (L // h)
        assert len(wg) == k
        err = np.abs(ref[:k] - wg).max() / np.abs(ref).max()
        assert err < 1e-12, (L, err)


def test_mutants_differ_from_the_definition():
    """Each float64 mutant the GPU bound has to reject changes the output, and the restatement without one is the
    definition itself."""
    rng = np.random.default_rng(5)
    n, h, w, L = 256, 64, 256, 2000
    a = torch.from_numpy(rng.standard_normal((2, L)))
    bias = torch.from_numpy(np.abs(rng.standard_normal((2, n // 2 + 1))) * 3)
    lens, voice = [L, L - 300], [1, 0]
    ref = dm.denoise64_batch(a, n, h, w, bias, 0.5, lens, voice)
    got, _ = dm.denoise64_parts(a, n, h, w, bias, 0.5, lens, voice)
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    for m in dm.DENOISE_MUTANTS:
        mut, _ = dm.denoise64_parts(a, n, h, w, bias, 0.5, lens, voice, mutant=m)
        assert (mut - ref).abs().max() > 1e-3 * ref.abs().max(), m


# ------------------------------------------------------------------------------------------------------------------
# the module's checks, without a device
# ------------------------------------------------------------------------------------------------------------------
class _FakeCuda(torch.Tensor):
    @property
    def is_cuda(self):
        return True


def _fake(*shape, grad=False, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype, requires_grad=grad).as_subclass(_FakeCuda)


def test_module_refusals():
    d = denoiser.Denoiser.from_bias(torch.zeros(2, 513))
    assert d.n_fft == 1024 and d.hop == 256 and d.win_length == 1024
    with pytest.raises(engine.EngineError, match="audio must be a CUDA tensor"):
        d(torch.zeros(2, 4096))
    with pytest.raises(engine.EngineError, match=r"fp32 \[B, L\] or \[B, 1, L\]"):
        d(_fake(2, 4096, dtype=torch.float64))
    with pytest.raises(engine.EngineError, match=r"fp32 \[B, L\] or \[B, 1, L\]"):
        d(_fake(2, 2, 4096))
    with pytest.raises(engine.EngineError, match="audio requires grad"):
        d(_fake(2, 4096, grad=True))
    with pytest.raises(engine.EngineError, match="dtype must be"):
        d(_fake(2, 4096), dtype=torch.float16)
    with pytest.raises(engine.EngineError, match="strength"):
        d(_fake(2, 4096), strength=float("nan"))
    for args, match in (((1000,), "filter_length 1000 is not a power of two"), ((4096,), "filter_length 4096"),
                        ((1024, 4, 1025), "win_length 1025"), ((1024, 4, 0), "win_length 0"), ((1024, 2048), "hop"),
                        ((1024, 2, 500), "hop 512 exceeds win_length 500")):
        with pytest.raises(engine.EngineError, match=match):
            denoiser.Denoiser.from_bias(torch.zeros(1, args[0] // 2 + 1), *args)
    with pytest.raises(engine.EngineError, match=r"fp32 \[V, 513\]"):
        denoiser.Denoiser.from_bias(torch.zeros(1, 512))
    with pytest.raises(engine.EngineError, match=r"fp32 \[V, 513\]"):
        denoiser.Denoiser.from_bias(torch.zeros(1, 513, dtype=torch.float64))
    with pytest.raises(engine.EngineError, match="mode"):
        denoiser.Denoiser(object(), mode="ones")
    with pytest.raises(engine.EngineError, match="at least one generator"):
        denoiser.Denoiser([])
    with pytest.raises(engine.EngineError, match="built from a bias"):
        d.refresh()


def test_module_under_no_grad_accepts_audio_that_requires_grad():
    """Grad mode off: an audio that requires grad passes the checks (no graph could be built), so the call gets as far as
    selecting the device, which the fake CUDA tensor does not have."""
    d = denoiser.Denoiser.from_bias(torch.zeros(1, 513))
    with pytest.raises(engine.EngineError, match="audio requires grad"):
        d(_fake(2, 4096, grad=True))
    with torch.no_grad():
        with pytest.raises(Exception) as e:
            d(_fake(2, 4096, grad=True))
    assert "requires grad" not in str(e.value)
