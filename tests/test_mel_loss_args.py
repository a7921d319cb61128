"""The multi-resolution mel loss without a GPU: every argument the C calls and the module refuse is reported (an error
code and a message naming it) before anything touches CUDA, the frame count and workspace sizes at the frame geometry's
borders, the tables against a float64 numpy restatement of librosa's window and Slaney filter bank at every supported
n_fft, and the table builder at n_fft 1024 against every field of the front end's mg_mel_tables_build.  Fake device
addresses stand in for buffers: a call that reached CUDA would fail with MG_ERR_CUDA instead."""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, mel_loss

INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL
N_FFTS = (128, 256, 512, 1024, 2048)


def _lib():
    return mel_loss._lib()


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _sizes(n_fft, hop, B, L):
    f, b = ctypes.c_size_t(), ctypes.c_size_t()
    rc = _lib().mg_mel_loss_workspace_bytes(len(n_fft), _ints(n_fft), _ints(hop), B, L, ctypes.byref(f), ctypes.byref(b))
    return rc, f.value, b.value


def _call(which, n_fft=(1024, 2048, 512), hop=(256, 512, 128), B=2, L=8192, tables=None, n_res=None, ws_bytes=None, **ptr):
    lib = _lib()
    n_res = len(n_fft) if n_res is None else n_res
    tabs = (ctypes.c_void_p * max(1, len(n_fft)))(*([256] * len(n_fft) if tables is None else tables))
    rc, f, b = _sizes(n_fft, hop, B, L)
    p = dict(x=256, y=512, loss=768, grad=1280, gx=4096, ws=8192, tabs=tabs, n_fft_arr=_ints(n_fft), hop_arr=_ints(hop))
    p.update(ptr)
    if which == "forward":
        rc = lib.mg_mel_loss_forward(n_res, p["tabs"], p["n_fft_arr"], p["hop_arr"], p["x"], p["y"], B, L, p["loss"], p["ws"],
                                     f if ws_bytes is None else ws_bytes, None)
    else:
        rc = lib.mg_mel_loss_backward(n_res, p["tabs"], p["n_fft_arr"], p["hop_arr"], p["x"], p["y"], B, L, p["grad"], p["gx"],
                                      p["ws"], b if ws_bytes is None else ws_bytes, None)
    return rc, lib.mg_last_error_string().decode()


def _frames(n, h, L):
    span = L + 2 * ((n - h) // 2)
    return 0 if span < n else 1 + (span - n) // h


@pytest.mark.parametrize("which", ["forward", "backward"])
def test_refusals_before_any_launch(which):
    fn = "mg_mel_loss_" + which
    ptrs = ["x", "y", "loss", "ws", "tabs", "n_fft_arr", "hop_arr"] if which == "forward" else \
        ["x", "y", "grad", "gx", "ws", "tabs", "n_fft_arr", "hop_arr"]
    names = dict(gx="grad_x", ws="workspace", tabs="tables", n_fft_arr="n_fft", hop_arr="hop")
    for k in ptrs:
        rc, msg = _call(which, **{k: None})
        assert rc == INVALID and msg.startswith(fn) and "%s is NULL" % names.get(k, k) in msg, (k, msg)
    for k, align in (("x", 4), ("y", 4), ("loss", 4), ("grad", 4), ("gx", 4), ("ws", 16)):
        if k not in ptrs:
            continue
        rc, msg = _call(which, **{k: 256 + align // 2})
        assert rc == INVALID and "%s must be %d-byte aligned" % (names.get(k, k), align) in msg, (k, msg)
    rc, msg = _call(which, tables=[256, 264, 256])
    assert rc == INVALID and "tables[1] must be 16-byte aligned" in msg
    rc, msg = _call(which, tables=[256, 256, None])
    assert rc == INVALID and "tables[2] is NULL" in msg
    for n in (64, 100, 1000, 4096, 0, -1024):
        rc, msg = _call(which, n_fft=(1024, n, 512))
        assert rc == INVALID and "n_fft[1]=%d is not a power of two in [128, 2048]" % n in msg, msg
    for h in (0, -3, 513):
        rc, msg = _call(which, hop=(256, 512, h))
        assert rc == INVALID and "hop[2]=%d is outside [1, n_fft=512]" % h in msg, msg
    # one frame needs L + 2 ((N - H) // 2) >= N: at (2048, 512) L >= 512, at (1024, 256) L >= 256
    for L in (511, 300, 1):
        rc, msg = _call(which, L=L)
        assert rc == INVALID and "L=%d samples are fewer than one frame of resolution" % L in msg, msg
    rc, msg = _call(which, L=(1 << 30) + 1, ws_bytes=1 << 62)
    assert rc == INVALID and "L=1073741825 samples, 1 to 2^30 supported" in msg, msg
    rc, msg = _call(which, L=0)
    assert rc == INVALID and "L=0 samples" in msg, msg
    for B in (0, -1):
        rc, msg = _call(which, B=B)
        assert rc == INVALID and "B=%d, at least 1 item needed" % B in msg, msg
    for n_res in (0, 9, -1):
        rc, msg = _call(which, n_res=n_res)
        assert rc == INVALID and "n_res=%d resolutions, 1 to 8 supported" % n_res in msg, msg
    rc, msg = _call(which, n_fft=(128,) * 9, hop=(1,) * 9)
    assert rc == INVALID and "n_res=9" in msg
    # B T CTAs past 2^31 - 1 at hop 1: 2^16 items of 2^15 + 1 frames
    rc, msg = _call(which, n_fft=(128,), hop=(1,), B=1 << 16, L=(1 << 15) + 2, ws_bytes=1 << 62)
    assert rc == INVALID and "B=65536 x 32769 frames of resolution 0 exceed 2^31 - 1 CTAs" in msg, msg
    # the gather's B ceil(L / 256) CTAs past 2^31 - 1 with few frames: hop = n_fft
    rc, msg = _call(which, n_fft=(2048,), hop=(2048,), B=1 << 9, L=1 << 30, ws_bytes=1 << 62)
    assert rc == INVALID and "sample blocks exceed 2^31 - 1 CTAs" in msg, msg
    rc0, f, b = _sizes((1024, 2048, 512), (256, 512, 128), 2, 8192)
    need = f if which == "forward" else b
    rc, msg = _call(which, ws_bytes=need - 1)
    assert rc == WS_SMALL and "workspace of %d bytes, %d needed" % (need - 1, need) in msg, msg
    rc, msg = _call(which, ws_bytes=0)
    assert rc == WS_SMALL


def test_workspace_call_refusals():
    lib = _lib()
    f = ctypes.c_size_t()
    rc = lib.mg_mel_loss_workspace_bytes(1, _ints([512]), _ints([128]), 2, 8192, ctypes.byref(f), None)
    assert rc == INVALID and b"backward_bytes is NULL" in lib.mg_last_error_string()
    rc = lib.mg_mel_loss_workspace_bytes(1, _ints([512]), None, 2, 8192, ctypes.byref(f), ctypes.byref(f))
    assert rc == INVALID and b"hop is NULL" in lib.mg_last_error_string()
    assert _sizes((512,), (128,), 2, 127)[0] == INVALID
    assert _sizes((512,), (0,), 2, 8192)[0] == INVALID
    assert _sizes((512,), (513,), 2, 8192)[0] == INVALID
    assert _sizes((512,) * 9, (128,) * 9, 2, 8192)[0] == INVALID
    assert _sizes((512,), (128,), 1, (1 << 30) + 1)[0] == INVALID
    assert _sizes((512,), (512,), 1, 1 << 30)[0] == 0
    assert lib.mg_mel_loss_frames(512, 128, (1 << 30) + 1) == 0
    assert lib.mg_mel_loss_frames(512, 128, 0) == 0


@pytest.mark.parametrize("n,h", [(128, 1), (128, 128), (128, 37), (256, 64), (512, 51), (1024, 256), (1024, 1024), (1024, 333),
                                 (2048, 512), (2048, 2047), (2048, 1)])
def test_frames_and_workspace_follow_the_frame_geometry(n, h):
    """At the one-frame minimum L, at L = 0, 1 and H - 1 mod H around it, with (N - H) odd and even, at H = 1 and H = N."""
    lib = _lib()
    p = (n - h) // 2
    lmin = n - 2 * p                       # H, or H + 1 when N - H is odd
    Ls = {lmin, lmin + 1, 8192, 220500}
    for m in range(1, 5):
        for r in (0, 1, h - 1):
            Ls.add(lmin + m * h + r - (1 if r == 0 and m else 0))
            Ls.add(m * h + r)
    for L in sorted(v for v in Ls if v >= 1):
        T = lib.mg_mel_loss_frames(n, h, L)
        assert T == _frames(n, h, L), (n, h, L)
        if T < 1:
            assert L < lmin and _sizes((n,), (h,), 1, L)[0] == INVALID
            continue
        for B in (1, 3, 16):
            rc, f, b = _sizes((n,), (h,), B, L)
            assert rc == 0
            assert f == -(-B * T * 4 // 256) * 256, (B, L)
            assert b == B * T * n * 4, (B, L)
    assert lib.mg_mel_loss_frames(n, h, lmin) == 1 and lib.mg_mel_loss_frames(n, h, lmin - 1) == 0
    assert lib.mg_mel_loss_frames(n, h, lmin + h - 1) == 1 and lib.mg_mel_loss_frames(n, h, lmin + h) == 2
    assert lib.mg_mel_loss_frames(n, 0, 8192) == 0 and lib.mg_mel_loss_frames(n, n + 1, 8192) == 0
    assert lib.mg_mel_loss_frames(n + 1, h, 8192) == 0


def test_reference_analysis_frames_equal_the_front_ends():
    lib = engine.lib()
    for L in (256, 257, 511, 512, 8192, 8193, 66167, 220500):
        assert _lib().mg_mel_loss_frames(1024, 256, L) == lib.mg_mel_frames(L), L


def test_workspace_sums_the_partials_and_takes_the_largest_frame_buffer():
    B, L = 16, 8192
    res = ((128, 256, 512, 1024, 2048), (32, 64, 128, 256, 512))
    rc, f, b = _sizes(*res, B, L)
    T = [_frames(n, h, L) for n, h in zip(*res)]
    assert rc == 0
    assert f == sum(-(-B * t * 4 // 256) * 256 for t in T)
    assert b == max(B * t * n * 4 for t, n in zip(T, res[0]))


# ------------------------------------------------------------------------------------------------------------------
# tables
# ------------------------------------------------------------------------------------------------------------------
def _hz_to_mel(f):
    f = np.asarray(f, np.float64)
    lin = f / (200.0 / 3)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-300) / 1000.0) / (np.log(6.4) / 27.0), lin)


def _mel_to_hz(m):
    m = np.asarray(m, np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp(np.log(6.4) / 27.0 * (m - 15.0)), (200.0 / 3) * m)


def filterbank64(sr, n_fft, n_mels, fmin, fmax):
    """librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=False, norm='slaney') in float64, as librosa states it."""
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    return w * (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]


def window64(n_fft, win_length):
    """scipy.signal.get_window('hann', win_length, fftbins=True), centred in n_fft as librosa.util.pad_center does."""
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win_length) / win_length) if win_length > 1 else np.ones(1)
    left = (n_fft - win_length) // 2
    return np.pad(w, (left, n_fft - win_length - left))


def parse(host, n_fft):
    """(window, twiddles [n_fft/2, 2], n_mels, kstart, kcount, woff, weights) of one mel-loss table."""
    ib = host.view(np.int32)
    base = 2 * n_fft
    n_mels = int(ib[base])
    ks, kc, wo = (ib[base + 4 + 512 * i:base + 4 + 512 * i + n_mels] for i in range(3))
    wts = host[base + 4 + 3 * 512:base + 4 + 3 * 512 + 2 * (n_fft // 2 + 1)]
    return host[:n_fft], host[n_fft:2 * n_fft].reshape(-1, 2), n_mels, ks, kc, wo, wts


def dense(ks, kc, wo, wts, n_fft):
    out = np.zeros((len(ks), n_fft // 2 + 1))
    for m in range(len(ks)):
        out[m, ks[m]:ks[m] + kc[m]] = wts[wo[m]:wo[m] + kc[m]]
    return out


TABLE_CASES = [(22050, 80, 55.0, 9000.0), (22050, 80, 0.0, 11025.0), (16000, 40, 0.0, 8000.0), (24000, 100, 20.0, 12000.0),
               (44100, 128, 0.0, 22050.0), (22050, 512, 0.0, 11025.0), (22050, 10, 55.0, 9000.0), (8000, 1, 0.0, 4000.0)]


@pytest.mark.parametrize("n", N_FFTS)
def test_tables_equal_float64_librosa(n):
    """Window and twiddles as the STFT loss builds them; each filter's sparse run holds exactly its positive bins, each
    weight its float64 value rounded to fp32; same-parity filters share no bin (the backward's two passes rely on it).
    At n_fft 128 most of 128 or 512 bands cover no bin: their runs are empty."""
    lib = _lib()
    assert lib.mg_mel_loss_tables_bytes(n) == 8 * n + 16 + 3 * 512 * 4 + -(-(2 * (n // 2 + 1) * 4) // 16) * 16
    empties = 0
    for sr, n_mels, fmin, fmax in TABLE_CASES + ([(22050, 128, 0.0, 11025.0)] if n == 128 else []):
        for w in sorted({n, n - 1, n // 2 + 1, 1}):
            host = mel_loss.build_tables(n, w, sr, n_mels, fmin, fmax)
            win, tw, nm, ks, kc, wo, wts = parse(host, n)
            assert np.array_equal(win, window64(n, w).astype(np.float32)), (n, w)
            assert np.array_equal(host[:2 * n], stft_loss_table(n, w))
            k = np.arange(n // 2)
            assert np.array_equal(tw, np.stack([np.cos(2 * np.pi * k / n), -np.sin(2 * np.pi * k / n)], 1).astype(np.float32))
            assert nm == n_mels
            ref = filterbank64(sr, n, n_mels, fmin, fmax)
            got = dense(ks, kc, wo, wts, n)
            for m in range(n_mels):
                pos = np.nonzero(ref[m] > 0)[0]
                if len(pos) == 0:
                    assert kc[m] == 0, (n, sr, n_mels, m)
                    empties += 1
                else:
                    # a bin whose float64 weight is a rounding error from 0 may fall either side of it
                    assert ks[m] <= pos[0] + 1 and ks[m] + kc[m] >= pos[-1], (n, sr, n_mels, m)
            assert np.all(np.abs(got - ref) <= 2 ** -23 * ref + 1e-12 * ref.max()), (n, sr, n_mels, np.abs(got - ref).max())
            for par in (0, 1):
                cover = np.zeros(n // 2 + 1, int)
                for m in range(par, n_mels, 2):
                    cover[ks[m]:ks[m] + kc[m]] += 1
                assert cover.max() <= 1, (n, sr, n_mels, par)
    if n == 128:
        assert empties > 0


def stft_loss_table(n, w):
    from melgan_multi_b200 import stft_loss
    return stft_loss.build_tables(n, w)


def test_builder_at_1024_reproduces_every_field_of_the_front_ends_tables():
    """mg_mel_tables_build (norm = 1, Slaney) and mg_mel_loss_tables_build at (1024, 1024) fill the same window,
    twiddles, n_mels, kstart, kcount, woff and weights, bit for bit."""
    from kernel_model import mel_option_cases
    L = engine.lib()
    L.mg_mel_tables_bytes.restype = ctypes.c_size_t
    L.mg_mel_tables_build.restype = ctypes.c_int
    L.mg_mel_tables_build.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
    nb = L.mg_mel_tables_bytes()
    cases = {c[:4] for c in mel_option_cases()} | {(22050, 80, 55.0, 9000.0), (22050, 128, 0.0, 11025.0)}
    for sr, n_mels, fmin, fmax in sorted(cases):
        front = np.zeros((nb + 3) // 4, np.float32)
        engine.check(L.mg_mel_tables_build(sr, n_mels, fmin, fmax, 1, front.ctypes.data))
        fi = front.view(np.int32)
        win, tw, nm, ks, kc, wo, wts = parse(mel_loss.build_tables(1024, 1024, sr, n_mels, fmin, fmax), 1024)
        assert np.array_equal(win.view(np.int32), fi[:1024])
        assert np.array_equal(tw.reshape(-1).view(np.int32), fi[1024:2048])
        assert nm == fi[2048] == n_mels
        assert np.array_equal(ks, fi[2049:2049 + n_mels]) and np.array_equal(kc, fi[2049 + 128:2049 + 128 + n_mels])
        assert np.array_equal(wo, fi[2049 + 256:2049 + 256 + n_mels])
        used = int(wo[-1] + kc[-1])
        assert np.array_equal(wts[:used].view(np.int32), fi[2049 + 384:2049 + 384 + used]), (sr, n_mels, fmin, fmax)


def test_table_build_refusals():
    lib = _lib()
    buf = np.zeros(8 * 2048, np.float32)
    p = buf.ctypes.data

    def refused(args, text):
        assert lib.mg_mel_loss_tables_build(*args) == INVALID, args
        msg = lib.mg_last_error_string()
        assert msg.startswith(b"mg_mel_loss_tables_build") and text in msg, msg

    for n in (64, 100, 4096):
        assert lib.mg_mel_loss_tables_bytes(n) == 0
        refused((n, 64, 22050, 80, 55.0, 9000.0, p), b"n_fft=%d is not a power of two" % n)
    for w in (0, -1, 1025):
        refused((1024, w, 22050, 80, 55.0, 9000.0, p), b"win_length=%d is outside [1, n_fft=1024]" % w)
    refused((1024, 1024, 0, 80, 0.0, 0.0, p), b"sampling_rate=0")
    for m in (0, -1, 513):
        refused((1024, 1024, 22050, m, 55.0, 9000.0, p), b"n_mels=%d is outside [1, 512]" % m)
    for fmin, fmax in ((-1.0, 9000.0), (9000.0, 9000.0), (100.0, 50.0), (0.0, 11026.0), (float("nan"), 9000.0), (0.0, float("nan"))):
        refused((1024, 1024, 22050, 80, fmin, fmax, p), b"fmin=")
    refused((1024, 1024, 22050, 80, 55.0, 9000.0, None), b"tables_host is NULL")
    assert lib.mg_mel_loss_tables_build(1024, 1024, 22050, 80, 0.0, 11025.0, p) == 0


# ------------------------------------------------------------------------------------------------------------------
# the module's dispatch, without a device
# ------------------------------------------------------------------------------------------------------------------
class _FakeCuda(torch.Tensor):
    """A CPU tensor that passes the module's CUDA check, so its dispatch runs without a device."""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def no_device(monkeypatch):
    calls = []

    def fake_forward(an, x, y):
        calls.append((tuple(x.shape), an.n))
        return torch.zeros(())
    monkeypatch.setattr(mel_loss, "_forward", fake_forward)
    return calls


def _fake(*shape, grad=False):
    return torch.zeros(*shape, requires_grad=grad).as_subclass(_FakeCuda)


def test_module_builds_a_graph_only_when_grad_is_needed(no_device):
    loss = mel_loss.MultiResolutionMelLoss()
    assert list(loss.parameters()) == []
    assert loss(_fake(2, 4096), _fake(2, 4096)).grad_fn is None
    with torch.no_grad():
        assert loss(_fake(2, 4096, grad=True), _fake(2, 4096)).grad_fn is None
    with torch.no_grad():                       # a y that requires grad is only refused where a graph could be built
        loss(_fake(2, 4096), _fake(2, 4096, grad=True))
    with torch.inference_mode():
        assert loss(_fake(2, 4096), _fake(2, 4096)).grad_fn is None
    out = loss(_fake(2, 4096, grad=True), _fake(2, 4096))
    assert out.requires_grad and "MelLoss" in type(out.grad_fn).__name__
    out = loss(_fake(2, 1, 4096, grad=True), _fake(2, 1, 4096))      # the generator's [B, 1, L]
    assert out.requires_grad
    assert no_device == [((2, 4096), 1)] * 6


def test_module_refusals(no_device):
    loss = mel_loss.MultiResolutionMelLoss()
    x = _fake(2, 4096, grad=True)
    with pytest.raises(engine.EngineError, match="x must be a CUDA tensor"):
        loss(torch.zeros(2, 4096), _fake(2, 4096))
    with pytest.raises(engine.EngineError, match="y must be a CUDA tensor"):
        loss(x, torch.zeros(2, 4096))
    with pytest.raises(engine.EngineError, match="differ in shape"):
        loss(x, _fake(2, 4097))
    with pytest.raises(engine.EngineError, match="differ in shape"):
        loss(_fake(2, 1, 4096), _fake(2, 4096))
    with pytest.raises(engine.EngineError, match="y requires grad"):
        loss(x, _fake(2, 4096, grad=True))
    for bad in (_fake(4096), _fake(2, 2, 4096), torch.zeros(2, 4096, dtype=torch.float64).as_subclass(_FakeCuda)):
        with pytest.raises(engine.EngineError, match="fp32"):
            loss(bad, bad)
    with pytest.raises(engine.EngineError, match="at least one frame"):
        loss(_fake(2, 255), _fake(2, 255))
    assert no_device == []
    for kw, match in (
            (dict(fft_sizes=(1024, 4096), hop_sizes=(256, 512), win_lengths=(1024, 4096), num_mels=(80, 80)), "n_fft=4096"),
            (dict(fft_sizes=(1000,), win_lengths=(1000,)), "n_fft=1000"),
            (dict(fft_sizes=(64,), hop_sizes=(16,), win_lengths=(64,)), "n_fft=64"),
            (dict(hop_sizes=(0,)), "hop_size 0"),
            (dict(hop_sizes=(1025,)), "hop_size 1025"),
            (dict(win_lengths=(1025,)), "win_length 1025"),
            (dict(win_lengths=(0,)), "win_length 0"),
            (dict(num_mels=(0,)), "num_mels 0"),
            (dict(num_mels=(513,)), "num_mels 513"),
            (dict(fmin=-1.0), "fmin"),
            (dict(fmin=9000.0), "fmin"),
            (dict(fmax=11026.0), "fmax"),
            (dict(sampling_rate=0, fmin=0.0, fmax=None), "sampling_rate 0"),
            (dict(fft_sizes=(1024, 512)), "differ in length"),
            (dict(fft_sizes=(), hop_sizes=(), win_lengths=(), num_mels=()), "0 resolutions"),
            (dict(fft_sizes=(128,) * 9, hop_sizes=(32,) * 9, win_lengths=(128,) * 9, num_mels=(10,) * 9), "9 resolutions")):
        with pytest.raises(engine.EngineError, match=match):
            mel_loss.MultiResolutionMelLoss(**kw)
    m = mel_loss.MultiResolutionMelLoss(fmax=None)
    assert m.fmax == 11025.0
