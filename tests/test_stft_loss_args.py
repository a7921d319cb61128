"""The multi-resolution STFT loss without a GPU: every argument the C calls refuse is reported (an error code and a
message naming it) before anything touches CUDA, the frame count and workspace sizes at the frame geometry's borders,
the tables against float64 numpy rounded once, and stft_loss.MultiResolutionSTFTLoss building an autograd graph only
when grad is enabled and x requires it.  Fake device addresses stand in for buffers: a call that reached CUDA would fail
with MG_ERR_CUDA instead."""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, stft_loss

INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL
DEFAULT = ((1024, 2048, 512), (120, 240, 50), (600, 1200, 240))


def _lib():
    return stft_loss._lib()


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _sizes(n_fft, hop, B, L):
    f, b = ctypes.c_size_t(), ctypes.c_size_t()
    rc = _lib().mg_stft_loss_workspace_bytes(len(n_fft), _ints(n_fft), _ints(hop), B, L, ctypes.byref(f), ctypes.byref(b))
    return rc, f.value, b.value


def _call(which, n_fft=(1024, 2048, 512), hop=(120, 240, 50), B=2, L=8192, tables=None, n_res=None, ws_bytes=None, **ptr):
    lib = _lib()
    n_res = len(n_fft) if n_res is None else n_res
    tabs = (ctypes.c_void_p * max(1, len(n_fft)))(*([256] * len(n_fft) if tables is None else tables))
    rc, f, b = _sizes(n_fft, hop, B, L)
    p = dict(x=256, y=512, sc=768, mag=1024, gsc=1280, gmag=1536, fws=2048, gx=4096, ws=8192, tabs=tabs, n_fft_arr=_ints(n_fft),
             hop_arr=_ints(hop))
    p.update(ptr)
    if which == "forward":
        rc = lib.mg_stft_loss_forward(n_res, p["tabs"], p["n_fft_arr"], p["hop_arr"], p["x"], p["y"], B, L, p["sc"], p["mag"], p["ws"],
                                      f if ws_bytes is None else ws_bytes, None)
    else:
        rc = lib.mg_stft_loss_backward(n_res, p["tabs"], p["n_fft_arr"], p["hop_arr"], p["x"], p["y"], B, L, p["gsc"], p["gmag"], p["fws"],
                                       p["gx"], p["ws"], b if ws_bytes is None else ws_bytes, None)
    return rc, lib.mg_last_error_string().decode()


@pytest.mark.parametrize("which", ["forward", "backward"])
def test_refusals_before_any_launch(which):
    fn = "mg_stft_loss_" + which
    ptrs = ["x", "y", "sc", "mag", "ws", "tabs", "n_fft_arr", "hop_arr"] if which == "forward" else \
        ["x", "y", "gsc", "gmag", "fws", "gx", "ws", "tabs", "n_fft_arr", "hop_arr"]
    names = dict(sc="sc_loss", mag="mag_loss", gsc="grad_sc", gmag="grad_mag", fws="forward_workspace", gx="grad_x", ws="workspace",
                 tabs="tables", n_fft_arr="n_fft", hop_arr="hop")
    for k in ptrs:
        rc, msg = _call(which, **{k: None})
        assert rc == INVALID and msg.startswith(fn) and "%s is NULL" % names.get(k, k) in msg, (k, msg)
    for k, align in (("x", 4), ("y", 4), ("sc", 4), ("mag", 4), ("gsc", 4), ("gmag", 4), ("gx", 4), ("ws", 16), ("fws", 16)):
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
    for h in (0, -3):
        rc, msg = _call(which, hop=(120, 240, h))
        assert rc == INVALID and "hop[2]=%d, at least 1 needed" % h in msg, msg
    for L in (1024, 1000, 600):
        rc, msg = _call(which, L=L)
        assert rc == INVALID and "L=%d samples, reflect padding by n_fft[1]/2=1024 needs more" % L in msg, msg
    rc, msg = _call(which, L=(1 << 30) + 1, ws_bytes=1 << 62)
    assert rc == INVALID and "L=1073741825 samples, at most 2^30 supported" in msg, msg
    for B in (0, -1):
        rc, msg = _call(which, B=B)
        assert rc == INVALID and "B=%d, at least 1 item needed" % B in msg, msg
    for n_res in (0, 9, -1):
        rc, msg = _call(which, n_res=n_res)
        assert rc == INVALID and "n_res=%d resolutions, 1 to 8 supported" % n_res in msg, msg
    rc, msg = _call(which, n_fft=(128,) * 9, hop=(1,) * 9)
    assert rc == INVALID and "n_res=9" in msg
    # B T CTAs past 2^31 - 1 at hop 1: 2^16 items of 2^15 + 1 frames
    rc, msg = _call(which, n_fft=(128,), hop=(1,), B=1 << 16, L=1 << 15, ws_bytes=1 << 62)
    assert rc == INVALID and "B=65536 x 32769 frames of resolution 0 exceed 2^31 - 1 CTAs" in msg, msg
    # the gather's B ceil(L / 256) CTAs past 2^31 - 1 with few frames: hop = L
    L = 1 << 30
    rc, msg = _call(which, n_fft=(128,), hop=(L,), B=1 << 9, L=L, ws_bytes=1 << 62)
    assert rc == INVALID and "sample blocks exceed 2^31 - 1 CTAs" in msg, msg
    rc0, f, b = _sizes((1024, 2048, 512), (120, 240, 50), 2, 8192)
    need = f if which == "forward" else b
    rc, msg = _call(which, ws_bytes=need - 1)
    assert rc == WS_SMALL and "workspace of %d bytes, %d needed" % (need - 1, need) in msg, msg
    rc, msg = _call(which, ws_bytes=0)
    assert rc == WS_SMALL


def test_workspace_call_refusals():
    lib = _lib()
    f = ctypes.c_size_t()
    rc = lib.mg_stft_loss_workspace_bytes(1, _ints([512]), _ints([50]), 2, 8192, ctypes.byref(f), None)
    assert rc == INVALID and b"backward_bytes is NULL" in lib.mg_last_error_string()
    rc = lib.mg_stft_loss_workspace_bytes(1, None, _ints([50]), 2, 8192, ctypes.byref(f), ctypes.byref(f))
    assert rc == INVALID and b"n_fft is NULL" in lib.mg_last_error_string()
    assert _sizes((512,), (50,), 2, 256)[0] == INVALID
    assert _sizes((512,), (0,), 2, 8192)[0] == INVALID
    assert _sizes((512,) * 9, (50,) * 9, 2, 8192)[0] == INVALID
    assert _sizes((512,), (50,), 1, (1 << 30) + 1)[0] == INVALID
    assert _sizes((512,), (1 << 20,), 1, 1 << 30)[0] == 0
    assert lib.mg_stft_loss_frames(512, 50, (1 << 30) + 1) == 0


def _frames(L, h):
    return 1 + L // h


@pytest.mark.parametrize("n,h", [(128, 1), (128, 128), (256, 64), (512, 50), (1024, 120), (1024, 1024), (2048, 240),
                                 (2048, 4096)])
def test_frames_and_workspace_follow_the_frame_geometry(n, h):
    lib = _lib()
    Ls = {n // 2 + 1, n // 2 + 2, 8192, 220500}
    for m in range(max(1, (n // 2 + 1) // h), (n // 2 + 1) // h + 4):
        Ls |= {m * h - 1, m * h, m * h + 1}
    for L in sorted(v for v in Ls if v > n // 2):
        T = lib.mg_stft_loss_frames(n, h, L)
        assert T == _frames(L, h), (n, h, L)
        for B in (1, 3, 16):
            rc, f, b = _sizes((n,), (h,), B, L)
            assert rc == 0
            assert f == 256 + -(-3 * B * T * 4 // 256) * 256, (B, L)
            assert b == B * T * n * 4, (B, L)
    assert lib.mg_stft_loss_frames(n, h, n // 2) == 0
    assert lib.mg_stft_loss_frames(n, 0, 8192) == 0
    assert lib.mg_stft_loss_frames(n + 1, h, 8192) == 0


def test_default_workspace_sums_and_takes_the_largest_frame_buffer():
    B, L = 16, 8192
    rc, f, b = _sizes(*DEFAULT[:2], B, L)
    T = [_frames(L, h) for h in DEFAULT[1]]
    assert rc == 0
    assert f == 256 + sum(-(-3 * B * t * 4 // 256) * 256 for t in T)
    assert b == max(B * t * n * 4 for t, n in zip(T, DEFAULT[0]))


@pytest.mark.parametrize("n", [128, 256, 512, 1024, 2048])
def test_tables_equal_float64_rounded_once(n):
    lib = _lib()
    assert lib.mg_stft_loss_tables_bytes(n) == 8 * n
    for w in sorted({1, 2, 3, n // 2 - 1, n // 2, 600 if n >= 600 else n - 1, n - 1, n}):
        host = stft_loss.build_tables(n, w)
        win = np.zeros(n)
        left = (n - w) // 2
        win[left:left + w] = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(w) / w) if w > 1 else 1.0
        assert np.array_equal(host[:n], win.astype(np.float32)), (n, w)
        k = np.arange(n // 2)
        tw = np.stack([np.cos(2 * np.pi * k / n), -np.sin(2 * np.pi * k / n)], 1).astype(np.float32).ravel()
        assert np.array_equal(host[n:], tw), (n, w)
        # the same window torch.stft pads: hann_window(w, periodic=True) centred in n
        ref = torch.nn.functional.pad(torch.hann_window(w, periodic=True, dtype=torch.float64), (left, n - w - left))
        assert np.abs(host[:n] - ref.numpy()).max() <= 2 ** -24


def test_table_build_refusals():
    lib = _lib()
    buf = np.zeros(2048 * 2, np.float32)
    for n in (64, 100, 4096):
        assert lib.mg_stft_loss_tables_bytes(n) == 0
        assert lib.mg_stft_loss_tables_build(n, 64, buf.ctypes.data) == INVALID
        assert b"n_fft=%d is not a power of two" % n in lib.mg_last_error_string()
    for w in (0, -1, 1025):
        assert lib.mg_stft_loss_tables_build(1024, w, buf.ctypes.data) == INVALID
        assert b"win_length=%d is outside [1, n_fft=1024]" % w in lib.mg_last_error_string()
    assert lib.mg_stft_loss_tables_build(1024, 600, None) == INVALID
    assert b"tables_host is NULL" in lib.mg_last_error_string()


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
        z = torch.zeros(())
        return z.clone(), z.clone(), torch.zeros(4)
    monkeypatch.setattr(stft_loss, "_forward", fake_forward)
    return calls


def _fake(*shape, grad=False):
    return torch.zeros(*shape, requires_grad=grad).as_subclass(_FakeCuda)


def test_module_builds_a_graph_only_when_grad_is_needed(no_device):
    loss = stft_loss.MultiResolutionSTFTLoss()
    assert list(loss.parameters()) == []
    sc, mag = loss(_fake(2, 4096), _fake(2, 4096))
    assert sc.grad_fn is None and mag.grad_fn is None
    with torch.no_grad():
        sc, mag = loss(_fake(2, 4096, grad=True), _fake(2, 4096))
    assert sc.grad_fn is None
    with torch.no_grad():                       # a y that requires grad is only refused where a graph could be built
        loss(_fake(2, 4096), _fake(2, 4096, grad=True))
    with torch.inference_mode():
        sc, mag = loss(_fake(2, 4096), _fake(2, 4096))
    assert sc.grad_fn is None
    sc, mag = loss(_fake(2, 4096, grad=True), _fake(2, 4096))
    assert sc.requires_grad and mag.requires_grad and "STFTLoss" in type(sc.grad_fn).__name__
    assert sc.grad_fn is mag.grad_fn
    assert no_device == [((2, 4096), 3)] * 5


def test_module_refusals(no_device):
    loss = stft_loss.MultiResolutionSTFTLoss()
    x = _fake(2, 4096, grad=True)
    with pytest.raises(engine.EngineError, match="x must be a CUDA tensor"):
        loss(torch.zeros(2, 4096), _fake(2, 4096))
    with pytest.raises(engine.EngineError, match="y must be a CUDA tensor"):
        loss(x, torch.zeros(2, 4096))
    with pytest.raises(engine.EngineError, match="differ in shape"):
        loss(x, _fake(2, 4097))
    with pytest.raises(engine.EngineError, match="y requires grad"):
        loss(x, _fake(2, 4096, grad=True))
    with pytest.raises(engine.EngineError, match="fp32"):
        loss(_fake(4096), _fake(4096))
    with pytest.raises(engine.EngineError, match="fp32"):
        loss(torch.zeros(2, 4096, dtype=torch.float64).as_subclass(_FakeCuda), _fake(2, 4096))
    with pytest.raises(engine.EngineError, match="needs L > 1024"):
        loss(_fake(2, 1024), _fake(2, 1024))
    assert no_device == []
    for args, match in (
            (((1024, 4096), (120, 240), (600, 1200)), "n_fft=4096"),
            (((1024, 1000), (120, 240), (600, 1000)), "n_fft=1000"),
            (((64,), (16,), (64,)), "n_fft=64"),
            (((1024,), (0,), (600,)), "hop_size 0"),
            (((1024,), (120,), (1025,)), "win_length 1025"),
            (((1024,), (120,), (0,)), "win_length 0"),
            (((1024, 512), (120,), (600, 240)), "differ in length"),
            (((), (), ()), "0 resolutions"),
            (((128,) * 9, (50,) * 9, (128,) * 9), "9 resolutions")):
        with pytest.raises(engine.EngineError, match=match):
            stft_loss.MultiResolutionSTFTLoss(*args)
    with pytest.raises(engine.EngineError, match="Hann"):
        stft_loss.MultiResolutionSTFTLoss(window="hamming_window")
