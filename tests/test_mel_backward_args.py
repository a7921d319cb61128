"""The mel front end's backward without a GPU: every argument mg_mel_spectrogram_backward refuses is reported (an error
code and a message naming it) before anything touches CUDA, mg_mel_backward_workspace_bytes at the frame geometry's
borders, and meldataset.mel_spectrogram building an autograd graph only when grad is enabled and the input requires it.
Fake device addresses stand in for buffers: a call that reached CUDA would fail with MG_ERR_CUDA instead."""
import ctypes

import numpy as np
import pytest
import torch

from kernel_model import mel_option_cases
from melgan_multi_b200 import engine, meldataset

INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL


def _lib():
    return meldataset._lib()


def backward(tables=256, audio=256, grad_mel=256, grad_audio=256, B=2, L=8192, ws=256, ws_bytes=None):
    lib = _lib()
    nbytes = lib.mg_mel_backward_workspace_bytes(B, L) if ws_bytes is None else ws_bytes
    rc = lib.mg_mel_spectrogram_backward(tables, audio, grad_mel, grad_audio, B, L, ws, nbytes, None)
    return rc, lib.mg_last_error_string()


def test_refusals_before_any_launch():
    for null in ("tables", "audio", "grad_mel", "grad_audio", "ws"):
        rc, msg = backward(**{null: None})
        assert rc == INVALID and b"mg_mel_spectrogram_backward: bad argument" in msg, null
    for B, L in ((0, 8192), (-1, 8192), (2, 0), (2, -5)):
        rc, msg = backward(B=B, L=L, ws_bytes=1 << 30)
        assert rc == INVALID and b"bad argument" in msg, (B, L)
    rc, msg = backward(L=255, ws_bytes=1 << 30)
    assert rc == INVALID and b"255 samples are fewer than one frame" in msg
    rc, msg = backward(tables=264)
    assert rc == INVALID and b"tables must be 16-byte aligned" in msg
    rc, msg = backward(ws=264)
    assert rc == INVALID and b"workspace must be 16-byte aligned" in msg
    need = _lib().mg_mel_backward_workspace_bytes(2, 8192)
    rc, msg = backward(ws_bytes=need - 1)
    assert rc == WS_SMALL and (b"workspace of %d bytes, %d needed" % (need - 1, need)) in msg
    rc, msg = backward(ws_bytes=0)
    assert rc == WS_SMALL
    # B * ceil(T / 2) CTAs past 2^31 - 1: 2^17 items of 2^15 + 1 frame pairs
    B, L = 1 << 17, 256 * (2 * ((1 << 15) + 1))
    rc, msg = backward(B=B, L=L, ws_bytes=1 << 62)
    assert rc == INVALID and b"exceed 2^31 - 1 CTAs" in msg


def test_workspace_bytes_follow_the_frame_geometry():
    lib = _lib()
    for L in (256, 257, 511, 512, 513, 767, 768, 1023, 1024, 1025, 8191, 8192, 8193, 220500):
        T = lib.mg_mel_frames(L)
        assert T == L // 256
        for B in (1, 3, 37, 70000):
            assert lib.mg_mel_backward_workspace_bytes(B, L) == B * T * 1024 * 4, (B, L)
    for B, L in ((0, 8192), (1, 0), (1, 255), (-3, 8192), (3, -1)):
        assert lib.mg_mel_backward_workspace_bytes(B, L) == 0, (B, L)
    pairs = 1 << 15
    L = 256 * 2 * pairs
    assert lib.mg_mel_backward_workspace_bytes((2 ** 31 - 1) // pairs, L) > 0
    assert lib.mg_mel_backward_workspace_bytes((2 ** 31 - 1) // pairs + 1, L) == 0


def test_same_parity_filters_share_no_bin():
    """The backward accumulates M^T (g / s) in two passes, even filters then odd ones, and relies on the filters of one
    parity covering disjoint bin runs; every table mg_mel_tables_build makes has that property."""
    lib = engine.lib()
    lib.mg_mel_tables_bytes.restype = ctypes.c_size_t
    lib.mg_mel_tables_build.restype = ctypes.c_int
    lib.mg_mel_tables_build.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
    n = lib.mg_mel_tables_bytes()
    for sr, n_mels, fmin, fmax, norm in mel_option_cases():
        host = np.zeros((n + 3) // 4, np.float32)
        engine.check(lib.mg_mel_tables_build(sr, n_mels, fmin, fmax, norm, host.ctypes.data))
        ints = host.view(np.int32)
        base = (1024 + 2 * 512) + 1   # win, tw, n_mels
        assert ints[base - 1] == n_mels
        kstart, kcount = ints[base:base + 128], ints[base + 128:base + 256]
        for par in (0, 1):
            cover = np.zeros(513, int)
            for m in range(par, n_mels, 2):
                cover[kstart[m]:kstart[m] + kcount[m]] += 1
            assert cover.max() <= 1, (sr, n_mels, fmin, fmax, norm, par)


class _FakeCuda(torch.Tensor):
    """A CPU tensor that passes mel_spectrogram's CUDA check, so the wrapper's dispatch runs without a device."""

    @property
    def is_cuda(self):
        return True


@pytest.fixture
def no_device(monkeypatch):
    calls = []

    def fake_forward(y2, tab, num_mels, T):
        calls.append((tuple(y2.shape), y2.dtype, num_mels, T))
        return torch.zeros((y2.shape[0], num_mels, T))
    monkeypatch.setattr(meldataset, "_forward", fake_forward)
    monkeypatch.setattr(meldataset, "_tables", lambda *a: torch.zeros(4))
    return calls


def _call(y):
    return meldataset.mel_spectrogram(y, 1024, 80, 22050, 256, 1024, 55.0, 9000.0, check_range=False)


def test_wrapper_builds_a_graph_only_when_grad_is_needed(no_device):
    y = torch.zeros(2, 1024).as_subclass(_FakeCuda)
    out = _call(y)
    assert out.grad_fn is None and not out.requires_grad
    leaf = torch.zeros(2, 1024, requires_grad=True)
    with torch.no_grad():
        out = _call(leaf.as_subclass(_FakeCuda))
    assert out.grad_fn is None and not out.requires_grad
    with torch.inference_mode():
        out = _call(torch.zeros(2, 1024).as_subclass(_FakeCuda))
    assert out.grad_fn is None
    out = _call(leaf.as_subclass(_FakeCuda))
    assert out.requires_grad and "MelSpectrogram" in type(out.grad_fn).__name__
    one = _call(torch.zeros(1024, dtype=torch.float64, requires_grad=True).as_subclass(_FakeCuda))
    assert one.shape == (80, 4) and one.requires_grad
    # every path launches the same forward on the same [B, L] fp32 view
    assert no_device == [((2, 1024), torch.float32, 80, 4)] * 4 + [((1, 1024), torch.float32, 80, 4)]


def test_wrapper_refuses_other_analyses_with_grad():
    y = torch.zeros(1024, requires_grad=True).as_subclass(_FakeCuda)
    with pytest.raises(engine.EngineError):
        meldataset.mel_spectrogram(y, 2048, 80, 22050, 256, 1024, 55.0, 9000.0)
    with pytest.raises(engine.EngineError):
        meldataset.mel_spectrogram(y, 1024, 80, 22050, 256, 1024, 55.0, 9000.0, center=True)
