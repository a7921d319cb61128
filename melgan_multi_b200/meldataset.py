"""GPU drop-in for ``mel_spectrogram`` of the reference's meldataset.py (/root/reference/meldataset.py:44-55).

Same signature and semantics -- zero-pad by (n_fft - hop_size) / 2, magnitude STFT with a periodic Hann window and
center=False, Slaney-normalised triangular mel filters (librosa ``norm=1`` of the API the reference was written against),
``log(clip(x, 1e-5))`` -- computed by one hand-written kernel (csrc/mg_mel.cu) on CUDA tensors, so the training loop's
validation pass (train.py:164) and a GPU-side data pipeline never go through librosa on the host.  When grad is enabled and
the input requires grad, the output is differentiable with respect to the audio (two more kernels compute the gradient),
so a mel-reconstruction loss on generated audio trains the generator; otherwise no graph is built.  Only the analysis
parameters of the reference's config.json (n_fft = win_size = 1024, hop_size = 256, center=False) exist as a kernel; anything
else raises.  CUDA only, like the rest of the package.  ``MelDataset`` (file IO, random cropping) is the reference's
loader and out of scope.
"""
import ctypes

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import engine as _engine

_TABLES = {}


def _tables(device, sampling_rate, num_mels, fmin, fmax, norm):
    key = (device, int(sampling_rate), int(num_mels), float(fmin), float(fmax), int(norm))
    t = _TABLES.get(key)
    if t is None:
        L = _engine.lib()
        L.mg_mel_tables_bytes.restype = ctypes.c_size_t
        L.mg_mel_tables_build.restype = ctypes.c_int
        L.mg_mel_tables_build.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
        n = L.mg_mel_tables_bytes()
        host = np.zeros((n + 3) // 4, np.float32)
        _engine.check(L.mg_mel_tables_build(key[1], key[2], key[3], key[4], key[5], host.ctypes.data))
        t = torch.from_numpy(host).to(device)
        _TABLES[key] = t
    return t


def mel_spectrogram(y, n_fft, num_mels, sampling_rate, hop_size, win_size, fmin, fmax, center=False, check_range=True,
                    norm=1):
    """y: CUDA float tensor [L] or [B, L] in [-1, 1] -> log-mel [num_mels, T] or [B, num_mels, T] (T = L / hop_size for whole
    hops).  ``check_range`` reproduces the reference's two asserts (one host sync); ``norm``: 1 = Slaney area normalisation
    (the reference's call), 0 = none, 2 = L1.  Non-finite audio (with check_range=False) propagates as in the reference's
    ``np.log(np.clip(x, 1e-5, None))``: every frame that reads a NaN or Inf sample is NaN in the bands its spectrum
    makes NaN (an Inf sample can also give +Inf), never log(1e-5); the other frames and items are unchanged.  The
    gradient is NaN exactly where torch autograd's float64 gradient is."""
    if not torch.is_tensor(y) or not y.is_cuda:
        raise _engine.EngineError("melgan_multi_b200.meldataset.mel_spectrogram needs a CUDA tensor (no CPU fallback; the "
                                  "reference's host path is librosa)")
    if (n_fft, hop_size, win_size) != (1024, 256, 1024) or center:
        raise _engine.EngineError("mel_spectrogram: the kernel implements the reference's analysis (n_fft = win_size = 1024, "
                                  "hop_size = 256, center=False) only")
    squeeze = y.dim() == 1
    y2 = (y[None] if squeeze else y).float().contiguous()
    if y2.dim() != 2:
        raise _engine.EngineError("mel_spectrogram: y must be [L] or [B, L]")
    if check_range:  # meldataset.py:45-46
        lo, hi = torch.aminmax(y2)
        assert float(lo) >= -1.0
        assert float(hi) <= 1.0
    L = _lib()
    B, n = y2.shape
    T = L.mg_mel_frames(n)
    if T < 1:
        raise _engine.EngineError("mel_spectrogram: %d samples are fewer than one frame" % n)
    tab = _tables(y2.device, sampling_rate, num_mels, fmin, fmax, norm)
    if torch.is_grad_enabled() and y2.requires_grad:
        out = _MelSpectrogram.apply(y2, tab, num_mels, T)
    else:
        out = _forward(y2, tab, num_mels, T)
    return out[0] if squeeze else out


def _lib():
    L = _engine.lib()
    L.mg_mel_frames.restype = ctypes.c_int
    L.mg_mel_frames.argtypes = [ctypes.c_int]
    L.mg_mel_spectrogram.restype = ctypes.c_int
    L.mg_mel_spectrogram.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.mg_mel_backward_workspace_bytes.restype = ctypes.c_size_t
    L.mg_mel_backward_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    L.mg_mel_spectrogram_backward.restype = ctypes.c_int
    L.mg_mel_spectrogram_backward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                              ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return L


def _forward(y2, tab, num_mels, T):
    """mg_mel_spectrogram on the current stream: y2 [B, L] contiguous fp32 -> [B, num_mels, T]."""
    B, n = y2.shape
    out = torch.empty((B, num_mels, T), dtype=torch.float32, device=y2.device)
    with torch.cuda.device(y2.device):
        _engine.check(_lib().mg_mel_spectrogram(tab.data_ptr(), y2.data_ptr(), out.data_ptr(), B, n,
                                                torch.cuda.current_stream().cuda_stream))
    return out


class _MelSpectrogram(torch.autograd.Function):
    """The same kernel output, with d loss / d audio from mg_mel_spectrogram_backward.  The backward allocates its
    workspace on the current stream and reads nothing back to the host, so it can be captured in a CUDA graph."""

    @staticmethod
    def forward(ctx, y2, tab, num_mels, T):
        ctx.save_for_backward(y2, tab)
        return _forward(y2, tab, num_mels, T)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_mel):
        y2, tab = ctx.saved_tensors
        B, n = y2.shape
        g = grad_mel.contiguous().float()
        grad = torch.empty_like(y2)
        L = _lib()
        nbytes = L.mg_mel_backward_workspace_bytes(B, n)
        with torch.cuda.device(y2.device):
            ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=y2.device)
            _engine.check(L.mg_mel_spectrogram_backward(tab.data_ptr(), y2.data_ptr(), g.data_ptr(), grad.data_ptr(), B, n,
                                                        ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream))
        return grad, None, None, None
