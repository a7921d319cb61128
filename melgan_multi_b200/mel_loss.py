"""Multi-resolution log-mel L1 loss on hand-written sm_90a kernels (csrc/mg_mel_loss.cu).

``MultiResolutionMelLoss`` is HiFi-GAN's mel reconstruction term ``l1(mel(y_hat), mel(y))`` (without its weight of 45),
averaged over one or more analyses as later GAN vocoders use it.  For each resolution (n_fft, hop, win_length, n_mels),
with the sampling rate, fmin and fmax shared: the audio is zero-padded by ``(n_fft - hop) // 2`` on each side and framed
with center=False (meldataset.py:48 generalised), windowed by a periodic Hann of length win_length centred in n_fft,
``|rfft|``, the librosa Slaney mel filter bank, ``log(clamp(., min=1e-5))``; the resolution's term is the mean of
``|mel_x - mel_y|`` over (item, band, frame), and ``forward(x, y)`` returns the mean over resolutions as a 0-d fp32
tensor.  At the defaults (the reference's config.json analysis) it equals
``F.l1_loss(meldataset.mel_spectrogram(x, ...), meldataset.mel_spectrogram(y, ...))``.  Differentiable with respect to
the predicted audio x (not the target y).  CUDA only, like the rest of the package: there is no CPU fallback.
"""
import ctypes

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import engine as _engine
from .stft_loss import MAX_RESOLUTIONS, _Analysis, _TablesModule, _workspace

MAX_MELS = 512
_LIB = None


def _lib():
    """The library with the mel-loss calls' ctypes signatures, set once."""
    global _LIB
    if _LIB is not None:
        return _LIB
    L = _engine.lib()
    L.mg_mel_loss_tables_bytes.restype = ctypes.c_size_t
    L.mg_mel_loss_tables_bytes.argtypes = [ctypes.c_int]
    L.mg_mel_loss_tables_build.restype = ctypes.c_int
    L.mg_mel_loss_tables_build.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                           ctypes.c_void_p]
    L.mg_mel_loss_frames.restype = ctypes.c_int
    L.mg_mel_loss_frames.argtypes = [ctypes.c_int] * 3
    L.mg_mel_loss_workspace_bytes.restype = ctypes.c_int
    L.mg_mel_loss_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                              ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)]
    L.mg_mel_loss_forward.restype = ctypes.c_int
    L.mg_mel_loss_forward.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                      ctypes.c_void_p]
    L.mg_mel_loss_backward.restype = ctypes.c_int
    L.mg_mel_loss_backward.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_size_t, ctypes.c_void_p]
    _LIB = L
    return L


def build_tables(n_fft, win_length, sampling_rate, n_mels, fmin, fmax):
    """Host float32 table of one resolution (window, twiddles, then n_mels and the sparse filter bank), from the library."""
    L = _lib()
    n = L.mg_mel_loss_tables_bytes(n_fft)
    if n == 0:
        raise _engine.EngineError("MultiResolutionMelLoss: n_fft=%d is not a power of two in [128, 2048]" % n_fft)
    host = np.zeros(n // 4, np.float32)
    _engine.check(L.mg_mel_loss_tables_build(n_fft, win_length, sampling_rate, n_mels, fmin, fmax, host.ctypes.data))
    return host


def frames(n_fft, hop, L):
    """Frames of an L-sample signal at (n_fft, hop): 1 + (L + 2 ((n_fft - hop) // 2) - n_fft) // hop, 0 if unsupported."""
    return _lib().mg_mel_loss_frames(n_fft, hop, L)


def _forward(an, x, y):
    """mg_mel_loss_forward on the current stream: the 0-d loss."""
    B, n = x.shape
    fbytes, _ = an.workspace_bytes(B, n)
    with torch.cuda.device(x.device):
        tabs = an.tables(x.device)
        ws = _workspace(fbytes, x.device)
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        _engine.check(_lib().mg_mel_loss_forward(an.n, tabs, an.n_fft, an.hop, x.data_ptr(), y.data_ptr(), B, n, loss.data_ptr(),
                                                 ws.data_ptr(), fbytes, torch.cuda.current_stream().cuda_stream))
    return loss


class _MelLoss(torch.autograd.Function):
    """The kernels' loss, with d loss / d x from mg_mel_loss_backward, which recomputes the spectra (the forward keeps
    nothing but x and y).  The backward allocates its workspace on the current stream and reads nothing back to the
    host, so it can be captured in a CUDA graph."""

    @staticmethod
    def forward(ctx, x, y, an):
        ctx.an = an
        ctx.save_for_backward(x, y)
        return _forward(an, x, y)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        x, y = ctx.saved_tensors
        an = ctx.an
        B, n = x.shape
        _, bbytes = an.workspace_bytes(B, n)
        g = grad_loss.float().contiguous()
        grad = torch.empty_like(x)
        with torch.cuda.device(x.device):
            ws = _workspace(bbytes, x.device)
            _engine.check(_lib().mg_mel_loss_backward(an.n, an.tables(x.device), an.n_fft, an.hop, x.data_ptr(), y.data_ptr(), B, n,
                                                      g.data_ptr(), grad.data_ptr(), ws.data_ptr(), bbytes,
                                                      torch.cuda.current_stream().cuda_stream))
        return grad, None, None


class MultiResolutionMelLoss(_TablesModule):
    """Multi-resolution log-mel L1 loss: ``forward(x, y) -> loss`` for predicted audio x and target audio y, fp32 CUDA
    tensors [B, L] or [B, 1, L] (the generator's output) of one shape.  The module has no parameters; it keeps each
    device's tables.  The defaults are the reference's analysis (config.json: n_fft 1024, hop 256, win 1024, 80 mels,
    22050 Hz, fmin 55, fmax 9000); several resolutions are passed as equal-length sequences; ``fmax=None`` means
    sampling_rate / 2.

    Supported: n_fft a power of two from 128 to 2048, 1 <= win_length <= n_fft, 1 <= hop <= n_fft, 1 <= n_mels <= 512
    (filters that cover no FFT bin are allowed: their band is log(1e-5) and gets no gradient), 0 <= fmin < fmax <=
    sampling_rate / 2, 1 to 8 resolutions, at least one frame at every resolution and L <= 2^30; anything else raises
    EngineError.  The tables are uploaded to a device by .to() / .cuda() or by the first call there; that first upload
    cannot happen inside a CUDA graph capture, so move the module to the device, or call it once, before capturing.  A
    graph is built only when grad is enabled and x requires grad; a y that requires grad is refused under grad mode.
    NaN or Inf samples propagate to the loss and the gradient as in float64 autograd of the definition; they are never
    clamped away."""

    def __init__(self, fft_sizes=(1024,), hop_sizes=(256,), win_lengths=(1024,), num_mels=(80,), sampling_rate=22050, fmin=55.0,
                 fmax=9000.0):
        super().__init__()
        name = "MultiResolutionMelLoss"
        fft_sizes, hop_sizes, win_lengths, num_mels = (tuple(int(v) for v in a) for a in (fft_sizes, hop_sizes, win_lengths, num_mels))
        if not len(fft_sizes) == len(hop_sizes) == len(win_lengths) == len(num_mels):
            raise _engine.EngineError("%s: fft_sizes, hop_sizes, win_lengths and num_mels differ in length" % name)
        if not 1 <= len(fft_sizes) <= MAX_RESOLUTIONS:
            raise _engine.EngineError("%s: %d resolutions, 1 to %d supported" % (name, len(fft_sizes), MAX_RESOLUTIONS))
        sampling_rate = int(sampling_rate)
        fmax = sampling_rate / 2.0 if fmax is None else float(fmax)
        fmin = float(fmin)
        if sampling_rate < 1:
            raise _engine.EngineError("%s: sampling_rate %d, at least 1 needed" % (name, sampling_rate))
        if not 0.0 <= fmin < fmax <= sampling_rate / 2.0:
            raise _engine.EngineError("%s: fmin %g and fmax %g, 0 <= fmin < fmax <= sampling_rate / 2 needed" % (name, fmin, fmax))
        for n, h, w, m in zip(fft_sizes, hop_sizes, win_lengths, num_mels):
            if not 1 <= h <= n:
                raise _engine.EngineError("%s: hop_size %d outside [1, fft_size %d]" % (name, h, n))
            if not 1 <= w <= n:
                raise _engine.EngineError("%s: win_length %d outside [1, fft_size %d]" % (name, w, n))
            if not 1 <= m <= MAX_MELS:
                raise _engine.EngineError("%s: num_mels %d outside [1, %d]" % (name, m, MAX_MELS))
        self.fft_sizes, self.hop_sizes, self.win_lengths, self.num_mels = fft_sizes, hop_sizes, win_lengths, num_mels
        self.sampling_rate, self.fmin, self.fmax = sampling_rate, fmin, fmax
        host = [build_tables(n, w, sampling_rate, m, fmin, fmax) for n, w, m in zip(fft_sizes, win_lengths, num_mels)]
        self._an = _Analysis(fft_sizes, hop_sizes, host, name, _lib().mg_mel_loss_workspace_bytes)

    def forward(self, x, y):
        name = "MultiResolutionMelLoss"
        for which, t in (("x", x), ("y", y)):
            if not torch.is_tensor(t) or not t.is_cuda:
                raise _engine.EngineError("%s: %s must be a CUDA tensor (no CPU fallback)" % (name, which))
            if t.dtype != torch.float32 or not (t.dim() == 2 or (t.dim() == 3 and t.shape[1] == 1)):
                raise _engine.EngineError("%s: %s must be fp32 [B, L] or [B, 1, L], got %s %s" % (name, which, t.dtype, tuple(t.shape)))
        if x.shape != y.shape:
            raise _engine.EngineError("%s: x %s and y %s differ in shape" % (name, tuple(x.shape), tuple(y.shape)))
        if x.device != y.device:
            raise _engine.EngineError("%s: x and y are on different devices" % name)
        grad = torch.is_grad_enabled()
        if grad and y.requires_grad:
            raise _engine.EngineError("%s: y requires grad; no gradient with respect to the target is computed (pass y.detach())"
                                      % name)
        if x.dim() == 3:
            x, y = x.squeeze(1), y.squeeze(1)
        B, n = x.shape
        short = [(f, h) for f, h in zip(self.fft_sizes, self.hop_sizes) if frames(f, h, n) < 1]
        if B < 1 or short:
            raise _engine.EngineError("%s: [B, L] = [%d, %d]; every resolution needs at least one frame and L <= 2^30 (%s)"
                                      % (name, B, n, ", ".join("n_fft %d hop %d" % s for s in short)))
        x, y = x.contiguous(), y.contiguous()
        if grad and x.requires_grad:
            return _MelLoss.apply(x, y, self._an)
        return _forward(self._an, x, y)
