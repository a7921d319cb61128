"""Multi-resolution STFT loss on hand-written sm_90a kernels (csrc/mg_stft_loss.cu).

``MultiResolutionSTFTLoss`` has the arguments, defaults and result of Parallel WaveGAN's module of that name, the
auxiliary loss of Parallel WaveGAN and Multi-band MelGAN: for each resolution (n_fft, hop, win_length) with a periodic
Hann window, ``X = torch.stft(x, n_fft, hop, win_length, window, center=True, pad_mode="reflect")``, the magnitudes
``sqrt(clamp(|X|^2, min=1e-7))`` of x and y, the spectral convergence ``||y_mag - x_mag||_F / ||y_mag||_F`` and the
log-magnitude distance ``mean |log y_mag - log x_mag|``; ``forward(x, y)`` returns their means over the resolutions as
two 0-d fp32 tensors ``(sc_loss, mag_loss)``.  Both are differentiable with respect to the predicted audio x (not the
target y).  CUDA only, like the rest of the package: there is no CPU fallback.
"""
import ctypes

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import engine as _engine

MAX_RESOLUTIONS = 8
_LIB = None


def _lib():
    """The library with the STFT-loss calls' ctypes signatures, set once."""
    global _LIB
    if _LIB is not None:
        return _LIB
    L = _engine.lib()
    L.mg_stft_loss_tables_bytes.restype = ctypes.c_size_t
    L.mg_stft_loss_tables_bytes.argtypes = [ctypes.c_int]
    L.mg_stft_loss_tables_build.restype = ctypes.c_int
    L.mg_stft_loss_tables_build.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    L.mg_stft_loss_frames.restype = ctypes.c_int
    L.mg_stft_loss_frames.argtypes = [ctypes.c_int] * 3
    L.mg_stft_loss_workspace_bytes.restype = ctypes.c_int
    L.mg_stft_loss_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                               ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)]
    L.mg_stft_loss_forward.restype = ctypes.c_int
    L.mg_stft_loss_forward.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.mg_stft_loss_backward.restype = ctypes.c_int
    L.mg_stft_loss_backward.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    _LIB = L
    return L


def build_tables(n_fft, win_length):
    """Host float32 table of one resolution (window zero-padded to n_fft, then the twiddles), from the library."""
    L = _lib()
    n = L.mg_stft_loss_tables_bytes(n_fft)
    if n == 0:
        raise _engine.EngineError("MultiResolutionSTFTLoss: n_fft=%d is not a power of two in [128, 2048]" % n_fft)
    host = np.zeros(n // 4, np.float32)
    _engine.check(L.mg_stft_loss_tables_build(n_fft, win_length, host.ctypes.data))
    return host


class _Analysis:
    """The resolutions of one loss module as the C calls take them, and each device's uploaded tables.  Tables are
    uploaded with a copy from pageable host memory, which a CUDA graph capture forbids: tables() uploads them before any
    capture (the module calls it from .to() / .cuda()), and a first call on a device inside a capture raises EngineError.
    owner names the module in messages; workspace_call is its mg_*_workspace_bytes."""

    def __init__(self, fft_sizes, hop_sizes, host, owner="MultiResolutionSTFTLoss", workspace_call=None):
        self.n = len(fft_sizes)
        self.n_fft = (ctypes.c_int * self.n)(*fft_sizes)
        self.hop = (ctypes.c_int * self.n)(*hop_sizes)
        self.host = host
        self.owner = owner
        self.workspace_call = workspace_call or _lib().mg_stft_loss_workspace_bytes
        self.device = {}

    def tables(self, device):
        d = self.device.get(device)
        if d is None:
            if torch.cuda.is_current_stream_capturing():
                raise _engine.EngineError("%s: the tables for %s are not uploaded yet and a CUDA graph capture forbids the "
                                          "copy; call the module once, or move it with .to(%s), before capturing"
                                          % (self.owner, device, device))
            tabs = [torch.from_numpy(h).to(device) for h in self.host]
            d = (tabs, (ctypes.c_void_p * self.n)(*[t.data_ptr() for t in tabs]))
            self.device[device] = d
        return d[1]

    def workspace_bytes(self, B, L):
        f, b = ctypes.c_size_t(), ctypes.c_size_t()
        _engine.check(self.workspace_call(self.n, self.n_fft, self.hop, B, L, ctypes.byref(f), ctypes.byref(b)))
        return f.value, b.value


class _TablesModule(torch.nn.Module):
    """A loss module whose .to(device) / .cuda() upload its _Analysis's tables there, so a first call inside a CUDA
    graph capture finds them."""

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        dev = fn(torch.empty(0)).device
        if dev.type == "cuda":
            self._an.tables(torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device()))
        return out


def _workspace(nbytes, device):
    return torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=device)


def _forward(an, x, y):
    """mg_stft_loss_forward on the current stream: (sc, mag, forward workspace)."""
    B, n = x.shape
    fbytes, _ = an.workspace_bytes(B, n)
    with torch.cuda.device(x.device):
        tabs = an.tables(x.device)
        ws = _workspace(fbytes, x.device)
        sc = torch.empty((), dtype=torch.float32, device=x.device)
        mag = torch.empty((), dtype=torch.float32, device=x.device)
        _engine.check(_lib().mg_stft_loss_forward(an.n, tabs, an.n_fft, an.hop, x.data_ptr(), y.data_ptr(), B, n, sc.data_ptr(),
                                                  mag.data_ptr(), ws.data_ptr(), fbytes, torch.cuda.current_stream().cuda_stream))
    return sc, mag, ws


class _STFTLoss(torch.autograd.Function):
    """The kernels' losses, with d loss / d x from mg_stft_loss_backward.  The backward allocates its workspace on the
    current stream and reads nothing back to the host, so it can be captured in a CUDA graph."""

    @staticmethod
    def forward(ctx, x, y, an):
        sc, mag, ws = _forward(an, x, y)
        ctx.an = an
        ctx.save_for_backward(x, y, ws)
        return sc, mag

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_sc, grad_mag):
        x, y, fws = ctx.saved_tensors
        an = ctx.an
        B, n = x.shape
        fbytes, bbytes = an.workspace_bytes(B, n)
        gsc = grad_sc.float().contiguous()
        gmag = grad_mag.float().contiguous()
        grad = torch.empty_like(x)
        with torch.cuda.device(x.device):
            ws = _workspace(bbytes, x.device)
            _engine.check(_lib().mg_stft_loss_backward(an.n, an.tables(x.device), an.n_fft, an.hop, x.data_ptr(), y.data_ptr(), B, n,
                                                       gsc.data_ptr(), gmag.data_ptr(), fws.data_ptr(), grad.data_ptr(),
                                                       ws.data_ptr(), bbytes, torch.cuda.current_stream().cuda_stream))
        return grad, None, None


class MultiResolutionSTFTLoss(_TablesModule):
    """Parallel WaveGAN's multi-resolution STFT loss: ``forward(x, y) -> (sc_loss, mag_loss)`` for predicted audio x and
    target audio y, fp32 CUDA tensors [B, L] of one shape.  The module has no parameters; it keeps each device's tables.

    Supported: n_fft a power of two from 128 to 2048, 1 <= win_length <= n_fft, hop >= 1, 1 to 8 resolutions, and
    n_fft / 2 < L <= 2^30 (torch.stft's reflect padding needs the lower bound); anything else raises EngineError.  The
    tables are uploaded to a device by .to() / .cuda() or by the first call there; that first upload cannot happen inside
    a CUDA graph capture, so move the module to the device, or call it once, before capturing.  A graph is built only when
    grad is enabled and x requires grad; a y that requires grad is refused under grad mode (no gradient with respect to
    the target is computed).  NaN or Inf samples propagate to the losses and the gradient as in float64 autograd of
    the definition; they are never clamped away."""

    def __init__(self, fft_sizes=(1024, 2048, 512), hop_sizes=(120, 240, 50), win_lengths=(600, 1200, 240),
                 window="hann_window"):
        super().__init__()
        if window != "hann_window":
            raise _engine.EngineError("MultiResolutionSTFTLoss: only the periodic Hann window is implemented")
        fft_sizes, hop_sizes, win_lengths = (tuple(int(v) for v in a) for a in (fft_sizes, hop_sizes, win_lengths))
        if not len(fft_sizes) == len(hop_sizes) == len(win_lengths):
            raise _engine.EngineError("MultiResolutionSTFTLoss: fft_sizes, hop_sizes and win_lengths differ in length")
        if not 1 <= len(fft_sizes) <= MAX_RESOLUTIONS:
            raise _engine.EngineError("MultiResolutionSTFTLoss: %d resolutions, 1 to %d supported" % (len(fft_sizes), MAX_RESOLUTIONS))
        for n, h, w in zip(fft_sizes, hop_sizes, win_lengths):
            if h < 1:
                raise _engine.EngineError("MultiResolutionSTFTLoss: hop_size %d, at least 1 needed" % h)
            if not 1 <= w <= n:
                raise _engine.EngineError("MultiResolutionSTFTLoss: win_length %d outside [1, fft_size %d]" % (w, n))
        self.fft_sizes, self.hop_sizes, self.win_lengths = fft_sizes, hop_sizes, win_lengths
        self._an = _Analysis(fft_sizes, hop_sizes, [build_tables(n, w) for n, w in zip(fft_sizes, win_lengths)])

    def forward(self, x, y):
        for name, t in (("x", x), ("y", y)):
            if not torch.is_tensor(t) or not t.is_cuda:
                raise _engine.EngineError("MultiResolutionSTFTLoss: %s must be a CUDA tensor (no CPU fallback)" % name)
            if t.dtype != torch.float32 or t.dim() != 2:
                raise _engine.EngineError("MultiResolutionSTFTLoss: %s must be fp32 [B, L], got %s %s" % (name, t.dtype, tuple(t.shape)))
        if x.shape != y.shape:
            raise _engine.EngineError("MultiResolutionSTFTLoss: x %s and y %s differ in shape" % (tuple(x.shape), tuple(y.shape)))
        if x.device != y.device:
            raise _engine.EngineError("MultiResolutionSTFTLoss: x and y are on different devices")
        grad = torch.is_grad_enabled()
        if grad and y.requires_grad:
            raise _engine.EngineError("MultiResolutionSTFTLoss: y requires grad; no gradient with respect to the target is "
                                      "computed (pass y.detach())")
        B, n = x.shape
        short = [f for f in self.fft_sizes if n <= f // 2]
        if B < 1 or short:
            raise _engine.EngineError("MultiResolutionSTFTLoss: [B, L] = [%d, %d]; reflect padding by fft_size / 2 needs L > %d"
                                      % (B, n, max(self.fft_sizes) // 2))
        x, y = x.contiguous(), y.contiguous()
        if grad and x.requires_grad:
            return _STFTLoss.apply(x, y, self._an)
        sc, mag, _ = _forward(self._an, x, y)
        return sc, mag
