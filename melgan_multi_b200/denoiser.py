"""Denoiser on hand-written sm_90a kernels (csrc/mg_denoise.cu): WaveGlow's ``Denoiser``, which removes a vocoder's own
bias -- the faint constant hum or hiss it leaves even on a silent mel.

The bias spectrum is the magnitude of the first STFT frame of the generator's audio for a zero mel (``mode="zeros"``) or
a standard-normal one (``mode="normal"``), ``[1, 80, 88]``, one row per voice.  ``forward`` computes, per item,
``S = torch.stft(a, n_fft, hop, win_length, hann, center=True, pad_mode="reflect")``, subtracts ``strength * bias``
from ``|S|``, clamps at 0, keeps the phase of S (phase 0 where ``|S| = 0``) and returns
``torch.istft(..., length=L)``: every step on the package's own kernels, for uniform, ragged and multi-voice batches,
in fp32 or 16-bit PCM.  ``Denoiser.stream`` applies the same denoiser to live audio, each session's samples
emitted once final and bit-identical to ``forward`` of the whole utterance.  Inference only.  CUDA only, like the rest of the package: there is no CPU fallback.
"""
import ctypes
import math

import torch

from . import engine as _engine
from . import stft_loss as _stft_loss
from .stft_loss import _Analysis, _TablesModule, _workspace

BIAS_MEL_FRAMES = 88  # WaveGlow's Denoiser: the bias audio is vocoded from an 80 x 88 mel
_LIB = None


def _lib():
    """The library with the denoiser calls' ctypes signatures, set once."""
    global _LIB
    if _LIB is not None:
        return _LIB
    L = _stft_loss._lib()
    L.mg_denoise_workspace_bytes.restype = ctypes.c_int
    L.mg_denoise_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.POINTER(ctypes.c_size_t)]
    L.mg_denoise_bias.restype = ctypes.c_int
    L.mg_denoise_bias.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                  ctypes.c_void_p]
    for name in ("mg_denoise_forward", "mg_denoise_forward_pcm16"):
        f = getattr(L, name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                      ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.mg_denoise_stream_state_bytes.restype = ctypes.c_size_t
    L.mg_denoise_stream_state_bytes.argtypes = [ctypes.c_int] * 4
    L.mg_denoise_stream_max_out.restype = ctypes.c_int
    L.mg_denoise_stream_max_out.argtypes = [ctypes.c_int] * 3
    L.mg_denoise_stream_create.restype = ctypes.c_int
    L.mg_denoise_stream_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t]
    L.mg_denoise_stream_destroy.restype = None
    L.mg_denoise_stream_destroy.argtypes = [ctypes.c_void_p]
    for name in ("mg_denoise_stream_step", "mg_denoise_stream_step_pcm16"):
        f = getattr(L, name)
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                      ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                      ctypes.c_void_p]
    L.mg_denoise_stream_dry_step.restype = ctypes.c_int
    L.mg_denoise_stream_dry_step.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    _LIB = L
    return L


def workspace_bytes(n_fft, hop, B, L_max, lengths=None):
    """Bytes of frame workspace a call needs: sum over items of (1 + L_i // hop) n_fft floats."""
    n = ctypes.c_size_t()
    lens = None if lengths is None else (ctypes.c_int * B)(*lengths)
    _engine.check(_lib().mg_denoise_workspace_bytes(n_fft, hop, B, L_max, lens, ctypes.byref(n)))
    return n.value


class Denoiser(_TablesModule):
    """WaveGlow's Denoiser over one generator or several: ``Denoiser(generator, filter_length=1024, n_overlap=4,
    win_length=1024, mode="zeros")``, hop = int(filter_length / n_overlap).  A list of generators gives one bias row per
    voice, in the order generate_voices takes them.  The bias is computed once, at construction, on the generators'
    device; call refresh() after their weights change.  ``Denoiser.from_bias(bias, ...)`` takes a caller's
    ``[V, filter_length // 2 + 1]`` bias instead.

    Supported: filter_length a power of two from 128 to 2048, 1 <= hop <= win_length <= filter_length, items of
    filter_length / 2 < L <= 2^30 samples, and analyses whose window-square envelope stays >= 1e-11 (torch.istft's NOLA
    condition); anything else raises EngineError.  The tables and bias move with .to(device); a first call on a device
    inside a CUDA graph capture is refused, so move the module or call it once before capturing."""

    def __init__(self, generator, filter_length=1024, n_overlap=4, win_length=1024, mode="zeros"):
        super().__init__()
        gens = list(generator) if isinstance(generator, (list, tuple)) else [generator]
        if not gens:
            raise _engine.EngineError("Denoiser needs at least one generator")
        if mode not in ("zeros", "normal"):
            raise _engine.EngineError("Denoiser: mode must be 'zeros' or 'normal' (got %r)" % (mode,))
        self._setup(filter_length, n_overlap, win_length)
        self._generators = gens
        self.mode = mode
        self.register_buffer("bias_spec", torch.empty(0))
        self.refresh()

    @classmethod
    def from_bias(cls, bias, filter_length=1024, n_overlap=4, win_length=1024):
        """A denoiser with a given bias spectrum [V, filter_length // 2 + 1] (fp32; any device, moved with .to())."""
        self = cls.__new__(cls)
        _TablesModule.__init__(self)
        self._setup(filter_length, n_overlap, win_length)
        self._generators = []
        self.mode = None
        if not torch.is_tensor(bias) or bias.dtype != torch.float32 or bias.dim() != 2 or bias.shape[1] != self.n_fft // 2 + 1 \
                or bias.shape[0] < 1:
            raise _engine.EngineError("Denoiser.from_bias: bias must be fp32 [V, %d], got %s" % (
                self.n_fft // 2 + 1, (bias.dtype, tuple(bias.shape)) if torch.is_tensor(bias) else type(bias).__name__))
        self.register_buffer("bias_spec", bias.detach().contiguous().clone())
        return self

    def _setup(self, filter_length, n_overlap, win_length):
        n, w = int(filter_length), int(win_length)
        if _stft_loss._lib().mg_stft_loss_tables_bytes(n) == 0:
            raise _engine.EngineError("Denoiser: filter_length %d is not a power of two in [128, 2048]" % n)
        hop = int(n / n_overlap) if n_overlap else 0
        if hop < 1:
            raise _engine.EngineError("Denoiser: hop = int(filter_length / n_overlap) = %d, at least 1 needed" % hop)
        if not 1 <= w <= n:
            raise _engine.EngineError("Denoiser: win_length %d outside [1, filter_length %d]" % (w, n))
        if hop > w:
            raise _engine.EngineError("Denoiser: hop %d exceeds win_length %d (torch.istft needs hop <= win_length)" % (hop, w))
        host = _stft_loss.build_tables(n, w)
        self.n_fft, self.hop, self.win_length = n, hop, w
        self._an = _Analysis((n,), (hop,), [host], "Denoiser")

    def refresh(self):
        """Recomputes the bias from the generators' current weights (WaveGlow computes it once, at construction)."""
        if not self._generators:
            raise _engine.EngineError("Denoiser.refresh: this denoiser was built from a bias, not from generators")
        dev = self._generators[0].conv_pre.weight_v.device
        if dev.type != "cuda":
            raise _engine.EngineError("Denoiser needs its generators on CUDA (no CPU fallback)")
        with torch.no_grad():
            rows = []
            for g in self._generators:
                mel = torch.zeros(1, 80, BIAS_MEL_FRAMES, device=dev) if self.mode == "zeros" else \
                    torch.randn(1, 80, BIAS_MEL_FRAMES, device=dev)
                rows.append(g.generate(mel).reshape(1, -1))
            audio = torch.cat(rows).contiguous()
            bias = torch.empty(len(rows), self.n_fft // 2 + 1, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _engine.check(_lib().mg_denoise_bias(self._an.tables(dev)[0], self.n_fft, audio.data_ptr(), audio.shape[0],
                                                     audio.shape[1], bias.data_ptr(), torch.cuda.current_stream().cuda_stream))
        self.bias_spec = bias
        return bias

    def forward(self, audio, strength=0.1, lengths=None, voice=None, dtype=torch.float32):
        """audio [B, L] or [B, 1, L] fp32 CUDA -> the denoised audio of the same shape, fp32 or (dtype=torch.int16) pcm16 of
        it written by the last kernel.  lengths: B item lengths in SAMPLES (256 times the mel lengths after
        Generator.generate), a list, a tuple or a CPU integer tensor; None: every item L.  voice: B bias rows (None: row
        0).  The samples past each length are not read and come out 0."""
        name = "Denoiser"
        pcm = _engine._pcm16(dtype)
        if not torch.is_tensor(audio) or not audio.is_cuda:
            raise _engine.EngineError("%s: audio must be a CUDA tensor (no CPU fallback)" % name)
        if audio.dtype != torch.float32 or not (audio.dim() == 2 or (audio.dim() == 3 and audio.shape[1] == 1)):
            raise _engine.EngineError("%s: audio must be fp32 [B, L] or [B, 1, L], got %s %s" % (name, audio.dtype, tuple(audio.shape)))
        if torch.is_grad_enabled() and audio.requires_grad:
            raise _engine.EngineError("%s: audio requires grad; the denoiser computes no gradient (pass audio.detach() or run "
                                      "under torch.no_grad())" % name)
        strength = float(strength)
        if not math.isfinite(strength):
            raise _engine.EngineError("%s: strength %r is not finite" % (name, strength))
        if self.bias_spec.device != audio.device:
            raise _engine.EngineError("%s: the bias is on %s, audio on %s (move the denoiser with .to())"
                                      % (name, self.bias_spec.device, audio.device))
        shape = audio.shape
        x = audio.reshape(shape[0], shape[-1]).contiguous()
        B, L = x.shape
        n, h = self.n_fft, self.hop
        if B < 1 or L <= n // 2:
            raise _engine.EngineError("%s: [B, L] = [%d, %d]; reflect padding by filter_length / 2 needs L > %d" % (name, B, L, n // 2))
        lens = None if lengths is None else _engine._host_ints(lengths, B, "lengths", n // 2 + 1, L + 1,
                                                               "lengths must lie in (filter_length / 2 = %d, L = %d]" % (n // 2, L))
        V = self.bias_spec.shape[0]
        ids = None if voice is None else _engine._voice_ids(voice, B, V)
        nbytes = ctypes.c_size_t()
        _engine.check(_lib().mg_denoise_workspace_bytes(n, h, B, L, lens, ctypes.byref(nbytes)))
        out = torch.empty((B, L), dtype=torch.int16 if pcm else torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            tabs = self._an.tables(x.device)
            ws = _workspace(nbytes.value, x.device)
            call = _lib().mg_denoise_forward_pcm16 if pcm else _lib().mg_denoise_forward
            _engine.check(call(tabs[0], n, h, self.win_length, x.data_ptr(), B, L, lens, self.bias_spec.data_ptr(), V, ids, strength,
                               out.data_ptr(), ws.data_ptr(), nbytes.value, torch.cuda.current_stream().cuda_stream))
        return out.reshape(shape)

    def stream(self, max_sessions=1, max_push_samples=256 * 32 + 1542, strength=0.1, dtype=torch.float32, state=None):
        """A DenoiserStream of this denoiser: up to max_sessions live sessions, at most max_push_samples new samples per
        session and step (the default takes GeneratorStream's output at its default max_push_frames=32), one strength for
        the handle's lifetime.  dtype: the default output format, torch.float32 or torch.int16."""
        return DenoiserStream(self, max_sessions, max_push_samples, strength, dtype, state)


class DenoiserStream:
    """Denoising of up to ``max_sessions`` live audio streams (mg_denoise_stream_*, contract in include/melgan_b200.h).
    Each step takes each session's newly received samples and returns the denoised samples that became final: E(R) of
    them once R samples have been received (E(R) = 0 for R <= n_fft / 2, else clamp((q + 1) hop - n_fft / 2, 0, R),
    q = (R - n_fft / 2) // hop), all L after the step that ends the utterance; their concatenation equals
    ``Denoiser.forward`` of the whole utterance bit for bit (same bias row and strength), in fp32 and int16.

    The bias and tables are read from the denoiser at every step, so refresh() between steps takes effect; the handle's
    state lives on the device the denoiser was on when the stream was opened, and a step after the denoiser was moved
    with .to() to another device is refused.  Chaining after a GeneratorStream needs no copy::

        a, c = gs.step_packed(mel, frames, flags, voice=v)
        y, m = ds.step_packed(a, c, flags, voice=v)

    One thread drives a handle at a time, and its steps must be enqueued on one CUDA stream (or otherwise ordered)."""

    def __init__(self, denoiser, max_sessions, max_push_samples, strength, dtype, state):
        self._dn = denoiser
        self.dtype = dtype
        _engine._pcm16(dtype)
        self.device = denoiser.bias_spec.device
        if self.device.type != "cuda":
            raise _engine.EngineError("Denoiser.stream: the denoiser is on %s; it needs CUDA (no CPU fallback)" % (self.device,))
        self.strength = float(strength)
        if not math.isfinite(self.strength):
            raise _engine.EngineError("Denoiser.stream: strength %r is not finite" % (self.strength,))
        self.max_sessions, self.max_push_samples = int(max_sessions), int(max_push_samples)
        n, h = denoiser.n_fft, denoiser.hop
        L = _lib()
        nbytes = L.mg_denoise_stream_state_bytes(n, h, self.max_sessions, self.max_push_samples)
        if nbytes == 0:
            raise _engine.EngineError("Denoiser.stream: max_sessions must lie in [1, 256] and max_push_samples in [1, 2^20]")
        if state is None:
            state = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if state.device != self.device or state.numel() * state.element_size() < nbytes or not state.is_contiguous():
            raise _engine.EngineError("Denoiser.stream: state must be a contiguous CUDA tensor of at least %d bytes on %s"
                                      % (nbytes, self.device))
        self.state = state
        self.max_out = L.mg_denoise_stream_max_out(n, h, self.max_push_samples)
        self._h = ctypes.c_void_p()
        _engine.check(L.mg_denoise_stream_create(ctypes.byref(self._h), n, h, denoiser.win_length, self.max_sessions,
                                                 self.max_push_samples, self.strength, state.data_ptr(),
                                                 state.numel() * state.element_size()))
        self._in = torch.zeros((self.max_sessions, self.max_push_samples), dtype=torch.float32, device=self.device)

    def step_packed(self, audio, counts, flags=None, voice=None, out=None):
        """The C step on a packed buffer: audio [n, stride] fp32 CUDA (slot i's new samples first, e.g. GeneratorStream's
        output), counts: n sample counts, flags: None or n ints (STREAM_END / STREAM_RESET), voice: None (bias row 0) or n
        bias rows.  Returns (out [n, max_out], per-slot sample counts as a list of ints).  out: None (a new tensor of the
        handle's dtype) or a contiguous fp32 or int16 CUDA tensor [n, max_out], whose dtype picks this step's format."""
        n = len(counts)
        if not self._h:
            raise _engine.EngineError("DenoiserStream: the stream is closed")
        bias = self._dn.bias_spec
        if bias.device != self.device:
            raise _engine.EngineError("DenoiserStream: the denoiser was moved to %s, this stream's state is on %s (open a new "
                                      "stream after .to())" % (bias.device, self.device))
        if audio is not None and (not torch.is_tensor(audio) or audio.device != self.device or audio.dtype != torch.float32
                                  or audio.dim() != 2 or audio.shape[0] < n or audio.stride(1) != 1):
            raise _engine.EngineError("DenoiserStream: audio must be an fp32 [n, stride] tensor on %s with unit-stride rows"
                                      % (self.device,))
        ids = None if voice is None else _engine._voice_ids(voice, n, bias.shape[0])
        if out is None:
            out = torch.empty((n, self.max_out), dtype=self.dtype, device=self.device)
        if out.dtype not in (torch.float32, torch.int16) or out.device != self.device or out.dim() != 2 or out.shape[0] < n \
                or out.shape[1] != self.max_out or not out.is_contiguous():
            raise _engine.EngineError("DenoiserStream: out must be a contiguous fp32 or int16 [%d, %d] tensor on %s"
                                      % (n, self.max_out, self.device))
        cnt_in = (ctypes.c_int * max(n, 1))(*[int(v) for v in counts])
        fl = (ctypes.c_int * max(n, 1))(*[int(v) for v in flags]) if flags is not None else None
        cnt = (ctypes.c_int * max(n, 1))()
        with torch.cuda.device(self.device):
            tabs = self._dn._an.tables(self.device)
            L = _lib()
            fn = L.mg_denoise_stream_step_pcm16 if out.dtype == torch.int16 else L.mg_denoise_stream_step
            _engine.check(fn(self._h, tabs[0], bias.data_ptr(), bias.shape[0], ids, audio.data_ptr() if audio is not None else None,
                             audio.stride(0) if audio is not None else 0, cnt_in, fl, n, out.data_ptr(), cnt,
                             torch.cuda.current_stream().cuda_stream))
        return out, [cnt[i] for i in range(n)]

    def step(self, chunks, end=None, reset=None, voice=None):
        """chunks: one entry per slot 0 .. n-1, each a [1, m] or [m] fp32 CUDA tensor (m <= max_push_samples) or None;
        end / reset / voice as for GeneratorStream.step.  Returns n [1, m_i] CUDA tensors of newly final denoised audio in
        the handle's dtype.  Asynchronous on the current stream: the lengths are known on return."""
        n = len(chunks)
        if n > self.max_sessions:
            raise _engine.EngineError("DenoiserStream: %d chunks for %d sessions" % (n, self.max_sessions))
        counts = []
        for i, c in enumerate(chunks):
            if c is None:
                counts.append(0)
                continue
            if not torch.is_tensor(c) or not (c.dim() == 1 or (c.dim() == 2 and c.shape[0] == 1)) \
                    or c.shape[-1] > self.max_push_samples:
                raise _engine.EngineError("DenoiserStream: chunk %d must be [1, m] or [m] with m <= %d, got %s"
                                          % (i, self.max_push_samples, tuple(c.shape) if torch.is_tensor(c) else type(c).__name__))
            if c.device != self.device or c.dtype != torch.float32:
                raise _engine.EngineError("DenoiserStream: chunks must be fp32 tensors on %s" % (self.device,))
            counts.append(int(c.shape[-1]))
            if counts[-1]:
                self._in[i, :counts[-1]].copy_(c.reshape(-1))
        flags = [(_engine.STREAM_END if end is not None and end[i] else 0) | (_engine.STREAM_RESET if reset is not None and reset[i]
                                                                                else 0) for i in range(n)]
        out, m = self.step_packed(self._in, counts, flags, voice=voice)
        return [out[i:i + 1, :k] for i, k in enumerate(m)]

    def close(self):
        if self._h:
            _lib().mg_denoise_stream_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
