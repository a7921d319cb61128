"""ctypes binding of libmelgan_b200.so (the C ABI in include/melgan_b200.h).

PyTorch is plumbing here: it owns device memory and streams; every kernel that runs on the hot
path lives in the shared library.  There is no CPU or eager-PyTorch fallback: if the library
is missing, or the device is not sm_90 (H100), calls raise.

Streams and threads: every call enqueues its work on the caller's current CUDA stream.  Inference calls of one
GeneratorDevice or DiscriminatorDevice (and so of one Generator, Discriminator or MultiScaleDiscriminator) may run
concurrently on distinct streams, from one host thread or several: the scratch memory a call writes (the generator's
workspace, the discriminator's status word and backward workspace, the status copy to the host) is kept per stream, is
allocated while that stream is current, and so is only ever used and freed in that stream's order (_PerStream).  Calls
on one stream are ordered by the stream.  Every read of the packed weights waits for the last pack, whichever stream
enqueued it (_PackedBlob).  Training steps that update the parameters need the caller's ordering, as in stock PyTorch.
A GeneratorStream handle is the exception: its steps must stay on one stream (GeneratorStream).
"""
import collections
import ctypes
import os
import threading
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmelgan_b200.so")
NUM_LAYERS = 30

_f32p = ctypes.POINTER(ctypes.c_float)
_lib = None


class EngineError(RuntimeError):
    pass


def lib():
    """Loads the shared library (once).  Raises if it has not been built: the product path never
    degrades to a fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(
                "libmelgan_b200.so is not built (%s). Run `python -m melgan_multi_b200.build` "
                "(needs nvcc); there is no CPU/PyTorch fallback for the hot path." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.mg_abi_version.restype = ctypes.c_int
        L.mg_last_error_string.restype = ctypes.c_char_p
        L.mg_device_check.restype = ctypes.c_int
        L.mg_gen_packed_bytes.restype = ctypes.c_size_t
        L.mg_gen_pack.restype = ctypes.c_int
        L.mg_gen_pack.argtypes = [ctypes.c_void_p] * 5
        L.mg_gen_workspace_bytes.restype = ctypes.c_size_t
        L.mg_gen_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
        L.mg_gen_forward.restype = ctypes.c_int
        L.mg_gen_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        L.mg_gen_forward_ragged.restype = ctypes.c_int
        L.mg_gen_forward_ragged.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        L.mg_gen_forward_precision.restype = ctypes.c_int
        L.mg_gen_forward_precision.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        L.mg_gen_forward_voices.restype = ctypes.c_int
        L.mg_gen_forward_voices.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_size_t, ctypes.c_void_p]
        L.mg_gen_forward_timed.restype = ctypes.c_int
        L.mg_gen_forward_timed.argtypes = L.mg_gen_forward.argtypes + [ctypes.POINTER(ctypes.c_float)]
        L.mg_gen_check_status.restype = ctypes.c_int
        L.mg_gen_check_status.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_convt.restype = ctypes.c_int
        L.mg_gen_convt.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                   ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_resblock.restype = ctypes.c_int
        L.mg_gen_resblock.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_upres.restype = ctypes.c_int
        L.mg_gen_upres.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                   ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_upres_post.restype = ctypes.c_int
        L.mg_gen_upres_post.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_resblock_config.restype = ctypes.c_char_p
        L.mg_gen_resblock_config.argtypes = [ctypes.c_int]
        L.mg_gen_convt_config.restype = ctypes.c_char_p
        L.mg_gen_convt_config.argtypes = [ctypes.c_int]
        L.mg_gen_conv_pre_config.restype = ctypes.c_char_p
        L.mg_gen_conv_pre_config.argtypes = []
        L.mg_gen_chain_kernel.restype = ctypes.c_int
        L.mg_gen_chain_kernel.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_conv_pre.restype = ctypes.c_int
        L.mg_gen_conv_pre.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_resblock_post.restype = ctypes.c_int
        L.mg_gen_resblock_post.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_disc_packed_bytes.restype = ctypes.c_size_t
        L.mg_disc_pack.restype = ctypes.c_int
        L.mg_disc_pack.argtypes = [ctypes.c_void_p] * 5
        L.mg_disc_forward.restype = ctypes.c_int
        L.mg_disc_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                      ctypes.c_void_p, ctypes.c_void_p]
        L.mg_gen_resup.restype = ctypes.c_int
        L.mg_gen_resup.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_void_p]
        L.mg_gen_set_pipeline.restype = ctypes.c_int
        L.mg_gen_set_pipeline.argtypes = [ctypes.c_int]
        L.mg_gen_stage_output.restype = ctypes.c_int
        L.mg_gen_stage_output.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_void_p]
        L.mg_gen_forward_launches.restype = ctypes.c_int
        L.mg_gen_forward_slices.restype = ctypes.c_int
        L.mg_gen_forward_slices.argtypes = [ctypes.c_int, ctypes.c_int]
        L.mg_gen_kernel_name.restype = ctypes.c_char_p
        L.mg_gen_kernel_name.argtypes = [ctypes.c_int]
        L.mg_msd_packed_bytes.restype = ctypes.c_size_t
        L.mg_msd_pack.restype = ctypes.c_int
        L.mg_msd_pack.argtypes = [ctypes.c_void_p] * 5
        L.mg_msd_lengths.restype = ctypes.c_int
        L.mg_msd_lengths.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        L.mg_msd_forward.restype = ctypes.c_int
        L.mg_msd_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_void_p]
        L.mg_msd_layer_forward.restype = ctypes.c_int
        L.mg_msd_layer_forward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.mg_disc_tc_element.restype = ctypes.c_int
        L.mg_disc_tc_element.argtypes = [ctypes.c_size_t] + [ctypes.POINTER(ctypes.c_int)] * 4
        L.mg_msd_grouped_backward_workspace_bytes.restype = ctypes.c_size_t
        L.mg_msd_grouped_backward_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.mg_msd_grouped_backward.restype = ctypes.c_int
        L.mg_msd_grouped_backward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6 + [
            ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_msd_post1_dgrad.restype = ctypes.c_int
        L.mg_msd_post1_dgrad.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_void_p, ctypes.c_void_p]
        L.mg_msd_post1_wgrad.restype = ctypes.c_int
        L.mg_msd_post1_wgrad.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.mg_msd_edge_backward_workspace_bytes.restype = ctypes.c_size_t
        L.mg_msd_edge_backward_workspace_bytes.argtypes = [ctypes.c_int] * 3
        L.mg_msd_edge_backward.restype = ctypes.c_int
        L.mg_msd_edge_backward.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6 + [
            ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
        L.mg_msd_scale_backward_workspace_bytes.restype = ctypes.c_size_t
        L.mg_msd_scale_backward_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
        L.mg_msd_scale_backward.restype = ctypes.c_int
        L.mg_msd_scale_backward.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 8 + [
            ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.mg_lrelu_backward.restype = ctypes.c_int
        L.mg_lrelu_backward.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_longlong, ctypes.c_void_p]
        L.mg_msd_wn_backward.restype = ctypes.c_int
        L.mg_msd_wn_backward.argtypes = [ctypes.c_void_p] * 6
        L.mg_adam_chunk.restype = ctypes.c_int
        L.mg_adam_step.restype = ctypes.c_int
        L.mg_adam_step.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int, ctypes.c_int] + [ctypes.c_float] * 5 + [
            ctypes.c_longlong, ctypes.c_void_p]
        L.mg_loss_workspace_bytes.restype = ctypes.c_size_t
        L.mg_loss_workspace_bytes.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.mg_loss_forward.restype = ctypes.c_int
        L.mg_loss_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        L.mg_loss_backward.restype = ctypes.c_int
        L.mg_loss_backward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.mg_msd_check_status.restype = ctypes.c_int
        L.mg_msd_check_status.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.mg_gen_engine_create.restype = ctypes.c_int
        L.mg_gen_engine_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int]
        L.mg_gen_engine_load_state.restype = ctypes.c_int
        L.mg_gen_engine_load_state.argtypes = [ctypes.c_void_p] * 4
        L.mg_gen_engine_forward.restype = ctypes.c_int
        L.mg_gen_engine_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                            ctypes.c_int]
        L.mg_gen_engine_forward_ragged.restype = ctypes.c_int
        L.mg_gen_engine_forward_ragged.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                   ctypes.c_void_p]
        L.mg_gen_engine_forward_precision.restype = ctypes.c_int
        L.mg_gen_engine_forward_precision.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                      ctypes.c_void_p, ctypes.c_int]
        L.mg_gen_engine_last_kernel_ms.restype = ctypes.c_int
        L.mg_gen_engine_last_kernel_ms.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float)]
        L.mg_gen_engine_destroy.restype = None
        L.mg_gen_engine_destroy.argtypes = [ctypes.c_void_p]
        L.mg_gen_stream_lookahead.restype = ctypes.c_int
        L.mg_gen_stream_state_bytes.restype = ctypes.c_size_t
        L.mg_gen_stream_state_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
        L.mg_gen_stream_max_out.restype = ctypes.c_int
        L.mg_gen_stream_max_out.argtypes = [ctypes.c_int]
        L.mg_gen_stream_create.restype = ctypes.c_int
        L.mg_gen_stream_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_size_t]
        L.mg_gen_stream_destroy.restype = None
        L.mg_gen_stream_destroy.argtypes = [ctypes.c_void_p]
        L.mg_gen_stream_step.restype = ctypes.c_int
        L.mg_gen_stream_step.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int] + [ctypes.c_void_p] * 3
        L.mg_gen_stream_check_status.restype = ctypes.c_int
        L.mg_gen_stream_check_status.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.mg_gen_stream_dry_step.restype = ctypes.c_int
        L.mg_gen_stream_dry_step.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] + [ctypes.c_void_p] * 3
        L.mg_gen_stream_step_voices.restype = ctypes.c_int
        L.mg_gen_stream_step_voices.argtypes = ([ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
                                                + [ctypes.c_void_p] * 3)
        L.mg_gen_forward_pcm16.restype = ctypes.c_int
        L.mg_gen_forward_pcm16.argtypes = L.mg_gen_forward_voices.argtypes
        L.mg_gen_stream_step_pcm16.restype = ctypes.c_int
        L.mg_gen_stream_step_pcm16.argtypes = L.mg_gen_stream_step_voices.argtypes
        L.mg_gen_engine_forward_pcm16.restype = ctypes.c_int
        L.mg_gen_engine_forward_pcm16.argtypes = L.mg_gen_engine_forward_precision.argtypes
        L.mg_gen_stream_dry_step_voices.restype = ctypes.c_int
        L.mg_gen_stream_dry_step_voices.argtypes = ([ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
                                                    + [ctypes.c_void_p] * 3)
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise EngineError("melgan_b200 error %d: %s" % (rc, lib().mg_last_error_string().decode()))


def _ptr_array(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def _host_ints(values, B, name, lo, hi, range_error):
    """B per-item values in [lo, hi) as a C int array: a list, a tuple or a CPU integer tensor.  A CUDA tensor is refused:
    reading it would synchronise the stream.  name and range_error word the errors."""
    if hasattr(values, "device") and hasattr(values, "is_floating_point"):
        if values.device.type != "cpu":
            raise EngineError("%s must be a list, a tuple or a CPU tensor (reading a CUDA tensor would synchronise)" % name)
        if values.is_floating_point() or values.dim() != 1:
            raise EngineError("%s must be a 1-D integer tensor" % name)
        values = values.tolist()
    values = [int(v) for v in values]
    if len(values) != B:
        raise EngineError("%s has %d entries for a batch of %d" % (name, len(values), B))
    bad = [v for v in values if not lo <= v < hi]
    if bad:
        raise EngineError("%s (got %d)" % (range_error, bad[0]))
    return (ctypes.c_int * B)(*values)


def _lengths(lengths, B, T_max):
    """Per-item mel lengths of a ragged batch, each in [1, T_max] (_host_ints)."""
    return _host_ints(lengths, B, "lengths", 1, T_max + 1, "lengths must lie in [1, T_max = %d]" % T_max)


def _voice_ids(voice, B, n_voices):
    """Per-item voice ids of a multi-voice batch, each in [0, n_voices) (_host_ints)."""
    return _host_ints(voice, B, "voice", 0, n_voices, "voice ids must lie in [0, n_voices = %d)" % n_voices)


PRECISIONS = {"fp32": 0, "bf16": 1}  # MG_GEN_PRECISION_FP32 / _BF16, include/melgan_b200.h


def _precision(precision):
    """The C code of an inference precision: "fp32" (three bf16 passes per product, fp32-equivalent audio) or "bf16"
    (one pass; the accuracy contract is at mg_gen_forward_precision in include/melgan_b200.h)."""
    if not isinstance(precision, str) or precision not in PRECISIONS:
        raise EngineError("precision must be one of %s (got %r)" % (", ".join(map(repr, PRECISIONS)), precision))
    return PRECISIONS[precision]


def _pcm16(dtype):
    """Whether an inference call returns 16-bit PCM: dtype torch.float32 (fp32 audio in [-1, 1]) or torch.int16 (pcm16 of
    that audio: 0 for NaN, else clamp(rint(32768 a), -32768, 32767), contract at mg_gen_forward_pcm16 in
    include/melgan_b200.h)."""
    import torch
    if dtype is torch.float32:
        return False
    if dtype is torch.int16:
        return True
    raise EngineError("dtype must be torch.float32 or torch.int16 (got %r)" % (dtype,))


def _pcm16_np(dtype):
    """_pcm16 for the host-buffer path: np.float32 or np.int16 (or their np.dtype)."""
    try:
        dt = np.dtype(dtype)
    except TypeError:
        dt = None
    if dt == np.float32 and not isinstance(dtype, str):
        return False
    if dt == np.int16 and not isinstance(dtype, str):
        return True
    raise EngineError("dtype must be np.float32 or np.int16 (got %r)" % (dtype,))


def _audio_out(torch, out, shape, pcm, device):
    """The caller's out= for audio of `shape` (None: a new tensor of the call's dtype).  An int16 out needs dtype=torch.int16
    and the reverse, on the call's device, contiguous and of the audio's shape."""
    dt = torch.int16 if pcm else torch.float32
    if out is None:
        return torch.empty(shape, dtype=dt, device=device)
    if pcm or out.dtype == torch.int16:
        if out.dtype != dt:
            raise EngineError("out is %s but dtype is %s" % (out.dtype, dt))
        if out.device != device or tuple(out.shape) != tuple(shape) or not out.is_contiguous():
            raise EngineError("out must be a contiguous %s tensor of shape %s on %s" % (dt, tuple(shape), device))
    return out


class _StatusWatch:
    """The tensor-core kernels bound every mbarrier wait and, on a timeout, raise a device status word and carry on (a hung
    GPU box is worse than a failed call).  A forward must therefore never be trusted silently: after each one the status
    word is copied to pinned host memory on the same stream (4 bytes, asynchronous), and the copy is inspected at the
    next forward of the same module, or at the next host synchronisation point the training loop has anyway
    (``discriminator_loss``' read-back, ``poll_status``).  A non-zero word raises EngineError.  Skipped while the stream
    is being captured into a CUDA graph (no host-visible copy can be made there; replays are checked by check_status).
    One watch serves one stream at a time (_PerStream): a second call in flight on another stream has its own slot and
    event."""
    _live = weakref.WeakSet()  # watches with a copy in flight

    def __init__(self, torch, device, what):
        self.torch, self.what = torch, what
        self.pin = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.event = torch.cuda.Event()
        self.pending = False

    def arm(self, status_word):
        """status_word: int32 CUDA tensor view [1] holding the pipeline's status after the work just enqueued."""
        if self.torch.cuda.is_current_stream_capturing():
            return
        self.pin.copy_(status_word, non_blocking=True)
        self.event.record()
        self.pending = True
        _StatusWatch._live.add(self)

    def check(self, wait=False):
        if not self.pending or self.torch.cuda.is_current_stream_capturing():
            return  # (event queries are illegal while this thread captures a CUDA graph)
        if wait:
            self.event.synchronize()
        elif not self.event.query():
            return
        self.pending = False
        _StatusWatch._live.discard(self)
        code = int(self.pin[0])
        if code:
            self.pin[0] = 0
            raise EngineError("%s: tensor-core pipeline wait timed out (role code %d); the outputs of that call are "
                              "invalid" % (self.what, code))


def poll_status(wait=False):
    """Checks every status copy in flight (all modules and streams, this process); ``wait=True`` blocks on the copies'
    events."""
    for w in list(_StatusWatch._live):
        w.check(wait)


class _StreamScratch:
    """The scratch buffers and the status watch one module uses on one CUDA stream."""

    def __init__(self, owner):
        self.owner = owner
        self.bufs = {}
        self._watch = None

    def buffer(self, name, nbytes, zeros=False):
        """The stream's buffer `name` of at least nbytes (grown on demand; an int32 tensor when zeros, else fp32).  Called
        with the stream current, so the caching allocator ties the memory to it: a buffer dropped by regrowth or
        eviction is handed out again only in this stream's order."""
        torch, device = self.owner.torch, self.owner.device
        t = self.bufs.get(name)
        if t is None or t.numel() * 4 < nbytes:
            n = (nbytes + 3) // 4
            t = self.bufs[name] = (torch.zeros(n, dtype=torch.int32, device=device) if zeros else
                                   torch.empty(n, dtype=torch.float32, device=device))
        if torch.cuda.is_current_stream_capturing():
            self.owner.hold(t)
        return t

    @property
    def watch(self):
        if self._watch is None:
            self._watch = self.owner.take_watch()
        return self._watch

    def check(self):
        """Raises for a timed-out wait of an earlier call of this module whose status copy has landed: this stream's
        previous call, or a call on a stream whose scratch has since been dropped (_PerStream.check_retired)."""
        self.owner.check_retired()
        if self._watch is not None:
            self._watch.check()

    def arm(self, status_word):
        if not self.owner.torch.cuda.is_current_stream_capturing():  # (no pinned allocation while capturing)
            self.watch.arm(status_word)


class _PerStream:
    """One _StreamScratch per CUDA stream of a module, keyed by the current stream's handle, so that calls on distinct
    streams or threads never share a byte of scratch memory.

    At most LIMIT streams keep their scratch, as many as PyTorch's pool hands out per priority (torch.cuda.Stream()):
    the least recently used one beyond them is dropped.  Its buffers return to the caching allocator's pool of their own
    stream, which keeps them reserved for that stream, so reserved memory follows the number of distinct streams that
    ever called, not LIMIT.  Its status watch is retired: the module's next call checks it without blocking (raising
    for a timed-out wait whose copy has landed), and once its copy has landed it is reused by a new stream's scratch,
    so pinned slots and events are bounded by LIMIT plus the copies still in flight.  Buffers a captured CUDA graph
    writes stay allocated for the module's lifetime."""
    LIMIT = 32

    def __init__(self, torch, device, what):
        self.torch, self.device, self.what = torch, device, what
        self._by_stream = collections.OrderedDict()
        self._held = []     # buffers captured CUDA graphs write
        self._retired = []  # watches of dropped scratch: copies in flight first, then idle ones for reuse
        self._lock = threading.Lock()  # streams of several host threads share the tables

    def current(self):
        key = self.torch.cuda.current_stream(self.device).cuda_stream
        with self._lock:
            s = self._by_stream.get(key)
            if s is None:
                s = self._by_stream[key] = _StreamScratch(self)
                while len(self._by_stream) > self.LIMIT:
                    _, old = self._by_stream.popitem(last=False)
                    if old._watch is not None:
                        self._retired.append(old._watch)
            else:
                self._by_stream.move_to_end(key)
        return s

    def hold(self, t):
        with self._lock:
            if not any(h is t for h in self._held):
                self._held.append(t)

    def take_watch(self):
        """An idle retired watch (no copy in flight), or a new one."""
        with self._lock:
            for i, w in enumerate(self._retired):
                if not w.pending:
                    return self._retired.pop(i)
        return _StatusWatch(self.torch, self.device, self.what)

    def check_retired(self):
        with self._lock:
            try:
                for w in self._retired:
                    w.check()  # (non-blocking; marks a landed copy checked before it raises)
            finally:
                idle = [w for w in self._retired if not w.pending]
                self._retired = [w for w in self._retired if w.pending] + idle[:self.LIMIT]


class _PackedBlob:
    """The packed weight blob of a GeneratorDevice / DiscriminatorDevice.  ``pack`` enqueues its writes on the caller's
    stream and records an event after them; until that event has completed, every read of ``packed`` makes the current
    stream wait for it, so a call on any stream reads the weights of the last pack, even when the pack is still queued
    behind other work on its own stream.  (A re-pack while calls on other streams still read the old weights needs the
    caller's ordering, as any parameter update does.)"""

    @property
    def packed(self):
        ev = self._pack_done
        if ev is not None and not self.torch.cuda.is_current_stream_capturing():  # (no event query while capturing)
            if ev.query():
                self._pack_done = None
            else:
                self.torch.cuda.current_stream(self.device).wait_event(ev)
        return self._packed

    def _pack_enqueued(self):
        if not self.torch.cuda.is_current_stream_capturing():
            ev = self.torch.cuda.Event()
            ev.record(self.torch.cuda.current_stream(self.device))
            self._pack_done = ev


# ------------------------------------------------------------------------------------------
# Device-pointer path (what models.Generator.forward uses with torch tensors)
# ------------------------------------------------------------------------------------------
class GeneratorDevice(_PackedBlob):
    """Packed weights + workspace cache on one CUDA device, driven with torch tensors.  Each CUDA stream gets its own
    workspace and status watch (_PerStream), so forwards on distinct streams or threads may run concurrently; the
    methods that read a workspace back (check_status, stage_output) read the current stream's."""

    def __init__(self, device):
        import torch
        self.torch = torch
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise EngineError("the native engine runs on CUDA devices only (got %s)" % (device,))
        with torch.cuda.device(self.device):
            check(lib().mg_device_check())
        self._packed = torch.empty((lib().mg_gen_packed_bytes() + 3) // 4, dtype=torch.float32, device=self.device)
        self._pack_done = None
        self._scratch = _PerStream(torch, self.device, "Generator.forward")

    @property
    def _ws(self):
        """The current stream's workspace (None before its first forward)."""
        return self._scratch.current().bufs.get("ws")

    @property
    def _watch(self):
        return self._scratch.current().watch

    def pack(self, vs, gs, bs):
        """vs/gs/bs: 30 contiguous fp32 CUDA tensors each (weight_v, weight_g, bias; reference order)."""
        torch = self.torch
        keep = []
        def ptrs(ts):
            out = []
            for t in ts:
                t = t.detach()
                if t.device != self.device or t.dtype != torch.float32:
                    raise EngineError("generator parameters must be fp32 tensors on %s" % (self.device,))
                t = t.contiguous()
                keep.append(t)
                out.append(t.data_ptr())
            return _ptr_array(out)
        if not (len(vs) == len(gs) == len(bs) == NUM_LAYERS):
            raise EngineError("expected %d layers" % NUM_LAYERS)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_pack(ptrs(vs), ptrs(gs), ptrs(bs), self._packed.data_ptr(), stream))
            self._pack_enqueued()
        del keep

    def workspace(self, B, T):
        """The current stream's workspace, grown to mg_gen_workspace_bytes(B, T)."""
        return self._scratch.current().buffer("ws", lib().mg_gen_workspace_bytes(B, T))

    def forward(self, mel, out=None, precision="fp32", dtype=None):
        """mel [B, 80, T] -> audio [B, 1, 256 T].  precision "fp32" (the default) or "bf16" (one bf16 pass per tensor-core
        product: inference only, contract at mg_gen_forward_precision in include/melgan_b200.h).  dtype torch.float32 (the
        default) or torch.int16: 16-bit PCM written by the last kernel, pcm16 of the float audio bit for bit (contract at
        mg_gen_forward_pcm16); out= must then be int16."""
        return self._forward(mel, None, None, None, out, precision, dtype)

    def forward_ragged(self, mel, lengths, out=None, precision="fp32", dtype=None):
        """Ragged batch (inference): mel [B, 80, T_max] with item i's frames [0, lengths[i]) valid (the rest is never read)
        -> audio [B, 1, 256 T_max]; item i's first 256 lengths[i] samples equal its own forward (at the same precision) bit
        for bit, the rest are 0.  lengths: a list, a tuple or a CPU integer tensor.  dtype as for forward.  Asynchronous,
        like forward."""
        return self._forward(mel, lengths, None, None, out, precision, dtype)

    def forward_voices(self, voices, mel, voice, lengths=None, out=None, precision="fp32", dtype=None):
        """Many voices in one forward (inference): item i of mel [B, 80, T_max] runs on the weights of voices[voice[i]] (a
        sequence of GeneratorDevice on this device, this one among them or not) -> audio [B, 1, 256 T_max], each item bit
        for bit its own forward on its own voice (at the same precision; 0 past 256 lengths[i] samples).  voice: B ids in
        [0, len(voices)), and lengths as in forward_ragged (None: every item T_max frames), each a list, a tuple or a CPU
        integer tensor.  Items sorted by voice run fastest (contract at mg_gen_forward_voices, include/melgan_b200.h).
        dtype as for forward.  Uses this module's scratch of the current stream.  Asynchronous, like forward."""
        return self._forward(mel, lengths, list(voices), voice, out, precision, dtype)

    def _forward(self, mel, lengths, voices, voice, out, precision, dtype):
        """forward, forward_ragged and forward_voices: lengths None (every item T_max frames) or B lengths; voices None
        (every item on this module's weights) or a list of GeneratorDevice with B voice ids."""
        torch = self.torch
        code = _precision(precision)
        pcm = _pcm16(torch.float32 if dtype is None else dtype)
        if mel.dim() != 3 or mel.shape[1] != 80:
            T = "T" if lengths is None and voices is None else "T_max"
            raise EngineError("mel must be [B, 80, %s], got %s" % (T, tuple(mel.shape)))
        if mel.device != self.device or mel.dtype != torch.float32:
            raise EngineError("mel must be an fp32 tensor on %s" % (self.device,))
        if voices is not None:
            if not voices:
                raise EngineError("forward_voices needs at least one voice")
            for v in voices:
                if not isinstance(v, GeneratorDevice) or v.device != self.device:
                    raise EngineError("every voice must be a GeneratorDevice on %s" % (self.device,))
        mel = mel.contiguous()
        B, _, T = mel.shape
        lens = None if lengths is None else _lengths(lengths, B, T)
        ids = None if voices is None else _voice_ids(voice, B, len(voices))
        out = _audio_out(torch, out, (B, 1, 256 * T), pcm, self.device)
        sc = self._scratch.current()
        sc.check()  # the previous forward's status word on this stream, if its copy has landed
        nbytes = lib().mg_gen_workspace_bytes(B, T)
        ws = sc.buffer("ws", nbytes)
        with torch.cuda.device(self.device):
            args = (mel.data_ptr(), out.data_ptr(), B, T, lens, code, ws.data_ptr(), ws.numel() * 4,
                    torch.cuda.current_stream().cuda_stream)
            if pcm or voices is not None:
                blobs = [v.packed.data_ptr() for v in voices or [self]]  # (each read orders this stream after its pack)
                fn = lib().mg_gen_forward_pcm16 if pcm else lib().mg_gen_forward_voices
                check(fn(_ptr_array(blobs), len(blobs), ids, *args))
            else:
                check(lib().mg_gen_forward_precision(self.packed.data_ptr(), *args))
            off = (nbytes - 256) // 4  # the status word sits after the activation buffers
            sc.arm(ws.view(torch.int32)[off:off + 1])
        return out

    def forward_timed(self, mel, out):
        """Like forward; returns {kernel name: device time in ms} for every launch of the forward."""
        torch = self.torch
        mel = mel.contiguous()
        B, _, T = mel.shape
        ws = self.workspace(B, T)
        n = lib().mg_gen_forward_launches()
        ms = (ctypes.c_float * 16)()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_forward_timed(self.packed.data_ptr(), mel.data_ptr(), out.data_ptr(), B, T,
                                             ws.data_ptr(), ws.numel() * 4, stream, ms))
        return [(lib().mg_gen_kernel_name(i).decode(), ms[i]) for i in range(n)]

    def _last_ws(self):
        ws = self._ws
        if ws is None:
            raise EngineError("no forward has run on the current stream of %s" % (self.device,))
        return ws

    def check_status(self, B, T):
        """Synchronises the current stream and raises if the tensor-core pipeline of the last [B, 80, T] forward on it
        timed out (for a replayed CUDA graph: call it on the stream the graph was captured on)."""
        torch = self.torch
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_check_status(self._last_ws().data_ptr(), B, T, stream))

    def convt(self, stage, x):
        """LeakyReLU -> ConvTranspose1d of stage 0..3 on the tensor cores; x [B, 512>>stage, Lin]; synchronous."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if C != (512 >> stage):
            raise EngineError("stage %d expects %d input channels" % (stage, 512 >> stage))
        y = torch.empty((B, 256 >> stage, L * (8 if stage < 2 else 2)), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_convt(self.packed.data_ptr(), stage, x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def resblock(self, stage, x):
        """One tensor-core ResBlock (stage 0..3) on x [B, 256>>stage, L]; synchronous."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if C != (256 >> stage):
            raise EngineError("stage %d expects %d channels" % (stage, 256 >> stage))
        y = torch.empty_like(x)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_resblock(self.packed.data_ptr(), stage, x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def upres(self, stage, x):
        """Stage 2 or 3 as one kernel: LeakyReLU -> ConvTranspose1d(k4, s2) -> ResBlock on x [B, 512>>stage, Lin];
        returns [B, 256>>stage, 2 Lin]; synchronous."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if stage not in (2, 3) or C != (512 >> stage):
            raise EngineError("upres: stage 2 / 3 expect 128 / 64 input channels")
        y = torch.empty((B, 256 >> stage, 2 * L), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_upres(self.packed.data_ptr(), stage, x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def upres_post(self, x):
        """The default chain's last kernel: LeakyReLU -> ConvTranspose1d(k4, s2) of stage 3 -> ResBlock -> LeakyReLU ->
        conv_post -> tanh on x [B, 64, Lin] -> audio [B, 1, 2 Lin]; synchronous."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if C != 64:
            raise EngineError("upres_post expects 64 input channels")
        y = torch.empty((B, 1, 2 * L), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_upres_post(self.packed.data_ptr(), x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def resup(self, stage, x):
        """ResBlock `stage` (0..2) + the next stage's LeakyReLU -> ConvTranspose1d at its tail, one kernel:
        x [B, 256>>stage, L] -> [B, 128>>stage, S L] (S = 8 for stage 0, else 2); synchronous parity entry point."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if stage not in (0, 1, 2) or C != (256 >> stage):
            raise EngineError("resup: stage 0..2 with 256>>stage channels")
        y = torch.empty((B, C // 2, L * (8 if stage == 0 else 2)), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_resup(self.packed.data_ptr(), stage, x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def conv_pre(self, mel):
        """conv_pre alone (models.py:46,62): mel [B, 80, T] -> [B, 512, T]; synchronous parity entry point."""
        torch = self.torch
        mel = mel.contiguous()
        B, _, T = mel.shape
        y = torch.empty((B, 512, T), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_conv_pre(self.packed.data_ptr(), mel.data_ptr(), y.data_ptr(), B, T, stream))
        return y

    # kernel k of the default chain: (input channels, output channels, output positions per input position)
    CHAIN_SHAPES = ((80, 512, 1), (512, 256, 8), (256, 256, 1), (256, 128, 8), (128, 128, 1), (128, 64, 2), (64, 64, 1), (64, 1, 2))

    def chain_kernel(self, k, x, lengths=None, precision="fp32", out=None):
        """Kernel k (0..7) of the default chain alone, as the forward and the stream launch it (mg_gen_chain_kernel):
        x [B, Cin, L_max] -> [B, Cout, R L_max] (CHAIN_SHAPES[k]); lengths: None (every item L_max) or B lengths in kernel
        k's input units (list, tuple or CPU tensor).  out: an optional fp32 CUDA tensor whose first B Cout R L_max elements
        receive the output (a view of them is returned), e.g. a NaN-filled buffer with a guard region after it.
        Synchronous."""
        torch = self.torch
        code = _precision(precision)
        if not isinstance(k, int) or not 0 <= k < len(self.CHAIN_SHAPES):
            raise EngineError("chain kernel index must be 0..7 (got %r)" % (k,))
        cin, cout, R = self.CHAIN_SHAPES[k]
        if x.dim() != 3 or x.shape[1] != cin:
            raise EngineError("chain kernel %d expects x [B, %d, L], got %s" % (k, cin, tuple(x.shape)))
        if x.device != self.device or x.dtype != torch.float32:
            raise EngineError("x must be an fp32 tensor on %s" % (self.device,))
        x = x.contiguous()
        B, _, L = x.shape
        lens = None if lengths is None else _lengths(lengths, B, L)
        n = B * cout * R * L
        if out is None:
            out = torch.empty(n, dtype=torch.float32, device=self.device)
        elif out.device != self.device or out.dtype != torch.float32 or not out.is_contiguous() or out.numel() < n:
            raise EngineError("out must be a contiguous fp32 tensor on %s of at least %d elements" % (self.device, n))
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_chain_kernel(self.packed.data_ptr(), k, x.data_ptr(), out.data_ptr(), B, L, lens, code, stream))
        return out.view(-1)[:n].view(B, cout, R * L)

    def resblock_post(self, x):
        """Last ResBlock + LeakyReLU -> conv_post -> tanh (models.py:66-69) on x [B, 32, L] -> audio [B, 1, L]; synchronous."""
        torch = self.torch
        x = x.contiguous()
        B, C, L = x.shape
        if C != 32:
            raise EngineError("resblock_post expects 32 channels")
        y = torch.empty((B, 1, L), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_resblock_post(self.packed.data_ptr(), x.data_ptr(), y.data_ptr(), B, L, stream))
        return y

    def stage_output(self, which, B, T):
        """Activation after conv_pre (0) or stage 0..2 (1..3) of the last forward on the current stream, NCL."""
        torch = self.torch
        shapes = [(B, 512, T), (B, 256, 8 * T), (B, 128, 64 * T), (B, 64, 128 * T)]
        out = torch.empty(shapes[which], dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_gen_stage_output(self._last_ws().data_ptr(), which, out.data_ptr(), B, T, stream))
        return out


STREAM_END, STREAM_RESET = 1, 2  # MG_GEN_STREAM_END / _RESET, include/melgan_b200.h


class GeneratorStream:
    """Incremental vocoding of up to ``max_sessions`` live mel streams (mg_gen_stream_*, contract in
    include/melgan_b200.h).  Each step pushes a few new frames per session and returns the audio samples that became final:
    256 t - lookahead_samples of them after t frames, all 256 t after the step that ends the utterance, and their
    concatenation equals Generator.generate of the whole mel bit for bit.

    packed_fn: a callable returning the GeneratorDevice whose packed weights a step reads (Generator._ensure_packed, so
    weights changed between steps are re-packed), or a list of them, one per voice (models.stream_voices): slot i then
    runs on the weights of voice[i] (mg_gen_stream_step_voices; an open utterance keeps the voice it was opened with until
    it ends or is reset).  state: optional caller-provided uint8 CUDA tensor of at least mg_gen_stream_state_bytes bytes
    (the stream never lets a byte it has not written reach an output).  dtype: the handle's audio format, torch.float32
    (the default) or torch.int16 (16-bit PCM, pcm16 of the float samples bit for bit: mg_gen_stream_step_pcm16).

    One thread drives a handle at a time, and all steps of one handle must be enqueued on one CUDA stream (or otherwise
    ordered), as for mg_gen_stream_step: the state and the mel staging buffer that ``step`` copies each chunk into are
    the handle's own, and the next step overwrites them in stream order.  Distinct handles of one generator may step
    concurrently on distinct streams or threads."""

    def __init__(self, packed_fn, device, max_sessions=1, max_push_frames=32, precision="fp32", state=None, dtype=None):
        import torch
        self.torch = torch
        self.dtype = torch.float32 if dtype is None else dtype
        _pcm16(self.dtype)
        self._packed_fn = packed_fn
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise EngineError("stream: the native engine runs on CUDA devices only (got %s)" % (device,))
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.precision = precision
        code = _precision(precision)
        self.max_sessions, self.max_push_frames = int(max_sessions), int(max_push_frames)
        nbytes = lib().mg_gen_stream_state_bytes(self.max_sessions, self.max_push_frames)
        if nbytes == 0:
            raise EngineError("stream: max_sessions must lie in [1, 256] and max_push_frames in [1, 65536]")
        if state is None:
            state = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if state.device != self.device or state.numel() * state.element_size() < nbytes or not state.is_contiguous():
            raise EngineError("stream: state must be a contiguous CUDA tensor of at least %d bytes on %s" % (nbytes, self.device))
        self.state = state
        self.lookahead_samples = lib().mg_gen_stream_lookahead()
        self.max_out = lib().mg_gen_stream_max_out(self.max_push_frames)
        self._h = ctypes.c_void_p()
        check(lib().mg_gen_stream_create(ctypes.byref(self._h), self.max_sessions, self.max_push_frames, code, state.data_ptr(),
                                         state.numel() * state.element_size()))
        self._mel = torch.zeros((self.max_sessions, 80, self.max_push_frames), dtype=torch.float32, device=self.device)

    def step_packed(self, mel, frames, flags=None, audio=None, voice=None):
        """The C step on a packed buffer: mel [n, 80, max_push_frames] fp32 CUDA (slot i's frames first), frames / flags: n
        ints, voice: None (every slot on the first voice) or n voice ids as for ``step``.  Returns (audio [n, max_out],
        per-slot sample counts as a list of ints).  audio: None (a new tensor of the handle's dtype) or a contiguous fp32 or
        int16 CUDA tensor [n, max_out], whose dtype picks this step's format (float and int16 steps may alternate)."""
        torch = self.torch
        n = len(frames)
        devs = self._packed_fn()
        devs = list(devs) if isinstance(devs, (list, tuple)) else [devs]
        for d in devs:
            if d.device != self.device:
                raise EngineError("stream: a voice's weights are on %s, the stream on %s" % (d.device, self.device))
        ids = None if voice is None else _voice_ids(voice, n, len(devs))
        if audio is None:
            audio = torch.empty((n, self.max_out), dtype=self.dtype, device=self.device)
        pcm = audio.dtype == torch.int16
        if pcm and (audio.device != self.device or audio.dim() != 2 or audio.shape[0] < n or audio.shape[1] != self.max_out
                    or not audio.is_contiguous()):
            raise EngineError("stream: int16 audio must be a contiguous [%d, %d] tensor on %s" % (n, self.max_out, self.device))
        fr = (ctypes.c_int * max(n, 1))(*[int(v) for v in frames])
        fl = (ctypes.c_int * max(n, 1))(*[int(v) for v in flags]) if flags is not None else None
        cnt = (ctypes.c_int * max(n, 1))()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            blobs = _ptr_array([d.packed.data_ptr() for d in devs])  # (each read orders this stream after its pack)
            fn = lib().mg_gen_stream_step_pcm16 if pcm else lib().mg_gen_stream_step_voices
            check(fn(self._h, blobs, len(devs), ids, mel.data_ptr() if mel is not None else None, fr, fl, n, audio.data_ptr(), cnt,
                     stream))
        return audio, [cnt[i] for i in range(n)]

    def step(self, chunks, end=None, reset=None, voice=None):
        """chunks: one entry per slot 0 .. n-1, each a [80, n_i] fp32 CUDA tensor (0 <= n_i <= max_push_frames) or None;
        end / reset: None or n booleans (end: the utterance ends after this chunk; reset: drop the slot's unfinished
        utterance first); voice: None (every slot on the first voice) or n voice ids (a list, a tuple or a CPU integer
        tensor) -- a slot's id may change only on a step that resets it or once its utterance has ended.  Returns n [1, m_i]
        CUDA tensors of newly final audio in the handle's dtype, owned by the caller.  Asynchronous on the current stream: the lengths are known on
        return, the values once the stream gets there."""
        n = len(chunks)
        if n > self.max_sessions:
            raise EngineError("stream: %d chunks for %d sessions" % (n, self.max_sessions))
        frames = []
        for i, c in enumerate(chunks):
            if c is None:
                frames.append(0)
                continue
            if c.dim() != 2 or c.shape[0] != 80 or c.shape[1] > self.max_push_frames:
                raise EngineError("stream: chunk %d must be [80, n] with n <= %d, got %s" % (i, self.max_push_frames, tuple(c.shape)))
            if c.device != self.device or c.dtype != self.torch.float32:
                raise EngineError("stream: chunks must be fp32 tensors on %s" % (self.device,))
            frames.append(int(c.shape[1]))
            if c.shape[1]:
                self._mel[i, :, :c.shape[1]].copy_(c)
        flags = [(STREAM_END if end is not None and end[i] else 0) | (STREAM_RESET if reset is not None and reset[i] else 0)
                 for i in range(n)]
        audio, counts = self.step_packed(self._mel, frames, flags, voice=voice)
        return [audio[i:i + 1, :m] for i, m in enumerate(counts)]

    def check_status(self):
        """Synchronises and raises if a tensor-core pipeline wait of any step so far timed out."""
        with self.torch.cuda.device(self.device):
            check(lib().mg_gen_stream_check_status(self._h, self.torch.cuda.current_stream().cuda_stream))

    def close(self):
        if self._h:
            lib().mg_gen_stream_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


D_CHANNELS = (16, 64, 256, 1024, 1024, 1024, 1)  # channels of the seven feature maps of one Discriminator


def msd_lengths(L):
    """Feature-map lengths [3][7] of the multi-scale discriminator for an input of L samples."""
    lens = (ctypes.c_int * 21)()
    check(lib().mg_msd_lengths(int(L), lens))
    return [[lens[s * 7 + l] for l in range(7)] for s in range(3)]


LOSS_L1, LOSS_ONE_MINUS_SQ, LOSS_SQ = 0, 1, 2  # row modes of mg_loss_forward (include/melgan_b200.h)


def _loss_tables(a, b, modes):
    import torch
    dev = a[0].device
    if dev.type != "cuda":
        raise EngineError("the fused loss kernels run on CUDA tensors only")
    keep_a, keep_b = [], []
    for t, u, m in zip(a, b, modes):
        if t.dtype != torch.float32 or t.device != dev or (m == LOSS_L1 and (u is None or u.shape != t.shape or u.device != dev)):
            raise EngineError("loss rows must be fp32 tensors of equal shape on one CUDA device")
        keep_a.append(t.contiguous())
        keep_b.append(u.contiguous() if m == LOSS_L1 else None)
    n = (ctypes.c_longlong * len(a))(*[t.numel() for t in keep_a])
    md = (ctypes.c_int * len(a))(*modes)
    pa = _ptr_array([t.data_ptr() for t in keep_a])
    pb = _ptr_array([u.data_ptr() if u is not None else 0 for u in keep_b])
    return dev, keep_a, keep_b, n, md, pa, pb


def loss_forward(a, b, modes):
    """Row means of a fused loss table (mg_loss_forward): a, b lists of CUDA tensors, modes list of LOSS_*; returns a
    float32 CUDA tensor [len(a)].  One reduction launch + one fixed-order combine, no host sync."""
    import torch
    dev, keep_a, keep_b, n, md, pa, pb = _loss_tables(a, b, modes)
    out = torch.empty(len(a), dtype=torch.float32, device=dev)
    nbytes = lib().mg_loss_workspace_bytes(n, len(a))
    ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        check(lib().mg_loss_forward(pa, pb, n, md, len(a), out.data_ptr(), ws.data_ptr(), nbytes, stream))
    return out


def loss_backward(a, b, modes, grad_out, need_b, out_a=None, out_b=None):
    """Gradients of the row means w.r.t. a (and b where need_b[i] and the row is an L1 pair), scaled by grad_out [rows].
    out_a / out_b: optional preallocated contiguous tensors to write into (e.g. the two halves of one stacked buffer)."""
    import torch
    dev, keep_a, keep_b, n, md, pa, pb = _loss_tables(a, b, modes)
    ga = list(out_a) if out_a is not None else [torch.empty_like(t) for t in keep_a]
    gb = (list(out_b) if out_b is not None else
          [torch.empty_like(u) if (u is not None and nb) else None for u, nb in zip(keep_b, need_b)])
    for t in ga + [u for u in gb if u is not None]:
        if not t.is_contiguous():
            raise EngineError("loss_backward: output gradients must be contiguous")
    pga = _ptr_array([t.data_ptr() for t in ga])
    pgb = _ptr_array([t.data_ptr() if t is not None else 0 for t in gb])
    grad_out = grad_out.to(device=dev, dtype=torch.float32).contiguous()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream().cuda_stream
        check(lib().mg_loss_backward(pa, pb, n, md, len(a), grad_out.data_ptr(), pga, pgb, stream))
    return ga, gb


class DiscriminatorDevice(_PackedBlob):
    """Packed discriminator weights on one CUDA device, driven with torch tensors: the three-scale stack of
    MultiScaleDiscriminator (ndisc = 3) or one stand-alone Discriminator (ndisc = 1).  The status word and the backward
    workspace are kept per CUDA stream (_PerStream), so calls on distinct streams or threads may run concurrently."""

    def __init__(self, device, ndisc=3):
        import torch
        self.torch = torch
        self.device = torch.device(device)
        self.ndisc = ndisc
        if self.device.type != "cuda":
            raise EngineError("the native engine runs on CUDA devices only (got %s)" % (device,))
        if ndisc not in (1, 3):
            raise EngineError("DiscriminatorDevice: ndisc must be 1 or 3")
        with torch.cuda.device(self.device):
            check(lib().mg_device_check())
        nbytes = lib().mg_msd_packed_bytes() if ndisc == 3 else lib().mg_disc_packed_bytes()
        self._packed = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=self.device)
        self._pack_done = None
        self._scratch = _PerStream(torch, self.device, "Discriminator forward")

    @property
    def status(self):
        """The current stream's status word (int32 [64], zeroed when first made): every call on the stream reports a
        timed-out tensor-core pipeline wait in it."""
        return self._scratch.current().buffer("status", 64 * 4, zeros=True)

    @property
    def _watch(self):
        return self._scratch.current().watch

    def pack(self, vs, gs, bs):
        """vs/gs/bs: 7 * ndisc fp32 CUDA tensors each (discriminator-major, layers in registration order)."""
        torch = self.torch
        if not (len(vs) == len(gs) == len(bs) == 7 * self.ndisc):
            raise EngineError("expected %d discriminator layers" % (7 * self.ndisc))
        keep = []

        def ptrs(ts):
            out = []
            for t in ts:
                t = t.detach()
                if t.device != self.device or t.dtype != torch.float32:
                    raise EngineError("discriminator parameters must be fp32 tensors on %s" % (self.device,))
                t = t.contiguous()
                keep.append(t)
                out.append(t.data_ptr())
            return _ptr_array(out)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            fn = lib().mg_msd_pack if self.ndisc == 3 else lib().mg_disc_pack
            check(fn(ptrs(vs), ptrs(gs), ptrs(bs), self._packed.data_ptr(), stream))
            self._pack_enqueued()

    def forward(self, y):
        """y [Bt, 1, L] -> list of ndisc lists of 7 feature maps [Bt, C, len] (fresh tensors)."""
        torch = self.torch
        if y.dim() != 3 or y.shape[1] != 1:
            raise EngineError("audio must be [B, 1, L], got %s" % (tuple(y.shape),))
        if y.device != self.device or y.dtype != torch.float32:
            raise EngineError("audio must be an fp32 tensor on %s" % (self.device,))
        y = y.contiguous()
        Bt, _, L = y.shape
        lens = msd_lengths(L)
        scratch = self._scratch.current()
        scratch.check()
        status = scratch.buffer("status", 64 * 4, zeros=True)
        fmaps = [[torch.empty((Bt, D_CHANNELS[l], lens[s][l]), dtype=torch.float32, device=self.device)
                  for l in range(7)] for s in range(self.ndisc)]
        ptrs = _ptr_array([f.data_ptr() for sc in fmaps for f in sc])
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            fn = lib().mg_msd_forward if self.ndisc == 3 else lib().mg_disc_forward
            check(fn(self.packed.data_ptr(), y.data_ptr(), Bt, L, ptrs, status.data_ptr(), stream))
            scratch.arm(status[:1])
        return fmaps

    def layer_forward(self, scale, layer, x, out=None):
        """Layer `layer` (1..6) of discriminator `scale` alone on x [Bt, Cin, Lin] (mg_msd_layer_forward, the launcher the
        forward runs): returns out [Bt, Cout, Lout], written into `out` (a flat fp32 buffer of at least that many elements,
        e.g. one filled with a marker to see what the kernel writes) when given.  Asynchronous: check_status() reports a
        timed-out pipeline wait."""
        torch = self.torch
        from .synth import DISCRIMINATOR_LAYERS
        _n, cin, cout, k, stride, _g, pad = DISCRIMINATOR_LAYERS[layer]
        if x.dim() != 3 or x.shape[1] != cin or x.device != self.device or x.dtype != torch.float32:
            raise EngineError("layer %d expects x [Bt, %d, L] fp32 on %s" % (layer, cin, self.device))
        x = x.contiguous()
        Bt, _, Lin = x.shape
        n = Bt * cout * ((Lin + 2 * pad - k) // stride + 1)
        if out is None:
            out = torch.empty(max(n, 1), dtype=torch.float32, device=self.device)
        if out.numel() < n or out.dtype != torch.float32 or not out.is_contiguous():
            raise EngineError("out must be a contiguous fp32 buffer of at least %d elements" % n)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_layer_forward(self.packed.data_ptr(), scale, layer, x.data_ptr(), out.data_ptr(), Bt, Lin,
                                             self.status.data_ptr(), stream))
        return out[:n].view(Bt, cout, n // (Bt * cout))

    def scale_backward(self, scale, x0, fmaps, grads, need_gx0):
        """The whole backward of discriminator `scale` in one host call (mg_msd_scale_backward): x0 [Bt, 1, L0] its input,
        fmaps the 7 maps its forward returned, grads the gradient w.r.t. each (None: none).  Returns (gx0 | None, dws[7],
        dbs[7]) -- gradients of the FOLDED weights in torch layout; entries of layers the gradient does not reach are None.
        The intermediate gradients live in the current stream's workspace, reused by every call on that stream (in the
        stream's order)."""
        torch = self.torch
        from .synth import DISCRIMINATOR_LAYERS
        x0 = x0.contiguous()
        Bt, _, L0 = x0.shape
        gs = [g.contiguous() if g is not None else None for g in grads]
        keep = [f.contiguous() for f in fmaps]
        dws = [torch.empty((cout, cin // groups, k), dtype=torch.float32, device=self.device)
               for _n, cin, cout, k, _s, groups, _p in DISCRIMINATOR_LAYERS]
        dbs = [torch.empty((cout,), dtype=torch.float32, device=self.device) for _n, _cin, cout, *_ in DISCRIMINATOR_LAYERS]
        gx0 = torch.empty_like(x0) if need_gx0 else None
        nbytes = lib().mg_msd_scale_backward_workspace_bytes(Bt, L0)
        sc = self._scratch.current()
        ws, status = sc.buffer("bwd", nbytes), sc.buffer("status", 64 * 4, zeros=True)
        reached = (ctypes.c_int * 7)()
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_scale_backward(
                self.packed.data_ptr(), scale, x0.data_ptr(), _ptr_array([f.data_ptr() for f in keep]),
                _ptr_array([g.data_ptr() if g is not None else None for g in gs]), gx0.data_ptr() if need_gx0 else None,
                _ptr_array([t.data_ptr() for t in dws]), _ptr_array([t.data_ptr() for t in dbs]), reached, ws.data_ptr(),
                ws.numel() * 4, Bt, L0, status.data_ptr(), stream))
        hit = [bool(r) for r in reached]
        return (gx0 if hit[0] else None), [w if h else None for w, h in zip(dws, hit)], [b if h else None for b, h in zip(dbs, hit)]

    def grouped_backward(self, scale, layer, dz, x, need_dx=True):
        """Gradients of grouped conv `layer` (1..4) of discriminator `scale`: dz [Bt, Cout, Lout] (already multiplied by
        LeakyReLU'), x [Bt, Cin, Lin] the layer input -> (dx or None, dw [Cout, 4, 41] w.r.t. the folded weight, db)."""
        torch = self.torch
        dz, x = dz.contiguous(), x.contiguous()
        Bt, cout, Lout = dz.shape
        _, cin, Lin = x.shape
        dx = torch.empty_like(x) if need_dx else None
        dw = torch.empty((cout, 4, 41), dtype=torch.float32, device=self.device)
        db = torch.empty(cout, dtype=torch.float32, device=self.device)
        nbytes = lib().mg_msd_grouped_backward_workspace_bytes(layer, Bt, Lout)
        ws = torch.empty((nbytes + 3) // 4, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_grouped_backward(self.packed.data_ptr(), scale, layer, dz.data_ptr(), x.data_ptr(),
                                                dx.data_ptr() if need_dx else None, dw.data_ptr(), db.data_ptr(),
                                                ws.data_ptr(), nbytes, Bt, Lin, Lout, stream))
        return dx, dw, db

    def post1_dgrad(self, scale, dz):
        """dx of conv_post1 of discriminator `scale` from dz [Bt, 1024, L] (wgmma, transposed weight copy of the blob)."""
        torch = self.torch
        dz = dz.contiguous()
        Bt, C, L = dz.shape
        if C != 1024:
            raise EngineError("post1_dgrad expects 1024 channels")
        dx = torch.empty_like(dz)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_post1_dgrad(self.packed.data_ptr(), scale, dz.data_ptr(), dx.data_ptr(), Bt, L,
                                           self.status.data_ptr(), stream))
        return dx

    def edge_backward(self, scale, layer, dz, x, need_dx=True):
        """(dx | None, dw, db) of conv_pre (layer 0) or conv_post2 (layer 6) of discriminator `scale`; dw in the torch layout."""
        torch = self.torch
        x, dz = x.contiguous(), dz.contiguous()
        Bt, L = x.shape[0], x.shape[2]
        cin, cout, k = (1, 16, 15) if layer == 0 else (1024, 1, 3)
        if tuple(x.shape) != (Bt, cin, L) or tuple(dz.shape) != (Bt, cout, L):
            raise EngineError(f"edge_backward(layer {layer}) expects x [Bt, {cin}, L] and dz [Bt, {cout}, L]")
        dx = torch.empty_like(x) if need_dx else None
        dw = torch.empty((cout, cin, k), dtype=torch.float32, device=x.device)
        db = torch.empty((cout,), dtype=torch.float32, device=x.device)
        nbytes = lib().mg_msd_edge_backward_workspace_bytes(layer, Bt, L)
        ws = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=x.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_edge_backward(self.packed.data_ptr(), scale, layer, dz.data_ptr(), x.data_ptr(),
                                             dx.data_ptr() if need_dx else None, dw.data_ptr(), db.data_ptr(),
                                             ws.data_ptr(), nbytes, Bt, L, stream))
        return dx, dw, db

    def post1_wgrad(self, x, dz):
        """(dW [1024, 1024, 5], db [1024]) of conv_post1 from its input x and dz, both [Bt, 1024, L] (wgmma, split-bf16)."""
        torch = self.torch
        x, dz = x.contiguous(), dz.contiguous()
        Bt, C, L = dz.shape
        if C != 1024 or tuple(x.shape) != (Bt, C, L):
            raise EngineError("post1_wgrad expects x and dz of shape [Bt, 1024, L]")
        dw = torch.empty((1024, 1024, 5), dtype=torch.float32, device=dz.device)
        db = torch.empty((1024,), dtype=torch.float32, device=dz.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_post1_wgrad(x.data_ptr(), dz.data_ptr(), dw.data_ptr(), db.data_ptr(), Bt, L,
                                           self.status.data_ptr(), stream))
        return dw, db

    def lrelu_backward(self, g1, g2, out):
        """(g1 + g2) * LeakyReLU'(out) in one launch; g1 or g2 may be None (not both)."""
        torch = self.torch
        if g1 is None:
            g1, g2 = g2, None
        g1 = g1.contiguous()
        g2 = g2.contiguous() if g2 is not None else None
        out = out.contiguous()
        dz = torch.empty_like(out)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_lrelu_backward(g1.data_ptr(), g2.data_ptr() if g2 is not None else None, out.data_ptr(),
                                          dz.data_ptr(), out.numel(), stream))
        return dz

    def wn_backward(self, vs, gs, dws):
        """(d weight_v, d weight_g) of the 7 * ndisc layers from the gradients of their folded weights (None: layer skipped)."""
        torch = self.torch
        vs = [t.detach().contiguous() for t in vs]
        gs = [t.detach().contiguous() for t in gs]
        dws = [t.contiguous() if t is not None else None for t in dws]
        dvs = [torch.empty_like(v) if d is not None else None for v, d in zip(vs, dws)]
        dgs = [torch.empty_like(g) if d is not None else None for g, d in zip(gs, dws)]

        pad = 21 - len(vs)  # the launch walks a 21-row table; a stand-alone Discriminator fills the rest with skipped rows

        def arr(ts, fill):
            return _ptr_array([t.data_ptr() if t is not None else None for t in ts] + [fill] * pad)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_wn_backward(arr(vs, vs[0].data_ptr()), arr(gs, gs[0].data_ptr()), arr(dws, None), arr(dvs, None),
                                           arr(dgs, None), stream))
        return dvs, dgs

    def check_status(self):
        torch = self.torch
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().mg_msd_check_status(self.status.data_ptr(), stream))


# ------------------------------------------------------------------------------------------
# Host-buffer path (no torch needed): numpy in, numpy out, copies inside the call
# ------------------------------------------------------------------------------------------
class GeneratorHost:
    """mg_gen_engine_* wrapper: the call a non-PyTorch host makes (host buffers in and out)."""

    def __init__(self, max_B=1, max_T=32):
        self._h = ctypes.c_void_p()
        check(lib().mg_gen_engine_create(ctypes.byref(self._h), max_B, max_T))

    def load_state(self, state):
        """state: mapping name -> float32 ndarray with the reference's state_dict keys."""
        from .synth import GENERATOR_LAYERS
        keep, vs, gs, bs = [], [], [], []
        for name, *_ in GENERATOR_LAYERS:
            for lst, suffix in ((vs, ".weight_v"), (gs, ".weight_g"), (bs, ".bias")):
                a = np.ascontiguousarray(state[name + suffix], dtype=np.float32)
                keep.append(a)
                lst.append(a.ctypes.data)
        check(lib().mg_gen_engine_load_state(self._h, _ptr_array(vs), _ptr_array(gs), _ptr_array(bs)))

    def forward(self, mel, out=None, precision="fp32", dtype=np.float32):
        """mel [B, 80, T] -> audio [B, 1, 256 T]; precision as for GeneratorDevice.forward.  dtype np.float32 (the default)
        or np.int16: 16-bit PCM, pcm16 of the float audio bit for bit (mg_gen_engine_forward_pcm16)."""
        return self._forward(mel, None, out, precision, dtype)

    @staticmethod
    def _out(out, shape, pcm):
        dt = np.int16 if pcm else np.float32
        if out is None:
            return np.empty(shape, dt)
        if pcm or out.dtype == np.int16:
            if out.dtype != dt or tuple(out.shape) != tuple(shape) or not out.flags.c_contiguous:
                raise EngineError("out must be a C-contiguous %s array of shape %s" % (np.dtype(dt).name, tuple(shape)))
        return out

    def forward_ragged(self, mel, lengths, out=None, precision="fp32", dtype=np.float32):
        """Ragged batch from host memory (mg_gen_engine_forward_ragged): mel [B, 80, T_max], lengths and precision as for
        GeneratorDevice.forward_ragged, dtype as for forward -> audio [B, 1, 256 T_max]."""
        return self._forward(mel, lengths, out, precision, dtype)

    def _forward(self, mel, lengths, out, precision, dtype):
        code = _precision(precision)
        pcm = _pcm16_np(dtype)
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        if mel.ndim != 3 or mel.shape[1] != 80:
            raise EngineError("mel must be [B, 80, %s]" % ("T" if lengths is None else "T_max"))
        B, _, T = mel.shape
        lens = None if lengths is None else _lengths(lengths, B, T)
        out = self._out(out, (B, 1, 256 * T), pcm)
        fn = lib().mg_gen_engine_forward_pcm16 if pcm else lib().mg_gen_engine_forward_precision
        check(fn(self._h, mel.ctypes.data, out.ctypes.data, B, T, lens, code))
        return out

    def forward_ptr(self, mel_ptr, out_ptr, B, T):
        """Raw host pointers (e.g. pinned torch tensors' data_ptr())."""
        check(lib().mg_gen_engine_forward(self._h, mel_ptr, out_ptr, B, T))

    HALO_FRAMES = 8  # the generator's receptive field is +-7 mel frames (SURVEY section 5); 8 for slack

    def stream(self, mel, chunk_frames=128, precision="fp32"):
        """Long-utterance streaming (BASELINE config 5): yields the audio of `mel` [1, 80, T] chunk by chunk, each chunk
        computed from its frames plus an 8-frame halo either side, so latency and memory are bounded by the chunk and the
        concatenation equals the whole-utterance result (every conv of the fused stages re-applies its zero padding only
        at the true ends, which a chunk touching an end reproduces exactly).  precision as for forward."""
        _precision(precision)  # (a bad value is refused before any chunk is computed)
        mel = np.ascontiguousarray(mel, dtype=np.float32)
        if mel.ndim != 3 or mel.shape[0] != 1 or mel.shape[1] != 80:
            raise EngineError("stream() takes one utterance [1, 80, T]")
        T, h = mel.shape[2], self.HALO_FRAMES
        for lo in range(0, T, chunk_frames):
            hi = min(T, lo + chunk_frames)
            a, b = max(0, lo - h), min(T, hi + h)
            audio = self.forward(mel[:, :, a:b], precision=precision)
            yield audio[:, :, (lo - a) * 256:(lo - a + hi - lo) * 256]

    def last_kernel_ms(self):
        ms = ctypes.c_float()
        check(lib().mg_gen_engine_last_kernel_ms(self._h, ctypes.byref(ms)))
        return ms.value

    def close(self):
        if self._h:
            lib().mg_gen_engine_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
