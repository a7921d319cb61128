"""Drop-in replacement for the reference's ``models`` module (/root/reference/models.py).

``train.py:13`` does ``from models import Generator, MultiScaleDiscriminator, feature_loss,
generator_loss, discriminator_loss``; this module exports the same five names with the same
constructor and ``forward`` signatures, the same ``state_dict`` keys, shapes and parameter
registration order (so reference checkpoints and Adam state load, SURVEY 8b), and leaves
``weight_g`` / ``weight_v`` / ``bias`` as ordinary leaf parameters so the reference's gradient
all-reduce wrapper (distributed.py:90-142) hooks them unchanged.

What runs where
  * ``Generator.forward`` (models.py:61-71 in the reference): eight hand-written sm_90a wgmma kernels in
    libmelgan_b200.so -- conv_pre, then LeakyReLU -> ConvTranspose1d and the fused six-conv ResBlock of each stage,
    the last stage as ONE kernel (its stride-2 ConvT, the ResBlock and LeakyReLU -> conv_post -> tanh) -- plus one launch that folds weight-norm for all 30 layers
    whenever the parameters changed.  CUDA only; a CPU tensor raises (the reference's CPU path lives in oracle/ as
    test infrastructure).
  * ``MultiScaleDiscriminator.forward`` (models.py:119-135, Discriminator.forward :87-103) on CUDA: real and generated
    audio are stacked into one batch and run through hand-written kernels -- AvgPool chain fused into each scale's
    conv_pre, grouped k41 convs and conv_post1 on wgmma -- after one launch that folds weight-norm for the 21 layers.
  * ``feature_loss`` / ``generator_loss`` / ``discriminator_loss`` (models.py:138-167) on CUDA tensors: every term of a
    loss is a row of one fused reduction launch (forward) and one gradient launch (backward).
  * Backward: the generator's runs as recomputation through stock PyTorch ops; the discriminators' walks the saved
    feature maps layer by layer on hand-written kernels only (grouped convs, conv_post1 dgrad / wgrad on wgmma,
    conv_pre / conv_post2, LeakyReLU, weight-norm): no cuDNN call in a discriminator's backward.
"""
import threading

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch._utils import _unflatten_dense_tensors
from torch.multiprocessing.reductions import StorageWeakRef
from torch.nn import AvgPool1d, Conv1d, ConvTranspose1d
from torch.nn.utils import weight_norm
from torch.optim.optimizer import register_optimizer_step_post_hook

from . import engine as _engine
from .optim import _bump_versions
from .synth import DISCRIMINATOR_LAYERS, GENERATOR_LAYERS

# Makes a module's lazy (re-)pack one step when host threads call it at once: the first caller packs (engine
# _PackedBlob orders every later read of the blob after that pack), the others see the weights already packed.
_PACK_LOCK = threading.Lock()


class _PackKey:
    """What a module's packed blob was folded from: every parameter's (data_ptr, _version), and a weak reference to each
    parameter's storage.  (data_ptr, _version) alone can recur: ``p.data = t`` keeps p's version counter, and the
    caching allocator may put t where a storage freed since the pack used to be (two ``vector_to_parameters`` calls in a
    row, ``.cpu()``, a new ``.data``, ``.cuda()``).  The freed storage's weak reference has expired then, so the key no
    longer matches.  A weak reference keeps no memory: a freed storage's bytes go back to the allocator as before."""

    def __init__(self, ts):
        self.key = tuple((t.data_ptr(), t._version) for t in ts)
        self.refs = [StorageWeakRef(t.untyped_storage()) for t in ts]

    def matches(self, ts):
        return self.key == tuple((t.data_ptr(), t._version) for t in ts) and not any(r.expired() for r in self.refs)


class _Repack:
    """The modules that fold their weight-norm parameters into a packed blob, keyed on every parameter (_PackKey).  The
    key sees in-place ops under no_grad, optimizer steps (the fused ones through _bump_after_fused_step) and
    ``load_state_dict``, and new storage (``p.data = t``, ``load_state_dict(assign=True)``, ``vector_to_parameters``,
    ``.to()``).  It cannot see an in-place write through ``p.data``, nor a write the host never issues, such as a
    replayed CUDA graph of an optimizer step.  Nor does it see ``torch._foreach_lerp_`` with a scalar weight, which
    ``swa_utils.AveragedModel``'s EMA update runs: on CUDA that op leaves the version counters as they were
    (torch 2.11)."""

    def _pack_if_changed(self, dev, vs, gs, bs):
        """dev.pack(vs, gs, bs) unless the blob was last folded from exactly these parameter values (call under
        _PACK_LOCK)."""
        ts = vs + gs + bs
        if self._packed_key is None or not self._packed_key.matches(ts):
            dev.pack(vs, gs, bs)
            self._packed_key = _PackKey(ts)

    def repack(self):
        """Makes the next call of this module, and of every module inside it, fold the parameters' current values.
        A stream or a ``generate_voices`` call built on it picks them up at its next step or call.  It does not reach
        a module that contains this one: call repack() on the module you will call, or on the outermost one."""
        with _PACK_LOCK:
            for m in self.modules():
                if isinstance(m, _Repack):
                    m._packed_key = None


@torch.compiler.disable  # in a compiled step, traced, the bump would be dropped
def _bump_after_fused_step(optimizer, args, kwargs):
    """torch.optim's fused steps (``Adam(fused=True)`` and the other ``fused`` optimizers) write the parameters without
    bumping their version counters, unlike the for-loop and foreach forms.  Bumping them here lets the modules' packed
    folds see the step, as autograd's saved-tensor checks then do too.  The hook is process-wide because an optimizer
    step does not say which modules its parameters belong to; for any other parameter the bump only does what the
    for-loop and foreach steps already do."""
    ps = [p for g in optimizer.param_groups if g.get("fused") for p in g["params"] if p.grad is not None]
    if ps:
        _bump_versions(ps)


register_optimizer_step_post_hook(_bump_after_fused_step)

_RES_DILATIONS = (1, 3, 9)


def get_padding(kernel_size, dilation=1):
    """'same' padding for an odd kernel (reference models.py:8-9)."""
    return (kernel_size * dilation - dilation) // 2


def _wn_conv(cin, cout, k, **kw):
    return weight_norm(Conv1d(cin, cout, k, **kw))


class ResBlock(nn.Module):
    """Parameter container with the reference's layout (models.py:12-30).  ``forward`` is the stock
    PyTorch restatement used only by the autograd (backward) path."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.convs1 = nn.ModuleList(
            [_wn_conv(in_channels, out_channels, 3, dilation=d, padding=get_padding(3, d)) for d in _RES_DILATIONS])
        self.convs2 = nn.ModuleList(
            [_wn_conv(in_channels, out_channels, 3, dilation=1, padding=get_padding(3, 1)) for _ in _RES_DILATIONS])

    def forward(self, x):
        for first, second in zip(self.convs1, self.convs2):
            x = second(F.leaky_relu(first(F.leaky_relu(x)))) + x
        return x


def _layer_modules(gen):
    """The 30 weight-normed modules of a Generator in reference registration order."""
    mods = [gen.conv_pre] + list(gen.ups)
    for rb in gen.resblocks:
        mods += list(rb.convs1) + list(rb.convs2)
    mods.append(gen.conv_post)
    return mods


def _owned_copies(tensors):
    """Copies of tensors (None stays None) carved out of one new allocation and filled by one multi-tensor copy."""
    src = [t for t in tensors if t is not None]
    if not src:
        return list(tensors)
    flat = torch.empty(sum(t.numel() for t in src), dtype=src[0].dtype, device=src[0].device)
    dst = _unflatten_dense_tensors(flat, src)  # src-shaped views of flat, made in one call (per-tensor views cost the host)
    torch._foreach_copy_(dst, src)
    it = iter(dst)
    return [next(it) if t is not None else None for t in tensors]


class _GeneratorFunction(torch.autograd.Function):
    """Forward on the fused sm_90a kernels; backward by recomputation through stock PyTorch ops (open row: native
    backward).  The recomputation -- 30 convs forward, their backward, weight-norm: ~600 launches that cost the host more
    than the GPU -- is captured ONCE per input shape as a pair of CUDA graphs (torch.cuda.make_graphed_callables) and
    replayed, so the step is no longer bound by eager launch overhead (MG_GEN_BWD_GRAPH=0: eager).
    Inputs: mel, then 30 x (weight_v, weight_g, bias).

    The gradients it returns belong to the caller on both paths.  A graphed backward writes them into static buffers of
    the graph that its next replay overwrites, so they are copied out (one flat allocation, one multi-tensor copy) before
    they are handed on: .grad accumulation across backward() calls, zero_grad(set_to_none=False), two calls in one loss
    and a mel.grad kept across later steps all see their own values.  The graph buffers are per module, so one module's
    backward must not run on two streams at once."""

    @staticmethod
    def forward(ctx, gen, mel, *params):
        ctx.gen = gen
        ctx.save_for_backward(mel, *params)
        ctx.graphed = gen._graphed_recompute(mel, params)  # built here (not inside backward): capture needs a quiet device
        return gen._engine_forward(mel)

    @staticmethod
    def backward(ctx, grad_out):
        gen = ctx.gen
        mel, *params = ctx.saved_tensors
        need_mel = ctx.needs_input_grad[1]
        graphed = ctx.graphed is not None and need_mel == ctx.graphed[1]
        with torch.enable_grad():
            mel_ = mel.detach().requires_grad_(need_mel)
            leaves = [p.detach().requires_grad_(True) for p in params]
            if graphed:
                y = ctx.graphed[0](mel_, *leaves)
            else:
                y = gen._torch_forward(mel_, leaves)
            wanted = ([mel_] if need_mel else []) + leaves
            grads = torch.autograd.grad(y, wanted, grad_out.contiguous(), allow_unused=True)
        if graphed:
            grads = _owned_copies(grads)
        grads = list(grads)
        gmel = grads.pop(0) if need_mel else None
        return (None, gmel, *grads)


class Generator(_Repack, nn.Module):
    """mel [B, 80, T] fp32 CUDA -> audio [B, 1, 256*T] (reference models.py:43-71).

    The weights are folded and packed at the first call and again whenever a parameter's _version or data_ptr changed:
    optimizer steps, in-place ops under no_grad, load_state_dict and p.data = t are seen.  In-place writes through
    p.data and replayed CUDA graphs (an optimizer step captured with capturable=True) are not, nor is an EMA update of
    swa_utils.AveragedModel on CUDA (_Repack): call repack() after them."""

    def __init__(self):
        super().__init__()
        self.conv_pre = _wn_conv(80, 512, 7, padding=3)
        self.ups = nn.ModuleList([
            weight_norm(ConvTranspose1d(cin, cout, k, k // 2, padding=k // 4))
            for _n, kind, cin, cout, k in GENERATOR_LAYERS if kind == "convT"])
        self.resblocks = nn.ModuleList([ResBlock(c, c) for c in (256, 128, 64, 32)])
        self.conv_post = _wn_conv(32, 1, 7, padding=3)
        self._dev = None          # engine.GeneratorDevice, created lazily on the parameters' device
        self._packed_key = None   # _PackKey of the parameters at the last pack

    # -- parameter plumbing -----------------------------------------------------------------
    def _param_triplets(self):
        mods = _layer_modules(self)
        return [m.weight_v for m in mods], [m.weight_g for m in mods], [m.bias for m in mods]

    def _ensure_packed(self):
        vs, gs, bs = self._param_triplets()
        dev = vs[0].device
        if dev.type != "cuda":
            raise _engine.EngineError(
                "melgan_multi_b200.Generator runs on CUDA (sm_90a) only; move the module with .to('cuda'). "
                "There is deliberately no CPU fallback.")
        with _PACK_LOCK:
            if self._dev is None or self._dev.device != dev:
                self._dev = _engine.GeneratorDevice(dev)
                self._packed_key = None
            self._pack_if_changed(self._dev, vs, gs, bs)
            return self._dev

    def _engine_forward(self, mel):
        return self._ensure_packed().forward(mel)

    def generate(self, x, lengths=None, precision="fp32", dtype=torch.float32):
        """Vocodes a batch in one forward (inference only: no autograd graph is built).  x [B, 80, T_max] fp32 CUDA.
        lengths None: every item has T_max frames.  Otherwise B mel lengths in [1, T_max] as a list, a tuple or a CPU integer
        tensor; the frames past each length are never read, and the audio [B, 1, 256 T_max] of item i starts with exactly
        the 256 lengths[i] samples of generate(x[i:i+1, :, :lengths[i]], precision=precision) and is 0 after them.
        precision "fp32" computes what self(x) computes; "bf16" runs one bf16 pass per tensor-core product (faster, audio
        about 1e-3 from float64 in relative L2: the contract is at mg_gen_forward_precision, include/melgan_b200.h).
        dtype torch.float32 returns audio in [-1, 1]; torch.int16 returns 16-bit PCM written by the last kernel, bit for bit
        pcm16 of the float audio: 0 for NaN, else clamp(rint(32768 a), -32768, 32767) (mg_gen_forward_pcm16)."""
        _engine._precision(precision)
        _engine._pcm16(dtype)
        if not x.is_cuda:
            raise _engine.EngineError("melgan_multi_b200.Generator.generate needs a CUDA tensor (no CPU fallback)")
        with torch.no_grad():
            return self._ensure_packed()._forward(x.detach().float(), lengths, None, None, None, precision, dtype)

    def stream(self, max_sessions=1, max_push_frames=32, precision="fp32", dtype=torch.float32):
        """A streaming vocoder over this generator's weights (inference only): up to max_sessions live mel streams, each
        step pushing at most max_push_frames new frames per session and returning the audio samples that became final
        (engine.GeneratorStream; the concatenation of a session's outputs equals generate() of its whole mel bit for bit).
        Weights changed between steps are re-packed at the next step, as in generate (after the writes the class
        docstring names, once repack() was called).  dtype: the format of every step's audio, as in
        generate (torch.int16: pcm16 of the float samples)."""
        _engine._pcm16(dtype)
        vs, _, _ = self._param_triplets()
        if vs[0].device.type != "cuda":
            raise _engine.EngineError("melgan_multi_b200.Generator.stream needs the module on CUDA (no CPU fallback)")
        self._ensure_packed()
        return _engine.GeneratorStream(self._ensure_packed, vs[0].device, max_sessions, max_push_frames, precision, dtype=dtype)

    def _graphed_recompute(self, mel, params):
        """(graphed stock-op forward+backward, mel_requires_grad) for this input shape, or None.  Cached per shape and per
        setting that picks the recompute's algorithms (cuDNN precision, benchmark and determinism, torch's deterministic
        mode: a graph replays the algorithms chosen at its capture); the graphs own static copies of nothing but
        activations and gradients -- parameters are call arguments."""
        import os
        if os.environ.get("MG_GEN_BWD_GRAPH", "1") == "0" or torch.cuda.is_current_stream_capturing():
            return None
        need_mel = bool(mel.requires_grad)
        key = (tuple(mel.shape), mel.device, need_mel, torch.backends.cudnn.conv.fp32_precision, torch.backends.cudnn.benchmark,
               torch.backends.cudnn.deterministic, torch.are_deterministic_algorithms_enabled())
        cache = self.__dict__.setdefault("_bwd_graphs", {})
        if key not in cache:
            if len(cache) >= 4:  # shapes keep changing (e.g. whole-utterance validation): stay eager for new ones
                return None
            sample = [mel.detach().clone().requires_grad_(need_mel)] + [p.detach().clone().requires_grad_(True) for p in params]
            try:
                with torch.enable_grad():  # (we are inside autograd.Function.forward, where grad mode is off)
                    fn = torch.cuda.make_graphed_callables(lambda m, *leaves: self._torch_forward(m, list(leaves)), tuple(sample))
            except Exception:  # capture refused (e.g. allocator / library state): the eager recompute still works
                fn = None
            cache[key] = fn
        return (cache[key], need_mel) if cache[key] is not None else None

    # -- stock-PyTorch restatement, used ONLY to differentiate (backward) ---------------------
    def _torch_forward(self, x, leaves):
        # (the same graph on channels_last 4-D tensors through conv2d saves cuDNN's nchw<->nhwc conversions --
        #  scripts/gen_bwd_layout_ab.py -- but picks TF32 kernels whose rounding puts the deepest
        #  layers' weight_g gradients AT the 5e-3 digest tolerance of tests/test_train_gpu.py on the small case: not taken)
        ws = [torch._weight_norm(leaves[3 * i], leaves[3 * i + 1], 0) for i in range(30)]
        bs = [leaves[3 * i + 2] for i in range(30)]
        x = F.conv1d(x, ws[0], bs[0], padding=3)
        for i in range(4):
            k = ws[1 + i].shape[2]
            x = F.conv_transpose1d(F.leaky_relu(x), ws[1 + i], bs[1 + i], stride=k // 2, padding=k // 4)
            for j, d in enumerate(_RES_DILATIONS):
                a, b = 5 + 6 * i + j, 5 + 6 * i + 3 + j
                h = F.conv1d(F.leaky_relu(x), ws[a], bs[a], padding=d, dilation=d)
                x = F.conv1d(F.leaky_relu(h), ws[b], bs[b], padding=1) + x
        return torch.tanh(F.conv1d(F.leaky_relu(x), ws[29], bs[29], padding=3))

    def forward(self, x):
        if not x.is_cuda:
            raise _engine.EngineError("melgan_multi_b200.Generator.forward needs a CUDA tensor (no CPU fallback)")
        if x.dtype != torch.float32:
            x = x.float()
        vs, gs, bs = self._param_triplets()
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in vs + gs + bs))
        if not needs_grad:
            return self._engine_forward(x)
        flat = []
        for v, g, b in zip(vs, gs, bs):
            flat += [v, g, b]
        return _GeneratorFunction.apply(self, x, *flat)


def generate_voices(generators, mel, voice, lengths=None, precision="fp32", dtype=torch.float32):
    """Vocodes a batch that mixes voices in one forward (inference only: no autograd graph is built).  generators: a
    sequence of Generator modules (a vocoder fine-tuned per speaker, say) on mel's CUDA device, each packed lazily as
    generate packs it.  mel [B, 80, T_max] fp32; voice: B ids in [0, len(generators)) as a list, a tuple or a CPU integer
    tensor; lengths as in Generator.generate (None: every item T_max frames).  Item i of the audio [B, 1, 256 T_max] is
    bit for bit generators[voice[i]].generate(mel[i:i+1, :, :lengths[i]], precision=precision), then 0.  Items need not be
    sorted by voice, but sorted ones run fastest.  dtype as in Generator.generate (torch.int16: 16-bit PCM)."""
    _engine._precision(precision)
    _engine._pcm16(dtype)
    if not mel.is_cuda:
        raise _engine.EngineError("melgan_multi_b200.generate_voices needs a CUDA tensor (no CPU fallback)")
    generators = list(generators)
    if not generators:
        raise _engine.EngineError("generate_voices needs at least one generator")
    with torch.no_grad():
        devs = []
        for g in generators:
            dev = g._ensure_packed()
            if dev.device != mel.device:
                raise _engine.EngineError("generate_voices: a generator is on %s, mel on %s" % (dev.device, mel.device))
            devs.append(dev)
        return devs[0].forward_voices(devs, mel.detach().float(), voice, lengths, precision=precision, dtype=dtype)


def stream_voices(generators, max_sessions=1, max_push_frames=32, precision="fp32", dtype=torch.float32):
    """A streaming vocoder whose live sessions run on several voices in one step (inference only): generators is a
    sequence of Generator modules on one CUDA device, each re-packed lazily at every step as Generator.stream does.  The
    returned engine.GeneratorStream's step(chunks, end=None, reset=None, voice=None) takes one voice id per slot (None:
    every slot on generators[0]); a slot keeps the voice its utterance was opened with until the utterance ends or the
    slot is reset.  The concatenation of a session's outputs equals generators[v].generate() of its whole mel bit for bit.
    dtype as in Generator.stream."""
    _engine._precision(precision)
    _engine._pcm16(dtype)
    generators = list(generators)
    if not generators:
        raise _engine.EngineError("stream_voices needs at least one generator")
    devices = set()
    for g in generators:
        vs, _, _ = g._param_triplets()
        if vs[0].device.type != "cuda":
            raise _engine.EngineError("melgan_multi_b200.stream_voices needs every generator on CUDA (no CPU fallback)")
        devices.add(vs[0].device)
    if len(devices) > 1:
        raise _engine.EngineError("stream_voices: the generators are on %s; they must share one device"
                                  % ", ".join(sorted(map(str, devices))))

    def packed():
        return [g._ensure_packed() for g in generators]
    packed()
    return _engine.GeneratorStream(packed, devices.pop(), max_sessions, max_push_frames, precision, dtype=dtype)


class Discriminator(_Repack, nn.Module):
    """One discriminator (reference models.py:74-103).  Inside ``MultiScaleDiscriminator`` (its only caller in the
    reference, models.py:109-113) the three of them run as one fused pipeline on the stacked real + generated batch;
    called on its own, ``forward(x)`` runs the same sm_90a kernels on this module's weights and returns
    ``(flattened logits, [7 feature maps])`` like the reference's.  CUDA only, no stock-op fallback.

    Called on its own it packs its own blob, apart from the enclosing MultiScaleDiscriminator's, and re-packs it as
    Generator does: a change of a parameter's _version or data_ptr is seen, whichever module it was made through;
    after an in-place write through p.data, a replayed CUDA graph or an AveragedModel EMA update call repack() (the
    enclosing module's repack() covers this one too, but this one's does not reach the enclosing module)."""

    def __init__(self):
        super().__init__()
        spec = {n: (cin, cout, k, s, g, p) for n, cin, cout, k, s, g, p in DISCRIMINATOR_LAYERS}
        def mk(n):
            cin, cout, k, s, g, p = spec[n]
            return weight_norm(Conv1d(cin, cout, k, s, groups=g, padding=p))
        self.conv_pre = mk("conv_pre")
        self.grouped_convs = nn.ModuleList([mk("grouped_convs.%d" % i) for i in range(4)])
        self.conv_post1 = mk("conv_post1")
        self.conv_post2 = mk("conv_post2")

    def layers(self):
        return [self.conv_pre] + list(self.grouped_convs) + [self.conv_post1, self.conv_post2]

    meanpools = ()   # what _MSDFunction walks for scale 0: no pooling

    def _param_triplets(self):
        mods = self.layers()
        return [m.weight_v for m in mods], [m.weight_g for m in mods], [m.bias for m in mods]

    def _engine_forward(self, x):
        vs, gs, bs = self._param_triplets()
        dev = vs[0].device
        with _PACK_LOCK:
            if getattr(self, "_dev", None) is None or self._dev.device != dev:
                self._dev = _engine.DiscriminatorDevice(dev, ndisc=1)
                self._packed_key = None
            self._pack_if_changed(self._dev, vs, gs, bs)
        return self._dev.forward(x)

    def forward(self, x):
        if not x.is_cuda:
            raise _engine.EngineError("melgan_multi_b200.Discriminator.forward needs a CUDA tensor (no CPU fallback)")
        x = x.float()
        vs, gs, bs = self._param_triplets()
        needs_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in vs + gs + bs))
        if needs_grad:
            flat = []
            for v, g, b in zip(vs, gs, bs):
                flat += [v, g, b]
            fmap = list(_MSDFunction.apply(self, 0, {}, x, *flat))
        else:
            fmap = self._engine_forward(x)[0]
        return torch.flatten(fmap[6], 1, -1), fmap


class _MSDFunction(torch.autograd.Function):
    """ONE discriminator of the stack as an autograd node: forward on the fused sm_90a kernels, backward layer by layer on
    the saved feature maps without recomputing the forward -- the grouped k41 convs (layers 1..4) and weight-norm on the
    hand-written kernels of csrc/mg_disc_bwd.cu (cuDNN launches one kernel per group for them), conv_post1 (88 % of the
    FLOPs) on the wgmma kernels of csrc/mg_conv_tc.cu (dgrad, transposed weight copy) and csrc/mg_wgrad_tc.cu (wgrad),
    conv_pre / conv_post2 on the bandwidth-bound kernels of csrc/mg_disc_edge_bwd.cu.  No aten / cuDNN call is left.

    The three scales of a MultiScaleDiscriminator are three nodes that share one forward: the first node to run launches the
    whole fused stack (real and generated stacked as one batch, the scales on forked streams) and parks the feature maps
    in ``cache``; the other two pick theirs up.  Separate nodes mean each discriminator's parameter gradients exist as soon
    as ITS backward is done, so the data-parallel wrapper (distributed.py) all-reduces them while the other scales'
    backward is still running.
    Inputs: scale index, cache dict, stacked audio [2B,1,L], then 7 x (weight_v, weight_g, bias) of that discriminator;
    outputs: its 7 feature maps."""

    @staticmethod
    def forward(ctx, host, s, cache, y2, *params):
        ctx.host, ctx.s = host, s
        if "fmaps" not in cache:
            cache["fmaps"] = host._engine_forward(y2)
        fm = tuple(cache["fmaps"][s])
        ctx.save_for_backward(y2, *params, *fm)
        return fm

    @staticmethod
    def backward(ctx, *grads):
        host, s, dev = ctx.host, ctx.s, ctx.host._dev
        saved = ctx.saved_tensors
        y2, params, fm = saved[0], saved[1:22], saved[22:]
        need_y = ctx.needs_input_grad[3]
        x0 = y2
        for k in range(s):  # the scale's input: the AvgPool chain of models.py:114-117,125-127
            x0 = host.meanpools[k](x0)
        # one host call walks the seven layers and enqueues every kernel (csrc/mg_disc_bwd_chain.cu): LeakyReLU', grouped convs,
        # conv_post1 dgrad / wgrad on wgmma, conv_pre / conv_post2 -- the step was bound by per-kernel Python launches
        g, dws, dbs = dev.scale_backward(s, x0, fm, grads, need_y)
        gy = None
        if need_y and g is not None:  # back through the (linear) AvgPool chain: differentiate it on zeros
            gy = g
            lens = [y2.shape[2], y2.shape[2] // 2 + 1]  # input lengths of pools 0, 1: AvgPool1d(4, 2, pad 2) gives L // 2 + 1
            for k in range(s - 1, -1, -1):
                with torch.enable_grad():
                    a = torch.zeros((y2.shape[0], 1, lens[k]), dtype=y2.dtype, device=y2.device).requires_grad_(True)
                    (gy,) = torch.autograd.grad(host.meanpools[k](a), a, gy)
        dvs, dgs = dev.wn_backward([params[3 * l] for l in range(7)], [params[3 * l + 1] for l in range(7)], dws)
        out = []
        for l in range(7):
            out += [dvs[l], dgs[l], dbs[l]]
        return (None, None, None, gy, *out)


class MultiScaleDiscriminator(_Repack, nn.Module):
    """Reference models.py:106-135: three Discriminators on y, pool(y), pool(pool(y)); returns
    (y_d_rs, y_d_gs, fmap_rs, fmap_gs).  On CUDA the whole stack runs in the hand-written kernels of
    libmelgan_b200.so with y and y_hat stacked into one batch (the reference calls each discriminator twice).

    The forward and its backward read weights packed at the first call and re-packed whenever a parameter's _version
    or data_ptr changed, as in Generator.  After an in-place write through p.data, a replayed CUDA graph or an
    AveragedModel EMA update call repack(), which also re-packs the three Discriminators for their stand-alone calls."""

    def __init__(self):
        super().__init__()
        self.discriminators = nn.ModuleList([Discriminator() for _ in range(3)])
        self.meanpools = nn.ModuleList([AvgPool1d(4, 2, padding=2), AvgPool1d(4, 4, padding=2)])
        self._dev = None
        self._packed_key = None

    def _param_triplets(self):
        mods = [m for d in self.discriminators for m in d.layers()]
        return [m.weight_v for m in mods], [m.weight_g for m in mods], [m.bias for m in mods]

    def _engine_forward(self, y2):
        vs, gs, bs = self._param_triplets()
        dev = vs[0].device
        with _PACK_LOCK:
            if self._dev is None or self._dev.device != dev:
                self._dev = _engine.DiscriminatorDevice(dev)
                self._packed_key = None
            self._pack_if_changed(self._dev, vs, gs, bs)
        return self._dev.forward(y2)

    # -- stock-PyTorch restatement on folded weights, used ONLY to differentiate (backward) -----------------
    def _torch_forward(self, y2, leaves):
        outs = []
        x_in = y2
        for s in range(3):
            if s > 0:
                x_in = self.meanpools[s - 1](x_in)
            x = x_in
            for l, (_n, _cin, _cout, _k, stride, groups, pad) in enumerate(DISCRIMINATOR_LAYERS):
                i = 3 * (7 * s + l)
                w = torch._weight_norm(leaves[i], leaves[i + 1], 0)
                x = F.conv1d(x, w, leaves[i + 2], stride=stride, padding=pad, groups=groups)
                if l < 6:
                    x = F.leaky_relu(x)
                outs.append(x)
        return outs

    def forward(self, y, y_hat):
        if not (y.is_cuda and y_hat.is_cuda):
            raise _engine.EngineError(
                "melgan_multi_b200.MultiScaleDiscriminator.forward needs CUDA tensors (no CPU fallback)")
        B = y.shape[0]
        y2 = torch.cat([y, y_hat], dim=0).float()
        vs, gs, bs = self._param_triplets()
        needs_grad = torch.is_grad_enabled() and (y2.requires_grad or any(p.requires_grad for p in vs + gs + bs))
        if needs_grad:
            cache, fmaps = {}, []
            for s in range(3):  # three autograd nodes, one fused forward launch (see _MSDFunction)
                flat = []
                for i in range(7 * s, 7 * s + 7):
                    flat += [vs[i], gs[i], bs[i]]
                fmaps.append(list(_MSDFunction.apply(self, s, cache, y2, *flat)))
        else:
            fmaps = self._engine_forward(y2)
        # The reference's four lists.  Every element is an ordinary autograd slice of the stacked map (any use of it
        # differentiates correctly), and is also tagged with the stacked tensor it is a half of: the package's own loss
        # functions then work on the stacked tensors directly -- one gradient tensor per map instead of two zero-padded
        # slice gradients and their sum (SliceBackward + add_: ~1000 launches per training step).
        def half(f, h, flat=False):
            t = f[h * B:(h + 1) * B]
            if flat:
                t = torch.flatten(t, 1, -1)
            t._mg_half = (f, h)
            return t
        y_d_rs, y_d_gs, fmap_rs, fmap_gs = [], [], [], []
        for s in range(3):
            fmap_rs.append([half(f, 0) for f in fmaps[s]])
            fmap_gs.append([half(f, 1) for f in fmaps[s]])
            y_d_rs.append(half(fmaps[s][6], 0, True))
            y_d_gs.append(half(fmaps[s][6], 1, True))
        return y_d_rs, y_d_gs, fmap_rs, fmap_gs


class _LossRows(torch.autograd.Function):
    """Row means of a loss table on the fused kernels (csrc/mg_loss.cu): forward = one reduction launch over every row +
    a fixed-order combine, backward = one launch writing every input gradient.  Inputs: rows of (a, b) CUDA tensors
    (b ignored unless the row is an L1 pair)."""

    @staticmethod
    def forward(ctx, modes, *tensors):
        k = len(modes)
        a, b = list(tensors[:k]), list(tensors[k:])
        ctx.modes, ctx.k = modes, k
        ctx.save_for_backward(*[t.detach() for t in tensors])
        return _engine.loss_forward(a, b, list(modes))

    @staticmethod
    def backward(ctx, grad_out):
        k, modes = ctx.k, ctx.modes
        saved = ctx.saved_tensors
        a, b = list(saved[:k]), list(saved[k:])
        need_b = [ctx.needs_input_grad[1 + k + i] and modes[i] == _engine.LOSS_L1 for i in range(k)]
        ga, gb = _engine.loss_backward(a, b, list(modes), grad_out, need_b)
        ga = [g if ctx.needs_input_grad[1 + i] else None for i, g in enumerate(ga)]
        return (None, *[g.view_as(t) if g is not None else None for g, t in zip(ga, a)],
                *[g.view_as(t) if g is not None else None for g, t in zip(gb, b)])


class _StackedLossRows(torch.autograd.Function):
    """The same row means, for rows that are halves (real / generated) of stacked discriminator outputs: forward reads the
    halves in place, backward writes each row's gradient straight into its half of ONE gradient tensor per stacked map.
    rows: tuple of (parent index, half of a, half of b or None, mode)."""

    @staticmethod
    def forward(ctx, rows, *parents):
        ctx.rows = rows
        ctx.save_for_backward(*parents)
        a, b = _StackedLossRows._views(rows, [p.detach() for p in parents])
        return _engine.loss_forward(a, [u if u is not None else t for t, u in zip(a, b)], [r[3] for r in rows])

    @staticmethod
    def _views(rows, tensors):
        a, b = [], []
        for pi, ha, hb, _mode in rows:
            t = tensors[pi]
            n = t.shape[0] // 2
            a.append(t[ha * n:(ha + 1) * n])
            b.append(t[hb * n:(hb + 1) * n] if hb is not None else None)
        return a, b

    @staticmethod
    def backward(ctx, grad_out):
        rows, parents = ctx.rows, ctx.saved_tensors
        covered = [set() for _ in parents]
        for pi, ha, hb, _mode in rows:
            covered[pi].add(ha)
            if hb is not None:
                covered[pi].add(hb)
        grads = [(torch.empty_like(p) if len(c) == 2 else torch.zeros_like(p)) if ctx.needs_input_grad[1 + i] else None
                 for i, (p, c) in enumerate(zip(parents, covered))]
        scratch = [g if g is not None else torch.empty_like(p) for g, p in zip(grads, parents)]
        a, b = _StackedLossRows._views(rows, [p.detach() for p in parents])
        ga, gb = _StackedLossRows._views(rows, scratch)
        modes = [r[3] for r in rows]
        _engine.loss_backward(a, [u if u is not None else t for t, u in zip(a, b)], modes, grad_out,
                              [u is not None for u in b], out_a=ga, out_b=gb)
        return (None, *grads)


def _stacked_rows(a, b, modes):
    """If every row is a tagged half of a stacked discriminator output (MultiScaleDiscriminator.forward), the table in
    (parent index, halves, mode) form plus the distinct parents; else None."""
    parents, index, rows = [], {}, []
    for t, u, m in zip(a, b, modes):
        ti = getattr(t, "_mg_half", None)
        ui = getattr(u, "_mg_half", None) if u is not None else None
        if ti is None or (u is not None and (ui is None or ui[0] is not ti[0])) or not ti[0].requires_grad:
            return None
        if id(ti[0]) not in index:
            index[id(ti[0])] = len(parents)
            parents.append(ti[0])
        rows.append((index[id(ti[0])], ti[1], ui[1] if ui is not None else None, m))
    return tuple(rows), parents


def _row_means(a, b, modes):
    """Row means of a loss table on the fused kernels.  CUDA tensors only, like the modules: there is no CPU path."""
    if not all(t.is_cuda for t in a):
        raise _engine.EngineError("melgan_multi_b200 loss functions need CUDA tensors (no CPU fallback)")
    st = _stacked_rows(a, b, modes) if torch.is_grad_enabled() else None
    if st is not None:
        return _StackedLossRows.apply(st[0], *st[1])
    b = [u if u is not None else t for t, u in zip(a, b)]  # placeholder rows keep the argument list rectangular
    return _LossRows.apply(tuple(modes), *a, *b)


def feature_loss(fmap_r, fmap_g):
    """10 * sum over the 21 feature-map pairs of mean |r - g| (reference models.py:138-144)."""
    rs = [r for maps in fmap_r for r in maps]
    gs = [g for maps in fmap_g for g in maps]
    return _row_means(rs, gs, [_engine.LOSS_L1] * len(rs)).sum() * 10


def discriminator_loss(disc_real_outputs, disc_generated_outputs):
    """LSGAN discriminator loss; returns (loss, real terms, generated terms) like models.py:147-159 (the two lists are
    Python floats, as in the reference -- read back with ONE host sync instead of six)."""
    k = len(disc_real_outputs)
    rows = list(disc_real_outputs) + list(disc_generated_outputs)
    means = _row_means(rows, [None] * (2 * k), [_engine.LOSS_ONE_MINUS_SQ] * k + [_engine.LOSS_SQ] * k)
    vals = means.detach().tolist()
    # the read-back above synchronised the stream: every forward enqueued before it has finished, so its pipeline status
    # word (engine._StatusWatch) can be inspected here at no cost -- a stalled tensor-core pipeline raises instead of training on
    _engine.poll_status()
    return means.sum(), vals[:k], vals[k:]


def generator_loss(disc_generated_outputs):
    """LSGAN generator loss (reference models.py:162-167)."""
    rows = list(disc_generated_outputs)
    return _row_means(rows, [None] * len(rows), [_engine.LOSS_ONE_MINUS_SQ] * len(rows)).sum()
