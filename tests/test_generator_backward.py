"""CPU: who owns the gradients that models._GeneratorFunction returns, and what keys the generator's recompute graphs.

The generator's backward replays a CUDA graph (torch.cuda.make_graphed_callables) whose backward hands out detached
aliases of the graph's static gradient buffers; the next replay of the same graph overwrites them.  A stand-in generator
reproduces that on the CPU: its graphed recompute is an autograd Function whose backward writes every gradient into one
persistent buffer per input and returns buffer.detach(), as Graphed.backward does.  Gradient accumulation, two calls in
one loss, zero_grad(set_to_none=False) and a gradient kept across a later backward must all see their own values,
bit for bit."""

import pytest
import torch

from melgan_multi_b200 import models


class _StandInGenerator:
    """What _GeneratorFunction calls on a Generator: y = tanh(w * mel) + b on [B, C, T], forward and recompute on the CPU."""

    def __init__(self):
        self.static = None     # the graph's gradient buffers: one per input, reused by every backward
        self.replays = 0

    def _engine_forward(self, mel):
        return self._torch_forward(mel, list(self.params)).detach()

    @staticmethod
    def _torch_forward(mel, leaves):
        w, b = leaves
        return torch.tanh(w * mel) + b

    def _graphed_recompute(self, mel, params):
        owner, need_mel = self, bool(mel.requires_grad)

        class Graphed(torch.autograd.Function):
            @staticmethod
            def forward(ctx, m, *leaves):
                ctx.save_for_backward(m, *leaves)
                return owner._torch_forward(m, list(leaves))

            @staticmethod
            def backward(ctx, gy):
                m, *leaves = ctx.saved_tensors
                with torch.enable_grad():
                    ins = [m.detach().requires_grad_(need_mel)] + [t.detach().requires_grad_(True) for t in leaves]
                    y = owner._torch_forward(ins[0], ins[1:])
                    grads = torch.autograd.grad(y, ins if need_mel else ins[1:], gy)
                grads = ([] if need_mel else [None]) + list(grads)
                if owner.static is None:
                    owner.static = [torch.empty_like(g) if g is not None else None for g in grads]
                for s, g in zip(owner.static, grads):
                    if s is not None:
                        s.copy_(g)
                owner.replays += 1
                return tuple(s.detach() if s is not None else None for s in owner.static)

        return Graphed.apply, need_mel


C, T = 4, 6


def _setup(seed=0):
    gen = _StandInGenerator()
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(1, C, 1, generator=g).requires_grad_(True)
    b = torch.randn(1, C, 1, generator=g).requires_grad_(True)
    gen.params = (w, b)
    return gen, w, b, g


def _call(gen, mel):
    return models._GeneratorFunction.apply(gen, mel, *gen.params)


def _data(g, B=2):
    return torch.randn(B, C, T, generator=g), torch.randn(B, C, T, generator=g)


def _separate(gen, mel, r):
    """(d/dw, d/db, d/dmel) of sum(r * y) through the plain autograd graph."""
    m = mel.detach().requires_grad_(True)
    y = gen._torch_forward(m, list(gen.params))
    return torch.autograd.grad((r * y).sum(), list(gen.params) + [m])


def test_two_calls_in_one_loss_get_the_sum_of_their_gradients():
    gen, w, b, g = _setup()
    (x1, r1), (x2, r2) = _data(g), _data(g)
    e1, e2 = _separate(gen, x1, r1), _separate(gen, x2, r2)
    x1, x2 = x1.requires_grad_(True), x2.requires_grad_(True)
    ((r1 * _call(gen, x1)).sum() + (r2 * _call(gen, x2)).sum()).backward()
    assert gen.replays == 2
    assert torch.equal(w.grad, e1[0] + e2[0]) and torch.equal(b.grad, e1[1] + e2[1])
    assert torch.equal(x1.grad, e1[2]) and torch.equal(x2.grad, e2[2])


def test_gradients_accumulate_over_backward_calls():
    gen, w, b, g = _setup(1)
    (x1, r1), (x2, r2) = _data(g), _data(g)
    e1, e2 = _separate(gen, x1, r1), _separate(gen, x2, r2)
    (r1 * _call(gen, x1)).sum().backward()
    (r2 * _call(gen, x2)).sum().backward()
    assert torch.equal(w.grad, e1[0] + e2[0]) and torch.equal(b.grad, e1[1] + e2[1])


def test_zeroed_gradients_are_not_doubled_by_the_next_step():
    gen, w, b, g = _setup(2)
    x, r = _data(g)
    e = _separate(gen, x, r)
    opt = torch.optim.SGD([w, b], lr=0.0)
    for _ in range(2):
        opt.zero_grad(set_to_none=False)
        (r * _call(gen, x)).sum().backward()
        assert torch.equal(w.grad, e[0]) and torch.equal(b.grad, e[1])


def test_returned_gradients_survive_a_later_backward():
    gen, w, b, g = _setup(3)
    (xa, ra), (xb, rb) = _data(g), _data(g)
    xa = xa.requires_grad_(True)
    (ra * _call(gen, xa)).sum().backward()
    held = [w.grad, b.grad, xa.grad]
    kept = [t.clone() for t in held]
    w.grad, b.grad = None, None  # zero_grad(): the caller still holds the old tensors
    (rb * _call(gen, xb.requires_grad_(True))).sum().backward()
    assert gen.replays == 2
    for h, k in zip(held, kept):
        assert torch.equal(h, k)
    assert not any(h.data_ptr() == s.data_ptr() for h in held for s in gen.static if s is not None)


def test_eager_recompute_gives_the_same_gradients():
    """No graph for this call (MG_GEN_BWD_GRAPH=0, a fifth shape, a call during capture): the eager recompute runs."""
    gen, w, b, g = _setup(4)
    x, r = _data(g)
    e = _separate(gen, x, r)
    gen._graphed_recompute = lambda mel, params: None
    (r * _call(gen, x.requires_grad_(True))).sum().backward()
    assert torch.equal(w.grad, e[0]) and torch.equal(b.grad, e[1]) and torch.equal(x.grad, e[2])


@pytest.fixture()
def stub_capture(monkeypatch):
    """Generator._graphed_recompute on the CPU: make_graphed_callables is replaced by a stub that counts captures."""
    captures = []

    def make_graphed_callables(fn, sample):
        captures.append(sample)
        return fn
    monkeypatch.setattr(torch.cuda, "make_graphed_callables", make_graphed_callables)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.delenv("MG_GEN_BWD_GRAPH", raising=False)
    return captures


def _params():
    gen = models.Generator()
    vs, gs, bs = gen._param_triplets()
    return gen, [t for trip in zip(vs, gs, bs) for t in trip]


def test_recompute_graphs_are_keyed_by_every_algorithm_setting(stub_capture):
    """A graph replays the algorithms chosen when it was captured: turning on cuDNN determinism or torch's deterministic
    mode after a capture must capture a new graph, as must a change of cuDNN precision or of mel's requires_grad."""
    gen, params = _params()
    mel = torch.zeros(1, 80, 3)
    old = (torch.backends.cudnn.deterministic, torch.are_deterministic_algorithms_enabled(),
           torch.is_deterministic_algorithms_warn_only_enabled(), torch.backends.cudnn.conv.fp32_precision)
    try:
        torch.backends.cudnn.deterministic = False
        torch.use_deterministic_algorithms(False)
        assert gen._graphed_recompute(mel, params) is not None and len(gen._bwd_graphs) == 1
        assert gen._graphed_recompute(mel, params) is not None and len(gen._bwd_graphs) == 1  # cached
        torch.backends.cudnn.deterministic = True
        assert gen._graphed_recompute(mel, params) is not None and len(gen._bwd_graphs) == 2
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert gen._graphed_recompute(mel, params) is not None and len(gen._bwd_graphs) == 3
        torch.backends.cudnn.conv.fp32_precision = "ieee" if old[3] != "ieee" else "tf32"
        assert gen._graphed_recompute(mel, params) is not None and len(gen._bwd_graphs) == 4
        gen._bwd_graphs.clear()
        mel.requires_grad_(True)
        fn, need_mel = gen._graphed_recompute(mel, params)
        assert need_mel and len(gen._bwd_graphs) == 1 and len(stub_capture) == 5
    finally:
        torch.backends.cudnn.deterministic = old[0]
        torch.use_deterministic_algorithms(old[1], warn_only=old[2])
        torch.backends.cudnn.conv.fp32_precision = old[3]


def test_recompute_graphs_stop_at_four_keys_and_honour_the_switch(stub_capture, monkeypatch):
    gen, params = _params()
    for T in range(1, 5):
        assert gen._graphed_recompute(torch.zeros(1, 80, T), params) is not None
    assert gen._graphed_recompute(torch.zeros(1, 80, 5), params) is None  # a fifth key runs eager
    assert gen._graphed_recompute(torch.zeros(1, 80, 2), params) is not None  # known keys still replay
    monkeypatch.setenv("MG_GEN_BWD_GRAPH", "0")
    assert gen._graphed_recompute(torch.zeros(1, 80, 2), params) is None
    assert len(gen._bwd_graphs) == 4 and len(stub_capture) == 4


def test_owned_copies_are_exact_and_share_no_storage():
    src = [torch.randn(3, 4, 5), None, torch.randn(7), torch.randn(2, 1)]
    out = models._owned_copies(src)
    assert out[1] is None
    for s, o in zip(src, out):
        if s is not None:
            assert torch.equal(s, o) and o.shape == s.shape and o.untyped_storage().data_ptr() != s.untyped_storage().data_ptr()
    assert models._owned_copies([None, None]) == [None, None]
