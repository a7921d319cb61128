"""GPU: the generator's gradients -- every element of all 90 parameter gradients and of the mel gradient -- against
float64 autograd of the reference graph (reference models.py:61-71 plus the 30 weight-norm pre-forward hooks, written out
below), on both recompute paths of models._GeneratorFunction: the CUDA-graph replay (one pair of graphs per cache key,
Generator._bwd_graphs) and the eager stock-op recompute (MG_GEN_BWD_GRAPH=0, a fifth key).

The loss is linear, L = sum(R * y) with a seeded R, so the upstream gradient is exactly R whatever the native forward's
~1e-5 error, and each LeakyReLU takes the branch an fp32 forward takes (see reference()): the comparison measures the
recompute's arithmetic alone.  One mean-square loss checks the plumbing of a
y-dependent upstream with its own looser bound.  Each tensor is held to TAU = (max|d| / max|g64|, ||d|| / ||g64||),
calibrated under cuDNN "ieee" (strict fp32) and printed as the worst ratio to the bound; three mutants of the float64
reference (a ResBlock dilation swapped, conv_post's bias gradient dropped, one ConvTranspose's padding off by one) must
exceed it by at least kernel_model.MUTANT_X.

The ownership tests are exact: under cuDNN determinism a gradient returned by the graphed backward must equal, bit for
bit, the same gradient computed on its own, however calls and backward() calls are combined."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_errors
from melgan_multi_b200 import models, synth
from kernel_model import MUTANT_X

pytestmark = pytest.mark.gpu

# (max-rel, l2-rel) per tensor, worst measured over this file on an H100 80GB HBM3 at 700 W.  ieee (strict fp32 convs):
# 2.4e-5 / 1.8e-5, fp32 rounding of the long wgrad / bias reductions (up to B * 256 T positions).  tf32 (10-bit operand
# mantissas): 1.6e-3 / 1.4e-3.  Mean-square loss: 3.7e-6 / 2.6e-6; its upstream 2 (y - target) / N also carries the native
# forward's error (~1e-5 of max|y|), hence the looser bound.
TAU_IEEE = (1e-4, 5e-5)
TAU_TF32 = (5e-3, 5e-3)
TAU_MSE = (5e-4, 5e-4)
SHAPES = [(1, 1), (1, 7), (3, 33), (16, 32), (1, 200)]
DIL = (1, 3, 9)


@pytest.fixture(autouse=True)
def ieee_deterministic():
    old = (torch.backends.cudnn.conv.fp32_precision, torch.backends.cudnn.deterministic)
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.conv.fp32_precision, torch.backends.cudnn.deterministic = old


def fresh(seed=1234):
    """A new module each time: a shared one would carry its recompute graphs from test to test."""
    gen = models.Generator()
    gen.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
    return gen.cuda().train()


def params(gen):
    """The 90 parameters as 30 x (weight_v, weight_g, bias), the order of _GeneratorFunction's inputs."""
    vs, gs, bs = gen._param_triplets()
    return [t for trip in zip(vs, gs, bs) for t in trip]


def inputs(B, T, seed):
    mel = torch.from_numpy(synth.mel_input(B, T, seed)).cuda()
    g = torch.Generator().manual_seed(seed + 77)
    return mel, torch.randn(B, 1, 256 * T, generator=g).cuda()


def generator_graph(mel, ws, bs, lrelu, dil=(DIL,) * 4, up_pad=(0, 0, 0, 0)):
    """The reference's Generator.forward on folded weights, with LeakyReLU passed in; dil and up_pad select mutants."""
    x = F.conv1d(mel, ws[0], bs[0], padding=3)
    for i in range(4):
        k = ws[1 + i].shape[2]
        x = F.conv_transpose1d(lrelu(x), ws[1 + i], bs[1 + i], stride=k // 2, padding=k // 4 + up_pad[i],
                               output_padding=2 * up_pad[i])
        for j, d in enumerate(dil[i]):
            a, b = 5 + 6 * i + j, 5 + 6 * i + 3 + j
            h = F.conv1d(lrelu(x), ws[a], bs[a], padding=d, dilation=d)
            x = F.conv1d(lrelu(h), ws[b], bs[b], padding=1) + x
    return torch.tanh(F.conv1d(lrelu(x), ws[29], bs[29], padding=3))


def reference(gen, mel, R, loss="linear", post_bias=True, **mutant):
    """float64 gradients of the loss w.r.t. the module's current parameters (90 tensors), then mel.

    Every product, sum and the weight-norm fold (from the module's own weight_v / weight_g) run in float64.  Only the
    branch each LeakyReLU takes comes from an fp32 forward of the same stock ops under the current cuDNN settings, as the
    recompute's own forward decides it: an input within fp32 rounding of zero may fall on either side, and where the
    float64 forward disagrees the derivative jumps by 0.99 of the upstream gradient -- a handful of such positions moves
    a bias or weight_g gradient by up to 3e-2 of its maximum, which says nothing about the backward's arithmetic."""
    ps = [p.detach() for p in params(gen)]
    branches = []

    def record(x):
        branches.append(x > 0)
        return F.leaky_relu(x)
    with torch.no_grad():
        generator_graph(mel, [torch._weight_norm(ps[3 * i], ps[3 * i + 1], 0) for i in range(30)], ps[2::3], record, **mutant)
    taken = iter(branches)

    def lrelu(x):
        return torch.where(next(taken), x, 0.01 * x)
    leaves = [p.double().requires_grad_(True) for p in ps]
    m = mel.detach().double().requires_grad_(True)
    ws = [g * v / (v * v).sum((1, 2), keepdim=True).sqrt() for v, g in zip(leaves[0::3], leaves[1::3])]
    bs = leaves[2::3]
    if not post_bias:
        bs = bs[:29] + [bs[29].detach()]
    y = generator_graph(m, ws, bs, lrelu, **mutant)
    L = (R.double() * y).sum() if loss == "linear" else ((y - R.double()) ** 2).mean()
    return [g if g is not None else torch.zeros_like(t)
            for g, t in zip(torch.autograd.grad(L, leaves + [m], allow_unused=True), leaves + [m])]


def run(gen, mel, R, need_mel=True, loss="linear"):
    """One forward + backward through the module: the 90 parameter gradients, then mel's (or None)."""
    gen.zero_grad()
    x = mel.detach().clone().requires_grad_(need_mel)
    y = gen(x)
    ((R * y).sum() if loss == "linear" else ((y - R) ** 2).mean()).backward()
    return [p.grad for p in params(gen)] + [x.grad]


def worst(got, ref, tau):
    """(largest ratio to the bound over the tensors, its tensor index, worst max-rel, worst l2-rel); None in got: skipped."""
    out, wm, wl = (0.0, None), 0.0, 0.0
    for i, (a, r) in enumerate(zip(got, ref)):
        if a is None:
            continue
        m, l2 = rel_errors(a.detach().cpu().numpy(), r.detach().cpu().numpy())
        out = max(out, (max(m / tau[0], l2 / tau[1]), i), key=lambda t: t[0])
        wm, wl = max(wm, m), max(wl, l2)
    return out + (wm, wl)


def check(got, ref, tau, what):
    ratio, i, m, l2 = worst(got, ref, tau)
    print("%s: worst ratio to the bound %.3f (tensor %s); worst max-rel %.2e, l2-rel %.2e" % (what, ratio, i, m, l2))
    assert ratio <= 1.0, (what, i, ratio)
    return ratio


def clones(grads):
    return [g.clone() if g is not None else None for g in grads]


def identical(a, b):
    return [i for i, (x, y) in enumerate(zip(a, b)) if (x is None) != (y is None) or (x is not None and not torch.equal(x, y))]


@pytest.mark.parametrize("B,T", SHAPES)
def test_gradients_meet_float64_on_the_graphed_and_the_eager_path(B, T, monkeypatch):
    """Graphed (a capture on this module's first call at this shape) against float64, then the same inputs eager
    (MG_GEN_BWD_GRAPH=0, read at each forward): bit-identical under cudnn.deterministic."""
    monkeypatch.delenv("MG_GEN_BWD_GRAPH", raising=False)
    gen = fresh()
    mel, R = inputs(B, T, 10 + T)
    graphed = clones(run(gen, mel, R))
    assert len(gen._bwd_graphs) == 1 and all(v is not None for v in gen._bwd_graphs.values())
    check(graphed, reference(gen, mel, R), TAU_IEEE, "graphed B=%d T=%d" % (B, T))
    monkeypatch.setenv("MG_GEN_BWD_GRAPH", "0")
    eager = run(gen, mel, R)
    assert len(gen._bwd_graphs) == 1
    assert not identical(graphed, eager), identical(graphed, eager)


def test_fifth_shape_runs_eager_and_every_shape_meets_float64(monkeypatch):
    monkeypatch.delenv("MG_GEN_BWD_GRAPH", raising=False)
    gen = fresh()
    for n, (B, T) in enumerate(SHAPES):
        mel, R = inputs(B, T, 20 + n)
        got = run(gen, mel, R)
        graphs = gen._bwd_graphs
        if n < 4:
            assert len(graphs) == n + 1 and all(v is not None for v in graphs.values())
        else:
            assert len(graphs) == 4 and all(k[0] != (B, 80, T) for k in graphs)
        check(got, reference(gen, mel, R), TAU_IEEE, "shape %d of 5, B=%d T=%d" % (n + 1, B, T))


def test_bound_rejects_mutants_of_the_reference():
    gen = fresh()
    mel, R = inputs(3, 33, 5)
    ref = reference(gen, mel, R)
    check(run(gen, mel, R), ref, TAU_IEEE, "B=3 T=33")
    for name, mutant in (("dilation swapped in ResBlock 2", dict(dil=(DIL, DIL, (1, 9, 3), DIL))),
                         ("conv_post bias gradient dropped", dict(post_bias=False)),
                         ("ups.1 padding off by one", dict(up_pad=(0, 1, 0, 0)))):
        ratio, i, _, _ = worst(reference(gen, mel, R, **mutant), ref, TAU_IEEE)
        print("mutant %s: %.1f x the bound (tensor %s)" % (name, ratio, i))
        assert ratio >= MUTANT_X, (name, ratio)


def test_mean_square_loss_meets_its_bound():
    gen = fresh()
    mel, target = inputs(3, 33, 6)
    target = 0.5 * target
    check(run(gen, mel, target, loss="mse"), reference(gen, mel, target, loss="mse"), TAU_MSE, "mean-square loss")


def test_precision_switch_captures_a_new_graph():
    """Default tf32 convs against their own bound; switching the module to ieee captures a second graph that meets the
    ieee bound (a graph captured under tf32 and replayed would not)."""
    gen = fresh()
    mel, R = inputs(3, 33, 7)
    torch.backends.cudnn.conv.fp32_precision = "tf32"
    tf32 = clones(run(gen, mel, R))
    assert len(gen._bwd_graphs) == 1
    check(tf32, reference(gen, mel, R), TAU_TF32, "tf32")
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    ref = reference(gen, mel, R)
    ieee = run(gen, mel, R)
    assert len(gen._bwd_graphs) == 2
    check(ieee, ref, TAU_IEEE, "ieee after tf32")
    assert worst(tf32, ref, TAU_IEEE)[0] > MUTANT_X  # tf32 was in effect: its gradients are far outside the ieee bound


def test_determinism_settings_capture_new_graphs():
    gen = fresh()
    mel, R = inputs(1, 7, 8)
    ref = reference(gen, mel, R)
    old = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    try:
        torch.backends.cudnn.deterministic = False
        check(run(gen, mel, R), ref, TAU_IEEE, "cudnn.deterministic off")
        assert len(gen._bwd_graphs) == 1
        torch.backends.cudnn.deterministic = True
        check(run(gen, mel, R), ref, TAU_IEEE, "cudnn.deterministic on")
        assert len(gen._bwd_graphs) == 2
        torch.use_deterministic_algorithms(True, warn_only=True)
        check(run(gen, mel, R), ref, TAU_IEEE, "deterministic algorithms")
        assert len(gen._bwd_graphs) == 3
    finally:
        torch.use_deterministic_algorithms(old[0], warn_only=old[1])


@pytest.mark.parametrize("first", [False, True])
def test_mel_gradient_on_and_off(first):
    """need_mel is part of the graph key: alternating mel.requires_grad on one module and shape keeps both graphs right."""
    gen = fresh()
    mel, R = inputs(2, 8, 9)
    ref = reference(gen, mel, R)
    for k in range(4):
        need = first if k % 2 == 0 else not first
        got = run(gen, mel, R, need_mel=need)
        assert (got[90] is not None) == need
        check(got, ref, TAU_IEEE, "call %d, mel.requires_grad=%s" % (k, need))
    assert sorted(k[2] for k in gen._bwd_graphs) == [False, True]


# -- ownership of the returned gradients: exact -------------------------------------------------------------------------

def test_two_calls_in_one_loss_get_the_sum_of_their_gradients():
    gen = fresh()
    (m1, r1), (m2, r2) = inputs(2, 8, 1), inputs(2, 8, 2)
    g1, g2 = clones(run(gen, m1, r1)), clones(run(gen, m2, r2))
    gen.zero_grad()
    x1, x2 = m1.clone().requires_grad_(True), m2.clone().requires_grad_(True)
    ((r1 * gen(x1)).sum() + (r2 * gen(x2)).sum()).backward()
    want = [a + b for a, b in zip(g1[:90], g2[:90])]
    bad = identical([p.grad for p in params(gen)] + [x1.grad, x2.grad], want + [g1[90], g2[90]])
    assert not bad, bad


def test_gradients_accumulate_over_backward_calls():
    gen = fresh()
    (m1, r1), (m2, r2) = inputs(2, 8, 1), inputs(2, 8, 2)
    g1, g2 = clones(run(gen, m1, r1)), clones(run(gen, m2, r2))
    gen.zero_grad()
    (r1 * gen(m1)).sum().backward()
    (r2 * gen(m2)).sum().backward()
    bad = identical([p.grad for p in params(gen)], [a + b for a, b in zip(g1[:90], g2[:90])])
    assert not bad, bad


def test_zero_grad_without_none_does_not_double_the_next_step():
    gen = fresh()
    mel, R = inputs(2, 8, 3)
    opt = torch.optim.Adam(gen.parameters(), 1e-3)
    steps = []
    for _ in range(2):
        opt.zero_grad(set_to_none=False)
        (R * gen(mel)).sum().backward()
        steps.append(clones([p.grad for p in params(gen)]))
    bad = identical(steps[0], steps[1])
    assert not bad, bad


def test_held_gradients_survive_a_later_backward():
    gen = fresh()
    (ma, ra), (mb, rb) = inputs(2, 8, 4), inputs(2, 8, 5)
    held = run(gen, ma, ra)
    kept = clones(held)
    run(gen, mb, rb)
    bad = identical(held, kept)
    assert not bad, bad


def test_frozen_layers_get_no_gradient_and_the_rest_meet_float64():
    gen = fresh()
    gen.conv_pre.requires_grad_(False)
    gen.ups[0].requires_grad_(False)
    frozen = {id(p) for p in list(gen.conv_pre.parameters()) + list(gen.ups[0].parameters())}
    mel, R = inputs(2, 8, 6)
    got = run(gen, mel, R)
    assert all((g is None) == (id(p) in frozen) for p, g in zip(params(gen), got))
    assert sum(g is None for g in got[:90]) == 6
    check(got, reference(gen, mel, R), TAU_IEEE, "conv_pre and ups.0 frozen")


@pytest.mark.parametrize("optimizer", ["torch", "multi_tensor"])
def test_gradient_after_an_optimizer_step_is_at_the_new_weights(optimizer):
    from melgan_multi_b200 import optim
    gen = fresh()
    mel, R = inputs(2, 8, 7)
    opt = (torch.optim.Adam if optimizer == "torch" else optim.Adam)(gen.parameters(), 1e-2, betas=(0.5, 0.9))
    before = reference(gen, mel, R)
    check(run(gen, mel, R), before, TAU_IEEE, "before the step")
    opt.step()
    opt.zero_grad()
    after = reference(gen, mel, R)
    assert worst(before, after, TAU_IEEE)[0] > MUTANT_X  # the step moved the gradient far beyond the bound
    check(run(gen, mel, R), after, TAU_IEEE, "after one %s Adam step" % optimizer)
