"""The training-side kernels -- the fused losses (csrc/mg_loss.cu) and the multi-tensor Adam (csrc/mg_optim.cu) -- against
float64 statements of their own arithmetic, at training size and at every chunk border.

Losses.  A row mean is held to |got - ref| <= TAU_L * mean|term| + 2^-24 |ref|, ref the float64 mean of the same fp32
inputs.  TAU_L = 2^-21 follows from the kernel's structure: each element's path is 64 fp32 additions in its thread, then 5
warp and 3 block tree levels, then a float64 combine -- 72 roundings of at most u/2 of a partial sum, with random signs
about sqrt(72) u / 2 = 4.2 u, doubled (the worst case, all of them one way, would be (64 + 8 + 2) u).  The gradients are
exact up to a few roundings: an L1 gradient has the sign of a - b (0 where a == b) and a magnitude within 2^-22 of
float64 autograd; an LSGAN row writes only its half of the stacked gradient and the other half is exactly 0.
test_loss_tau_calibration_on_emulated_reduction checks both sides of TAU_L on the CPU (the emulation: <= 0.13 of the
bound; the last chunk dropped, bf16 partial sums or fp16 per-thread sums: >= 14x).

Adam.  Each step is checked on the kernel's own previous state (so errors do not compound), element-wise:
    |m - m64| <= 8u Ma,   |v - v64| <= 12u Va,   |p - p64| <= 4u |p64| + 8u step (Ma / den64) (1 + Va / v64)
with u = 2^-24, Ma = |b1 m| + (1 - b1)(|g| + wd |p|), Va = b2 v + (1 - b2)(|g| + wd |p|)^2, den64 = sqrt(v64) / sqrt(bc2) + eps
and step = lr / bc1 -- a few ulps of the parameter plus a few ulps of the update and of its inputs.
test_adam_bound_calibration_on_emulated_kernel checks both sides on the CPU (the emulation: 0.33 of the bound; bc1 used for
both corrections, moments stored in bf16, eps inside the square root: >= 8000x).

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s): worst ratio to the bound
    loss rows at training size 0.28 (B = 16) / 0.19 (B = 3); chunk borders 0.22 (24 rows); Adam 0.33 (worst of steps 1, 2,
    10, 1000 over the generator and MSD sets).  The race test fails without the upload wait: a step off by 1.6e-4 (~lr).
"""
import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth

U = 2.0 ** -24
TAU_L = 2.0 ** -21
CHUNK = 16384          # kLossChunk
ADAM_CHUNK = 4096      # kAdamChunk
F32 = np.float32


# ------------------------------------------------------------------------------------------------------------------
# losses: the bound, calibrated on the CPU
# ------------------------------------------------------------------------------------------------------------------
def terms64(a, b, mode):
    a = a.double()
    return (a - b.double()).abs() if mode == 0 else (1 - a) ** 2 if mode == 1 else a * a


def loss_ratio(got, a, b, mode):
    """|got - ref| / (TAU_L mean|term| + 2^-24 |ref|) of one row."""
    t = terms64(a, b, mode)
    ref = float(t.mean())
    return abs(float(got) - ref) / (TAU_L * float(t.abs().mean()) + U * abs(ref))


def emulate_row(terms, drop_last_chunk=False, partial_bf16=False, thread_fp16=False):
    """loss_partial_kernel + loss_final_kernel on an aligned row of fp32 terms: per thread, float4 groups at
    4 t + 1024 i added as (t0 + t1) + (t2 + t3), the scalar tail, the xor-shuffle tree, the 8-warp tree; the CTA partials
    combined in float64 and divided by n."""
    n = terms.size
    acc = F32 if not thread_fp16 else np.float16
    parts = []
    for base in range(0, n, CHUNK):
        seg = terms[base:min(base + CHUNK, n)]
        n4 = seg.size & ~3
        s = np.zeros(256, acc)
        g = seg[:n4].reshape(-1, 4)
        for i in range(0, g.shape[0], 256):
            blk = g[i:i + 256]
            add = (blk[:, 0] + blk[:, 1]) + (blk[:, 2] + blk[:, 3])
            s[:blk.shape[0]] = (s[:blk.shape[0]] + add.astype(acc)).astype(acc)
        for j in range(n4, seg.size):
            s[j - n4] = acc(s[j - n4] + acc(seg[j]))
        s = s.astype(F32)
        for o in (16, 8, 4, 2, 1):           # lane l ends with the tree over its xor partners; lane 0 is read
            s = s + s[np.arange(256) ^ o]
        r = s[::32]
        p = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        if partial_bf16:
            p = torch.tensor(float(p)).to(torch.bfloat16).item()
        parts.append(float(p))
    if drop_last_chunk and len(parts) > 1:
        parts = parts[:-1]
    return F32(sum(parts) / n)


@pytest.mark.parametrize("n,mode", [(3 * CHUNK + 1, 0), (CHUNK, 1), (5 * CHUNK + 7, 2), (2 * CHUNK - 3, 0)])
def test_loss_tau_calibration_on_emulated_reduction(n, mode):
    """The fp32 emulation of the reduction uses < 0.5 of the bound; each wrong variant exceeds it by >= 8x."""
    gen = torch.Generator().manual_seed(n + mode)
    a, b = torch.randn(n, generator=gen) * 0.3 + 0.2, torch.randn(n, generator=gen) * 0.3
    if mode == 0:
        t = (a - b).abs()
    else:
        t = (1 - a) ** 2 if mode == 1 else a * a
    t = t.numpy().astype(F32)
    good = loss_ratio(emulate_row(t), a, b, mode)
    wrong = {name: loss_ratio(emulate_row(t, **{key: True}), a, b, mode)
             for name, key in (("last chunk dropped", "drop_last_chunk"), ("bf16 partial sums", "partial_bf16"),
                               ("fp16 per-thread sums", "thread_fp16"))}
    if n <= CHUNK:
        del wrong["last chunk dropped"]   # one chunk: nothing to drop
    print("\nn=%d mode %d: emulation %.3f of the bound; %s" % (n, mode, good, ", ".join("%s %.0f" % kv for kv in wrong.items())))
    assert good < 0.5, good
    assert min(wrong.values()) >= 8, wrong


# ------------------------------------------------------------------------------------------------------------------
# losses on the GPU: training size through the stacked path
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def msd():
    m = models.MultiScaleDiscriminator()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    return m.cuda().train()


def _check_l1_grad(got, a, b, scale, extra=None):
    """got: gradient of scale * mean|a - b| (+ extra, a float64 gradient added by another loss) w.r.t. a."""
    d = a.double() - b.double()
    mag = scale / a.numel()
    ref = torch.sign(d) * mag + (extra if extra is not None else 0)
    if extra is None:
        assert torch.equal(torch.sign(got), torch.sign(d)), "L1 gradient sign"
    tol = 2.0 ** -22 * (mag + (extra.abs() if extra is not None else 0))
    assert bool(((got.double() - ref).abs() <= tol).all()), float(((got.double() - ref).abs() / tol).max())


@pytest.mark.gpu
@pytest.mark.parametrize("B", [16, 3])
def test_losses_at_training_size_through_the_stacked_path(msd, B):
    """Config 3 (B = 16 x 8192) and B = 3 (odd: the second half of every stacked map is not 16-byte aligned): values of
    every row against float64, the totals of the generator and discriminator steps, and the full stacked gradients."""
    y = torch.from_numpy(synth.audio_input(B, 8192, 40 + B)).cuda()
    y_hat = torch.from_numpy(synth.audio_input(B, 8192, 50 + B)).cuda().requires_grad_(True)
    worst = 0.0
    # generator step: feature_loss + generator_loss on the same stacked parents
    dr, dg, fr, fg = msd(y, y_hat)
    parents = [t._mg_half[0] for maps in fr for t in maps]      # 21 stacked maps; every 7th is a logit map
    if B % 2:
        assert any(p[B:].data_ptr() % 16 for p in parents)
    with torch.no_grad():
        rows = engine.loss_forward([p[:B] for p in parents], [p[B:] for p in parents], [engine.LOSS_L1] * 21)
        for i, p in enumerate(parents):
            r = loss_ratio(rows[i], p[:B], p[B:], 0)
            assert r <= 1, (i, r)
            worst = max(worst, r)
        lsg = engine.loss_forward([p[B:] for p in parents[6::7]], [None] * 3, [engine.LOSS_ONE_MINUS_SQ] * 3)
        for i, p in enumerate(parents[6::7]):
            worst = max(worst, loss_ratio(lsg[i], p[B:], None, 1))
    lf, lg = models.feature_loss(fr, fg), models.generator_loss(dg)
    p64 = [p.detach().double().requires_grad_(True) for p in parents]
    f64 = 10 * sum((p[:B] - p[B:]).abs().mean() for p in p64)
    g64 = sum(((1 - p[B:]) ** 2).mean() for p in p64[6::7])
    for got, ref, terms in ((lf, f64, [10 * (p[:B] - p[B:]).abs().mean() for p in p64]),
                            (lg, g64, [((1 - p[B:]) ** 2).mean() for p in p64[6::7]])):
        tol = sum(TAU_L * float(t) for t in terms) + 32 * U * abs(float(ref))
        assert abs(float(got) - float(ref)) <= tol, (float(got), float(ref), tol)
    # gradients: feature_loss alone, generator_loss alone (the real half exactly 0), and their sum through autograd
    gf = torch.autograd.grad(lf, parents, retain_graph=True)
    gg = torch.autograd.grad(lg, parents[6::7], retain_graph=True)
    gs = torch.autograd.grad(lf + lg, parents)
    rf = torch.autograd.grad(f64, p64, retain_graph=True)
    rg = torch.autograd.grad(g64, p64[6::7])
    for i, p in enumerate(parents):
        _check_l1_grad(gf[i][:B], p[:B], p[B:], 10.0)
        _check_l1_grad(-gf[i][B:], p[:B], p[B:], 10.0)
        extra = rg[i // 7] if i % 7 == 6 else None
        ref = rf[i] + (extra if extra is not None else 0)
        tol = 2.0 ** -22 * (rf[i].abs() + (extra.abs() if extra is not None else 0))
        assert bool(((gs[i].double() - ref).abs() <= tol).all()), i
    for i, p in enumerate(parents[6::7]):
        assert bool((gg[i][:B] == 0).all()), "generator_loss wrote the real half"
        assert bool(((gg[i][B:].double() - rg[i][B:]).abs() <= 2.0 ** -22 * rg[i][B:].abs()).all())
    # discriminator step: real rows (1 - a)^2 and generated rows a^2 on the two halves of each logit map
    dr, dg, _, _ = msd(y, y_hat.detach())
    dl, rl, gl = models.discriminator_loss(dr, dg)
    logits = [t._mg_half[0] for t in dr]
    l64 = [p.detach().double().requires_grad_(True) for p in logits]
    r64 = [((1 - p[:B]) ** 2).mean() for p in l64]
    q64 = [(p[B:] ** 2).mean() for p in l64]
    for i, p in enumerate(logits):
        for got, half, mode in ((rl[i], p[:B], 1), (gl[i], p[B:], 2)):
            r = loss_ratio(got, half, None, mode)
            assert r <= 1, (i, mode, r)
            worst = max(worst, r)
    tot64 = sum(r64) + sum(q64)
    assert abs(float(dl) - float(tot64)) <= sum(TAU_L * float(t) for t in r64 + q64) + 8 * U * float(tot64)
    gd = torch.autograd.grad(dl, logits)
    rd = torch.autograd.grad(tot64, l64)
    for g, r in zip(gd, rd):
        assert bool(((g.double() - r).abs() <= 2.0 ** -22 * r.abs()).all())
    print("\nB=%d: worst loss row %.3f of the bound" % (B, worst))


# ------------------------------------------------------------------------------------------------------------------
# losses on the GPU: row and chunk borders through engine.loss_forward / loss_backward
# ------------------------------------------------------------------------------------------------------------------
BORDER_N = [1, 3, 4, 5, CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 1]


def _row_table(count, seed):
    """count rows cycling through the border sizes, modes and alignments (a misaligned with b aligned and the reverse):
    rows of several chunks put row boundaries in the middle of the grid."""
    gen = torch.Generator().manual_seed(seed)
    a, b, modes = [], [], []
    for i in range(count):
        n = BORDER_N[i % len(BORDER_N)]
        mode = i % 3
        oa, ob = (1, 0) if i % 4 == 1 else (0, 3) if i % 4 == 2 else (2, 2) if i % 4 == 3 else (0, 0)
        ba = (torch.randn(n + 4, generator=gen) * 0.5).cuda()
        bb = (torch.randn(n + 4, generator=gen) * 0.5).cuda()
        ta, tb = ba[oa:oa + n], bb[ob:ob + n]
        if i % 5 == 0:
            tb[: n // 2] = ta[: n // 2]                  # exact ties: the L1 gradient must be 0 there
        a.append(ta)
        b.append(tb)
        modes.append(mode)
    return a, b, modes


@pytest.mark.gpu
@pytest.mark.parametrize("count", [8, 24])
def test_loss_rows_at_chunk_borders(count):
    a, b, modes = _row_table(count, count)
    assert sum(1 for t in a if t.data_ptr() % 16) >= count // 4
    out = engine.loss_forward(a, b, modes)
    worst = 0.0
    for i in range(count):
        r = loss_ratio(out[i], a[i], b[i], modes[i])
        assert r <= 1, (i, a[i].numel(), modes[i], r)
        worst = max(worst, r)
    assert torch.equal(out, engine.loss_forward(a, b, modes))
    gout = torch.linspace(0.5, 3.0, count, device="cuda")
    ga, gb = engine.loss_backward(a, b, modes, gout, [True] * count)
    for i in range(count):
        n, sc = a[i].numel(), float(gout[i]) / a[i].numel()
        x, d = a[i].double(), a[i].double() - b[i].double()
        if modes[i] == 0:
            assert torch.equal(torch.sign(ga[i]), torch.sign(d)) and torch.equal(gb[i], -ga[i]), i
            ref = torch.sign(d) * sc
        else:
            assert gb[i] is None or modes[i] != 0
            ref = -2 * (1 - x) * sc if modes[i] == 1 else 2 * x * sc
        assert bool(((ga[i].double() - ref).abs() <= 2.0 ** -22 * ref.abs()).all()), (i, n, modes[i])
    print("\n%d rows: worst %.3f of the bound" % (count, worst))


# ------------------------------------------------------------------------------------------------------------------
# Adam: the bound, calibrated on the CPU
# ------------------------------------------------------------------------------------------------------------------
def adam64(p, g, m, v, t, lr, b1, b2, eps, wd):
    """One float64 Adam step from (p, m, v) with the fp32 hyper-parameters the kernel receives; returns the new state
    and the magnitudes the bound needs."""
    lr, b1, b2, eps, wd = (float(F32(x)) for x in (lr, b1, b2, eps, wd))
    p, g, m, v = (x.double() for x in (p, g, m, v))
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    gr = g + wd * p
    m1 = b1 * m + (1 - b1) * gr
    v1 = b2 * v + (1 - b2) * gr * gr
    den = v1.sqrt() / bc2 ** 0.5 + eps
    step = lr / bc1
    p1 = p - step * m1 / den
    ga = g.abs() + wd * p.abs()
    Ma = (b1 * m).abs() + (1 - b1) * ga
    Va = b2 * v + (1 - b2) * ga * ga
    return p1, m1, v1, dict(Ma=Ma, Va=Va, den=den, step=step)


def adam_ratio(got, ref):
    """Worst ratio to the bound of (p, m, v) against adam64's (p1, m1, v1, magnitudes)."""
    (p, m, v), (p1, m1, v1, k) = got, ref
    rm = (m.double() - m1).abs() / (8 * U * k["Ma"]).clamp_min(1e-300)
    rv = (v.double() - v1).abs() / (12 * U * k["Va"]).clamp_min(1e-300)
    up = k["step"] * k["Ma"] / k["den"] * (1 + k["Va"] / v1.clamp_min(1e-300))
    rp = (p.double() - p1).abs() / (4 * U * p1.abs() + 8 * U * up).clamp_min(1e-300)
    return max(float(rm.max()), float(rv.max()), float(rp.max()))


def emulate_adam(p, g, m, v, t, lr, b1, b2, eps, wd, bc1_both=False, bf16_moments=False, eps_in_sqrt=False):
    """adam_kernel in float32, in its expression order (bias corrections from float64 pow, as the launcher does)."""
    f = lambda x: x.float()
    lr, b1, b2, eps, wd = (float(F32(x)) for x in (lr, b1, b2, eps, wd))
    bc1 = torch.tensor(1 - b1 ** t, dtype=torch.float32)
    bc2s = torch.tensor((1 - b2 ** t) ** 0.5, dtype=torch.float32)
    if bc1_both:
        bc2s = bc1
    b1f, b2f, wdf, epsf = (torch.tensor(x, dtype=torch.float32) for x in (b1, b2, wd, eps))
    gr = f((g.double() + wdf.double() * p.double()))      # fmaf(wd, p, g)
    mn = b1f * m + (1 - b1f) * gr
    vn = b2f * v + (1 - b2f) * gr * gr
    if bf16_moments:
        mn, vn = mn.bfloat16().float(), vn.bfloat16().float()
    step = torch.tensor(lr, dtype=torch.float32) / bc1
    den = (vn + epsf).sqrt() / bc2s if eps_in_sqrt else vn.sqrt() / bc2s + epsf
    return p - step * mn / den, mn, vn


ADAM_CASES = [(t, betas, wd) for t in (1, 2, 10, 1000) for betas in ((0.5, 0.9), (0.9, 0.999)) for wd in (0.0, 0.01)]


def _adam_state(n, t, seed, device="cpu"):
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen) * 0.1
    g = torch.randn(n, generator=gen) * torch.rand(n, generator=gen) * 1e-2
    g[::97] = 0
    if t == 1:
        m, v = torch.zeros(n), torch.zeros(n)
    else:
        m = torch.randn(n, generator=gen) * 1e-3
        v = (torch.randn(n, generator=gen) * 1e-3) ** 2
    return [x.to(device) for x in (p, g, m, v)]


def test_adam_bound_calibration_on_emulated_kernel():
    """The fp32 emulation uses < 0.5 of the bound in every case; each wrong variant exceeds it by >= 8x (in the cases
    where it differs from Adam at all: with betas (0.5, 0.9) both corrections are 1 by step 1000)."""
    good, wrong = 0.0, {"bc1 for both corrections": 0.0, "bf16 moments": 0.0, "eps inside the square root": 0.0}
    for i, (t, (b1, b2), wd) in enumerate(ADAM_CASES):
        p, g, m, v = _adam_state(20000, t, i)
        hp = (t, 1e-3 * (1 + 0.1 * i), b1, b2, 1e-8, wd)
        ref = adam64(p, g, m, v, *hp)
        good = max(good, adam_ratio(emulate_adam(p, g, m, v, *hp), ref))
        for name, kw in (("bc1 for both corrections", "bc1_both"), ("bf16 moments", "bf16_moments"),
                         ("eps inside the square root", "eps_in_sqrt")):
            wrong[name] = max(wrong[name], adam_ratio(emulate_adam(p, g, m, v, *hp, **{kw: True}), ref))
    print("\nAdam emulation %.3f of the bound; wrong variants: %s" % (good, ", ".join("%s %.0f" % kv for kv in wrong.items())))
    assert good < 0.5, good
    assert min(wrong.values()) >= 8, wrong


# ------------------------------------------------------------------------------------------------------------------
# Adam on the GPU
# ------------------------------------------------------------------------------------------------------------------
def _param_shapes():
    """The generator's 90 and the MSD's 63 parameter tensors (conv_post1 weight_v: 5.2 M elements), plus sizes at the
    4096-element chunk border."""
    g = [tuple(p.shape) for p in models.Generator().parameters()]
    d = [tuple(p.shape) for p in models.MultiScaleDiscriminator().parameters()]
    return {"generator": g + [(1,), (ADAM_CHUNK - 1,), (ADAM_CHUNK,), (ADAM_CHUNK + 1,)], "msd": d}


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["generator", "msd"])
@pytest.mark.parametrize("betas,wd", [((0.5, 0.9), 0.0), ((0.9, 0.999), 0.01)])
def test_adam_steps_against_float64_on_the_kernels_own_state(which, betas, wd):
    """Steps 1, 2, 10 and 1000, lr changed between steps as a scheduler does; each step from the kernel's own state."""
    from melgan_multi_b200.optim import Adam
    shapes = _param_shapes()[which]
    if which == "msd":
        assert len(shapes) == 63 and max(int(np.prod(s)) for s in shapes) == 1024 * 1024 * 5
    gen = torch.Generator(device="cuda").manual_seed(len(shapes))
    ps = [(torch.randn(s, device="cuda", generator=gen) * 0.1).requires_grad_(True) for s in shapes]
    opt = Adam(ps, 2e-4, betas=betas, weight_decay=wd)
    worst = 0.0
    for k, t in enumerate((1, 2, 10, 1000)):
        if k >= 2:   # jump to step t - 1, keeping the kernel's moments
            sd = opt.state_dict()
            for st in sd["state"].values():
                st["step"] = torch.tensor(float(t - 1))
            opt.load_state_dict(sd)
        lr = 2e-4 * (1 - 0.2 * k)
        opt.param_groups[0]["lr"] = lr
        for p in ps:
            p.grad = torch.randn(p.shape, device="cuda", generator=gen) * torch.rand(p.shape, device="cuda", generator=gen) * 1e-2
        before = [(p.detach().clone(), opt.state[p]["exp_avg"].clone() if t > 1 else torch.zeros_like(p),
                   opt.state[p]["exp_avg_sq"].clone() if t > 1 else torch.zeros_like(p)) for p in ps]
        opt.step()
        for p, (p0, m0, v0) in zip(ps, before):
            ref = adam64(p0, p.grad, m0, v0, t, lr, betas[0], betas[1], 1e-8, wd)
            r = adam_ratio((p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]), ref)
            assert r <= 1, (which, t, tuple(p.shape), r)
            worst = max(worst, r)
    assert int(opt.state_dict()["state"][0]["step"]) == 1000
    print("\n%s betas %s wd %g: worst %.3f of the bound" % (which, betas, wd, worst))


@pytest.mark.gpu
def test_adam_steps_queued_behind_a_busy_stream_use_their_own_gradients():
    """A host that runs steps ahead of the GPU: the stream is held by a bounded sleep while three steps, each with fresh
    gradient tensors at new addresses, are enqueued without a sync.  Each step must read its own gradients, not a later
    step's pointer table."""
    from melgan_multi_b200.optim import Adam
    gen = torch.Generator(device="cuda").manual_seed(3)
    ps = [(torch.randn(n, device="cuda", generator=gen) * 0.1).requires_grad_(True) for n in (1, 4097, 70000)]
    opt = Adam(ps, 1e-3, betas=(0.5, 0.9))
    for p in ps:
        p.grad = torch.randn_like(p) * 1e-2
    opt.step()   # builds the table (its first upload is synchronous)
    grads = [[torch.randn(p.shape, device="cuda", generator=gen) * 1e-2 for p in ps] for _ in range(3)]
    state = [(p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone()) for p in ps]
    torch.cuda.synchronize()
    torch.cuda._sleep(2 * 10 ** 9)    # about one second of the stream's time
    for gs in grads:
        for p, g in zip(ps, gs):
            p.grad = g
        opt.step()
    torch.cuda.synchronize()
    for i, p in enumerate(ps):
        p64, m64, v64 = state[i]
        for k in range(3):
            p64, m64, v64, _ = adam64(p64, grads[k][i], m64, v64, 2 + k, 1e-3, 0.5, 0.9, 1e-8, 0.0)
        err = float((p.detach().double() - p64).abs().max())
        assert err <= 1e-4 * 1e-3, (i, err)   # a step on another step's gradients is off by ~lr
