"""Every discriminator backward kernel on its OWN recorded inputs, against a float64 statement of its own gradient, at the
training size, at the ragged lengths and at every tile and chunk border of its launch geometry; the one-call chain
(mg_msd_scale_backward) against the kernels it is made of; weight-norm backward against float64 autograd.

Section 1 runs the stacked (real, generated) forward, takes the gradients of the feature-map L1 loss plus the LSGAN
generator term w.r.t. the 21 returned maps through the package's loss functions, and walks each scale from the logits
down through the per-kernel entry points (lrelu_backward, edge_backward, post1_dgrad, post1_wgrad, grouped_backward).
Layer l gets the dz the engine produced for it and the map the forward recorded, so an error can be neither hidden by nor
blamed on another layer.  Every element of dx, dW and db is held to

    |g - g64| <= tau * A2 + 2^-20 * |g64|,

with g64 = torch.nn.grad.conv1d_input / conv1d_weight / sum(dz) in float64 on the same fp32 inputs, and A2 the
root-sum-square of the products that make up the element (the same float64 call on squared operands; sqrt(sum dz^2)
for db).  tau depends on the arithmetic of the kernel:
  * split-bf16 wgmma (conv_post1 dgrad and wgrad): TAU = 2^-12, as for the forward (test_layer_isolation_gpu);
    test_tau_calibration_on_emulated_split_bf16_backward checks it at the two backward contractions.  These two also get
    a relative term for the tensor cores' accumulation (wgmma_rel): 2^-24 |g64| per MMA that adds into one accumulator.
    Without it the wgrad dW at config 3, scale 0 (768 MMAs, elements with |g64| = 9.6 A2) reaches 1.07 of the bound,
    0.87 TAU A2 away from an exact 3-pass emulation on the same operands, which itself uses 0.35.
  * fp32 SIMT: a sum of n products accumulated one after another in fp32 carries a rounding error that grows like
    2^-24 sqrt(n) A2 (random signs), so tau_simt(n) = 2^-20 sqrt(n), 16x that scale.  Dropping one typical product of
    the n (about A2 / sqrt(n)) is then 2^20 / n of the bound, >= 8x up to n = 2^17.  n follows from the kernel:
    176 = 16 channels x 11 taps (grouped_dx4_kernel), 164 = 4 x 41 (grouped_dx1_kernel), 240 = 16 x 15 (conv_pre dx),
    3 (conv_post2 dx); tiles per chunk x 128 plus the chunk count of the combine (grouped dW and db); 512 plus the tile
    count (conv_pre dW and db); Bt L / 256 per thread plus the 8-level tree (conv_post2 dW and db); the stage count plus
    8 (conv_post1 db).  test_tau_calibration_on_emulated_fp32_sums checks both sides at those n.
  * LeakyReLU' (lrelu_grad_kernel) is bit-identical to (g1 + g2) * where(out > 0, 1, slope) in float32.

Measured on an H100 80GB HBM3 (400 W power limit), printed by the tests (-s).  Worst ratio to the bound at config 3
(32 x 8192), worst of the three scales, dx / dW / db (the ragged lengths stay at or below these):
    conv_pre 0.250 / 0.655 / 0.632, grouped_convs.0-3 0.247 / 0.636 / 0.540, 0.203 / 0.264 / 0.230,
    0.214 / 0.173 / 0.144, 0.232 / 0.130 / 0.108, conv_post1 0.244 / 0.390 / 0.104, conv_post2 0.108 / 0.105 / 0.014;
    weight-norm backward 0.237.  CPU calibration: fp32 sums 0.05 - 0.16 of tau_simt(n), one product dropped >= 13x;
    split-bf16 backward 0.06 - 0.08 of TAU, one pass dropped >= 13.8x.  The GPU tests of this file take about 20 s.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv1d_input, conv1d_weight

from melgan_multi_b200 import engine, synth
from kernel_model import ddev, dstate  # noqa: F401 (fixtures)
from kernel_model import (POST1_PAD, POST1_ROWS, REL, SIMT_N, TAU, WG_PANEL, WG_STAGE, bf16_rn, cdiv, folded64,
                          post1_lengths, post1_straddles, tau_simt, upstream)

LAYERS = synth.DISCRIMINATOR_LAYERS
SLOPE = 0.01  # kSlope (csrc/mg_layout.h)
SIZES = [(32, 8192), (2, 64), (6, 257), (4, 2050), (2, 4097)]  # config 3 and the ragged lengths of test_disc_gpu.py

# launch geometry of the kernels (csrc/mg_disc_bwd.cu, mg_disc_edge_bwd.cu, mg_conv_tc.cu, mg_wgrad_tc.cu)
DX4_TILE = 512                   # grouped_dx4_kernel: input positions per CTA, a quad of positions per thread
DX1_TILE, DX1_VEC = 128, 8       # grouped_dx1_kernel: positions per CTA, per thread (two float4 stores if p + 8 <= Lin)
DW_TILE = 128                    # grouped_dw4_kernel / grouped_dw1_kernel: output positions per tile
PRE_TILE, PRE_HALO = 512, 7      # disc_pre_bwd_kernel
POST2_THREADS = 256              # disc_post2_dw_kernel: threads along the flattened (item, position) axis


def grouped_plan(layer, Bt, Lout):
    """(tiles per item, tiles per chunk, chunks) of the grouped weight-gradient launch, read back from the library: the
    workspace holds one [groups][165 * COG] partial per chunk, and chunks = ceil(total / tiles per chunk) determines the
    tiles per chunk as ceil(total / chunks)."""
    _n, _cin, cout, _k, _s, groups, _p = LAYERS[layer]
    per_chunk = groups * 165 * (cout // groups) * 4
    nbytes = engine.lib().mg_msd_grouped_backward_workspace_bytes(layer, Bt, Lout)
    assert nbytes > 0 and nbytes % per_chunk == 0, (layer, Bt, Lout, nbytes)
    tiles = cdiv(Lout, DW_TILE)
    chunks = nbytes // per_chunk
    tpc = cdiv(Bt * tiles, chunks)
    assert cdiv(Bt * tiles, tpc) == chunks
    return tiles, tpc, chunks


def kernel_ns(layer, Bt, Lin, Lout):
    """{gradient: n} of the kernels that compute layer `layer`'s backward at this size: the fp32 products one output
    element accumulates in sequence, or None for the split-bf16 wgmma kernels."""
    if layer == 0:
        n = PRE_TILE + Bt * cdiv(Lin, PRE_TILE)
        return {"dx": 16 * 15, "dw": n, "db": n}
    if layer == 5:
        return {"dx": None, "dw": None, "db": cdiv(Bt * cdiv(Lout, WG_PANEL), WG_STAGE // WG_PANEL) + 8}
    if layer == 6:
        n = cdiv(Bt * Lin, POST2_THREADS) + 8
        return {"dx": 3, "dw": n, "db": n}
    _tiles, tpc, chunks = grouped_plan(layer, Bt, Lout)
    n = tpc * DW_TILE + chunks
    return {"dx": 176 if layer < 4 else 164, "dw": n, "db": n}


def wgmma_rel(layer, Bt, L):
    """{gradient: extra relative term} of conv_post1's wgmma kernels: the tensor cores add each MMA into the fp32
    accumulator without rounding to nearest, an error of up to 2^-24 of the running sum per MMA that does not average out
    (measured at config 3, scale 0: the wgrad dW sits 0.87 TAU A2 from an exact 3-pass emulation where |g64| = 9.6 A2).
    n_mma = the MMAs that add into one accumulator: 3 passes x K / 16."""
    if layer != 5:
        return {}
    stages = cdiv(Bt * cdiv(L, WG_PANEL), WG_STAGE // WG_PANEL)
    return {"dx": 2.0 ** -24 * 3 * (1024 * 5 // 16), "dw": 2.0 ** -24 * 3 * (stages * WG_STAGE // 16)}


def bound_ratio(got, ref, a2, tau, rel=0.0):
    """Worst |g - g64| / (tau A2 + (2^-20 + rel) |g64|) (<= 1: within the bound)."""
    assert got is not None and tuple(got.shape) == tuple(ref.shape), (None if got is None else tuple(got.shape), tuple(ref.shape))
    d = (got.double() - ref).abs()
    return float((d / (tau * a2 + (REL + rel) * ref.abs()).clamp_min(1e-300)).max())


def layer_weights(dstate, s):
    return [folded64(dstate, "discriminators.%d.%s" % (s, n))[0] for n, *_ in LAYERS]


def run_layer(dd, s, l, x, dz, need_dx):
    """(dx | None, dw, db) of layer l of scale s through its per-kernel entry points."""
    if l in (0, 6):
        return dd.edge_backward(s, l, dz, x, need_dx)
    if l == 5:
        dw, db = dd.post1_wgrad(x, dz)
        return (dd.post1_dgrad(s, dz) if need_dx else None), dw, db
    return dd.grouped_backward(s, l, dz, x, need_dx)


def check_layer(l, x, dz, dx, dw, db, w64):
    """{gradient: worst ratio to the bound} of one layer's kernel outputs against float64 on the same fp32 inputs."""
    _n, _cin, _cout, _k, stride, groups, pad = LAYERS[l]
    ns = kernel_ns(l, x.shape[0], x.shape[2], dz.shape[2])
    assert all(n is None or n <= max(SIMT_N) for n in ns.values()), ("n beyond the calibrated range", l, ns)
    taus = {k: TAU if n is None else tau_simt(n) for k, n in ns.items()}
    rels = wgmma_rel(l, x.shape[0], dz.shape[2])
    x64, dz64 = x.double(), dz.double()
    out = {}
    if dx is not None:
        ref = conv1d_input(x.shape, w64, dz64, stride, pad, 1, groups)
        a2 = conv1d_input(x.shape, w64 * w64, dz64 * dz64, stride, pad, 1, groups).sqrt()
        out["dx"] = bound_ratio(dx, ref, a2, taus["dx"], rels.get("dx", 0.0))
    ref = conv1d_weight(x64, w64.shape, dz64, stride, pad, 1, groups)
    a2 = conv1d_weight(x64 * x64, w64.shape, dz64 * dz64, stride, pad, 1, groups).sqrt()
    out["dw"] = bound_ratio(dw, ref, a2, taus["dw"], rels.get("dw", 0.0))
    out["db"] = bound_ratio(db, dz64.sum(dim=(0, 2)), dz64.square().sum(dim=(0, 2)).sqrt(), taus["db"])
    return out


def walk(dd, s, x0, fm, grads, need_gx0, w64=None, ratios=None):
    """The backward of scale s composed layer by layer from the per-kernel entry points, in the order and with the operands
    of mg_msd_scale_backward; returns (gx0 | None, dws[7], dbs[7]) like DiscriminatorDevice.scale_backward.  With w64 each
    kernel is also held to float64 on the inputs it was given, the worst ratios going into ratios[(s, layer, gradient)]."""
    g, gx0, dws, dbs = None, None, [None] * 7, [None] * 7
    for l in range(6, -1, -1):
        go = grads[l]
        if g is None and go is None:
            continue
        if l == 6:
            dz = go
        else:
            dz = dd.lrelu_backward(g, go, fm[l])
            if w64 is not None:
                a = g if go is None else go if g is None else g + go
                assert torch.equal(dz, a * torch.where(fm[l] > 0, 1.0, SLOPE)), ("lrelu_backward", s, l)
        x = x0 if l == 0 else fm[l - 1]
        dx, dws[l], dbs[l] = run_layer(dd, s, l, x, dz, l > 0 or need_gx0)
        if w64 is not None:
            for k, r in check_layer(l, x, dz, dx, dws[l], dbs[l], w64[l]).items():
                ratios[(s, l, k)] = max(ratios.get((s, l, k), 0.0), r)
        g = dx
        if l == 0:
            gx0 = dx
    return gx0, dws, dbs


def scale_input(y, s):
    """The input of discriminator s as training computes it (fp32 AvgPool chain of MultiScaleDiscriminator)."""
    x = y
    for k in range(s):
        x = F.avg_pool1d(x, 4, 2 if k == 0 else 4, padding=2)
    return x


def forward(dd, Bt, L):
    y = torch.from_numpy(synth.audio_input(Bt, L, 11 * L + Bt)).cuda()
    fm = dd.forward(y)
    dd.check_status()
    return y, fm


# ------------------------------------------------------------------------------------------------------------------
# the two taus, calibrated on the CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIMT_N)
def test_tau_calibration_on_emulated_fp32_sums(n):
    """An fp32 sum of n products accumulated in sequence (one rounding per fmaf) uses < 0.5 of tau_simt(n); the same sum
    with one typical product left out exceeds it by >= 8x (median over elements)."""
    rng = np.random.default_rng(n)
    m = 4096
    x = rng.standard_normal((n, m)).astype(np.float32)
    x = np.where(x > 0, x, np.float32(SLOPE) * x)  # post-LeakyReLU operands, like the layers' inputs
    p = x.astype(np.float64) * rng.standard_normal((n, m)).astype(np.float32)  # exact products of fp32 operands
    ref = p.sum(axis=0)
    bound = tau_simt(n) * np.sqrt((p * p).sum(axis=0)) + REL * np.abs(ref)

    def fp32_sum(skip):
        acc = np.zeros(m, np.float32)
        for i in range(n):
            if i != skip:
                acc = (acc + p[i]).astype(np.float32)
        return acc

    full = float((np.abs(fp32_sum(-1) - ref) / bound).max())
    dropped = float(np.median(np.abs(fp32_sum(n // 2) - ref) / bound))
    print("n=%d: fp32 sum %.3f of the bound, one product dropped %.1f" % (n, full, dropped))
    assert full < 0.5, (n, full)
    assert dropped >= 8, (n, dropped)


def split_bilinear(f, a, b, passes=(0, 1, 2)):
    """A bilinear contraction f(a, b) the way the tensor cores run it on fp32 operands: passes (ah, bh), (al, bh), (ah, bl)
    of the bf16 hi / lo split, exact products accumulated (in float64 here, rounded to fp32 at the end)."""
    ah, bh = bf16_rn(a), bf16_rn(b)
    al, bl = bf16_rn(a - ah), bf16_rn(b - bh)
    ops = [(ah, bh), (al, bh), (ah, bl)]
    return sum(f(ops[p][0].double(), ops[p][1].double()) for p in passes).float()


@pytest.mark.parametrize("which,Bt,L", [("wgrad", 1, 3), ("wgrad", 3, 65), ("wgrad", 32, 17), ("wgrad", 32, 65),
                                        ("wgrad", 32, 128), ("dgrad", 2, 64)])
def test_tau_calibration_on_emulated_split_bf16_backward(which, Bt, L):
    """conv_post1's two backward contractions -- wgrad (A = dz, B = x, K = Bt L up to 32 x 128) and dgrad (A = dz, B = the
    transposed weight, K = 1024 x 5) -- pass the element-wise bound at TAU with margin in the 3-pass split, and fail it
    by >= 8x with any one pass dropped."""
    gen = torch.Generator().manual_seed(Bt * 1000 + L)
    C = 1024 if which == "dgrad" else 16
    dz = torch.randn(Bt, C, L, generator=gen)
    if which == "wgrad":
        x = F.leaky_relu(torch.randn(Bt, C, L, generator=gen))
        f = lambda a, b: conv1d_weight(b, (C, C, 5), a, 1, 2)
        a, b, K = dz, x, Bt * L
        ref = f(dz.double(), x.double())
        a2 = conv1d_weight(x.double() ** 2, (C, C, 5), dz.double() ** 2, 1, 2).sqrt()
    else:
        w = (torch.rand(C, 16, 5, generator=gen) * 2 - 1) / (C * 5) ** 0.5
        f = lambda a, b: conv1d_input((Bt, 16, L), b, a, 1, 2)
        a, b, K = dz, w, C * 5
        ref = f(dz.double(), w.double())
        a2 = conv1d_input((Bt, 16, L), w.double() ** 2, dz.double() ** 2, 1, 2).sqrt()
    full = bound_ratio(split_bilinear(f, a, b), ref, a2, TAU)
    dropped = [bound_ratio(split_bilinear(f, a, b, [p for p in range(3) if p != q]), ref, a2, TAU) for q in range(3)]
    print("%s K=%d: 3-pass %.3f of the bound, one pass dropped %s" % (which, K, full, " ".join("%.1f" % r for r in dropped)))
    assert full < 0.5, (K, full)
    assert min(dropped) >= 8, (K, dropped)


# ------------------------------------------------------------------------------------------------------------------
# 1. every backward kernel on its own recorded inputs
# ------------------------------------------------------------------------------------------------------------------
def report(ratios, head):
    lines = [head]
    for s in range(3):
        lines.append("  scale %d: " % s + ", ".join(
            "%s %s" % (LAYERS[l][0], "/".join("%s %.3f" % (k, ratios[(s, l, k)]) for k in ("dx", "dw", "db")
                                                if (s, l, k) in ratios)) for l in range(7)))
    print("\n".join(lines))


@pytest.mark.gpu
@pytest.mark.parametrize("Bt,L", SIZES)
def test_backward_kernels_on_their_own_inputs(ddev, dstate, Bt, L):
    """Gradients of the generator step (feature-map L1 + LSGAN) on the maps the forward returned; each scale walked from
    the logits down, every element of every dx / dW / db against float64, LeakyReLU' bit for bit."""
    y, fm = forward(ddev, Bt, L)
    G = upstream(fm, "generator")
    ratios = {}
    for s in range(3):
        walk(ddev, s, scale_input(y, s), fm[s], G[s], True, layer_weights(dstate, s), ratios)
    torch.cuda.synchronize()
    assert int(ddev.status[0].item()) == 0
    report(ratios, "\n(Bt=%d, L=%d) worst ratio to the bound:" % (Bt, L))
    bad = {k: r for k, r in ratios.items() if r > 1}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------
# 2. tile and chunk borders of the launch geometry
# ------------------------------------------------------------------------------------------------------------------
def dx4_lengths():
    """grouped_dx4_kernel (layers 1-3, input lengths): around the first two CTA borders, Lin % 4 != 0 included; the output
    lengths (Lin - 1) // 4 + 1 then sit around the dW kernel's 128-output tile (127, 128, 129)."""
    T = DX4_TILE
    return [5, T - 4, T - 1, T, T + 1, T + 3, 2 * T, 2 * T + 1]


def dx1_lengths():
    """grouped_dx1_kernel and grouped_dw1_kernel (layer 4, Lin = Lout): around the 128-position CTA and tile, with the
    two-float4 store (Lin % 4 == 0, p + 8 <= Lin), its scalar fallback at a multiple of 4 (last thread past the end) and
    Lin % 4 != 0."""
    T, V = DX1_TILE, DX1_VEC
    return [5, V, T - 1, T, T + 1, T + V // 2, T + V, 2 * T - 1, 2 * T, 2 * T + V // 2]


def pre_lengths():
    """disc_pre_bwd_kernel: 512-position tiles staged with a 7-position halo; shorter than the 15 taps, at the tile end,
    one past it and where the last tile ends inside the previous tile's halo."""
    T, H = PRE_TILE, PRE_HALO
    return [5, T - H, T - 1, T, T + 1, T + H, 2 * T, 2 * T + H]


BORDER_CASES = ([(l, L) for l in (1, 2, 3) for L in dx4_lengths()] + [(4, L) for L in dx1_lengths()] +
                [(0, L) for L in pre_lengths()] + [(5, L) for L in post1_lengths()])
# (layer, Bt, Lout) of the grouped weight-gradient chunk plan: chunks that straddle two items with a short last chunk,
# a single chunk, and the plan of layer 1 (264 chunks wanted) past its first straddle
CHUNK_CASES = [(3, 3, 891), (3, 1, 128), (4, 3, 891), (4, 1, 100), (1, 3, DW_TILE * 91)]


def chunk_claims(layer, Bt, Lout):
    """(a chunk straddles two items, the last chunk is short, one chunk) of the plan at this size."""
    tiles, tpc, chunks = grouped_plan(layer, Bt, Lout)
    straddle = any((c * tpc) // tiles != (min(Bt * tiles, (c + 1) * tpc) - 1) // tiles for c in range(chunks))
    return straddle, (Bt * tiles) % tpc != 0, chunks == 1


def test_border_cases_sit_on_the_kernel_borders():
    """The border lengths and chunk-plan cases are where their descriptions say (CPU: geometry and the library's plan)."""
    d4 = dx4_lengths()
    assert any(L % 4 for L in d4) and {DX4_TILE - 1, DX4_TILE, DX4_TILE + 1, 2 * DX4_TILE, 2 * DX4_TILE + 1} <= set(d4)
    assert {DW_TILE - 1, DW_TILE, DW_TILE + 1} <= {(L - 1) // 4 + 1 for L in d4}  # the dW tile, in output positions
    d1 = dx1_lengths()
    last = lambda L: DX1_VEC * ((L - 1) // DX1_VEC)  # first position of the last thread (16 threads x 8 per CTA)
    assert any(L % 4 == 0 and last(L) + DX1_VEC <= L for L in d1)   # every thread takes the vector store
    assert any(L % 4 == 0 and last(L) + DX1_VEC > L for L in d1)    # aligned rows, last thread on the scalar path
    assert any(L % 4 for L in d1)
    assert {DW_TILE - 1, DW_TILE, DW_TILE + 1} <= set(d1) and any(L % DW_TILE == 0 and L > DW_TILE for L in d1)
    pre = pre_lengths()
    assert min(pre) < 15 and {PRE_TILE - 1, PRE_TILE, PRE_TILE + 1} <= set(pre)
    assert any(L % PRE_TILE == PRE_HALO for L in pre) and any(L % PRE_TILE == PRE_TILE - PRE_HALO for L in pre)
    p1 = post1_lengths()
    assert any(L < 5 for L in p1) and any(L % 4 for L in p1) and any(L % 8 and L % 4 == 0 for L in p1)
    assert any(cdiv(L, WG_PANEL) % (WG_STAGE // WG_PANEL) for L in p1 if L > WG_STAGE)  # last stage part-filled
    assert any(POST1_ROWS % (L + POST1_PAD) == 0 and L + POST1_PAD < POST1_ROWS for L in p1)
    assert any(L + POST1_PAD == POST1_ROWS for L in p1) and any(post1_straddles(3, L) for L in p1)
    claims = {c: chunk_claims(*c) for c in CHUNK_CASES}
    for i, what in enumerate(("straddle", "short last chunk", "single chunk")):
        assert any(v[i] for v in claims.values()), (what, claims)
    assert claims[(3, 3, 891)][:2] == (True, True) and claims[(4, 3, 891)][:2] == (True, True)
    assert claims[(3, 1, 128)][2] and claims[(4, 1, 100)][2]


def border_inputs(layer, Bt, Lin, seed):
    _n, cin, cout, k, stride, _g, pad = LAYERS[layer]
    gen = torch.Generator().manual_seed(seed)
    Lout = (Lin + 2 * pad - k) // stride + 1
    x = torch.rand(Bt, 1, Lin, generator=gen) * 2 - 1 if layer == 0 else F.leaky_relu(torch.randn(Bt, cin, Lin, generator=gen))
    return x.cuda(), torch.randn(Bt, cout, Lout, generator=gen).cuda()


def check_at(dd, w64, layer, Bt, Lin):
    x, dz = border_inputs(layer, Bt, Lin, 1000 * layer + 10 * Lin + Bt)
    dx, dw, db = run_layer(dd, 1, layer, x, dz, True)
    r = check_layer(layer, x, dz, dx, dw, db, w64[layer])
    assert max(r.values()) <= 1, (layer, Bt, Lin, r)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("layer,Lin", BORDER_CASES)
def test_backward_kernels_at_tile_borders(ddev, dstate, layer, Lin):
    """Random operands at each border length, Bt = 1 and 3, every element under the bound."""
    w64 = layer_weights(dstate, 1)
    for Bt in (1, 3):
        check_at(ddev, w64, layer, Bt, Lin)
    torch.cuda.synchronize()
    assert int(ddev.status[0].item()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("layer,Bt,Lout", CHUNK_CASES)
def test_grouped_weight_gradient_chunk_plan(ddev, dstate, layer, Bt, Lout):
    Lin = Lout * LAYERS[layer][4]
    r = check_at(ddev, layer_weights(dstate, 1), layer, Bt, Lin)
    print("layer %d Bt=%d Lout=%d plan %s claims %s: %s" % (layer, Bt, Lout, grouped_plan(layer, Bt, Lout),
                                                           chunk_claims(layer, Bt, Lout), r))


# ------------------------------------------------------------------------------------------------------------------
# 3. the one-call chain equals its parts
# ------------------------------------------------------------------------------------------------------------------
def assert_same(chain, parts, what):
    (cx, cws, cbs), (px, pws, pbs) = chain, parts
    for name, a, b in [("gx0", cx, px)] + [("dw%d" % l, a, b) for l, (a, b) in enumerate(zip(cws, pws))] + \
                      [("db%d" % l, a, b) for l, (a, b) in enumerate(zip(cbs, pbs))]:
        assert (a is None) == (b is None), (what, name, a is None, b is None)
        assert a is None or torch.equal(a, b), (what, name, float((a - b).abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("Bt,L", SIZES)
def test_scale_backward_equals_its_kernels(ddev, Bt, L):
    """mg_msd_scale_backward bit for bit against the layer-by-layer composition, every scale, three gradient patterns:
    the generator step (all seven maps, gx0), the discriminator step (logits only, no gx0), one intermediate map (the
    layers above it unreached); and twice in a row (fixed summation order)."""
    y, fm = forward(ddev, Bt, L)
    for pattern, need in (("generator", True), ("discriminator", False), ("map 3", True)):
        G = upstream(fm, pattern)
        for s in range(3):
            x0 = scale_input(y, s)
            chain = ddev.scale_backward(s, x0, fm[s], G[s], need)
            assert_same(chain, walk(ddev, s, x0, fm[s], G[s], need), (pattern, s))
            if pattern == "map 3":
                assert all(chain[1][l] is None and chain[2][l] is None for l in (4, 5, 6))
                assert all(chain[1][l] is not None for l in range(4))
            if pattern == "discriminator":
                assert chain[0] is None
            if pattern == "generator":
                assert_same(chain, ddev.scale_backward(s, x0, fm[s], G[s], need), ("repeat", s))
    torch.cuda.synchronize()
    assert int(ddev.status[0].item()) == 0


@pytest.mark.gpu
def test_standalone_discriminator_backward_equals_scale_0(ddev, dstate):
    """A stand-alone Discriminator blob (ndisc = 1) with scale 0's weights gives scale 0's gradients bit for bit."""
    one = engine.DiscriminatorDevice("cuda:0", ndisc=1)
    names = ["discriminators.0.%s" % n for n, *_ in LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    one.pack([to(dstate[n + ".weight_v"]) for n in names], [to(dstate[n + ".weight_g"]) for n in names],
             [to(dstate[n + ".bias"]) for n in names])
    y, fm = forward(ddev, 6, 257)
    G = upstream(fm, "generator")
    assert_same(one.scale_backward(0, y, fm[0], G[0], True), ddev.scale_backward(0, y, fm[0], G[0], True), "standalone")


# ------------------------------------------------------------------------------------------------------------------
# 4. weight-norm backward
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_weight_norm_backward_matches_float64(ddev, dstate):
    """disc_wn_backward_kernel on the chain's dW against float64 autograd of torch._weight_norm, all 21 layers, every
    element.  With p_i = dW_i v_i the dot <dW, v> has A2 = sqrt(sum p_i^2); dg = <dW, v> / |v| is held to tau A2 / |v|,
    dv_j = (g / |v|)(dW_j - <dW, v> v_j / |v|^2) to tau (|g| / |v|) sqrt(dW_j^2 + v_j^2 A2^2 / |v|^4), with tau_simt
    of the per-thread strided sum plus the 7-level reduction.  Scale 2 gets the gradient of map 3 only: its layers 4-6
    are passed as None and must come back as None."""
    y, fm = forward(ddev, 6, 257)
    G = upstream(fm, "generator")
    dws = []
    for s in range(3):
        grads = G[s] if s < 2 else [g if l == 3 else None for l, g in enumerate(G[s])]
        dws += ddev.scale_backward(s, scale_input(y, s), fm[s], grads, False)[1]
    names = ["discriminators.%d.%s" % (s, n) for s in range(3) for n, *_ in LAYERS]
    vs = [torch.from_numpy(dstate[n + ".weight_v"]).cuda() for n in names]
    gs = [torch.from_numpy(dstate[n + ".weight_g"]).cuda() for n in names]
    dvs, dgs = ddev.wn_backward(vs, gs, dws)
    worst = 0.0
    for i, (v, g, dw, dv, dg) in enumerate(zip(vs, gs, dws, dvs, dgs)):
        if dw is None:
            assert dv is None and dg is None, names[i]
            continue
        _n, cin, _cout, k, _s, groups, _p = LAYERS[i % 7]
        tau = tau_simt(cdiv(cin // groups * k, 128) + 7)
        v64, g64 = v.double().requires_grad_(True), g.double().requires_grad_(True)
        rdv, rdg = torch.autograd.grad(torch._weight_norm(v64, g64, 0), (v64, g64), dw.double())
        v64, g64, dw64 = v64.detach(), g64.detach(), dw.double()
        nv = v64.square().sum(dim=(1, 2), keepdim=True).sqrt()
        a2 = (dw64 * v64).square().sum(dim=(1, 2), keepdim=True).sqrt()
        r = max(bound_ratio(dg, rdg, a2 / nv, tau),
                bound_ratio(dv, rdv, (g64.abs() / nv) * (dw64.square() + v64.square() * a2.square() / nv ** 4).sqrt(), tau))
        assert r <= 1, (names[i], r)
        worst = max(worst, r)
    assert sum(d is None for d in dvs) == 3
    print("\nweight-norm backward: worst ratio to the bound %.3f" % worst)
