"""Every discriminator forward kernel at each tile and packed-item border of its launch geometry, against float64; the
fp32 SIMT grouped convs (MG_DISC_GROUP=simt) at the same lengths.

The input lengths are derived from the launch geometry (mirrored from the kernels' sources, here and in kernel_model)
rather than picked by hand: for each border length of a kernel, find_L gives the shortest input that puts it at that
layer.  Around it:
  * disc_group_tc_kernel (grouped_convs.0-2): ni = 134 // (ceil(Lout/2) + 6) items share a CTA as virtual rows while two
    fit (Lout <= 122); from Lout = 123 each CTA is one 256-output tile of one item; odd Lout takes the scalar store;
  * disc_group4_tc_kernel (grouped_convs.3): ni = 133 // (ceil(L/8) + 5) items per tile, one single-item tile up to
    L = 1024, ceil(L/1024) tiles per item beyond; stores masked per output at 8 kb + e < L;
  * conv_rows_tc_kernel<Post1Cfg> (conv_post1): 128 virtual rows at a pitch of L + 2 per item;
  * disc_pre_kernel<scale>: 256-output tiles with a 7-sample halo, the AvgPool chain evaluated inside the load (lengths at
    each scale, from the shortest and the longest input that give them, so the pooling windows end on both parities);
  * disc_post2_kernel: 8 positions per CTA.
Packed geometries run Bt = 1, ni - 1, ni, ni + 1 and 2 ni + 1 (a part-filled last CTA, an item that starts a new one),
the others Bt = 1 and 3.  test_border_cases_sit_on_the_kernel_borders checks on the CPU that the cases really contain
each claimed situation.

Each call goes through the C ABI into feature maps filled with NaN, so a store that a mask skips shows up as a
non-finite element instead of a stale value the allocator handed back.  Layer l is held to float64 on the map the engine
returned for layer l - 1 (layer 0: the float64 AvgPool chain of y), with the element-wise bound of
test_layer_isolation_gpu, |y - y64| <= tau A2 + 2^-20 |y64|:
  * tensor-core layers (grouped convs, conv_post1): TAU = 2^-12, the 3-pass split-bf16 bound;
  * fp32 SIMT layers: tau_simt(n) of test_disc_backward_isolation_gpu with n the roundings one output goes through:
    conv_pre 15 products + 3 pooling adds per AvgPool level (15 / 18 / 21 at scales 0 / 1 / 2), conv_post2 96 products
    per thread + 2 shuffle adds + the 8-partial combine (106), the SIMT grouped convs 4 ci x 41 taps (164).
Every item of every batch is bit-identical to its own Bt = 1 call, a repeated call is bit-identical, and a stand-alone
Discriminator (mg_disc_forward) with scale 0's weights gives scale 0's maps bit for bit.

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s).  Worst ratio to the bound over all 103
border lengths, scale 0 / 1 / 2:
    conv_pre           disc_pre_kernel                 0.182 / 0.281 / 0.216
    grouped_convs.0-2  disc_group_tc_kernel            0.114 / 0.108 / 0.116,  0.109 / 0.118 / 0.096,
                                                       0.121 / 0.115 / 0.105
    grouped_convs.3    disc_group4_tc_kernel           0.108 / 0.111 / 0.113
    conv_post1         conv_rows_tc_kernel<Post1Cfg>   0.327 / 0.321 / 0.342
    conv_post2         disc_post2_kernel               0.098 / 0.091 / 0.080
  MG_DISC_GROUP=simt, 107 lengths:
    grouped_convs.0-3  disc_group_kernel               0.224 / 0.207 / 0.197,  0.275 / 0.259 / 0.221,
                                                       0.279 / 0.270 / 0.239,  0.264 / 0.400 / 0.239
The GPU tests of this file take 60 - 70 s.  Value-only changes to the kernels each fail most of the lengths: the bias
of the last packed item dropped in disc_group_tc_kernel (79 of 103, first caught by the item bit-identity), the lone last
output of an odd Lout left unstored (100, by the NaN fill), the last lane of disc_group4_tc_kernel left unstored when
L % 8 != 0 (90, by the NaN fill), the last sample dropped from the pooling windows of disc_pre_kernel (103, by the
float64 bound of conv_pre at scale 1).
"""
import math

import pytest
import torch

from melgan_multi_b200 import engine, synth
from kernel_model import ddev, dstate  # noqa: F401 (fixtures)
from kernel_model import (GROUP4_TARGETS, GROUP_TARGETS, LANE4, POST1_PAD, POST1_ROWS, SIMT_N, TAU, batches,
                          conv_bound_ratio, folded64, group4_plan, group_tc_plan, post1_lengths, post1_straddles, tau_simt)

LAYERS = synth.DISCRIMINATOR_LAYERS
GROUP_BT_LIMIT = 65535  # mg_msd_forward / mg_disc_forward (csrc/mg_api.cu): items go on grid.y / grid.z

# launch geometry of the forward kernels
TILE = 256                       # dg::TILE (csrc/mg_disc_tc.cu): outputs per disc_group_tc_kernel CTA, 128 rows x 2 parities
PRE_TILE, PRE_HALO = 256, 7      # disc_pre_kernel (csrc/mg_disc.cu): outputs per CTA, halo on each side
POST2_TILE = 8                   # disc_post2_kernel (csrc/mg_disc.cu): positions per CTA
SIMT_TILE = 128                  # disc_group_kernel (csrc/mg_disc.cu): outputs per CTA; input windows from 4 (t0 - 5)
                                 # (stride 4) and t0 - 20 (stride 1)

N_PRE = (15, 18, 21)             # conv_pre: 15 products + 3 adds per AvgPool level, per scale
N_POST2 = 32 * 3 + 2 + 8         # conv_post2: per-thread products, shuffle adds, combine of the 8 warp partials
N_SIMT_GROUP = 4 * 41            # disc_group_kernel: input channels x taps, one fmaf chain


# ------------------------------------------------------------------------------------------------------------------
# geometry, on the CPU
# ------------------------------------------------------------------------------------------------------------------
def scale_length(L, s):
    """Input length of discriminator s: y, AvgPool1d(4, 2, pad 2)(y), then AvgPool1d(4, 4, pad 2) of that."""
    if s >= 1:
        L = L // 2 + 1
    if s == 2:
        L = L // 4 + 1
    return L


def msd_lengths(L):
    """Feature-map lengths [3][7] for an input of L samples (the conv output-length formula, layer by layer)."""
    out = []
    for s in range(3):
        n, row = scale_length(L, s), []
        for _name, _cin, _cout, k, stride, _g, pad in LAYERS:
            n = (n + 2 * pad - k) // stride + 1
            row.append(n)
        out.append(row)
    return out


def find_L(scale, layer, target):
    """The smallest input length that gives `target` outputs at (scale, layer), None if none does (lengths are
    non-decreasing in L, so a bisection finds it)."""
    at = lambda L: msd_lengths(L)[scale][layer]
    hi = 1
    while at(hi) < target:
        hi *= 2
    lo = 1
    while lo < hi:
        mid = (lo + hi) // 2
        lo, hi = (mid + 1, hi) if at(mid) < target else (lo, mid)
    return lo if at(lo) == target else None


PRE_TARGETS = (1, 2, 3, 4, 5, 255, 256, 257, 511, 512, 513)                     # Ls of conv_pre, every scale
POST2_TARGETS = (1, 2, 7, 8, 9, 15, 16, 17)                                      # L of conv_post2
SIMT_TARGETS = GROUP_TARGETS + (SIMT_TILE - 1, SIMT_TILE, SIMT_TILE + 1)         # Lout of the SIMT grouped convs


def shortest(layer, target):
    """The smallest L over the three scales that gives `target` at `layer`."""
    return min(L for L in (find_L(s, layer, target) for s in range(3)) if L is not None)


def border_cases():
    """{L: set of Bt} of the tensor-core sweep."""
    cases = {}
    add = lambda L, bts: cases.setdefault(L, set()).update(bts)
    for layer in (1, 2, 3):
        for T in GROUP_TARGETS:
            add(shortest(layer, T), batches(group_tc_plan(T)[1]))
    for T in GROUP4_TARGETS:
        add(shortest(4, T), batches(group4_plan(T)[0]))
    for T in post1_lengths():
        add(shortest(5, T), {1, 3})
    for T in POST2_TARGETS:
        add(shortest(6, T), {1, 3})
    for s in range(3):
        for T in PRE_TARGETS:  # the shortest and the longest input of this Ls, and the shortest of the other parity
            first, last = find_L(s, 0, T), find_L(s, 0, T + 1) - 1
            for L in {first, min(first + 1, last), last}:
                add(L, {1, 3})
    return cases


def simt_cases():
    """{L: Bt} of the SIMT grouped-conv sweep: the tensor-core sweep's lengths and largest batch, plus the SIMT tile
    borders at every grouped layer."""
    cases = {L: max(bts) for L, bts in border_cases().items()}
    for layer in (1, 2, 3, 4):
        for T in SIMT_TARGETS:
            cases.setdefault(shortest(layer, T), 3)
    return cases


CASES = border_cases()
SIMT_CASES = simt_cases()


def geometry(L, Bt):
    """Every (scale, layer) situation of one call, as a list of dicts."""
    out = []
    for s, row in enumerate(msd_lengths(L)):
        for l in (1, 2, 3):
            rp, ni = group_tc_plan(row[l])
            out.append(dict(kind="group_tc", s=s, l=l, Lout=row[l], ni=ni, Bt=Bt, L=L))
        ni, segs = group4_plan(row[4])
        out.append(dict(kind="group4", s=s, l=4, Lout=row[4], ni=ni, segs=segs, Bt=Bt, L=L))
        out.append(dict(kind="post1", s=s, l=5, Lout=row[5], Bt=Bt, L=L))
        out.append(dict(kind="post2", s=s, l=6, Lout=row[6], Bt=Bt, L=L))
        out.append(dict(kind="pre", s=s, l=0, Lout=row[0], Bt=Bt, L=L))
    return out


def test_msd_lengths_mirror_the_library():
    for L in list(range(1, 5001)) + [8192, 7745, 7809, 16385, 31169, 65473, 65537, 131073, 1 << 20]:
        assert msd_lengths(L) == engine.msd_lengths(L), L


def test_find_L_gives_the_shortest_input():
    for s in range(3):
        for l in range(7):
            for T in (1, 2, 17, 122, 123, 489, 1025):
                L = find_L(s, l, T)
                assert L is not None and msd_lengths(L)[s][l] == T and (L == 1 or msd_lengths(L - 1)[s][l] < T), (s, l, T)
    assert [shortest(3, 122), shortest(3, 123), shortest(3, 257)] == [7745, 7809, 16385]
    assert [shortest(4, 488), shortest(4, 1024), shortest(4, 1025)] == [31169, 65473, 65537]
    assert find_L(1, 0, 256) == 510 and find_L(2, 0, 256) == 2038


def test_border_cases_sit_on_the_kernel_borders():
    """Each situation the module docstring names is in the sweep (CPU: the geometry of the launches)."""
    geo = [g for L, bts in CASES.items() for Bt in bts for g in geometry(L, Bt)]
    grp = [g for g in geo if g["kind"] == "group_tc"]
    g4 = [g for g in geo if g["kind"] == "group4"]
    # grouped_convs.0-2: the last packed length (ni = 2) and the first single-item tile, at each of the three layers
    last = max(T for T in range(1, 4 * TILE) if group_tc_plan(T)[1] > 1)
    assert (last, group_tc_plan(last)[1], group_tc_plan(last + 1)[1]) == (122, 2, 1)
    for l in (1, 2, 3):
        at = {g["Lout"] for g in grp if g["l"] == l}
        assert {1, 2, 3, 13, 14, last, last + 1, TILE - 1, TILE, TILE + 1, 2 * TILE, 2 * TILE + 1} <= at, (l, sorted(at))
    assert {group_tc_plan(T)[1] for T in (1, 2, 3, 13, 14, 121, 122)} == {19, 16, 10, 2}
    # a part-filled last CTA with an item that starts a new one, in every packed geometry of a target
    for T in GROUP_TARGETS:
        ni = group_tc_plan(T)[1]
        if ni > 1:
            assert any(g["Lout"] == T and g["Bt"] > ni and g["Bt"] % ni for g in grp), T
    for T in GROUP4_TARGETS:
        ni = group4_plan(T)[0]
        if ni > 1:
            assert any(g["Lout"] == T and g["Bt"] > ni and g["Bt"] % ni for g in g4), T
    # odd Lout (scalar store path) packed and in 256-output tiles; Lout % 256 != 0 in tiles
    assert any(g["Lout"] % 2 and g["ni"] > 1 for g in grp) and any(g["Lout"] % 2 and g["ni"] == 1 for g in grp)
    assert any(g["ni"] == 1 and g["Lout"] % TILE == 1 for g in grp)
    # grouped_convs.3: ni 22 -> 19, the last ni = 2, the single tiles, more than one tile per item, L % 8 != 0 in each
    assert [group4_plan(L)[0] for L in (8, 9, 488, 489, 1024)] == [22, 19, 2, 1, 1]
    assert group4_plan(1024)[1] == 1 and group4_plan(1025)[1] == 2
    assert {1, 7, 8, 9, 487, 488, 489, 1023, 1024, 1025, 2048, 2049} <= {g["Lout"] for g in g4}
    assert any(g["segs"] > 1 and g["Bt"] > 1 for g in g4)
    for cond in (lambda g: g["ni"] > 1, lambda g: g["ni"] == 1 and g["segs"] == 1, lambda g: g["segs"] > 1):
        assert any(cond(g) and g["Lout"] % LANE4 for g in g4)
    # conv_post1: an item's L + 2 rows straddle two 128-row tiles; items that tile the rows exactly
    p1 = [g for g in geo if g["kind"] == "post1"]
    assert any(post1_straddles(g["Bt"], g["Lout"]) for g in p1)
    assert any(POST1_ROWS % (g["Lout"] + POST1_PAD) == 0 and g["Bt"] * (g["Lout"] + POST1_PAD) > POST1_ROWS for g in p1)
    # conv_pre: shorter than the taps, and each side of the first two tile borders, at every scale; the pooled scales
    # from inputs of both parities for one Ls
    pre = [g for g in geo if g["kind"] == "pre"]
    for s in range(3):
        at = {g["Lout"] for g in pre if g["s"] == s}
        assert {1, 5, PRE_TILE - 1, PRE_TILE, PRE_TILE + 1, 2 * PRE_TILE - 1, 2 * PRE_TILE, 2 * PRE_TILE + 1} <= at, s
        if s:
            for T in (PRE_TILE, 2 * PRE_TILE + 1):
                assert {g["L"] % 2 for g in pre if g["s"] == s and g["Lout"] == T} == {0, 1}, (s, T)
    # conv_post2: each side of the 8-position CTA
    at = {g["Lout"] for g in geo if g["kind"] == "post2"}
    assert {1, POST2_TILE - 1, POST2_TILE, POST2_TILE + 1, 2 * POST2_TILE, 2 * POST2_TILE + 1} <= at
    # the SIMT grouped convs: each side of the 128-output tile, at every grouped layer
    simt = {(s, l): set() for s in range(3) for l in (1, 2, 3, 4)}
    for L in SIMT_CASES:
        for s, row in enumerate(msd_lengths(L)):
            for l in (1, 2, 3, 4):
                simt[(s, l)].add(row[l])
    for l in (1, 2, 3, 4):
        assert {SIMT_TILE - 1, SIMT_TILE, SIMT_TILE + 1} <= set().union(*(simt[(s, l)] for s in range(3))), l


def test_simt_n_within_the_calibrated_range():
    """Every n the GPU tests use lies inside the range test_tau_calibration_on_emulated_fp32_sums calibrates."""
    for n in N_PRE + (N_POST2, N_SIMT_GROUP):
        assert min(SIMT_N) <= n <= max(SIMT_N), n


def test_forward_refuses_batches_beyond_the_grid():
    """Bt > 65535 is refused with MG_ERR_INVALID_ARGUMENT before any CUDA call (fake pointers: nothing is touched)."""
    L = engine.lib()
    p = 256
    maps = engine._ptr_array([p] * 21)
    for fn, name in ((L.mg_msd_forward, b"mg_msd_forward"), (L.mg_disc_forward, b"mg_disc_forward")):
        assert fn(p, p, GROUP_BT_LIMIT + 1, 64, maps, p, None) == -1
        msg = L.mg_last_error_string()
        assert name in msg and b"65535" in msg, msg
        assert fn(p, p, 1 << 30, 8192, maps, p, None) == -1


# ------------------------------------------------------------------------------------------------------------------
# on the GPU
# ------------------------------------------------------------------------------------------------------------------
KERNELS = {"tc": ("disc_pre_kernel", "disc_group_tc_kernel", "disc_group_tc_kernel", "disc_group_tc_kernel",
                  "disc_group4_tc_kernel", "conv_rows_tc_kernel<Post1Cfg>", "disc_post2_kernel"),
           "simt": (None, "disc_group_kernel<16, 4>", "disc_group_kernel<16, 4>", "disc_group_kernel<16, 4>",
                    "disc_group_kernel<4, 1>", None, None)}


@pytest.fixture(scope="module")
def disc0(dstate):
    """A stand-alone Discriminator (mg_disc_pack) with scale 0's weights."""
    one = engine.DiscriminatorDevice("cuda:0", ndisc=1)
    names = ["discriminators.0.%s" % n for n, *_ in LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    one.pack([to(dstate[n + ".weight_v"]) for n in names], [to(dstate[n + ".weight_g"]) for n in names],
             [to(dstate[n + ".bias"]) for n in names])
    return one


@pytest.fixture(scope="module")
def worst():
    """{(path, layer, scale): worst ratio to the bound}, printed when the module's tests are done."""
    w = {}
    yield w
    lines = ["\nworst ratio to the bound over the border lengths, scale 0 / 1 / 2:"]
    for path in ("tc", "simt"):
        for l in range(7):
            r = [w.get((path, l, s)) for s in range(3)]
            if any(v is not None for v in r):
                lines.append("  %-16s %-30s " % (LAYERS[l][0], KERNELS[path][l]) +
                             " / ".join("-" if v is None else "%.3f" % v for v in r))
    print("\n".join(lines))


def forward(dev, y):
    """dev's forward (mg_msd_forward, or mg_disc_forward for a stand-alone Discriminator) through the C ABI into maps
    filled with NaN; every element must come back finite."""
    Bt, _, L = y.shape
    lens, nd = msd_lengths(L), dev.ndisc
    maps = [[torch.full((Bt, engine.D_CHANNELS[l], lens[s][l]), math.nan, device=y.device) for l in range(7)]
            for s in range(nd)]
    lib = engine.lib()
    stream = torch.cuda.current_stream().cuda_stream
    fn = lib.mg_msd_forward if nd == 3 else lib.mg_disc_forward
    engine.check(fn(dev.packed.data_ptr(), y.data_ptr(), Bt, L, engine._ptr_array([m.data_ptr() for sc in maps for m in sc]),
                    dev.status.data_ptr(), stream))
    engine.check(lib.mg_msd_check_status(dev.status.data_ptr(), stream))
    for s in range(nd):
        for l in range(7):
            assert bool(torch.isfinite(maps[s][l]).all()), ("an output element was not written", Bt, L, s, LAYERS[l][0])
    return maps


def assert_same(a, b, what):
    for s, (sa, sb) in enumerate(zip(a, b)):
        for l, (x, y) in enumerate(zip(sa, sb)):
            assert torch.equal(x, y), (what, s, LAYERS[l][0], float((x - y).abs().max()))


def audio(Bt, L):
    """Bt rows of U(-1, 1) audio; row i does not depend on Bt."""
    return torch.from_numpy(synth.audio_input(Bt, L, L)).cuda()


def check_layers(dstate, y, maps, layers, taus):
    """{(layer, scale): worst ratio to the bound} of each layer on its own input: the map the engine returned for the
    layer before it, the float64 AvgPool chain of y for layer 0.  taus(layer, scale) -> tau."""
    out = {}
    x0 = y.double()
    for s in range(3):
        if s:
            x0 = torch.nn.functional.avg_pool1d(x0, 4, 2 if s == 1 else 4, padding=2)
        for l in layers:
            name, _cin, _cout, _k, stride, groups, pad = LAYERS[l]
            w, b = folded64(dstate, "discriminators.%d.%s" % (s, name))
            x = x0 if l == 0 else maps[s][l - 1].double()
            r = conv_bound_ratio(maps[s][l], x, w, b, stride, pad, groups, lrelu=l < 6, tau=taus(l, s))
            assert r <= 1, (y.shape, s, name, r)
            out[(l, s)] = r
    return out


def tc_tau(l, s):
    return tau_simt(N_PRE[s]) if l == 0 else tau_simt(N_POST2) if l == 6 else TAU


@pytest.mark.gpu
@pytest.mark.parametrize("L", sorted(CASES))
def test_forward_at_borders(ddev, dstate, disc0, worst, monkeypatch, L):
    """At each border length: every batch of the case written in full, each item bit-identical to its own Bt = 1 call, a
    repeated call and the stand-alone Discriminator bit-identical, every layer of the largest batch within its bound."""
    monkeypatch.delenv("MG_DISC_GROUP", raising=False)
    bts = sorted(CASES[L])
    assert bts[0] == 1 and len(bts) > 1
    y = audio(bts[-1], L)
    singles = [forward(ddev, y[i:i + 1]) for i in range(bts[-1])]
    for Bt in bts[1:]:
        full = forward(ddev, y[:Bt])
        for i in range(Bt):
            assert_same([[m[i:i + 1] for m in sc] for sc in full], singles[i], ("item", i, "of", Bt, L))
    assert_same(full, forward(ddev, y), ("repeat", L))
    assert_same(full[:1], forward(disc0, y), ("stand-alone Discriminator", L))
    for (l, s), r in check_layers(dstate, y, full, range(7), tc_tau).items():
        worst[("tc", l, s)] = max(worst.get(("tc", l, s), 0.0), r)


@pytest.mark.gpu
@pytest.mark.parametrize("L", sorted(SIMT_CASES))
def test_simt_grouped_convs_at_borders(ddev, dstate, worst, monkeypatch, L):
    """MG_DISC_GROUP=simt (read at every forward): the fp32 SIMT grouped convs, every output written, each within
    tau_simt(164) of float64 on its own input."""
    monkeypatch.setenv("MG_DISC_GROUP", "simt")
    y = audio(SIMT_CASES[L], L)
    maps = forward(ddev, y)
    for (l, s), r in check_layers(dstate, y, maps, (1, 2, 3, 4), lambda l, s: tau_simt(N_SIMT_GROUP)).items():
        worst[("simt", l, s)] = max(worst.get(("simt", l, s), 0.0), r)
