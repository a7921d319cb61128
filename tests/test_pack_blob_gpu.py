"""The pack kernels against float64: every byte of the generator's blob (pack_kernel, csrc/mg_pack.cu) and of the
discriminators' blobs (disc_pack_kernel, csrc/mg_disc.cu), every weight in every copy.

Why.  Every emulation test of the generator and discriminator kernels reads the weights' bf16 halves back out of the
blob, so a wrong weight in the blob is invisible to it: the emulation reads the same wrong value the kernel reads.  A lo
half truncated instead of rounded, an index collision that leaves a slot holding the previous pack or uninitialised
memory, or a hi half rounded half-away instead of to even (seen by bf16 inference alone) all stay far under the goldens'
end-to-end tolerance.  This module holds the blobs to an independent reference instead.

The fold and its bound.  Both pack kernels fold w = g v / ||v|| per norm row of `inner` elements in one CTA of 128
threads: each thread sums n = ceil(inner / 128) squares with fmaf, a 5-level xor-shuffle tree and red[0] + red[1] +
red[2] + red[3] combine the partial sums, then an IEEE sqrtf, an IEEE division g / sqrtf(ss) and one fp32 multiply
scale * v.  Every term of ss is non-negative, so with u = 2^-24 the computed ss is ss (1 + d), |d| <= (n + 8) u to first
order (n roundings in a thread, 5 in the tree, 3 in the final adds); the square root halves that and adds u, the
division and the multiply add u each:
    |w32 - w64| <= (n + 14) u / 2 + O(u^2) |w64|   ->   (ceil(inner / 128) + 15) 2^-25 |w64| + 2^-149   (fold_bound)
with one spare unit for the second-order terms (at most 55 u / 2 here) and one subnormal ulp for folds below the normal
range.  w64 is synth.fold_weight_norm's formula without its final rounding (kernel_model.fold64).  Where v is 0, w32
must be exactly 0.  test_fold_bound_calibration (CPU): a float32 emulation of that exact order stays under 0.5 of the
bound for every layer shape of both blobs, and three value mutants of the fold exceed it by at least MUTANT_X.

The split copies are held bit for bit: hi = bf16_rn(w32), lo = bf16_rn(w32 - hi), w32 the fp32 copy of the same weight
in the same blob, bf16_rn torch's round-to-nearest-even (the kernels' split rounds the fold to fp32 first, then
converts: no contraction reaches lo).  conv_post1 of a discriminator has no fp32 copy: its transposed copy must equal
the forward copy at (ci, co, 4 - tap), each lo is at most half a bf16 ulp of its hi, and |hi + lo - w64| <= 2^-16 |w64|
+ fold_bound + 2^-133 (a bf16 subnormal ulp).  Biases are bit copies; Toeplitz structural zeros and the 4 KiB zero row of
the conv_post1 dgrad launch are +0.0.

Layouts (CPU).  kernel_model restates the generator's fp32 layout next to its tensor-core layouts and lists each copy's
byte range and the padding between regions for both blobs (gen_regions, disc_regions).  The restated map from
(layer, row, column, tap, half) to an offset is injective and, with the declared padding, tiles each blob exactly; the
tensor-core offsets agree with mg_gen_tc_weight_offset (every element of conv_pre, ups.3, the last ResBlock conv and the
fused ups.3 copy, and a seeded sample of the rest) and mg_disc_tc_element, the sizes with the library's.

GPU.  Each blob is packed through the C entry points (mg_gen_pack, mg_msd_pack, mg_disc_pack) into a buffer with GUARD
bytes on both sides, twice, once pre-filled with each of two sentinel bytes: a byte is unwritten exactly when it holds
the first sentinel after the first pack and the second after the second, whatever value a written byte has.  Exactly the
declared padding and the guards are unwritten, and both packs wrote the same bytes.  The states: the seeded synth states
and an edge state (edge_state) whose first rows in every layer have g = 0, negative g, one-hot v (the fold is exactly
+-g) with g on a bf16 rounding tie (1 + 2^-8, even below, where half-away rounding differs; 1 + 3 2^-8, odd below),
one fp32 ulp either side of a tie, g on a tie of the lo half, a subnormal g; v from 2^-80 to 2^50 in one row (folds
down to 2^-130: subnormal); and subnormal v entries in an ordinary row.  Re-pack: the edge state packed over the seeded
one leaves exactly the edge state's blob, and packing it again writes the same bytes.  Production path: after an
optim.Adam step, the next forward's automatic re-pack of a models.Generator and of a models.MultiScaleDiscriminator
holds the fold of the updated parameters, and so does the re-pack after repack() following a write through p.data that
no version counter sees; a stand-alone Discriminator loaded with scale 0's weights packs scale 0's block bit for bit.

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s).  Worst ratio to fold_bound over the folds
in the normal range, seeded / edge state: generator fp32 copies 0.377 / 0.377 (a ResBlock conv; every layer 0.2 - 0.38),
discriminators' grouped convs 0.39 / 0.39, conv_pre 0.29 / 0.29, conv_post2 0.11 / 0.07; conv_post1's split rule
0.458 / 0.500.  The edge state's subnormal folds reach 0.499: their rounding is half of the 2^-149 term.  After an Adam
step and after repack() the re-packed blobs stay at 0.40 (generator) and 0.46 (discriminators).  The calibration's
float32 emulation reaches 0.10 - 0.39 of the bound.  The GPU tests of this file take 49 s (25 s in the tests), most of
it the float64 reference and the host-side reads of the 156 MB of MSD blobs.

Value-only pack mutants, each built once from a modified copy and run once: failing tests of this file, and the older
tests that catch them (of test_resblock_emulation_gpu's and test_disc_emulation_gpu's blob checks, test_generator_gpu and
test_disc_gpu).
    (1) pack_kernel truncates the lo half of resblocks.1.convs1.0: 4 of 11 (both generator states, the re-pack, the
        production path; 22000 - 24000 of 49152 lo halves differ); older: none.
    (2) hi rounded half-away instead of to even (every generator copy): 4 of 11 (seeded: 1 of conv_pre's 286720 hi halves,
        a tie of the random weights; edge: 3, its tie rows); older: none.
    (3) up_weight_index folds the last co-group of ups.0 and ups.1 onto its neighbour: 4 of 11 (1 MiB of ups.0's and
        512 KiB of ups.1's copy unwritten); older: the 7 blob-pattern checks and 24 of test_generator_gpu.
    (4) the fused ups.2 / ups.3 copy has its tap flipped: 4 of 11; older: the 7 blob-pattern checks, 15 of
        test_generator_gpu.
    (5) ss omits red[3]: 4 of 11 (conv_pre up to 3e5 x the bound; rows with inner <= 96 have nothing in warp 3); older:
        the 7 blob-pattern checks, 15 of test_generator_gpu.
    (6) the discriminators' conv_pre fp32 copy written [co][tap]: 7 of 11 (every discriminator test); older: 12 of
        test_disc_gpu.
    (7) the dgrad zero-row memset skipped: 7 of 11 (4 KiB unwritten per blob; the zero row is not +0.0 after a re-pack
        and in the module's blob); older: test_disc_gpu's stand-alone forward and backward.
"""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth
from kernel_model import (BLOB_BYTES, GEN_BLOB_BYTES, GEN_FP32_BYTES, GEN_LAYERS, GEN_TC_START, LAYERS, MUTANT_X,
                          TC_START, ZERO_START, bf16_rn, cdiv, disc_bias_offset, disc_fp32_index, disc_regions, fold64,
                          fold_bound, fp32_blob_bytes, gen_bias_offset, gen_fp32_index, gen_grid, gen_regions,
                          gen_split_copies, lib_offset, post1_offset, slots)

THREADS = 128                 # the pack kernels' CTA: one norm row each
SENTINELS = (0xA5, 0x3C)      # the two fills of a guarded buffer
GUARD = 4096                  # bytes either side of a blob (keeps the 256-byte alignment mg_msd_pack / mg_disc_pack need)
POST1_SPLIT = 2.0 ** -16      # conv_post1: |hi + lo - w32| <= 2^-16 |w32| (two roundings to 8 significant bits)
BF16_SUB = 2.0 ** -133        # a bf16 subnormal ulp


def gen_inner(l):
    _n, kind, cin, cout, k = GEN_LAYERS[l]
    return (cin if kind == "conv" else cout) * k


def disc_inner(l):
    _n, cin, _cout, k, _s, groups, _p = LAYERS[l]
    return cin // groups * k


INNERS = sorted({gen_inner(l) for l in range(len(GEN_LAYERS))} | {disc_inner(l) for l in range(len(LAYERS))})


# ------------------------------------------------------------------------------------------------------------------
# CPU: the fold's bound
# ------------------------------------------------------------------------------------------------------------------
FOLD_MUTANTS = ("one element dropped from ss", "ss rounded to bf16", "one warp's partial dropped")


def fold32(g, v, mutant=None):
    """The pack kernels' fold in float32, in their order, of v [rows, inner] and g [rows]: thread t sums v[j]^2 for j = t,
    t + 128, .. with fmaf (emulated in float64: the square is exact, the add rounded twice), a xor-shuffle tree per warp,
    red[0] + red[1] + red[2] + red[3], g / sqrtf(ss), scale * v."""
    rows, inner = v.shape
    n = cdiv(inner, THREADS)
    vp = np.zeros((rows, n * THREADS), np.float32)
    vp[:, :inner] = v
    if mutant == "one element dropped from ss":
        vp[:, 0] = 0
    vp = vp.reshape(rows, n, THREADS)
    ss = np.zeros((rows, THREADS), np.float32)
    for i in range(n):
        e = vp[:, i].astype(np.float64)
        ss = (e * e + ss.astype(np.float64)).astype(np.float32)
    lanes = ss.reshape(rows, 4, 32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, np.arange(32) ^ o]
    red = lanes[:, :, 0].copy()
    if mutant == "one warp's partial dropped":  # the last warp that holds an element
        red[:, (min(inner, THREADS) - 1) // 32] = 0
    total = ((red[:, 0] + red[:, 1]) + red[:, 2]) + red[:, 3]
    if mutant == "ss rounded to bf16":
        total = bf16_rn(torch.from_numpy(total)).numpy()
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = g.astype(np.float32) / np.sqrt(total)
        return scale[:, None] * v


def bound_ratio(w32, w64, inner):
    with np.errstate(invalid="ignore"):
        r = np.abs(w32.astype(np.float64) - w64) / fold_bound(w64, inner)
    return np.nan_to_num(r, nan=np.inf, posinf=np.inf)


def test_layer_shapes():
    assert INNERS == [15, 96, 128, 164, 192, 224, 256, 384, 560, 768, 2048, 3072, 4096, 5120]


@pytest.mark.parametrize("inner", INNERS)
def test_fold_bound_calibration(inner):
    """A float32 emulation of the kernels' order stays under 0.5 of fold_bound; each fold mutant exceeds it by
    >= MUTANT_X.  Rows: half synth-like U(-1, 1), half with magnitudes 2^U(-10, 10); g of either sign."""
    rs = np.random.RandomState(inner)
    rows = 256
    v = rs.uniform(-1, 1, (rows, inner))
    v[rows // 2:] = np.sign(v[rows // 2:]) * 2.0 ** rs.uniform(-10, 10, (rows - rows // 2, inner))
    v = v.astype(np.float32)
    g = (rs.uniform(0.5, 1.5, rows) * rs.choice((-1, 1), rows)).astype(np.float32)
    w64 = fold64(g, v)
    clean = float(bound_ratio(fold32(g, v), w64, inner).max())
    print("\ninner %4d: float32 emulation %.3f of the bound" % (inner, clean), end="")
    assert clean < 0.5, (inner, clean)
    for m in FOLD_MUTANTS:
        rm = float(bound_ratio(fold32(g, v, m), w64, inner).max())
        print(", %s %.0fx" % (m, rm), end="")
        assert rm >= MUTANT_X, (inner, m, rm)


def test_fold_reference_is_synths():
    """fold64 is synth.fold_weight_norm before its final rounding."""
    st = synth.discriminator_state(5)
    for n, *_ in LAYERS:
        g, v = st["discriminators.1.%s.weight_g" % n], st["discriminators.1.%s.weight_v" % n]
        assert np.array_equal(fold64(g, v).astype(np.float32), synth.fold_weight_norm(g, v)), n


# ------------------------------------------------------------------------------------------------------------------
# CPU: the layouts
# ------------------------------------------------------------------------------------------------------------------
def gen_images():
    """{region name: (byte offsets, bytes per element)} of every element the generator's pack writes."""
    out = {}
    for l, (name, kind, _ci, cout, _k) in enumerate(GEN_LAYERS):
        grid = gen_grid(l)
        out["fp32 " + name] = (gen_fp32_index(l, *grid).ravel(), 4)
        out["bias " + name] = (4 * (gen_bias_offset(l) + np.arange(cout)), 4)
        for copy, off in gen_split_copies(l).items():
            out[copy + " " + name] = (np.concatenate([off(*grid, h).ravel() for h in (0, 1)]), 2)
    return out


def disc_images():
    """{region name: (byte offsets, bytes per element)} of every element of one discriminator's blob: the pack's writes
    and the zero row."""
    out = {}
    for l, (name, cin, cout, k, _s, groups, _p) in enumerate(LAYERS):
        if l != 5:
            co, ci, tap = np.meshgrid(np.arange(cout), np.arange(cin // groups), np.arange(k), indexing="ij")
            out["fp32 " + name] = (disc_fp32_index(l, co, ci, tap).ravel(), 4)
        out["bias " + name] = (4 * (disc_bias_offset(l) + np.arange(cout)), 4)
    for l in (1, 2, 3, 4):
        out["toeplitz " + LAYERS[l][0]] = (slots(l)[0], 2)
    out["tc conv_post1"] = (slots(5)[0], 2)
    out["tcT conv_post1"] = (slots(6)[0], 2)
    out["zero row"] = (ZERO_START + 4 * np.arange(1024), 4)
    return out


def check_tiling(regions, images, total):
    assert regions[0][1] == 0 and regions[-1][2] == total
    for (n0, _s0, e0, _p0), (n1, s1, _e1, _p1) in zip(regions, regions[1:]):
        assert e0 == s1, (n0, n1)
    assert sorted(n for n, _s, _e, p in regions if not p) == sorted(images)
    for name, start, end, pad in regions:
        if pad:
            assert 0 < end - start < 256, (name, start, end)  # alignment padding only
            continue
        off, width = images[name]
        assert (end - start) % width == 0 and off.size == (end - start) // width, (name, off.size, end - start)
        assert np.array_equal(np.sort(off), start + width * np.arange(off.size)), name


def test_generator_layout_tiles_the_blob():
    """The restated map is injective and its image, with the one padding region, tiles the generator's blob."""
    assert engine.lib().mg_gen_packed_bytes() == GEN_BLOB_BYTES
    assert GEN_TC_START == fp32_blob_bytes() and GEN_FP32_BYTES == 4 * (4524290 - 4353)  # all G params but the g scalars
    check_tiling(gen_regions(), gen_images(), GEN_BLOB_BYTES)


def test_discriminator_layout_tiles_the_blob():
    assert engine.lib().mg_disc_packed_bytes() == BLOB_BYTES and engine.lib().mg_msd_packed_bytes() == 3 * BLOB_BYTES
    check_tiling(disc_regions(), disc_images(), BLOB_BYTES)


def test_generator_tc_layout_matches_the_library():
    """mg_gen_tc_weight_offset(front, layer, co, ci, tap, h) on every element of conv_pre, ups.3, the last ResBlock
    conv and the fused ups.3 copy, on 4000 seeded elements of every other copy, and -1 outside each layer."""
    f = lib_offset()
    rs = np.random.RandomState(11)
    for l, (name, kind, *_r) in enumerate(GEN_LAYERS):
        grid = [a.ravel() for a in gen_grid(l)]
        for copy, off in gen_split_copies(l).items():
            n = grid[0].size
            pick = np.arange(n) if l in (0, 4, 28) else rs.choice(n, min(4000, n), replace=False)
            a, b, t = (x[pick] for x in grid)
            co, ci = (a, b) if kind == "conv" else (b, a)
            front, layer = (1, l - 1) if copy == "upf" else (0, l)
            for h in (0, 1):
                want = off(a, b, t, h).tolist()
                got = [f(front, layer, *e, h) for e in zip(co.tolist(), ci.tolist(), t.tolist())]
                if got != want:
                    i = next(i for i, (x, y) in enumerate(zip(got, want)) if x != y)
                    raise AssertionError((name, copy, int(co[i]), int(ci[i]), int(t[i]), h, got[i], want[i]))
    none = 2 ** 64 - 1
    for args in ((0, 29, 0, 0, 0, 0), (0, 5, 256, 0, 0, 0), (0, 28, 0, 0, 3, 0), (0, 1, 0, 512, 0, 0), (0, 0, 0, 80, 0, 0),
                 (1, 4, 0, 0, 0, 0), (1, 3, 0, 64, 0, 0), (1, 2, 0, 0, 4, 0), (0, 5, 0, 0, 0, 2)):
        assert f(*args) == none, args


def test_discriminator_tc_layout_matches_the_library():
    """mg_disc_tc_element at both ends of every tensor-core copy and on 500 seeded elements of each."""
    fn = engine.lib().mg_disc_tc_element
    for copy in range(1, 7):
        off, h, co, ci, tap = slots(copy)
        order = np.argsort(off)
        pick = np.concatenate([order[:8], order[-8:], np.random.RandomState(copy).choice(off.size, 500, replace=False)])
        for j in pick:
            out = [ctypes.c_int(-9) for _ in range(4)]
            got = (fn(int(off[j]), *(ctypes.byref(v) for v in out)),) + tuple(v.value for v in out)
            assert got == (int(h[j]), copy, int(co[j]), int(ci[j]), int(tap[j])), (copy, int(off[j]), got)
    for bad in (0, TC_START - 2, ZERO_START, BLOB_BYTES):
        assert fn(bad, *(ctypes.byref(ctypes.c_int()) for _ in range(4))) == -1, bad


# ------------------------------------------------------------------------------------------------------------------
# the states
# ------------------------------------------------------------------------------------------------------------------
TIE = 1 + 2.0 ** -8  # halfway between the bf16 neighbours 1 (even) and 1 + 2^-7
ONE_HOT_G = {
    "one-hot, g on a tie (even below)": TIE,
    "one-hot, g on a negative tie": -TIE,
    "one-hot, g on a tie (odd below)": 1 + 3 * 2.0 ** -8,
    "one-hot, g one ulp above a tie": TIE + 2.0 ** -23,
    "one-hot, g one ulp below a tie": TIE - 2.0 ** -23,
    "one-hot, g on a tie of the lo half": 1 + 2.0 ** -9 + 2.0 ** -17,
    "one-hot, subnormal g": 5.5 * 2.0 ** -133 + 2.0 ** -149,
}
EDGE_KINDS = ("g = 0", "g < 0", "v from 2^-80 to 2^50", "subnormal v entries") + tuple(ONE_HOT_G)


def edge_rows(v, g, l, rs):
    """Rows 0 .. of one layer's v [rows, inner] and g [rows] (in place): row r gets EDGE_KINDS[(r + l) % len], so layers
    of one row (conv_post, conv_post2) see different kinds."""
    rows, inner = v.shape
    for r in range(min(rows, len(EDGE_KINDS))):
        kind = EDGE_KINDS[(r + l) % len(EDGE_KINDS)]
        if kind == "g = 0":
            g[r] = 0
        elif kind == "g < 0":
            g[r] = -abs(g[r]) - 0.25
        elif kind == "v from 2^-80 to 2^50":  # ||v||^2 <= 5120 2^100: inside fp32; folds down to 2^-130
            e = np.round(np.linspace(-80, 50, inner))
            v[r] = rs.choice((-1, 1), inner) * rs.uniform(1, 2, inner) * 2.0 ** rs.permutation(e)
        elif kind == "subnormal v entries":
            k = rs.choice(inner, max(1, inner // 4), replace=False)
            v[r, k] = rs.choice((-1, 1), k.size) * np.floor(2.0 ** rs.uniform(0, 23, k.size)) * 2.0 ** -149
        else:  # v = +-2^k: ss, its root, g / 2^k and the product are exact (k <= 0 for a subnormal g, so g / 2^k is)
            v[r] = 0
            top = 1 if ONE_HOT_G[kind] < 2.0 ** -126 else 21
            v[r, rs.randint(inner)] = rs.choice((-1, 1)) * 2.0 ** rs.randint(-20, top)
            g[r] = ONE_HOT_G[kind]


def edge_state(state, prefixed_names, seed):
    """A copy of an ordinary state dict with edge rows in every layer (layers numbered in the given order)."""
    rs = np.random.RandomState(seed)
    sd = {k: v.copy() for k, v in state.items()}
    for l, n in enumerate(prefixed_names):
        v, g = sd[n + ".weight_v"], sd[n + ".weight_g"]
        v2 = v.reshape(v.shape[0], -1).astype(np.float64)
        g1 = g.reshape(-1).astype(np.float64)
        edge_rows(v2, g1, l, rs)
        sd[n + ".weight_v"] = v2.astype(np.float32).reshape(v.shape)
        sd[n + ".weight_g"] = g1.astype(np.float32).reshape(g.shape)
    return sd


def test_edge_state_rows_are_what_they_claim():
    """The float32 edge values are exact (ties, subnormals), and the range row's norm stays inside fp32."""
    gs = edge_state(synth.generator_state(1234), [n for n, *_ in GEN_LAYERS], 5)
    for l, (n, *_r) in enumerate(GEN_LAYERS):
        v, g = gs[n + ".weight_v"], gs[n + ".weight_g"].reshape(-1)
        v2 = v.reshape(v.shape[0], -1)
        for r in range(min(v.shape[0], len(EDGE_KINDS))):
            kind = EDGE_KINDS[(r + l) % len(EDGE_KINDS)]
            if kind in ONE_HOT_G:
                assert float(g[r]) == ONE_HOT_G[kind] and np.count_nonzero(v2[r]) == 1, (n, kind)
            if kind == "v from 2^-80 to 2^50":
                assert float((v2[r].astype(np.float64) ** 2).sum()) < 2.0 ** 127, n
            if kind == "subnormal v entries":
                sub = (v2[r] != 0) & (np.abs(v2[r]) < 2.0 ** -126)
                assert sub.sum() >= 1, n
    sub = [x for x in ONE_HOT_G.values() if 0 < x < 2.0 ** -126]
    assert sub and all(float(np.float32(x)) == x for x in ONE_HOT_G.values())


# ------------------------------------------------------------------------------------------------------------------
# GPU: packing into guarded buffers
# ------------------------------------------------------------------------------------------------------------------
BLOBS = ("generator", "msd", "discriminator")


def layer_names(blob):
    if blob == "generator":
        return [n for n, *_ in GEN_LAYERS]
    if blob == "msd":
        return ["discriminators.%d.%s" % (d, n) for d in range(3) for n, *_ in LAYERS]
    return [n for n, *_ in LAYERS]


def blob_bytes(blob):
    return {"generator": GEN_BLOB_BYTES, "msd": 3 * BLOB_BYTES, "discriminator": BLOB_BYTES}[blob]


def scale0(msd_state):
    p = "discriminators.0."
    return {k[len(p):]: v for k, v in msd_state.items() if k.startswith(p)}


_STATES = {}


def state(blob, which):
    """The seeded synth state or its edge state (the stand-alone discriminator: scale 0 of the MSD's)."""
    key = ("generator" if blob == "generator" else "msd", which)
    if key not in _STATES:
        if key[0] == "generator":
            base = synth.generator_state(1234)
        else:
            base = synth.discriminator_state(4321)
        _STATES[key] = base if which == "seeded" else edge_state(base, layer_names(key[0]), 77)
    st = _STATES[key]
    return scale0(st) if blob == "discriminator" else st


def pack_into(blob, st, buf):
    """Packs st through the blob's C entry point into buf[GUARD:GUARD + blob_bytes]."""
    names = layer_names(blob)
    ts = {p: [torch.from_numpy(np.ascontiguousarray(st[n + "." + p])).cuda() for n in names]
          for p in ("weight_v", "weight_g", "bias")}
    arr = lambda xs: (ctypes.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
    fn = getattr(engine.lib(), {"generator": "mg_gen_pack", "msd": "mg_msd_pack", "discriminator": "mg_disc_pack"}[blob])
    assert (buf.data_ptr() + GUARD) % 256 == 0
    engine.check(fn(arr(ts["weight_v"]), arr(ts["weight_g"]), arr(ts["bias"]), buf.data_ptr() + GUARD,
                    torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


def guarded(blob, sentinel):
    return torch.full((2 * GUARD + blob_bytes(blob),), sentinel, dtype=torch.uint8, device="cuda")


def unwritten_mask(blob):
    """What a pack must leave alone, over a guarded buffer: the guards and the declared padding of each blob."""
    m = np.zeros(2 * GUARD + blob_bytes(blob), bool)
    m[:GUARD] = m[GUARD + blob_bytes(blob):] = True
    if blob == "generator":
        copies, regions = [0], gen_regions()
    else:
        copies, regions = [BLOB_BYTES * d for d in range(3 if blob == "msd" else 1)], disc_regions()
    for base in copies:
        for _n, s, e, pad in regions:
            if pad:
                m[GUARD + base + s:GUARD + base + e] = True
    return m


def check_coverage(blob, r1, r2):
    """r1, r2: the buffers after packing into the fills SENTINELS[0] and [1].  Exactly the guards and the padding are
    unwritten, and every written byte is the same in both."""
    a, b = r1.cpu().numpy(), r2.cpu().numpy()
    unwritten = (a == SENTINELS[0]) & (b == SENTINELS[1])
    want = unwritten_mask(blob)
    if not np.array_equal(unwritten, want):
        regions = gen_regions() if blob == "generator" else disc_regions()
        bad = []
        copies = [0] if blob != "msd" else [BLOB_BYTES * d for d in range(3)]
        for d, base in enumerate(copies):
            for name, s, e, pad in regions:
                sl = slice(GUARD + base + s, GUARD + base + e)
                n = int((unwritten[sl] != want[sl]).sum())
                if n:
                    bad.append((d, name, "%d bytes %s" % (n, "written" if pad else "unwritten")))
        for name, sl in (("guard before", slice(0, GUARD)), ("guard after", slice(GUARD + blob_bytes(blob), None))):
            if not unwritten[sl].all():
                bad.append((name, int((~unwritten[sl]).sum())))
        raise AssertionError((blob, bad[:12]))
    assert np.array_equal(a[~want], b[~want]), (blob, "two packs of one state differ")
    return a[GUARD:GUARD + blob_bytes(blob)]


# ------------------------------------------------------------------------------------------------------------------
# GPU: every value
# ------------------------------------------------------------------------------------------------------------------
def split_bits(w32):
    """(hi, lo) bf16 bit patterns of the exact split of fp32 values: hi = bf16_rn(w), lo = bf16_rn(w - hi)."""
    t = torch.from_numpy(np.ascontiguousarray(w32, np.float32))
    hi = t.to(torch.bfloat16)
    lo = (t - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16).numpy().view(np.uint16), lo.view(torch.int16).numpy().view(np.uint16)


def check_fp32(w32, w64, v, inner, what, worst):
    r = bound_ratio(w32, w64, inner)
    sub = np.abs(w64) < 2.0 ** -126  # reported apart: their rounding is half the bound's subnormal ulp
    for key, sel in ((what, ~sub), ("subnormal folds", sub)):
        if sel.any():
            worst[key] = max(worst.get(key, 0.0), float(r[sel].max()))
    assert float(r.max()) <= 1, (what, float(r.max()), np.unravel_index(int(np.argmax(r)), r.shape))
    nz = (v == 0) & (w32 != 0)
    assert not nz.any(), (what, "nonzero weight where v == 0", int(nz.sum()))


def check_halves(got_hi, got_lo, w32, what):
    hi, lo = split_bits(w32)
    for h, got, want in ((0, got_hi, hi), (1, got_lo, lo)):
        bad = got != want
        if bad.any():
            i = np.unravel_index(int(np.argmax(bad)), bad.shape)
            raise AssertionError((what, "hi" if h == 0 else "lo", "%d of %d differ from the exact split" % (bad.sum(), bad.size),
                                  "first at %s: 0x%04x, want 0x%04x (w32 %r)" % (i, got[i], want[i], float(w32[i]))))


def check_bias(f32, offset, b, what):
    got = f32[offset:offset + b.size].view(np.uint32)
    assert np.array_equal(got, np.ascontiguousarray(b, np.float32).view(np.uint32)), (what, "bias is not a bit copy")


_GRIDS = {}


def grid_offsets(key, fn):
    if key not in _GRIDS:
        _GRIDS[key] = fn()
    return _GRIDS[key]


def check_generator_blob(blob, st, worst):
    """Every value of a generator blob (uint8 numpy) against the float64 fold of st."""
    f32, u16 = blob.view(np.float32), blob.view(np.uint16)
    for l, (name, _kind, _ci, _co, _k) in enumerate(GEN_LAYERS):
        v, g = st[name + ".weight_v"], st[name + ".weight_g"]
        grid = grid_offsets(("g", l), lambda: gen_grid(l))
        w32 = f32[grid_offsets(("g32", l), lambda: gen_fp32_index(l, *grid) // 4)]
        check_fp32(w32, fold64(g, v), v, gen_inner(l), "fp32 " + name, worst)
        for copy, off in gen_split_copies(l).items():
            o = grid_offsets(("g16", l, copy), lambda: [off(*grid, h) // 2 for h in (0, 1)])
            check_halves(u16[o[0]], u16[o[1]], w32, (name, copy))
        check_bias(f32, gen_bias_offset(l), st[name + ".bias"], name)


def check_discriminator_blob(blob, st, prefix, worst):
    """Every value of one discriminator's blob (uint8 numpy) against the float64 fold of st's layers prefix + name."""
    f32, u16 = blob.view(np.float32), blob.view(np.uint16)
    for l, (name, cin, cout, k, _s, groups, _p) in enumerate(LAYERS):
        v, g = st[prefix + name + ".weight_v"], st[prefix + name + ".weight_g"]
        w64 = fold64(g, v)
        if l != 5:
            idx = grid_offsets(("d32", l), lambda: disc_fp32_index(l, *np.meshgrid(
                np.arange(cout), np.arange(cin // groups), np.arange(k), indexing="ij")) // 4)
            w32 = f32[idx]
            check_fp32(w32, w64, v, disc_inner(l), "fp32 " + name, worst)
        if 1 <= l <= 4:
            off, h, co, ci, tap = grid_offsets(("slots", l), lambda: slots(l))
            live = h < 2
            wv = w32[co[live], ci[live], tap[live]]
            hi, lo = split_bits(wv)
            want = np.where(h[live] == 0, hi, lo)
            got = u16[off[live] // 2]
            bad = got != want
            assert not bad.any(), (name, "toeplitz", "%d of %d halves differ from the exact split" % (bad.sum(), bad.size))
            assert not u16[off[~live] // 2].any(), (name, "a structural zero is not +0.0")
        if l == 5:
            off, h, co, ci, tap = grid_offsets(("slots", 5), lambda: slots(5))
            fwd = u16[off // 2]
            tr = u16[grid_offsets(("post1T",), lambda: post1_offset(co, ci, tap, h, True)) // 2]
            assert np.array_equal(fwd, tr), (name, "the transposed copy differs from the forward copy at (ci, co, 4 - tap)")
            hi = (fwd[0::2].astype(np.uint32) << 16).view(np.float32).astype(np.float64)  # h is the fastest index of the slots
            lo = (fwd[1::2].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
            e = np.frexp(hi)[1]
            half_ulp = np.where(hi != 0, np.ldexp(1.0, e - 9), 0)
            assert (np.abs(lo) <= half_ulp).all(), (name, "a lo half exceeds half a bf16 ulp of hi")
            w = w64[co[0::2], ci[0::2], tap[0::2]]
            r = np.abs(hi + lo - w) / (POST1_SPLIT * np.abs(w) + fold_bound(w, disc_inner(5)) + BF16_SUB)
            worst["split " + name] = max(worst.get("split " + name, 0.0), float(r.max()))
            assert worst["split " + name] <= 1, (name, worst["split " + name])
        check_bias(f32, disc_bias_offset(l), st[prefix + name + ".bias"], name)
    assert not blob[ZERO_START:BLOB_BYTES].any(), "the dgrad zero row is not +0.0"


def check_values(blob, data, st, worst):
    if blob == "generator":
        check_generator_blob(data, st, worst)
    elif blob == "msd":
        for d in range(3):
            check_discriminator_blob(data[d * BLOB_BYTES:(d + 1) * BLOB_BYTES], st, "discriminators.%d." % d, worst)
    else:
        check_discriminator_blob(data, st, "", worst)


def report(title, worst):
    items = sorted(worst.items(), key=lambda kv: -kv[1])
    print("\n%s: worst ratio to the bound %.3f (%s); per copy: %s" % (
        title, items[0][1], items[0][0], ", ".join("%s %.3f" % kv for kv in items)))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["seeded", "edge"])
@pytest.mark.parametrize("blob", BLOBS)
def test_every_byte_every_weight(blob, which):
    st = state(blob, which)
    r1 = guarded(blob, SENTINELS[0])
    pack_into(blob, st, r1)
    r2 = guarded(blob, SENTINELS[1])
    pack_into(blob, st, r2)
    data = check_coverage(blob, r1, r2)
    worst = {}
    check_values(blob, data, st, worst)
    report("%s %s" % (blob, which), worst)


@pytest.mark.gpu
@pytest.mark.parametrize("blob", BLOBS)
def test_repack_over_another_state(blob):
    """The edge state packed over the seeded one leaves exactly the edge state's blob; a second pack writes the same
    bytes, and the guards and the padding keep their fill."""
    buf = guarded(blob, SENTINELS[0])
    pack_into(blob, state(blob, "seeded"), buf)
    pack_into(blob, state(blob, "edge"), buf)
    first = buf.clone()
    pack_into(blob, state(blob, "edge"), buf)
    assert torch.equal(buf, first), (blob, "a second pack of one state changed the blob")
    keep = torch.from_numpy(unwritten_mask(blob)).cuda()
    assert bool((buf[keep] == SENTINELS[0]).all()), (blob, "a guard or the padding was written")
    worst = {}
    check_values(blob, buf[GUARD:GUARD + blob_bytes(blob)].cpu().numpy(), state(blob, "edge"), worst)


def module_state(m):
    return {k: t.detach().cpu().numpy() for k, t in m.state_dict().items()}


def packed_bytes(dev):
    return dev.packed.view(torch.uint8).cpu().numpy()


def step_and_write(module, forward):
    """An Adam step (the next forward re-packs), then a write through p.data that no version counter sees and repack();
    yields after each re-packing forward."""
    gen = torch.Generator(device="cuda").manual_seed(3)
    opt = torch.optim.Adam(module.parameters(), lr=1e-2)
    for p in module.parameters():
        p.grad = torch.randn(p.shape, generator=gen, device="cuda")
    opt.step()
    with torch.no_grad():
        forward()
    yield "after an Adam step"
    for p in module.parameters():
        p.data.add_(torch.randn(p.shape, generator=gen, device="cuda"), alpha=1e-2)
    module.repack()
    with torch.no_grad():
        forward()
    yield "after a write through p.data and repack()"


@pytest.mark.gpu
def test_generator_repacks_the_updated_parameters():
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda()
    mel = torch.from_numpy(synth.mel_input(1, 4, 3)).cuda()
    with torch.no_grad():
        g(mel)
    before = packed_bytes(g._dev)
    for when in step_and_write(g, lambda: g(mel)):
        data = packed_bytes(g._dev)
        assert not np.array_equal(data, before), when
        worst = {}
        check_generator_blob(data, module_state(g), worst)
        report("Generator " + when, worst)
        before = data


@pytest.mark.gpu
def test_discriminators_repack_the_updated_parameters():
    msd = models.MultiScaleDiscriminator()
    msd.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(4321).items()})
    msd = msd.cuda()
    y = torch.from_numpy(synth.audio_input(1, 2048, 5)).cuda()
    with torch.no_grad():
        msd(y, y)
    before = packed_bytes(msd._dev)
    for when in step_and_write(msd, lambda: msd(y, y)):
        data = packed_bytes(msd._dev)
        assert not np.array_equal(data, before), when
        worst = {}
        check_values("msd", data, module_state(msd), worst)
        report("MultiScaleDiscriminator " + when, worst)
        before = data
    d = models.Discriminator()
    d.load_state_dict(msd.discriminators[0].state_dict())
    d = d.cuda()
    with torch.no_grad():
        d(y)
    written = ~unwritten_mask("discriminator")[GUARD:GUARD + BLOB_BYTES]  # (the padding is never written)
    own, block = packed_bytes(d._dev), before[:BLOB_BYTES]
    differ = [n for n, s, e, pad in disc_regions() if not pad and not np.array_equal(own[s:e], block[s:e])]
    assert np.array_equal(own[written], block[written]), ("the stand-alone blob differs from scale 0's", differ)
