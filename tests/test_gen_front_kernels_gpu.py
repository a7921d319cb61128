"""conv_pre and the four ConvTranspose kernels against a float64 emulation of their OWN arithmetic, at every tile and item
border of their launch geometry, on uniform and ragged batches, at fp32 and bf16; the default chain's ResBlock kernels on
the same ragged tables.

Emulation.  Each kernel multiplies bf16 operands exactly and accumulates in fp32.  The reference here is that arithmetic
with the accumulation in float64:
  * x is split into hi = bf16_rn(x), lo = bf16_rn(x - hi), as split2_bf16 does (csrc/mg_tc.cuh); the ConvTs split
    LeakyReLU(x) = fmaxf(x, x * 0.01f), taken in fp32;
  * the weights' hi and lo halves are read back from the packed blob (at the layout kernel_model restates), not re-split from a
    float64 fold: a few dozen of the ~1 M folded fp32 weights sit within an ulp of a bf16 rounding midpoint, and a
    re-split would round them the other way, a 2^-8 error on that product;
  * fp32 runs the passes (xh, wh) + (xl, wh) + (xh, wl), bf16 (up0, up1) the first alone; the bias is added exactly.
Bound, element-wise:

    |y - y_emu| <= TAU_E * A2 + 2^-22 * |y_emu|,      A2 = sqrt(conv64(x^2, w^2))   (test_layer_isolation_gpu)

so what is left is the fp32 accumulation.  The 2^-12 bound of test_layer_isolation_gpu, against the exact product, has to
leave room for the split itself, so a defect that touches only lo halves, which carry about 2^-8 of each value -- a stale
lo half of a ring slot, an unwritten lo half of some rows, a wrong lo k-panel offset at a tile edge -- lands close to it:
zeroing the lo half of one k-panel of one row gives 1.3 - 3.4x that bound (test_tau_calibration prints both).
test_tau_calibration (CPU) holds TAU_E to both sides: a float32-accumulated emulation stays under 0.5 of the bound at every
(Cin, K, S) here (at most 0.28 of a 2^-16 bound), and each value-only mutant of the operands exceeds it by >= 4x (>= 20x at
2^-16) -- the lo half of one k-panel of one row zeroed, one pass dropped for one k-panel, LeakyReLU applied to the halves
after the split, and (bf16) the hi operand truncated instead of rounded (at fp32 the lo half absorbs most of a truncated
hi).  On the H100 the MMAs' fp32 accumulation reached 1.43 x 2^-16 (up0 at fp32, as far from the tile borders and item
ends as at them), so TAU_E = 3 x 2^-16, about twice that.

Geometry (from the strings the library reports, so a re-tiling moves the tested lengths with it):
  * conv_pre  conv_rows_tc_kernel<ConvCfg<80,512,7,ROWS,N>>: tiles of ROWS virtual rows, each item's positions followed by
    PAD = 3 zero rows; one CTA per (tile, group of N output channels);
  * up0       convt_tc_kernel<UpCfg<0,ROWS,NG>>: tiles of ROWS input rows, one zero row after each item; CTAs per (tile, NG);
  * up1       convt_resident_tc_kernel<UpCfg<1,ROWS,NG>>: the same rows, one CTA per tile looping over the channel groups;
  * up2, up3  convt_stream_tc_kernel<StreamCfg<S,ROWS,MAXSEG,NSX>>: persistent CTAs walking tiles of ROWS rows.
Uniform batches put an item's end, and the end of its zero rows, one row before, on and after tile borders 1 - 3, with
B = 1, 2, 3; plus a short last tile, batches that leave the last CTA part-filled and more CTAs than two waves of the SMs.
Ragged tables (GeneratorDevice.chain_kernel, lengths in the kernel's input units): item ends at every offset of a tile,
items of 1 and 2 positions (a conv_pre tap reaches across a whole item) with many items per tile, and 256 runs that do not
merge.  Inputs hold NaN past every length; outputs are NaN-filled (a payload no kernel writes) with a guard after the
buffer.  Per item: the valid outputs are within the bound, every output past them still holds the fill (kernel 7:
exactly 0.0, its documented zero tail), the guard is untouched, and the item equals its own uniform call bit for bit.  The
ResBlock kernels (2, 4, 6, 7) get the same tables at both precisions -- NaN, guard and own-call checks, and at fp32 each
item against the float64 layers at ROW_TOL.  conv_pre and up2 keep three passes under bf16: bit-identical to fp32.

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s): worst ratio to the bound at TAU_E = 3 x 2^-16,
uniform batches (within 2 rows of a tile border or item end / elsewhere) and ragged tables:
    conv_pre  fp32  0.259 / 0.276   0.286          up2  fp32  0.130 / 0.153   0.149
    up0       fp32  0.452 / 0.461   0.477          up3  fp32  0.071 / 0.084     -
    up0       bf16  0.171 / 0.171   0.186
    up1       fp32  0.237 / 0.277   0.254
    up1       bf16  0.091 / 0.100   0.095
ResBlock chain kernels on the ragged tables at fp32, worst per-row error: 2 res0 2.5e-5, 4 res1 1.7e-5, 6 res2 1.2e-5,
7 up3+res3+post 2.1e-5.  The GPU tests of this file take about 15 s.  Value-only mutants of the kernels, failing
(B, L) cases / ragged items of the test that catches them:
    up0's converter stores lo = 0 for k-panel 1 of A row 0 (the row carried in from the tile before)    19 / 29, 194 / 445
    conv_pre's tail_rows (A rows 128 - 133) store lo = 0                                                 31 / 40, 262 / 509
    convt_store adds the bias twice to the hi float4 of an item's last row       up0, up1 at fp32 and bf16: 29 / 29, 445 / 445
    Bf16<UpCfg<1>>'s converter stores row 1's first k-panel hi truncated, not rounded                    28 / 29, 442 / 445
The generator's other GPU tests catch each of these too (test_tc_gpu's oracle comparisons, at 1e-4 of the output's max,
the first three; test_bf16_inference_gpu's ragged bit-identity the fourth).
"""
import ctypes
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine
from kernel_model import g64, gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import (MUTANT_X, REL_E, ROW_TOL, SHAPE, TAU_E, bf16_of, bf16_rn, fill_faults, gen_weight_offset,
                          lib_offset, lrelu32, nan_buffer, row_errors, split_passes, split_rn, up_tc_bytes, valid_mask,
                          weight_grid)

OLD_TAU, OLD_REL = 2.0 ** -12, 2.0 ** -20  # test_layer_isolation_gpu, against the exact product
NUM_SMS = 132  # kNumSMs (csrc/mg_common.cuh)

KERNELS = ("pre", "up0", "up1", "up2", "up3")
LAYER = {"pre": 0, "up0": 1, "up1": 2, "up2": 3, "up3": 4}
CHAIN = {"pre": 0, "up0": 1, "up1": 3, "up2": 5}  # index in the default chain (up3 runs fused into kernel 7)
RES_TABLES = {2: "up0", 4: "up1", 6: "up2", 7: "up3"}  # ResBlock chain kernel -> whose ragged tables it runs
RES_STAGE = {2: 0, 4: 1, 6: 2, 7: 3}
# (B, L) with more CTAs than two waves of the SMs (persistent kernels: more than two passes of the grid)
WAVES = {"pre": (64, 200), "up0": (40, 64), "up1": (64, 300), "up2": (40, 1000), "up3": (40, 1000)}


# ------------------------------------------------------------------------------------------------------------------
# geometry (pure functions: tested without a GPU)
# ------------------------------------------------------------------------------------------------------------------
def parse(kernel, name):
    """The tile geometry of a configuration string: ROWS per tile, PAD zero rows per item, CTAs per tile, persistent."""
    if kernel == "pre":
        m = re.fullmatch(r"conv_rows_tc_kernel<ConvCfg<80,512,7,(\d+),(\d+)>>", name)
        if not m:
            raise ValueError("not conv_pre's configuration: %r" % (name,))
        rows, n = (int(v) for v in m.groups())
        return dict(ROWS=rows, PAD=3, PER_TILE=512 // n, persistent=False)
    s = int(kernel[2])
    pat = {0: r"convt_tc_kernel<UpCfg<0,(\d+),(\d+)>>", 1: r"convt_resident_tc_kernel<UpCfg<1,(\d+),(\d+)>>"}.get(
        s, r"convt_stream_tc_kernel<StreamCfg<%d,(\d+),\d+,\d+>>" % s)
    m = re.fullmatch(pat, name)
    if not m:
        raise ValueError("not the configuration of %s: %r" % (kernel, name))
    rows = int(m.group(1))
    return dict(ROWS=rows, PAD=1, PER_TILE=(256 // int(m.group(2))) if s == 0 else 1, persistent=s >= 2)


def geometry(kernel):
    lib = engine.lib()
    name = lib.mg_gen_conv_pre_config() if kernel == "pre" else lib.mg_gen_convt_config(int(kernel[2]))
    return parse(kernel, name.decode())


def ctas(g, B, L):
    """CTAs of a uniform launch (persistent kernels: tiles, walked by at most NUM_SMS CTAs)."""
    return -(-B * (L + g["PAD"]) // g["ROWS"]) * g["PER_TILE"]


def uniform_cases(g, kernel):
    """(B, L): for B = 1, 2, 3 the batch's last position, or its last zero row, one row before, on and after tile borders
    1 - 3; a short last tile; part-filled last CTAs; more CTAs than two waves."""
    R, P = g["ROWS"], g["PAD"]
    out = set()
    for B in (1, 2, 3):
        for k in (1, 2, 3):
            for t in (k * R - 1, k * R, k * R + 1):
                for rows in (t, t + P):  # B (L + P) rows: the last zero row, or the last position (rows - P), ends at t
                    if rows % B == 0 and rows // B - P >= 1:
                        out.add((B, rows // B - P))
    out |= {(1, 1), (4, 1), (5, 7), (9, 7), (3, R // 2 + 1), (7, 30), WAVES[kernel]}
    return sorted(out)


def ragged_tables(g):
    """name -> lengths (input units) of the ragged batches of a kernel with geometry g."""
    R, P = g["ROWS"], g["PAD"]
    rs = np.random.RandomState(R * 10 + P)
    # R items of R + 1 and 2 R + 1 virtual rows alternately: item i ends at offset i + 1 of a tile, no two runs merge
    offsets = [(R + 1 if i % 2 == 0 else 2 * R + 1) - P for i in range(min(R, 256))]
    short = [int(v) for v in rs.choice([1, 2, 1, 2, 3], 120)] + [R + 5, 1, 2, 2 * R, 1]
    runs = []
    while len(runs) < 256:
        v = int(rs.randint(1, R + 1))
        if not runs or v != runs[-1]:
            runs.append(v)
    return {"offsets": offsets, "short": short, "runs256": runs}


def item_ends(g, lengths):
    """Virtual row after each item's last position, and after its last zero row."""
    v = np.cumsum([L + g["PAD"] for L in lengths])
    return v - g["PAD"], v


KNOWN = {"pre": "conv_rows_tc_kernel<ConvCfg<80,512,7,128,128>>", "up0": "convt_tc_kernel<UpCfg<0,64,32>>",
         "up1": "convt_resident_tc_kernel<UpCfg<1,64,32>>", "up2": "convt_stream_tc_kernel<StreamCfg<2,128,3,4>>",
         "up3": "convt_stream_tc_kernel<StreamCfg<3,128,3,4>>"}


def test_parsers_on_known_geometry():
    assert parse("pre", KNOWN["pre"]) == dict(ROWS=128, PAD=3, PER_TILE=4, persistent=False)
    assert parse("up0", KNOWN["up0"]) == dict(ROWS=64, PAD=1, PER_TILE=8, persistent=False)
    assert parse("up1", KNOWN["up1"]) == dict(ROWS=64, PAD=1, PER_TILE=1, persistent=False)
    assert parse("up3", KNOWN["up3"]) == dict(ROWS=128, PAD=1, PER_TILE=1, persistent=True)
    assert ctas(parse("pre", KNOWN["pre"]), 1, 125) == 4 and ctas(parse("pre", KNOWN["pre"]), 1, 126) == 8
    for k, bad in (("pre", KNOWN["up0"]), ("up0", KNOWN["up1"]), ("up2", KNOWN["up3"]), ("up1", "convt_tc_kernel")):
        with pytest.raises(ValueError):
            parse(k, bad)
    assert (1, 125) in uniform_cases(parse("pre", KNOWN["pre"]), "pre")  # 128 rows: the zero rows end on border 1


@pytest.mark.parametrize("kernel", KERNELS)
def test_library_reports_the_geometry(kernel):
    g = geometry(kernel)
    assert g["ROWS"] % 64 == 0 and g["PER_TILE"] >= 1, g


@pytest.mark.parametrize("kernel", KERNELS)
def test_sweeps_contain_every_situation(kernel):
    g = parse(kernel, KNOWN[kernel])
    R = g["ROWS"]
    cases = uniform_cases(g, kernel)
    for k in (1, 2, 3):
        for d in (-1, 0, 1):
            for B in (1, 2, 3):
                last = [c for c in cases if c[0] == B and B * (c[1] + g["PAD"]) - g["PAD"] == k * R + d]
                zero = [c for c in cases if c[0] == B and B * (c[1] + g["PAD"]) == k * R + d]
                assert B > 1 or (last and zero), (kernel, k, d)  # B = 1 reaches every border; B = 2, 3 where divisible
            assert any(B > 1 and B * (L + g["PAD"]) in (k * R + d, k * R + d + g["PAD"]) for B, L in cases), (kernel, k, d)
    rows = [B * (L + g["PAD"]) for B, L in cases]
    assert any(0 < r % R <= R // 8 for r in rows)  # a short last tile
    assert any(B > 1 and r % R for (B, _), r in zip(cases, rows))  # a part-filled last CTA of a multi-item batch
    assert max(ctas(g, B, L) for B, L in cases) > 2 * NUM_SMS
    tables = ragged_tables(g)
    _, zero_ends = item_ends(g, tables["offsets"])
    assert set(zero_ends % R) == set(range(R)) and len(tables["offsets"]) <= 256
    short = tables["short"]
    assert {1, 2} <= set(short) and (g["PAD"] < 3 or any(L + 3 < 7 for L in short))  # a k7 tap spans a whole item
    assert max(np.bincount(np.floor_divide(item_ends(g, short)[1] - 1, R))) > R // (1 + 2 * g["PAD"])  # many items a tile
    runs = tables["runs256"]
    assert len(runs) == 256 and all(a != b for a, b in zip(runs, runs[1:]))
    for t in tables.values():
        assert all(L >= 1 for L in t)


# ------------------------------------------------------------------------------------------------------------------
# where the blob keeps conv_pre's and the ConvTs' weights (restated in kernel_model.gen_weight_offset)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", range(5))
def test_layout_restatement_matches_the_library(layer):
    """Every weight of conv_pre and a seeded sample of each ConvT's, both halves; out-of-range arguments give -1."""
    off, none = lib_offset(), ctypes.c_size_t(-1).value
    a, b, tap = (g.ravel() for g in weight_grid(layer))
    if layer:
        pick = np.random.RandomState(layer).choice(a.size, min(a.size, 20000), replace=False)
        a, b, tap = a[pick], b[pick], tap[pick]
    for h in (0, 1):
        want = gen_weight_offset(layer, a, b, tap, h)
        got = np.array([off(0, layer, int(co_or_ci), int(ci_or_co), int(t), h) for co_or_ci, ci_or_co, t in zip(
            (a if layer == 0 else b), (b if layer == 0 else a), tap)], dtype=np.int64)
        assert np.array_equal(got, want), (layer, h, int(np.argmax(got != want)))
    cin, cout, _, K = SHAPE[("pre", "up0", "up1", "up2", "up3")[layer]]
    assert off(0, layer, cout, 0, 0, 0) == none and off(0, layer, 0, cin, 0, 0) == none and off(0, layer, 0, 0, K, 0) == none
    assert off(0, layer, 0, 0, 0, 2) == none and off(0, -1, 0, 0, 0, 0) == none
    # the blocks follow each other: ups.0 right after the last ResBlock conv, conv_pre right after ups.3
    assert off(0, 1, 0, 0, 0, 0) == off(0, 28, 0, 0, 0, 0) + 12 * 32 * 32
    assert off(0, 0, 0, 0, 0, 0) == off(0, 4, 0, 0, 0, 0) + up_tc_bytes(3)


# ------------------------------------------------------------------------------------------------------------------
# argument checks of the new entry points (no CUDA call is reached)
# ------------------------------------------------------------------------------------------------------------------
def test_chain_kernel_refuses_bad_arguments_before_any_cuda_call():
    lib = engine.lib()
    p, x, y = ctypes.c_void_p(256), ctypes.c_void_p(512), ctypes.c_void_p(1024)
    lens = lambda *v: (ctypes.c_int * len(v))(*v)
    call = lambda **kw: lib.mg_gen_chain_kernel(*[kw.get(n, d) for n, d in (
        ("packed", p), ("k", 0), ("x", x), ("y", y), ("B", 2), ("L", 8), ("lengths", lens(8, 3)), ("precision", 0),
        ("stream", None))])
    bad = [dict(packed=None), dict(x=None), dict(y=None), dict(y=x), dict(x=ctypes.c_void_p(520)),
           dict(y=ctypes.c_void_p(1028)), dict(packed=ctypes.c_void_p(260)), dict(k=-1), dict(k=8), dict(B=0),
           dict(B=257), dict(L=0), dict(B=1 << 20, L=1 << 9), dict(lengths=lens(0, 3)), dict(lengths=lens(8, 9)),
           dict(lengths=lens(-1, 1)), dict(precision=2), dict(precision=-1)]
    for kw in bad:
        assert call(**kw) == -1, kw
        assert b"mg_gen_chain_kernel" in lib.mg_last_error_string(), kw
    engine.check(lib.mg_gen_set_pipeline(2))  # another chain: refused like the stream
    try:
        assert call() == -1 and b"default chain" in lib.mg_last_error_string()
    finally:
        engine.check(lib.mg_gen_set_pipeline(-1))
    assert lib.mg_gen_convt_config(-1) == b"" and lib.mg_gen_convt_config(4) == b""


# ------------------------------------------------------------------------------------------------------------------
# the emulation, and TAU_E calibrated on the CPU
# ------------------------------------------------------------------------------------------------------------------
def conv_fn(kernel):
    S = SHAPE[kernel][2]
    if kernel == "pre":
        return lambda a, w: F.conv1d(a, w, padding=3)
    return lambda a, w: F.conv_transpose1d(a, w, stride=S, padding=S // 2)


def operand(kernel, x):
    """The fp32 value the kernel splits: x (conv_pre) or LeakyReLU(x) (the ConvTs)."""
    return x if kernel == "pre" else lrelu32(x)


def bound(emu, a2):
    return TAU_E * a2 + REL_E * emu.abs()


def ratio(y, emu, a2):
    return (y.double() - emu).abs() / bound(emu, a2).clamp_min(1e-300)


# (kernel name, Cin, K, S) under test; the calibration uses 32 or 64 output channels of each
CALIBRATION = [("pre", 80, 7, 1), ("up0", 512, 16, 8), ("up1", 256, 16, 8), ("up2", 128, 4, 2), ("up3", 64, 4, 2)]


@pytest.mark.parametrize("kernel,cin,k,S", CALIBRATION)
def test_tau_calibration(kernel, cin, k, S):
    """A float32-accumulated emulation stays under 0.5 of the bound at fp32 and bf16; each value-only mutant of the
    operands exceeds it by >= 8x.  Also printed: each mutant against the 2^-12 bound of test_layer_isolation_gpu."""
    gen = torch.Generator().manual_seed(cin * 100 + k)
    x = torch.randn(2, cin, 300, generator=gen)
    if kernel == "pre":
        w = (torch.rand(64, cin, k, generator=gen) * 2 - 1) / (cin * k) ** 0.5
    else:
        w = (torch.rand(cin, 32, k, generator=gen) * 2 - 1) / (cin * 2) ** 0.5
    conv = conv_fn(kernel)
    a = operand(kernel, x)
    ah, al = split_rn(a)
    wh, wl = split_rn(w)
    a64, w64 = a.double(), w.double()
    a2 = conv(a64 * a64, w64 * w64).sqrt()
    exact = conv(a64, w64)
    old = lambda y: float(((y - exact).abs() / (OLD_TAU * a2 + OLD_REL * exact.abs()).clamp_min(1e-300)).max())
    r = lambda y, emu: float(ratio(y, emu, a2).max())
    emu3, emu1 = split_passes(conv, ah, al, wh, wl), split_passes(conv, ah, al, wh, wl, "bf16")
    f = lambda t: t.float()
    f32_3 = (conv(f(ah), f(wh)) + conv(f(al), f(wh)) + conv(f(ah), f(wl))).double()
    f32_1 = conv(f(ah), f(wh)).double()
    mutants = {}
    m = al.clone()
    m[:, 8:16, 150] = 0
    mutants["lo of one k-panel of one row zeroed"] = (split_passes(conv, ah, m, wh, wl), emu3)
    drop_xl = al.clone()
    drop_xl[:, 8:16, :] = 0
    drop_wl = wl.clone()
    if kernel == "pre":
        drop_wl[:, 8:16, :] = 0
    else:
        drop_wl[8:16] = 0
    mutants["pass (xl, wh) dropped for one k-panel"] = (split_passes(conv, ah, drop_xl, wh, wl), emu3)
    mutants["pass (xh, wl) dropped for one k-panel"] = (split_passes(conv, ah, al, wh, drop_wl), emu3)
    trunc = (a.view(torch.int32) & -65536).view(torch.float32).double()
    mutants["hi truncated (bf16)"] = (split_passes(conv, trunc, None, wh, None, "bf16"), emu1)
    if kernel != "pre":
        xh, xl = split_rn(x)
        mutants["LeakyReLU after the split"] = (
            split_passes(conv, bf16_rn(lrelu32(xh.float())).double(), bf16_rn(lrelu32(xl.float())).double(), wh, wl), emu3)
    clean3, clean1 = r(f32_3, emu3), r(f32_1, emu1)
    print("\n%s (Cin %d, K %d, S %d): float32 accumulation %.3f (fp32) / %.3f (bf16) of the bound" % (
        kernel, cin, k, S, clean3, clean1))
    assert clean3 < 0.5 and clean1 < 0.5, (clean3, clean1)
    for name, (y, emu) in mutants.items():
        rm = r(y, emu)
        print("  %-40s %7.1f x the bound, %.2f x the 2^-12 bound" % (name, rm, old(y)))
        assert rm >= MUTANT_X, (kernel, name, rm)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def halves(gdev):
    """layer -> (hi, lo) of its weights in torch layout, fp32, read back from the packed blob."""
    blob = gdev.packed.view(torch.int16)
    out = {}
    for layer in range(5):
        grid = weight_grid(layer)
        out[layer] = tuple(bf16_of(blob, gen_weight_offset(layer, *grid, h)) for h in (0, 1))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("layer", range(5))
def test_blob_holds_the_split_of_the_folded_weights(g64, halves, layer):
    hi, lo = halves[layer]
    w = g64.w["conv_pre" if layer == 0 else "ups.%d" % (layer - 1)][0]
    assert hi.shape == w.shape
    # hi is the round-to-nearest of the pair; where lo rounded up to half an ulp of hi, hi + lo is a tie and either
    # neighbour is nearest (about 2^-10 of the weights)
    rn = bf16_rn(hi + lo)
    assert bool(((rn == hi) | (2 * (hi + lo) == hi + rn)).all()), layer
    assert bool((lo.abs() <= 2.0 ** -8 * hi.abs()).all()), layer
    d = ((hi.double() + lo.double()) - w).abs()
    assert bool((d <= 2.0 ** -16 * w.abs() + 2.0 ** -40).all()), (layer, float((d / w.abs().clamp_min(1e-30)).max()))


def run(gdev, kernel, x, lengths=None, precision="fp32"):
    """(output [B, Cout, R L] in a FILL-ed buffer, the buffer) of a ConvT / conv_pre kernel or ResBlock chain kernel."""
    B, _, L = x.shape
    if isinstance(kernel, int):
        _, cout, R = gdev.CHAIN_SHAPES[kernel]
    else:
        _, cout, R, _ = SHAPE[kernel]
    buf = nan_buffer(B * cout * R * L)
    if kernel == "up3":  # (no chain kernel of its own: mg_gen_convt)
        assert lengths is None and precision == "fp32"
        stream = torch.cuda.current_stream().cuda_stream
        engine.check(engine.lib().mg_gen_convt(gdev.packed.data_ptr(), 3, x.data_ptr(), buf.data_ptr(), B, L, stream))
        return buf[:B * cout * R * L].view(B, cout, R * L), buf
    k = kernel if isinstance(kernel, int) else CHAIN[kernel]
    return gdev.chain_kernel(k, x, lengths, precision, out=buf), buf


def own_call_faults(gdev, kernel, x, y, lengths, R, precision):
    """Items that differ from their own uniform call."""
    out = set()
    for i, L in enumerate(lengths):
        own, _ = run(gdev, kernel, x[i:i + 1, :, :L].contiguous(), None, precision)
        if not torch.equal(own[0], y[i, :, :R * L]):
            out.add(i)
    return out


def emulation(g64, halves, kernel, x, lengths, precision):
    """(y_emu, A2) of the whole batch in float64; positions past each length are zero in x (an item's own padding)."""
    _, _, R, _ = SHAPE[kernel]
    B, _, L = x.shape
    xv = torch.where(valid_mask(lengths, 1, L)[:, None, :], x, torch.zeros((), device=x.device))
    a = operand(kernel, xv)
    ah, al = split_rn(a)
    wh, wl = (t.double() for t in halves[LAYER[kernel]])
    w64, b64 = g64.w["conv_pre" if kernel == "pre" else "ups.%d" % (LAYER[kernel] - 1)]
    emu = split_passes(conv_fn(kernel), ah, al, wh, wl, precision) + b64[None, :, None]
    a64 = a.double()
    return emu, conv_fn(kernel)(a64 * a64, w64 * w64).sqrt()


def item_ratios(y, emu, a2, lengths, R):
    r = torch.where(valid_mask(lengths, R, y.shape[-1])[:, None, :], ratio(y, emu, a2), torch.zeros((), device=y.device))
    return r.flatten(1).amax(1)  # NaN (an output never written, or computed from NaN) propagates and fails


def where_worst(y, emu, a2, g, R, B, L):
    r = ratio(y, emu, a2)
    i, c, t = np.unravel_index(int(torch.argmax(torch.nan_to_num(r, nan=1e30))), tuple(r.shape))
    row = i * (L + g["PAD"]) + t // R
    return "item %d, channel %d, output %d (virtual row %d, offset %d in its tile)" % (i, c, t, row, row % g["ROWS"])


def inputs(cin, B, L, seed, lengths=None):
    x = torch.randn(B, cin, L, generator=torch.Generator().manual_seed(seed)).cuda()
    if lengths is not None:
        x[~valid_mask(lengths, 1, L)[:, None, :].expand_as(x)] = float("nan")
    return x


UNIFORM = [("pre", "fp32"), ("up0", "fp32"), ("up0", "bf16"), ("up1", "fp32"), ("up1", "bf16"), ("up2", "fp32"),
           ("up3", "fp32")]


def near_border(g, B, L, R, band=2):
    """[B, R L]: outputs whose input position lies within `band` rows of a tile border or of its item's ends."""
    p = torch.arange(R * L, device="cuda") // R
    v = torch.arange(B, device="cuda")[:, None] * (L + g["PAD"]) + p[None, :]
    off = v % g["ROWS"]
    return (off <= band) | (off >= g["ROWS"] - band) | (p[None, :] <= band) | (p[None, :] >= L - 1 - band)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,precision", UNIFORM)
def test_uniform_batches_at_tile_borders(gdev, g64, halves, kernel, precision):
    g = geometry(kernel)
    cin, _, R, _ = SHAPE[kernel]
    worst, at, near_w, far_w, fails = 0.0, "", 0.0, 0.0, []
    cases = uniform_cases(g, kernel)
    for B, L in cases:
        x = inputs(cin, B, L, 7919 * LAYER[kernel] + 31 * B + L)
        y, buf = run(gdev, kernel, x, None, precision)
        emu, a2 = emulation(g64, halves, kernel, x, [L] * B, precision)
        r = float(item_ratios(y, emu, a2, [L] * B, R).max())
        if not r <= 1:
            fails.append((B, L, r, where_worst(y, emu, a2, g, R, B, L)))
        if fill_faults(y, buf, [L] * B, R):
            fails.append((B, L, "outputs past the end or the guard written"))
        rr, near = ratio(y, emu, a2).amax(1), near_border(g, B, L, R)
        near_w = max(near_w, float(rr[near].max()) if near.any() else 0.0)
        far_w = max(far_w, float(rr[~near].max()) if (~near).any() else 0.0)
        if r > worst:
            worst, at = r, "(B %d, L %d) %s" % (B, L, where_worst(y, emu, a2, g, R, B, L))
    print("\n%s %s uniform: worst %.3f of the bound at %s; within 2 rows of a tile border or item end %.3f, elsewhere %.3f"
          % (kernel, precision, worst, at, near_w, far_w))
    assert not fails, ("%d of %d (B, L) fail" % (len({f[:2] for f in fails}), len(cases)), fails[:4])


RAGGED = [("pre", "fp32"), ("up0", "fp32"), ("up0", "bf16"), ("up1", "fp32"), ("up1", "bf16"), ("up2", "fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,precision", RAGGED)
def test_ragged_tables(gdev, g64, halves, kernel, precision):
    g = geometry(kernel)
    cin, _, R, _ = SHAPE[kernel]
    worst, at, fails, total = 0.0, "", [], 0
    for name, lengths in ragged_tables(g).items():
        B, L = len(lengths), max(lengths)
        x = inputs(cin, B, L, 104729 * LAYER[kernel] + B, lengths)
        y, buf = run(gdev, kernel, x, lengths, precision)
        emu, a2 = emulation(g64, halves, kernel, x, lengths, precision)
        r = item_ratios(y, emu, a2, lengths, R)
        bound_bad = set(torch.nonzero(~(r <= 1)).flatten().tolist())
        fill_bad = fill_faults(y, buf, lengths, R)
        own_bad = own_call_faults(gdev, kernel, x, y, lengths, R, precision)
        total += B
        fails += [(name, i, lengths[i], float(r[i]), i in fill_bad, i in own_bad) for i in sorted(bound_bad | fill_bad | own_bad)]
        if float(r.max()) > worst:
            i = int(torch.argmax(r))
            worst, at = float(r.max()), "table %s, item %d of %d positions" % (name, i, lengths[i])
    print("\n%s %s ragged: worst %.3f of the bound (%s)" % (kernel, precision, worst, at))
    # (table, item, length, ratio to the bound, written past its end, differs from its own call)
    assert not fails, ("%d of %d items fail" % (len(fails), total), fails[:6])


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("k", [2, 4, 6, 7])
def test_resblock_kernels_on_the_ragged_tables(gdev, g64, k, precision):
    cin, _, R = gdev.CHAIN_SHAPES[k]
    stage = RES_STAGE[k]
    worst = 0.0
    for name, lengths in ragged_tables(geometry(RES_TABLES[k])).items():
        B, L = len(lengths), max(lengths)
        x = inputs(cin, B, L, 1299709 * k + B, lengths)
        y, buf = run(gdev, k, x, lengths, precision)
        bad = fill_faults(y, buf, lengths, R, zero_tail=k == 7)
        assert not bad, (k, name, "outputs past the end or the guard written", sorted(bad)[:8])
        bad = own_call_faults(gdev, k, x, y, lengths, R, precision)
        assert not bad, (k, name, "items differ from their own calls", sorted(bad)[:8])
        if precision == "fp32":
            for i, Li in enumerate(lengths):
                x64 = x[i:i + 1, :, :Li].double()
                ref = g64.post(g64.resblock(3, g64.convt(3, x64))) if k == 7 else g64.resblock(stage, x64)
                e = float(row_errors(y[i:i + 1, :, :R * Li], ref).max())
                assert e < ROW_TOL, (k, name, i, Li, e)
                worst = max(worst, e)
    print("\nchain kernel %d %s ragged tables: %s" % (
        k, precision, "worst per-row error %.2e" % worst if precision == "fp32" else "fill, guard and own calls"))


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["pre", "up2"])
def test_bf16_keeps_three_passes_where_documented(gdev, kernel):
    g = geometry(kernel)
    cin = SHAPE[kernel][0]
    for lengths in [[L] * B for B, L in uniform_cases(g, kernel)[:6]] + list(ragged_tables(g).values()):
        x = inputs(cin, len(lengths), max(lengths), 17 * len(lengths) + max(lengths), lengths)
        y32, _ = run(gdev, kernel, x, lengths, "fp32")
        y16, _ = run(gdev, kernel, x, lengths, "bf16")
        assert torch.equal(y32.view(torch.int32), y16.view(torch.int32)), (kernel, len(lengths), max(lengths))
