"""The 64- and 32-channel ResBlock kernels with their weights stacked [hi | lo] along the MMA N dimension
(csrc/mg_layout.h tc_stacked, csrc/mg_res_tc.cu).

(a) layout, no GPU: inside a chunk of KC input channels the bf16 element of (k-panel kp, half h, output row co, e) sits at
    ((kp * 2 + h) * C + co) * 8 + e, so one k-panel is 2 C rows of 16 bytes -- hi rows [0, C), lo rows [C, 2 C) -- and
    consecutive k-panels are 2 C * 16 bytes apart, which is the leading-byte-offset of the B descriptor; chunk order and
    chunk size are those of the wider stages.  Restated in numpy against mg_gen_tc_weight_offset for every weight of the
    stage-2 / 3 ResBlock convs and of the two fused front ConvTs.  With a GPU the packed blob is read back and hi + lo of
    every such weight must reproduce the folded fp32 weight to split-bf16 precision, |lo| <= 2^-8 |hi|.
(b) stage codes 2, 12, 13, 14, 4 and 22 against the float64 layer reference at the tile-border lengths of
    test_kernel_borders_gpu, same tolerance.
(c) the bf16 variants (codes 2 and 14, reached through the bf16 forward) against the float64 emulation of
    test_bf16_inference_gpu at their border lengths.
"""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, synth
from test_bf16_inference_gpu import _emulation_bound, gen  # noqa: F401 (fixture)
from test_kernel_borders_gpu import config, lengths, input_shape, run_code
from test_layer_isolation_gpu import ROW_TOL, Gen64, g64, gdev, gstate, row_errors  # noqa: F401 (fixtures)

NARROW = (64, 32)
STAGE_OF = {64: 2, 32: 3}


def tc_kc(C):
    return 4096 // C if C >= 128 else C


def fp32_blob_bytes():
    n = 80 * 512 * 7 + 32 * 7 + 512 + 1
    for i in range(4):
        cin, cout, k = 512 >> i, 256 >> i, (16 if i < 2 else 4)
        n += cin * cout * k + cout + 6 * (cout * cout * 3 + cout)
    return (n * 4 + 255) // 256 * 256


def res_base(layer):
    """Byte offset of a ResBlock conv's tensor-core block: after the fp32 blob, 12 C^2 bytes per conv in layer order."""
    return fp32_blob_bytes() + sum(12 * (256 >> ((l - 5) // 6)) ** 2 for l in range(5, layer))


def in_chunk(C, co, cik, h):
    """bf16 element index inside a chunk (numpy arrays welcome): stacked for C <= 64, halves back to back above."""
    KC = tc_kc(C)
    if C <= 64:
        return ((cik // 8 * 2 + h) * C + co) * 8 + cik % 8
    return ((h * (KC // 8) + cik // 8) * C + co) * 8 + cik % 8


def lib_offset():
    f = engine.lib().mg_gen_tc_weight_offset
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.c_int] * 6
    return f


@pytest.mark.parametrize("C", NARROW + (128,))
def test_in_chunk_scatter_matches_the_descriptors(C):
    """Every (co, ci, tap, half) of one c1 conv of the stage: chunk = (tap, K-slice) in consumption order, then the
    in-chunk order the B descriptor of resblock_tc_kernel walks."""
    off = lib_offset()
    stage = {128: 1, 64: 2, 32: 3}[C]
    layer, KC = 5 + 6 * stage + 1, tc_kc(C)
    chunk_elems = 2 * KC * C
    base = res_base(layer)
    assert off(0, 5, 0, 0, 0, 0) == fp32_blob_bytes()
    for tap in range(3):
        for ci in range(0, C, 3 if C > 64 else 1):
            for h in (0, 1):
                for co in (0, 1, 7, 8, C // 2, C - 1):
                    want = base + 2 * ((tap * (C // KC) + ci // KC) * chunk_elems + in_chunk(C, co, ci % KC, h))
                    assert off(0, layer, co, ci, tap, h) == want, (C, tap, ci, h, co)
    if C <= 64:
        # what the descriptors rely on: rows 16 bytes apart, lo rows C rows after the hi rows, k-panels 2 C rows apart
        o = lambda co, ci, h: off(0, layer, co, ci, 0, h)
        assert o(1, 0, 0) - o(0, 0, 0) == 16 and o(0, 0, 1) - o(0, 0, 0) == C * 16
        assert o(0, 8, 0) - o(0, 0, 0) == 2 * C * 16 and o(0, 1, 0) - o(0, 0, 0) == 2
        assert o(C - 1, KC - 1, 1) - o(0, 0, 0) == 4 * C * KC - 2  # the last element of the chunk


@pytest.mark.parametrize("C", NARROW)
def test_front_convt_chunks_are_stacked_too(C):
    off = lib_offset()
    stage, KC = STAGE_OF[C], tc_kc(C)
    base = off(1, stage, 0, 0, 0, 0)
    assert base == res_base(29) + sum((512 >> s) * (256 >> s) * (16 if s < 2 else 4) * 4 for s in range(4)) \
        + 80 * 512 * 7 * 4 + (0 if stage == 2 else 4 * (2 * 64 // 64) * 4 * 64 * 64)
    for k in range(4):
        for ci in range(2 * C):
            for h in (0, 1):
                for co in (0, 5, C - 1):
                    want = base + 2 * ((k * (2 * C // KC) + ci // KC) * 2 * KC * C + in_chunk(C, co, ci % KC, h))
                    assert off(1, stage, co, ci, k, h) == want, (C, k, ci, h, co)
    assert off(1, 1, 0, 0, 0, 0) == ctypes.c_size_t(-1).value and off(0, 29, 0, 0, 0, 0) == ctypes.c_size_t(-1).value


def _bf16_at(blob_u16, byte_offsets):
    v = blob_u16[torch.from_numpy(byte_offsets // 2).cuda()].to(torch.int32) << 16
    return v.view(torch.float32).double()


@pytest.mark.gpu
@pytest.mark.parametrize("C", NARROW)
def test_packed_blob_holds_hi_and_lo_where_the_descriptors_read_them(gdev, g64, C):
    blob = gdev.packed.view(torch.int16).to(torch.int32) & 0xFFFF
    stage, KC = STAGE_OF[C], tc_kc(C)
    co, ci, tap = np.meshgrid(np.arange(C), np.arange(C), np.arange(3), indexing="ij")
    for j in range(3):
        for which in ("convs1", "convs2"):
            layer = 5 + 6 * stage + j + (3 if which == "convs2" else 0)
            w = g64.w["resblocks.%d.%s.%d" % (stage, which, j)][0]  # [co][ci][tap], float64
            idx = lambda h: res_base(layer) + 2 * ((tap * (C // KC) + ci // KC) * 2 * KC * C + in_chunk(C, co, ci % KC, h))
            hi, lo = _bf16_at(blob, idx(0)), _bf16_at(blob, idx(1))
            assert float((hi + lo - w).abs().max()) <= 2.0 ** -15 * float(w.abs().max()), (layer, "hi + lo")
            assert bool((lo.abs() <= 2.0 ** -8 * hi.abs() + 1e-30).all()), (layer, "lo rows")
    w = g64.w["ups.%d" % stage][0]  # [ci][co][k]
    ci, co, k = np.meshgrid(np.arange(2 * C), np.arange(C), np.arange(4), indexing="ij")
    base = lib_offset()(1, stage, 0, 0, 0, 0)
    idx = lambda h: base + 2 * ((k * (2 * C // KC) + ci // KC) * 2 * KC * C + in_chunk(C, co, ci % KC, h))
    hi, lo = _bf16_at(blob, idx(0)), _bf16_at(blob, idx(1))
    assert float((hi + lo - w).abs().max()) <= 2.0 ** -15 * float(w.abs().max())
    assert bool((lo.abs() <= 2.0 ** -8 * hi.abs() + 1e-30).all())


@pytest.mark.gpu
@pytest.mark.parametrize("code", [2, 12, 13, 14, 4, 22])
def test_narrow_codes_at_tile_borders(gdev, g64, code):
    g = config(code)
    worst = 0.0
    for L in lengths(g):
        for B in (1, 3):
            rs = np.random.RandomState(code * 7919 + L * 13 + B)
            x = torch.from_numpy(rs.standard_normal(input_shape(g, code, B, L)).astype(np.float32)).cuda()
            y, ref, _x64 = run_code(gdev, g64, code, x)
            assert y.shape == ref.shape
            e = float(row_errors(y, ref).max())
            assert e < ROW_TOL, (code, B, L, e)
            worst = max(worst, e)
    print("\ncode %d: %d lengths, worst per-row error %.2e" % (code, len(lengths(g)), worst))


@pytest.mark.gpu
@pytest.mark.parametrize("code,per_frame", [(2, 128), (14, 256)])
def test_bf16_variants_at_their_borders(gen, g64, code, per_frame):
    Ts = sorted({t for L in lengths(config(code)) for t in (-(-L // per_frame), -(-L // per_frame) + 1) if t >= 1})
    worst = 0.0
    for T in Ts:
        mel = torch.from_numpy(synth.mel_input(1, T, 700 + T)).cuda()
        worst = max(worst, _emulation_bound(gen, g64, mel, (code, T))[4])
    print("\nbf16 code %d: T = %s, worst (kernel - 2e-5) / emulation %.2f" % (code, Ts, worst))
