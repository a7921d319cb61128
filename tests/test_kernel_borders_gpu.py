"""The ResBlock kernels at every kind of tile and cluster border, with the lengths derived from the geometry the library
reports (mg_gen_resblock_config), so a re-tiling moves the tested lengths with it.

Tiling (launch_resblock and the edge-aware comment of resblock_tc_kernel, csrc/mg_res_tc.cu): a cluster of CS CTAs covers
PC = CS P consecutive positions (P = 64 NRB per CTA).  Cluster 0 starts at position 0; cluster c > 0 starts at
(PC - HALO) + (c - 1) PVB - HL.  A cluster keeps the outputs it owns: not its left HL rows (c > 0) and not its right HALO
rows when more sequence follows, so the ownership borders sit at PC - HALO + k PVB, and a cluster k + 1 appears at
L = PC + k PVB + 1.  Inside a cluster the CTAs exchange their border rows instead of recomputing a halo.

Every length runs with B = 1 and 3 against the float64 restatement of the kernel's layers (test_layer_isolation_gpu):
per (item, channel) row max|d| / max|ref| < 1e-4 (the residual branch alone < 3e-4 for the plain ResBlocks), and the
error within 20 rows of a border may not exceed 4x the largest error elsewhere in the same call (+ 1e-7 of the row
scale): the arithmetic is the same on every row, only the data movement differs at a border.

Measured on an H100 80GB HBM3 (700 W power limit), printed by test_border_sweep (-s): worst per-row error, worst
branch error (plain ResBlocks), worst (error near a border) / (error elsewhere) of one call:
    code  0  2.2e-5  2.2e-4  1.25        code  4  5.2e-6     -    1.08        code 20  2.3e-5  -  1.15
    code  1  1.2e-5  8.3e-5  1.21        code 12  2.9e-5     -    1.31        code 21  3.1e-5  -  1.14
    code  2  7.5e-6  4.8e-5  1.06        code 13  3.8e-5     -    0.96        code 22  3.0e-5  -  1.30
    code  3  5.5e-6  2.3e-5  1.02        code 14  1.0e-5     -    1.02
Every chain variant (tail masks 0, 2, .., 14) against float64: worst per-item error 7.0e-6 at (3, 5), 9.3e-6 at (40, 32).
"""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth
from kernel_model import g64, gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import (BAND, BRANCH_TOL, ROW_TOL, borders, config, ctas, input_shape, lengths, parse_config, row_errors,
                          run_with_reference)

CODES = (0, 1, 2, 3, 4, 12, 13, 14, 20, 21, 22)
BORDER_X = 4.0   # border error <= BORDER_X * interior error + FLOOR
FLOOR = 1e-7


def test_config_strings_parse_for_every_stage_code():
    """Every stage code the pipeline uses reports a configuration, and its tiling covers each length exactly once."""
    lib = engine.lib()
    assert lib.mg_gen_resblock_config(5) == b"" and lib.mg_gen_resblock_config(-1) == b""
    for code in CODES:
        g = config(code)
        assert g["C"] == 256 >> {4: 3, 12: 2, 13: 3, 14: 3}.get(code, code % 10)
        assert bool(g["POST"]) == (code in (4, 14)) and bool(g["UPF"]) == (12 <= code <= 14)
        assert g["UPT"] == ({20: 8, 21: 2, 22: 2}.get(code, 0))
        assert g["PVB"] > 0
        for L in list(range(1, 3 * g["PC"])) + lengths(g):
            owned = sorted((lo, hi) for (_c, _r, _o, lo, hi) in ctas(g, L) if hi > lo)
            assert owned[0][0] == 0 and owned[-1][1] == L and all(a[1] == b[0] for a, b in zip(owned, owned[1:])), (code, L)


def test_upres_post_entry_point_validates_before_launching():
    lib, p = engine.lib(), ctypes.c_void_p(256)
    assert lib.mg_gen_upres_post(None, p, ctypes.c_void_p(512), 1, 4, None) == -1
    assert lib.mg_gen_upres_post(p, p, p, 1, 4, None) == -1  # x and audio must differ
    assert lib.mg_gen_upres_post(p, p, ctypes.c_void_p(512), 0, 4, None) == -1
    assert b"mg_gen_upres_post" in lib.mg_last_error_string()


def test_parser_and_lengths_on_known_geometry():
    g = parse_config("resblock_tc_kernel<RbCfg<256,1,1,2,4,0,0,0,4>>")
    assert (g["P"], g["PC"], g["HALO"], g["HL"], g["PVB"]) == (64, 256, 16, 16, 224)
    Ls = lengths(g)
    for L in (239, 240, 241, 255, 256, 257, 463, 464, 465, 480, 481, 703, 704, 705, 63, 64, 65, 288, 289, 352, 417):
        assert L in Ls, L
    assert borders(g, 257) == [64, 128, 192, 240] and borders(g, 200) == [64, 128, 192]
    g = parse_config("resblock_tc_kernel<RbCfg<32,8,2,1,4,1,1,0,1>>")
    assert (g["P"], g["HALO"], g["HL"], g["PVB"]) == (512, 19, 19, 474)
    assert all(L % 2 == 0 for L in lengths(g)) and 986 in lengths(g) and 512 in lengths(g)
    g = parse_config("resblock_tc_kernel<RbCfg<256,1,1,2,4,0,0,8,1>>")
    assert (g["HL"], g["PVB"]) == (17, 31)
    with pytest.raises(ValueError):
        parse_config("convt_tc_kernel")


# ------------------------------------------------------------------------------------------------------------------
# the sweep
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("code", CODES)
def test_border_sweep(gdev, g64, code):
    """Stage code `code` at every length of lengths(), B = 1 and 3 (measured values: the module docstring)."""
    g = config(code)
    S = g["UPT"] or 1
    worst_rows = worst_branch = worst_border = 0.0
    for L in lengths(g):
        for B in (1, 3):
            rs = np.random.RandomState(code * 100003 + L * 7 + B)
            x = torch.from_numpy(rs.standard_normal(input_shape(g, code, B, L)).astype(np.float32)).cuda()
            y, ref, x64 = run_with_reference(gdev, g64, code, x)
            assert y.shape == ref.shape, (code, L, tuple(y.shape), tuple(ref.shape))
            e = row_errors(y, ref)
            rows = float(e.max())
            assert rows < ROW_TOL, (code, B, L, rows)
            worst_rows = max(worst_rows, rows)
            if code <= 3 and borders(g, L):  # (a few positions alone: the branch is small against the error x leaves)
                branch = float(row_errors(y.double() - x64, ref - x64).max())
                assert branch < BRANCH_TOL, (code, B, L, branch)
                worst_branch = max(worst_branch, branch)
            # output index t of a tail ConvT belongs to input position (t + S / 2) // S
            n = y.shape[-1]
            near = torch.zeros(n, dtype=torch.bool, device=y.device)
            for b in borders(g, L):
                t = S * b - S // 2 if S > 1 else b
                near[max(0, t - BAND * S):min(n, t + BAND * S + 1)] = True
            if near.any() and not near.all():
                eb, ei = float(e[..., near].max()), float(e[..., ~near].max())
                assert eb <= BORDER_X * ei + FLOOR, (code, B, L, eb, ei, borders(g, L))
                worst_border = max(worst_border, eb / max(ei, 1e-30))
    print("\ncode %d (%s): %d lengths, rows %.2e, branch %s, border / interior %.2f" % (
        code, engine.lib().mg_gen_resblock_config(code).decode(), len(lengths(g)), worst_rows,
        "%.2e" % worst_branch if code <= 3 else "-", worst_border))


# ------------------------------------------------------------------------------------------------------------------
# bitwise: batch independence and determinism of the clustered stages, every chain variant against float64
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("stage,L", [(0, 500), (1, 600)])
def test_clustered_stage_items_equal_their_single_item_calls(gdev, stage, L):
    """More than two waves of clusters: every item of the batch equals the same item run alone, and two identical calls
    are bit-identical."""
    g = config(stage)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 2 * (sms // g["CS"]) + 1
    rs = np.random.RandomState(50 + stage)
    x = torch.from_numpy(rs.standard_normal((B, g["C"], L)).astype(np.float32)).cuda()
    y1 = gdev.resblock(stage, x)
    y2 = gdev.resblock(stage, x)
    assert torch.equal(y1, y2)
    for b in range(B):
        assert torch.equal(gdev.resblock(stage, x[b:b + 1]), y1[b:b + 1]), (stage, b)


@pytest.fixture(scope="module")
def torch_gen64(gstate):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in gstate.items()})
    g = g.cuda().double()
    vs, gs, bs = g._param_triplets()
    return g, [t.detach() for trip in zip(vs, gs, bs) for t in trip]


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(3, 5), (40, 32)])
def test_every_tail_mask_chain_matches_float64(gdev, torch_gen64, B, T):
    """Each of the eight chains (ConvT of stage 1, 2, 3 fused at the tail of the ResBlock before it, or not) against
    Generator._torch_forward in float64, per item; (40, 32) runs as two batch slices."""
    g, leaves = torch_gen64
    mel = torch.from_numpy(synth.mel_input(B, T, 900 + B)).cuda()
    with torch.no_grad():
        ref = g._torch_forward(mel.double(), leaves)
    lib = engine.lib()
    assert lib.mg_gen_forward_slices(B, T) == (2 if B == 40 else 1)
    worst = 0.0
    try:
        for mask in range(0, 16, 2):
            engine.check(lib.mg_gen_set_pipeline(mask))
            y = gdev.forward(mel)
            gdev.check_status(B, T)
            e = float(row_errors(y, ref).max())
            assert e < ROW_TOL, (mask, e)
            worst = max(worst, e)
    finally:
        engine.check(lib.mg_gen_set_pipeline(-1))
    print("\n(B=%d, T=%d) every tail mask: worst per-item max-rel %.2e" % (B, T, worst))
