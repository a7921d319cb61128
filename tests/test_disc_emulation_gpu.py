"""The discriminator's split-bf16 tensor-core kernels against a float64 emulation of their OWN arithmetic: the grouped
convs (disc_group_tc_kernel, disc_group4_tc_kernel), conv_post1's forward and data gradient (conv_rows_tc_kernel<Post1Cfg>,
<Post1DgradCfg>) and its weight gradient (post1_wgrad_tc_kernel); and the four tensor-core weight copies the pack writes.

Blob.  disc_pack_kernel keeps, per discriminator, a Toeplitz copy of grouped_convs.0-2 (each weight once per output parity,
zero slots where a panel's tap falls outside 0..40), the 8-outputs-per-lane Toeplitz copy of grouped_convs.3 (each weight
once per e), conv_post1's copy and its transposed, tap-flipped copy for the data gradient.  The layouts are restated in
kernel_model (numpy) and checked against mg_disc_tc_element on every element of one group per copy and a seeded sample of the rest.
On the GPU: every element of the grouped copies is split_bf16 of the fp32 folded weight in the blob, hi = bf16_rn(w),
lo = bf16_rn(w - hi), bit for bit, every structural zero +0.0; conv_post1's transposed copy equals the forward copy at
(ci, co, 4 - tap) bit for bit, each lo is at most half a bf16 ulp of its hi and hi + lo is within 2^-16 |w64| of the float64
fold (bit for bit the split of the exact weight for the exact-operand state).  A lo half truncated in the pack, or one
duplicate written from the wrong tap, is about 2^-17 of a weight: far under any value bound, and invisible to an
emulation that reads its halves back from the same blob.

Emulation.  Operands are split as split2_bf16 splits them, the weights' halves read back from the blob, and the passes
accumulated in float64:
  * grouped convs: one accumulator gets (xh, wh) + (xl, wh), another (xh, wl); kernel: their fp32 sum + bias, then
    LeakyReLU fmaxf(v, v * 0.01f);
  * conv_post1 forward: (xh, wh) + (xl, wh) + (xh, wl) + bias, LeakyReLU; the data gradient the same passes on the
    transposed copy, zero bias, no activation;
  * wgrad: (dzh, xh) + (dzl, xh) + (dzh, xl) over every item's positions, zero padding at each item's ends.
Bound, element-wise:  |y - y_emu| <= TAU_E A2 + (REL_E + rel) |y_emu|  with A2 = sqrt(conv64(x^2, w^2)) and, after a
LeakyReLU, TAU_E A2 scaled by 0.01 where y_emu is negative by more than TAU_E A2.  rel = 2^-24 per MMA that adds into one
accumulator (3 K / 16) for the data and weight gradients only, the tensor cores' truncating accumulation that
test_disc_backward_isolation_gpu measured; it grows with K, so at training size (K = 4096 positions) it hides a lo-half
defect of one stage, and the exact-operand cases below are what see it.  test_tau_calibration (CPU): a float32-accumulated
emulation stays under 0.5 of the bound, each operand mutant exceeds it by >= 4x.

Random operands at the border lengths of the launch geometry, each layer called alone (mg_msd_layer_forward) on an input
of the length that puts it there: grouped_convs.0-2 at the GROUP_TARGETS output lengths, grouped_convs.3 at GROUP4_TARGETS,
Bt = 1, ni - 1, ni, ni + 1, 2 ni + 1 for the packed geometries (test_disc_forward_borders_gpu), conv_post1 and its two
gradients at post1_lengths with Bt = 1 and 3 (test_disc_backward_isolation_gpu); plus config 3 (32 x 8192) on the maps
and the gradients the engine produced, where the layer call must also equal the forward's map bit for bit.  Outputs go to
NaN-filled buffers with a guard after them that must still hold the fill.

Exact operands.  A second discriminator state whose folds are exact: each v row of layers 1-5 is sparse +-1 with n in
{1, 4, 16, 64} nonzeros (the fold g / sqrtf(n) is a power-of-two scaling), g, the biases, x and dz are hi + lo with
|hi| in {1, 1.25, 1.5, 1.75} 2^e and |lo| in {1, 1.5} 2^(e - 10), below half a bf16 ulp of hi, so split_bf16 returns
exactly those two nonzero halves.  Every product of the three passes is then a multiple of 2^(ex + ew - 13) and the sum of
their magnitudes stays under 2^21 of that quantum, so every output is exact in fp32 whatever the order and the rounding of
the adds (test_exact_operands_sum_exactly proves it on the CPU, in three orders with round-to-nearest and truncation), and
the kernel must match the float64 emulation bit for bit.  An extra (xl, wl) pass is 2^-20 of a product: visible on the
rows with n = 1.  The nonzeros are routed so that every Toeplitz slot (k-panel, phase or channel pair, parity or e,
position, output column) of grouped_convs.0-3, every (tap, k-panel) of conv_post1 and of its transposed copy, and every
k-panel, stage, ring slot and item end of the weight gradient at config-3 size carries a nonzero product
(test_exact_operands_cover_every_slot).

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s).  Worst ratio to the bound (worst
|y - y_emu| / A2 in units of 2^-16), border lengths / config 3:
    grouped_convs.0  0.286 (0.30) / 0.295 (0.29)      conv_post1        0.275 (6.14) / 0.306 (4.68)
    grouped_convs.1  0.310 (0.31) / 0.333 (0.31)      conv_post1 dgrad  0.279 (6.38) / 0.261 (6.63)
    grouped_convs.2  0.337 (0.38) / 0.317 (1.01)      conv_post1 wgrad  0.124 (0.62) / 0.360 (13.84)
    grouped_convs.3  0.395 (3.21) / 0.395 (2.41)
conv_post1's forward and data gradient reached 6.4 x 2^-16 A2 at K = 5120, twice the generator's TAU_E alone: hence the
accumulation term for all three conv_post1 kernels, not only the gradients.  The GPU tests of this file take about 30 s.
Value-only kernel mutants, each run once:
    mutant                                                                   new tests failing      older tests failing
    disc_pack_kernel truncates the lo half of conv_post1's transposed copy  the blob checks (3)    none
    disc_group_tc_kernel stores lo = 0 for ci 0 of the second position of   grouped 0-2 random,    49 forward-border
      unit 0 of phase 0 (the first unit of a tile)                           exact, config 3 (7)    lengths and 8 others
    disc_group4_tc_kernel's pass 1 skips k-panel 2 of channel pair 1         grouped 3 random,      103 + 18
                                                                             exact, config 3 (3)
    conv_post1's tail_rows (A rows 128 - 131) store lo = 0                   conv_post1 random,     43 + 13
                                                                             exact, config 3 (3)
    post1_wgrad_tc_kernel stores lo(dz) = 0 for k-panel 0 of the last stage  exact wgrad at config  config 3 of the backward
      when there are more than 12 stages                                     3, config 3 (2)        isolation, 5 of test_disc_gpu
The pack truncation is the one no older test sees (its 2^-17 error passes every value bound).  The unit-0 element had to be
the second position: the first position of a tile's first unit only ever meets the zero slots of q = -1.  The exact
state does not see the pack truncation either, by design (its lo halves are exact in bf16); the blob checks do.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv1d_weight

from melgan_multi_b200 import engine, synth
from kernel_model import ddev, dstate  # noqa: F401 (fixtures)
from kernel_model import (BLOB_BYTES, G4TC_GROUP, G4TC_START, GROUP4_TARGETS, GROUP_TARGETS, GROUPS, GTC_GROUP, TC_BYTES,
                          TC_START, TCT_START, WG_PANEL, WG_STAGE, batches, cdiv, disc_bias_offset, disc_weight_offset,
                          folded64, group4_plan, group_tc_plan, gtc_start, guard_ok, nan_buffer, post1_lengths,
                          post1_offset, post1_straddles, slots, split_np, split_passes, split_rn, toeplitz_slots, upstream)

LAYERS = synth.DISCRIMINATOR_LAYERS
TAU_E = 3 * 2.0 ** -16       # the generator's emulation bound (test_gen_front_kernels_gpu), K = 1024 x 5
TAU_G = 2.0 ** -16           # the grouped convs, K = 4 x 41: their MMAs add 28 partial sums into an output, not 960
REL_E = 2.0 ** -22
MUTANT_X = 4                 # each operand mutant exceeds the bound by at least this factor
SLOPE32 = float(np.float32(0.01))
EXACT_N = (64, 16, 4, 1)     # nonzeros per v row of the exact-operand state
EX, EW = 0, -4               # exponents of the exact operands' hi halves: x and dz, weights


# ------------------------------------------------------------------------------------------------------------------
# the blob of one discriminator: kernel_model's restatement of csrc/mg_layout.h against the library
# ------------------------------------------------------------------------------------------------------------------
def tc_element(offset):
    out = [ctypes.c_int(-9) for _ in range(4)]
    h = engine.lib().mg_disc_tc_element(int(offset), *(ctypes.byref(v) for v in out))
    return (h,) + tuple(v.value for v in out)


def test_blob_size_matches_the_library():
    assert engine.lib().mg_disc_packed_bytes() == BLOB_BYTES
    assert engine.lib().mg_msd_packed_bytes() == 3 * BLOB_BYTES


@pytest.mark.parametrize("copy", range(1, 7))
def test_layout_restatement_matches_the_library(copy):
    """Each copy's restated slots fill its byte range exactly once; mg_disc_tc_element agrees on every element of one group
    (grouped copies) or one ring slot column (conv_post1: 128 rows x 16 channels, all taps) and on a seeded sample."""
    off, h, co, ci, tap = slots(copy)
    start, nbytes = {1: (gtc_start(1), 4 * GTC_GROUP), 2: (gtc_start(2), 16 * GTC_GROUP), 3: (gtc_start(3), 64 * GTC_GROUP),
                     4: (G4TC_START, 256 * G4TC_GROUP), 5: (TC_START, TC_BYTES), 6: (TCT_START, TC_BYTES)}[copy]
    assert off.size * 2 == nbytes and np.array_equal(np.sort(off), start + 2 * np.arange(off.size)), copy
    if copy <= 4:
        cog = 16 if copy <= 3 else 4
        first = np.nonzero((co // cog) == GROUPS[copy] // 2)[0]
    else:
        first = np.nonzero((co < 128) & (ci >= 16) & (ci < 32))[0]
    pick = np.concatenate([first, np.random.RandomState(copy).choice(off.size, 3000, replace=False)])
    for j in pick:
        want = (int(h[j]), copy, int(co[j]), int(ci[j]), int(tap[j]))
        assert tc_element(off[j]) == want, (copy, int(off[j]), tc_element(off[j]), want)
    for bad in (0, TC_START - 2, TCT_START + TC_BYTES, BLOB_BYTES, TC_START + 1):
        assert tc_element(bad)[0] == -1, bad


# ------------------------------------------------------------------------------------------------------------------
# the exact-operand state
# ------------------------------------------------------------------------------------------------------------------
def exact_values(rs, shape, e):
    """hi + lo with hi = +-(1 + k/4) 2^e and lo = +-(1 + j/2) 2^(e - 10): both halves nonzero, lo under half a bf16 ulp
    of hi (also below a power of two), so split_bf16 gives back exactly hi and lo."""
    hi = rs.choice([-1.0, 1.0], shape) * (1 + rs.randint(0, 4, shape) / 4) * 2.0 ** e
    lo = rs.choice([-1.0, 1.0], shape) * (1 + rs.randint(0, 2, shape) / 2) * 2.0 ** (e - 10)
    return (hi + lo).astype(np.float32)


def exact_rows(rs, rows, inner, pattern):
    """[rows, inner] of +-1 with pattern[j % 4] nonzeros in row j, taken as consecutive chunks of one permutation of the
    inner index (wrapping), so every inner index is hit once the chunks add up to `inner`."""
    v = np.zeros((rows, inner), np.float32)
    perm, at = rs.permutation(inner), 0
    for j in range(rows):
        n = pattern[j % 4]
        v[j, perm[(at + np.arange(n)) % inner]] = rs.choice([-1.0, 1.0], n)
        at += n
    return v


def exact_layer(rs, l):
    """(v, g, bias) of layer l (1..5): rows sparse +-1, g = (hi + lo) sqrt(n) so that the fold w = g v / sqrt(n) has
    |hi| in [2^EW, 2^(EW + 1)) in every row; bias a multiple of 2^(EX + EW - 3)."""
    _n, cin, cout, k, _s, groups, _p = LAYERS[l]
    cig, cog = cin // groups, cout // groups
    v = np.zeros((cout, cig * k), np.float32)
    if groups == 1:
        # conv_post1 (row n = EXACT_N[co % 4]).  The 32 rows of n = 64 of a 128-row output group hold one (ci, tap) of
        # every (128-channel group of ci, tap) -- for the transposed copy, whose k-panels are 8 co -- and, between them,
        # one of every (8-channel k-panel of ci, tap) of the forward copy
        for cg in range(cout // 128):
            fwd = rs.permutation(((np.arange(cig // 8)[:, None] * 8 + rs.randint(0, 8, (cig // 8, k))) * k + np.arange(k)).ravel())
            for j in range(128):
                n, co = EXACT_N[j % 4], 128 * cg + j
                pick = rs.choice(cig * k, n, replace=False)
                if n == 64:
                    tr = ((np.arange(cig // 128)[:, None] * 128 + rs.randint(0, 128, (cig // 128, k))) * k + np.arange(k)).ravel()
                    pick = np.unique(np.concatenate([tr, fwd[20 * (j // 4):20 * (j // 4 + 1)]]))
                    rest = rs.permutation(np.setdiff1d(np.arange(cig * k), pick))
                    pick = np.concatenate([pick, rest[:n - pick.size]])
                v[co, pick] = rs.choice([-1.0, 1.0], n)
    else:  # one permutation per output column c of a group, its rows are the column's rows of every group
        pattern = (64, 64, 64, 1) if groups == 4 else EXACT_N
        for c in range(cog):
            v[c::cog] = exact_rows(rs, groups, cig * k, pattern[c % 4:] + pattern[:c % 4])
    n = (v != 0).sum(1)
    g = exact_values(rs, (cout,), EW) * np.sqrt(n).astype(np.float32)
    bias = (rs.randint(-7, 8, cout) * 2.0 ** (EX + EW - 3)).astype(np.float32)
    return v.reshape(cout, cig, k), g.reshape(cout, 1, 1), bias


def exact_state(seed=97):
    """synth.discriminator_state with layers 1-5 of all three discriminators replaced by exact ones."""
    st = synth.discriminator_state(seed)
    rs = np.random.RandomState(seed)
    for d in range(3):
        for l in range(1, 6):
            base = "discriminators.%d.%s" % (d, LAYERS[l][0])
            st[base + ".weight_v"], st[base + ".weight_g"], st[base + ".bias"] = exact_layer(rs, l)
    return st


_EXACT = {}


def exact_weights():
    """(state, [3][7] folded fp32 weights, exact) of the exact-operand state, built once."""
    if not _EXACT:
        st = exact_state()
        w = [[None] * 7 for _ in range(3)]
        for d in range(3):
            for l in range(1, 6):
                base = "discriminators.%d.%s" % (d, LAYERS[l][0])
                v, g = st[base + ".weight_v"], st[base + ".weight_g"]
                w[d][l] = (g.astype(np.float64) / np.sqrt((v != 0).sum((1, 2), keepdims=True)) * v).astype(np.float32)
        _EXACT.update(state=st, w=w)
    return _EXACT["state"], _EXACT["w"]


def test_exact_state_folds_to_split_halves():
    """The fold of every exact layer is exact in fp32 (float64 fold == fp32 fold) and splits into two nonzero halves
    with hi in [2^EW, 2^(EW + 1)) in magnitude; the exact x values split the same way."""
    st, w = exact_weights()
    for d in range(3):
        for l in range(1, 6):
            base = "discriminators.%d.%s" % (d, LAYERS[l][0])
            w64 = synth.fold_weight_norm(st[base + ".weight_g"], st[base + ".weight_v"])
            assert np.array_equal(w64, w[d][l]), (d, l)
            nz = w[d][l] != 0
            hi, lo = split_np(w[d][l][nz])
            assert np.all((np.abs(hi) >= 2.0 ** EW) & (np.abs(hi) < 2.0 ** (EW + 1)) & (lo != 0)), (d, l)
            assert np.array_equal(hi + lo, w[d][l][nz].astype(np.float64)), (d, l)
    x = exact_values(np.random.RandomState(1), (100000,), EX)
    hi, lo = split_np(x)
    assert np.all((lo != 0) & (np.abs(hi) >= 2.0 ** EX)) and np.array_equal(hi + lo, x.astype(np.float64))


def test_exact_operands_cover_every_slot():
    """Every Toeplitz slot of grouped_convs.0-3 (the output column included) holds a nonzero weight of the exact state;
    every (k-panel, tap) of conv_post1 and of its transposed copy does; the rows take every n of EXACT_N."""
    _st, w = exact_weights()
    for d in range(3):
        for l in (1, 2, 3, 4):
            off, h, co, ci, tap = toeplitz_slots(l)
            live = h < 2
            cog = 16 if l <= 3 else 4
            nz = w[d][l][co[live], ci[live], tap[live]] != 0
            # per (slot position inside a group block, i.e. offset within the block): nonzero in some group
            block = GTC_GROUP if l <= 3 else G4TC_GROUP
            rel = (off[live] - off.min()) % block
            hit = np.zeros(block // 2, bool)
            hit[rel[nz] // 2] = True
            want = np.zeros(block // 2, bool)
            want[rel // 2] = True
            assert np.array_equal(hit, want), (d, l, int((want & ~hit).sum()))
            assert {1, 64} <= set((w[d][l] != 0).sum((1, 2)).tolist()) <= set(EXACT_N), (d, l)
        wp = w[d][5] != 0
        # forward: every (k-panel of ci, tap) per 128-row output group; transposed: every (k-panel of co, tap) per ci group
        assert wp.reshape(8, 128, 128, 8, 5).any(axis=(1, 3)).all(), d
        assert wp.reshape(128, 8, 8, 128, 5).any(axis=(1, 3)).all(), d
        assert set(wp.sum((1, 2)).tolist()) == set(EXACT_N), d


def wgrad_dz(rs, Bt, L):
    """Exact dz for the weight gradient: row co of every item sparse, EXACT_N[co % 4] nonzeros over all Bt L positions,
    consecutive chunks of one permutation of the positions (every position hit)."""
    dz = np.zeros((1024, Bt * L), np.float32)
    mask = exact_rows(rs, 1024, Bt * L, EXACT_N) != 0
    dz[mask] = exact_values(rs, (int(mask.sum()),), EX)
    return np.ascontiguousarray(dz.reshape(1024, Bt, L).transpose(1, 0, 2))


WGRAD_EXACT = [(32, 128), (3, 65), (5, 17)]  # config 3 (conv_post1 at scale 0 of 32 x 8192), L % 8 != 0 with short items


def test_exact_wgrad_covers_every_stage():
    """At each WGRAD_EXACT size, every k-panel of every stage (so every ring slot) and both ends of every item carry a
    nonzero dz; config 3 runs 128 stages, past the 12 a part of the tests' mutants keys on."""
    for Bt, L in WGRAD_EXACT:
        dz = wgrad_dz(np.random.RandomState(Bt * 1000 + L), Bt, L)
        assert (dz != 0).any(1).all(), (Bt, L)  # every (item, position): every k-panel, stage, ring slot, item end
        assert {1, 64} <= set((dz != 0).sum((0, 2)).tolist()) <= set(EXACT_N)
    assert wgrad_stages(32, 128) == 128 and any(L % WG_PANEL for _Bt, L in WGRAD_EXACT)


def wgrad_stages(Bt, L):
    return cdiv(Bt * cdiv(L, WG_PANEL), WG_STAGE // WG_PANEL)


def wgrad_k(Bt, L):
    """K of the weight-gradient launch: every item padded to whole k-panels, the batch to whole stages."""
    return wgrad_stages(Bt, L) * WG_STAGE


def passes_terms(a, w):
    """Product terms of the split passes, one output per row: a [outputs, n], w [n] fp32 -> (terms of (ah, wh), (al, wh),
    (ah, wl)) [outputs, 3 n], and those of the absent (al, wl) [outputs, n]."""
    ah, al = split_np(a)
    wh, wl = split_np(w)
    return np.concatenate([ah * wh, al * wh, ah * wl], 1), al * wl


def fp32_sum(terms, order, truncate):
    """Sum of the float64 terms [n_out, n] in float32, in the given column order, rounding each add to nearest or
    towards zero."""
    acc = np.zeros(terms.shape[0], np.float32)
    for j in order:
        s = acc.astype(np.float64) + terms[:, j]  # exact: both fit in 53 bits here
        r = s.astype(np.float32)
        if truncate:
            over = np.abs(r.astype(np.float64)) > np.abs(s)
            r = np.where(over, np.nextafter(r, np.float32(0)), r)
        acc = r
    return acc


def test_exact_operands_sum_exactly():
    """For outputs of every exact case -- a grouped conv row, conv_post1 and its data gradient (a column of the weight)
    and the weight gradient (a sparse dz row against x) -- the fp32 sum of the three passes' products and the bias is
    the same in forward, reverse and shuffled order with round-to-nearest and with truncation, and equals the float64 sum;
    with n = 1 the absent (xl, wl) pass would change it."""
    _st, w = exact_weights()
    rs = np.random.RandomState(5)
    cases = []
    for l in (1, 4, 5):
        wl = w[0][l].reshape(w[0][l].shape[0], -1)
        cases += [("layer %d row %d" % (l, r), wl[r]) for r in range(0, wl.shape[0], max(1, wl.shape[0] // 64))]
    wt = w[0][5].transpose(1, 0, 2).reshape(1024, -1)
    cases += [("dgrad column %d" % c, wt[c]) for c in range(0, 1024, 16)]
    dz = wgrad_dz(np.random.RandomState(32 * 1000 + 128), 32, 128).transpose(1, 0, 2).reshape(1024, -1)
    cases += [("wgrad dz row %d" % c, dz[c]) for c in range(0, 1024, 16)]
    extra_seen = False
    for name, row in cases:
        nz = np.nonzero(row)[0]
        a = exact_values(rs, (256, nz.size), EX)  # 256 outputs: the operand they meet at the row's nonzeros
        t, t_ll = passes_terms(a, row[nz])
        bias = rs.randint(-7, 8, (256, 1)) * 2.0 ** (EX + EW - 3)
        t = np.concatenate([t, bias], 1)
        exact = t.sum(1)
        orders = [np.arange(t.shape[1]), np.arange(t.shape[1])[::-1], rs.permutation(t.shape[1])]
        for order in orders:
            for trunc in (False, True):
                got = fp32_sum(t, order, trunc).astype(np.float64)
                assert np.array_equal(got, exact), (name, trunc)
        if nz.size == 1:
            with_ll = (exact + t_ll.sum(1)).astype(np.float32).astype(np.float64)
            assert not np.any(with_ll == exact), name
            extra_seen = True
    assert extra_seen


# ------------------------------------------------------------------------------------------------------------------
# the emulation, and the bound calibrated on the CPU
# ------------------------------------------------------------------------------------------------------------------
def conv_fn(kind, l=None):
    """f(a, w) of a kernel's contraction: grouped conv l, conv_post1 forward / data gradient (a conv on the transposed
    weights [ci][co][k']), or the weight gradient (a = dz, w = x: returns [co][ci][tap])."""
    if kind == "group":
        _n, _ci, _co, _k, stride, groups, pad = LAYERS[l]
        return lambda a, w: F.conv1d(a, w, stride=stride, padding=pad, groups=groups)
    if kind in ("post1", "dgrad"):
        return lambda a, w: F.conv1d(a, w, padding=2)
    return lambda a, w: conv1d_weight(w, (a.shape[1], w.shape[1], 5), a, 1, 2)


def act(pre):
    return torch.where(pre > 0, pre, pre * SLOPE32)


def ratio(y, pre, a2, lrelu, acc=0.0, tau=TAU_E):
    """|y - y_emu| / bound, element-wise; pre: the float64 emulation before the activation."""
    emu = act(pre) if lrelu else pre
    t = tau * a2 + acc * (a2 + pre.abs())
    if lrelu:
        t = torch.where(pre > -t, t, t * SLOPE32)
    return (y.double() - emu).abs() / (t + REL_E * emu.abs()).clamp_min(1e-300)


def mma_acc(kind, K):
    """The accumulation term of conv_post1's kernels: 2^-23 per MMA that adds into one accumulator (3 passes x K / 16),
    times A2 + |y_emu| (the partial sums' scale): the tensor cores truncate each add, an error of up to an ulp of the
    running sum that does not average out; none for the grouped convs (28 MMAs)."""
    return 2.0 ** -23 * 3 * K / 16 if kind != "group" else 0.0


# (kind, layer, Cin, K per output, operand shapes) of the calibration: the grouped convs at their K = 4 x 41, conv_post1
# and its data gradient at K = 1024 x 5 (64 output channels), the weight gradient at the border sizes' K = Bt L
CALIBRATION = [("group", 1, None), ("group", 4, None), ("post1", 5, None), ("dgrad", 5, None),
               ("wgrad", 5, (3, 65)), ("wgrad", 5, (3, 127))]


def calibration_operands(kind, l, size, gen):
    if kind == "group":
        _n, cin, _co, k, _s, groups, _p = LAYERS[l]
        cout = 4 * (LAYERS[l][2] // groups)
        a = F.leaky_relu(torch.randn(2, 4 * 4, 300, generator=gen))
        w = (torch.rand(cout, 4, 41, generator=gen) * 2 - 1) / (4 * 41) ** 0.5
        f = lambda x, ww: F.conv1d(x, ww, stride=LAYERS[l][4], padding=20, groups=4)
        return a, w, f, 4 * 41
    if kind in ("post1", "dgrad"):
        a = F.leaky_relu(torch.randn(2, 1024, 64, generator=gen)) if kind == "post1" else torch.randn(2, 1024, 64, generator=gen)
        w = (torch.rand(64, 1024, 5, generator=gen) * 2 - 1) / (1024 * 5) ** 0.5
        return a, w, conv_fn(kind), 1024 * 5
    Bt, L = size
    dz = torch.randn(Bt, 16, L, generator=gen)
    x = F.leaky_relu(torch.randn(Bt, 64, L, generator=gen))
    return dz, x, conv_fn("wgrad"), Bt * L


@pytest.mark.parametrize("kind,l,size", CALIBRATION)
def test_tau_calibration(kind, l, size):
    """A float32-accumulated emulation stays under 0.5 of the bound; each value-only operand mutant exceeds it by >= 4x:
    the lo half of one 16-byte unit (8 consecutive K elements of one row) zeroed, pass (al, wh) or (ah, wl) dropped for
    one k-panel, the A operand's hi truncated instead of rounded."""
    gen = torch.Generator().manual_seed(100 * l + len(kind) + (size[1] if size else 0))
    a, w, f, K = calibration_operands(kind, l, size, gen)
    ah, al = split_rn(a)
    wh, wl = split_rn(w)
    a64, w64 = a.double(), w.double()
    a2 = f(a64 * a64, w64 * w64).sqrt()
    pre = split_passes(f, ah, al, wh, wl)
    acc = mma_acc(kind, K)
    lrelu = kind in ("group", "post1")
    r = lambda y: float(ratio(act(y) if lrelu else y, pre, a2, lrelu, acc, TAU_G if kind == "group" else TAU_E).max())
    fl = lambda t: t.float()
    clean = r((f(fl(ah), fl(wh)) + f(fl(al), fl(wh)) + f(fl(ah), fl(wl))).double())
    passes = lambda al_=al, wh1=wh, wl_=wl: f(ah, wh) + f(al_, wh1) + f(ah, wl_)  # wh1: the weights pass (al, wh) sees
    # value-only mutants the kernels' structure allows
    mut = {}
    if kind == "wgrad":  # A = dz over K = positions, B = x; a 16-byte unit and a k-panel are 8 positions of one item
        m = al.clone()
        m[1, 3, 8:16] = 0
        mut["lo of one 8-position unit of one dz row zeroed"] = passes(al_=m)
        m = al.clone()
        m[1, :, 8:16] = 0
        mut["pass (dzl, xh) dropped for one k-panel"] = passes(al_=m)
        m = wl.clone()
        m[1, :, 8:16] = 0
        mut["pass (dzh, xl) dropped for one k-panel"] = passes(wl_=m)
    else:  # K = (ci, tap); a k-panel is 8 channels at one tap (conv_post1), 2 taps 4 apart x 4 channels (grouped)
        m = al.clone()
        if kind == "group":
            m[0, 0:4, [149, 153]] = 0  # the two positions x 4 channels of one unit of a phase buffer
        else:
            m[0, 8:16, 30] = 0
        mut["lo of one 16-byte unit zeroed"] = passes(al_=m)
        panel = (slice(None), slice(None), [9, 13]) if kind == "group" else (slice(None), slice(8, 16), 3)
        m = wh.clone()
        m[panel] = 0
        mut["pass (xl, wh) dropped for one k-panel"] = passes(wh1=m)
        m = wl.clone()
        m[panel] = 0
        mut["pass (xh, wl) dropped for one k-panel"] = passes(wl_=m)
    th = (a.view(torch.int32) & -65536).view(torch.float32).double()
    mut["A hi truncated, lo of the rounded split"] = f(th, wh) + f(al, wh) + f(th, wl)
    print("\n%s l=%d K=%d: float32 accumulation %.3f of the bound" % (kind, l, K, clean))
    assert clean < 0.5, (kind, clean)
    for name, y in mut.items():
        rm = r(y)
        print("  %-50s %7.1f x the bound" % (name, rm))
        # at K = 5120 the accumulation term leaves a lo-half defect of one k-panel near the bound: the exact-operand
        # cases are what see those
        assert rm >= MUTANT_X or (K == 5120 and "hi truncated" not in name), (kind, name, rm)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the blob
# ------------------------------------------------------------------------------------------------------------------
def msd_device(state):
    dd = engine.DiscriminatorDevice("cuda:0")
    names = ["discriminators.%d.%s" % (d, n) for d in range(3) for n, *_ in LAYERS]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dd.pack([to(state[n + ".weight_v"]) for n in names], [to(state[n + ".weight_g"]) for n in names],
            [to(state[n + ".bias"]) for n in names])
    return dd


@pytest.fixture(scope="module")
def xdev():
    """The exact-operand state, packed."""
    return msd_device(exact_weights()[0])


def blob_i16(dd, s):
    return dd.packed.view(torch.int16)[s * BLOB_BYTES // 2:(s + 1) * BLOB_BYTES // 2]


def bits(blob, off):
    return blob[torch.from_numpy(np.ascontiguousarray(off // 2)).cuda()]


def as_float(b16):
    return (b16.to(torch.int32) << 16).view(torch.float32)


def split_bits(w):
    hi = w.to(torch.bfloat16)
    return hi.view(torch.int16), (w - hi.float()).to(torch.bfloat16).view(torch.int16)


def fp32_grouped(dd, s, l):
    """Layer l's fp32 folded weights in the blob, torch layout [Cout][4][41]."""
    _n, _cin, cout, _k, _s, groups, _p = LAYERS[l]
    cog = cout // groups
    f = dd.packed[s * BLOB_BYTES // 4:(s + 1) * BLOB_BYTES // 4]
    blk = f[disc_weight_offset(l):disc_weight_offset(l) + cout * 164].view(groups, 164, cog)
    return blk.permute(0, 2, 1).reshape(cout, 4, 41)


_SLOTS = {}


def cached_slots(copy):
    if copy not in _SLOTS:
        _SLOTS[copy] = slots(copy)
    return _SLOTS[copy]


def check_blob(dd, s, w_exact=None, w64=None):
    blob = blob_i16(dd, s)
    for l in (1, 2, 3, 4):
        off, h, co, ci, tap = cached_slots(l)
        got = bits(blob, off)
        hz = torch.from_numpy(h).cuda()
        w = fp32_grouped(dd, s, l)
        live = h < 2
        wv = w[torch.from_numpy(co[live]).cuda(), torch.from_numpy(ci[live]).cuda(), torch.from_numpy(tap[live]).cuda()]
        hi, lo = split_bits(wv)
        want = torch.where(hz[torch.from_numpy(live).cuda()] == 0, hi, lo)
        assert torch.equal(got[torch.from_numpy(live).cuda()], want), (s, l, "a half differs from split_bf16 of the fp32 weight")
        assert bool((got[hz == 2] == 0).all()), (s, l, "a structural zero is not +0.0")
        if w_exact is not None:
            assert torch.equal(w, torch.from_numpy(w_exact[l]).cuda()), (s, l, "fp32 fold")
    off5, h5, co5, ci5, tap5 = cached_slots(5)
    off6 = post1_offset(co5, ci5, tap5, h5, True)
    fwd, tr = bits(blob, off5), bits(blob, off6)
    assert torch.equal(fwd, tr), (s, "the transposed copy differs from the forward copy at (ci, co, 4 - tap)")
    hi, lo = as_float(fwd[0::2]).double(), as_float(fwd[1::2]).double()  # h is the fastest index of post1_slots
    assert np.array_equal(h5[0::2], np.zeros(h5.size // 2)) and np.array_equal(h5[1::2], np.ones(h5.size // 2))
    e = torch.frexp(hi.float())[1].double()  # |hi| in [2^(e-1), 2^e): half a bf16 ulp is 2^(e - 9)
    assert bool((lo.abs() <= torch.where(hi != 0, torch.ldexp(torch.ones_like(hi), (e - 9).long()), 0 * hi)).all()), s
    idx = [torch.from_numpy(a[0::2]).cuda() for a in (co5, ci5, tap5)]
    if w64 is not None:
        w = w64[idx[0], idx[1], idx[2]]
        d = (hi + lo - w).abs()
        assert bool((d <= 2.0 ** -16 * w.abs() + 2.0 ** -40).all()), (s, float((d / w.abs().clamp_min(1e-30)).max()))
    if w_exact is not None:
        whi, wlo = split_bits(torch.from_numpy(w_exact[5]).cuda()[idx[0], idx[1], idx[2]])
        assert torch.equal(fwd[0::2], whi) and torch.equal(fwd[1::2], wlo), s


@pytest.mark.gpu
@pytest.mark.parametrize("s", range(3))
def test_blob_holds_the_split_of_the_folded_weights(ddev, dstate, xdev, s):
    w64 = folded64(dstate, "discriminators.%d.conv_post1" % s)[0]
    check_blob(ddev, s, w64=w64)
    check_blob(xdev, s, w_exact=exact_weights()[1][s], w64=torch.from_numpy(exact_weights()[1][s][5]).cuda().double())


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ------------------------------------------------------------------------------------------------------------------
def halves(dd, s, l):
    """(wh, wl) float64 of layer l (1..5) read back from the tensor-core copy, torch layout; l = 6: conv_post1's halves
    from its transposed copy, as the data gradient's weights [ci][co][k']."""
    blob = blob_i16(dd, s)
    if l <= 4:
        off, h, co, ci, tap = cached_slots(l)
        live = h < 2
        out = []
        for half in (0, 1):
            sel = live & (h == half)
            w = torch.zeros(LAYERS[l][2], 4, 41, dtype=torch.float32, device="cuda")
            w[tuple(torch.from_numpy(a[sel]).cuda() for a in (co, ci, tap))] = as_float(bits(blob, off[sel]))
            out.append(w.double())
        return tuple(out)
    off, h, co, ci, tap = cached_slots(5)
    if l == 6:
        off = post1_offset(co, ci, tap, h, True)
    w = as_float(bits(blob, off)).view(1024, 1024, 5, 2).double()
    wh, wl = w[..., 0], w[..., 1]
    if l == 6:
        wh, wl = (t.permute(1, 0, 2).flip(2).contiguous() for t in (wh, wl))
    return wh, wl


_HALVES = {}


def cached_halves(dd, s, l):
    key = (id(dd), s, l)
    if key not in _HALVES:
        _HALVES[key] = halves(dd, s, l)
    return _HALVES[key]


def bias_of(dd, s, l):
    f = dd.packed[s * BLOB_BYTES // 4:(s + 1) * BLOB_BYTES // 4]
    return f[disc_bias_offset(l):disc_bias_offset(l) + LAYERS[l][2]].double()


def run_layer(dd, s, l, x):
    """layer_forward into a FILL-ed buffer: (y, guard intact)."""
    _n, _cin, cout, k, stride, _g, pad = LAYERS[l]
    Bt, _, Lin = x.shape
    n = Bt * cout * ((Lin + 2 * pad - k) // stride + 1)
    buf = nan_buffer(n)
    y = dd.layer_forward(s, l, x, out=buf)
    dd.check_status()
    return y, guard_ok(buf, n)


def forward_emulation(dd, s, l, x):
    """(pre-activation emulation, A2) of layer l on fp32 x."""
    kind = "group" if l <= 4 else "post1"
    f = conv_fn(kind, l)
    wh, wl = cached_halves(dd, s, l)
    ah, al = split_rn(x)
    pre = split_passes(f, ah, al, wh, wl) + bias_of(dd, s, l)[None, :, None]
    w = wh + wl
    x64 = x.double()
    return pre, f(x64 * x64, w * w).sqrt()


def run_dgrad(dd, s, dz):
    Bt, C, L = dz.shape
    buf = nan_buffer(dz.numel())
    engine.check(engine.lib().mg_msd_post1_dgrad(dd.packed.data_ptr(), s, dz.data_ptr(), buf.data_ptr(), Bt, L,
                                                 dd.status.data_ptr(), torch.cuda.current_stream().cuda_stream))
    dd.check_status()
    return buf[:dz.numel()].view(Bt, C, L), guard_ok(buf, dz.numel())


def run_wgrad(dd, x, dz):
    Bt, C, L = dz.shape
    dw, db = nan_buffer(1024 * 1024 * 5), nan_buffer(1024)
    engine.check(engine.lib().mg_msd_post1_wgrad(x.data_ptr(), dz.data_ptr(), dw.data_ptr(), db.data_ptr(), Bt, L,
                                                 dd.status.data_ptr(), torch.cuda.current_stream().cuda_stream))
    dd.check_status()
    return dw[:1024 * 1024 * 5].view(1024, 1024, 5), guard_ok(dw, 1024 * 1024 * 5) and guard_ok(db, 1024)


def dgrad_emulation(dd, s, dz):
    wh, wl = cached_halves(dd, s, 6)
    ah, al = split_rn(dz)
    f = conv_fn("dgrad")
    w = wh + wl
    d64 = dz.double()
    return split_passes(f, ah, al, wh, wl), f(d64 * d64, w * w).sqrt()


def wgrad_emulation(x, dz):
    ah, al = split_rn(dz)
    bh, bl = split_rn(x)
    f = conv_fn("wgrad")
    return split_passes(f, ah, al, bh, bl), f(dz.double() ** 2, x.double() ** 2).sqrt()


class Worst:
    """Worst ratio to the bound and worst |y - y_emu| / A2 per kernel, printed at the end of the module."""

    def __init__(self):
        self.r, self.t = {}, {}

    def add(self, key, y, pre, a2, lrelu, acc=0.0, tau=TAU_E):
        r = ratio(y, pre, a2, lrelu, acc, tau)
        emu = act(pre) if lrelu else pre
        t = (y.double() - emu).abs() / a2.clamp_min(1e-300)
        self.r[key] = max(self.r.get(key, 0.0), float(torch.nan_to_num(r, nan=1e30).max()))
        self.t[key] = max(self.t.get(key, 0.0), float(torch.nan_to_num(t, nan=1e30).max()))
        return float(torch.nan_to_num(r, nan=1e30).max())


@pytest.fixture(scope="module")
def worst():
    w = Worst()
    yield w
    lines = ["\nworst ratio to the bound (worst |y - y_emu| / A2 in units of 2^-16):"]
    for k in sorted(w.r):
        lines.append("  %-28s %.3f  (%.2f)" % (k, w.r[k], w.t[k] / 2.0 ** -16))
    print("\n".join(lines))


def grouped_cases(l):
    """(Lin, Bt) of layer l: each GROUP(4)_TARGETS output length with the batches of its packed geometry."""
    out = []
    for T in (GROUP_TARGETS if l <= 3 else GROUP4_TARGETS):
        if l <= 3:
            Lin, ni = 4 * T - T % 4, group_tc_plan(T)[1]
        else:
            Lin, ni = T, group4_plan(T)[0]
        out += [(Lin, Bt) for Bt in sorted(batches(ni))]
    return out


def random_input(cin, Bt, L, seed, signed=False):
    x = torch.randn(Bt, cin, L, generator=torch.Generator().manual_seed(seed))
    return (x if signed else F.leaky_relu(x)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("l", [1, 2, 3, 4])
def test_grouped_convs_random(ddev, worst, monkeypatch, l):
    monkeypatch.delenv("MG_DISC_GROUP", raising=False)
    fails = []
    for Lin, Bt in grouped_cases(l):
        s = (Lin + Bt) % 3
        x = random_input(LAYERS[l][1], Bt, Lin, 1000 * l + 7 * Lin + Bt)
        y, guard = run_layer(ddev, s, l, x)
        pre, a2 = forward_emulation(ddev, s, l, x)
        r = worst.add("grouped_convs.%d" % (l - 1), y, pre, a2, True, tau=TAU_G)
        if not (r <= 1 and guard):
            fails.append((Lin, Bt, s, r, guard))
    assert not fails, fails[:6]


@pytest.mark.gpu
def test_post1_random(ddev, worst):
    """conv_post1's forward, data gradient and weight gradient at the border lengths, Bt = 1 and 3."""
    fails = []
    for L in post1_lengths():
        for Bt in (1, 3):
            s = (L + Bt) % 3
            x = random_input(1024, Bt, L, 31 * L + Bt)
            y, guard = run_layer(ddev, s, 5, x)
            pre, a2 = forward_emulation(ddev, s, 5, x)
            r = worst.add("conv_post1", y, pre, a2, True, mma_acc("post1", 5120))
            dz = random_input(1024, Bt, L, 37 * L + Bt, signed=True)
            dx, g2 = run_dgrad(ddev, s, dz)
            pre_d, a2_d = dgrad_emulation(ddev, s, dz)
            rd = worst.add("conv_post1 dgrad", dx, pre_d, a2_d, False, mma_acc("dgrad", 5120))
            dw, g3 = run_wgrad(ddev, x, dz)
            pre_w, a2_w = wgrad_emulation(x, dz)
            rw = worst.add("conv_post1 wgrad", dw, pre_w, a2_w, False, mma_acc("wgrad", wgrad_k(Bt, L)))
            if not (max(r, rd, rw) <= 1 and guard and g2 and g3):
                fails.append((L, Bt, s, r, rd, rw, guard, g2, g3, post1_straddles(Bt, L)))
    assert not fails, fails[:6]


@pytest.mark.gpu
def test_config3_on_the_engine_maps_and_gradients(ddev, worst, monkeypatch):
    """Config 3 (32 x 8192): each tensor-core layer of each scale called alone on the map the forward produced equals
    the forward's map bit for bit and is within the bound; conv_post1's gradients on the dz the engine produced for the
    generator step."""
    monkeypatch.delenv("MG_DISC_GROUP", raising=False)
    Bt, L = 32, 8192
    y = torch.from_numpy(synth.audio_input(Bt, L, 11 * L + Bt)).cuda()
    fm = ddev.forward(y)
    ddev.check_status()
    G = upstream(fm, "generator")
    for s in range(3):
        for l in range(1, 6):
            out, guard = run_layer(ddev, s, l, fm[s][l - 1])
            assert guard and torch.equal(out, fm[s][l]), (s, l, "layer call differs from the forward")
            pre, a2 = forward_emulation(ddev, s, l, fm[s][l - 1])
            r = worst.add("config 3 " + LAYERS[l][0], out, pre, a2, True, mma_acc("post1" if l == 5 else "group", 5120),
                          TAU_G if l <= 4 else TAU_E)
            assert r <= 1, (s, l, r)
        dx6, _dw6, _db6 = ddev.edge_backward(s, 6, G[s][6], fm[s][5], True)
        dz = ddev.lrelu_backward(dx6, G[s][5], fm[s][5])
        Lp = dz.shape[2]
        dx, g2 = run_dgrad(ddev, s, dz)
        pre, a2 = dgrad_emulation(ddev, s, dz)
        rd = worst.add("config 3 conv_post1 dgrad", dx, pre, a2, False, mma_acc("dgrad", 5120))
        dw, g3 = run_wgrad(ddev, fm[s][4], dz)
        pre, a2 = wgrad_emulation(fm[s][4], dz)
        rw = worst.add("config 3 conv_post1 wgrad", dw, pre, a2, False, mma_acc("wgrad", wgrad_k(Bt, Lp)))
        assert g2 and g3 and rd <= 1 and rw <= 1, (s, rd, rw, g2, g3)


# ------------------------------------------------------------------------------------------------------------------
# GPU: exact operands, bit for bit
# ------------------------------------------------------------------------------------------------------------------
def exact_input(cin, Bt, L, seed):
    return torch.from_numpy(exact_values(np.random.RandomState(seed), (Bt, cin, L), EX)).cuda()


def exact_grouped_cases(l):
    """Packed tiles with a part-filled last CTA, a single tile, several tiles (the first unit of a later tile holds data)."""
    if l <= 3:
        return [(4 * T - T % 4, Bt) for T, Bt in ((13, 11), (122, 3), (123, 1), (257, 2), (513, 1))]
    return [(T, Bt) for T, Bt in ((9, 20), (489, 2), (1025, 2), (2049, 1))]


def exact_mismatch(y, want):
    d = y.view(torch.int32) != want.view(torch.int32)
    return int(d.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("l", [1, 2, 3, 4, 5])
def test_exact_forward_bit_for_bit(xdev, monkeypatch, l):
    monkeypatch.delenv("MG_DISC_GROUP", raising=False)
    cases = exact_grouped_cases(l) if l <= 4 else [(L, 3) for L in post1_lengths()]
    fails = []
    for Lin, Bt in cases:
        for s in range(3):
            x = exact_input(LAYERS[l][1], Bt, Lin, 100 * l + 10 * s + Lin)
            y, guard = run_layer(xdev, s, l, x)
            pre, _a2 = forward_emulation(xdev, s, l, x)
            p32 = pre.float()
            assert torch.equal(p32.double(), pre), (l, Lin, Bt, s, "the emulation is not exact in fp32")
            want = torch.maximum(p32, p32 * torch.tensor(0.01, dtype=torch.float32, device="cuda"))
            bad = exact_mismatch(y, want)
            if bad or not guard:
                fails.append((Lin, Bt, s, bad, guard))
    assert not fails, (l, fails[:6])


@pytest.mark.gpu
def test_exact_dgrad_bit_for_bit(xdev):
    fails = []
    for L in post1_lengths():
        for s in range(3):
            dz = exact_input(1024, 3, L, 7 * L + s)
            dx, guard = run_dgrad(xdev, s, dz)
            pre, _a2 = dgrad_emulation(xdev, s, dz)
            assert torch.equal(pre.float().double(), pre), (L, s)
            bad = exact_mismatch(dx, pre.float())
            if bad or not guard:
                fails.append((L, s, bad, guard))
    assert not fails, fails[:6]


@pytest.mark.gpu
@pytest.mark.parametrize("Bt,L", WGRAD_EXACT)
def test_exact_wgrad_bit_for_bit(xdev, Bt, L):
    x = exact_input(1024, Bt, L, 11 * L + Bt)
    dz = torch.from_numpy(wgrad_dz(np.random.RandomState(Bt * 1000 + L), Bt, L)).cuda()
    dw, guard = run_wgrad(xdev, x, dz)
    pre, _a2 = wgrad_emulation(x, dz)
    assert torch.equal(pre.float().double(), pre)
    bad = exact_mismatch(dw, pre.float())
    assert guard and not bad, (Bt, L, bad, guard)


# ------------------------------------------------------------------------------------------------------------------
# argument checks of the layer entry point (no CUDA call is reached)
# ------------------------------------------------------------------------------------------------------------------
def test_layer_forward_refuses_bad_arguments_before_any_cuda_call():
    lib = engine.lib()
    p, x, y, st = ctypes.c_void_p(256), ctypes.c_void_p(512), ctypes.c_void_p(1024), ctypes.c_void_p(2048)
    call = lambda **kw: lib.mg_msd_layer_forward(*[kw.get(n, d) for n, d in (
        ("packed", p), ("scale", 0), ("layer", 1), ("x", x), ("out", y), ("Bt", 2), ("Lin", 64), ("status", st),
        ("stream", None))])
    bad = [dict(packed=None), dict(x=None), dict(out=None), dict(status=None), dict(out=x), dict(scale=-1), dict(scale=3),
           dict(layer=0), dict(layer=7), dict(Bt=0), dict(Bt=65536), dict(Lin=0), dict(layer=6, Lin=0),
           dict(layer=3, Bt=65535, Lin=1 << 20)]
    for kw in bad:
        assert call(**kw) == -1, kw
        assert b"mg_msd_layer_forward" in lib.mg_last_error_string(), kw
