"""Each ResBlock conv of resblock_tc_kernel against a float64 emulation of its OWN arithmetic, one conv at a time, at every
cluster, CTA and item border of the launch geometry, on uniform and ragged batches, at fp32 and bf16.

Why one conv at a time.  The kernel splits its intermediate values on chip (hi = bf16_rn(v), lo = bf16_rn(v - hi)), so an
emulation of six chained convs cannot follow its splits: a 2^-24 difference in v can move a bf16 rounding.  Each conv is
therefore observed on an operand the host knows exactly, by choosing the weights (an ordinary generator state through
GeneratorDevice.pack; the fold is g / sqrtf(||v||^2), so a one-hot v row with g = 1 folds to exactly 1.0, hi = 1, lo = 0,
and g = 0 folds to exactly 0).  The kernel's code path does not depend on the weight values: the ring, the multicast, the
stacked chunks, every hand-off and the halo exchange run unchanged.  Seven packs (PATTERNS), each isolating the same conv
index in all four stages at once:
  * c1[j]  c1[j] seeded, c2[j] the centre-tap identity, every other c2 zero; biases seeded (pend carries them).  Output
           x + sum_i b2[i] + hl(lrelu(h)), h = c1[j](split(lrelu(x + sum_{i<j} b2[i]))) + b1[j], hl(v) = hi + lo.
  * c2[j]  c1[j] the centre-tap identity (its output hl(lrelu(x_j)) + b1 is exact in fp32), c2[j] seeded, other c2 zero.
  * fused  every c2 zero (the ResBlock is x + sum b2): observes the front ConvT (codes 12, 13, 14), the tail ConvT with its
           fp32 fix-up at position L (codes 20, 21, 22) and conv_post (codes 4, 14) with seeded weights.
In the six ResBlock patterns the front and tail ConvTs are one-hot (one nonzero tap per input channel): the front sends
the first C input channels to the even outputs and the other C to the odd ones, the tail sends half of the channels
through x[s] taps and half through x[s - 1] taps, so the fix-up at L carries ResBlock values.  conv_post keeps seeded
weights (one output channel cannot observe channels separately); the bound goes through it by root-sum-square.

Emulation (float64; the kernel's documented arithmetic, csrc/mg_res_tc.cu): X = split(lrelu32(v)), zero outside [0, L);
the weights' halves read back from the blob; passes (xh,wh) + (xl,wh) + (xh,wl) at fp32, (xh,wh) at bf16; b1 added at
read-back; c2 accumulates onto R and y = R + pend with pend the fp32 running sum of the b2; the tail fix-up an fp32 dot
product of lrelu(x[L-1]) with the fp32 ConvT weights; conv_post and tanh in fp32.  Every output is held to an interval:
  * one conv:   TAU_E A2 + REL_E |y_emu|  (test_gen_front_kernels_gpu), + RHO |x| for a c2 at C >= 128, whose three
                passes go onto the fp32 residual inside the MMA (at C <= 64 only xh * wl and then D do: ULP_E covers it);
  * an exact observation: HL_E |v| for hl(v) = hi + lo, ULP_E of the magnitudes of each fp32 add onto x and pend; at bf16
                the identity reads bf16_rn(lrelu(h)): the interval is [bf16_rn(lrelu(h - B)), bf16_rn(lrelu(h + B))];
  * conv_post:  POST_RSS sqrt(conv(B^2, w^2)) + POST_E sum |products| + TANH_E (tanh is 1-Lipschitz).  A bf16
                interval is a rounding, up to its whole width on every channel, so one root-sum-square fell short
                (2.3x, chain kernel 7 at bf16): POST_RSS = 4;
  * fix-up:     FIX_E (sum |products| + |bias|) (fp32 weights: no split).
test_calibration (CPU) holds the bound to both sides: a float32-accumulated emulation stays under 0.5 of it and each
value-only operand mutant exceeds it by at least MUTANT_X.

Where (geometry from the strings the library reports): every lengths(config(code)) of the eleven stage codes (cluster
ownership borders, every count of live CTAs in the last cluster, CTA-rank borders, L - 1 on a tile's first or last row)
with B = 1 and 3, all seven patterns at fp32 through the parity entry points; chain kernels 2, 4, 6, 7 at bf16 on the same
lengths; and ragged tables built from the ResBlock's own geometry (RbCfg border lengths, 1, 2, 8, 9, 10, HALO +- 1, P +- 1
and short items up to 256, several waves of clusters) for chain kernels 2, 4, 6, 7 at both precisions and every
pattern.  Ragged inputs hold NaN past each length, outputs are NaN-filled with a guard; per item: within the interval,
nothing written past its end (kernel 7: an exact 0 tail), the guard intact, bit-identical to its own call (a uniform
call of the items of its length; the kernels are batch-independent, test_kernel_borders_gpu).

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s).  Residual term: a c2 needed at most
5.31 x 2^-20 |x| (code 0; code 1: 1.60 x 2^-20; codes 2, 3, 12, 13: none), so RHO = 11 x 2^-20 at C >= 128.  Worst
ratio to the bound, within BAND rows of a border / elsewhere (c1 = worst of c1[0..2], likewise c2):
    code  c1           c2           fused          code  c1           c2           fused
     0    0.978/0.974  0.602/0.595  0 (exact)       13   0.970/0.977  0.172/0.177  0.081/0.092
     1    0.975/0.975  0.331/0.328  0 (exact)       14   0.038/0.045  0.007/0.009  0.007/0.007
     2    0.953/0.976  0.275/0.368  0 (exact)       20   0.982/0.977  0.978/0.975  0.219/0.181
     3    0.945/0.971  0.213/0.221  0 (exact)       21   0.964/0.975  0.977/0.976  0.116/0.133
     4    0.035/0.042  0.007/0.008  0.053/0.062     22   0.974/0.977  0.973/0.977  0.066/0.071
    12    0.978/0.978  0.246/0.333  0.142/0.170
    bf16 chain kernels 2, 4, 6: c1 1.000 (an identity read of bf16_rn(lrelu(h)) sits on an end of its interval),
    c2 0.263 / 0.130 / 0.319, fused exact; kernel 7: c1 0.621, c2 0.006, fused 0.003.
The c1 ratios near 1 are the observation, not the conv: hl(v) - v reaches 2^-16 |v| for v just above a power of two,
and the tail codes see every pattern through hl(lrelu(y)).  Ragged tables, worst item: kernels 2 / 4 / 6 / 7 at fp32
c1 0.975 / 0.976 / 0.973 / 0.040, c2 0.581 / 0.325 / 0.365 / 0.008; at bf16 c1 1.000 / 1.000 / 1.000 / 0.603, c2
0.253 / 0.122 / 0.406 / 0.007; fused exact except kernel 7 (0.007 / 0.004).  Borders never exceed the rest of the call
by more than BORDER_X.  The GPU tests of this file take 79 s.

Value-only kernel mutants, each built once from a modified copy and run once: failing cases of this file (uniform
(B, L) cases / ragged items), and the older generator tests that catch them.
    (a) stage 3's stacked c2 drops xh * wl of one k-step: codes 3, 4, 13, 14 in every c2 pattern, 31 - 38 of 32 - 38
        cases each, kernel 7 fp32 ragged 251 - 255 of 256 items (up to 83x the bound); older: test_border_sweep,
        test_narrow_codes_at_tile_borders, test_tc_gpu, test_layer_isolation_gpu (34 tests).
    (b) stage 0's cluster exchange sends Xl panel KP + 1 for panel KP at hand-off 2 (the input of c1[1]): code 0 c1.1
        70 of 76 cases, kernel 2 fp32 ragged 36 of 256 items (up to 22x); older: test_border_sweep[0], the fp32 ragged
        ResBlock check of test_gen_front_kernels_gpu, test_generator_layers_on_their_own_inputs (4 tests).
    (c) Bf16<Rb1> writes k-panel 0 of hand-off 3 truncated, not rounded: kernel 4 bf16 c1.1 52 of 52 and c2.1 51 of 52
        cases, 255 and 253 of 256 ragged items (up to 14000x); NO older test catches it (226 generator tests pass).
    (d) the tail fix-up rounds its fp32 weights to bf16: codes 20, 21, 22 fused, 38 of 38 cases each (300 - 750x);
        older: test_border_sweep[20 - 22], test_tc_gpu's tail ConvT tests and others (26 tests).
    (e) conv_post's quad reduction drops the partner lane's tap-3 sum for the last 128 rows of a CTA: codes 4 and 14 in
        every pattern (36 of 38 / 30 of 32 cases), kernel 7 at both precisions (30 of 32 cases; 18 of 256 ragged items,
        those long enough to have such rows); older: test_border_sweep, test_bf16_inference_gpu and others (48 tests).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, synth
from kernel_model import gstate  # noqa: F401 (fixture)
from kernel_model import (BAND, DILATIONS, MUTANT_X, REL_E, TAU_E, Gen64, bf16_of, bf16_rn, borders, config, fill_faults,
                          front_index, gen_weight_offset, input_shape, lengths, lrelu32, nan_buffer, res_index, split_op,
                          split_passes, split_rn, weight_grid)

RHO = 11 * 2.0 ** -20  # residual term of a C >= 128 c2 (per |x|): about twice the worst measured (module docstring)
HL_E = 2.0 ** -16    # |hi + lo - v| <= 2^-16 |v| (two bf16 roundings of 8 significant bits)
ULP_E = 2.0 ** -21   # a few fp32 ulps per add onto x and pend
POST_RSS = 4.0      # conv_post: the input bound carried as POST_RSS root-sum-squares (module docstring)
POST_E = 2.0 ** -21  # conv_post's fp32 sums (and the fp32 fold of its weights), per sum |products|
TANH_E = 2.0 ** -21  # tanhf, absolute
FIX_E = 2.0 ** -20   # the tail fix-up's fp32 dot product, per sum |products|
BORDER_X = 4.0       # ratio within BAND rows of a border <= BORDER_X * ratio elsewhere + BORDER_FLOOR
BORDER_FLOOR = 0.1

CODES = (0, 1, 2, 3, 4, 12, 13, 14, 20, 21, 22)
STAGE = {0: 0, 1: 1, 2: 2, 3: 3, 4: 3, 12: 2, 13: 3, 14: 3, 20: 0, 21: 1, 22: 2}
CHAIN_CODE = {2: 0, 4: 1, 6: 2, 7: 14}  # ResBlock kernels of the default chain -> stage code
PATTERNS = ("c1.0", "c1.1", "c1.2", "c2.0", "c2.1", "c2.2", "fused")


# ------------------------------------------------------------------------------------------------------------------
# the patterns (ordinary generator states)
# ------------------------------------------------------------------------------------------------------------------
def tail_tap(C, ci):
    """One-hot tail ConvT of a C-channel ResBlock (C -> C / 2, stride S): (co, tap) of input channel ci.  The first half
    uses x[s] taps (phase pad + co % pad), the second half x[s - 1] taps (phase co % pad, so pad > phase: the fix-up)."""
    S = 8 if C == 256 else 2
    pad = S // 2
    co = ci % (C // 2)
    return co, (pad + co % pad) if ci < C // 2 else S + co % pad


def front_tap(C, ci):
    """One-hot front ConvT (2C -> C, k4, s2): ci < C -> even outputs out[2s] = x[s] (tap 1), else odd ones (tap 2)."""
    return ci % C, 1 if ci < C else 2


def pattern_state(base, pat):
    sd = {k: v.copy() for k, v in base.items()}

    def identity(name):
        v = np.zeros_like(sd[name + ".weight_v"])
        c = v.shape[0]
        v[np.arange(c), np.arange(c), 1] = 1.0
        sd[name + ".weight_v"], sd[name + ".weight_g"] = v, np.ones_like(sd[name + ".weight_g"])

    def zero(name):
        sd[name + ".weight_g"] = np.zeros_like(sd[name + ".weight_g"])

    def one_hot(name, tap_of, C):
        v = np.zeros_like(sd[name + ".weight_v"])
        for ci in range(v.shape[0]):
            co, k = tap_of(C, ci)
            v[ci, co, k] = 1.0
        sd[name + ".weight_v"], sd[name + ".weight_g"] = v, np.ones_like(sd[name + ".weight_g"])

    for s in range(4):
        for j in range(3):
            if pat == "fused" or j != int(pat[3]):
                zero("resblocks.%d.convs2.%d" % (s, j))
        if pat != "fused":
            j = int(pat[3])
            identity("resblocks.%d.convs%d.%d" % (s, 2 if pat[:2] == "c1" else 1, j))
    if pat != "fused":
        one_hot("ups.1", tail_tap, 256)
        one_hot("ups.2", tail_tap, 128)  # = front_tap(64, .): the same tensor serves code 21's tail and code 12's front
        one_hot("ups.3", tail_tap, 64)   # = front_tap(32, .)
    return sd


def test_shared_convt_patterns_agree():
    for C in (64, 32):
        assert all(tail_tap(2 * C, ci) == front_tap(C, ci) for ci in range(2 * C)), C


def fold32(g, v):
    """The pack kernel's fold, g / sqrtf(sum v^2) * v, in fp32 (a sequential sum: one-hot or any v row of this test)."""
    g32, v32 = torch.from_numpy(g).float(), torch.from_numpy(v).float()
    ss = (v32 * v32).flatten(1).sum(1).reshape(g32.shape)
    return (g32 / torch.sqrt(ss)) * v32


@pytest.mark.parametrize("pat", PATTERNS)
def test_patterns_fold_exactly(gstate, pat):
    """Identity and one-hot layers fold to exactly 1.0 and 0.0, zeroed ones to 0.0, in float64 and in fp32."""
    sd = pattern_state(gstate, pat)
    for name, kind, *_ in synth.GENERATOR_LAYERS:
        g, v = sd[name + ".weight_g"], sd[name + ".weight_v"]
        w64 = synth.fold_weight_norm(g, v).astype(np.float64)
        w32 = fold32(g, v).double().numpy()
        if not g.any():
            assert not w64.any() and not w32.any(), name
        elif (v != 0).sum() == v.shape[0]:  # one nonzero per norm row
            assert set(np.unique(w64)) == {0.0, 1.0} and np.array_equal(w64, w32), name
            assert (w64 != 0).sum() == v.shape[0], name
    n_id = sum(1 for name, *_ in synth.GENERATOR_LAYERS if (sd[name + ".weight_v"] != 0).sum() == sd[name + ".weight_v"].shape[0])
    assert n_id == (0 if pat == "fused" else 4 + 3), (pat, n_id)
    n_zero = sum(1 for name, *_ in synth.GENERATOR_LAYERS if not sd[name + ".weight_g"].any())
    assert n_zero == 4 * (3 if pat == "fused" else 2), (pat, n_zero)


# ------------------------------------------------------------------------------------------------------------------
# the emulation: (mid, rad) of every output, |y - mid| <= rad
# ------------------------------------------------------------------------------------------------------------------
class Pattern:
    """One pattern's weights: float64 folds (Gen64), fp32 biases, and the bf16 halves the kernels read."""

    def __init__(self, state, pat, halves, device):
        self.pat, self.device = pat, device
        self.g64 = Gen64(state, device)
        self.b32 = {n: torch.from_numpy(state[n + ".bias"]).to(device) for n, *_ in synth.GENERATOR_LAYERS}
        self.halves = halves  # (kind, stage, j) -> (hi, lo) float64 in torch layout; kind "c1", "c2", "front", "tail"

    def pend(self, s, upto):
        """fp32 running sum of b2[0 .. upto) of stage s, as the kernel adds them (pend starts at 0)."""
        p = torch.zeros_like(self.b32["resblocks.%d.convs2.0" % s])
        for i in range(upto):
            p = p + self.b32["resblocks.%d.convs2.%d" % (s, i)]
        return p[None, :, None]


def conv_d(a, w, d):
    return F.conv1d(a, w, padding=d, dilation=d)


def resblock_emu(P, s, r, prec):
    """(mid, rad, rabs) of ResBlock s on the exact fp32 input r; rad excludes RHO * rabs."""
    pat, r64 = P.pat, r.double()
    pend_all = P.pend(s, 3)
    if pat == "fused":
        y = (r + pend_all).double()
        return y, ULP_E * y.abs(), torch.zeros_like(y)
    j = int(pat[3])
    d = DILATIONS[j]
    xj = r + P.pend(s, j)
    a = lrelu32(xj)
    ah, al = split_op(a, prec)
    base = r64 + pend_all.double()
    if pat[:2] == "c1":
        w64, b64 = P.g64.w["resblocks.%d.convs1.%d" % (s, j)]
        wh, wl = P.halves[("c1", s, j)]
        h = split_passes(lambda u, w: conv_d(u, w, d), ah, al, wh, wl, prec) + b64[None, :, None]
        a64 = a.double()
        B = TAU_E * conv_d(a64 * a64, w64 * w64, d).sqrt() + REL_E * h.abs()
        vlo, vhi = F.leaky_relu(h - B), F.leaky_relu(h + B)
        if prec == "bf16":
            vlo, vhi = bf16_rn(vlo), bf16_rn(vhi)
        else:
            vlo, vhi = vlo - HL_E * vlo.abs(), vhi + HL_E * vhi.abs()
        mid, half = base + (vlo + vhi) / 2, (vhi - vlo) / 2
        mag = r64.abs() + pend_all.double().abs() + torch.maximum(vlo.abs(), vhi.abs())
        return mid, half + ULP_E * mag, torch.zeros_like(mid)
    # c2[j]: c1[j] is the identity, so its output hl(a) + b1 (bf16: hi + b1) is exact in fp32
    b1 = P.b32["resblocks.%d.convs1.%d" % (s, j)][None, :, None]
    hv = ((ah + al).float() if al is not None else ah.float()) + b1
    v = lrelu32(hv)
    vh, vl = split_op(v, prec)
    w64, _ = P.g64.w["resblocks.%d.convs2.%d" % (s, j)]
    wh, wl = P.halves[("c2", s, j)]
    c = split_passes(lambda u, w: conv_d(u, w, 1), vh, vl, wh, wl, prec)
    v64 = v.double()
    mid = base + c
    rad = TAU_E * conv_d(v64 * v64, w64 * w64, 1).sqrt() + REL_E * c.abs() + ULP_E * (
        r64.abs() + pend_all.double().abs() + c.abs())
    return mid, rad, r64.abs()


def front_emu(P, s, x, prec):
    """The fused front ConvT of stage s on x [B, 2C, Lin]: (r fp32 exact, None) for the one-hot patterns, else
    (mid, rad) of its seeded output."""
    b = P.b32["ups.%d" % s][None, :, None]
    a = lrelu32(x)
    ah, al = split_op(a, prec)
    conv = lambda u, w: F.conv_transpose1d(u, w, stride=2, padding=1)
    if P.pat != "fused":
        w01 = P.g64.w["ups.%d" % s][0]
        hl = ah + al if al is not None else ah
        return (conv(hl, w01).float() + b), None
    w64, b64 = P.g64.w["ups.%d" % s]
    wh, wl = P.halves[("front", s, 0)]
    mid = split_passes(conv, ah, al, wh, wl, prec) + b64[None, :, None]
    a64 = a.double()
    return mid, TAU_E * conv(a64 * a64, w64 * w64).sqrt() + REL_E * mid.abs()


def post_emu(P, mid, rad):
    w, b = P.g64.w["conv_post"]
    a = F.leaky_relu(mid)
    z = F.conv1d(a, w, b, padding=3)
    bound = POST_RSS * F.conv1d(rad * rad, w * w, padding=3).sqrt() + POST_E * (F.conv1d(a.abs(), w.abs(), padding=3) + b.abs()[None, :, None])
    return torch.tanh(z), bound + TANH_E


def tail_emu(P, s, mid, rad):
    """The tail ConvT (stage s + 1) on the ResBlock output, with the fix-up outputs at position L."""
    name = "ups.%d" % (s + 1)
    S = 8 if s == 0 else 2
    pad, L = S // 2, mid.shape[-1]
    conv = lambda u, w: F.conv_transpose1d(u, w, stride=S, padding=pad)
    w64, b64 = P.g64.w[name]
    bias = b64[None, :, None]
    if P.pat != "fused":  # one-hot 0 / 1 weights: monotone, so the interval maps through
        vlo, vhi = F.leaky_relu(mid - rad), F.leaky_relu(mid + rad)
        vlo, vhi = vlo - HL_E * vlo.abs(), vhi + HL_E * vhi.abs()
        lo, hi = conv(vlo, w64) + bias, conv(vhi, w64) + bias
        return (lo + hi) / 2, (hi - lo) / 2 + ULP_E * (torch.maximum(lo.abs(), hi.abs()) + bias.abs())
    a = lrelu32(mid.float())  # (fused: the ResBlock output is exact, rad is a few ulps)
    ah, al = split_rn(a)
    wh, wl = P.halves[("tail", s, 0)]
    out = split_passes(conv, ah, al, wh, wl, "fp32") + bias
    a64 = a.double()
    rad_out = TAU_E * conv(a64 * a64, w64 * w64).sqrt() + REL_E * out.abs() + conv(rad, w64.abs())
    # fix-up: outputs [S L - pad, S L) from x[L - 1] and the fp32 weights
    last = a64[..., L - 1:L]
    fix = conv(last, w64)[..., S - pad:S] + bias  # (a one-position ConvT: outputs [-pad, S + pad); x[s-1] taps at S..)
    fix_abs = conv(last.abs(), w64.abs())[..., S - pad:S] + bias.abs()
    out[..., S * L - pad:] = fix
    rad_out[..., S * L - pad:] = FIX_E * fix_abs + conv(rad[..., L - 1:L], w64.abs())[..., S - pad:S]
    return out, rad_out


def emulate(P, code, x, prec="fp32"):
    """(mid, rad, rabs) of stage code `code` on x (input of the kernel, every position valid); |y - mid| <= rad + RHO
    rabs (rabs: the residual under a c2, zero past the ResBlock)."""
    s = STAGE[code]
    if code in (12, 13, 14):
        r, rad_r = front_emu(P, s, x, prec)
        if rad_r is None:
            mid, rad, rabs = resblock_emu(P, s, r, prec)
        else:  # fused: the ResBlock adds pend
            pend = P.pend(s, 3).double()
            mid, rabs = r + pend, torch.zeros_like(r)
            rad = rad_r + ULP_E * (mid.abs() + pend.abs())
    else:
        mid, rad, rabs = resblock_emu(P, s, x, prec)
    if code in (4, 14):
        mid, rad = post_emu(P, mid, rad + rho(mid.shape[1]) * rabs)
        return mid, rad, torch.zeros_like(mid)
    if code >= 20:
        mid, rad = tail_emu(P, s, mid, rad + rho(mid.shape[1]) * rabs)
        return mid, rad, torch.zeros_like(mid)
    return mid, rad, rabs


def rho(C):
    """The residual term of a c2 on C channels.  At C <= 64 the c2 MMAs put only the xh * wl products and then D onto R
    (stacked weights): a couple of fp32 roundings, which ULP_E covers."""
    return RHO if C >= 128 else 0.0


def ratio(y, emu):
    mid, rad, rabs = emu
    return (y.double() - mid).abs() / (rad + rho(mid.shape[1]) * rabs).clamp_min(1e-300)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the observation model against the float64 layers, and the bound's calibration
# ------------------------------------------------------------------------------------------------------------------
def cpu_halves(state):
    out = {}
    for s in range(4):
        for j in range(3):
            for kind, grp in (("c1", "convs1"), ("c2", "convs2")):
                n = "resblocks.%d.%s.%d" % (s, grp, j)
                out[(kind, s, j)] = split_rn(fold32(state[n + ".weight_g"], state[n + ".weight_v"]))
    for s in (1, 2, 3):
        w = split_rn(fold32(state["ups.%d.weight_g" % s], state["ups.%d.weight_v" % s]))
        out[("tail", s - 1, 0)] = w
        out[("front", s, 0)] = w
    return out


def reference64(g, code, x):
    """The float64 layers (kernel_model.Gen64) of stage code `code`."""
    s = STAGE[code]
    if code in (12, 13, 14):
        x = g.convt(s, x)
    y = g.resblock(s, x)
    if code in (4, 14):
        return g.post(y)
    if code >= 20:
        return g.convt(s + 1, y)
    return y


@pytest.mark.parametrize("pat", PATTERNS)
def test_emulator_matches_the_float64_layers(gstate, pat):
    """On the CPU, with the split of the fp32 fold as the blob, every stage code's emulation of a pattern agrees with the
    float64 layers of the same pattern's weights, within the split error: the identity routes, the sum b2 carry and the
    one-hot ConvT taps are what the emulator assumes."""
    sd = pattern_state(gstate, pat)
    P = Pattern(sd, pat, cpu_halves(sd), "cpu")
    g = Gen64(sd, "cpu")
    for code in CODES:
        C = 256 >> STAGE[code]
        shape = (2, 2 * C, 20) if code in (12, 13, 14) else (2, C, 40)
        x = torch.randn(*shape, generator=torch.Generator().manual_seed(code + 100 * PATTERNS.index(pat)))
        mid, rad, rabs = emulate(P, code, x)
        ref = reference64(g, code, x.double())
        assert mid.shape == ref.shape, (code, tuple(mid.shape), tuple(ref.shape))
        scale = ref.abs().amax(-1, keepdim=True).clamp_min(float(ref.abs().max()) / 8)
        e = float(((mid - ref).abs() / scale).max())
        assert e < 2.0 ** -12, (pat, code, e)
        assert float((rad / scale).max()) < 2.0 ** -5, (pat, code)  # the interval stays an observation, not a shrug
        assert not bool(rabs.any()) or pat[:2] == "c2", (pat, code)


@pytest.mark.parametrize("C,d,kind", [(C, d, "c1") for C in (256, 32) for d in DILATIONS] + [(256, 1, "c2"), (32, 1, "c2")])
def test_calibration(C, d, kind):
    """A float32-accumulated emulation stays under 0.5 of the bound; each value-only operand mutant exceeds it by
    >= MUTANT_X: a lo k-panel zeroed in one row, the xh * wl half of one stacked k-step dropped, one pass dropped, and
    (bf16) the hi operand truncated instead of rounded."""
    gen = torch.Generator().manual_seed(C * 10 + d)
    x = torch.randn(2, C, 300, generator=gen)
    w = (torch.rand(C, C, 3, generator=gen) * 2 - 1) / (3 * C) ** 0.5
    r = torch.randn(2, C, 300, generator=gen) if kind == "c2" else torch.zeros(2, C, 300)
    dd = d if kind == "c1" else 1
    conv = lambda u, ww: conv_d(u, ww, dd)
    a = lrelu32(x)
    ah, al = split_rn(a)
    wh, wl = split_rn(w)
    a64, w64, r64 = a.double(), w.double(), r.double()
    a2 = conv(a64 * a64, w64 * w64).sqrt()
    res = (rho(C) + ULP_E) * r64.abs() if kind == "c2" else 0.0

    def ratio_of(y, emu):
        c = (emu - r64).abs()
        return float(((y.double() - emu).abs() / (TAU_E * a2 + REL_E * c + res)).max())

    emu3, emu1 = r64 + split_passes(conv, ah, al, wh, wl, "fp32"), r64 + split_passes(conv, ah, al, wh, wl, "bf16")
    # float32, in the kernel's order: per (tap, 16-channel k-step, pass) an fp32 partial sum onto the accumulator
    f = lambda t: t.float()

    def f32(ops):
        acc = r.clone()
        for tap in range(3):
            for k0 in range(0, C, 16):
                for xa, ww in ops:
                    wt = torch.zeros(C, 16, 3)
                    wt[:, :, tap] = f(ww)[:, k0:k0 + 16, tap]
                    acc = acc + conv(f(xa)[:, k0:k0 + 16], wt)
        return acc.double()

    clean3 = ratio_of(f32([(ah, wh), (al, wh), (ah, wl)]), emu3)
    clean1 = ratio_of(f32([(ah, wh)]), emu1)
    mutants = {}
    m = al.clone()
    m[:, 8:16, 150] = 0
    mutants["lo of one k-panel of one row zeroed"] = (r64 + split_passes(conv, ah, m, wh, wl, "fp32"), emu3)
    dwl = wl.clone()
    dwl[:, 16:32, 1] = 0
    mutants["xh * wl of one stacked k-step dropped"] = (r64 + split_passes(conv, ah, al, wh, dwl, "fp32"), emu3)
    mutants["pass (xl, wh) dropped"] = (r64 + split_passes(conv, ah, torch.zeros_like(al), wh, wl, "fp32"), emu3)
    trunc = (a.view(torch.int32) & -65536).view(torch.float32).double()
    mutants["hi truncated (bf16)"] = (r64 + conv(trunc, wh), emu1)
    print("\nC %d, dilation %d, %s: float32 accumulation %.3f (fp32) / %.3f (bf16) of the bound" % (C, dd, kind, clean3, clean1))
    assert clean3 < 0.5 and clean1 < 0.5, (clean3, clean1)
    for name, (y, emu) in mutants.items():
        rm = ratio_of(y, emu)
        print("  %-40s %7.1f x the bound" % (name, rm))
        assert rm >= MUTANT_X, (C, d, kind, name, rm)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def blob_halves(dev):
    blob = dev.packed.view(torch.int16)
    out = {}
    for s in range(4):
        C = 256 >> s
        co, ci, tap = np.meshgrid(np.arange(C), np.arange(C), np.arange(3), indexing="ij")
        for j in range(3):
            for kind, l in (("c1", 5 + 6 * s + j), ("c2", 5 + 6 * s + 3 + j)):
                out[(kind, s, j)] = tuple(bf16_of(blob, res_index(C, l, co, ci, tap, h)).double() for h in (0, 1))
    for s in (1, 2, 3):  # the tail ConvT streams ups.s's blob (the ConvT kernel's own layout)
        out[("tail", s - 1, 0)] = tuple(bf16_of(blob, gen_weight_offset(1 + s, *weight_grid(1 + s), h)).double() for h in (0, 1))
    for s in (2, 3):
        C = 256 >> s
        ci, co, k = np.meshgrid(np.arange(2 * C), np.arange(C), np.arange(4), indexing="ij")
        out[("front", s, 0)] = tuple(bf16_of(blob, front_index(C, s, ci, co, k, h)).double() for h in (0, 1))
    return out


@pytest.fixture(scope="module")
def packs(gstate):
    """pattern -> (GeneratorDevice, Pattern with the halves read back from its blob)."""
    out = {}
    order = [n for n, *_ in synth.GENERATOR_LAYERS]
    for pat in PATTERNS:
        sd = pattern_state(gstate, pat)
        dev = engine.GeneratorDevice("cuda:0")
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        dev.pack([to(sd[n + ".weight_v"]) for n in order], [to(sd[n + ".weight_g"]) for n in order],
                 [to(sd[n + ".bias"]) for n in order])
        torch.cuda.synchronize()
        out[pat] = (dev, Pattern(sd, pat, blob_halves(dev), "cuda"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("pat", PATTERNS)
def test_blob_holds_the_patterns(packs, pat):
    """The one-hot and identity weights are hi = 1, lo = 0 and the zeroed convs 0, at the offsets the descriptors read;
    the seeded ones are the split of the fold."""
    _, P = packs[pat]
    for key, (hi, lo) in P.halves.items():
        kind, s, j = key
        if kind in ("c1", "c2"):
            w = P.g64.w["resblocks.%d.convs%s.%d" % (s, kind[1], j)][0]
        else:
            w = P.g64.w["ups.%d" % (s + 1 if kind == "tail" else s)][0]
        assert hi.shape == w.shape, key
        if not bool((w != 0).any()) or bool(((w == 0) | (w == 1)).all()):
            assert torch.equal(hi, w) and not bool(lo.any()), (pat, key)
        else:
            assert float((hi + lo - w).abs().max()) <= 2.0 ** -15 * float(w.abs().max()), (pat, key)
    if pat != "fused":
        j = int(pat[3])
        ident = P.halves[("c2" if pat[:2] == "c1" else "c1", 0, j)][0]
        assert float(ident.sum()) == 256 and float(ident[:, :, 1].diagonal().sum()) == 256, pat


def run_code(dev, code, x):
    if code <= 3:
        return dev.resblock(code, x)
    if code == 4:
        return dev.resblock_post(x)
    if code in (12, 13):
        return dev.upres(code - 10, x)
    if code == 14:
        return dev.upres_post(x)
    return dev.resup(code - 20, x)


def near_mask(g, code, B, L, n):
    """[n] outputs within BAND rows of an ownership border or of the item's ends."""
    S = g["UPT"] or 1
    near = torch.zeros(n, dtype=torch.bool, device="cuda")
    for b in borders(g, L) + [0, L]:
        t = S * b - S // 2 if S > 1 else b
        near[max(0, t - BAND * S):min(n, t + BAND * S + 1)] = True
    return near


class Tally:
    def __init__(self):
        self.near = self.far = self.rho = 0.0
        self.fails = []

    def add(self, y, emu, near, tag):
        r = ratio(y, emu).amax(dim=(0, 1))
        worst = float(torch.nan_to_num(r, nan=1e30).max())
        if not worst <= 1:
            i = int(torch.argmax(torch.nan_to_num(r, nan=1e30)))
            self.fails.append(tag + (round(worst, 2), i))
        if near is not None:
            self.near = max(self.near, float(r[near].max()) if near.any() else 0.0)
            self.far = max(self.far, float(r[~near].max()) if (~near).any() else 0.0)
        mid, rad, rabs = emu
        if bool(rabs.any()):  # what of |y - mid| the RHO term has to cover, per |x|
            ex = ((y.double() - mid).abs() - rad).clamp_min(0) / rabs.clamp_min(1e-30)
            self.rho = max(self.rho, float(torch.nan_to_num(ex, nan=0).max()))
        return worst


@pytest.mark.gpu
@pytest.mark.parametrize("pat", PATTERNS)
@pytest.mark.parametrize("code", CODES)
def test_uniform_lengths_fp32(packs, code, pat):
    dev, P = packs[pat]
    g = config(code)
    T = Tally()
    for L in lengths(g):
        for B in (1, 3):
            rs = np.random.RandomState(code * 100003 + L * 7 + B)
            x = torch.from_numpy(rs.standard_normal(input_shape(g, code, B, L)).astype(np.float32)).cuda()
            y = run_code(dev, code, x)
            emu = emulate(P, code, x)
            assert y.shape == emu[0].shape, (code, B, L)
            T.add(y, emu, near_mask(g, code, B, L, y.shape[-1]), (B, L))
    print("\ncode %d %s fp32: near borders %.3f, elsewhere %.3f of the bound%s" % (
        code, pat, T.near, T.far, ", residual term needed %.2f x 2^-20" % (T.rho * 2 ** 20) if pat[:2] == "c2" else ""))
    assert not T.fails, ("%d of %d (B, L) fail" % (len(T.fails), 2 * len(lengths(g))), T.fails[:4])
    assert T.near <= BORDER_X * T.far + BORDER_FLOOR, (T.near, T.far)


def chain_input(code, g, B, L, seed):
    rs = np.random.RandomState(seed)
    return torch.from_numpy(rs.standard_normal(input_shape(g, code, B, L)).astype(np.float32)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("pat", PATTERNS)
@pytest.mark.parametrize("k", [2, 4, 6, 7])
def test_uniform_lengths_bf16(packs, k, pat):
    dev, P = packs[pat]
    code = CHAIN_CODE[k]
    g = config(code)
    T = Tally()
    for L in lengths(g):
        for B in (1, 3):
            x = chain_input(code, g, B, L, code * 7 + L * 13 + B)
            y = dev.chain_kernel(k, x, None, "bf16")
            T.add(y, emulate(P, code, x, "bf16"), near_mask(g, code, B, L, y.shape[-1]), (B, L))
    print("\nchain kernel %d %s bf16: near borders %.3f, elsewhere %.3f of the bound" % (k, pat, T.near, T.far))
    assert not T.fails, ("%d of %d (B, L) fail" % (len(T.fails), 2 * len(lengths(g))), T.fails[:4])
    assert T.near <= BORDER_X * T.far + BORDER_FLOOR, (T.near, T.far)


def ragged_lengths(code):
    """Item lengths (ResBlock positions) of one ragged launch: the RbCfg border lengths, 1, 2, 8, 9, 10, HALO +- 1, P +- 1,
    then short items up to 256 of them (several waves of clusters)."""
    g = config(code)
    Ls = lengths(g) + [1, 2, 8, 9, 10, g["HALO"] - 1, g["HALO"], g["HALO"] + 1, g["P"] - 1, g["P"], g["P"] + 1]
    if g["UPF"]:
        Ls = [L + L % 2 for L in Ls]
    rs = np.random.RandomState(code + 7)
    Ls = [int(v) for v in rs.permutation(Ls)]
    Ls += [int(v) for v in rs.randint(1, 11, 256 - len(Ls)) * (2 if g["UPF"] else 1)]
    return Ls


@pytest.mark.parametrize("code", sorted(CHAIN_CODE.values()))
def test_ragged_tables_reach_every_kind_of_length(code):
    g = config(code)
    Ls = ragged_lengths(code)
    assert len(Ls) == 256 and min(Ls) >= 1 and (not g["UPF"] or all(L % 2 == 0 for L in Ls))
    even = (lambda L: L + L % 2) if g["UPF"] else (lambda L: L)
    for L in lengths(g) + [1, 2, 8, 9, 10, g["HALO"] - 1, g["HALO"] + 1, g["P"] - 1, g["P"] + 1]:
        assert even(L) in Ls, (code, L)
    units = lambda L: 1 + ((L - g["PC"] + g["PVB"] - 1) // g["PVB"] if L > g["PC"] else 0)
    assert g["CS"] * sum(units(L) for L in Ls) > 2 * 132  # more CTAs than two waves of the SMs


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("pat", PATTERNS)
@pytest.mark.parametrize("k", [2, 4, 6, 7])
def test_ragged_tables(packs, k, pat, precision):
    dev, P = packs[pat]
    code = CHAIN_CODE[k]
    g = config(code)
    cin, _, R = dev.CHAIN_SHAPES[k]
    per = 2 if g["UPF"] else 1  # ResBlock positions per input position
    lens = [L // per for L in ragged_lengths(code)]
    B, Lmax = len(lens), max(lens)
    x = chain_input(code, g, B, Lmax * per, 31 * k + PATTERNS.index(pat))
    valid = torch.arange(Lmax, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    x[~valid[:, None, :].expand_as(x)] = float("nan")
    buf = nan_buffer(B * dev.CHAIN_SHAPES[k][1] * R * Lmax)
    y = dev.chain_kernel(k, x, lens, precision, out=buf)
    bad = {}
    for i in fill_faults(y, buf, lens, R, zero_tail=k == 7):
        bad.setdefault(i, []).append("written past its end or the guard")
    T = Tally()
    for Li in sorted(set(lens)):
        idx = [i for i, v in enumerate(lens) if v == Li]
        xi = x[idx, :, :Li].contiguous()
        own = dev.chain_kernel(k, xi, None, precision)
        yi = y[idx, :, :R * Li]
        for n, i in enumerate(idx):
            if not torch.equal(own[n], yi[n]):
                bad.setdefault(i, []).append("differs from its own call")
        r = ratio(yi, emulate(P, code, xi, precision)).flatten(1).amax(1)
        for n, i in enumerate(idx):
            if not float(r[n]) <= 1:
                bad.setdefault(i, []).append("%.2f x the bound" % float(r[n]))
        T.near = max(T.near, float(torch.nan_to_num(r, nan=1e30).max()))
    print("\nchain kernel %d %s %s ragged: %d items, worst %.3f of the bound" % (k, pat, precision, B, T.near))
    assert not bad, ("%d of %d items fail" % (len(bad), B), sorted((lens[i], v) for i, v in bad.items())[:6])
