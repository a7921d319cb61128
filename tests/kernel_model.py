"""What the tests know about the kernels, stated once: the split-bf16 arithmetic, where the packed blobs keep each weight,
the launch geometry the library reports, guarded output buffers, the float64 layer models and the fixtures that pack
them.  A change to a kernel's layout or tiling updates its restatement here; the test files import what they use by name.

The fixtures are module-scoped: each test module that imports one gets its own packed state."""
import ctypes
import math
import random
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, models, synth
from oracle import cport


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------------------------
# 1. split arithmetic: hi = bf16_rn(v), lo = bf16_rn(v - hi), and the tensor cores' passes over the halves
# ------------------------------------------------------------------------------------------------------------------
# 2^-16 covers a float32-accumulated emulation with room (test_tau_calibration); the H100's MMA accumulation measured up to
# 1.43 x 2^-16 (up0, spread over the whole tile rather than at its borders: test_gen_front_kernels_gpu), so TAU_E is about
# twice that
TAU_E = 3 * 2.0 ** -16
REL_E = 2.0 ** -22
MUTANT_X = 4  # each operand mutant exceeds the bound by at least this factor


def bf16_rn(v):
    return v.to(torch.bfloat16).to(v.dtype)


def bf16_rn64(t):
    """bf16_rn, returned as float64."""
    return t.to(torch.bfloat16).to(torch.float64)


def lrelu32(x):
    return torch.maximum(x, x * torch.tensor(0.01, dtype=torch.float32, device=x.device))


def split_rn(v):
    """hi = bf16_rn(v), lo = bf16_rn(v - hi) of an fp32 tensor (split2_bf16), as float64."""
    hi = bf16_rn(v)
    return hi.double(), bf16_rn(v - hi).double()


def split_np(v):
    """split_rn of an fp32 numpy array, as float64 numpy arrays."""
    hi, lo = split_rn(torch.from_numpy(np.ascontiguousarray(v, np.float32)))
    return hi.numpy(), lo.numpy()


def split_op(a, prec):
    """split_rn(a); bf16 runs one pass per product, so it has no lo half."""
    ah, al = split_rn(a)
    return ah, (None if prec == "bf16" else al)


def split_passes(f, ah, al, wh, wl, prec="fp32"):
    """float64 sum of the passes of a bilinear f on split operands (no bias): (ah, wh) + (al, wh) + (ah, wl) at fp32,
    summed as (ah + al, wh) + (ah, wl) since (ah + al) and each product are exact in float64; (ah, wh) alone at bf16."""
    return f(ah, wh) if prec == "bf16" else f(ah + al, wh) + f(ah, wl)


def split_conv(x, w, stride, padding, groups, passes=(0, 1, 2)):
    """The tensor cores' arithmetic on fp32 operands: hi = bf16(v), lo = bf16(v - hi); passes (xh, wh), (xl, wh), (xh, wl)
    accumulated in fp32."""
    xh, wh = bf16_rn(x), bf16_rn(w)
    xl, wl = bf16_rn(x - xh), bf16_rn(w - wh)
    ops = [(xh, wh), (xl, wh), (xh, wl)]
    y = torch.zeros(())
    for p in passes:
        y = y + F.conv1d(ops[p][0], ops[p][1], None, stride=stride, padding=padding, groups=groups)
    return y


# ------------------------------------------------------------------------------------------------------------------
# 2. reading the packed blobs
# ------------------------------------------------------------------------------------------------------------------
def bf16_of(blob_i16, offsets):
    """The bf16 values at byte offsets (numpy) of an int16 view of a packed blob, as fp32."""
    idx = torch.from_numpy(np.ascontiguousarray(offsets // 2)).to(blob_i16.device)
    return (blob_i16[idx].to(torch.int32) << 16).view(torch.float32)


def lib_offset():
    f = engine.lib().mg_gen_tc_weight_offset
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.c_int] * 6
    return f


# ------------------------------------------------------------------------------------------------------------------
# 3. the generator's blob (restated from csrc/mg_layout.h)
# ------------------------------------------------------------------------------------------------------------------
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


def res_index(C, layer, co, ci, tap, h):
    """Byte offset of half h of ResBlock conv `layer`'s w[co][ci][tap]: chunks of (tap, K-slice) in consumption order."""
    KC = tc_kc(C)
    return res_base(layer) + 2 * ((tap * (C // KC) + ci // KC) * 2 * KC * C + in_chunk(C, co, ci % KC, h))


def front_index(C, s, ci, co, k, h):
    """Byte offset of half h of W[ci][co][k] of the front ConvT of the fused stage-s kernel (ResBlock-style chunks)."""
    assert C == 256 >> s, (C, s)
    return upf_index(s, ci, co, k, h)


# (Cin, Cout, R = outputs per input position, K); layer index in the blob: pre 0, up s -> 1 + s
SHAPE = {"pre": (80, 512, 1, 7), "up0": (512, 256, 8, 16), "up1": (256, 128, 8, 16), "up2": (128, 64, 2, 4),
         "up3": (64, 32, 2, 4)}


def up_tc_bytes(s):
    return (512 >> s) * (256 >> s) * (16 if s < 2 else 4) * 4


def up_base(s):
    """ConvT s's block: after the 24 ResBlock convs, the ConvTs in stage order; conv_pre after the four."""
    return res_base(29) + sum(up_tc_bytes(i) for i in range(s))


def gen_weight_offset(layer, a, b, tap, h):
    """Byte offset of half h of w[a = co][b = ci][tap] (conv_pre, layer 0) or W[a = ci][b = co][tap] (ups[layer - 1]);
    numpy arrays welcome.  conv_pre: ring slots of (128-channel group, 16-channel chunk, tap), each [half][k-panel][co][8];
    a ConvT: slots of (NG-channel group, 16-channel chunk), each [tap][half][k-panel][phase * NG + co][8]."""
    if layer == 0:
        co, ci, NG = a, b, 128
        i = ((((co // NG * 5 + ci // 16) * 7 + tap) * 2 + h) * 2 + ci % 16 // 8) * NG * 8 + co % NG * 8 + ci % 8
        return up_base(4) + 2 * i
    s = layer - 1
    ci, co = a, b
    S, NG, CIN = (8 if s < 2 else 2), (64 if s == 2 else 32), 512 >> s
    phi, t = tap % S, tap // S
    i = ((((co // NG * (CIN // 16) + ci // 16) * 2 + t) * 2 + h) * 2 + ci % 16 // 8) * (S * NG) * 8 + (phi * NG + co % NG) * 8 + ci % 8
    return up_base(s) + 2 * i


def weight_grid(layer):
    """Index arrays over the whole weight tensor of conv_pre (layer 0) or ups[layer - 1], in its torch layout."""
    k = ("pre", "up0", "up1", "up2", "up3")[layer]
    cin, cout, _, K = SHAPE[k]
    dims = (cout, cin, K) if layer == 0 else (cin, cout, K)
    return np.meshgrid(*(np.arange(n) for n in dims), indexing="ij")


# the fp32 part of the blob: every layer's folded weights in layer order, then every bias (csrc/mg_layout.h weight_offset,
# bias_offset); Conv1d w[co][ci][tap] at [ci][tap][co], ConvTranspose1d W[ci][co][k] at [ci][co][k % S][k // S] (S = K / 2)
GEN_LAYERS = synth.GENERATOR_LAYERS  # (name, kind, Cin, Cout, K); layer l of the blob is GEN_LAYERS[l]


def gen_fp32_weight_offset(l):
    """Float offset of layer l's fp32 weights."""
    return sum(cin * cout * k for _n, _kind, cin, cout, k in GEN_LAYERS[:l])


def gen_bias_offset(l):
    """Float offset of layer l's bias."""
    return gen_fp32_weight_offset(len(GEN_LAYERS)) + sum(cout for _n, _kind, _ci, cout, _k in GEN_LAYERS[:l])


GEN_FP32_BYTES = 4 * gen_bias_offset(len(GEN_LAYERS))
GEN_TC_START = cdiv(GEN_FP32_BYTES, 256) * 256


def gen_fp32_index(l, a, b, tap):
    """Byte offset of the fp32 copy of layer l's weight at [a][b][tap] of its torch layout (a = co, b = ci for a Conv1d;
    a = ci, b = co for a ConvTranspose1d); numpy arrays welcome."""
    _n, kind, cin, cout, K = GEN_LAYERS[l]
    o = gen_fp32_weight_offset(l)
    if kind == "conv":
        return 4 * (o + (b * K + tap) * cout + a)
    S = K // 2
    return 4 * (o + ((a * cout + b) * S + tap % S) * 2 + tap // S)


def upf_base(s):
    """The fused stride-2 ConvT copies (stages 2, 3) follow conv_pre's block: 2C x C x 4 taps x (hi, lo) each."""
    return up_base(4) + 80 * 512 * 7 * 4 + (32 * 64 * 64 if s == 3 else 0)


def upf_index(s, ci, co, k, h):
    """Byte offset of half h of ups[s]'s W[ci][co][k] in its fused-kernel copy (ResBlock-style chunks, 4 taps over 2C
    input channels); numpy arrays welcome.  front_index without the library."""
    C = 256 >> s
    KC = tc_kc(C)
    return upf_base(s) + 2 * ((k * (2 * C // KC) + ci // KC) * 2 * KC * C + in_chunk(C, co, ci % KC, h))


GEN_BLOB_BYTES = upf_base(3) + 32 * 32 * 32


def gen_grid(l):
    """Index arrays (a, b, tap) over layer l's whole weight tensor in its torch layout (v's layout: a is the norm row)."""
    _n, kind, cin, cout, K = GEN_LAYERS[l]
    dims = (cout, cin, K) if kind == "conv" else (cin, cout, K)
    return np.meshgrid(*(np.arange(n) for n in dims), indexing="ij")


def gen_split_copies(l):
    """{copy name: offset function (a, b, tap, h) -> byte offset} of layer l's split-bf16 copies, in torch-layout
    indices: conv_pre's ring slots, a ConvT's ring slots (and the fused copy of stages 2 and 3), a ResBlock conv's chunks;
    conv_post has none."""
    if l == 0:
        return {"tc": lambda a, b, t, h: gen_weight_offset(0, a, b, t, h)}
    if l <= 4:
        out = {"tc": lambda a, b, t, h: gen_weight_offset(l, a, b, t, h)}
        if l >= 3:
            out["upf"] = lambda a, b, t, h: upf_index(l - 1, a, b, t, h)
        return out
    if l <= 28:
        C = GEN_LAYERS[l][3]
        return {"tc": lambda a, b, t, h: res_index(C, l, a, b, t, h)}
    return {}


def gen_regions():
    """[(name, start, end, padding)] of the generator's blob in address order: the fp32 weights and biases, the padding to
    the 256-byte aligned tensor-core region, the 24 ResBlock convs, the four ConvTs, conv_pre, the two fused ConvTs."""
    L = len(GEN_LAYERS)
    out = [("fp32 " + GEN_LAYERS[l][0], 4 * gen_fp32_weight_offset(l), 4 * gen_fp32_weight_offset(l + 1), False) for l in range(L)]
    out += [("bias " + GEN_LAYERS[l][0], 4 * gen_bias_offset(l), 4 * gen_bias_offset(l + 1), False) for l in range(L)]
    out.append(("padding", GEN_FP32_BYTES, GEN_TC_START, True))
    out += [("tc " + GEN_LAYERS[l][0], res_base(l), res_base(l + 1), False) for l in range(5, 29)]
    out += [("tc ups.%d" % s, up_base(s), up_base(s) + up_tc_bytes(s), False) for s in range(4)]
    out.append(("tc conv_pre", up_base(4), upf_base(2), False))
    out += [("upf ups.2", upf_base(2), upf_base(3), False), ("upf ups.3", upf_base(3), GEN_BLOB_BYTES, False)]
    return out


# ------------------------------------------------------------------------------------------------------------------
# 4. the blob of one discriminator (restated from csrc/mg_layout.h) and its launch geometry
# ------------------------------------------------------------------------------------------------------------------
LAYERS = synth.DISCRIMINATOR_LAYERS


def _fp32_floats():
    w = sum(0 if n == "conv_post1" else cout * (cin // g) * k for n, cin, cout, k, _s, g, _p in LAYERS)
    return w + sum(cout for _n, _ci, cout, *_ in LAYERS)


def disc_weight_offset(l):
    """Float offset of layer l's fp32 weights (grouped layers: [group][ci 4][tap 41][co within group])."""
    return sum(0 if n == "conv_post1" else cout * (cin // g) * k for n, cin, cout, k, _s, g, _p in LAYERS[:l])


def disc_bias_offset(l):
    return disc_weight_offset(7) + sum(cout for _n, _ci, cout, *_ in LAYERS[:l])


TC_BYTES = 1024 * 1024 * 5 * 4
GTC_GROUP, G4TC_GROUP = 7 * 2 * 2 * 64 * 16, 6 * 2 * 2 * 64 * 16
GROUPS = {1: 4, 2: 16, 3: 64, 4: 256}
TC_START = cdiv(_fp32_floats() * 4, 256) * 256
GTC_START = TC_START + TC_BYTES
G4TC_START = GTC_START + (4 + 16 + 64) * GTC_GROUP
TCT_START = G4TC_START + 256 * G4TC_GROUP
BLOB_BYTES = TCT_START + TC_BYTES + 4096


def gtc_start(l):
    return GTC_START + sum(GROUPS[i] for i in range(1, l)) * GTC_GROUP


D_FP32_BYTES = 4 * _fp32_floats()
ZERO_START = TCT_START + TC_BYTES  # 1024 zero floats: the conv_post1 dgrad launch's "bias"


def disc_fp32_index(l, co, ci, tap):
    """Byte offset of the fp32 copy of layer l's w[co][ci][tap] (every layer but conv_post1): conv_pre [tap][co 16],
    grouped [group][ci 4][tap 41][co within group], conv_post2 [ci][tap]; numpy arrays welcome."""
    _n, cin, cout, k, _s, groups, _p = LAYERS[l]
    o = disc_weight_offset(l)
    if l == 0:
        return 4 * (o + tap * cout + co)
    if l <= 4:
        cog = cout // groups
        return 4 * (o + ((co // cog * (cin // groups) + ci) * k + tap) * cog + co % cog)
    assert l == 6, l
    return 4 * (o + ci * k + tap)


def disc_regions():
    """[(name, start, end, padding)] of one discriminator's blob in address order: the fp32 weights (none for conv_post1)
    and biases, the padding to the 256-byte aligned tensor-core part, conv_post1's copy, the Toeplitz copies of
    grouped_convs.0-2 and .3, conv_post1's transposed copy, the zero row."""
    out = [("fp32 " + LAYERS[l][0], 4 * disc_weight_offset(l), 4 * disc_weight_offset(l + 1), False) for l in range(7) if l != 5]
    out += [("bias " + LAYERS[l][0], 4 * disc_bias_offset(l), 4 * disc_bias_offset(l + 1), False) for l in range(7)]
    out.append(("padding", D_FP32_BYTES, TC_START, True))
    out.append(("tc conv_post1", TC_START, GTC_START, False))
    out += [("toeplitz " + LAYERS[l][0], gtc_start(l), gtc_start(l + 1), False) for l in (1, 2, 3)]
    out += [("toeplitz " + LAYERS[4][0], G4TC_START, TCT_START, False), ("tcT conv_post1", TCT_START, ZERO_START, False),
            ("zero row", ZERO_START, BLOB_BYTES, False)]
    return out


def toeplitz_slots(l):
    """Every bf16 element of layer l's Toeplitz copy (l = 1..4) as arrays (offset, h, co, ci, tap), h = 2 for a structural
    zero.  l = 1..3: block row n = [half][parity e][co 16], element (pos, ci) of k-panel kp of phase r holds tap
    4 q + r, q = 2 kp + pos - 1 - e.  l = 4: n = [half][e 8][co 4], element i of k-panel kp of channel ci holds tap
    8 kp + i - e."""
    if l <= 3:
        grp, kp, r, half, e, col, pos, ci = np.meshgrid(*(np.arange(v) for v in (GROUPS[l], 7, 4, 2, 2, 16, 2, 4)), indexing="ij")
        n = half * 32 + e * 16 + col
        idx = (((kp * 2 + r // 2) * 2 + r % 2) * 64 + n) * 8 + pos * 4 + ci
        off = gtc_start(l) + grp * GTC_GROUP + 2 * idx
        q = 2 * kp + pos - 1 - e
        tap = 4 * q + r
        valid = (q >= 0) & (tap <= 40)
        co = grp * 16 + col
    else:
        grp, kp, ci, half, e, col, i = np.meshgrid(*(np.arange(v) for v in (256, 6, 4, 2, 8, 4, 8)), indexing="ij")
        n = half * 32 + e * 4 + col
        idx = (((kp * 2 + ci // 2) * 2 + ci % 2) * 64 + n) * 8 + i
        off = G4TC_START + grp * G4TC_GROUP + 2 * idx
        tap = 8 * kp + i - e
        valid = (tap >= 0) & (tap <= 40)
        co = grp * 4 + col
    h = np.where(valid, half, 2)
    return tuple(a.ravel() for a in (off, h, co, ci, tap))


def post1_offset(co, ci, tap, h, transposed=False):
    """Byte offset of half h of conv_post1's w[co][ci][tap]: ring slots of (128-channel group, 16-channel chunk, tap), each
    [half][k-panel][row][8]; the transposed copy holds it at row ci, column co, tap 4 - tap.  numpy arrays welcome."""
    a, b, t = (ci, co, 4 - tap) if transposed else (co, ci, tap)
    i = (((((a // 128) * 64 + b // 16) * 5 + t) * 2 + h) * 2 + (b % 16) // 8) * 1024 + (a % 128) * 8 + b % 8
    return (TCT_START if transposed else TC_START) + 2 * i


def post1_slots(transposed):
    co, ci, tap, h = np.meshgrid(np.arange(1024), np.arange(1024), np.arange(5), np.arange(2), indexing="ij")
    return tuple(a.ravel() for a in (post1_offset(co, ci, tap, h, transposed), h, co, ci, tap))


def slots(copy):
    """(offset, h, co, ci, tap) of every element of copy 1..6 (mg_disc_tc_element's numbering)."""
    return toeplitz_slots(copy) if copy <= 4 else post1_slots(copy == 6)


PANELS = 7                       # kDgPanels (csrc/mg_layout.h): an item's halo is PANELS - 1 units
UNITS = 134                      # dg::UNITS = 128 + kDgPanels - 1: 16-byte units (output pairs) per phase buffer
PANELS4 = 6                      # kDg4Panels (csrc/mg_layout.h)
UNITS4 = 133                     # dg4::UNITS = 128 + kDg4Panels - 1 (disc_group4_tc_kernel): units of 8 positions
LANE4 = 8                        # disc_group4_tc_kernel: outputs per accumulator row
POST1_ROWS, POST1_PAD = 128, 2   # conv_rows_tc_kernel<Post1Cfg> / <Post1DgradCfg> (csrc/mg_conv_tc.cu): virtual rows per
                                 # CTA, zero rows after each item (L + 2 rows per item)
WG_PANEL, WG_STAGE = 8, 32       # post1_wgrad_tc_kernel: positions per k-panel (per item) and per stage

GROUP_TARGETS = (1, 2, 3, 13, 14, 121, 122, 123, 124, 255, 256, 257, 512, 513)  # Lout of grouped_convs.0-2
GROUP4_TARGETS = (1, 7, 8, 9, 487, 488, 489, 1023, 1024, 1025, 2048, 2049)      # L of grouped_convs.3


def group_tc_plan(Lout):
    """(rp, ni) of launch_disc_group_tc: ni items per CTA at a pitch of rp units (the item's ceil(Lout / 2) output pairs
    + 6 halo units) while two fit, else (None, 1): 256-output tiles of one item."""
    rp = cdiv(Lout, 2) + PANELS - 1
    ni = UNITS // rp
    return (rp, ni) if ni > 1 else (None, 1)


def group4_plan(L):
    """(ni, segs) of launch_disc_group4_tc: ni = 133 // (nb + 5) items per tile with nb = ceil(L / 8) lanes each; items
    longer than 128 lanes take segs = ceil(nb / 128) tiles of one item."""
    nb = cdiv(L, LANE4)
    ni = UNITS4 // (nb + PANELS4 - 1)
    return (ni, 1) if ni >= 1 else (1, cdiv(nb, 128))


def batches(ni):
    return {1, ni - 1, ni, ni + 1, 2 * ni + 1} - {0} if ni > 1 else {1, 3}


def post1_lengths():
    """conv_post1 dgrad (128 virtual rows, L + 2 rows per item) and wgrad (8-position k-panels per item, 32-position
    stages): L < 5, L % 4 != 0, L % 8 != 0, part-filled stages, items that tile the 128 rows exactly or straddle two."""
    R, P = POST1_ROWS, POST1_PAD
    return [1, 3, 4, 5, 7, WG_PANEL + 1, 17, WG_STAGE - 1, WG_STAGE, WG_STAGE + 1, R // 2 - P, R // 2 - P + 1, 65,
            R - P, R - P + 1]


def post1_straddles(Bt, L):
    """An item's L + 2 virtual rows straddle two 128-row tiles of the dgrad launch."""
    return any((i * (L + POST1_PAD)) // POST1_ROWS != ((i + 1) * (L + POST1_PAD) - 1) // POST1_ROWS for i in range(Bt))


def tau_simt(n):
    """Element-wise tau of an fp32 SIMT sum of n products (test_disc_backward_isolation_gpu's module docstring)."""
    return 2.0 ** -20 * math.sqrt(n)


SIMT_N = (3, 24, 164, 176, 240, 393, 1024, 2048)  # calibrated n; every n a GPU test uses must be <= the largest


def upstream(fm, pattern):
    """Gradients w.r.t. the 21 stacked maps fm[s][l] (first half real, second half generated), through the package's
    loss functions: "generator" = feature-map L1 + LSGAN generator term (every map), "discriminator" = the LSGAN
    discriminator loss (the logits only), "map 3" = the generator step's gradient on map 3 alone."""
    leaves = [[f.detach().clone().requires_grad_(True) for f in sc] for sc in fm]
    B = leaves[0][0].shape[0] // 2
    d_r = [torch.flatten(sc[6][:B], 1) for sc in leaves]
    d_g = [torch.flatten(sc[6][B:], 1) for sc in leaves]
    if pattern == "discriminator":
        loss = models.discriminator_loss(d_r, d_g)[0]
    else:
        loss = models.feature_loss([[f[:B] for f in sc] for sc in leaves], [[f[B:] for f in sc] for sc in leaves])
        loss = loss + models.generator_loss(d_g)
    flat = [f for sc in leaves for f in sc]
    gr = torch.autograd.grad(loss, flat, allow_unused=True)
    G = [list(gr[7 * s:7 * s + 7]) for s in range(3)]
    if pattern == "map 3":
        G = [[g if l == 3 else None for l, g in enumerate(Gs)] for Gs in G]
    return G


# ------------------------------------------------------------------------------------------------------------------
# 5. the ResBlock kernels' launch geometry (pure functions of the configuration string the library reports)
# ------------------------------------------------------------------------------------------------------------------
BAND = 20        # rows either side of a border


def parse_config(name):
    """"resblock_tc_kernel<RbCfg<C,NRB,RPW,NCP,NSTAGE,POST,UPF,UPT,CS>>" -> dict with the tiling constants."""
    m = re.fullmatch(r"resblock_tc_kernel<RbCfg<(\d+(?:,\d+){8})>>", name)
    if not m:
        raise ValueError("not a ResBlock configuration: %r" % (name,))
    C, NRB, RPW, NCP, NSTAGE, POST, UPF, UPT, CS = (int(v) for v in m.group(1).split(","))
    g = dict(C=C, NRB=NRB, RPW=RPW, NCP=NCP, NSTAGE=NSTAGE, POST=POST, UPF=UPF, UPT=UPT, CS=CS)
    g["P"] = 64 * NRB
    g["HALO"] = 16 + 3 * POST
    g["HL"] = g["HALO"] + (UPT > 0)
    g["PC"] = CS * g["P"]
    g["PVB"] = g["PC"] - g["HALO"] - g["HL"]
    return g


def config(code):
    return parse_config(engine.lib().mg_gen_resblock_config(code).decode())


def ctas(g, L):
    """[(cluster, rank, o, first owned, end of owned)] of one item at length L, positions in the ResBlock's own
    coordinates; exactly the index arithmetic of resblock_tc_kernel."""
    P, CS, PC, PVB, HALO, HL = g["P"], g["CS"], g["PC"], g["PVB"], g["HALO"], g["HL"]
    n = 1 + ((L - PC + PVB - 1) // PVB if L > PC else 0)
    out = []
    for c in range(n):
        oc = 0 if c == 0 else (PC - HALO) + (c - 1) * PVB - HL
        for r in range(CS):
            o = oc + r * P
            p_lo = 0 if (c == 0 or r > 0) else HL
            p_hi = P if (r < CS - 1 or oc + PC >= L) else P - HALO
            out.append((c, r, o, o + p_lo, min(o + p_hi, L)))
    return out


def borders(g, L):
    """Positions where ownership passes from one CTA to the next (cluster and CTA-rank borders) inside [1, L)."""
    return sorted({lo for (_c, _r, _o, lo, hi) in ctas(g, L) if 0 < lo < L and hi > lo})


def lengths(g):
    """Lengths that put a border next to the end of the sequence or a CTA at a special fill."""
    P, CS, PC, PVB, HALO, HL = g["P"], g["CS"], g["PC"], g["PVB"], g["HALO"], g["HL"]
    out = set()
    for k in range(3):  # the first three cluster borders: ownership border, and the length at which cluster k + 1 appears
        for b in (PC - HALO + k * PVB, PC + k * PVB):
            out |= {b - 1, b, b + 1}
    if CS > 1:  # the first CTA-rank border inside a cluster
        out |= {P - 1, P, P + 1}
    for c in (1, 2):  # the last cluster (the second or third) with 1, 2, .. CS CTAs holding rows
        oc = PC - HALO + (c - 1) * PVB - HL
        lo_L, hi_L = PC + (c - 1) * PVB + 1, PC + c * PVB  # lengths with exactly c + 1 clusters
        for m in range(1, CS + 1):
            a, b = max(oc + (m - 1) * P + 1, lo_L), min(oc + m * P, hi_L)
            if a <= b:
                out |= {a, b}
    for c in range(3):  # L - 1 on the first or the last row of a CTA (the tail ConvT's fp32 fix-up for position L)
        oc = 0 if c == 0 else PC - HALO + (c - 1) * PVB - HL
        for r in range(CS):
            o = oc + r * P
            for L in (o + 1, o + P):
                if any(oo in (L - 1, L - P) and lo <= L - 1 < hi for (_c, _r, oo, lo, hi) in ctas(g, L)):
                    out.add(L)
    if g["UPF"]:  # the output length of a stride-2 ConvT is even: the even neighbours of an odd length
        out = {v for L in out for v in ((L,) if L % 2 == 0 else (L - 1, L + 1))}
    return sorted(L for L in out if L >= 1)


def input_shape(g, code, B, L):
    if g["UPF"]:
        return (B, 2 * g["C"], L // 2)
    return (B, g["C"], L)


def cluster_border_frames():
    """Mel lengths whose stage-0 (x8) or stage-1 (x64) length lies at or next to a cluster or CTA-rank border."""
    out = set()
    for code, scale in ((0, 8), (1, 64)):
        for L in lengths(config(code)):
            out |= {max(1, L // scale), (L + scale - 1) // scale}
    return sorted(out)


# ------------------------------------------------------------------------------------------------------------------
# 6. guarded output buffers
# ------------------------------------------------------------------------------------------------------------------
GUARD = 1024  # floats after each output buffer
FILL = 0x7FC0DEAD  # quiet NaN with a payload: arithmetic on NaN gives the canonical NaN, never this


def nan_buffer(n):
    return torch.full((n + GUARD,), FILL, dtype=torch.int32, device="cuda").view(torch.float32)


def guard_ok(buf, n):
    return bool((buf.view(torch.int32)[n:] == FILL).all())


def valid_mask(lengths, R, n, device="cuda"):
    """[B, n]: True at the first R lengths[i] of n positions of item i (the outputs of its own positions)."""
    lens = torch.tensor(lengths, device=device)
    return torch.arange(n, device=device)[None, :] < R * lens[:, None]


def fill_faults(y, buf, lengths, R, zero_tail=False):
    """Items with an output past their valid ones that no longer holds FILL (zero_tail: that is not +0.0); all items
    if the guard after the buffer was overwritten."""
    if not bool((buf.view(torch.int32)[y.numel():] == FILL).all()):
        return set(range(len(lengths)))
    past = ~valid_mask(lengths, R, y.shape[-1])[:, None, :]
    bad = (past & (y.contiguous().view(torch.int32) != (0 if zero_tail else FILL))).flatten(1).any(1)
    return set(torch.nonzero(bad).flatten().tolist())


# ------------------------------------------------------------------------------------------------------------------
# 7. the float64 layer models, their bounds, and the fixtures that pack the weights
# ------------------------------------------------------------------------------------------------------------------
TAU = 2.0 ** -12
REL = 2.0 ** -20
ROW_TOL = 1e-4      # per (item, channel) row, max|d| / max|ref|
BRANCH_TOL = 3e-4   # the residual branch (y - x) alone, per row
DILATIONS = (1, 3, 9)


# float64 restatements of the layers (reference models.py:32-40, 61-71, 87-103)
def folded64(state, name, device="cuda"):
    w = synth.fold_weight_norm(state[name + ".weight_g"], state[name + ".weight_v"])
    return (torch.from_numpy(w).to(device, torch.float64), torch.from_numpy(state[name + ".bias"]).to(device, torch.float64))


def fold64(g, v):
    """synth.fold_weight_norm without its final rounding to fp32: w = g v / ||v|| in float64, norm over every axis but 0."""
    v64 = v.astype(np.float64)
    norm = np.sqrt((v64 ** 2).sum(axis=tuple(range(1, v.ndim)), keepdims=True))
    return g.astype(np.float64).reshape(norm.shape) * v64 / norm


def fold_bound(w64, inner):
    """|w32 - w64| allowed to the pack kernels' fp32 fold of a norm row of `inner` elements (test_pack_blob_gpu's module
    docstring): (ceil(inner / 128) + 15) 2^-25 |w64|, plus one subnormal ulp."""
    return (cdiv(inner, 128) + 15) * 2.0 ** -25 * np.abs(w64) + 2.0 ** -149


class Gen64:
    """The generator's layers in float64 on the GPU."""

    def __init__(self, state, device="cuda"):
        self.w = {n: folded64(state, n, device) for n, *_ in synth.GENERATOR_LAYERS}

    def conv_pre(self, mel):
        w, b = self.w["conv_pre"]
        return F.conv1d(mel, w, b, padding=3)

    def convt(self, stage, x):
        w, b = self.w["ups.%d" % stage]
        k = w.shape[2]
        return F.conv_transpose1d(F.leaky_relu(x), w, b, stride=k // 2, padding=k // 4)

    def resblock(self, stage, x):
        for j, d in enumerate(DILATIONS):
            w1, b1 = self.w["resblocks.%d.convs1.%d" % (stage, j)]
            w2, b2 = self.w["resblocks.%d.convs2.%d" % (stage, j)]
            h = F.conv1d(F.leaky_relu(x), w1, b1, padding=d, dilation=d)
            x = F.conv1d(F.leaky_relu(h), w2, b2, padding=1) + x
        return x

    def post(self, x):
        w, b = self.w["conv_post"]
        return torch.tanh(F.conv1d(F.leaky_relu(x), w, b, padding=3))


def conv_bound_ratio(got, x64, w64, b64, stride=1, padding=0, groups=1, lrelu=False, tau=TAU):
    """Worst |y - y64| / (tau A2 + 2^-20 |y64 before the activation|) of one conv (<= 1: within the bound)."""
    pre = F.conv1d(x64, w64, b64, stride=stride, padding=padding, groups=groups)
    a2 = F.conv1d(x64 * x64, w64 * w64, None, stride=stride, padding=padding, groups=groups).sqrt()
    ref = F.leaky_relu(pre) if lrelu else pre
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    d = (got.double() - ref).abs()
    return float((d / (tau * a2 + REL * pre.abs()).clamp_min(1e-300)).max())


def row_errors(got, ref):
    """|got - ref| / max|ref| of its (item, channel) row, element-wise.  The row scale is at least 1/8 of the largest
    |ref| of the call: a row of a few positions can cancel to near zero (y = x + branch at L = 1), and its error is then
    that of the rows around it, not a fraction of its own value."""
    d = (got.double() - ref).abs()
    a = ref.abs()
    return d / a.amax(dim=-1, keepdim=True).clamp_min(float(a.max()) / 8).clamp_min(1e-30)


def run_with_reference(dev, g64, code, x):
    """(kernel output, float64 reference, float64 ResBlock input or None) of stage code `code` on x."""
    x64 = x.double()
    if code <= 3:
        return dev.resblock(code, x), g64.resblock(code, x64), x64
    if code == 4:
        return dev.resblock_post(x), g64.post(g64.resblock(3, x64)), None
    if code in (12, 13):
        s = code - 10
        c64 = g64.convt(s, x64)
        return dev.upres(s, x), g64.resblock(s, c64), c64
    if code == 14:
        return dev.upres_post(x), g64.post(g64.resblock(3, g64.convt(3, x64))), None
    s = code - 20
    return dev.resup(s, x), g64.convt(s + 1, g64.resblock(s, x64)), None


@pytest.fixture(scope="module")
def gstate():
    return synth.generator_state(1234)


@pytest.fixture(scope="module")
def gdev(gstate):
    gd = engine.GeneratorDevice("cuda:0")
    order = [n for n, *_ in synth.GENERATOR_LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    gd.pack([to(gstate[n + ".weight_v"]) for n in order], [to(gstate[n + ".weight_g"]) for n in order],
            [to(gstate[n + ".bias"]) for n in order])
    return gd


@pytest.fixture(scope="module")
def g64(gstate):
    return Gen64(gstate)


@pytest.fixture(scope="module")
def gen(gstate):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in gstate.items()})
    return g.cuda().eval()


@pytest.fixture(scope="module")
def dstate():
    return synth.discriminator_state(4321)


@pytest.fixture(scope="module")
def ddev(dstate):
    dd = engine.DiscriminatorDevice("cuda:0")
    names = ["discriminators.%d.%s" % (d, n) for d in range(3) for n, *_ in synth.DISCRIMINATOR_LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    dd.pack([to(dstate[n + ".weight_v"]) for n in names], [to(dstate[n + ".weight_g"]) for n in names],
            [to(dstate[n + ".bias"]) for n in names])
    return dd


# the bf16 inference mode in float64: exact (q = no_rounding), or its emulation (q = bf16_rn64 at the inputs of the
# single-pass layers; test_bf16_inference_gpu's module docstring)
EMU_X = 2.0        # kernel error <= EMU_X * emulation error + EMU_FLOOR, per item
EMU_FLOOR = 2e-5


def no_rounding(t):
    return t


def convt64(g, s, x, q):
    w, b = g.w["ups.%d" % s]
    k = w.shape[2]
    return F.conv_transpose1d(q(F.leaky_relu(x)), q(w), b, stride=k // 2, padding=k // 4)


def resblock64(g, s, x, q):
    for j, d in enumerate(DILATIONS):
        w1, b1 = g.w["resblocks.%d.convs1.%d" % (s, j)]
        w2, b2 = g.w["resblocks.%d.convs2.%d" % (s, j)]
        h = F.conv1d(q(F.leaky_relu(x)), q(w1), b1, padding=d, dilation=d)
        x = F.conv1d(q(F.leaky_relu(h)), q(w2), b2, padding=1) + x
    return x


def forward64(g, mel, emulate):
    """Exact float64 forward (emulate=False) or the bf16 emulation, mel [B, 80, T] -> audio [B, 1, 256 T]."""
    q = bf16_rn64 if emulate else no_rounding
    x = g.conv_pre(mel.double())
    for s in range(4):
        x = resblock64(g, s, convt64(g, s, x, no_rounding if s == 2 else q), q)
    return g.post(x)


def forward64_items(g, mel, emulate, chunk=16):
    return torch.cat([forward64(g, mel[i:i + chunk], emulate) for i in range(0, mel.shape[0], chunk)])


def item_max_abs(y, ref):
    return (y.double() - ref).abs().flatten(1).amax(dim=1)


def bf16_emulation_bound(gen, g64, mel, what):
    """bf16 forward of mel, its per-item error against exact float64 and the emulation's; asserts the bound."""
    y = gen.generate(mel, precision="bf16")
    gen._dev.check_status(mel.shape[0], mel.shape[2])
    exact = forward64_items(g64, mel, False)
    emu = forward64_items(g64, mel, True)
    e_k, e_e = item_max_abs(y, exact), item_max_abs(emu, exact)
    ratio = float(((e_k - EMU_FLOOR) / e_e).max())
    assert bool((e_k <= EMU_X * e_e + EMU_FLOOR).all()), (what, e_k.tolist(), e_e.tolist())
    return y, exact, e_k, e_e, ratio


# ragged generator batches
def ragged_batch(lens, seed):
    """mel [B, 80, max(lens)] of seeded per-item inputs, NaN past each length."""
    T = max(lens)
    mel = np.full((len(lens), 80, T), np.nan, np.float32)
    for i, L in enumerate(lens):
        mel[i, :, :L] = synth.mel_input(1, L, seed + i)[0]
    return torch.from_numpy(mel).cuda()


def check_items(gen, mel, lens, audio):
    assert audio.shape == (len(lens), 1, 256 * mel.shape[2])
    with torch.no_grad():
        for i, L in enumerate(lens):
            own = gen(mel[i:i + 1, :, :L].contiguous())
            assert torch.equal(audio[i:i + 1, :, :256 * L], own), (i, L)
            assert bool((audio[i, :, 256 * L:] == 0).all()), (i, L)
    gen._dev.check_status(len(lens), mel.shape[2])


# the C oracle
TOL = 1e-4


def oracle_resblock(state, stage, x):
    """ResBlock.forward (models.py:32-40) with the oracle's primitives."""
    lr = lambda a: np.where(a > 0, a, a * np.float32(0.01)).astype(np.float32)
    for j, d in enumerate((1, 3, 9)):
        n1, n2 = "resblocks.%d.convs1.%d" % (stage, j), "resblocks.%d.convs2.%d" % (stage, j)
        w1 = cport.fold_weight_norm(state[n1 + ".weight_g"], state[n1 + ".weight_v"])
        w2 = cport.fold_weight_norm(state[n2 + ".weight_g"], state[n2 + ".weight_v"])
        h = cport.conv1d(lr(x), w1, state[n1 + ".bias"], 1, d, d, 1)
        x = cport.conv1d(lr(h), w2, state[n2 + ".bias"], 1, 1, 1, 1) + x
    return x


# the training step's reference gradients
def train_case():
    return dict(B=2, T=4, mel_seed=21, audio_seed=22)  # tests/golden/make_golden.py TRAIN_CASE


def check_grad_digest(golden_grads, prefix, named_params, rtol):
    """Every parameter's gradient against the reference digest (L2 norm, sum, first 16 values)."""
    worst = 0.0
    for n, p in named_params:
        g = p.grad.detach().double().reshape(-1).cpu()
        l2 = float(golden_grads[prefix + n + "/l2"])
        scale = max(l2, 1e-12)
        if n.endswith("weight_g") and g.numel() == 1:
            # d weight_g = <dw, v> / ||v|| of a ONE-row layer (conv_post, conv_post2): a projection that cancels to a value far
            # below |dw| |v| (1e-5 against 1e-2 at B=16), so its error is set by the size of dw, i.e. of the sibling weight_v's
            # gradient, not by its own magnitude
            scale = max(scale, 0.02 * float(golden_grads[prefix + n[:-1] + "v/l2"]))
        assert abs(float(g.norm()) - l2) <= rtol * scale, (prefix, n, float(g.norm()), l2)
        assert abs(float(g.sum()) - float(golden_grads[prefix + n + "/sum"])) <= rtol * scale * max(1.0, g.numel() ** 0.5), (prefix, n)
        head = golden_grads[prefix + n + "/head"]
        err = np.abs(g[:16].numpy() - head).max()
        assert err <= rtol * max(np.abs(head).max(), scale / max(1.0, g.numel() ** 0.5)), (prefix, n, err)
        worst = max(worst, abs(float(g.norm()) - l2) / scale)
    return worst


# ------------------------------------------------------------------------------------------------------------------
# 8. the mel front end's options
# ------------------------------------------------------------------------------------------------------------------
DEFAULT = (22050, 80, 55.0, 9000.0, 1)                           # the reference's config.json: sr, n_mels, fmin, fmax, norm
NORMS = {0: None, 1: 1, 2: "l1"}


def mel_option_cases():
    full = []
    for sr in (16000, 22050, 24000, 44100):
        for n_mels in (1, 40, 80, 128):
            for norm in (0, 1, 2):
                for fmin in (0.0, 55.0):
                    for fmax in sorted({8000.0, 9000.0, sr / 2.0}):
                        if fmax <= sr / 2.0:
                            full.append((sr, n_mels, fmin, fmax, norm))
    picked = random.Random(2024).sample(full, 28)
    # the reference's setting; every thread of a frame a mel (128) at each norm; filters that cover no bin
    must = [DEFAULT, (44100, 128, 0.0, 22050.0, 0), (44100, 128, 55.0, 9000.0, 1), (22050, 128, 0.0, 11025.0, 2),
            (16000, 1, 0.0, 8000.0, 1), (44100, 128, 0.0, 4000.0, 1)]
    return must + [c for c in picked if c not in must]
