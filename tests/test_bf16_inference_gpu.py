"""The bf16 inference mode (mg_gen_forward_precision, Generator.generate(..., precision="bf16")): one bf16 pass per
tensor-core product in the ConvTs of stages 0, 1 and 3 and in every ResBlock conv, against a float64 emulation of
exactly that arithmetic.

The emulation (float64, on the GPU) rounds LeakyReLU(x) and the folded weights to bf16 (round to nearest even) at the
inputs of those layers and computes everything else exactly: conv_pre and the stride-2 ConvT of stage 2 (three passes
in the kernels), the biases, the residual adds and conv_post + tanh (fp32 in the kernels).  What the kernels add to the
emulation's own error is fp32 accumulation and the rounding of operands that have drifted by that much, so a forward is
held to  max|y - y64| <= 2 x (max|emulation - y64|) + 2e-5  per item, y64 the exact float64 forward.

Measured on an H100 80GB HBM3 (400 W power limit), printed by the tests (-s):
    config 2, N(0,1) / log-mel-like: rel-L2 vs float64 9.8e-4 / 1.6e-3 (SNR 60.1 / 55.9 dB), max|d| 1.8e-4 / 3.1e-4;
        at the stored reference positions worst item rel-L2 1.0e-3 / 1.7e-3; kernel max|d| / emulation max|d| <= 1.12
    goldens (T = 1 .. 1000): worst (max|d| - 2e-5) / emulation 0.98;  63 border lengths: 1.05
    stage taps, worst row max|d| / max|ref|: up0+res0 5.2e-3, up1+res1 5.2e-3, up2+res2 6.9e-3, up3+res3+post 2.6e-3
"""
import ctypes
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cases
from melgan_multi_b200 import engine, models, synth
from test_kernel_borders_gpu import config, lengths as border_lengths
from test_layer_isolation_gpu import Gen64, g64, gdev, gstate, row_errors  # noqa: F401 (fixtures)

DILATIONS = (1, 3, 9)
EMU_X = 2.0        # kernel error <= EMU_X * emulation error + EMU_FLOOR, per item
EMU_FLOOR = 2e-5
ROW_TOL = 3e-2     # stage isolation: per (item, channel) row, max|d| / max|ref| against exact float64
ITEMS = (0, 15, 16, 31, 32, 47, 48, 63)  # the borders of config 2's four batch slices
CHAIN_CODES = {0: 8, 1: 64, 2: 128, 14: 256}  # bf16 ResBlock stage codes of the default chain -> positions per mel frame


# ------------------------------------------------------------------------------------------------------------------
# float64 references: exact, and the bf16 emulation
# ------------------------------------------------------------------------------------------------------------------
def _bf16(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _same(t):
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
    q = _bf16 if emulate else _same
    x = g.conv_pre(mel.double())
    for s in range(4):
        x = resblock64(g, s, convt64(g, s, x, _same if s == 2 else q), q)
    return g.post(x)


def forward64_items(g, mel, emulate, chunk=16):
    return torch.cat([forward64(g, mel[i:i + chunk], emulate) for i in range(0, mel.shape[0], chunk)])


def item_max_abs(y, ref):
    return (y.double() - ref).abs().flatten(1).amax(dim=1)


@pytest.fixture(scope="module")
def gen(gstate):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in gstate.items()})
    return g.cuda().eval()


def _emulation_bound(gen, g64, mel, what):
    """bf16 forward of mel, its per-item error against exact float64 and the emulation's; asserts the bound."""
    y = gen.generate(mel, precision="bf16")
    gen._dev.check_status(mel.shape[0], mel.shape[2])
    exact = forward64_items(g64, mel, False)
    emu = forward64_items(g64, mel, True)
    e_k, e_e = item_max_abs(y, exact), item_max_abs(emu, exact)
    ratio = float(((e_k - EMU_FLOOR) / e_e).max())
    assert bool((e_k <= EMU_X * e_e + EMU_FLOOR).all()), (what, e_k.tolist(), e_e.tolist())
    return y, exact, e_k, e_e, ratio


# ------------------------------------------------------------------------------------------------------------------
# 1 + 3: config 2 at full size, and the mode is really on
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def config2_golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "config2_outputs.npz"))


@pytest.mark.gpu
@pytest.mark.parametrize("realistic", [False, True])
def test_config2_full_size(gen, g64, config2_golden, realistic):
    """B = 64, T = 32, all 64 items: per item, at the stored positions of the reference's output, rel-L2 <= 4e-3 and
    max|d| <= 1e-3; against float64 everywhere within twice the emulation's error.  bf16 must differ from the fp32 path
    by rel-L2 >= 2e-4 (the three-pass path sits at ~2e-6 from float64: a silent fall-back to it fails), and fp32 through
    mg_gen_forward_precision is mg_gen_forward bit for bit."""
    B, T = 64, 32
    mel = torch.from_numpy(synth.mel_input(B, T, 0, realistic)).cuda()
    y, exact, e_k, e_e, ratio = _emulation_bound(gen, g64, mel, ("config2", realistic))
    pos = torch.from_numpy(config2_golden["gen_B64_T32_positions"]).cuda()
    ref = torch.from_numpy(config2_golden["gen_B64_T32_s0_r%d" % int(realistic)]).cuda().double()
    d = y[:, :, pos].double() - ref
    rel = d.flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1)
    mx = d.abs().flatten(1).amax(dim=1)
    assert float(rel.max()) <= 4e-3 and float(mx.max()) <= 1e-3, (float(rel.max()), float(mx.max()))
    full = (y.double() - exact)
    rel_all = float(full.norm() / exact.norm())
    snr = -20 * math.log10(rel_all)
    y32 = gen.generate(mel)
    rel_32 = float((y.double() - y32.double()).norm() / y32.double().norm())
    assert rel_32 >= 2e-4, rel_32
    # the fp32 code of the new entry point is the old path
    dev, L = gen._dev, engine.lib()
    out = torch.empty_like(y32)
    ws = dev.workspace(B, T)
    engine.check(L.mg_gen_forward_precision(dev.packed.data_ptr(), mel.data_ptr(), out.data_ptr(), B, T, None, 0, ws.data_ptr(),
                                            ws.numel() * 4, torch.cuda.current_stream().cuda_stream))
    dev.check_status(B, T)
    assert torch.equal(out, y32)
    print("\nconfig 2 %s: vs float64 rel-L2 %.2e (worst item %.2e), max|d| %.2e, SNR %.1f dB; at the golden positions "
          "worst item rel-L2 %.2e, max|d| %.2e; kernel / emulation max|d| worst %.2f; bf16 vs fp32 rel-L2 %.2e" % (
              "log-mel-like" if realistic else "N(0,1)", rel_all,
              float((full.flatten(1).norm(dim=1) / exact.flatten(1).norm(dim=1)).max()), float(e_k.max()), snr,
              float(rel.max()), float(mx.max()), ratio, rel_32))


# ------------------------------------------------------------------------------------------------------------------
# 2: every generator golden
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", cases.GEN_CASES + [(1, 1000, 0, False)])
def test_goldens_within_twice_the_emulation_error(gen, g64, golden, case):
    """The cases of reference_outputs.npz (T = 1, 7, 32, 33, 16 and 1000): per item, error against float64 <= 2x the
    emulation's + 2e-5.  The float64 forward itself is checked against the stored reference output first."""
    B, T, seed, realistic = case
    mel = torch.from_numpy(synth.mel_input(B, T, seed, realistic)).cuda()
    y, exact, e_k, e_e, ratio = _emulation_bound(gen, g64, mel, case)
    if T == 1000:
        ref, got = golden["gen_T1000_head"], exact[0, 0, :4096]
    else:
        ref, got = golden[cases.gen_key(*case)], exact
    assert float(np.abs(got.cpu().numpy() - ref).max()) < 1e-4 * max(float(np.abs(ref).max()), 1e-3)
    print("\n%s: max|d| %s, emulation %s, worst (kernel - 2e-5) / emulation %.2f" % (
        case, " ".join("%.2e" % v for v in e_k.tolist()), " ".join("%.2e" % v for v in e_e.tolist()), ratio))


# ------------------------------------------------------------------------------------------------------------------
# 4: stage isolation from the chain's own taps
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_stage_taps_against_float64(gdev, g64):
    """Config 2 in bf16, each stage on the tap the chain produced for it: conv_pre's tap is the fp32 forward's bit for bit;
    ConvT + ResBlock of stages 0-2 and up3 + ResBlock 3 + post per (item, channel) row within 3e-2 of float64."""
    B, T = 64, 32
    L = engine.lib()
    assert L.mg_gen_forward_launches() == 8  # the default chain
    mel = torch.from_numpy(synth.mel_input(B, T, 300 + T)).cuda()
    gdev.forward(mel)
    tap0 = gdev.stage_output(0, B, T)
    audio = gdev.forward(mel, precision="bf16")
    taps = [gdev.stage_output(i, B, T) for i in range(4)]
    gdev.check_status(B, T)
    assert torch.equal(taps[0], tap0)
    items = list(ITEMS)
    worst = []
    for s in range(4):
        x = taps[s][items].double()
        y64 = resblock64(g64, s, convt64(g64, s, x, _same), _same)
        got, ref = (taps[s + 1][items], y64) if s < 3 else (audio[items], g64.post(y64))
        r = float(row_errors(got, ref).max())
        worst.append(r)
        assert r <= ROW_TOL, (s, r)
    print("\nbf16 stage taps, worst row max|d| / max|ref|: up0+res0 %.2e, up1+res1 %.2e, up2+res2 %.2e, up3+res3+post %.2e"
          % tuple(worst))


# ------------------------------------------------------------------------------------------------------------------
# 5: ragged batches, host engine, determinism
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ragged_items_equal_their_own_bf16_forward(gen, gstate):
    """16 seeded lengths in [1, 300], NaN past each length (cut into batch slices): each item is its own bf16 forward bit for
    bit followed by zeros; the host engine gives the same bits as the device path; two identical calls are identical."""
    lens = [int(v) for v in np.random.default_rng(31).integers(1, 301, 16)]
    B, T = len(lens), max(lens)
    mel_np = synth.mel_input(B, T, 77)
    for i, n in enumerate(lens):
        mel_np[i, :, n:] = np.nan
    mel = torch.from_numpy(mel_np).cuda()
    y = gen.generate(mel, lens, precision="bf16")
    y2 = gen.generate(mel, lens, precision="bf16")
    gen._dev.check_status(B, T)
    assert torch.equal(y, y2)
    for i, n in enumerate(lens):
        own = gen.generate(mel[i:i + 1, :, :n].contiguous(), precision="bf16")
        assert torch.equal(y[i, 0, :256 * n], own[0, 0]), (i, n)
        assert not bool(y[i, 0, 256 * n:].any()), (i, n)
    gen._dev.check_status(1, lens[-1])
    host = engine.GeneratorHost(B, T)
    try:
        host.load_state(gstate)
        yh = host.forward_ragged(mel_np, lens, precision="bf16")
        yu = host.forward(mel_np[:1, :, :lens[0]], precision="bf16")
    finally:
        host.close()
    assert np.array_equal(yh, y.cpu().numpy())
    assert np.array_equal(yu[0, 0], y[0, 0, :256 * lens[0]].cpu().numpy())


# ------------------------------------------------------------------------------------------------------------------
# 6: tile and cluster borders
# ------------------------------------------------------------------------------------------------------------------
def border_frames():
    """Mel lengths that put an end of the sequence at (or one frame either side of) every tile and cluster border of the
    default chain's bf16 ResBlock kernels, derived from the geometry the library reports (test_kernel_borders_gpu)."""
    out = set()
    for code, k in CHAIN_CODES.items():
        for L in border_lengths(config(code)):
            t = -(-L // k)
            out |= {v for v in (t - 1, t, t + 1) if v >= 1}
    return sorted(out)


@pytest.mark.gpu
def test_borders_within_twice_the_emulation_error(gen, g64):
    """Every border length of border_frames() as its own B = 1 forward, within the bound of the goldens."""
    worst = 0.0
    Ts = border_frames()
    for T in Ts:
        mel = torch.from_numpy(synth.mel_input(1, T, 500 + T)).cuda()
        _y, _exact, _e_k, _e_e, ratio = _emulation_bound(gen, g64, mel, T)
        worst = max(worst, ratio)
    print("\n%d border lengths (T = %s): worst (kernel - 2e-5) / emulation %.2f" % (len(Ts), Ts, worst))


# ------------------------------------------------------------------------------------------------------------------
# 7: no GPU needed
# ------------------------------------------------------------------------------------------------------------------
def test_precision_strings():
    assert engine._precision("fp32") == 0 and engine._precision("bf16") == 1
    for bad in ("fp16", "BF16", "", None, 1, b"bf16"):
        with pytest.raises(engine.EngineError, match="precision"):
            engine._precision(bad)
    with pytest.raises(engine.EngineError, match="precision"):  # before the CUDA check
        models.Generator().generate(torch.zeros(2, 80, 4), precision="fp16")
    with pytest.raises(engine.EngineError, match="CUDA"):
        models.Generator().generate(torch.zeros(2, 80, 4), precision="bf16")


def test_precision_entry_points_validate_before_cuda():
    L, p = engine.lib(), ctypes.c_void_p(256)
    ws = L.mg_gen_workspace_bytes(2, 8)
    lens = (ctypes.c_int * 2)(8, 3)

    def fwd(precision, lengths=None, B=2, ws_bytes=ws, packed=p):
        rc = L.mg_gen_forward_precision(packed, p, p, B, 8, lengths, precision, p, ws_bytes, None)
        return rc, L.mg_last_error_string()

    for bad in (2, -1, 99):
        rc, msg = fwd(bad)
        assert rc == -1 and b"unknown precision %d" % bad in msg, msg
    rc, msg = fwd(1, packed=None)
    assert rc == -1 and b"null argument" in msg
    rc, msg = fwd(1, lens, ws_bytes=ws - 1)
    assert rc == -4 and b"workspace" in msg
    rc, msg = fwd(1, (ctypes.c_int * 2)(8, 9))
    assert rc == -1 and b"lengths[1] = 9" in msg
    rc, msg = fwd(0, B=0)
    assert rc == -1 and b"B >= 1" in msg
    assert L.mg_gen_engine_forward_precision(None, p, p, 2, 8, None, 7) == -1
    assert b"unknown precision 7" in L.mg_last_error_string()
    assert L.mg_gen_engine_forward_precision(None, p, p, 2, 8, lens, 1) == -1
    assert b"mg_gen_engine_forward_precision: null argument" in L.mg_last_error_string()


@pytest.mark.parametrize("mask", [2, 8, 14])
def test_bf16_refuses_a_non_default_chain(mask):
    L, p = engine.lib(), ctypes.c_void_p(256)
    ws = L.mg_gen_workspace_bytes(1, 4)
    engine.check(L.mg_gen_set_pipeline(mask))
    try:
        assert L.mg_gen_forward_precision(p, p, p, 1, 4, None, 1, p, ws, None) == -1
        msg = L.mg_last_error_string()
        assert b"default chain" in msg and b"tail mask %d" % mask in msg, msg
        assert L.mg_gen_engine_forward_precision(None, p, p, 1, 4, None, 1) == -1
        assert b"default chain" in L.mg_last_error_string()
        # fp32 still takes every chain (the call then stops at its null packed weights)
        assert L.mg_gen_forward_precision(None, p, p, 1, 4, None, 0, p, ws, None) == -1
        assert b"null argument" in L.mg_last_error_string()
    finally:
        engine.check(L.mg_gen_set_pipeline(-1))


def test_border_frames_cover_every_bf16_code():
    Ts = border_frames()
    assert Ts == sorted(set(Ts)) and Ts[0] >= 1
    for code, k in CHAIN_CODES.items():
        for L in border_lengths(config(code)):
            assert -(-L // k) in Ts, (code, L)
