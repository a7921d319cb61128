"""Every generator and discriminator kernel on its OWN recorded input, against a float64 restatement of that one layer
(torch.nn.functional on the GPU, weights folded by synth.fold_weight_norm), at the sizes users run.

A layer's input is what the engine itself produced for the layer before it (the generator's stage taps, the
discriminators' returned feature maps), so an error can be neither hidden by nor blamed on the layers in front of it.

Single-conv layers (generator conv_pre; discriminator conv_pre, grouped convs, conv_post1, conv_post2) are held to an
element-wise bound,

    |y - y64| <= TAU * A2 + 2^-20 * |y64|,      A2 = sqrt(conv64(x^2, w^2)),

where A2 is the root-sum-square of the products that make up the output.  The 3-pass split-bf16 arithmetic drops the
lo*lo term and the residual of the lo split, about 2^-16 of each product; losing one of the three passes leaves about
2^-9 of each product.  Either error has random signs and grows like the root of the number of products, so against A2
the two stay about 2^7 apart at any K.  LeakyReLU and tanh are 1-Lipschitz, so the bound of the pre-activation carries
through them (the 2^-20 term uses the pre-activation).  test_tau_calibration_on_emulated_split_bf16 checks both sides of
TAU on the CPU with an emulation of the split.

The ResBlock kernels (six chained convs, no per-element bound) are held per (item, channel) row: max|d| / max|ref| <
1e-4; for the unfused stages also the residual branch alone, against the float64 ConvT output the branch was added to.

Measured on an H100 80GB HBM3 (700 W power limit), printed by the tests (-s).  Worst |y - y64| as a fraction of
the bound at TAU = 2^-12 (the CPU emulation of the split: 0.06 - 0.10; with one pass dropped: >= 21):
    generator conv_pre                 config 2: 0.088    config 5: 0.098
    discriminators, config 3 (worst of the three scales; the ragged lengths stay at or below these)
        conv_pre 0.011, grouped_convs.0-3 0.109 / 0.117 / 0.098 / 0.115, conv_post1 0.314, conv_post2 0.004
Worst per-row max|d| / max|ref| (branch alone in brackets), config 2 / config 5:
    up0+res0 2.8e-5 (1.8e-4) / 2.7e-5 (1.4e-4), up1+res1 1.9e-5 (7.1e-5) / 1.5e-5 (6.0e-5),
    up2+res2 1.7e-5 (4.5e-5) / 1.6e-5 (4.7e-5), up3+res3+post 6.5e-6 / 8.4e-6
(The branch of up0+res0 also carries the ConvT kernel's own error, which the float64 input of the branch does not.)
"""
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, synth
from kernel_model import ddev, dstate, g64, gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import BRANCH_TOL, ROW_TOL, conv_bound_ratio, folded64, row_errors, split_conv


# ------------------------------------------------------------------------------------------------------------------
# the bound itself, calibrated on the CPU (split_conv: the split's arithmetic, conv_bound_ratio: the bound; kernel_model)
# ------------------------------------------------------------------------------------------------------------------
# (Cin, Cout, k, stride, groups): K = Cin / groups * k from 15 to 5120 -- the discriminators' conv_pre, a grouped conv,
# the generator's conv_pre and ResBlock convs, conv_post2, conv_post1
CALIBRATION = [(1, 16, 15, 1, 1), (64, 64, 41, 4, 16), (80, 128, 7, 1, 1), (256, 64, 3, 1, 1), (1024, 1, 3, 1, 1),
               (1024, 32, 5, 1, 1)]


@pytest.mark.parametrize("cin,cout,k,stride,groups", CALIBRATION)
def test_tau_calibration_on_emulated_split_bf16(cin, cout, k, stride, groups):
    """The 3-pass split passes the element-wise bound with margin; dropping any one of its passes fails it by >= 8x."""
    gen = torch.Generator().manual_seed(cin * 1000 + k)
    K = cin // groups * k
    x = F.leaky_relu(torch.randn(2, cin, 2048 if cin == 1 else 512, generator=gen))
    w = (torch.rand(cout, cin // groups, k, generator=gen) * 2 - 1) / K ** 0.5
    pad = k // 2
    x64, w64 = x.double(), w.double()
    full = conv_bound_ratio(split_conv(x, w, stride, pad, groups), x64, w64, None, stride, pad, groups)
    dropped = [conv_bound_ratio(split_conv(x, w, stride, pad, groups, [p for p in range(3) if p != q]), x64, w64, None,
                                stride, pad, groups) for q in range(3)]
    print("K=%d: 3-pass %.3f of the bound, one pass dropped %s" % (K, full, " ".join("%.1f" % r for r in dropped)))
    assert full < 0.5, (K, full)
    assert min(dropped) >= 8, (K, dropped)


# ------------------------------------------------------------------------------------------------------------------
# generator: every kernel of the default chain on its own recorded input
# ------------------------------------------------------------------------------------------------------------------
CHAIN = ["conv_pre", "up0", "res0", "up1", "res1", "up2", "res2", "up3+res3+post"]
ITEMS = (0, 15, 16, 31, 32, 47, 48, 63)  # the borders of config 2's four batch slices


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(64, 32), (1, 1000)])
def test_generator_layers_on_their_own_inputs(gdev, g64, B, T):
    """Config 2 (B = 64, T = 32: four batch slices) and config 5 (B = 1, T = 1000), every position of the checked items."""
    L = engine.lib()
    engine.check(L.mg_gen_set_pipeline(0))
    try:
        assert [L.mg_gen_kernel_name(i).decode() for i in range(L.mg_gen_forward_launches())] == CHAIN
        mel = torch.from_numpy(synth.mel_input(B, T, 300 + T)).cuda()
        audio = gdev.forward(mel)
        taps = [gdev.stage_output(i, B, T) for i in range(4)]
        gdev.check_status(B, T)
    finally:
        engine.check(L.mg_gen_set_pipeline(-1))
    items = [i for i in ITEMS if i < B]
    x = mel[items].double()
    w, b = g64.w["conv_pre"]
    r = conv_bound_ratio(taps[0][items], x, w, b, padding=3)
    print("\n(B=%d, T=%d) conv_pre: %.3f of the bound" % (B, T, r))
    assert r <= 1, ("conv_pre", r)
    for s in range(4):
        x = taps[s][items].double()
        c64 = g64.convt(s, x)
        y64 = g64.resblock(s, c64)
        if s == 3:
            got, ref, name = audio[items], g64.post(y64), "up3+res3+post"
        else:
            got, ref, name = taps[s + 1][items], y64, "up%d+res%d" % (s, s)
        rows = float(row_errors(got, ref).max())
        msg = "(B=%d, T=%d) %s: rows %.2e" % (B, T, name, rows)
        if s < 3:
            branch = float(row_errors(got.double() - c64, ref - c64).max())
            msg += ", branch %.2e" % branch
            assert branch < BRANCH_TOL, (name, branch)
        print(msg)
        assert rows < ROW_TOL, (name, rows)


# ------------------------------------------------------------------------------------------------------------------
# discriminators: all 21 layers, layer l on the feature map the engine returned for layer l - 1
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Bt,L", [(32, 8192), (2, 64), (6, 257), (4, 2050), (2, 4097)])
def test_discriminator_layers_on_their_own_inputs(ddev, dstate, Bt, L):
    """Config 3 (32 stacked items of 8192 samples) and the ragged lengths of test_disc_gpu.py (real and generated
    stacked): every element of every layer of the three scales."""
    y = torch.from_numpy(synth.audio_input(Bt, L, 7 * L + Bt)).cuda()
    fm = ddev.forward(y)
    ddev.check_status()
    x0 = y.double()
    worst = [0.0] * 7
    for s in range(3):
        if s == 1:
            x0 = F.avg_pool1d(x0, 4, 2, padding=2)
        elif s == 2:
            x0 = F.avg_pool1d(x0, 4, 4, padding=2)
        for l, (name, _cin, _cout, _k, stride, groups, pad) in enumerate(synth.DISCRIMINATOR_LAYERS):
            w, b = folded64(dstate, "discriminators.%d.%s" % (s, name))
            x = x0 if l == 0 else fm[s][l - 1].double()
            r = conv_bound_ratio(fm[s][l], x, w, b, stride, pad, groups, lrelu=l < 6)
            assert r <= 1, (s, name, r)
            worst[l] = max(worst[l], r)
    print("\n(Bt=%d, L=%d) worst ratio to the bound per layer: %s" % (
        Bt, L, ", ".join("%s %.3f" % (n, r) for (n, *_), r in zip(synth.DISCRIMINATOR_LAYERS, worst))))
