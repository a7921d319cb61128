"""GPU parity of the multi-scale discriminator forward (through the C ABI) against the reference's golden
outputs and the C oracle.  fp32 SIMT layers are exact to summation order; conv_post1 runs split-bf16 on
wgmma (~1e-5).  Asserted at 1e-4 (north_star tolerance: 1e-3)."""
import numpy as np
import pytest
import torch

import cases
from conftest import rel_errors
from melgan_multi_b200 import engine, synth
from oracle import cport

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def dstate():
    return synth.discriminator_state(4321)


@pytest.fixture(scope="module")
def msd_module(dstate):
    from melgan_multi_b200 import models
    m = models.MultiScaleDiscriminator()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in dstate.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def folded(dstate):
    return cport.fold_discriminators(dstate)


@pytest.mark.parametrize("case", cases.MSD_CASES)
def test_msd_matches_reference_golden(golden, msd_module, case):
    B, L, seed = case
    y = torch.from_numpy(synth.audio_input(B, L, seed)).cuda()
    y_hat = torch.from_numpy(synth.audio_input(B, L, seed + 7)).cuda()
    with torch.no_grad():
        rs, gs, frs, fgs = msd_module(y, y_hat)
    msd_module._dev.check_status()
    tag = "msd_B%d_L%d_s%d" % (B, L, seed)
    for i in range(3):
        for nm, lg, fm in (("r", rs, frs), ("g", gs, fgs)):
            ref = golden["%s_logit_%s%d" % (tag, nm, i)]
            got = lg[i].cpu().numpy()
            assert got.shape == ref.shape
            m, l2 = rel_errors(got, ref)
            assert m < TOL and l2 < TOL, (i, nm, m, l2)
            for j in range(7):
                a = fm[i][j].cpu().numpy()
                assert tuple(golden["%s_fmap_%s%d_%d_shape" % (tag, nm, i, j)]) == a.shape
                head = golden["%s_fmap_%s%d_%d_head" % (tag, nm, i, j)]
                m, _ = rel_errors(a[:, :4, :48], head)
                assert m < TOL, (i, j, nm, m)
                s = golden["%s_fmap_%s%d_%d_sum" % (tag, nm, i, j)]
                assert abs(np.abs(a.astype(np.float64)).sum() - s[1]) < 1e-4 * s[1], (i, j, nm)


@pytest.mark.parametrize("B,L", [(1, 64), (3, 257), (2, 2050), (1, 4097)])
def test_msd_matches_oracle_on_ragged_lengths(msd_module, folded, B, L):
    """Odd lengths exercise the AvgPool / stride-4 edges of every layer (the reference's pooled lengths are odd)."""
    y = synth.audio_input(B, L, 3 * L)
    y_hat = synth.audio_input(B, L, 3 * L + 1)
    ref = cport.msd_forward(folded, y, y_hat)
    with torch.no_grad():
        got = msd_module(torch.from_numpy(y).cuda(), torch.from_numpy(y_hat).cuda())
    msd_module._dev.check_status()
    for i in range(3):
        for k in (0, 1):  # logits real / generated
            m, l2 = rel_errors(got[k][i].cpu().numpy(), ref[k][i])
            assert m < TOL and l2 < TOL, ("logit", i, k, m, l2)
        for k in (2, 3):  # feature maps real / generated
            for j in range(7):
                m, l2 = rel_errors(got[k][i][j].cpu().numpy(), ref[k][i][j])
                assert m < TOL and l2 < TOL, ("fmap", i, j, k, m, l2)


def test_losses_on_native_outputs_match_reference(golden, msd_module):
    from melgan_multi_b200 import models
    B, L, seed = cases.MSD_CASES[0]
    y = torch.from_numpy(synth.audio_input(B, L, seed)).cuda()
    y_hat = torch.from_numpy(synth.audio_input(B, L, seed + 7)).cuda()
    with torch.no_grad():
        rs, gs, frs, fgs = msd_module(y, y_hat)
    tag = "msd_B%d_L%d_s%d" % (B, L, seed)
    assert abs(models.feature_loss(frs, fgs).item() / float(golden[tag + "_feature_loss"]) - 1) < 1e-4
    assert abs(models.generator_loss(gs).item() / float(golden[tag + "_generator_loss"]) - 1) < 1e-4
    dl, rl, gl = models.discriminator_loss(rs, gs)
    np.testing.assert_allclose([dl.item()] + rl + gl, golden[tag + "_discriminator_loss"], rtol=1e-4)


def test_fused_losses_match_torch_formulas_and_gradients():
    """csrc/mg_loss.cu against the reference's formulas (models.py:138-167) in plain torch, values and input gradients;
    ragged sizes exercise the vector/tail split and multi-CTA rows."""
    from melgan_multi_b200 import models
    gen = torch.Generator(device="cpu").manual_seed(7)
    shapes = [(2, 16, 4097), (2, 64, 1025), (2, 1024, 17), (2, 1, 17), (3, 5, 33333)]
    fr = [[torch.randn(s, generator=gen).cuda().requires_grad_(True) for s in shapes]]
    fg = [[torch.randn(s, generator=gen).cuda().requires_grad_(True) for s in shapes]]
    dr = [torch.randn(4, n, generator=gen).cuda().requires_grad_(True) for n in (128, 65, 17)]
    dg = [torch.randn(4, n, generator=gen).cuda().requires_grad_(True) for n in (128, 65, 17)]
    loss = models.feature_loss(fr, fg) + models.generator_loss(dg)
    dl, rl, gl = models.discriminator_loss(dr, dg)
    (loss + dl).backward()
    got = [t.grad.clone() for t in fr[0] + fg[0] + dr + dg]
    for t in fr[0] + fg[0] + dr + dg:
        t.grad = None
    ref = sum((r - g).abs().mean() for r, g in zip(fr[0], fg[0])) * 10 + sum(((1 - g) ** 2).mean() for g in dg)
    ref_r = [((1 - r) ** 2).mean() for r in dr]
    ref_g = [(g ** 2).mean() for g in dg]
    ref_dl = sum(ref_r) + sum(ref_g)
    (ref + ref_dl).backward()
    assert abs(loss.item() / ref.item() - 1) < 1e-5 and abs(dl.item() / ref_dl.item() - 1) < 1e-5
    np.testing.assert_allclose(rl + gl, [v.item() for v in ref_r + ref_g], rtol=1e-5)
    for g, t in zip(got, fr[0] + fg[0] + dr + dg):
        assert torch.allclose(g, t.grad, rtol=1e-5, atol=1e-9)
    # bit-reproducible (fixed-order combine of the per-CTA partial sums)
    with torch.no_grad():
        assert models.feature_loss(fr, fg).item() == models.feature_loss(fr, fg).item()


def test_msd_backward_reaches_parameters_and_input(msd_module):
    """train.py:117 backpropagates the generator loss THROUGH the discriminators into y_hat (and into D's leaves)."""
    msd_module.zero_grad()
    y = torch.from_numpy(synth.audio_input(2, 1024, 5)).cuda()
    y_hat = torch.from_numpy(synth.audio_input(2, 1024, 6)).cuda().requires_grad_(True)
    rs, gs, frs, fgs = msd_module(y, y_hat)
    from melgan_multi_b200 import models
    loss = models.feature_loss(frs, fgs) + models.generator_loss(gs)
    loss.backward()
    assert y_hat.grad is not None and torch.isfinite(y_hat.grad).all() and y_hat.grad.abs().sum() > 0
    for n, p in msd_module.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    msd_module.zero_grad()


def test_msd_is_deterministic_and_batch_items_are_independent(msd_module):
    y = torch.from_numpy(synth.audio_input(3, 1500, 11)).cuda()
    yh = torch.from_numpy(synth.audio_input(3, 1500, 12)).cuda()
    with torch.no_grad():
        a = msd_module(y, yh)
        b = msd_module(y, yh)
        one = msd_module(y[1:2], yh[1:2])
    for i in range(3):
        assert torch.equal(a[0][i], b[0][i]) and torch.equal(a[1][i], b[1][i])
        for j in range(7):
            assert torch.equal(a[2][i][j], b[2][i][j]) and torch.equal(a[3][i][j], b[3][i][j])
            assert torch.equal(a[2][i][j][1:2], one[2][i][j]) and torch.equal(a[3][i][j][1:2], one[3][i][j])


@pytest.mark.parametrize("layer,Bt,Lin", [(1, 3, 1025), (1, 2, 4096), (2, 2, 257), (3, 2, 65), (3, 5, 300), (4, 3, 17), (4, 2, 130)])
def test_grouped_conv_backward_matches_torch(msd_module, layer, Bt, Lin):
    """csrc/mg_disc_bwd.cu (dx, dw, db of the grouped k41 convs) against autograd of F.conv1d in strict fp32; ragged
    lengths cover the stride-4 phase logic at both edges and partial tiles."""
    import torch.nn.functional as F
    from melgan_multi_b200.synth import DISCRIMINATOR_LAYERS
    old = torch.backends.cudnn.conv.fp32_precision
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    try:
        with torch.no_grad():
            msd_module(torch.zeros(1, 1, 64).cuda(), torch.zeros(1, 1, 64).cuda())  # makes sure the weights are packed
        scale = 1
        _n, cin, cout, k, stride, groups, pad = DISCRIMINATOR_LAYERS[layer]
        conv = msd_module.discriminators[scale].layers()[layer]
        w = torch._weight_norm(conv.weight_v, conv.weight_g, 0).detach().requires_grad_(True)
        gen = torch.Generator(device="cpu").manual_seed(100 * layer + Lin)
        x = torch.randn(Bt, cin, Lin, generator=gen).cuda().requires_grad_(True)
        out = F.conv1d(x, w, None, stride, pad, 1, groups)
        dz = torch.randn(out.shape, generator=gen).cuda()
        rdx, rdw = torch.autograd.grad(out, (x, w), dz)
        dx, dw, db = msd_module._dev.grouped_backward(scale, layer, dz, x.detach())
        for got, ref in ((dx, rdx), (dw, rdw), (db, dz.sum(dim=(0, 2)))):
            m, l2 = rel_errors(got.cpu().numpy(), ref.cpu().numpy())
            assert m < 2e-5 and l2 < 2e-5, (m, l2)
        assert msd_module._dev.grouped_backward(scale, layer, dz, x.detach(), need_dx=False)[0] is None
    finally:
        torch.backends.cudnn.conv.fp32_precision = old


@pytest.mark.parametrize("Bt,L", [(32, 128), (32, 65), (32, 17), (32, 32), (32, 16), (32, 8), (3, 17), (2, 20), (5, 7), (1, 3),
                                  (2, 130)])
def test_conv_post1_gradients_match_fp64(msd_module, Bt, L):
    """csrc/mg_wgrad_tc.cu (dW, db) and the transposed-blob dgrad of conv_post1 (models.py:84,96) against autograd of F.conv1d
    in float64: the lengths conv_post1 sees at config 3 (32 stacked items of 8192 samples: 128 / 65 / 17 positions at
    scales 0 / 1 / 2; at 65 every item's last k-panel is padded and items meet inside a stage), other 32-item lengths, and
    ragged ones (L % 4 != 0: scalar loads; L % 8 != 0: padded k-panels; L < 5: every tap touches the zero padding; K extent
    not a multiple of 32)."""
    import torch.nn.functional as F
    with torch.no_grad():
        msd_module(torch.zeros(1, 1, 64).cuda(), torch.zeros(1, 1, 64).cuda())  # makes sure the weights are packed
    scale = 2
    conv = msd_module.discriminators[scale].layers()[5]
    w = torch._weight_norm(conv.weight_v, conv.weight_g, 0).detach().double().requires_grad_(True)
    gen = torch.Generator(device="cpu").manual_seed(1000 * Bt + L)
    x = torch.randn(Bt, 1024, L, generator=gen).cuda()
    dz = torch.randn(Bt, 1024, L, generator=gen).cuda()
    xd = x.double().requires_grad_(True)
    rdx, rdw = torch.autograd.grad(F.conv1d(xd, w, None, 1, 2), (xd, w), dz.double())
    dev = msd_module._dev
    dw, db = dev.post1_wgrad(x, dz)
    dx = dev.post1_dgrad(scale, dz)
    torch.cuda.synchronize()
    assert int(dev.status[0].item()) == 0
    for name, got, ref in (("dw", dw, rdw), ("db", db, dz.double().sum(dim=(0, 2))), ("dx", dx, rdx)):
        m, l2 = rel_errors(got.cpu().numpy(), ref.float().cpu().numpy())
        # (the sums run over 5120 products: the dropped lo*lo term of the 3-pass split leaves ~2e-5 of the maximum on dx)
        assert m < 5e-5 and l2 < 3e-5, (name, m, l2)


@pytest.mark.parametrize("layer,Bt,L", [(0, 3, 1300), (0, 2, 8192), (0, 2, 5), (0, 1, 512), (6, 3, 33), (6, 32, 128), (6, 2, 1), (6, 5, 65)])
def test_edge_layer_backward_matches_fp64(msd_module, layer, Bt, L):
    """csrc/mg_disc_edge_bwd.cu (dx, dw, db of conv_pre and conv_post2, models.py:77,85) against autograd of F.conv1d in float64:
    tile boundaries (512 positions), sequences shorter than the kernel, single positions."""
    import torch.nn.functional as F
    from melgan_multi_b200.synth import DISCRIMINATOR_LAYERS
    with torch.no_grad():
        msd_module(torch.zeros(1, 1, 64).cuda(), torch.zeros(1, 1, 64).cuda())  # makes sure the weights are packed
    scale = 1
    _n, cin, cout, k, stride, groups, pad = DISCRIMINATOR_LAYERS[layer]
    conv = msd_module.discriminators[scale].layers()[layer]
    w = torch._weight_norm(conv.weight_v, conv.weight_g, 0).detach().double().requires_grad_(True)
    gen = torch.Generator(device="cpu").manual_seed(77 * layer + 13 * Bt + L)
    x = torch.randn(Bt, cin, L, generator=gen).cuda()
    dz = torch.randn(Bt, cout, L, generator=gen).cuda()
    xd = x.double().requires_grad_(True)
    rdx, rdw = torch.autograd.grad(F.conv1d(xd, w, None, stride, pad), (xd, w), dz.double())
    dx, dw, db = msd_module._dev.edge_backward(scale, layer, dz, x)
    for name, got, ref in (("dx", dx, rdx), ("dw", dw, rdw), ("db", db, dz.double().sum(dim=(0, 2)))):
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        m, l2 = rel_errors(got.cpu().numpy(), ref.float().cpu().numpy())
        assert m < 1e-5 and l2 < 1e-5, (name, m, l2)
    assert msd_module._dev.edge_backward(scale, layer, dz, x, need_dx=False)[0] is None


def test_standalone_discriminator_forward_and_backward(golden, dstate, msd_module):
    """Discriminator.forward on its own (reference models.py:87-103: returns (flattened logits, 7 feature maps)): scale 0 of
    the reference golden is exactly discriminators[0] applied to y, so the stand-alone module must reproduce it; its
    gradients must equal those of the same discriminator run inside the multi-scale stack's autograd function."""
    from melgan_multi_b200 import models
    B, L, seed = cases.MSD_CASES[0]
    d = models.Discriminator()
    d.load_state_dict({k[len("discriminators.0."):]: torch.from_numpy(v) for k, v in dstate.items()
                       if k.startswith("discriminators.0.")})
    d = d.cuda()
    y = torch.from_numpy(synth.audio_input(B, L, seed)).cuda()
    with torch.no_grad():
        logits, fmap = d(y)
    d._dev.check_status()
    tag = "msd_B%d_L%d_s%d" % (B, L, seed)
    ref = golden[tag + "_logit_r0"]
    assert logits.shape == ref.shape and len(fmap) == 7
    m, l2 = rel_errors(logits.cpu().numpy(), ref)
    assert m < TOL and l2 < TOL, (m, l2)
    for j in range(7):
        a = fmap[j].cpu().numpy()
        assert tuple(golden["%s_fmap_r0_%d_shape" % (tag, j)]) == a.shape
        m, _ = rel_errors(a[:, :4, :48], golden["%s_fmap_r0_%d_head" % (tag, j)])
        assert m < TOL, (j, m)
    # backward: loss on the logits and one feature map, against the strict-fp32 stock-op restatement of the same layers
    old = torch.backends.cudnn.conv.fp32_precision
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    try:
        yg = y.clone().requires_grad_(True)
        logits, fmap = d(yg)
        (logits.square().mean() + fmap[2].abs().mean()).backward()
        got = {n: p.grad.clone() for n, p in d.named_parameters()}
        gy = yg.grad.clone()
        d.zero_grad()
        import torch.nn.functional as F
        yr = y.clone().requires_grad_(True)
        x, maps = yr, []
        for l, (name, _cin, _cout, _k, stride, groups, pad) in enumerate(synth.DISCRIMINATOR_LAYERS):
            mod = d.layers()[l]
            w = torch._weight_norm(mod.weight_v, mod.weight_g, 0)
            x = F.conv1d(x, w, mod.bias, stride=stride, padding=pad, groups=groups)
            if l < 6:
                x = F.leaky_relu(x)
            maps.append(x)
        (maps[6].flatten(1).square().mean() + maps[2].abs().mean()).backward()
        for n, p in d.named_parameters():
            scale = p.grad.norm().item() + 1e-12
            assert (got[n] - p.grad).norm().item() <= 2e-3 * scale, (n, (got[n] - p.grad).norm().item(), scale)
        assert (gy - yr.grad).norm().item() <= 2e-3 * yr.grad.norm().item()
    finally:
        torch.backends.cudnn.conv.fp32_precision = old
