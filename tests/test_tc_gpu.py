"""GPU parity of the tensor-core (wgmma, split-bf16) path against the C oracle / reference goldens.
Tolerance: north_star allows 1e-3 relative; the 3-pass split keeps us near 1e-5, asserted at 1e-4."""
import numpy as np
import pytest
import torch

import cases
from conftest import rel_errors
from melgan_multi_b200 import engine, synth
from oracle import cport
from kernel_model import gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import TOL, oracle_resblock

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("stage,B,L", [(3, 2, 2100), (2, 2, 1000), (1, 2, 500), (0, 2, 200), (3, 1, 5), (0, 1, 8),
                                       (1, 1, 224), (1, 1, 225),
                                       # stage 0 (4-CTA clusters of 64-position tiles, 256 positions with a 16-row halo
                                       # only at the cluster's outer edges): lengths inside one cluster, one cluster and
                                       # one over, several clusters, odd tails; test_kernel_borders_gpu.py derives the
                                       # border lengths of every stage from the kernels' configuration
                                       (0, 1, 129), (0, 2, 144), (0, 3, 256), (0, 1, 257), (0, 2, 480), (0, 1, 481), (0, 2, 1000),
                                       (0, 1, 128), (0, 64, 256)])
def test_resblock_tc_matches_oracle(gstate, gdev, stage, B, L):
    C = 256 >> stage
    rs = np.random.RandomState(stage * 100 + L)
    x = rs.standard_normal((B, C, L)).astype(np.float32)
    ref = oracle_resblock(gstate, stage, x)
    y = gdev.resblock(stage, torch.from_numpy(x).cuda()).cpu().numpy()
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (stage, B, L, m, l2)


@pytest.mark.parametrize("stage,B,L", [(0, 2, 32), (0, 64, 32), (0, 1, 1), (0, 3, 130), (1, 2, 256), (1, 1, 5),
                                       (2, 2, 700), (2, 1, 1), (3, 2, 1500), (3, 1, 511), (3, 1, 512), (3, 1, 513)])
def test_convt_tc_matches_oracle(gstate, gdev, stage, B, L):
    cin = 512 >> stage
    S, pad = (8, 4) if stage < 2 else (2, 1)
    rs = np.random.RandomState(stage * 1000 + L + B)
    x = rs.standard_normal((B, cin, L)).astype(np.float32)
    name = "ups.%d" % stage
    w = cport.fold_weight_norm(gstate[name + ".weight_g"], gstate[name + ".weight_v"])
    lr = np.where(x > 0, x, x * np.float32(0.01)).astype(np.float32)
    ref = cport.conv_transpose1d(lr, w, gstate[name + ".bias"], S, pad)
    y = gdev.convt(stage, torch.from_numpy(x).cuda()).cpu().numpy()
    assert y.shape == ref.shape
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (stage, B, L, m, l2)


@pytest.mark.parametrize("stage,B,L", [(2, 2, 500), (2, 1, 1), (2, 1, 223), (2, 1, 224), (2, 3, 447), (2, 1, 4096),
                                       (1, 2, 300), (1, 1, 2), (1, 1, 222), (1, 1, 223), (1, 2, 2048),
                                       (0, 1, 3), (0, 2, 128), (0, 1, 129), (0, 3, 256), (0, 1, 223), (0, 2, 224), (0, 1, 600),
                                       (0, 64, 256)])
def test_resblock_with_tail_convt_matches_oracle(gstate, gdev, stage, B, L):
    """ResBlock `stage` + the NEXT stage's LeakyReLU -> ConvTranspose1d fused at its tail (what the tail-fused pipelines run:
    res0+up1, res1+up2, res2+up3) against the oracle's ResBlock followed by its conv_transpose1d.  Lengths straddle the tile
    borders of the tail-fused tiling (one more halo row on the left, position L owned by the last tile)."""
    C = 256 >> stage
    S, pad = (8, 4) if stage == 0 else (2, 1)
    rs = np.random.RandomState(9000 + 100 * stage + L + B)
    x = rs.standard_normal((B, C, L)).astype(np.float32)
    h = oracle_resblock(gstate, stage, x)
    name = "ups.%d" % (stage + 1)
    w = cport.fold_weight_norm(gstate[name + ".weight_g"], gstate[name + ".weight_v"])
    lr = np.where(h > 0, h, h * np.float32(0.01)).astype(np.float32)
    ref = cport.conv_transpose1d(lr, w, gstate[name + ".bias"], S, pad)
    y = gdev.resup(stage, torch.from_numpy(x).cuda()).cpu().numpy()
    assert y.shape == ref.shape
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (stage, B, L, m, l2)


@pytest.mark.parametrize("stage,B,Lin", [(2, 2, 500), (2, 1, 1), (2, 1, 64), (2, 3, 129), (2, 1, 2048), (3, 2, 1050), (3, 1, 1),
                                         (3, 1, 128), (3, 1, 255), (3, 2, 256), (3, 1, 4096)])
def test_fused_convt_resblock_matches_oracle(gstate, gdev, stage, B, Lin):
    """Stage 2 / 3 as ONE kernel (LeakyReLU -> ConvT k4 s2 -> ResBlock; what the default pipeline runs for stage 3) against the oracle's
    conv_transpose1d + ResBlock; odd and tiny lengths cover the pair de-interleave at both sequence ends, long ones the
    tile borders."""
    cin = 512 >> stage
    rs = np.random.RandomState(stage * 777 + Lin + B)
    x = rs.standard_normal((B, cin, Lin)).astype(np.float32)
    name = "ups.%d" % stage
    w = cport.fold_weight_norm(gstate[name + ".weight_g"], gstate[name + ".weight_v"])
    lr = np.where(x > 0, x, x * np.float32(0.01)).astype(np.float32)
    ref = oracle_resblock(gstate, stage, cport.conv_transpose1d(lr, w, gstate[name + ".bias"], 2, 1))
    y = gdev.upres(stage, torch.from_numpy(x).cuda()).cpu().numpy()
    assert y.shape == ref.shape
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (stage, B, Lin, m, l2)


@pytest.mark.parametrize("case", cases.GEN_CASES)
def test_tc_pipeline_matches_golden(golden, gstate, case):
    B, T, seed, realistic = case
    eng = engine.GeneratorHost(B, T)
    eng.load_state(gstate)
    y = eng.forward(synth.mel_input(B, T, seed, realistic))
    eng.close()
    m, l2 = rel_errors(y, golden[cases.gen_key(*case)])
    assert m < TOL and l2 < TOL, (case, m, l2)


@pytest.mark.parametrize("B,T", [(1, 1), (2, 32), (64, 32), (3, 130), (1, 1000)])
def test_conv_pre_kernel_matches_oracle(gstate, gdev, B, T):
    """conv_pre alone (conv_rows_tc_kernel<80,512,k7>; models.py:46,62) against the oracle's conv1d."""
    x = synth.mel_input(B, T, 50 + T)
    w = cport.fold_weight_norm(gstate["conv_pre.weight_g"], gstate["conv_pre.weight_v"])
    ref = cport.conv1d(x, w, gstate["conv_pre.bias"], 1, 3, 1, 1)
    y = gdev.conv_pre(torch.from_numpy(x).cuda()).cpu().numpy()
    assert y.shape == ref.shape
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (B, T, m, l2)


@pytest.mark.parametrize("B,L", [(2, 2100), (1, 5), (1, 1), (3, 487), (1, 488), (2, 8192)])
def test_resblock_post_tanh_matches_oracle(gstate, gdev, B, L):
    """The last stage's kernel on its own: ResBlock(32) -> LeakyReLU -> conv_post(32->1, k7) -> tanh fused in one epilogue
    (models.py:66-69) against the oracle's ResBlock + conv1d + tanh; lengths straddle the 512-position tiles (valid part 474)."""
    rs = np.random.RandomState(4000 + L)
    x = rs.standard_normal((B, 32, L)).astype(np.float32)
    h = oracle_resblock(gstate, 3, x)
    lr = np.where(h > 0, h, h * np.float32(0.01)).astype(np.float32)
    w = cport.fold_weight_norm(gstate["conv_post.weight_g"], gstate["conv_post.weight_v"])
    ref = np.tanh(cport.conv1d(lr, w, gstate["conv_post.bias"], 1, 3, 1, 1).astype(np.float64))
    y = gdev.resblock_post(torch.from_numpy(x).cuda()).cpu().numpy()
    assert y.shape == ref.shape == (B, 1, L)
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (B, L, m, l2)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_accuracy_margin_vs_strict_fp32_restatement(seed):
    """Accuracy margin of the 3-pass split-bf16 pipeline at config 2 over several weight seeds and both input
    distributions (N(0,1) and log-mel-like U(-11.5, 2), meldataset.py:22), against the stock-op restatement of the same
    module in STRICT fp32 on the same GPU (the goldens pin one weight seed; this sweeps more).  Tolerance of north_star: 1e-3;
    asserted at 1e-4 for the generator and 2e-4 for the discriminators' feature maps."""
    from melgan_multi_b200 import models
    old = torch.backends.cudnn.conv.fp32_precision
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    try:
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1000 + seed).items()})
        g = g.cuda().eval()
        vs, gs, bs = g._param_triplets()
        leaves = [t for trip in zip(vs, gs, bs) for t in trip]
        for realistic in (False, True):
            x = torch.from_numpy(synth.mel_input(64, 32, seed, realistic)).cuda()
            with torch.no_grad():
                m, l2 = rel_errors(g(x).cpu().numpy(), g._torch_forward(x, leaves).cpu().numpy())
            assert m < 1e-4 and l2 < 1e-4, (seed, realistic, m, l2)
        d = models.MultiScaleDiscriminator()
        d.load_state_dict({k: torch.from_numpy(v) for k, v in synth.discriminator_state(2000 + seed).items()})
        d = d.cuda().eval()
        vs, gs, bs = d._param_triplets()
        dleaves = [t for trip in zip(vs, gs, bs) for t in trip]
        y = torch.from_numpy(synth.audio_input(8, 8192, seed)).cuda()
        yh = torch.from_numpy(synth.audio_input(8, 8192, 100 + seed)).cuda()
        with torch.no_grad():
            _, _, fr, fg = d(y, yh)
            ref = d._torch_forward(torch.cat([y, yh]), dleaves)
        for s in range(3):
            for l in range(7):
                got = torch.cat([fr[s][l], fg[s][l]])
                m, l2 = rel_errors(got.cpu().numpy(), ref[7 * s + l].cpu().numpy())
                assert m < 2e-4 and l2 < 2e-4, (seed, s, l, m, l2)
    finally:
        torch.backends.cudnn.conv.fp32_precision = old
