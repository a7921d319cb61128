"""The streaming stride-2 ConvT kernel (stages 2 and 3, convt_stream_tc_kernel) on its own, against a float64
restatement of LeakyReLU -> ConvTranspose1d, element by element:

    |y - y64| <= TAU * A2 + 2^-20 * |y64|,      A2 = sqrt(conv_transpose64(lrelu(x)^2, w^2))

(test_layer_isolation_gpu's bound and TAU).  The lengths come from the tile geometry the library reports
(mg_gen_convt_config): a tile is ROWS virtual rows of the batch's items concatenated with one zero row after each, the
grid is min(tiles, SMs) persistent CTAs, and up to MAXSEG item segments of a tile are staged by bulk copy (rows of
items shorter than that allows are read straight from global memory).  Each item must equal its own B = 1 call bit
for bit, and two calls in a row must be bit-identical.  Ragged batches run through the whole generator, where stage 2's
ConvT is a chain kernel of its own."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, models
from kernel_model import gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import REL, TAU, check_items, folded64, ragged_batch

CONFIG_RE = r"convt_stream_tc_kernel<StreamCfg<(\d+),(\d+),(\d+),(\d+)>>"


def geometry(stage):
    m = re.fullmatch(CONFIG_RE, engine.lib().mg_gen_convt_config(stage).decode())
    assert m, stage
    st, rows, maxseg, nsx = (int(v) for v in m.groups())
    assert st == stage
    return dict(ROWS=rows, MAXSEG=maxseg, NSX=nsx)


def test_convt_config_names_report_every_stage():
    """Stages 2 and 3 report their streaming geometry, the stride-8 stages their tiles; unknown stages nothing."""
    for s in (2, 3):
        g = geometry(s)
        assert g["ROWS"] % 64 == 0 and g["MAXSEG"] >= 3 and g["NSX"] >= 2, g
    assert re.fullmatch(r"convt_tc_kernel<UpCfg<0,\d+,\d+>>", engine.lib().mg_gen_convt_config(0).decode())
    assert re.fullmatch(r"convt_resident_tc_kernel<UpCfg<1,\d+,\d+>>", engine.lib().mg_gen_convt_config(1).decode())
    assert engine.lib().mg_gen_convt_config(4) == b"" and engine.lib().mg_gen_convt_config(-1) == b""


def border_cases(stage):
    """(B, Lin) around the tile borders: one item of Lin + 1 virtual rows ending just before, on and after a tile border
    (and the first row of a tile being an item's zero row), tiles that span two and three items, items shorter than
    the staged segments allow (more than MAXSEG items in one tile), row strides that are not a multiple of 4 floats, a
    short last tile, and more tiles than two passes of a persistent grid."""
    R = geometry(stage)["ROWS"]
    out = []
    for k in (1, 2, 3):
        out += [(1, k * R - 2), (1, k * R - 1), (1, k * R), (2, k * R - 1), (3, k * R + 1)]
    out += [(3, R // 2 + 1), (4, R - 40), (5, 1), (9, 7), (7, 30), (6, 63), (5, 64), (2, 333), (3, 1001)]
    out += [(200, 4 * R)]  # 200 (4R + 1) / R > 800 tiles: more than two passes of an H100's 132 persistent CTAs
    return sorted(set(out))


def bound_ratio(state, stage, x, y):
    """Worst |y - y64| / (TAU A2 + 2^-20 |y64|) over every element."""
    w, b = folded64(state, "ups.%d" % stage)
    k = w.shape[2]
    a = F.leaky_relu(x.double())
    ref = F.conv_transpose1d(a, w, b, stride=k // 2, padding=k // 4)
    a2 = F.conv_transpose1d(a * a, w * w, None, stride=k // 2, padding=k // 4).sqrt()
    assert y.shape == ref.shape
    return float(((y.double() - ref).abs() / (TAU * a2 + REL * ref.abs()).clamp_min(1e-300)).max())


def inputs(stage, B, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 512 >> stage, L, generator=g).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [2, 3])
def test_convt_stream_config2(gstate, gdev, stage):
    """The bench workload's shape (config 2: 64 items of 32 mel frames), every element within the bound; two calls agree bit
    for bit, and items 0, 31 and 63 equal their own B = 1 calls."""
    L = 32 * (64 if stage == 2 else 128)
    x = inputs(stage, 64, L, 20 + stage)
    y = gdev.convt(stage, x)
    r = bound_ratio(gstate, stage, x, y)
    print("stage %d config 2: worst ratio to the bound %.3f" % (stage, r))
    assert r <= 1.0, r
    assert torch.equal(gdev.convt(stage, x), y)
    for i in (0, 31, 63):
        assert torch.equal(gdev.convt(stage, x[i:i + 1].contiguous()), y[i:i + 1]), i


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [2, 3])
def test_convt_stream_tile_borders(gstate, gdev, stage):
    worst = 0.0
    for B, L in border_cases(stage):
        x = inputs(stage, B, L, 1000 * stage + 7 * B + L)
        y = gdev.convt(stage, x)
        r = bound_ratio(gstate, stage, x, y)
        worst = max(worst, r)
        assert r <= 1.0, (B, L, r)
        assert torch.equal(gdev.convt(stage, x), y), (B, L)
        for i in sorted({0, B // 2, B - 1}):
            assert torch.equal(gdev.convt(stage, x[i:i + 1].contiguous()), y[i:i + 1]), (B, L, i)
    print("stage %d tile borders: worst ratio to the bound %.3f" % (stage, worst))


@pytest.mark.gpu
def test_convt_stream_ragged(gstate):
    """Ragged batches through the generator (stage 2's ConvT is its own chain kernel): item boundaries of the stage-2 input
    (64 positions per mel frame + one zero row) at every offset into a tile, NaN past each length; each item equals its
    own forward bit for bit and the audio past its end is 0."""
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in gstate.items()})
    g = g.cuda().eval()
    R = geometry(2)["ROWS"]
    lens = [1, 2, 3, R // 64, R // 64 + 1, 2 * R // 64 - 1, 7, 32, 31, 33, 5, 1, 20]
    rs = np.random.RandomState(5)
    rs.shuffle(lens)
    mel = ragged_batch(lens, 300)
    with torch.no_grad():
        audio = g.generate(mel, torch.tensor(lens))
    check_items(g, mel, lens, audio)
