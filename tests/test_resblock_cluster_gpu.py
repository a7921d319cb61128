"""The clustered ResBlock kernels (stage 0: 4-CTA clusters of 64-position tiles, stage 1: 2-CTA clusters of 128-position
tiles) against the C oracle, at lengths around the cluster borders: halos only at a cluster's outer edges, border rows
exchanged between the CTAs of a cluster, CTAs of a cluster with no valid rows."""
import numpy as np
import pytest
import torch

from conftest import rel_errors
from kernel_model import gdev, gstate  # noqa: F401 (fixtures)
from kernel_model import TOL, oracle_resblock

pytestmark = pytest.mark.gpu

# (stage, cluster positions CS * P, outputs of a cluster with more sequence on both sides)
CLUSTER = {0: (256, 224), 1: (256, 224)}


def _lengths(stage):
    pc, pv = CLUSTER[stage]
    first = pc - 16  # outputs of cluster 0 when more clusters follow
    return [
        pc, pc - 1, pc + 1,  # exactly one cluster, one short, one over
        pc + 4,  # a second cluster whose upper CTAs hold no valid rows
        first + pv, first + pv + 1,  # the border between clusters 1 and 2
        40, 1,  # shorter than one CTA's tile
    ]


@pytest.mark.parametrize("stage,B,L", [(s, B, L) for s in (0, 1) for L in _lengths(s) for B in (1, 3)]
                         + [(0, 64, 256), (1, 2, 2048), (1, 1, 1000)])
def test_clustered_resblock_matches_oracle(gstate, gdev, stage, B, L):
    C = 256 >> stage
    rs = np.random.RandomState(1000 * stage + L + B)
    x = rs.standard_normal((B, C, L)).astype(np.float32)
    ref = oracle_resblock(gstate, stage, x)
    y = gdev.resblock(stage, torch.from_numpy(x).cuda()).cpu().numpy()
    m, l2 = rel_errors(y, ref)
    assert m < TOL and l2 < TOL, (stage, B, L, m, l2)
