"""Print the phase timeline (SM cycles) of one interior CTA of the tensor-core ResBlock kernel, per stage (clustered
stages: also the waits on the cluster neighbours' halo rows, and how many clusters the GPU keeps resident; codes 12 and 14:
also the phases of the fused front ConvT, and of conv_post)."""
import ctypes
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import engine, synth

state = synth.generator_state(1234)
gd = engine.GeneratorDevice("cuda:0")
order = [n for n, *_ in synth.GENERATOR_LAYERS]
to = lambda a: torch.from_numpy(a).cuda()
gd.pack([to(state[n + ".weight_v"]) for n in order], [to(state[n + ".weight_g"]) for n in order],
        [to(state[n + ".bias"]) for n in order])
L = engine.lib()
L.mg_gen_resblock_trace.restype = ctypes.c_int
L.mg_gen_resblock_trace.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_void_p]
# stage codes: the plain ResBlocks 0..3 (res0, res1, res2 of the default chain), 14 (its up3+res3+post) and 12 (up2+res2);
# config 2
for stage in (0, 1, 2, 3, 14, 12):
    C, Lp = (32, 8192) if stage == 14 else (64, 4096) if stage == 12 else (256 >> stage, 32 * [8, 64, 128, 256][stage])
    x = torch.randn(64, 2 * C, Lp // 2, device="cuda") if stage >= 12 else torch.randn(64, C, Lp, device="cuda")
    y = torch.empty(64, 1, Lp, device="cuda") if stage == 14 else torch.empty_like(x)
    tr = np.zeros(128, np.int64)
    for _ in range(2):
        engine.check(L.mg_gen_resblock_trace(gd.packed.data_ptr(), stage, x.data_ptr(), y.data_ptr(), 64, Lp, tr.ctypes.data))
    t0 = tr[0]
    e = lambda i: int(tr[i] - t0)
    clustered = tr[127] > 0
    print("stage %d (C=%d): load %d | total %d cycles" % (stage, C, e(1), e(20))
          + (" | max active clusters %d" % tr[127] if clustered else ""))
    if stage >= 12:  # the fused front ConvT, and the conv_post epilogue of code 14
        print("  front: operand in shared memory +%d | ConvT MMAs +%d | de-interleave +%d | slack rows + first hand-off +%d"
              % (e(21), tr[22] - tr[21], tr[23] - tr[22], tr[1] - tr[23])
              + (" | conv_post: per-tap sums %d, then to the stored audio %d" % (tr[26] - tr[24], tr[25] - tr[26]) if stage == 14 else ""))
    for c in range(6):
        print("  conv %d: X handed @%7d (+%5d after the previous hand-off) | mma: recv +%5d, weights +%5d, issued +%6d | acc ready @%7d (mma phase %6d) | epilogue %6d"
              % (c, e(2 + 3 * c), tr[2 + 3 * c] - tr[1 + 3 * c], tr[64 + 3 * c] - tr[2 + 3 * c], tr[65 + 3 * c] - tr[64 + 3 * c], tr[66 + 3 * c] - tr[65 + 3 * c],
                 e(3 + 3 * c), tr[3 + 3 * c] - tr[2 + 3 * c], (tr[4 + 3 * c] - tr[3 + 3 * c]) if c < 5 else (tr[20] - tr[18]))
              + (" | halo: wait full %5d, wait free %5d" % (tr[89 + 2 * c] - tr[88 + 2 * c],
                                                         (tr[101 + 2 * c] - tr[100 + 2 * c]) if c > 0 else 0) if clustered else ""))
