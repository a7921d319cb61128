"""CPU checks of the streaming vocoder (mg_gen_stream_*): the look-ahead and the window table restated in float64 on the
model's own layers, the host bookkeeping over seeded push schedules, and argument errors reported before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, synth
from oracle import torch_port

END, RESET = engine.STREAM_END, engine.STREAM_RESET
DIL = (1, 3, 9)


@pytest.fixture(scope="module")
def weights():
    ws, bs = torch_port.fold_state(synth.generator_state(1234))
    return [w.double() for w in ws], [b.double() for b in bs]


def lrelu(x):
    return F.leaky_relu(x, 0.1)


def resblock(ws, bs, i, x):
    for j, d in enumerate(DIL):
        a, b = 5 + 6 * i + j, 5 + 6 * i + 3 + j
        h = F.conv1d(lrelu(x), ws[a], bs[a], padding=d, dilation=d)
        x = F.conv1d(lrelu(h), ws[b], bs[b], padding=1) + x
    return x


def upsample(ws, bs, i, x):
    k = ws[1 + i].shape[2]
    return F.conv_transpose1d(lrelu(x), ws[1 + i], bs[1 + i], stride=k // 2, padding=k // 4)


# the default chain's eight kernels as float64 layer groups: (input channels, output / input scale, function)
def kernels(ws, bs):
    return [
        (80, 1, lambda x: F.conv1d(x, ws[0], bs[0], padding=3)),
        (512, 8, lambda x: upsample(ws, bs, 0, x)),
        (256, 1, lambda x: resblock(ws, bs, 0, x)),
        (256, 8, lambda x: upsample(ws, bs, 1, x)),
        (128, 1, lambda x: resblock(ws, bs, 1, x)),
        (128, 2, lambda x: upsample(ws, bs, 2, x)),
        (64, 1, lambda x: resblock(ws, bs, 2, x)),
        (64, 2, lambda x: torch.tanh(F.conv1d(lrelu(resblock(ws, bs, 3, upsample(ws, bs, 3, x))), ws[29], bs[29], padding=3))),
    ]


# exact outputs of a window [lo, hi) per kernel: (a, b) with the exact range [r lo + a, r hi - b)
TABLE = [(3, 3), (4, 4), (16, 16), (4, 4), (16, 16), (1, 1), (16, 16), (20, 20)]


def test_lookahead_is_the_models_receptive_field(weights):
    """Which audio samples mel frame t reaches, from the derivative of the float64 chain along a change of frame t (forward
    mode: a +1 perturbation's effect on the edge samples, ~1e-19, would be lost in rounding of the samples themselves)."""
    ws, bs = weights
    T, t = 24, 12
    mel = torch.from_numpy(synth.mel_input(1, T, 5)).double()
    tangent = torch.zeros_like(mel)
    tangent[0, :, t] = 1.0

    def chain(x):
        for _cin, _r, f in kernels(ws, bs):
            x = f(x)
        return x
    _, d = torch.func.jvp(chain, (mel,), (tangent,))
    changed = np.nonzero(d[0, 0].numpy())[0]
    look = engine.lib().mg_gen_stream_lookahead()
    # right side: frame t first reaches sample 256 t - lookahead, so [0, 256 t - lookahead) is final after frames [0, t)
    assert changed[0] == 256 * t - look == 1530
    # left side: the same reach, so a window needs 1542 samples of left context
    assert changed[-1] == 256 * (t + 1) - 1 + look == 4869
    assert len(changed) == changed[-1] - changed[0] + 1
    assert engine.lib().mg_gen_stream_max_out(8) == 256 * 8 + look


@pytest.mark.parametrize("k", range(8))
def test_window_table_per_kernel(weights, k):
    """Each kernel run on a window [lo, hi) of its input, zero-padded outside, matches the whole input's outputs exactly on
    the table's range and differs just outside it (the table is tight); at lo = 0 and at hi = the end it is exact to the
    edge."""
    ws, bs = weights
    cin, r, f = kernels(ws, bs)[k]
    a, b = TABLE[k]
    N = 90
    g = torch.Generator().manual_seed(k)
    x = torch.randn(1, cin, N, generator=g, dtype=torch.float64)
    with torch.no_grad():
        whole = f(x)
        for lo, hi in ((9, 70), (0, 70), (9, N)):
            y = f(x[:, :, lo:hi])
            s = r * lo + (a if lo > 0 else 0)
            e = r * hi - (b if hi < N else 0)
            got, ref = y[..., s - r * lo:e - r * lo], whole[..., s:e]
            assert torch.allclose(got, ref, rtol=0, atol=1e-10), (k, lo, hi)
            if lo > 0:
                assert (y[..., s - 1 - r * lo] - whole[..., s - 1]).abs().max() > 1e-6, (k, "left bound not tight")
            if hi < N:
                assert (y[..., e - r * lo] - whole[..., e]).abs().max() > 1e-6, (k, "right bound not tight")


def handle(S, P, precision=0):
    h = ctypes.c_void_p()
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    # create makes no CUDA call and a dry step never touches the state: any aligned address will do
    assert engine.lib().mg_gen_stream_create(ctypes.byref(h), S, P, precision, ctypes.c_void_p(1 << 20), nbytes) == 0
    return h


def dry_step(h, frames, flags):
    n = len(frames)
    cnt, items, nbytes = (ctypes.c_int * n)(), (ctypes.c_int * 8)(), ctypes.c_longlong()
    rc = engine.lib().mg_gen_stream_dry_step(h, (ctypes.c_int * n)(*frames), (ctypes.c_int * n)(*flags), n, cnt, items,
                                             ctypes.byref(nbytes))
    assert rc == 0, engine.lib().mg_last_error_string()
    return list(cnt), list(items), nbytes.value


@pytest.mark.parametrize("seed", range(4))
def test_bookkeeping_follows_the_contract(seed):
    rng = np.random.default_rng(seed)
    S, P = 16, int(rng.choice([1, 4, 8, 32]))
    look = engine.lib().mg_gen_stream_lookahead()
    h = handle(S, P)
    try:
        t, emitted = [0] * S, [0] * S
        for _ in range(300):
            frames = [int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))])) for _ in range(S)]
            flags = []
            for i in range(S):
                fl = RESET if rng.random() < 0.02 else 0
                if rng.random() < 0.08 and (t[i] + frames[i] > 0 or fl):
                    fl |= END
                if fl & RESET:
                    t[i] = emitted[i] = 0
                if (fl & END) and t[i] + frames[i] == 0:
                    frames[i] = 1
                flags.append(fl)
            cnt, items, nbytes = dry_step(h, frames, flags)
            assert all(0 <= v <= S for v in items) and nbytes >= 0
            for i in range(S):
                t[i] += frames[i]
                emitted[i] += cnt[i]
                assert 0 <= cnt[i] <= 256 * P + look
                if flags[i] & END:
                    assert emitted[i] == 256 * t[i]
                    t[i] = emitted[i] = 0
                else:
                    assert emitted[i] == max(0, 256 * t[i] - look)
        # a handle advanced without the device refuses real steps
        p = ctypes.c_void_p(256)
        one = (ctypes.c_int * 1)(1)
        assert engine.lib().mg_gen_stream_step(h, p, p, one, None, 1, p, (ctypes.c_int * 1)(), None) == -1
        assert b"dry_step" in engine.lib().mg_last_error_string()
    finally:
        engine.lib().mg_gen_stream_destroy(h)


def test_stream_argument_errors_are_reported_before_any_cuda_call():
    L = engine.lib()
    p = ctypes.c_void_p(1 << 20)
    nbytes = L.mg_gen_stream_state_bytes(4, 8)
    assert nbytes > 0 and L.mg_gen_stream_state_bytes(0, 8) == 0 and L.mg_gen_stream_state_bytes(257, 8) == 0
    assert L.mg_gen_stream_state_bytes(4, 0) == 0 and L.mg_gen_stream_max_out(0) == 0
    h = ctypes.c_void_p()
    assert L.mg_gen_stream_create(None, 4, 8, 0, p, nbytes) == -1
    assert L.mg_gen_stream_create(ctypes.byref(h), 4, 8, 0, None, nbytes) == -1
    assert L.mg_gen_stream_create(ctypes.byref(h), 0, 8, 0, p, nbytes) == -1 and b"max_sessions" in L.mg_last_error_string()
    assert L.mg_gen_stream_create(ctypes.byref(h), 257, 8, 0, p, nbytes) == -1
    assert L.mg_gen_stream_create(ctypes.byref(h), 4, 0, 0, p, nbytes) == -1 and b"max_push_frames" in L.mg_last_error_string()
    assert L.mg_gen_stream_create(ctypes.byref(h), 4, 8, 2, p, nbytes) == -1 and b"precision" in L.mg_last_error_string()
    assert L.mg_gen_stream_create(ctypes.byref(h), 4, 8, 0, p, nbytes - 1) == -4  # MG_ERR_WORKSPACE_TOO_SMALL
    assert L.mg_gen_stream_create(ctypes.byref(h), 4, 8, 0, ctypes.c_void_p((1 << 20) + 16), nbytes) == -1
    assert b"aligned" in L.mg_last_error_string()
    # another chain: create refused, the default restored by mg_gen_set_pipeline(-1)
    assert L.mg_gen_set_pipeline(10) == 0
    try:
        assert L.mg_gen_stream_create(ctypes.byref(h), 4, 8, 0, p, nbytes) == -1 and b"default chain" in L.mg_last_error_string()
    finally:
        assert L.mg_gen_set_pipeline(-1) == 0
    h = handle(4, 8)
    try:
        cnt = (ctypes.c_int * 4)()

        def step(frames, flags=None, mel=p, n=None):
            n = len(frames) if n is None else n
            fl = (ctypes.c_int * len(frames))(*flags) if flags is not None else None
            return L.mg_gen_stream_step(h, p, mel, (ctypes.c_int * len(frames))(*frames), fl, n, p, cnt, None)

        assert step([9]) == -1 and b"max_push_frames" in L.mg_last_error_string()
        assert step([-1]) == -1
        assert step([0, 0, 0, 0, 0]) == -1 and b"max_sessions" in L.mg_last_error_string()
        assert step([0], [END]) == -1 and b"no frames" in L.mg_last_error_string()
        assert step([0], [4]) == -1 and b"flags" in L.mg_last_error_string()
        assert step([3], mel=None) == -1 and b"null mel" in L.mg_last_error_string()
        assert L.mg_gen_stream_step(h, None, p, (ctypes.c_int * 1)(1), None, 1, p, cnt, None) == -1
        assert L.mg_gen_stream_step(h, p, p, None, None, 1, p, cnt, None) == -1
        assert L.mg_gen_stream_step(h, p, p, (ctypes.c_int * 1)(1), None, 1, p, None, None) == -1
        assert L.mg_gen_set_pipeline(14) == 0
        try:
            assert step([1]) == -1 and b"default chain" in L.mg_last_error_string()
        finally:
            assert L.mg_gen_set_pipeline(-1) == 0
        # a handle that has not stepped has nothing to check
        assert L.mg_gen_stream_check_status(h, None) == 0
    finally:
        L.mg_gen_stream_destroy(h)
