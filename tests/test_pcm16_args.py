"""16-bit PCM output without a GPU: every argument mg_gen_forward_pcm16, mg_gen_stream_step_pcm16 and
mg_gen_engine_forward_pcm16 refuse is reported (an error code and a message naming it) before anything touches CUDA, and
so are the Python wrappers' errors.  Fake device addresses stand in for buffers: a call that reached CUDA would fail with
MG_ERR_CUDA instead."""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models

MAX_B = 256  # MG_GEN_RAGGED_MAX_B, include/melgan_b200.h
END, RESET = engine.STREAM_END, engine.STREAM_RESET
INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL


def _ints(v):
    return (ctypes.c_int * max(len(v), 1))(*v)


def _blobs(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def forward(blobs, n_voices, voice, B=3, T=8, lens=None, precision=0, ws_bytes=None, mel=256, audio=256, ws=256):
    L = engine.lib()
    nbytes = L.mg_gen_workspace_bytes(B, T) if ws_bytes is None else ws_bytes
    rc = L.mg_gen_forward_pcm16(blobs, n_voices, None if voice is None else _ints(voice), mel, audio, B, T,
                                None if lens is None else _ints(lens), precision, ws, nbytes, None)
    return rc, L.mg_last_error_string()


def test_forward_refusals_with_voices():
    two = _blobs([256, 512])
    for voice, what in (([0, 2, 1], b"voice[1] = 2"), ([0, -1, 1], b"voice[1] = -1")):
        rc, msg = forward(two, 2, voice)
        assert rc == INVALID and what in msg and b"mg_gen_forward_pcm16" in msg
    rc, msg = forward(_blobs([256, None]), 2, [0, 0, 0])
    assert rc == INVALID and b"packed[1] is NULL" in msg
    rc, msg = forward(_blobs([256, 520]), 2, [0, 1, 0])
    assert rc == INVALID and b"packed[1] must be 16-byte aligned" in msg
    rc, msg = forward(two, 0, [0, 0, 0])
    assert rc == INVALID and b"n_voices = 0" in msg
    rc, msg = forward(None, 2, [0, 0, 0])
    assert rc == INVALID and b"null packed" in msg
    rc, msg = forward(two, 2, [0, 1, 0], lens=[4, 9, 8])
    assert rc == INVALID and b"lengths[1] = 9" in msg
    rc, msg = forward(two, 2, [0, 1, 0], lens=[4, 0, 8])
    assert rc == INVALID and b"lengths[1] = 0" in msg
    rc, msg = forward(two, 2, [0, 1, 0], precision=7)
    assert rc == INVALID and b"unknown precision 7" in msg
    rc, msg = forward(two, 2, [0, 1, 0], B=0)
    assert rc == INVALID and b"B >= 1" in msg
    rc, msg = forward(two, 2, [0, 1, 0], T=0)
    assert rc == INVALID and b"T >= 1" in msg
    for null in ("mel", "audio", "ws"):
        rc, msg = forward(two, 2, [0, 1, 0], **{null: None})
        assert rc == INVALID and b"null argument" in msg, null
    rc, msg = forward(two, 2, [0, 1, 0], ws=264)
    assert rc == INVALID and b"aligned" in msg
    rc, msg = forward(two, 2, [0, 1, 0], ws_bytes=1024)
    assert rc == WS_SMALL and b"workspace" in msg
    B = MAX_B + 1  # runs, not items, are limited, as for mg_gen_forward_voices
    rc, msg = forward(two, 2, [i % 2 for i in range(B)], B=B)
    assert rc == INVALID and b"257 runs" in msg
    rc, msg = forward(two, 2, [0] * B, B=B, ws_bytes=1024)
    assert rc == WS_SMALL


def test_forward_refusals_without_voices():
    """voice NULL: every item on packed[0], refused as mg_gen_forward_precision refuses (a ragged batch has at most
    MG_GEN_RAGGED_MAX_B items), and the blobs are still checked."""
    one = _blobs([256])
    rc, msg = forward(one, 1, None, lens=[4, 9, 8])
    assert rc == INVALID and b"lengths[1] = 9" in msg
    rc, msg = forward(one, 1, None, lens=[1] * (MAX_B + 1), B=MAX_B + 1)
    assert rc == INVALID and b"MG_GEN_RAGGED_MAX_B" in msg
    rc, msg = forward(one, 1, None, B=1 << 13, T=1 << 12)
    assert rc == INVALID and b"too large" in msg
    rc, msg = forward(one, 1, None, precision=-1)
    assert rc == INVALID and b"unknown precision -1" in msg
    rc, msg = forward(_blobs([None]), 1, None)
    assert rc == INVALID and b"packed[0] is NULL" in msg
    rc, msg = forward(_blobs([256, 520]), 2, None)
    assert rc == INVALID and b"packed[1] must be 16-byte aligned" in msg
    rc, msg = forward(None, 1, None)
    assert rc == INVALID and b"null packed" in msg
    rc, msg = forward(one, 0, None)
    assert rc == INVALID and b"n_voices = 0" in msg
    rc, msg = forward(one, 1, None, audio=None)
    assert rc == INVALID and b"null argument" in msg
    rc, msg = forward(one, 1, None, ws_bytes=16)
    assert rc == WS_SMALL


@pytest.mark.parametrize("mask", [2, 4, 8, 14])
def test_other_chains_refused(mask):
    """Only the default chain has an int16 last kernel: any other is refused at both precisions, with or without voices,
    by every new entry point -- also at fp32, where the float calls run it."""
    L = engine.lib()
    engine.check(L.mg_gen_set_pipeline(mask))
    try:
        for precision in (0, 1):
            for blobs, n, voice in ((_blobs([256, 512]), 2, [0, 1, 0]), (_blobs([256]), 1, None)):
                rc, msg = forward(blobs, n, voice, precision=precision)
                assert rc == INVALID and b"default chain" in msg
            rc = L.mg_gen_engine_forward_pcm16(None, ctypes.c_void_p(256), ctypes.c_void_p(256), 2, 4, None, precision)
            assert rc == INVALID and b"default chain" in L.mg_last_error_string()
    finally:
        engine.check(L.mg_gen_set_pipeline(-1))


def test_engine_refusals():
    L = engine.lib()
    p = ctypes.c_void_p(256)

    def call(e=None, mel=p, audio=p, B=2, T=4, lens=None, precision=0):
        rc = L.mg_gen_engine_forward_pcm16(e, mel, audio, B, T, None if lens is None else _ints(lens), precision)
        return rc, L.mg_last_error_string()

    for kw, what in ((dict(precision=3), b"unknown precision 3"), (dict(B=0), b"B >= 1"), (dict(T=0), b"T >= 1"),
                     (dict(lens=[1, 5]), b"lengths[1] = 5"), (dict(lens=[0, 1]), b"lengths[0] = 0"),
                     (dict(B=MAX_B + 1, lens=[1] * (MAX_B + 1)), b"MG_GEN_RAGGED_MAX_B"), (dict(), b"null argument"),
                     (dict(e=p, mel=None), b"null argument"), (dict(e=p, audio=None), b"null argument")):
        rc, msg = call(**kw)
        assert rc == INVALID and what in msg and b"mg_gen_engine_forward_pcm16" in msg, kw


def handle(S, P):
    h = ctypes.c_void_p()
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    # create makes no CUDA call and a refused or dry step never touches the state: any aligned address will do
    assert engine.lib().mg_gen_stream_create(ctypes.byref(h), S, P, 0, ctypes.c_void_p(1 << 20), nbytes) == 0
    return h


def test_stream_step_refusals_before_any_cuda_call():
    L = engine.lib()
    p = ctypes.c_void_p(1 << 20)
    h = handle(4, 8)
    try:
        cnt = (ctypes.c_int * 4)()

        def step(blobs, n_voices, voice, frames=(3, 1), flags=None, mel=p, audio=p, out=cnt, s=h):
            fl = None if flags is None else _ints(flags)
            rc = L.mg_gen_stream_step_pcm16(s, blobs, n_voices, None if voice is None else _ints(voice), mel, _ints(frames),
                                            fl, len(frames), audio, out, None)
            return rc, L.mg_last_error_string()

        two = _blobs([256, 512])
        for args, kw, what in (((two, 0, [0, 0]), {}, b"n_voices = 0"), ((None, 2, [0, 1]), {}, b"null argument"),
                               ((_blobs([256, None]), 2, [0, 1]), {}, b"packed[1] is NULL"),
                               ((_blobs([256, 520]), 2, [0, 0]), {}, b"packed[1] must be 16-byte aligned"),
                               ((two, 2, [0, 2]), {}, b"voice[1] = 2"), ((two, 2, [-1, 0]), {}, b"voice[0] = -1"),
                               ((two, 2, [0, 1]), dict(frames=(9, 1)), b"max_push_frames"),
                               ((two, 2, [0, 1]), dict(frames=(0, 1), flags=(END, 0)), b"no frames"),
                               ((two, 2, [0, 1]), dict(flags=(0, 4)), b"flags"),
                               ((two, 2, [0, 1]), dict(mel=None), b"null mel"),
                               ((two, 2, [0, 1]), dict(audio=None), b"null argument"),
                               ((two, 2, [0, 1]), dict(out=None), b"null argument"),
                               ((two, 2, [0, 1]), dict(s=None), b"null argument"),
                               ((two, 2, [0, 1, 0, 1, 0]), dict(frames=(0,) * 5), b"max_sessions")):
            rc, msg = step(*args, **kw)
            assert rc == INVALID and what in msg and b"mg_gen_stream_step_pcm16" in msg, what
        assert L.mg_gen_set_pipeline(14) == 0
        try:
            rc, msg = step(two, 2, [0, 1])
            assert rc == INVALID and b"default chain" in msg
        finally:
            assert L.mg_gen_set_pipeline(-1) == 0
        # a handle advanced by a dry step refuses real steps of either format
        cnt1, items, nbytes = (ctypes.c_int * 4)(), (ctypes.c_int * 8)(), ctypes.c_longlong()
        assert L.mg_gen_stream_dry_step_voices(h, 2, _ints([1]), _ints([2]), None, 1, cnt1, items, ctypes.byref(nbytes)) == 0
        rc, msg = step(two, 2, [0], frames=(1,))
        assert rc == INVALID and b"advanced by mg_gen_stream_dry_step" in msg
        # nothing above reached the device: the handle has nothing to check
        assert L.mg_gen_stream_check_status(h, None) == 0
    finally:
        L.mg_gen_stream_destroy(h)


def test_dry_step_counts_are_the_float_steps():
    """The dry step describes the float step whichever format later steps use: its counts and copy bytes do not depend on
    anything the int16 step adds (the handle is the same)."""
    L = engine.lib()
    a, b = handle(2, 8), handle(2, 8)
    try:
        for frames, flags in (([3, 8], [0, 0]), ([8, 0], [0, 0]), ([1, 2], [END, RESET])):
            res = []
            for h in (a, b):
                cnt, items, nbytes = (ctypes.c_int * 2)(), (ctypes.c_int * 8)(), ctypes.c_longlong()
                assert L.mg_gen_stream_dry_step(h, _ints(frames), _ints(flags), 2, cnt, items, ctypes.byref(nbytes)) == 0
                res.append((list(cnt), list(items), nbytes.value))
            assert res[0] == res[1]
            assert res[0][2] > 0
    finally:
        L.mg_gen_stream_destroy(a)
        L.mg_gen_stream_destroy(b)


def test_python_dtype_validation():
    assert engine._pcm16(torch.float32) is False and engine._pcm16(torch.int16) is True
    for bad in (torch.float16, torch.bfloat16, torch.int32, torch.uint8, np.int16, "int16", None):
        with pytest.raises(engine.EngineError, match="dtype"):
            engine._pcm16(bad)
    assert engine._pcm16_np(np.float32) is False and engine._pcm16_np(np.int16) is True
    assert engine._pcm16_np(np.dtype("int16")) is True
    for bad in (np.float64, np.int32, np.uint16, "int16", torch.int16):
        with pytest.raises(engine.EngineError, match="dtype"):
            engine._pcm16_np(bad)
    assert engine._audio_out(torch, None, (2, 1, 512), True, torch.device("cpu")).dtype == torch.int16
    with pytest.raises(engine.EngineError, match="dtype"):
        engine._audio_out(torch, torch.zeros(2, 1, 512, dtype=torch.int16), (2, 1, 512), False, torch.device("cpu"))
    with pytest.raises(engine.EngineError, match="dtype"):
        engine._audio_out(torch, torch.zeros(2, 1, 512), (2, 1, 512), True, torch.device("cpu"))
    with pytest.raises(engine.EngineError, match="shape"):
        engine._audio_out(torch, torch.zeros(2, 1, 256, dtype=torch.int16), (2, 1, 512), True, torch.device("cpu"))
    with pytest.raises(engine.EngineError, match="int16 array"):
        engine.GeneratorHost._out(np.zeros((2, 1, 512), np.float32), (2, 1, 512), True)
    with pytest.raises(engine.EngineError, match="float32 array"):
        engine.GeneratorHost._out(np.zeros((2, 1, 512), np.int16), (2, 1, 512), False)


def test_python_refusals_without_a_device():
    g = models.Generator()
    mel = torch.zeros(2, 80, 4)
    with pytest.raises(engine.EngineError, match="dtype"):
        g.generate(mel, dtype=torch.float16)
    with pytest.raises(engine.EngineError, match="CUDA"):
        g.generate(mel, dtype=torch.int16)
    with pytest.raises(engine.EngineError, match="dtype"):
        models.generate_voices([g], mel, [0, 0], dtype=torch.int32)
    with pytest.raises(engine.EngineError, match="dtype"):
        g.stream(dtype=torch.float64)
    with pytest.raises(engine.EngineError, match="CUDA"):
        g.stream(dtype=torch.int16)
    with pytest.raises(engine.EngineError, match="dtype"):
        models.stream_voices([g], dtype=torch.bfloat16)
