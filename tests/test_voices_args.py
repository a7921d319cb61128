"""Multi-voice batches without a GPU: every argument mg_gen_forward_voices refuses is reported (MG_ERR_INVALID_ARGUMENT and
a message naming it) before anything touches CUDA, and so are the Python wrappers' errors."""
import ctypes

import pytest
import torch

from melgan_multi_b200 import engine, models

MAX_B = 256  # MG_GEN_RAGGED_MAX_B, include/melgan_b200.h


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def _blobs(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def call(blobs, n_voices, voice, B=3, T=8, lens=None, precision=0, ws_bytes=None):
    L, p = engine.lib(), ctypes.c_void_p(256)
    ws = L.mg_gen_workspace_bytes(B, T) if ws_bytes is None else ws_bytes
    rc = L.mg_gen_forward_voices(blobs, n_voices, voice, p, p, B, T, lens, precision, p, ws, None)
    return rc, L.mg_last_error_string()


def test_refused_arguments():
    two = _blobs([256, 512])
    rc, msg = call(two, 2, _ints([0, 2, 1]))
    assert rc == -1 and b"voice[1] = 2" in msg and b"n_voices = 2" in msg
    rc, msg = call(two, 2, _ints([0, -1, 1]))
    assert rc == -1 and b"voice[1] = -1" in msg
    rc, msg = call(_blobs([256, None]), 2, _ints([0, 0, 0]))
    assert rc == -1 and b"packed[1] is NULL" in msg
    rc, msg = call(_blobs([256, 520]), 2, _ints([0, 1, 0]))
    assert rc == -1 and b"packed[1] must be 16-byte aligned" in msg
    rc, msg = call(two, 0, _ints([0, 0, 0]))
    assert rc == -1 and b"n_voices = 0" in msg
    rc, msg = call(None, 2, _ints([0, 0, 0]))
    assert rc == -1 and b"null packed or voice" in msg
    rc, msg = call(two, 2, None)
    assert rc == -1 and b"null packed or voice" in msg
    rc, msg = call(two, 2, _ints([0, 1, 0]), lens=_ints([4, 9, 8]))
    assert rc == -1 and b"lengths[1] = 9" in msg
    rc, msg = call(two, 2, _ints([0, 1, 0]), precision=7)
    assert rc == -1 and b"unknown precision 7" in msg
    rc, msg = call(two, 2, _ints([0, 1, 0]), B=0)
    assert rc == -1 and b"B >= 1" in msg
    rc, msg = call(two, 2, _ints([0, 1, 0]), ws_bytes=1024)
    assert rc == -4 and b"workspace" in msg  # MG_ERR_WORKSPACE_TOO_SMALL, as for mg_gen_forward_precision


def test_runs_not_items_are_limited():
    two = _blobs([256, 512])
    B = MAX_B + 1
    rc, msg = call(two, 2, _ints([i % 2 for i in range(B)]), B=B)  # every item its own run
    assert rc == -1 and b"257 runs" in msg and b"MG_GEN_RAGGED_MAX_B" in msg
    rc, msg = call(two, 2, _ints([0] * B), B=B, ws_bytes=1024)  # one run: B may exceed the limit
    assert rc == -4 and b"workspace" in msg


@pytest.mark.parametrize("mask", [2, 8])
def test_other_chains_refused(mask):
    two = _blobs([256, 512])
    engine.check(engine.lib().mg_gen_set_pipeline(mask))
    try:
        for precision in (0, 1):
            rc, msg = call(two, 2, _ints([0, 1, 0]), precision=precision)
            assert rc == -1 and b"default chain" in msg
    finally:
        engine.check(engine.lib().mg_gen_set_pipeline(-1))


def test_python_voice_validation():
    assert list(engine._voice_ids([0, 2, 1], 3, 3)) == [0, 2, 1]
    assert list(engine._voice_ids(torch.tensor([1, 0], dtype=torch.int64), 2, 2)) == [1, 0]
    for bad, what in (([0, 1], "entries"), ([0, 3, 1], "n_voices = 3"), ([0, -1, 1], "n_voices = 3"),
                      (torch.tensor([0.0, 1.0, 2.0]), "integer"), (torch.zeros(3, dtype=torch.int32, device="meta"), "CPU tensor")):
        with pytest.raises(engine.EngineError, match="voice") as e:
            engine._voice_ids(bad, 3, 3)
        assert what in str(e.value)


def test_python_refusals_without_a_device():
    g = models.Generator()
    mel = torch.zeros(2, 80, 4)
    with pytest.raises(engine.EngineError, match="CUDA"):
        models.generate_voices([g], mel, [0, 0])
    with pytest.raises(engine.EngineError, match="precision"):
        models.generate_voices([g], mel, [0, 0], precision="fp16")
