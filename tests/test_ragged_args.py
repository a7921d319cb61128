"""Ragged batches without a GPU: every argument error of mg_gen_forward_ragged / mg_gen_engine_forward_ragged and of the
Python wrappers is reported (negative code + message, or EngineError) before anything touches CUDA."""
import ctypes

import pytest
import torch

from melgan_multi_b200 import engine, models

MAX_B = 256  # MG_GEN_RAGGED_MAX_B, include/melgan_b200.h


def _ints(v):
    return (ctypes.c_int * len(v))(*v)


def test_forward_ragged_argument_errors():
    L, p = engine.lib(), ctypes.c_void_p(256)
    ws = L.mg_gen_workspace_bytes(3, 8)

    def call(B, T, lens, ws_bytes=ws):
        rc = L.mg_gen_forward_ragged(p, p, p, B, T, lens, p, ws_bytes, None)
        return rc, L.mg_last_error_string()

    rc, msg = call(3, 8, None)
    assert rc == -1 and b"null lengths" in msg
    rc, msg = call(3, 8, _ints([4, 0, 8]))
    assert rc == -1 and b"lengths[1] = 0" in msg
    rc, msg = call(3, 8, _ints([4, 9, 8]))
    assert rc == -1 and b"lengths[1] = 9" in msg and b"T_max = 8" in msg
    rc, msg = call(0, 8, _ints([1]))
    assert rc == -1 and b"B >= 1" in msg
    rc, msg = call(MAX_B + 1, 8, _ints([1] * (MAX_B + 1)))
    assert rc == -1 and b"MG_GEN_RAGGED_MAX_B" in msg
    rc, msg = call(3, 8, _ints([4, 1, 8]), ws - 1)
    assert rc == -4 and b"workspace" in msg  # MG_ERR_WORKSPACE_TOO_SMALL, as for mg_gen_forward
    assert L.mg_gen_forward_ragged(None, p, p, 3, 8, _ints([4, 1, 8]), p, ws, None) == -1
    assert b"null argument" in L.mg_last_error_string()


def test_engine_forward_ragged_argument_errors():
    L, p = engine.lib(), ctypes.c_void_p(256)
    assert L.mg_gen_engine_forward_ragged(None, p, p, 2, 8, None) == -1
    assert b"null lengths" in L.mg_last_error_string()
    assert L.mg_gen_engine_forward_ragged(None, p, p, 2, 8, _ints([8, 9])) == -1
    assert b"lengths[1] = 9" in L.mg_last_error_string()
    assert L.mg_gen_engine_forward_ragged(None, p, p, MAX_B + 1, 8, _ints([1] * (MAX_B + 1))) == -1
    assert b"MG_GEN_RAGGED_MAX_B" in L.mg_last_error_string()
    assert L.mg_gen_engine_forward_ragged(None, p, p, 0, 8, _ints([1])) == -1
    assert L.mg_gen_engine_forward_ragged(None, p, p, 2, 8, _ints([8, 1])) == -1  # valid lengths, no engine
    assert b"mg_gen_engine_forward_ragged: null argument" in L.mg_last_error_string()


def test_python_lengths_validation():
    assert list(engine._lengths([3, 1, 8], 3, 8)) == [3, 1, 8]
    assert list(engine._lengths((2, 2), 2, 2)) == [2, 2]
    assert list(engine._lengths(torch.tensor([5, 1], dtype=torch.int64), 2, 5)) == [5, 1]
    for bad, what in (([3, 1], "entries"), ([3, 0, 8], "[1, T_max"), ([3, 9, 8], "[1, T_max"),
                      (torch.tensor([1.0, 2.0, 3.0]), "integer"), (torch.ones(3, dtype=torch.int32, device="meta"), "CPU tensor")):
        with pytest.raises(engine.EngineError, match=r"lengths") as e:
            engine._lengths(bad, 3, 8)
        assert what in str(e.value)


def test_generate_refuses_cpu_tensors():
    g = models.Generator()
    with pytest.raises(engine.EngineError, match="CUDA"):
        g.generate(torch.zeros(2, 80, 4), [4, 2])
