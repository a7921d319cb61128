"""GPU cross-check of the product (wgmma split-bf16) generator against an independent second implementation: the
first-generation fp32 SIMT kernels, built into the TEST-ONLY library libmelgan_b200_simt_test.so (csrc/testlib).  The
product library does not contain that code; this file is the only thing that loads it."""
import ctypes

import numpy as np
import pytest
import torch

import cases
from conftest import rel_errors
from melgan_multi_b200 import build, engine, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def simt():
    L = ctypes.CDLL(build.TEST_LIB)
    L.mg_simt_gen_forward.restype = ctypes.c_int
    L.mg_simt_gen_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_void_p, ctypes.c_void_p]
    L.mg_simt_last_error_string.restype = ctypes.c_char_p
    return L


@pytest.fixture(scope="module")
def dev():
    state = synth.generator_state(1234)
    gd = engine.GeneratorDevice("cuda:0")
    order = [n for n, *_ in synth.GENERATOR_LAYERS]
    to = lambda a: torch.from_numpy(a).cuda()
    gd.pack([to(state[n + ".weight_v"]) for n in order], [to(state[n + ".weight_g"]) for n in order],
            [to(state[n + ".bias"]) for n in order])
    return gd


def simt_forward(simt, dev, mel):
    B, _, T = mel.shape
    out = torch.empty((B, 1, 256 * T), dtype=torch.float32, device="cuda")
    ws = dev.workspace(B, T)
    rc = simt.mg_simt_gen_forward(dev.packed.data_ptr(), mel.data_ptr(), out.data_ptr(), B, T, ws.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream)
    assert rc == 0, simt.mg_simt_last_error_string()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", cases.GEN_CASES)
def test_simt_matches_reference_golden(golden, simt, dev, case):
    B, T, seed, realistic = case
    y = simt_forward(simt, dev, torch.from_numpy(synth.mel_input(B, T, seed, realistic)).cuda()).cpu().numpy()
    m, l2 = rel_errors(y, golden[cases.gen_key(*case)])
    assert m < 2e-5 and l2 < 2e-5, (case, m, l2)  # fp32 FFMA: exact to summation order


def test_config2_two_independent_implementations_agree(simt, dev):
    """Config 2 (B=64, T=32): fp32 SIMT vs split-bf16 wgmma."""
    x = torch.from_numpy(synth.mel_input(64, 32, 0)).cuda()
    y_simt = simt_forward(simt, dev, x).cpu().numpy()
    y_tc = dev.forward(x).cpu().numpy()
    m, l2 = rel_errors(y_tc, y_simt)
    assert m < 1e-4 and l2 < 1e-4, (m, l2)
