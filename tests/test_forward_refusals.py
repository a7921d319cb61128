"""Every generator forward entry point refuses each single bad argument with the same code and a message naming the entry
point and the fault, before any CUDA call (no GPU needed): one table of faults, checked against all ten entry points, and
the Python wrappers' errors for bad mel, lengths, voice, precision and dtype.

Fake, 16-byte aligned device addresses stand in for buffers: a call that got past its checks would fail with MG_ERR_CUDA
instead.  A host-buffer call cannot be given a live engine without a device, so those rows pass engine = NULL as well;
mg_gen_engine_forward_ragged, _precision and _pcm16 check every other argument first, which is what their rows pin."""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine

INVALID, WS_SMALL = -1, -4  # MG_ERR_INVALID_ARGUMENT, MG_ERR_WORKSPACE_TOO_SMALL
P = 256                     # a fake device address (aligned)
MAX_B = 256                 # MG_GEN_RAGGED_MAX_B


def _ints(v):
    return None if v is None else (ctypes.c_int * max(len(v), 1))(*v)


def _ptrs(v):
    return None if v is None else (ctypes.c_void_p * len(v))(*v)


def _single(blobs):
    return None if blobs is None else blobs[0]


# entry point -> call(L, request); the request's fields are what the entry point takes
ENTRIES = {
    "mg_gen_forward": lambda L, r: L.mg_gen_forward(
        _single(r["blobs"]), r["mel"], r["audio"], r["B"], r["T"], r["ws"], r["ws_bytes"], None),
    "mg_gen_forward_ragged": lambda L, r: L.mg_gen_forward_ragged(
        _single(r["blobs"]), r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]), r["ws"], r["ws_bytes"], None),
    "mg_gen_forward_precision": lambda L, r: L.mg_gen_forward_precision(
        _single(r["blobs"]), r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]), r["precision"], r["ws"], r["ws_bytes"],
        None),
    "mg_gen_forward_voices": lambda L, r: L.mg_gen_forward_voices(
        _ptrs(r["blobs"]), r["n_voices"], _ints(r["voice"]), r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]),
        r["precision"], r["ws"], r["ws_bytes"], None),
    "mg_gen_forward_pcm16": lambda L, r: L.mg_gen_forward_pcm16(
        _ptrs(r["blobs"]), r["n_voices"], _ints(r["voice"]), r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]),
        r["precision"], r["ws"], r["ws_bytes"], None),
    "mg_gen_forward_pcm16/voice=NULL": lambda L, r: L.mg_gen_forward_pcm16(
        _ptrs(r["blobs"]), r["n_voices"], None, r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]), r["precision"],
        r["ws"], r["ws_bytes"], None),
    "mg_gen_forward_timed": lambda L, r: L.mg_gen_forward_timed(
        _single(r["blobs"]), r["mel"], r["audio"], r["B"], r["T"], r["ws"], r["ws_bytes"], None, r["kernel_ms"]),
    "mg_gen_engine_forward": lambda L, r: L.mg_gen_engine_forward(r["engine"], r["mel"], r["audio"], r["B"], r["T"]),
    "mg_gen_engine_forward_ragged": lambda L, r: L.mg_gen_engine_forward_ragged(
        r["engine"], r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"])),
    "mg_gen_engine_forward_precision": lambda L, r: L.mg_gen_engine_forward_precision(
        r["engine"], r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]), r["precision"]),
    "mg_gen_engine_forward_pcm16": lambda L, r: L.mg_gen_engine_forward_pcm16(
        r["engine"], r["mel"], r["audio"], r["B"], r["T"], _ints(r["lengths"]), r["precision"]),
}

SINGLE = ("mg_gen_forward", "mg_gen_forward_ragged", "mg_gen_forward_precision", "mg_gen_forward_timed")
ARRAY = ("mg_gen_forward_voices", "mg_gen_forward_pcm16", "mg_gen_forward_pcm16/voice=NULL")
VOICES = ("mg_gen_forward_voices", "mg_gen_forward_pcm16")
DEVICE = SINGLE + ARRAY
HOST = ("mg_gen_engine_forward_ragged", "mg_gen_engine_forward_precision", "mg_gen_engine_forward_pcm16")
LENGTHS = ("mg_gen_forward_ragged", "mg_gen_forward_precision") + ARRAY + HOST
PRECISION = ("mg_gen_forward_precision",) + ARRAY + ("mg_gen_engine_forward_precision", "mg_gen_engine_forward_pcm16")
DEFAULT_CHAIN_ONLY = ARRAY + ("mg_gen_engine_forward_pcm16",)

# (fault, request fields changed, code, {entry points: message substring}); an entry point missing from a row does not
# take the argument, or accepts the value.  mg_gen_forward_timed checks alignment as mg_gen_forward does (it used to hand a
# misaligned blob or workspace to the kernels).
FAULTS = [
    ("null packed", dict(blobs=None), INVALID,
     {SINGLE: "null argument", ("mg_gen_forward_voices",): "null packed or voice array",
      ("mg_gen_forward_pcm16", "mg_gen_forward_pcm16/voice=NULL"): "null packed"}),
    ("null blob", dict(blobs=[None, 512]), INVALID, {SINGLE: "null argument", ARRAY: "packed[0] is NULL"}),
    ("misaligned blob", dict(blobs=[P + 8, 512]), INVALID,
     {SINGLE: "packed/workspace must be 16-byte aligned", ARRAY: "packed[0] must be 16-byte aligned"}),
    ("misaligned second blob", dict(blobs=[P, 520]), INVALID, {ARRAY: "packed[1] must be 16-byte aligned"}),
    ("null blob second", dict(blobs=[P, None]), INVALID, {ARRAY: "packed[1] is NULL"}),
    ("n_voices 0", dict(n_voices=0), INVALID, {ARRAY: "n_voices = 0"}),
    ("null mel", dict(mel=None), INVALID, {DEVICE + HOST: "null argument"}),
    ("null audio", dict(audio=None), INVALID, {DEVICE + HOST: "null argument"}),
    ("null workspace", dict(ws=None), INVALID, {DEVICE: "null argument"}),
    ("misaligned workspace", dict(ws=P + 8), INVALID, {DEVICE: "aligned"}),
    ("short workspace", dict(ws_short=True), WS_SMALL, {DEVICE: "workspace"}),
    ("B 0", dict(B=0), INVALID, {DEVICE + HOST: "B >= 1"}),
    ("T 0", dict(T=0), INVALID, {DEVICE + HOST: "T >= 1"}),
    ("B*T too large", dict(B=1 << 13, T=1 << 12), INVALID, {DEVICE + HOST: "too large"}),
    ("null lengths", dict(lengths=None), INVALID, {("mg_gen_forward_ragged", "mg_gen_engine_forward_ragged"): "null lengths"}),
    ("length past T_max", dict(lengths=[4, 9, 8]), INVALID, {LENGTHS: "lengths[1] = 9 is outside [1, T_max = 8]"}),
    ("length 0", dict(lengths=[4, 0, 8]), INVALID, {LENGTHS: "lengths[1] = 0"}),
    ("too many items", dict(B=MAX_B + 1, lengths=[1] * (MAX_B + 1), voice=[i % 2 for i in range(MAX_B + 1)]), INVALID,
     {tuple(e for e in LENGTHS if e not in VOICES): "B = 257 exceeds MG_GEN_RAGGED_MAX_B",
      VOICES: "257 runs of equal length and voice exceed MG_GEN_RAGGED_MAX_B"}),
    ("voice id past n_voices", dict(voice=[0, 2, 1]), INVALID, {VOICES: "voice[1] = 2 is outside [0, n_voices = 2)"}),
    ("voice id negative", dict(voice=[0, -1, 1]), INVALID, {VOICES: "voice[1] = -1"}),
    ("null voice", dict(voice=None), INVALID, {("mg_gen_forward_voices",): "null packed or voice array"}),
    ("unknown precision", dict(precision=7), INVALID, {PRECISION: "unknown precision 7"}),
    ("other chain at fp32", dict(chain=2), INVALID, {DEFAULT_CHAIN_ONLY: "default chain"}),
    ("other chain at bf16", dict(chain=2, precision=1), INVALID, {PRECISION: "default chain"}),
    ("null kernel_ms", dict(kernel_ms=None), INVALID, {("mg_gen_forward_timed",): "null argument"}),
    ("null engine", dict(), INVALID, {("mg_gen_engine_forward",) + HOST: "null argument"}),
]

CASES = [pytest.param(entry, change, code, what, id="%s-%s" % (fault.replace(" ", "_"), entry))
         for fault, change, code, expect in FAULTS for entries, what in expect.items() for entry in entries]


def _request(change):
    r = dict(blobs=[P, 512], voice=[0, 1, 0], lengths=[4, 1, 8], B=3, T=8, precision=0, mel=P, audio=P, ws=P,
             kernel_ms=(ctypes.c_float * 16)(), engine=None)
    r.update({k: v for k, v in change.items() if k not in ("ws_short", "chain")})
    r["n_voices"] = change.get("n_voices", 2)
    r["ws_bytes"] = engine.lib().mg_gen_workspace_bytes(max(r["B"], 1), max(r["T"], 1)) - (1 if change.get("ws_short") else 0)
    return r


@pytest.mark.parametrize("entry, change, code, what", CASES)
def test_single_fault_refused(entry, change, code, what):
    L = engine.lib()
    engine.check(L.mg_gen_set_pipeline(change.get("chain", -1)))
    try:
        rc = ENTRIES[entry](L, _request(change))
    finally:
        engine.check(L.mg_gen_set_pipeline(-1))
    msg = L.mg_last_error_string().decode()
    assert rc == code and what in msg and msg.startswith(entry.split("/")[0] + ":"), (rc, msg)


def test_every_entry_point_is_in_the_table():
    assert {e for _, _, _, expect in FAULTS for entries in expect for e in entries} == set(ENTRIES)


# ---- the Python wrappers --------------------------------------------------------------------------------------------

def _device():
    """A GeneratorDevice whose device is the CPU: every wrapper check runs, and nothing past them can."""
    d = object.__new__(engine.GeneratorDevice)
    d.torch, d.device = torch, torch.device("cpu")
    return d


def _host():
    h = object.__new__(engine.GeneratorHost)
    h._h = ctypes.c_void_p()
    return h


MEL = torch.zeros(2, 80, 4)
DEVICE_CALLS = {
    "forward": lambda d, mel=MEL, lengths=None, voice=None, **kw: d.forward(mel, **kw),
    "forward_ragged": lambda d, mel=MEL, lengths=(4, 2), voice=None, **kw: d.forward_ragged(mel, lengths, **kw),
    "forward_voices": lambda d, mel=MEL, lengths=None, voice=(0, 0), **kw: d.forward_voices([d], mel, voice, lengths, **kw),
}
DEVICE_REFUSALS = [
    ("precision", dict(precision="fp16"), "precision must be one of 'fp32', 'bf16' (got 'fp16')"),
    ("dtype", dict(dtype=torch.float16), "dtype must be torch.float32 or torch.int16"),
    ("mel channels", dict(mel=torch.zeros(2, 79, 4)), "mel must be [B, 80, {T}], got (2, 79, 4)"),
    ("mel rank", dict(mel=torch.zeros(80, 4)), "mel must be [B, 80, {T}], got (80, 4)"),
    ("mel dtype", dict(mel=torch.zeros(2, 80, 4, dtype=torch.float64)), "mel must be an fp32 tensor on cpu"),
    ("lengths entries", dict(lengths=[4]), "lengths has 1 entries for a batch of 2"),
    ("lengths range", dict(lengths=[4, 5]), "lengths must lie in [1, T_max = 4] (got 5)"),
    ("lengths float", dict(lengths=torch.tensor([4.0, 2.0])), "lengths must be a 1-D integer tensor"),
    ("lengths device", dict(lengths=torch.ones(2, dtype=torch.int32, device="meta")), "lengths must be a list, a tuple or a CPU tensor"),
    ("voice range", dict(voice=[0, 1]), "voice ids must lie in [0, n_voices = 1) (got 1)"),
    ("voice entries", dict(voice=[0]), "voice has 1 entries for a batch of 2"),
    ("voice float", dict(voice=torch.tensor([0.0, 0.0])), "voice must be a 1-D integer tensor"),
]


def _applicable(calls, refusals):
    """(method, refusal) pairs where the method takes the argument the refusal is about"""
    takes = {"lengths": ("forward_ragged", "forward_voices"), "voice": ("forward_voices",)}
    return [pytest.param(m, kw, message, id="%s-%s" % (m, what.replace(" ", "_"))) for what, kw, message in refusals
            for m in sorted(calls) if m in takes.get(what.split()[0], calls)]


@pytest.mark.parametrize("method, kw, message", _applicable(DEVICE_CALLS, DEVICE_REFUSALS))
def test_device_wrappers_refuse(method, kw, message):
    with pytest.raises(engine.EngineError) as e:
        DEVICE_CALLS[method](_device(), **kw)
    assert str(e.value).startswith(message.format(T="T" if method == "forward" else "T_max"))


def test_forward_voices_refuses_bad_voices():
    d = _device()
    with pytest.raises(engine.EngineError, match="at least one voice"):
        d.forward_voices([], MEL, [0, 0])
    with pytest.raises(engine.EngineError, match="every voice must be a GeneratorDevice on cpu"):
        d.forward_voices([d, object()], MEL, [0, 0])


HOST_MEL = np.zeros((2, 80, 4), np.float32)
HOST_CALLS = {
    "forward": lambda h, mel=HOST_MEL, lengths=None, **kw: h.forward(mel, **kw),
    "forward_ragged": lambda h, mel=HOST_MEL, lengths=(4, 2), **kw: h.forward_ragged(mel, lengths, **kw),
}
HOST_REFUSALS = [
    ("precision", dict(precision="fp16"), "precision must be one of 'fp32', 'bf16' (got 'fp16')"),
    ("dtype", dict(dtype=np.float64), "dtype must be np.float32 or np.int16"),
    ("mel channels", dict(mel=np.zeros((2, 79, 4), np.float32)), "mel must be [B, 80, {T}]"),
    ("lengths entries", dict(lengths=[4]), "lengths has 1 entries for a batch of 2"),
    ("lengths range", dict(lengths=[0, 4]), "lengths must lie in [1, T_max = 4] (got 0)"),
    ("out dtype", dict(dtype=np.int16, out=np.zeros((2, 1, 1024), np.float32)), "out must be a C-contiguous int16 array"),
]


@pytest.mark.parametrize("method, kw, message", _applicable(HOST_CALLS, HOST_REFUSALS))
def test_host_wrappers_refuse(method, kw, message):
    with pytest.raises(engine.EngineError) as e:
        HOST_CALLS[method](_host(), **kw)
    assert str(e.value).startswith(message.format(T="T" if method == "forward" else "T_max"))
