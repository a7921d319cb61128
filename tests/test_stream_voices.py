"""Streams of many voices without a GPU (mg_gen_stream_step_voices, mg_gen_stream_dry_step_voices): every refusal is
reported (MG_ERR_INVALID_ARGUMENT and a message naming it) before any CUDA call, a slot's voice binds on the step that
opens its utterance and changes only at RESET or after END, and at one voice the plan is mg_gen_stream_dry_step's."""
import ctypes

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models

END, RESET = engine.STREAM_END, engine.STREAM_RESET


def _ints(v):
    return (ctypes.c_int * max(len(v), 1))(*v)


def _blobs(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def handle(S, P):
    h = ctypes.c_void_p()
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    # create makes no CUDA call and a dry step never touches the state: any aligned address will do
    assert engine.lib().mg_gen_stream_create(ctypes.byref(h), S, P, 0, ctypes.c_void_p(1 << 20), nbytes) == 0
    return h


def dry(h, n_voices, voice, frames, flags):
    """(rc, out_samples, kernel_items, copy_bytes) of one dry step; voice None passes NULL."""
    n = len(frames)
    cnt, items, nbytes = (ctypes.c_int * max(n, 1))(), (ctypes.c_int * 8)(), ctypes.c_longlong()
    rc = engine.lib().mg_gen_stream_dry_step_voices(h, n_voices, None if voice is None else _ints(voice), _ints(frames),
                                                    _ints(flags), n, cnt, items, ctypes.byref(nbytes))
    return rc, list(cnt)[:n], list(items), nbytes.value


def dry_one(h, frames, flags):
    n = len(frames)
    cnt, items, nbytes = (ctypes.c_int * max(n, 1))(), (ctypes.c_int * 8)(), ctypes.c_longlong()
    rc = engine.lib().mg_gen_stream_dry_step(h, _ints(frames), _ints(flags), n, cnt, items, ctypes.byref(nbytes))
    return rc, list(cnt)[:n], list(items), nbytes.value


def test_step_refusals_before_any_cuda_call():
    L = engine.lib()
    p = ctypes.c_void_p(1 << 20)
    h = handle(4, 8)
    try:
        cnt = (ctypes.c_int * 4)()

        def step(blobs, n_voices, voice, frames=(3, 1), flags=None, mel=p, audio=p, out=cnt):
            fl = None if flags is None else _ints(flags)
            rc = L.mg_gen_stream_step_voices(h, blobs, n_voices, None if voice is None else _ints(voice), mel, _ints(frames),
                                             fl, len(frames), audio, out, None)
            return rc, L.mg_last_error_string()

        two = _blobs([256, 512])
        rc, msg = step(two, 0, [0, 0])
        assert rc == -1 and b"n_voices = 0" in msg
        rc, msg = step(two, -3, None)
        assert rc == -1 and b"n_voices = -3" in msg
        rc, msg = step(None, 2, [0, 1])
        assert rc == -1 and b"null argument" in msg
        rc, msg = step(_blobs([256, None]), 2, [0, 1])
        assert rc == -1 and b"packed[1] is NULL" in msg
        rc, msg = step(_blobs([256, 520]), 2, [0, 0])
        assert rc == -1 and b"packed[1] must be 16-byte aligned" in msg  # checked even when no slot uses it
        rc, msg = step(two, 2, [0, 2])
        assert rc == -1 and b"voice[1] = 2" in msg and b"n_voices = 2" in msg
        rc, msg = step(two, 2, [-1, 0])
        assert rc == -1 and b"voice[0] = -1" in msg
        # what mg_gen_stream_step refuses, refused here too
        rc, msg = step(two, 2, [0, 1], frames=(9, 1))
        assert rc == -1 and b"max_push_frames" in msg
        rc, msg = step(two, 2, [0, 1], frames=(0, 1), flags=(END, 0))
        assert rc == -1 and b"no frames" in msg
        rc, msg = step(two, 2, [0, 1], flags=(0, 4))
        assert rc == -1 and b"flags" in msg
        rc, msg = step(two, 2, [0, 1], mel=None)
        assert rc == -1 and b"null mel" in msg
        rc, msg = step(two, 2, [0, 1], audio=None)
        assert rc == -1 and b"null argument" in msg
        rc, msg = step(two, 2, [0, 1], out=None)
        assert rc == -1 and b"null argument" in msg
        rc, msg = step(two, 2, [0, 1, 0, 1, 0], frames=(0,) * 5)
        assert rc == -1 and b"max_sessions" in msg
        assert L.mg_gen_set_pipeline(14) == 0
        try:
            rc, msg = step(two, 2, [0, 1])
            assert rc == -1 and b"default chain" in msg
        finally:
            assert L.mg_gen_set_pipeline(-1) == 0
        # the one-voice call names itself
        assert L.mg_gen_stream_step(h, None, p, _ints([1]), None, 1, p, cnt, None) == -1
        assert b"mg_gen_stream_step:" in L.mg_last_error_string()
        # nothing above reached the device: the handle has nothing to check
        assert L.mg_gen_stream_check_status(h, None) == 0
    finally:
        L.mg_gen_stream_destroy(h)


def test_dry_step_refusals():
    h = handle(4, 8)
    try:
        rc, *_ = dry(h, 0, None, [1], [0])
        assert rc == -1 and b"n_voices = 0" in engine.lib().mg_last_error_string()
        rc, *_ = dry(h, 3, [3], [1], [0])
        assert rc == -1 and b"voice[0] = 3" in engine.lib().mg_last_error_string()
        assert dry(h, 3, [1, 2], [4, 2], [0, 0])[0] == 0  # opens slots 0 (voice 1) and 1 (voice 2)
        rc, *_ = dry(h, 3, [2, 2], [1, 1], [0, 0])
        msg = engine.lib().mg_last_error_string()
        assert rc == -1 and b"voice[0] = 2" in msg and b"bound to voice 1" in msg and b"RESET" in msg
        rc, *_ = dry(h, 3, [1, 1], [0, 0], [0, 0])
        assert rc == -1 and b"voice[1] = 1" in engine.lib().mg_last_error_string()  # a 0-frame push is still a step of it
        rc, *_ = dry(h, 3, None, [0, 0], [0, 0])  # NULL: voice 0, not slot 0's voice
        assert rc == -1 and b"bound to voice 1" in engine.lib().mg_last_error_string()
        # refused steps changed nothing: the slots still hold 4 and 2 frames in voices 1 and 2
        rc, cnt, _, _ = dry(h, 3, [1, 2], [0, 0], [END, END])
        assert rc == 0 and cnt == [256 * 4, 256 * 2]
    finally:
        engine.lib().mg_gen_stream_destroy(h)


@pytest.mark.parametrize("seed", range(4))
def test_binding_over_seeded_schedules(seed):
    """A model of the binding rule against the planner: a switch is accepted on a free slot, at RESET and after END,
    refused mid-utterance (and a refused step changes nothing); n_voices changes between steps."""
    rng = np.random.default_rng(seed)
    S, P = 12, int(rng.choice([1, 4, 8, 32]))
    look = engine.lib().mg_gen_stream_lookahead()
    h = handle(S, P)
    seen = {"free_slot": 0, "switch_reset": 0, "switch_after_end": 0, "refused": 0}
    try:
        # per slot: frames of the open utterance (0: none open), samples emitted, the last voice bound (kept after the
        # utterance closes, to tell a switch), whether the last utterance closed by END
        t, emitted, bound, ended = [0] * S, [0] * S, [None] * S, [False] * S
        for _ in range(250):
            n_voices = int(rng.integers(1, 6))
            n = int(rng.integers(1, S + 1))
            frames = [int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))])) for _ in range(n)]
            flags, voice = [], []
            for i in range(n):
                fl = RESET if rng.random() < 0.05 else 0
                if rng.random() < 0.1 and (t[i] + frames[i] > 0 or fl):
                    fl |= END
                if (fl & END) and (0 if fl & RESET else t[i]) + frames[i] == 0:
                    frames[i] = 1
                flags.append(fl)
                keep = bound[i] is not None and not (fl & RESET) and bound[i] < n_voices and rng.random() < 0.9
                voice.append(bound[i] if keep else int(rng.integers(0, n_voices)))
            # what the rule predicts: a slot with an open utterance and no RESET must keep its voice
            bad = [i for i in range(n) if t[i] > 0 and not (flags[i] & RESET) and voice[i] != bound[i]]
            rc, cnt, items, nbytes = dry(h, n_voices, voice, frames, flags)
            if bad:
                assert rc == -1, (voice, bound)
                assert b"voice[%d]" % bad[0] in engine.lib().mg_last_error_string()
                seen["refused"] += 1
                continue
            assert rc == 0, engine.lib().mg_last_error_string()
            assert all(0 <= v <= n for v in items) and nbytes >= 0
            for i in range(n):
                if t[i] > 0 and flags[i] & RESET and voice[i] != bound[i]:
                    seen["switch_reset"] += 1
                elif t[i] == 0 and ended[i] and voice[i] != bound[i]:
                    seen["switch_after_end"] += 1
                elif t[i] == 0 and not ended[i]:
                    seen["free_slot"] += 1
                if flags[i] & RESET:
                    t[i] = emitted[i] = 0
                    ended[i] = False
                t[i] += frames[i]
                emitted[i] += cnt[i]
                if t[i] > 0:
                    bound[i] = voice[i]
                    ended[i] = False
                if flags[i] & END:
                    assert emitted[i] == 256 * t[i]
                    t[i] = emitted[i] = 0
                    ended[i] = True
                else:
                    assert emitted[i] == max(0, 256 * t[i] - look)
        assert all(v > 0 for v in seen.values()), seen
    finally:
        engine.lib().mg_gen_stream_destroy(h)


@pytest.mark.parametrize("seed", range(3))
def test_one_voice_plans_like_dry_step(seed):
    """At one voice (NULL ids, or every id 0) the twin gives mg_gen_stream_dry_step's counts, items and copy bytes; and
    since the walk only renumbers items, any assignment of voices gives the same."""
    rng = np.random.default_rng(100 + seed)
    S, P = 16, int(rng.choice([2, 8, 32]))
    hs = [handle(S, P) for _ in range(4)]
    try:
        t = [0] * S
        for _ in range(200):
            frames = [int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))])) for _ in range(S)]
            flags = []
            for i in range(S):
                fl = RESET if rng.random() < 0.02 else 0
                t0 = 0 if fl & RESET else t[i]
                if rng.random() < 0.08 and (t0 + frames[i] > 0 or fl):
                    fl |= END
                if (fl & END) and t0 + frames[i] == 0:
                    frames[i] = 1
                flags.append(fl)
                t[i] = 0 if fl & END else t0 + frames[i]
            ref = dry_one(hs[0], frames, flags)
            assert ref[0] == 0
            assert dry(hs[1], 1, None, frames, flags) == ref
            assert dry(hs[2], 1, [0] * S, frames, flags) == ref
            # slot i always on voice i % 3: never a switch, so never refused
            assert dry(hs[3], 3, [i % 3 for i in range(S)], frames, flags) == ref
    finally:
        for h in hs:
            engine.lib().mg_gen_stream_destroy(h)


def test_python_refusals_without_a_device():
    with pytest.raises(engine.EngineError, match="at least one"):
        models.stream_voices([])
    with pytest.raises(engine.EngineError, match="CUDA"):
        models.stream_voices([models.Generator()])
    with pytest.raises(engine.EngineError, match="precision"):
        models.stream_voices([models.Generator()], precision="fp16")
    with pytest.raises(engine.EngineError, match="voice"):
        engine._voice_ids([0, 3], 2, 3)
    assert list(engine._voice_ids(torch.tensor([2, 0]), 2, 3)) == [2, 0]
