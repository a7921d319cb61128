"""Streams of many voices on the GPU (models.stream_voices / mg_gen_stream_step_voices): each session's concatenated audio
equals its own voice's whole-utterance forward bit for bit, however the voices are spread over the slots.

Every voice comes from a different seed, so an item that ran on a neighbour's blob would show in its audio.  The planner
walks the sessions by voice, so each kernel's items come in voice runs; the border test puts a voice change one conv_pre
row before, at and one row after a conv_pre tile border, and one step has more stride-2 ConvT tiles than twice the SMs,
so persistent CTAs walk from one voice into another."""
import re

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth

pytestmark = pytest.mark.gpu
SEEDS = (1234, 2718, 3141, 5772)
END, RESET = engine.STREAM_END, engine.STREAM_RESET


@pytest.fixture(scope="module")
def voices():
    out = []
    for seed in SEEDS:
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
        out.append(g.cuda().eval())
    return out


def mel_of(T, seed):
    return torch.from_numpy(synth.mel_input(1, T, seed)).cuda()


def nan_stream(voices, S, P, precision):
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    state = torch.full(((nbytes + 3) // 4,), float("nan"), device="cuda").view(torch.uint8)
    return engine.GeneratorStream(lambda: [g._ensure_packed() for g in voices], "cuda", S, P, precision, state=state)


def guarded_step(st, mel, frames, flags, voice, guard=256):
    """One step into a NaN-filled output buffer with a guard after it: every slot's samples written, nothing else."""
    n = len(frames)
    buf = torch.full((n * st.max_out + guard,), float("nan"), device="cuda")
    rows = buf[:n * st.max_out].view(n, st.max_out)
    _, counts = st.step_packed(mel, frames, flags, audio=rows, voice=voice)
    for i, m in enumerate(counts):
        assert not bool(torch.isnan(rows[i, :m]).any()), (i, m)
        assert bool(torch.isnan(rows[i, m:]).all()), (i, m)
    assert bool(torch.isnan(buf[n * st.max_out:]).all())
    return [rows[i, :m].clone() for i, m in enumerate(counts)], counts


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sessions_equal_their_voice_forward(voices, precision):
    """16 utterances, voices at random, through 8 slots on seeded push schedules (0-, 1- and full pushes, END on a 0-frame
    push); slots are reused in other voices after END, and four utterances open with a RESET that drops an unfinished
    throw-away utterance of another voice in their slot."""
    rng = np.random.default_rng(23)
    lens = [1, 2, 5, 6, 7, 31, 32, 33, 257, 600, 3, 64, 100, 17, 45, 9]
    utts = [mel_of(T, 300 + i) for i, T in enumerate(lens)]
    uvoice = [int(v) for v in rng.integers(0, len(voices), len(lens))]
    after_reset = {2, 6, 9, 12}
    S, P = 8, 32
    st = nan_stream(voices, S, P, precision)
    look = st.lookahead_samples
    queue = list(range(len(lens)))
    slot_utt, pos, last_voice = [None] * S, [0] * S, [None] * S
    drop = [None] * S  # a throw-away utterance in progress: [frames still to push, its voice, the utterance that follows]
    out = {u: [] for u in queue}
    switches = {"end": 0, "reset": 0}
    mel = torch.zeros((S, 80, P), device="cuda")
    refused = False
    while queue or any(u is not None for u in slot_utt) or any(d is not None for d in drop):
        frames, flags = [0] * S, [0] * S
        voice = [int(v) for v in rng.integers(0, len(voices), S)]  # a free slot takes any id
        for i in range(S):
            if drop[i] is not None and drop[i][0] == 0:  # RESET drops it and opens the next utterance in another voice
                _, old, u = drop[i]
                drop[i] = None
                uvoice[u] = (old + 1 + u % 3) % len(voices)
                slot_utt[i], pos[i] = u, 0
                flags[i] = RESET
                switches["reset"] += 1
            elif slot_utt[i] is None and drop[i] is None and queue:
                u = queue.pop(0)
                if u in after_reset:
                    drop[i] = [int(rng.integers(3, 41)), int(rng.integers(0, len(voices))), u]
                else:
                    if last_voice[i] is not None and last_voice[i] != uvoice[u]:
                        switches["end"] += 1
                    slot_utt[i], pos[i] = u, 0
            if drop[i] is not None:
                n = min(int(rng.choice([1, P, int(rng.integers(0, P + 1))])), drop[i][0])
                frames[i], voice[i] = n, drop[i][1]
                if n:
                    mel[i, :, :n] = mel_of(n, 7 + i)[0]
                drop[i][0] -= n
                continue
            u = slot_utt[i]
            if u is None:
                continue
            voice[i] = last_voice[i] = uvoice[u]
            T = lens[u]
            n = min(int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))])), T - pos[i])
            if flags[i] & RESET:
                n = max(n, 1)  # (a RESET with no frames would leave the slot free: let it open the utterance)
            frames[i] = n
            if n:
                mel[i, :, :n] = utts[u][0, :, pos[i]:pos[i] + n]
            pos[i] += n
            if pos[i] == T and (n == 0 or rng.random() > 0.3):
                flags[i] |= END
        if not refused:  # a changed id on an open slot is refused, and the refused step changes nothing
            open_slots = [i for i in range(S) if slot_utt[i] is not None and pos[i] - frames[i] > 0 and not flags[i] & RESET]
            if open_slots:
                bad = list(voice)
                bad[open_slots[0]] = (bad[open_slots[0]] + 1) % len(voices)
                with pytest.raises(engine.EngineError, match="bound to voice"):
                    st.step_packed(mel, frames, flags, voice=bad)
                refused = True
        got, counts = guarded_step(st, mel, frames, flags, voice)
        for i in range(S):
            u = slot_utt[i]
            if u is None:
                continue
            out[u].append(got[i])
            total = sum(x.numel() for x in out[u])
            assert total == (256 * pos[i] if flags[i] & END else max(0, 256 * pos[i] - look)), (u, pos[i], total)
            if flags[i] & END:
                slot_utt[i] = None
    st.check_status()
    assert refused and switches["reset"] == len(after_reset) and switches["end"] > 0, switches
    for u, T in enumerate(lens):
        got = torch.cat(out[u])
        ref = voices[uvoice[u]].generate(utts[u], precision=precision)[0, 0]
        assert got.numel() == 256 * T
        assert torch.equal(got, ref), (precision, u, T, uvoice[u], float((got - ref).abs().max()))


def _run_two_steps(voices, first, lens, voice, P, precision="fp32", seed=0):
    """Sessions i: a first push of first[i] frames (not ended), then the rest (lens[i] - first[i] <= P) with END.  Every
    session's audio must equal its voice's whole forward."""
    S = len(lens)
    st = nan_stream(voices, S, P, precision)
    mels = [mel_of(L, seed + i) for i, L in enumerate(lens)]
    m = torch.zeros((S, 80, P), device="cuda")
    for i in range(S):
        m[i, :, :first[i]] = mels[i][0, :, :first[i]]
    a, _ = guarded_step(st, m, first, [0] * S, voice)
    m = torch.zeros((S, 80, P), device="cuda")
    for i in range(S):
        m[i, :, :lens[i] - first[i]] = mels[i][0, :, first[i]:]
    b, _ = guarded_step(st, m, [L - f for L, f in zip(lens, first)], [END] * S, voice)
    st.check_status()
    for i in range(S):
        ref = voices[voice[i]].generate(mels[i], precision=precision)[0, 0]
        assert torch.equal(torch.cat([a[i], b[i]]), ref), (i, lens[i], voice[i], precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_voice_change_at_conv_pre_tile_borders(voices, precision):
    """On a first push the conv_pre window is the pushed frames (f >= 4 makes it run), f + PAD rows of its grid.  Voices
    0, 1 and 2 end one row before, at and one row after a tile border (each voice starts a tile), voice 3 follows; the
    slots are shuffled, so only the planner's walk puts each voice's items together."""
    m = re.fullmatch(r"conv_rows_tc_kernel<ConvCfg<80,512,(\d+),(\d+),\d+>>", engine.lib().mg_gen_conv_pre_config().decode())
    pad, rows = int(m.group(1)) // 2, int(m.group(2))
    P = 32

    def segment(d):  # first pushes (n - 1 of 4 frames, then one of f) whose rows end d past a tile border
        for n in range(1, 2 * rows + 2):
            for f in range(4, P + 1):
                if ((n - 1) * (4 + pad) + f + pad - d) % rows == 0:
                    return [4] * (n - 1) + [f]
        raise AssertionError((rows, d))
    first, voice = [], []
    for v, d in enumerate((-1, 0, 1)):
        seg = segment(d)
        first += seg
        voice += [v] * len(seg)
    first += [5, 13]
    voice += [3, 3]
    assert len(first) <= 256
    rng = np.random.default_rng(3)
    perm = rng.permutation(len(first))
    first = [first[j] for j in perm]
    voice = [voice[j] for j in perm]
    lens = [f + int(rng.integers(1, 20)) for f in first]
    _run_two_steps(voices, first, lens, voice, P, precision, seed=500)


def test_persistent_convt_crosses_voices(voices):
    """One step whose stride-2 ConvT (up2) has more than 2 x SMs tiles, voices interleaved slot by slot."""
    name = engine.lib().mg_gen_convt_config(2).decode()
    rows = int(re.fullmatch(r"\w+<(?:Up|Stream)Cfg<2,(\d+)(?:,\d+)+>>", name).group(1))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    P, S = 32, 64
    # an open session's final positions at up2's input after a first push of P frames (the host's exact_hi chain), its
    # whole window there: Lin + 1 rows of the ConvT grid
    F = P
    for r, a in ((1, 3), (8, 4), (1, 16), (8, 4), (1, 16)):
        F = r * F - a
    assert S * (F + 1) > 2 * sms * rows, (F, rows, sms)
    voice = [i % len(voices) for i in range(S)]
    lens = [P + 1 + i % 7 for i in range(S)]
    _run_two_steps(voices, [P] * S, lens, voice, P, seed=700)


def test_one_voice_equals_generator_stream(voices):
    rng = np.random.default_rng(9)
    S, P = 6, 8
    lens = [int(v) for v in rng.integers(1, 60, S)]
    mel = torch.from_numpy(synth.mel_input(S, max(lens), 11)).cuda()
    g = voices[1]
    pairs = [(models.stream_voices([g], S, P), g.stream(S, P), None),
             (models.stream_voices(voices, S, P), g.stream(S, P), [1] * S)]
    for sv, ref, voice in pairs:
        pos = [0] * S
        while any(p >= 0 for p in pos):
            chunks, end = [], []
            for i in range(S):
                if pos[i] < 0:
                    chunks.append(None)
                    end.append(False)
                    continue
                n = min(int(rng.integers(0, P + 1)), lens[i] - pos[i])
                chunks.append(mel[i, :, pos[i]:pos[i] + n])
                pos[i] += n
                end.append(pos[i] == lens[i])
            a = sv.step(chunks, end=end, voice=voice)
            b = ref.step(chunks, end=end)
            for x, y in zip(a, b):
                assert torch.equal(x, y)
            pos = [-1 if e else p for p, e in zip(pos, end)]
        sv.check_status()


def _schedule(lens, voice, P, seed):
    """Per step: (chunks, end, voice) pushing random 0..P frames per session until each ends."""
    rng = np.random.default_rng(seed)
    mels = [mel_of(L, seed + i) for i, L in enumerate(lens)]
    pos, steps = [0] * len(lens), []
    while any(p >= 0 for p in pos):
        chunks, end = [], []
        for i, L in enumerate(lens):
            if pos[i] < 0:
                chunks.append(None)
                end.append(False)
                continue
            n = min(int(rng.integers(0, P + 1)), L - pos[i])
            chunks.append(mels[i][0, :, pos[i]:pos[i] + n])
            pos[i] += n
            end.append(pos[i] == L)
        steps.append((chunks, end, voice))
        pos = [-1 if e else p for p, e in zip(pos, end)]
    return steps


def _drive(st, steps):
    outs = [[] for _ in steps[0][0]]
    for chunks, end, voice in steps:
        for i, a in enumerate(st.step(chunks, end=end, voice=voice)):
            outs[i].append(a)
    return [torch.cat(o, dim=1) for o in outs]


def test_two_handles_on_two_streams_equal_serial(voices):
    P = 16
    plans = [_schedule([40, 7, 90, 23], [3, 0, 1, 3], P, 800), _schedule([12, 70, 33], [2, 2, 0], P, 900)]
    serial = [_drive(models.stream_voices(voices, 4, P), s) for s in plans]
    torch.cuda.synchronize()
    handles = [models.stream_voices(voices, 4, P) for _ in plans]
    streams = [torch.cuda.Stream() for _ in plans]
    cur = torch.cuda.current_stream()
    outs = [[[] for _ in s[0][0]] for s in plans]
    for k in range(max(len(s) for s in plans)):  # the two handles' steps interleaved, each on its own stream
        for h, (st, s) in enumerate(zip(handles, plans)):
            if k >= len(s):
                continue
            streams[h].wait_stream(cur)
            with torch.cuda.stream(streams[h]):
                chunks, end, voice = s[k]
                for i, a in enumerate(st.step(chunks, end=end, voice=voice)):
                    a.record_stream(cur)
                    outs[h][i].append(a)
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for h in range(len(plans)):
        for i, ref in enumerate(serial[h]):
            assert torch.equal(torch.cat(outs[h][i], dim=1), ref), (h, i)
        handles[h].check_status()
