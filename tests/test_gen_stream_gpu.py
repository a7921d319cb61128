"""The streaming vocoder on the GPU (mg_gen_stream_*, Generator.stream): every session's concatenated output equals the
whole-utterance forward bit for bit, under seeded push schedules, at both precisions, with NaN-filled state and output
buffers."""
import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, synth
from kernel_model import gen, gstate  # noqa: F401 (fixtures)
from kernel_model import cluster_border_frames

pytestmark = pytest.mark.gpu

END, RESET = engine.STREAM_END, engine.STREAM_RESET


def mel_of(T, seed):
    return torch.from_numpy(synth.mel_input(1, T, seed)).cuda()


def nan_stream(gen, S, P, precision):
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    state = torch.full(((nbytes + 3) // 4,), float("nan"), device="cuda").view(torch.uint8)
    return engine.GeneratorStream(gen._ensure_packed, "cuda", S, P, precision, state=state)


class Runner:
    """Drives a stream slot by slot from queues of utterances, checking every step's counts and output buffer."""

    def __init__(self, st, guard=256):
        self.st, self.guard = st, guard
        self.look = st.lookahead_samples

    def step(self, frames, flags, mel):
        st = self.st
        n = len(frames)
        buf = torch.full((n * st.max_out + self.guard,), float("nan"), device="cuda")
        audio, counts = st.step_packed(mel, frames, flags, audio=buf[:n * st.max_out].view(n, st.max_out))
        rows = buf[:n * st.max_out].view(n, st.max_out)
        for i, m in enumerate(counts):
            assert not bool(torch.isnan(rows[i, :m]).any()), (i, m)
            assert bool(torch.isnan(rows[i, m:]).all()), (i, m)
        assert bool(torch.isnan(buf[n * st.max_out:]).all())
        return [rows[i, :m].clone() for i, m in enumerate(counts)], counts


def run_schedule(gen, st, utterances, n_slots, rng, P, p_end_empty=0.3):
    """Serve `utterances` (list of mel [1, 80, T]) through n_slots slots, each slot taking the next utterance when its last
    one ended.  Returns the concatenated audio of each utterance."""
    run = Runner(st)
    queue = list(range(len(utterances)))
    slot_utt = [None] * n_slots
    pos = [0] * n_slots
    out = {u: [] for u in queue}
    mel = torch.zeros((n_slots, 80, P), device="cuda")
    while queue or any(u is not None for u in slot_utt):
        frames, flags = [0] * n_slots, [0] * n_slots
        for i in range(n_slots):
            if slot_utt[i] is None and queue:
                slot_utt[i], pos[i] = queue.pop(0), 0
            u = slot_utt[i]
            if u is None:
                continue
            T = utterances[u].shape[2]
            n = int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))]))
            n = min(n, T - pos[i])
            frames[i] = n
            if n:
                mel[i, :, :n] = utterances[u][0, :, pos[i]:pos[i] + n]
            pos[i] += n
            # END with the last frames, or on a later 0-frame push
            if pos[i] == T and (n == 0 or rng.random() > p_end_empty):
                flags[i] = END
        got, counts = run.step(frames, flags, mel)
        for i in range(n_slots):
            u = slot_utt[i]
            if u is None:
                continue
            out[u].append(got[i])
            total = sum(x.numel() for x in out[u])
            T_pushed = pos[i]
            want = 256 * T_pushed if flags[i] & END else max(0, 256 * T_pushed - run.look)
            assert total == want, (u, T_pushed, total, want)
            if flags[i] & END:
                slot_utt[i] = None
    return [torch.cat(out[u]) for u in range(len(utterances))]


def test_chain_is_translation_invariant(gen):
    """The interior audio of mel[:, :, a:] equals the whole forward's bit for bit: no kernel's arithmetic depends on where
    a position falls in its tile.  The stream's equality contract rests on this."""
    T, look = 96, engine.lib().mg_gen_stream_lookahead()
    mel = mel_of(T, 3)
    for precision in ("fp32", "bf16"):
        whole = gen.generate(mel, precision=precision)[0, 0]
        for a in (1, 3, 8, 13, 29):
            sub = gen.generate(mel[:, :, a:].contiguous(), precision=precision)[0, 0]
            n = 256 * (T - a)
            assert torch.equal(sub[look:n - look], whole[256 * a + look:256 * a + n - look]), (precision, a)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sessions_equal_their_whole_forward(gen, precision):
    lens = [1, 2, 5, 6, 7, 31, 32, 33, 257, 1000] + cluster_border_frames()[:4]
    rng = np.random.default_rng(17)
    utts = [mel_of(T, 100 + i) for i, T in enumerate(lens)]
    P = 32
    st = nan_stream(gen, 8, P, precision)  # 14 utterances through 8 slots: slots are reused after END
    got = run_schedule(gen, st, utts, 8, rng, P)
    st.check_status()
    for u, T in enumerate(lens):
        ref = gen.generate(utts[u], precision=precision)[0, 0]
        assert got[u].numel() == 256 * T
        assert torch.equal(got[u], ref), (precision, T, float((got[u] - ref).abs().max()))
    gen._dev.check_status(1, max(lens))


def test_reset_mid_utterance(gen):
    P = 16
    st = nan_stream(gen, 2, P, "fp32")
    run = Runner(st)
    a, b = mel_of(40, 1), mel_of(23, 2)
    mel = torch.zeros((2, 80, P), device="cuda")
    for k in range(2):  # 32 frames of utterance a in slot 1, never ended
        mel[1] = a[0, :, 16 * k:16 * k + 16]
        run.step([0, 16], [0, 0], mel)
    out, pos = [], 0
    first = True
    while pos < 23:
        n = min(7, 23 - pos)
        mel[1, :, :n] = b[0, :, pos:pos + n]
        pos += n
        got, counts = run.step([0, n], [0, (RESET if first else 0) | (END if pos == 23 else 0)], mel)
        first = False
        out.append(got[1])
    assert torch.equal(torch.cat(out), gen.generate(b)[0, 0])
    st.check_status()


def test_many_sessions_small_pushes(gen):
    rng = np.random.default_rng(5)
    S, P = 256, 4
    lens = [int(v) for v in rng.integers(1, 41, S)]
    T = max(lens)
    mel = torch.from_numpy(synth.mel_input(S, T, 9)).cuda()
    st = gen.stream(S, P)
    outs = [[] for _ in range(S)]
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
        got = st.step(chunks, end=end)
        for i in range(S):
            if pos[i] >= 0:
                outs[i].append(got[i][0])
                if end[i]:
                    pos[i] = -1
    st.check_status()
    ref = gen.generate(mel, lens)
    for i, L in enumerate(lens):
        assert torch.equal(torch.cat(outs[i]), ref[i, 0, :256 * L]), i


def test_step_is_asynchronous(gen):
    P = 8
    st = gen.stream(4, P)
    mels = [mel_of(20, 40 + i) for i in range(4)]
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)  # ~0.1 s of device time queued ahead of the step
    got = st.step([m[0, :, :P] for m in mels])
    ev = torch.cuda.Event()
    ev.record()
    look = st.lookahead_samples
    assert [g.shape[1] for g in got] == [256 * 8 - look] * 4
    got2 = st.step([m[0, :, P:2 * P] for m in mels], end=[False, False, False, False])
    got3 = st.step([m[0, :, 2 * P:20] for m in mels], end=[True] * 4)
    assert [g.shape[1] for g in got2] == [256 * 8] * 4
    assert [g.shape[1] for g in got3] == [256 * 4 + look] * 4
    assert not ev.query()  # the counts were known while the device was still sleeping
    torch.cuda.synchronize()
    for i in range(4):
        assert torch.equal(torch.cat([got[i][0], got2[i][0], got3[i][0]]), gen.generate(mels[i])[0, 0])
    st.check_status()


def test_other_chain_is_refused(gen):
    L = engine.lib()
    st = gen.stream(2, 8)
    assert L.mg_gen_set_pipeline(10) == 0
    try:
        with pytest.raises(engine.EngineError, match="default chain"):
            st.step([mel_of(8, 1)[0]])
        with pytest.raises(engine.EngineError, match="default chain"):
            gen.stream(2, 8)
    finally:
        assert L.mg_gen_set_pipeline(-1) == 0
    m = mel_of(8, 1)
    got = st.step([m[0]], end=[True])
    assert torch.equal(got[0][0], gen.generate(m)[0, 0])
    st.check_status()
