"""16-bit PCM output on the GPU: on every inference path and at both precisions, the int16 audio is bit for bit pcm16 of
the matching float call's audio, computed here on the host in float64:

    pcm16(a) = 0 if a is NaN, else clamp(rint(32768 a), -32768, 32767)    (rint: half to even)

Outputs go to sentinel-filled int16 buffers with guard regions before and after them, so a store outside the audio
(or a missing one) shows.  The data are made to hold the contract's edge cases, and the tests assert that they do:
samples at exactly +-1.0 (a generator whose conv_post drives tanh into saturation), samples with 32768 a exactly at a
half (ties).  NaN audio (a NaN mel frame) is int16 0: test_nonfinite_gpu holds every int16 path to that, item by item,
against float64."""
import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth
from kernel_model import ragged_batch

pytestmark = pytest.mark.gpu

END, RESET = engine.STREAM_END, engine.STREAM_RESET
SENT = 0x5A5A     # int16 sentinel of the guarded buffers
GUARD = 2048      # int16 elements before and after each output
SEEDS = (1234, 77, 4242)


def pcm16_np(a):
    """The contract in float64: a is fp32 audio (any shape) -> int16."""
    a = np.asarray(a, dtype=np.float32)
    s = np.clip(np.rint(32768.0 * a.astype(np.float64)), -32768, 32767)
    s[np.isnan(a)] = 0
    return s.astype(np.int16)


def pcm16_of(t):
    return pcm16_np(t.detach().cpu().numpy())


def guarded(shape):
    """(int16 CUDA view of `shape`, the whole sentinel-filled buffer with GUARD elements either side)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), SENT, dtype=torch.int16, device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def guards_ok(buf):
    return bool((buf[:GUARD] == SENT).all()) and bool((buf[-GUARD:] == SENT).all())


def make_gen(seed):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
    return g.cuda().eval()


@pytest.fixture(scope="module")
def gens():
    return [make_gen(s) for s in SEEDS]


def loud(seed, mel, lens, bias, spread=30.0):
    """The generator of `seed` with conv_post's gain raised and `bias` added to its bias, so that on mel its pre-tanh
    values spread about `bias` with a standard deviation of `spread`: at 30, tanh returns exactly +-1.0 (beyond about
    +-9.01) for a large share of the samples on both sides; at 1.5 most samples lie in (-1, 1) with large magnitudes,
    where a float32 sample is most often an odd multiple of 2^-16 (a tie).  The pre-tanh values of the unmodified
    generator are atanh of its audio."""
    g = make_gen(seed)
    a = g.generate(mel, lens).double()
    b0 = float(g.conv_post.bias.detach())
    z = torch.cat([torch.atanh(a[i, 0, :256 * L].clamp(-0.999999, 0.999999)) - b0 for i, L in enumerate(lens)])
    k = spread / float(z.std())
    with torch.no_grad():  # z' = b0 + k (z - b0) + shift = k (z - b0 - mean) + bias
        g.conv_post.weight_g.mul_(k)
        g.conv_post.bias.add_(bias - b0 - k * float(z.mean()))
    return g


def check_generate(gen, mel, lengths=None, precision="fp32"):
    """generate(dtype=int16) into a guarded buffer against pcm16 of generate(); returns the float audio."""
    B, _, T = mel.shape
    ref = gen.generate(mel, lengths, precision=precision)
    out, buf = guarded((B, 1, 256 * T))
    got = gen._ensure_packed().forward(mel, out=out, precision=precision, dtype=torch.int16) if lengths is None else \
        gen._ensure_packed().forward_ragged(mel, lengths, out=out, precision=precision, dtype=torch.int16)
    assert got.data_ptr() == out.data_ptr() and got.dtype == torch.int16
    gen._dev.check_status(B, T)
    assert guards_ok(buf)
    assert np.array_equal(out.cpu().numpy(), pcm16_of(ref))
    # the default out of generate() is int16 too, and equal
    again = gen.generate(mel, lengths, precision=precision, dtype=torch.int16)
    assert again.dtype == torch.int16 and again.shape == (B, 1, 256 * T) and torch.equal(again, out)
    return ref


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("B,T", [(64, 32), (7, 600), (4, 1), (1, 1)])
def test_uniform(gens, precision, B, T):
    """Config 2 (B = 64, T = 32: four batch slices), an uneven four-slice cut (7 x 600), and one-frame items."""
    mel = torch.from_numpy(synth.mel_input(B, T, 11 + B + T)).cuda()
    if (B, T) in ((64, 32), (7, 600)):
        assert engine.lib().mg_gen_forward_slices(B, T) == 4
    check_generate(gens[0], mel, precision=precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_ragged(gens, precision):
    """One-frame items among longer ones (NaN mel past every length, never read); the tails past 256 L_i are int16 0."""
    lens = [1, 7, 1, 33, 2, 64, 1, 40]
    mel = ragged_batch(lens, 500)
    ref = check_generate(gens[1], mel, lens, precision=precision)
    got = gens[1].generate(mel, lens, precision=precision, dtype=torch.int16).cpu().numpy()
    for i, L in enumerate(lens):
        assert not np.any(got[i, :, 256 * L:]), i
        assert not bool(torch.isnan(ref[i, :, :256 * L]).any())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("order", ["interleaved", "sorted"])
def test_voices(gens, precision, order):
    lens = [5, 1, 17, 32, 9, 1, 24, 3, 12]
    voice = [i % 3 for i in range(len(lens))] if order == "interleaved" else sorted(i % 3 for i in range(len(lens)))
    mel = ragged_batch(lens, 900)
    ref = models.generate_voices(gens, mel, voice, lens, precision=precision)
    out, buf = guarded((len(lens), 1, 256 * mel.shape[2]))
    got = models.generate_voices(gens, mel, voice, lens, precision=precision, dtype=torch.int16)
    dev = gens[0]._ensure_packed()
    dev.forward_voices([g._ensure_packed() for g in gens], mel, voice, lens, out=out, precision=precision, dtype=torch.int16)
    dev.check_status(len(lens), mel.shape[2])
    assert guards_ok(buf)
    want = pcm16_of(ref)
    assert np.array_equal(out.cpu().numpy(), want) and np.array_equal(got.cpu().numpy(), want)
    # uniform voices (lengths None) too
    mel_u = torch.from_numpy(synth.mel_input(6, 8, 3)).cuda()
    ref_u = models.generate_voices(gens, mel_u, [2, 0, 1, 1, 0, 2], precision=precision)
    got_u = models.generate_voices(gens, mel_u, [2, 0, 1, 1, 0, 2], precision=precision, dtype=torch.int16)
    assert np.array_equal(got_u.cpu().numpy(), pcm16_of(ref_u))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("bias", [5.0, -5.0])
def test_saturation_and_ties(gens, precision, bias):
    """tanh returns exactly +-1.0 for large arguments: +1.0 must give 32767 (a plain cast of 32768 would wrap to -32768)
    and -1.0 -32768.  The same data hold samples whose 32768 a is exactly at a half, rounded half to even."""
    lens = [64, 1, 64, 25, 64, 64]
    mel = ragged_batch(lens, 1300)
    g = loud(SEEDS[0], mel, lens, bias)
    ref = check_generate(g, mel, lens, precision=precision)
    a = ref.cpu().numpy()
    got = g.generate(mel, lens, precision=precision, dtype=torch.int16).cpu().numpy()
    pos, neg = a == 1.0, a == -1.0
    n_pos, n_neg = np.count_nonzero(pos), np.count_nonzero(neg)
    assert min(n_pos, n_neg) > 100 and (n_pos > n_neg) == (bias > 0), (n_pos, n_neg)
    assert np.all(got[pos] == 32767) and np.all(got[neg] == -32768)
    # ties, on data that hold many: rounded half to even (32767.5 is clamped to 32767 instead)
    wide = loud(SEEDS[0], mel, lens, 0.0, spread=1.5)
    ref_w = check_generate(wide, mel, lens, precision=precision)
    n_ties = 0
    for a, gg in ((a, g), (ref_w.cpu().numpy(), wide)):
        got = gg.generate(mel, lens, precision=precision, dtype=torch.int16).cpu().numpy().astype(np.float64)
        s = 32768.0 * a.astype(np.float64)
        tie = np.isfinite(s) & (s - np.floor(s) == 0.5) & (s < 32767)
        n_ties += int(np.count_nonzero(tie))
        assert np.all(got[tie] % 2 == 0) and np.all(np.abs(got[tie] - s[tie]) == 0.5)
    assert n_ties > 0


def nan_stream(gens, S, P, precision, dtype):
    nbytes = engine.lib().mg_gen_stream_state_bytes(S, P)
    state = torch.full(((nbytes + 3) // 4,), float("nan"), device="cuda").view(torch.uint8)
    return engine.GeneratorStream(lambda: [g._ensure_packed() for g in gens], "cuda", S, P, precision, state=state, dtype=dtype)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_stream_sessions(gens, precision):
    """Utterances of several voices through reused slots with seeded pushes, END and RESET, on a NaN-filled state; float
    and int16 steps alternate on one handle.  Every step writes into a guarded, sentinel-filled buffer of its format.
    Each session's concatenated int16 output (float steps' samples converted here) is pcm16 of its voice's generate()."""
    rng = np.random.default_rng(31)
    lens = [1, 3, 7, 31, 33, 90, 2, 64, 17, 5, 129, 8]
    utts = [torch.from_numpy(synth.mel_input(1, T, 2000 + i)).cuda() for i, T in enumerate(lens)]
    uvoice = [int(v) for v in rng.integers(0, len(gens), len(lens))]
    S, P = 4, 16
    st = nan_stream(gens, S, P, precision, torch.int16)
    queue = list(range(len(lens)))
    slot, pos = [None] * S, [0] * S
    drop = [0] * S  # frames of a throw-away utterance still to push before a RESET opens the queued one
    pending = [None] * S
    out = {u: [] for u in queue}
    mel = torch.zeros((S, 80, P), device="cuda")
    formats = {torch.int16: 0, torch.float32: 0}
    step_no = 0
    while queue or any(u is not None for u in slot) or any(pending):
        frames, flags, voice = [0] * S, [0] * S, [0] * S
        for i in range(S):
            if slot[i] is None and pending[i] is None and queue:
                u = queue.pop(0)
                if u % 4 == 1:  # opened by a RESET over an unfinished utterance of another voice
                    pending[i], drop[i] = u, int(rng.integers(2, 30))
                else:
                    slot[i], pos[i] = u, 0
            if pending[i] is not None:
                if drop[i] > 0:
                    n = min(drop[i], int(rng.integers(1, P + 1)))
                    frames[i], voice[i] = n, (uvoice[pending[i]] + 1) % len(gens)
                    mel[i, :, :n] = torch.from_numpy(synth.mel_input(1, n, 9 + i)).cuda()[0]
                    drop[i] -= n
                    continue
                slot[i], pos[i], pending[i] = pending[i], 0, None
                flags[i] = RESET
            u = slot[i]
            if u is None:
                continue
            voice[i] = uvoice[u]
            n = min(int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))])), lens[u] - pos[i])
            if flags[i] & RESET:
                n = max(n, 1)
            frames[i] = n
            if n:
                mel[i, :, :n] = utts[u][0, :, pos[i]:pos[i] + n]
            pos[i] += n
            if pos[i] == lens[u] and (n == 0 or rng.random() > 0.3):
                flags[i] |= END
        dt = torch.int16 if step_no % 2 == 0 else torch.float32
        step_no += 1
        buf = (torch.full((S * st.max_out + 2 * GUARD,), SENT, dtype=torch.int16, device="cuda") if dt == torch.int16 else
               torch.full((S * st.max_out + 2 * GUARD,), float("nan"), device="cuda"))
        rows = buf[GUARD:GUARD + S * st.max_out].view(S, st.max_out)
        _, counts = st.step_packed(mel, frames, flags, audio=rows, voice=voice)
        fill = SENT if dt == torch.int16 else None
        for i, m in enumerate(counts):
            tail = rows[i, m:]
            assert bool((tail == fill).all()) if fill is not None else bool(torch.isnan(tail).all()), (i, m)
            if dt == torch.float32:
                assert not bool(torch.isnan(rows[i, :m]).any())
        edge = buf[:GUARD], buf[-GUARD:]
        for e in edge:
            assert bool((e == fill).all()) if fill is not None else bool(torch.isnan(e).all())
        formats[dt] += 1
        for i in range(S):
            u = slot[i]
            if u is None:
                continue
            piece = rows[i, :counts[i]].cpu().numpy()
            out[u].append(piece if dt == torch.int16 else pcm16_np(piece))
            if flags[i] & END:
                slot[i] = None
    st.check_status()
    assert formats[torch.int16] > 3 and formats[torch.float32] > 3
    for u, T in enumerate(lens):
        ref = gens[uvoice[u]].generate(utts[u], precision=precision)
        got = np.concatenate(out[u])
        assert got.shape == (256 * T,), (u, got.shape)
        assert np.array_equal(got, pcm16_of(ref)[0, 0]), u


def test_stream_handle_format(gens):
    """models.stream_voices(dtype=int16) / Generator.stream(dtype=int16): step returns int16 slices."""
    mel = torch.from_numpy(synth.mel_input(1, 20, 5)).cuda()
    for st in (models.stream_voices(gens, 2, 8, dtype=torch.int16), gens[1].stream(2, 8, dtype=torch.int16)):
        voice = [1, 1] if st._packed_fn is not None and isinstance(st._packed_fn(), list) else None
        pieces = []
        for lo in range(0, 20, 8):
            hi = min(20, lo + 8)
            outs = st.step([mel[0, :, lo:hi], None], end=[hi == 20, False], voice=voice)
            assert all(o.dtype == torch.int16 for o in outs)
            pieces.append(outs[0])
        st.check_status()
        got = torch.cat(pieces, dim=1).cpu().numpy()[0]
        assert np.array_equal(got, pcm16_of(gens[1].generate(mel))[0, 0])
        st.close()


@pytest.mark.parametrize("pinned", [False, True])
def test_host_engine(pinned):
    """GeneratorHost(dtype=np.int16): pinned and pageable output buffers, uniform and ragged, both precisions."""
    state = synth.generator_state(SEEDS[0])
    eng = engine.GeneratorHost(8, 64)
    try:
        eng.load_state(state)
        lens = [64, 1, 13, 40, 2, 64, 9, 33]
        mel = np.full((8, 80, 64), np.nan, np.float32)
        for i, L in enumerate(lens):
            mel[i, :, :L] = synth.mel_input(1, L, 70 + i)[0]
        for precision in ("fp32", "bf16"):
            for ragged in (False, True):
                m = mel if ragged else np.nan_to_num(mel)
                if pinned:
                    t = torch.full((8 * 256 * 64 + 2 * GUARD,), SENT, dtype=torch.int16).pin_memory()
                    whole = t.numpy()
                else:
                    whole = np.full(8 * 256 * 64 + 2 * GUARD, SENT, np.int16)
                out = whole[GUARD:-GUARD].reshape(8, 1, 256 * 64)
                if ragged:
                    ref = eng.forward_ragged(m, lens, precision=precision)
                    got = eng.forward_ragged(m, lens, out=out, precision=precision, dtype=np.int16)
                else:
                    ref = eng.forward(m, precision=precision)
                    got = eng.forward(m, out=out, precision=precision, dtype=np.int16)
                assert got is out
                assert np.all(whole[:GUARD] == SENT) and np.all(whole[-GUARD:] == SENT)
                assert np.array_equal(out, pcm16_np(ref)), (precision, ragged)
                assert np.array_equal(eng.forward(m[:3, :, :5], precision=precision, dtype=np.int16),
                                      pcm16_np(eng.forward(m[:3, :, :5], precision=precision)))
    finally:
        eng.close()


def test_two_streams_in_flight(gens):
    """Two int16 forwards on two CUDA streams at once, on one module: each equals its serial result."""
    mels = [torch.from_numpy(synth.mel_input(16, 48, 40 + k)).cuda() for k in range(2)]
    lens = [[48, 1, 30, 17] * 4, None]
    serial = [gens[0].generate(mels[k], lens[k], dtype=torch.int16) for k in range(2)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    outs = [None, None]
    for _ in range(3):
        for k in range(2):
            streams[k].wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(streams[k]):
                outs[k] = gens[0].generate(mels[k], lens[k], dtype=torch.int16)
        torch.cuda.synchronize()
        for k in range(2):
            assert torch.equal(outs[k], serial[k]), k
    for k in range(2):
        assert np.array_equal(serial[k].cpu().numpy(), pcm16_of(gens[0].generate(mels[k], lens[k])))
