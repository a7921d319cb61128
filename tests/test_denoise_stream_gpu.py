"""The streaming denoiser (csrc/mg_denoise_stream.cu through denoiser.DenoiserStream) against Denoiser.forward of each
whole utterance, bit for bit: every n_fft, three (hop, win_length) shapes, seeded push schedules with 0- and 1-sample
pushes, full pushes and END at every length class, fp32 and int16 alternating, several voices per handle, chained after
Generator.stream and models.stream_voices, and the hygiene of the state and output buffers, NaN / Inf, concurrent
handles and asynchronous steps."""
import numpy as np
import pytest
import torch

import denoise_model as dm
from kernel_model import gen, gstate  # noqa: F401  (module-scoped fixtures)
from melgan_multi_b200 import denoiser, engine, models, synth

# (hop, win_length) per n_fft: hop < n/2, hop > n/2 with a short window, and a short window with a small hop
SHAPES = lambda n: [(n // 4, n), (5 * n // 8, 3 * n // 4), (n // 8, n // 2)]


def _bias(n, V, seed):
    rng = np.random.default_rng(seed)
    rows = np.abs(np.fft.rfft(rng.standard_normal((V, n)) * 0.02 * np.hanning(n), axis=1))
    return torch.from_numpy(rows.astype(np.float32))


def _audio(L, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 22050.0
    a = sum(rng.uniform(0.05, 0.25) * np.sin(2 * np.pi * rng.uniform(60, 6000) * t + rng.uniform(0, 6.3)) for _ in range(4))
    return torch.from_numpy((a + 0.01 * rng.standard_normal(L)).astype(np.float32)).cuda()


def _lengths(n, h, w, rng, k):
    """k NOLA-clean utterance lengths: the shortest legal one, and L mod h = 0, 1 and h - 1, then random."""
    out = []
    cands = [n // 2 + 1, 3 * h * (n // h + 1), 3 * h * (n // h + 1) + 1, 4 * h * (n // h + 1) - 1]
    while len(out) < k:
        L = cands.pop(0) if cands else int(rng.integers(n // 2 + 1, 6 * n))
        if dm.nola_ok(n, h, w, L):
            out.append(L)
    return out


def _run(ds, utts, rng, P, voice=None, fmt="alternate"):
    """Streams utts (list of 1-D CUDA tensors) through ds, one slot each, on seeded schedules of 0-, 1-, random and P-sample
    pushes; returns each utterance's concatenated output as float (fmt "float"), int16 ("int16") or steps alternating."""
    S = len(utts)
    pos = [0] * S
    outs = [[] for _ in range(S)]
    done = [False] * S
    step = 0
    while not all(done):
        chunks, end = [], []
        for i, a in enumerate(utts):
            if done[i]:
                chunks.append(None)
                end.append(False)
                continue
            m = int(rng.choice([0, 1, P, int(rng.integers(0, P + 1))]))
            m = min(m, a.shape[0] - pos[i])
            chunks.append(a[pos[i]:pos[i] + m])
            pos[i] += m
            end.append(pos[i] == a.shape[0] and rng.random() < 0.7)
        pcm = fmt == "int16" or (fmt == "alternate" and step % 2 == 1)
        out = torch.empty((S, ds.max_out), dtype=torch.int16 if pcm else torch.float32, device="cuda")
        counts = [c.shape[0] if c is not None else 0 for c in chunks]
        for i, c in enumerate(chunks):
            if counts[i]:
                ds._in[i, :counts[i]].copy_(c)
        flags = [engine.STREAM_END if e else 0 for e in end]
        y, m = ds.step_packed(ds._in, counts, flags, voice=voice, out=out)
        for i in range(S):
            outs[i].append((y[i, :m[i]].clone(), pcm))
            if end[i]:
                done[i] = True
        step += 1
    return outs


def _same(a, b):
    """Bit-identical (NaN payloads and signed zeros included)."""
    if a.dtype == torch.float32:
        return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _check(outs, refs, refs16):
    for i, parts in enumerate(outs):
        off = 0
        for p, pcm in parts:
            k = p.shape[0]
            assert _same(p, (refs16 if pcm else refs)[i][off:off + k]), (i, off, pcm)
            off += k
        assert off == refs[i].shape[0]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [128, 256, 512, 1024, 2048])
def test_stream_is_bit_identical_to_forward(n):
    rng = np.random.default_rng(n)
    for shape, (h, w) in enumerate(SHAPES(n)):
        dn = denoiser.Denoiser.from_bias(_bias(n, 1, n + shape), n, n / (h + 0.5), w).cuda()  # hop = int(n / n_overlap)
        assert dn.hop == h
        lens = _lengths(n, h, w, rng, 12)
        utts = [_audio(L, 100 * n + j) for j, L in enumerate(lens)]
        P = int(rng.choice([h, 3 * n]))
        ds = dn.stream(len(utts), P, strength=0.3)
        refs = [dn(a[None], strength=0.3)[0] for a in utts]
        refs16 = [dn(a[None], strength=0.3, dtype=torch.int16)[0] for a in utts]
        _check(_run(ds, utts, rng, P), refs, refs16)
        ds.close()


@pytest.mark.gpu
def test_voices_and_slot_reuse():
    n, h, w = 1024, 256, 1024
    bias = _bias(n, 3, 5)
    dn = denoiser.Denoiser.from_bias(bias, n, 4, w).cuda()
    rng = np.random.default_rng(3)
    lens = [700, 2000, 513, 4096, 3000, 1537]
    utts = [_audio(L, j) for j, L in enumerate(lens)]
    voice = [2, 0, 1, 1, 2, 0]
    ds = dn.stream(6, 600)
    refs = [dn(a[None], voice=[v])[0] for a, v in zip(utts, voice)]
    refs16 = [dn(a[None], voice=[v], dtype=torch.int16)[0] for a, v in zip(utts, voice)]
    _check(_run(ds, utts, rng, 600, voice=voice), refs, refs16)
    # every slot reused in another voice after END
    voice2 = [(v + 1) % 3 for v in voice]
    utts2 = [_audio(L + 17, 50 + j) for j, L in enumerate(lens)]
    refs = [dn(a[None], voice=[v])[0] for a, v in zip(utts2, voice2)]
    refs16 = [dn(a[None], voice=[v], dtype=torch.int16)[0] for a, v in zip(utts2, voice2)]
    _check(_run(ds, utts2, rng, 600, voice=voice2), refs, refs16)
    # RESET mid-utterance, then a new utterance in another voice on the same slot
    a = _audio(3000, 77)
    ds.step([a[:600]], voice=[0])
    with pytest.raises(engine.EngineError, match="bound to voice 0"):
        ds.step([a[600:700]], voice=[1])
    y1 = ds.step([a[:600]], reset=[True], voice=[1])
    y2 = ds.step([a[600:1200]], voice=[1])
    y3 = ds.step([a[1200:1800]], end=[True], voice=[1])
    assert torch.equal(torch.cat([y1[0][0], y2[0][0], y3[0][0]]), dn(a[None, :1800], voice=[1])[0])
    # one voice equals the single-voice handle
    one = denoiser.Denoiser.from_bias(bias[1:2].clone(), n, 4, w).cuda()
    s1 = one.stream(1, 600)
    z = [s1.step([a[k:k + 600]], end=[k + 600 >= 3000])[0][0] for k in range(0, 3000, 600)]
    assert torch.equal(torch.cat(z), one(a[None])[0]) and torch.equal(torch.cat(z), dn(a[None], voice=[1])[0])


def _gen2(seed):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
    return g.cuda().eval()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_chained_after_the_generator_stream(gen, precision):  # noqa: F811
    T = [40, 7, 33, 12]
    mels = [torch.from_numpy(synth.mel_input(1, t, 11 + i)).cuda() for i, t in enumerate(T)]
    dn = denoiser.Denoiser(gen)
    P = 8
    gs = gen.stream(4, P, precision=precision)
    ds = dn.stream(4, gs.max_out)
    got = [[] for _ in T]
    pos = [0] * 4
    mel = torch.zeros(4, 80, P, device="cuda")
    step = 0
    with torch.no_grad():
        while any(p < t for p, t in zip(pos, T)):
            frames, flags = [], []
            for i, t in enumerate(T):
                k = min(P if step % 3 else 1, t - pos[i]) if pos[i] < t else 0
                if k:
                    mel[i, :, :k] = mels[i][0, :, pos[i]:pos[i] + k]
                pos[i] += k
                frames.append(k)
                flags.append(engine.STREAM_END if k and pos[i] == t else 0)
            a, c = gs.step_packed(mel, frames, flags)
            out = torch.empty(4, ds.max_out, dtype=torch.int16 if step % 2 else torch.float32, device="cuda")
            y, m = ds.step_packed(a, c, flags, out=out)
            for i in range(4):
                got[i].append(y[i, :m[i]].clone())
            step += 1
        for i, t in enumerate(T):
            audio = gen.generate(mels[i], precision=precision)
            ref = dn(audio, lengths=[256 * t])[0, 0]
            ref16 = dn(audio, lengths=[256 * t], dtype=torch.int16)[0, 0]
            off = 0
            for p in got[i]:
                assert _same(p, (ref16 if p.dtype == torch.int16 else ref)[off:off + p.shape[0]]), (i, off)
                off += p.shape[0]
            assert off == 256 * t


@pytest.mark.gpu
def test_chained_after_stream_voices(gen):  # noqa: F811
    g2 = _gen2(99)
    dn = denoiser.Denoiser([gen, g2])
    T = [20, 9, 31]
    voice = [1, 0, 1]
    mels = [torch.from_numpy(synth.mel_input(1, t, 31 + i)).cuda() for i, t in enumerate(T)]
    P = 4
    gs = models.stream_voices([gen, g2], 3, P)
    ds = dn.stream(3, gs.max_out)
    outs = [[] for _ in T]
    pos = [0] * 3
    mel = torch.zeros(3, 80, P, device="cuda")
    with torch.no_grad():
        while any(p < t for p, t in zip(pos, T)):
            frames, flags = [], []
            for i, t in enumerate(T):
                k = min(P, t - pos[i]) if pos[i] < t else 0
                if k:
                    mel[i, :, :k] = mels[i][0, :, pos[i]:pos[i] + k]
                pos[i] += k
                frames.append(k)
                flags.append(engine.STREAM_END if k and pos[i] == t else 0)
            a, c = gs.step_packed(mel, frames, flags, voice=voice)
            y, m = ds.step_packed(a, c, flags, voice=voice)
            for i in range(3):
                outs[i].append(y[i, :m[i]].clone())
        for i, t in enumerate(T):
            g = [gen, g2][voice[i]]
            ref = dn(g.generate(mels[i]), lengths=[256 * t], voice=[voice[i]])[0, 0]
            assert _same(torch.cat(outs[i]), ref), i


@pytest.mark.gpu
def test_poisoned_state_guarded_output_and_256_sessions():
    n, h, w = 512, 128, 512
    dn = denoiser.Denoiser.from_bias(_bias(n, 2, 9), n, 4, w).cuda()
    S, P = 256, 300
    nbytes = denoiser._lib().mg_denoise_stream_state_bytes(n, h, S, P)
    state = torch.full((nbytes // 4 + 64,), float("nan"), device="cuda").view(torch.uint8)
    ds = dn.stream(S, P, state=state)
    rng = np.random.default_rng(1)
    lens = [int(rng.integers(n // 2 + 1, 3000)) for _ in range(S)]
    lens = [L if dm.nola_ok(n, h, w, L) else L + 1 for L in lens]
    utts = [_audio(L, 1000 + j) for j, L in enumerate(lens)]
    voice = [j % 2 for j in range(S)]
    pos = [0] * S
    got = [[] for _ in range(S)]
    guard = 64
    while any(p < L for p, L in zip(pos, lens)):
        counts = [min(int(rng.integers(0, P + 1)), L - p) for p, L in zip(pos, lens)]
        flags = []
        for i in range(S):
            if counts[i]:
                ds._in[i, :counts[i]].copy_(utts[i][pos[i]:pos[i] + counts[i]])
            pos[i] += counts[i]
            flags.append(engine.STREAM_END if counts[i] and pos[i] == lens[i] else 0)
        buf = torch.full((S * ds.max_out + guard,), float("nan"), device="cuda")
        out = buf[:S * ds.max_out].view(S, ds.max_out)
        y, m = ds.step_packed(ds._in, counts, flags, voice=voice, out=out)
        assert bool(torch.isnan(buf[S * ds.max_out:]).all())
        for i in range(S):
            assert bool(torch.isnan(out[i, m[i]:]).all())  # nothing past the count is written
            got[i].append(out[i, :m[i]].clone())
    for i in range(S):
        assert torch.equal(torch.cat(got[i]), dn(utts[i][None], voice=[voice[i]])[0]), i


@pytest.mark.gpu
def test_nonfinite_samples_stay_in_their_session():
    n, h, w = 1024, 256, 1024
    dn = denoiser.Denoiser.from_bias(_bias(n, 1, 4), n, 4, w).cuda()
    utts = [_audio(5000, j) for j in range(4)]
    utts[1][2500] = float("nan")
    utts[2][777] = float("inf")
    ds = dn.stream(4, 700)
    rng = np.random.default_rng(8)
    refs = [dn(a[None])[0] for a in utts]
    refs16 = [dn(a[None], dtype=torch.int16)[0] for a in utts]
    outs = _run(ds, utts, rng, 700)
    _check(outs, refs, refs16)  # bit for bit, NaN and Inf where forward has them
    assert bool(torch.isnan(refs[1]).any()) and not bool(torch.isnan(refs[0]).any()) and not bool(torch.isnan(refs[3]).any())


@pytest.mark.gpu
def test_two_handles_on_two_streams_equal_serial_stepping():
    n = 1024
    dn = denoiser.Denoiser.from_bias(_bias(n, 1, 6), n, 4, n).cuda()
    utts = [_audio(6000 + 13 * j, 200 + j) for j in range(8)]
    refs = [dn(a[None])[0] for a in utts]
    res = {}
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    handles = [dn.stream(4, 500), dn.stream(4, 500)]
    torch.cuda.synchronize()
    for k in range(2):
        res[k] = [[] for _ in range(4)]
    for off in range(0, 6200, 500):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                chunks = [u[off:off + 500] if off < u.shape[0] else None for u in utts[4 * k:4 * k + 4]]
                end = [c is not None and off + 500 >= u.shape[0] for c, u in zip(chunks, utts[4 * k:4 * k + 4])]
                ys = handles[k].step(chunks, end=end)
                for i in range(4):
                    res[k][i].append(ys[i])
    torch.cuda.synchronize()
    for k in range(2):
        for i in range(4):
            assert torch.equal(torch.cat([y[0] for y in res[k][i]]), refs[4 * k + i])


@pytest.mark.gpu
def test_step_is_asynchronous():
    n = 1024
    dn = denoiser.Denoiser.from_bias(_bias(n, 1, 2), n, 4, n).cuda()
    ds = dn.stream(2, 2048)
    a = [_audio(3000, 1), _audio(3000, 2)]
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    y1 = ds.step([x[:2048] for x in a])
    y2 = ds.step([x[2048:] for x in a], end=[True, True])
    ev = torch.cuda.Event()
    ev.record()
    e = (2048 - 512) // 256 * 256 + 256 - 512
    assert [y.shape[1] for y in y1] == [e, e] and [y.shape[1] for y in y2] == [3000 - e] * 2
    assert not ev.query()
    torch.cuda.synchronize()
    for i in range(2):
        assert torch.equal(torch.cat([y1[i][0], y2[i][0]]), dn(a[i][None])[0])


@pytest.mark.gpu
def test_moved_denoiser_is_refused():
    dn = denoiser.Denoiser.from_bias(_bias(1024, 1, 2), 1024, 4, 1024).cuda()
    ds = dn.stream(1, 100)
    dn.cpu()
    with pytest.raises(engine.EngineError, match="moved"):
        ds.step([torch.zeros(10, device="cuda")])
