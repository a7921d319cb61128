"""The denoiser (csrc/mg_denoise.cu through denoiser.Denoiser) against its float64 definition (denoise_model.denoise64,
torch.stft / torch.istft on the CPU) at every n_fft, hop and window shape, bit-exactness across ragged, uniform and
voiced batches, the bias spectrum, int16 output, NaN / Inf, poisoned buffers, determinism, streams, CUDA graphs, and
through the generator.

Error model.  Per frame f, E_f = TAU_F ||w . frame_f||_2 is the error of each bin of the fp32 forward FFT (the per-bin
RMS model of test_stft_loss_gpu.py).  The bin rule X -> max(|X| - c, 0) X / |X| is non-expansive (soft thresholding),
so each output bin is off by at most dY_k = E_f + 4 u |X_k|.  The inverse real transform takes a bin error to at most
(2 / n) sum_k dY_k per frame sample, its own rounding adds 2 TAU_F ||Y_f||_2 / (n / 2) and the scale and window 4 u
|y|; so a frame sample is off by at most |w_n| D_f + u |w_n y_n|.  The overlap-add sums c = n / hop + 3 such terms and
the envelope as many, so per output sample
    bound_i = (sum_f |w| D_f + c u sum_f |w y_f|) / env_i + c u |out_i|.
The module prints the worst ratio |got - ref| / bound seen for each case, and checks that the bound rejects each
float64 mutant of the definition (denoise_model.DENOISE_MUTANTS) by at least kernel_model.MUTANT_X.
"""
import threading

import numpy as np
import pytest
import torch

import denoise_model as dm
import kernel_model as km
from kernel_model import gen, gstate  # noqa: F401  (module-scoped fixtures)
from melgan_multi_b200 import denoiser, engine, models, synth

U = 2.0 ** -24
TAU_F = 2.0 ** -17
WORST = {}
REJECT = {}  # each mutant's smallest max(|mutant - ref| / bound) over the cases that try it


def _note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst ratios to the bound: " + ", ".join("%s %.3g" % kv for kv in sorted(WORST.items())))
    print("mutants rejected by at least: " + ", ".join("%s %.3g" % kv for kv in sorted(REJECT.items())))


def _signals(B, L, seed):
    """Smooth seeded audio: a few partials with random phase plus a little noise, in [-1, 1]."""
    rng = np.random.default_rng(seed)
    t = np.arange(L) / 22050.0
    out = np.zeros((B, L))
    for b in range(B):
        for _ in range(4):
            out[b] += rng.uniform(0.05, 0.25) * np.sin(2 * np.pi * rng.uniform(60, 6000) * t + rng.uniform(0, 2 * np.pi))
        out[b] += 0.01 * rng.standard_normal(L)
    return out.astype(np.float32)


def _bias(n, V, seed, scale=1.0):
    """V bias rows of the size of a noise floor's |X|: |rfft| of windowed noise, smoothed, times scale."""
    rng = np.random.default_rng(seed)
    rows = np.abs(np.fft.rfft(rng.standard_normal((V, n)) * 0.02 * np.hanning(n), axis=1)) * scale
    return torch.from_numpy(rows.astype(np.float32))


def _poison_tails(x, lengths, seed):
    """x with loud different audio past each item's length (a kernel reading it shows)."""
    x = x.copy()
    rng = np.random.default_rng(seed)
    for i, L in enumerate(lengths):
        x[i, L:] = rng.uniform(-1, 1, x.shape[1] - L)
    return x


def bound(n, h, parts, out64, Lmax):
    c = n // h + 3
    res = torch.zeros(len(parts), Lmax, dtype=torch.float64)
    for i, p in enumerate(parts):
        win, T, L = p["win"].abs(), p["T"], p["L"]
        E = TAU_F * p["xw"].norm(dim=-1, keepdim=True)
        dY = E + 4 * U * p["X"].abs()
        ymax = p["y"].abs().amax(-1, keepdim=True)
        D = (2.0 / n) * dY.sum(-1, keepdim=True) + 2 * TAU_F * p["Y"].abs().norm(dim=-1, keepdim=True) / (n // 2) + 4 * U * ymax
        per = win * D + c * U * p["yw"].abs()  # [T, n]
        acc = torch.zeros(n + h * (T - 1), dtype=torch.float64)
        for t in range(T):
            acc[t * h:t * h + n] += per[t]
        seg = acc[n // 2:n // 2 + L]
        env = p["env"][:seg.shape[0]]
        res[i, :seg.shape[0]] = seg / env + c * U * out64[i, :seg.shape[0]].abs()
    return res


def _run(d, x, strength, lengths=None, voice=None, dtype=torch.float32):
    with torch.no_grad():
        return d(torch.from_numpy(x).cuda(), strength, lengths=lengths, voice=voice, dtype=dtype)


def check(n, h, w, x, bias, strength, lengths=None, voice=None, key=None, mutants=False):
    d = denoiser.Denoiser.from_bias(bias, n, n / (h + 0.5), w).cuda()  # (hop = int(n / n_overlap) = h exactly)
    assert d.hop == h
    got = _run(d, x, strength, lengths, voice).cpu().double()
    ref, parts = dm.denoise64_parts(x, n, h, w, bias, strength, lengths, voice)
    defn = dm.denoise64_batch(x, n, h, w, bias, strength, lengths, voice)
    assert (ref - defn).abs().max() <= 1e-12 * max(1.0, float(defn.abs().max()))
    b = bound(n, h, parts, ref, x.shape[1])
    err = (got - ref).abs()
    bad = err > b
    assert not bad.any(), (key, torch.nonzero(bad)[:5].tolist(), err[bad][:5].tolist(), b[bad][:5].tolist())
    _note(key or "n=%d h=%d w=%d" % (n, h, w), float((err / b.clamp_min(1e-300)).max()))
    if lengths is not None:
        for i, L in enumerate(lengths):
            assert bool((got[i, L:] == 0).all())
    if mutants:
        for m in dm.DENOISE_MUTANTS:
            mut, _ = dm.denoise64_parts(x, n, h, w, bias, strength, lengths, voice, mutant=m)
            r = float(((mut - ref).abs() / b.clamp_min(1e-300)).max())
            assert r >= km.MUTANT_X, (m, r)
            REJECT[m] = min(REJECT.get(m, float("inf")), r)
    return got


def _cases():
    out = []
    for n in (128, 256, 512, 1024, 2048):
        w_odd = n - n // 4 + 1
        for w in (n, w_odd):
            for h in (n // 4, n // 2, n // 8 + 1 if (n // 8) % 2 == 0 else n // 8):
                out.append((n, h, w))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", _cases())
def test_against_float64(n, h, w):
    L = 5 * n + 37
    lens = [L, L - n // 2 - 5, n // 2 + 1 + (n // 8)]
    x = _poison_tails(_signals(3, L, n + h + w), lens, 7)
    check(n, h, w, x, _bias(n, 2, n), 0.5, lens, [1, 0, 1], mutants=(n, h, w) in ((512, 128, 512), (1024, 129, 769)))


@pytest.mark.gpu
def test_mutants_at_the_default_analysis():
    L = 8192 + 100
    lens = [L, 6000]
    x = _poison_tails(_signals(2, L, 3), lens, 4)
    check(1024, 256, 1024, x, _bias(1024, 2, 5), 1.0, lens, [1, 0], key="default mutants", mutants=True)


@pytest.mark.gpu
def test_special_strengths():
    n, h, w = 1024, 256, 1024
    x = _signals(2, 8192, 11)
    bias = _bias(n, 1, 12)
    got = check(n, h, w, x, bias, 0.0, key="strength 0")
    # strength 0 reproduces the input within the same bound (the definition at strength 0 is the identity to 1e-12)
    ref = torch.from_numpy(x).double()
    assert float((got - ref).abs().max()) < 1e-4
    d = denoiser.Denoiser.from_bias(torch.full((1, n // 2 + 1), 1.0), n).cuda()
    big = _run(d, x, 1e6)
    assert bool((big == 0).all())


@pytest.mark.gpu
def test_ragged_items_equal_their_own_calls():
    n, h, w = 1024, 256, 1024
    lens = [8192, 5000, 513, 8191, 2560, 8192]
    x = _poison_tails(_signals(6, 8192, 21), lens, 22)
    d = denoiser.Denoiser.from_bias(_bias(n, 1, 23), n).cuda()
    for dt in (torch.float32, torch.int16):
        got = _run(d, x, 0.7, lens, dtype=dt)
        for i, L in enumerate(lens):
            own = _run(d, np.ascontiguousarray(x[i:i + 1, :L]), 0.7, dtype=dt)
            assert torch.equal(got[i, :L], own[0]), (i, dt)
            assert bool((got[i, L:] == 0).all())
    same = _run(d, x, 0.7, [8192] * 6)
    assert torch.equal(same, _run(d, x, 0.7))
    assert torch.equal(_run(d, x[:, None, :].copy(), 0.7)[:, 0], same)  # [B, 1, L] in, same shape out


@pytest.mark.gpu
def test_voices_equal_single_voice_calls():
    n, h, w = 512, 128, 512
    V = 4
    bias = _bias(n, V, 31, scale=2.0)
    L = 6000
    x = _signals(8, L, 32)
    d = denoiser.Denoiser.from_bias(bias, n, 4, w).cuda()
    singles = [denoiser.Denoiser.from_bias(bias[v:v + 1].clone(), n, 4, w).cuda() for v in range(V)]
    for voice in ([0, 0, 1, 1, 2, 2, 3, 3], [0, 1, 2, 3, 0, 1, 2, 3], [3, 1, 0, 2, 1, 0, 3, 2]):
        lens = [L - 97 * i for i in range(8)]
        got = _run(d, x, 0.8, lens, voice)
        for i, v in enumerate(voice):
            own = _run(singles[v], np.ascontiguousarray(x[i:i + 1, :lens[i]]), 0.8)
            assert torch.equal(got[i, :lens[i]], own[0]), (voice, i)


def _gen(seed):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
    return g.cuda().eval()


@pytest.mark.gpu
def test_bias_is_frame_zero_of_the_generators_own_audio(gen):  # noqa: F811
    n, w = 1024, 1024
    d = denoiser.Denoiser(gen)
    with torch.no_grad():
        a = gen.generate(torch.zeros(1, 80, denoiser.BIAS_MEL_FRAMES, device="cuda")).reshape(1, -1).cpu().double()
    S = torch.stft(a[0], n, 256, w, torch.hann_window(w, dtype=torch.float64), center=True, pad_mode="reflect",
                   return_complex=True)[:, 0].abs()
    xw = torch.nn.functional.pad(a[None], (n // 2, n // 2), mode="reflect")[0, 0, :n] * dm.hann64(w, n)
    b = TAU_F * xw.norm() + 4 * U * S
    err = (d.bias_spec[0].cpu().double() - S).abs()
    assert bool((err <= b).all()), float((err / b).max())
    _note("bias", float((err / b).max()))
    g2 = _gen(99)
    both = denoiser.Denoiser([gen, g2])
    assert both.bias_spec.shape == (2, n // 2 + 1)
    assert torch.equal(both.bias_spec[0], d.bias_spec[0])
    assert torch.equal(both.bias_spec[1], denoiser.Denoiser(g2).bias_spec[0])
    assert not torch.equal(both.bias_spec[0], both.bias_spec[1])
    nrm = denoiser.Denoiser(gen, mode="normal")
    assert nrm.bias_spec.shape == (1, n // 2 + 1) and not torch.equal(nrm.bias_spec, d.bias_spec)
    # refresh() follows the weights
    old = d.bias_spec.clone()
    with torch.no_grad():
        gen.conv_post.bias.add_(0.01)
    try:
        d.refresh()
        assert not torch.equal(old, d.bias_spec)
    finally:
        with torch.no_grad():
            gen.conv_post.bias.sub_(0.01)
        d.refresh()
    assert torch.equal(old, d.bias_spec)


@pytest.mark.gpu
def test_int16_is_pcm16_of_the_float_output():
    n = 1024
    lens = [8192, 3001, 700]
    x = _signals(3, 8192, 41) * 4  # loud enough to saturate
    x[0, 100:140] = np.nan
    d = denoiser.Denoiser.from_bias(_bias(n, 2, 42), n).cuda()
    for kw in (dict(), dict(lengths=lens), dict(lengths=lens, voice=[1, 0, 1])):
        f = _run(d, x, 0.3, **kw)
        i16 = _run(d, x, 0.3, dtype=torch.int16, **kw)
        ref = torch.clamp(torch.round(f * 32768.0), -32768, 32767)
        ref = torch.where(torch.isnan(f), torch.zeros_like(ref), ref).to(torch.int16)
        assert i16.dtype == torch.int16 and torch.equal(i16, ref), kw
        assert bool((i16 == 32767).any()) and bool((i16 == -32768).any()) and bool(torch.isnan(f).any())


@pytest.mark.gpu
def test_nan_and_inf_reach_exactly_what_float64_reaches():
    n, h, w = 512, 128, 512
    L = 4000
    x = _signals(4, L, 51)
    x[1, 1000] = np.nan
    x[2, 2000] = np.inf
    x[3, 3] = -np.inf
    clean = x.copy()
    clean[1:] = _signals(3, L, 52)
    bias = _bias(n, 1, 53)
    d = denoiser.Denoiser.from_bias(bias, n, 4, w).cuda()
    got = _run(d, x, 0.5).cpu()
    ref = dm.denoise64_batch(x, n, h, w, bias, 0.5)
    assert torch.equal(torch.isfinite(got), torch.isfinite(ref))
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    assert bool(torch.isfinite(got[0]).all())
    other = _run(d, clean, 0.5).cpu()
    assert torch.equal(got[0], other[0])  # the clean item does not change by a bit


@pytest.mark.gpu
def test_buffer_hygiene():
    n, h, w = 1024, 256, 1024
    lens = [8192, 4000, 1000]
    B, L = 3, 8192
    x = torch.from_numpy(_signals(B, L, 61)).cuda()
    bias = _bias(n, 2, 62).cuda()
    d = denoiser.Denoiser.from_bias(bias, n).cuda()
    ref = _run(d, x.cpu().numpy(), 0.5, lens, [1, 0, 1])
    L_ = denoiser._lib()
    lens_c = engine._host_ints(lens, B, "lengths", 513, L + 1, "")
    voice_c = engine._host_ints([1, 0, 1], B, "voice", 0, 2, "")
    wsb = denoiser.workspace_bytes(n, h, B, L, lens)
    tabs = d._an.tables(x.device)
    for pcm in (False, True):
        out = km.nan_buffer(B * L // (2 if pcm else 1))
        ws = km.nan_buffer(wsb // 4)
        call = L_.mg_denoise_forward_pcm16 if pcm else L_.mg_denoise_forward
        engine.check(call(tabs[0], n, h, w, x.data_ptr(), B, L, lens_c, bias.data_ptr(), 2, voice_c, 0.5, out.data_ptr(),
                          ws.data_ptr(), wsb, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        nfl = B * L // (2 if pcm else 1)
        assert km.guard_ok(out, nfl) and km.guard_ok(ws, wsb // 4)
        got = out[:nfl].view(torch.int16 if pcm else torch.float32).view(B, L)
        want = _run(d, x.cpu().numpy(), 0.5, lens, [1, 0, 1], dtype=torch.int16) if pcm else ref
        assert torch.equal(got, want), pcm


@pytest.mark.gpu
def test_repeat_streams_and_graphs():
    n = 1024
    lens = [8192, 5000, 3000, 700]
    x = torch.from_numpy(_signals(4, 8192, 71)).cuda()
    d = denoiser.Denoiser.from_bias(_bias(n, 2, 72), n).cuda()
    with torch.no_grad():
        first = d(x, 0.4, lens, [0, 1, 1, 0])
        # repeated calls are bit-identical and enqueue without a host synchronisation
        torch.cuda.set_sync_debug_mode("error")
        try:
            outs = [d(x, 0.4, lens, [0, 1, 1, 0]) for _ in range(5)]
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert all(torch.equal(o, first) for o in outs)
        # two streams from two threads
        res = [None, None]
        inputs = [x, x.flip(0).contiguous()]
        serial = [d(inputs[0], 0.4, lens, [0, 1, 1, 0]), d(inputs[1], 0.4, lens[::-1], [1, 0, 0, 1])]

        def worker(k):
            s = torch.cuda.Stream()
            with torch.cuda.stream(s), torch.no_grad():
                for _ in range(3):
                    res[k] = d(inputs[k], 0.4, lens if k == 0 else lens[::-1], [0, 1, 1, 0] if k == 0 else [1, 0, 0, 1])
            s.synchronize()
        ts = [threading.Thread(target=worker, args=(k,)) for k in (0, 1)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert torch.equal(res[0], serial[0]) and torch.equal(res[1], serial[1])
        # CUDA graph capture and replay after .to(device)
        d2 = denoiser.Denoiser.from_bias(_bias(n, 2, 72), n).to("cuda")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            d2(x, 0.4, lens, [0, 1, 1, 0])  # warm the allocator on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            y = d2(x, 0.4, lens, [0, 1, 1, 0])
        x.mul_(0.5)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, d(x, 0.4, lens, [0, 1, 1, 0]))
        # a first call inside a capture is refused: the tables' upload cannot be captured
        d3 = denoiser.Denoiser.from_bias(_bias(n, 2, 72).cuda(), n)
        g2 = torch.cuda.CUDAGraph()
        with pytest.raises(engine.EngineError, match="CUDA graph capture forbids the copy"):
            with torch.cuda.graph(g2):
                d3(x, 0.4)


@pytest.mark.gpu
@pytest.mark.parametrize("ragged", [False, True])
def test_end_to_end_after_generate(gen, ragged):  # noqa: F811
    B, T = (64, 32) if not ragged else (6, 40)
    lens = None if not ragged else [40, 7, 33, 12, 40, 3]
    mel = torch.from_numpy(synth.mel_input(B, T, 81)).cuda()
    d = denoiser.Denoiser(gen)
    with torch.no_grad():
        audio = gen.generate(mel, lens)
        samples = None if lens is None else [256 * v for v in lens]
        got16 = d(audio, lengths=samples, dtype=torch.int16)
        got = d(audio, lengths=samples)
    assert got16.shape == audio.shape and got16.dtype == torch.int16
    a = audio[:, 0].cpu().numpy()
    ref, parts = dm.denoise64_parts(a, 1024, 256, 1024, d.bias_spec.cpu(), 0.1, samples)
    b = bound(1024, 256, parts, ref, a.shape[1])
    err = (got[:, 0].cpu().double() - ref).abs()
    assert bool((err <= b).all()), float((err / b).max())
    _note("generate %s" % ("ragged" if ragged else "config-2"), float((err / b.clamp_min(1e-300)).max()))
    pcm = torch.clamp(torch.round(got * 32768.0), -32768, 32767).to(torch.int16)
    assert torch.equal(got16, pcm)
