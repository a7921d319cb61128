"""What the kernels do with a value that is not finite: a NaN or +-Inf mel frame from an fp16 acoustic model, a generator
that diverged in training, a corrupt voice checkpoint.  Every case runs two calls on the same seeded inputs, a clean one
and a poisoned one with NaN, +Inf or -Inf at chosen positions, and requires:

1. containment: every other item, session, voice, stream slot or loss row of the poisoned call is bit for bit the clean
   call's, and so is every output of the poisoned item outside its allowed footprint;
2. no swallowing: every output the float64 reference makes NaN is NaN in the kernel (0 in int16 audio: pcm16 of NaN);
3. footprint: the allowed footprint is the float64 reference's own non-finite set, found by propagating the poison (as
   NaN) through the restatements the suite already has: kernel_model.forward64 for the generator, float64 F.conv1d and
   the AvgPool chain for the discriminators, a numpy statement with np.clip semantics for the mel front end.  Where a
   kernel's operand window is wider than the reference's taps, the footprint grows by exactly that reach, taken from
   the launch geometry of kernel_model (disc_group_tc_kernel: PANELS 16-byte units of 8 input positions per output
   pair; disc_group4_tc_kernel: PANELS4 units per lane of LANE4 outputs), never across an item border.  The growth each
   kernel shows is printed.  A +-Inf operand is split as hi = bf16(x), lo = x - hi = NaN, so inside the footprint a
   kernel may give NaN where the reference gives +-Inf (or +-1 after tanh); nowhere else.

The mel forward used to clamp with fmaxf(s, 1e-5f), which returns 1e-5 for a NaN band sum: log(1e-5) = -11.51 where
np.clip (and torch.clamp) give NaN, so a NaN or Inf in generated audio passed through a mel-L1 loss as silence with zero
gradient.  It now clamps with s < 1e-5f ? 1e-5f : s.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: the file runs in about 35 s; growth beyond float64's
footprint, in outputs, is 2 for grouped_convs.0-2, 6 for grouped_convs.3 and 0 for conv_pre, conv_post1, conv_post2 and
every generator kernel.

Mutants (each value-only: every finite output is unchanged) and what this file did with each on that card:
  - mel_kernel clamping with fmaxf again: test_mel_forward fails for NaN, +Inf and -Inf (no swallowing: -11.51 where
    the reference is NaN);
  - disc_group_tc_kernel loading an item's last virtual-row halo unit from its neighbour's first positions (in bounds,
    multiplied by structural zero slots only): test_msd_forward fails in 6 cases, short and long (long items share CTAs
    at the deeper layers), by containment;
  - the stream's window assembly adding 0 x (the slot's stored tail) to every window position, so an old utterance's
    tail reaches the slot's next one after END or RESET: test_stream_slot_reuse fails in all 4 cases (containment);
  - loss_row giving a row's last CTA to the next row: test_loss_rows fails for all three loss functions."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from melgan_multi_b200 import engine, meldataset, models, optim, synth
from oracle import mel_oracle as mo

NAN, INF = float("nan"), float("inf")
POISONS = {"nan": NAN, "+inf": INF, "-inf": -INF}
NFFT, HOP, PAD, CLIP = 1024, 256, 384, 1e-5
WIN64 = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(NFFT) / NFFT)
DLAYERS = synth.DISCRIMINATOR_LAYERS
# kernel_model's disc launch geometry, restated here so that the CPU part needs no library
from kernel_model import LANE4, PANELS, PANELS4, UNITS, UNITS4, cdiv, fold64, group4_plan, group_tc_plan  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------
# references and footprints (no device)
# ------------------------------------------------------------------------------------------------------------------
def mel64(y, fb):
    """The reference's log-mel of float64 y [B, L] in numpy: log(np.clip(fb @ |rfft(window * frame)|, 1e-5, None))."""
    T = y.shape[-1] // HOP
    yp = np.pad(np.asarray(y, np.float64), ((0, 0), (PAD, PAD)))
    idx = HOP * np.arange(T)[:, None] + np.arange(NFFT)[None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        mag = np.abs(np.fft.rfft(yp[:, idx] * WIN64, axis=-1))          # [B, T, 513]
        return np.log(np.clip(np.einsum("mk,btk->bmt", fb, mag), CLIP, None))


def same_bits(a, b):
    """Element-wise: equal bits, or both NaN (a NaN's payload is not part of any contract here)."""
    if a.dtype == torch.int16:
        return a == b
    ai, bi = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return (ai == bi) | (torch.isnan(a) & torch.isnan(b))


def window_mask(bad, lo, hi, stride=1, group=1, n_out=None):
    """[..., n_out] bool: output t (grouped by `group` consecutive outputs, g = t // group) whose operand window
    [stride * group * g + lo, stride * group * g + hi] of input positions holds a True of bad [..., n_in].  Positions
    outside [0, n_in) are zero padding (never bad): the window never leaves the item."""
    n_in = bad.shape[-1]
    c = torch.cumsum(torch.nn.functional.pad(bad.to(torch.int64), (1, 0)), dim=-1)   # c[i] = bad count in [0, i)
    g = torch.arange(n_out, device=bad.device) // group
    a = (stride * group * g + lo).clamp(0, n_in)
    b = (stride * group * g + hi + 1).clamp(0, n_in)
    return (c[..., b] - c[..., a]) > 0


def disc_window(l, Lout):
    """(lo, hi, group) of the input window each output of disc layer l reads in the kernel: the reference's taps for
    conv_pre, conv_post1, conv_post2 (no structural slots); grouped_convs.0-2 read PANELS units of 8 positions per output
    pair from 4 (t0 - (PANELS - 1)); grouped_convs.3 reads PANELS4 units of 8 positions per lane of LANE4 outputs from
    LANE4 kb - 20.  Reference windows are [stride t - pad, stride t - pad + k - 1]."""
    _n, _ci, _co, k, s, _g, p = DLAYERS[l]
    if 1 <= l <= 3:
        return -4 * (PANELS - 1), -4 * (PANELS - 1) + 8 * PANELS - 1, 2
    if l == 4:
        return -p, -p + 8 * PANELS4 - 1, LANE4
    return -p, -p + k - 1, 1


def test_structural_windows_cover_the_taps():
    """Each kernel window contains the reference's taps of every output it serves, and grows it by the reach printed."""
    for l, (n, _ci, _co, k, s, _g, p) in enumerate(DLAYERS):
        lo, hi, grp = disc_window(l, 64)
        for t in range(64):
            base = s * grp * (t // grp)
            assert base + lo <= s * t - p and s * t - p + k - 1 <= base + hi, (n, t)
        print("%s: kernel window [%d, %d] per %d outputs, taps [-%d, %d]" % (n, lo, hi, grp, p, k - 1 - p))
    assert group_tc_plan(20)[1] > 1 and group_tc_plan(400)[1] == 1 and UNITS == 128 + PANELS - 1 and UNITS4 == 128 + PANELS4 - 1


def test_mel64_propagates_nan_like_np_clip():
    """The numpy statement: a NaN sample makes the frames that read it NaN; silence is log(1e-5), not NaN."""
    fb = mo.mel_filterbank64(22050, NFFT, 80, 55.0, 9000.0, 1)
    y = np.zeros((1, 4 * HOP))
    y[0, 600] = NAN
    m = mel64(y, fb)
    frames = {t for t in range(4) if HOP * t - PAD <= 600 < HOP * t - PAD + NFFT}
    assert set(np.nonzero(np.isnan(m[0]).all(axis=0))[0]) == frames and not np.isnan(m[0][:, [t for t in range(4) if t not in frames]]).any()
    assert np.all(mel64(np.zeros((1, HOP)), fb) == np.log(CLIP))


# ------------------------------------------------------------------------------------------------------------------
# the generator
# ------------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu
_FOOT = {}


def gen_module(state):
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    return g.cuda().eval()


@pytest.fixture(scope="module")
def gstates():
    return [synth.generator_state(s) for s in (1234, 77, 4242)]


@pytest.fixture(scope="module")
def gens(gstates):
    return [gen_module(s) for s in gstates]


@pytest.fixture(scope="module")
def g64s(gstates):
    from kernel_model import Gen64
    return [Gen64(s) for s in gstates]


def footprint(g64, mel_item, frames, value):
    """(footprint, float64 reference) of one item [80, L] with `value` at `frames`: the footprint is the NaN set of
    forward64 with NaN there, the reference is forward64 with `value` there; both [256 L]."""
    from kernel_model import forward64
    m = mel_item.double().clone()
    m[:, frames] = NAN
    key = (id(g64), m.shape[1], tuple(frames))
    if key not in _FOOT:
        _FOOT[key] = torch.isnan(forward64(g64, m[None], False)[0, 0])
    if value != value:
        return _FOOT[key], None
    m[:, frames] = value
    return _FOOT[key], forward64(g64, m[None], False)[0, 0]


def check_item_audio(clean, got, foot, ref, what):
    """One poisoned item's audio [n] (float or int16) against the clean call's, its footprint and reference."""
    n = foot.numel()
    clean, got = clean[:n], got[:n]
    eq = same_bits(got, clean)
    assert bool(eq[~foot].all()), (what, "outside the footprint", torch.nonzero(~eq & ~foot)[:5].flatten().tolist())
    pcm = got.dtype == torch.int16
    is_nan = (got == 0) if pcm else torch.isnan(got)
    ref_nan = foot if ref is None else torch.isnan(ref)
    assert bool(is_nan[ref_nan].all()), (what, "swallowed", int((ref_nan & ~is_nan).sum()))
    if ref is not None:  # +-Inf: inside the footprint the kernel gives the reference's value or NaN
        r32 = ref.float()
        want = torch.from_numpy(pcm16_np(r32.cpu().numpy())).cuda() if pcm else r32
        ok = is_nan | (got == want)
        assert bool(ok[foot].all()), (what, "inside the footprint", int((~ok & foot).sum()))
    return int(foot.sum())


def pcm16_np(a):
    a = np.asarray(a, dtype=np.float32)
    s = np.clip(np.rint(32768.0 * a.astype(np.float64)), -32768, 32767)
    s[np.isnan(a)] = 0
    return s.astype(np.int16)


def check_batch(clean, got, poisons, lens, g64_of, mel, what):
    """clean / got [B, 1, 256 T]; poisons {item: (frames, value)}; the float64 models per item (g64_of(i))."""
    for i in range(clean.shape[0]):
        if i not in poisons:
            assert bool(same_bits(got[i], clean[i]).all()), (what, "item", i)
            continue
        frames, value = poisons[i]
        L = lens[i]
        foot, ref = footprint(g64_of(i), mel[i, :, :L], frames, value)
        check_item_audio(clean[i, 0], got[i, 0], foot, ref, (what, i, frames))
        assert bool(same_bits(got[i, 0, 256 * L:], clean[i, 0, 256 * L:]).all()), (what, i, "past the length")


def resblock_border_frames(T):
    """Frames next to a cluster or CTA-rank border of the stage-0 (x8) and stage-1 (x64) ResBlocks and of the fused
    stride-2 ConvT + ResBlock of stages 2 (x128) and 3 (x256), for an item of T frames (kernel_model.borders)."""
    from kernel_model import borders, config
    out = set()
    for code, scale in ((0, 8), (1, 64), (12, 128), (13, 256)):
        for b in borders(config(code), scale * T):
            out |= {(b - 1) // scale, b // scale}
    return sorted(f for f in out if 0 < f < T - 1)


def poison_mel(mel, poisons):
    m = mel.clone()
    for i, (frames, value) in poisons.items():
        m[i, :, frames] = value
    return m


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("poison", list(POISONS))
def test_generate_uniform_sliced(gens, g64s, precision, poison):
    """B = 64, T = 32 runs as four batch slices of 16 items: poisoned items at the first and last item of a slice, at the
    first and last frame, next to ResBlock borders and in the interior; float and int16 audio."""
    B, T = 64, 32
    assert engine.lib().mg_gen_forward_slices(B, T) == 4
    mel = torch.from_numpy(synth.mel_input(B, T, 5)).cuda()
    v = POISONS[poison]
    bf = resblock_border_frames(T)
    poisons = {0: ([0], v), 15: ([T - 1], v), 16: ([bf[0]], v), 31: ([bf[-1]], v), 47: ([T // 2], v)}
    bad = poison_mel(mel, poisons)
    for dtype in (torch.float32, torch.int16):
        clean = gens[0].generate(mel, precision=precision, dtype=dtype)
        got = gens[0].generate(bad, precision=precision, dtype=dtype)
        if precision == "fp32":
            check_batch(clean, got, poisons, [T] * B, lambda i: g64s[0], mel, ("uniform", dtype))
        else:  # bf16: the footprint is structural; the same sets as fp32's
            check_batch(clean, got, poisons, [T] * B, lambda i: g64s[0], mel, ("uniform bf16", dtype))
    print("uniform %s %s: footprint growth 0 samples (generator)" % (precision, poison))


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("poison", list(POISONS))
def test_generate_ragged(gens, g64s, precision, poison):
    """Items of different lengths share CTAs and tiles: poison the first frame, the last valid frame and a frame next to a
    ResBlock border of one item; its neighbours stay bit for bit."""
    from kernel_model import ragged_batch
    lens = [40, 1, 64, 7, 64, 33, 2]
    mel = ragged_batch(lens, 300)
    v = POISONS[poison]
    poisons = {0: ([0], v), 1: ([0], v), 2: ([resblock_border_frames(64)[0]], v), 3: ([6], v), 5: ([32], v)}
    bad = poison_mel(mel, poisons)
    for dtype in (torch.float32, torch.int16):
        clean = gens[1].generate(mel, lens, precision=precision, dtype=dtype)
        got = gens[1].generate(bad, lens, precision=precision, dtype=dtype)
        check_batch(clean, got, poisons, lens, lambda i: g64s[1], mel, ("ragged", precision, dtype))


@gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("order", ["interleaved", "sorted"])
def test_generate_voices(gens, g64s, precision, order):
    """generate_voices: NaN frames in items of two voices; then NaN in one weight_v of voice 1 (repack()): the other
    voices' items stay bit for bit, voice 1's are NaN wherever float64 makes them NaN, and after the weight is restored
    the whole batch is the clean run again."""
    lens = [5, 1, 17, 32, 9, 1, 24, 3, 12]
    voice = [i % 3 for i in range(len(lens))]
    if order == "sorted":
        voice = sorted(voice)
    from kernel_model import ragged_batch, Gen64, forward64
    mel = ragged_batch(lens, 900)
    poisons = {2: ([16], NAN), 3: ([0], -INF), 6: ([11], INF)}
    bad = poison_mel(mel, poisons)
    for dtype in (torch.float32, torch.int16):
        clean = models.generate_voices(gens, mel, voice, lens, precision=precision, dtype=dtype)
        got = models.generate_voices(gens, bad, voice, lens, precision=precision, dtype=dtype)
        check_batch(clean, got, poisons, lens, lambda i: g64s[voice[i]], mel, ("voices", precision, dtype))
    # a corrupt voice: one NaN in ups.1's weight_v (its fold makes that whole input-channel row NaN)
    g1 = gens[1]
    clean = models.generate_voices(gens, mel, voice, lens, precision=precision)
    with torch.no_grad():
        keep = g1.ups[1].weight_v[3, 5, 2].item()
        g1.ups[1].weight_v.data[3, 5, 2] = NAN
    g1.repack()
    try:
        got = models.generate_voices(gens, mel, voice, lens, precision=precision)
        got16 = models.generate_voices(gens, mel, voice, lens, precision=precision, dtype=torch.int16)
        st = {k: v.detach().cpu().numpy().copy() for k, v in g1.state_dict().items()}
        g64 = Gen64(st)
        for i, L in enumerate(lens):
            if voice[i] != 1:
                assert bool(same_bits(got[i], clean[i]).all()), ("other voice", i)
                continue
            ref_nan = torch.isnan(forward64(g64, mel[i:i + 1, :, :L].double(), False)[0, 0])
            assert bool(ref_nan.any())
            assert bool(torch.isnan(got[i, 0, :256 * L])[ref_nan].all()) and bool((got16[i, 0, :256 * L] == 0)[ref_nan].all()), i
            assert bool(same_bits(got[i, 0, :256 * L], clean[i, 0, :256 * L])[~ref_nan].all()), i
    finally:
        with torch.no_grad():
            g1.ups[1].weight_v.data[3, 5, 2] = keep
        g1.repack()
    again = models.generate_voices(gens, mel, voice, lens, precision=precision)
    assert bool(same_bits(again, clean).all())


@gpu
@pytest.mark.parametrize("pinned", [False, True])
def test_host_engine(gstates, g64s, pinned):
    """GeneratorHost: uniform and ragged batches into pinned or pageable int16 and float buffers."""
    eng = engine.GeneratorHost(8, 64)
    try:
        eng.load_state(gstates[0])
        lens = [64, 1, 13, 40, 2, 64, 9, 33]
        mel = np.zeros((8, 80, 64), np.float32)
        for i, L in enumerate(lens):
            mel[i, :, :L] = synth.mel_input(1, L, 70 + i)[0]
        poisons = {0: ([63], NAN), 3: ([0], INF), 7: ([32], -INF)}
        bad = mel.copy()
        for i, (fr, v) in poisons.items():
            bad[i, :, fr] = v
        for precision in ("fp32", "bf16"):
            for ragged in (False, True):
                for dt in (np.float32, np.int16):
                    whole = (torch.zeros(8 * 256 * 64, dtype=torch.int16 if dt == np.int16 else torch.float32).pin_memory().numpy()
                             if pinned else np.zeros(8 * 256 * 64, dt))
                    out = whole.reshape(8, 1, 256 * 64)
                    run = (lambda m, o=None: eng.forward_ragged(m, lens, out=o, precision=precision, dtype=dt)) if ragged else \
                          (lambda m, o=None: eng.forward(m, out=o, precision=precision, dtype=dt))
                    clean = torch.from_numpy(np.array(run(mel))).cuda()
                    got = run(bad, out)
                    assert got is out
                    got = torch.from_numpy(np.array(got)).cuda()
                    check_batch(clean, got, poisons, lens if ragged else [64] * 8, lambda i: g64s[0], torch.from_numpy(mel).cuda(),
                                ("host", precision, ragged, dt))
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------
# streams
# ------------------------------------------------------------------------------------------------------------------
def push_all(st, utts, P, voice=None, nan_at=None, reset_after=None):
    """Push utterances (one per slot, [80, T_i] each) in chunks of at most P frames, END with the last chunk; returns
    each slot's concatenated audio."""
    S = len(utts)
    pos, out = [0] * S, [[] for _ in range(S)]
    while any(pos[i] < utts[i].shape[1] for i in range(S)):
        chunks, end = [], []
        for i in range(S):
            n = min(P - (i % 3), utts[i].shape[1] - pos[i])
            chunks.append(utts[i][:, pos[i]:pos[i] + n].contiguous() if n > 0 else None)
            pos[i] += max(n, 0)
            end.append(n > 0 and pos[i] == utts[i].shape[1])
        outs = st.step(chunks, end=end, voice=voice)
        for i, o in enumerate(outs):
            if chunks[i] is not None:
                out[i].append(o[0])
    return [torch.cat(o) for o in out]


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16])
@pytest.mark.parametrize("voices", [False, True])
def test_stream_sessions(gens, dtype, voices):
    """A NaN frame (and an Inf frame) pushed in one session: the other sessions' audio is bit for bit generate() of their
    mel, the poisoned session's is generate() of its poisoned mel."""
    lens = [40, 23, 57]
    utts = [torch.from_numpy(synth.mel_input(1, T, 60 + i)).cuda()[0] for i, T in enumerate(lens)]
    bad = [u.clone() for u in utts]
    bad[1][:, 9] = NAN
    bad[1][:, 20] = INF
    voice = [0, 1, 2] if voices else None
    st = models.stream_voices(gens, 3, 8, dtype=dtype) if voices else gens[0].stream(3, 8, dtype=dtype)
    got = push_all(st, bad, 8, voice=voice)
    st.check_status()
    for i in range(3):
        g = gens[voice[i]] if voices else gens[0]
        want = g.generate(bad[i][None], dtype=dtype)[0, 0]
        assert bool(same_bits(got[i], want).all()), i
        if i != 1:
            assert bool(same_bits(got[i], g.generate(utts[i][None], dtype=dtype)[0, 0]).all()), i
    assert bool(torch.isnan(got[1]).any()) if dtype == torch.float32 else bool((got[1] == 0).any())
    st.close()


@gpu
@pytest.mark.parametrize("how", ["end", "reset"])
@pytest.mark.parametrize("voices", [False, True])
def test_stream_slot_reuse(gens, how, voices):
    """A slot whose utterance saw NaN frames (its stored tails hold NaN), then END or RESET, then a clean utterance on the
    same slot: bit for bit a stream that never saw the NaN."""
    P = 8
    first = torch.from_numpy(synth.mel_input(1, 30, 81)).cuda()[0]
    first[:, 21:] = NAN  # the last frames: every tail of the slot holds NaN when the utterance ends or is reset
    nxt = torch.from_numpy(synth.mel_input(1, 37, 82)).cuda()[0]
    other = torch.from_numpy(synth.mel_input(1, 60, 83)).cuda()[0]
    voice = [1, 2] if voices else None
    st = models.stream_voices(gens, 2, P, dtype=torch.float32) if voices else gens[0].stream(2, P)
    pos = 0
    outs1 = []
    while pos < 30:  # slot 0: the poisoned utterance, slot 1: a clean one running alongside
        n = min(P, 30 - pos)
        end = how == "end" and pos + n == 30
        o = st.step([first[:, pos:pos + n].contiguous(), other[:, pos:pos + n].contiguous()], end=[end, False], voice=voice)
        outs1.append(o[1][0])
        pos += n
    pos2, got = 0, []
    while pos2 < 37 or pos < 60:
        n = min(P, 37 - pos2)
        m = min(P, 60 - pos)
        o = st.step([nxt[:, pos2:pos2 + n].contiguous() if n else None, other[:, pos:pos + m].contiguous() if m else None],
                    end=[n > 0 and pos2 + n == 37, m > 0 and pos + m == 60], reset=[how == "reset" and pos2 == 0, False],
                    voice=voice)
        if n:
            got.append(o[0][0])
        if m:
            outs1.append(o[1][0])
        pos2 += n
        pos += m
    st.check_status()
    g0 = gens[1] if voices else gens[0]
    g1 = gens[2] if voices else gens[0]
    assert bool(same_bits(torch.cat(got), g0.generate(nxt[None])[0, 0]).all())
    assert bool(same_bits(torch.cat(outs1), g1.generate(other[None])[0, 0]).all())
    st.close()


# ------------------------------------------------------------------------------------------------------------------
# the mel front end
# ------------------------------------------------------------------------------------------------------------------
def mel_gpu(y):
    return meldataset.mel_spectrogram(y, NFFT, 80, 22050, HOP, NFFT, 55.0, 9000.0, check_range=False)


def mel_positions(L):
    """A sample at a frame's first position (window 0), one next to a frame edge, one in the interior."""
    return [HOP * 2 - PAD + NFFT, HOP * 3 - PAD + 1, L // 2 + 77]


@gpu
@pytest.mark.parametrize("poison", list(POISONS))
def test_mel_forward(poison):
    """A poisoned sample makes exactly the reference's frames non-finite; NaN where np.clip gives NaN (never log(1e-5))."""
    B, L = 3, 24 * HOP
    y = (torch.rand(B, L, generator=torch.Generator().manual_seed(3)) * 1.6 - 0.8).cuda()
    fb = mo.mel_filterbank64(22050, NFFT, 80, 55.0, 9000.0, 1)
    clean = mel_gpu(y)
    for p in mel_positions(L):
        bad = y.clone()
        bad[1, p] = POISONS[poison]
        got = mel_gpu(bad)
        for i in (0, 2):
            assert bool(same_bits(got[i], clean[i]).all()), (p, i)
        yn = bad[1:2].double().cpu().numpy()
        yn[0, p] = NAN
        foot = torch.from_numpy(np.isnan(mel64(yn, fb)[0])).cuda()
        ref = torch.from_numpy(mel64(bad[1:2].double().cpu().numpy(), fb)[0]).cuda()
        assert bool(same_bits(got[1], clean[1])[~foot].all()), p
        g = got[1]
        ref_nan = torch.isnan(ref)
        assert bool(torch.isnan(g)[ref_nan].all()), (p, "swallowed", g[ref_nan & ~torch.isnan(g)][:4].tolist())
        ok = torch.isnan(g) | (g == ref.float())
        assert bool(ok[foot].all()), (p, g[foot & ~ok][:4].tolist(), ref[foot & ~ok][:4].tolist())


def mel_graph64(y, fb):
    T = y.shape[-1] // HOP
    frames = F.pad(y, (PAD, PAD)).unfold(-1, NFFT, HOP)[:, :T]
    mag = torch.fft.rfft(frames * torch.from_numpy(WIN64).to(y), dim=-1).abs()
    return torch.log(torch.clamp(torch.einsum("mk,btk->bmt", torch.from_numpy(fb).to(y), mag), min=CLIP))


@gpu
@pytest.mark.parametrize("where", ["audio", "grad_mel"])
def test_mel_backward(where):
    """mg_mel_spectrogram_backward with NaN in one item's audio or grad_mel: the NaN set of the gradient is float64
    torch autograd's, the other items' gradients are the clean call's bit for bit."""
    B, L = 3, 20 * HOP
    y = (torch.rand(B, L, generator=torch.Generator().manual_seed(9)) * 1.6 - 0.8).cuda()
    fb = mo.mel_filterbank64(22050, NFFT, 80, 55.0, 9000.0, 1)
    T = L // HOP
    gmel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(10)).cuda()

    def grad(yy, gg):
        yy = yy.clone().requires_grad_(True)
        return torch.autograd.grad(mel_gpu(yy), yy, gg)[0]
    clean = grad(y, gmel)
    for p in (mel_positions(L) if where == "audio" else [(5, 0), (40, 7), (79, T - 1)]):
        yb, gb = y.clone(), gmel.clone()
        if where == "audio":
            yb[1, p] = NAN
        else:
            gb[1, p[0], p[1]] = NAN
        got = grad(yb, gb)
        for i in (0, 2):
            assert bool(same_bits(got[i], clean[i]).all()), (p, i)
        y64 = yb[1:2].double().cpu().requires_grad_(True)
        ref = torch.autograd.grad(mel_graph64(y64, fb), y64, gb[1:2].double().cpu())[0][0]
        ref_nan = torch.isnan(ref).cuda()
        assert bool(ref_nan.any())
        assert torch.equal(torch.isnan(got[1]), ref_nan), (p, int(torch.isnan(got[1]).sum()), int(ref_nan.sum()))


# ------------------------------------------------------------------------------------------------------------------
# the discriminators
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dstate():
    return synth.discriminator_state(4321)


@pytest.fixture(scope="module")
def msd(dstate):
    m = models.MultiScaleDiscriminator()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in dstate.items()})
    return m.cuda()


def dweights(dstate, s):
    out = []
    for n, *_ in DLAYERS:
        k = "discriminators.%d.%s" % (s, n)
        out.append((torch.from_numpy(fold64(dstate[k + ".weight_g"], dstate[k + ".weight_v"])).cuda(),
                    torch.from_numpy(dstate[k + ".bias"].astype(np.float64)).cuda()))
    return out


def pooled64(y64, s):
    x = y64
    for k in range(s):
        x = F.avg_pool1d(x, 4, 2 if k == 0 else 4, padding=2)
    return x


GROWTH = {}


def check_disc_scale(fm_clean, fm_got, x_got, ws, items, what):
    """The seven maps of one scale: items not in `items` bit for bit; for each poisoned item and layer, with the kernel's
    own input of that layer: outside the kernel window footprint bit for bit, NaN wherever float64 conv1d of that input
    is NaN, +-Inf or NaN where it is +-Inf.  Records the growth (outputs beyond the reference footprint) per layer."""
    B = fm_got[0].shape[0]
    others = [i for i in range(B) if i not in items]
    xin = x_got
    for l, (n, _ci, _co, k, s, g, p) in enumerate(DLAYERS):
        got, clean = fm_got[l], fm_clean[l]
        assert bool(same_bits(got[others], clean[others]).all()), (what, n, "other items")
        x = xin[items].double()
        bad_in = (~torch.isfinite(x)).any(dim=1)                        # [b, Lin]
        w, b = ws[l]
        xn = torch.where(torch.isfinite(x), x, torch.full_like(x, NAN))
        foot_ref = torch.isnan(F.conv1d(xn, w, b, stride=s, padding=p, groups=g))
        ref = F.conv1d(x, w, b, stride=s, padding=p, groups=g)
        if l < 6:
            ref = F.leaky_relu(ref)
        lo, hi, grp = disc_window(l, got.shape[-1])
        foot = foot_ref | window_mask(bad_in, lo, hi, s, grp, got.shape[-1])[:, None, :]
        gi, ci = got[items], clean[items]
        eq = same_bits(gi, ci)
        assert bool(eq[~foot].all()), (what, n, "outside the kernel window")
        gn = torch.isnan(gi)
        assert bool(gn[torch.isnan(ref)].all()), (what, n, "swallowed")
        inf = torch.isinf(ref)
        assert bool((gn | (gi.double() == ref))[inf].all()), (what, n, "+-Inf")
        grown = ~eq & ~foot_ref
        if bool(grown.any()):
            idx = torch.nonzero(grown.any(dim=1))[:, 1]
            ref_idx = torch.nonzero(foot_ref.any(dim=1))[:, 1]
            d = int((idx[:, None] - ref_idx[None, :]).abs().min(dim=1).values.max()) if ref_idx.numel() else -1
        else:
            d = 0
        GROWTH[n] = max(GROWTH.get(n, 0), d)
        xin = fm_got[l]


def disc_batch(B, L, seed):
    return (torch.rand(B, 1, L, generator=torch.Generator().manual_seed(seed)) * 1.8 - 0.9).cuda()


# (L, why): items of 20 outputs at grouped_convs.0 share a CTA as virtual rows; 1600 has several tiles per item
DISC_LENGTHS = {"short": 320, "long": 6400}


@gpu
@pytest.mark.parametrize("size", list(DISC_LENGTHS))
@pytest.mark.parametrize("poison", list(POISONS))
def test_msd_forward(msd, dstate, size, poison):
    """The stacked real + generated batch of MultiScaleDiscriminator: poison one generated item at its first sample, its
    last and in the interior (short: the items share CTAs as virtual rows at every grouped layer of every scale; long:
    each item has its own tiles), all three scales."""
    L = DISC_LENGTHS[size]
    B = 5
    lens = engine.msd_lengths(L)
    if size == "short":
        assert group_tc_plan(lens[0][1])[1] > 1 and group4_plan(lens[0][4])[0] > 1
    else:
        assert group_tc_plan(lens[0][1])[1] == 1
    y, yh = disc_batch(B, L, 1), disc_batch(B, L, 2)
    with torch.no_grad():
        msd(y, yh)  # packs the blob
        clean = msd._dev.forward(torch.cat([y, yh]))
    v = POISONS[poison]
    for pos in (0, L - 1, L // 2 + 3):
        bad = yh.clone()
        bad[2, 0, pos] = v
        y2 = torch.cat([y, bad])
        with torch.no_grad():
            got = msd._dev.forward(y2)
        for s in range(3):
            ws = dweights(dstate, s)
            x0 = pooled64(y2.double(), s)
            check_disc_scale(clean[s], got[s], x0, ws, [B + 2], (size, poison, pos, s))
    torch.cuda.synchronize()
    print("disc growth (outputs beyond float64's footprint):", GROWTH)


@gpu
@pytest.mark.parametrize("poison", ["nan", "+inf"])
def test_discriminator_alone(dstate, poison):
    """The stand-alone Discriminator on its own blob: same rule, items of a virtual-row batch."""
    d = models.Discriminator()
    d.load_state_dict({k[len("discriminators.0."):]: torch.from_numpy(v) for k, v in dstate.items() if k.startswith("discriminators.0.")})
    d = d.cuda()
    x = disc_batch(6, 400, 3)
    with torch.no_grad():
        _, clean = d(x)
        bad = x.clone()
        bad[3, 0, 200] = POISONS[poison]
        _, got = d(bad)
    check_disc_scale(clean, got, bad, dweights(dstate, 0), [3], ("alone", poison))


@gpu
@pytest.mark.parametrize("scale", [0, 1, 2])
def test_msd_scale_backward(msd, dstate, scale):
    """mg_msd_scale_backward with NaN in one item's upstream gradient (one position of feature map 3, then the logits):
    the other items' gx0 is the clean call's bit for bit, dw / db are NaN exactly where float64 autograd's are.  The
    float64 autograd runs on the CPU, whose im2col forms every product: cuDNN's float64 weight gradient of the grouped
    convs leaves some taps of a NaN row finite."""
    B, L = 6, 1600
    y2 = disc_batch(B, L, 4)
    with torch.no_grad():
        msd(y2[:3], y2[3:])
        fm = msd._dev.forward(y2)[scale]
    x0 = pooled64(y2.double(), scale).float()
    rng = torch.Generator().manual_seed(5)
    grads = [torch.randn(f.shape, generator=rng).cuda() if l in (3, 6) else None for l, f in enumerate(fm)]
    gx0_c, dw_c, db_c = msd._dev.scale_backward(scale, x0, fm, grads, True)
    gx0_c = gx0_c.clone()
    ws = dweights(dstate, scale)
    for l in (3, 6):
        gb = [g.clone() if g is not None else None for g in grads]
        gb[l][4, 0, gb[l].shape[-1] // 3] = NAN
        gx0, dw, db = msd._dev.scale_backward(scale, x0, fm, gb, True)
        others = [0, 1, 2, 3, 5]
        assert bool(same_bits(gx0[others], gx0_c[others]).all()), l
        # float64 autograd of the same chain on the same input
        leaves = [(w.cpu().requires_grad_(True), b.cpu().requires_grad_(True)) for w, b in ws]
        x = x0.double().cpu().requires_grad_(True)
        h, outs = x, []
        for li, (n, _ci, _co, k, s, g, p) in enumerate(DLAYERS):
            h = F.conv1d(h, leaves[li][0], leaves[li][1], stride=s, padding=p, groups=g)
            if li < 6:
                h = F.leaky_relu(h)
            outs.append(h)
        pairs = [(o, g.double().cpu()) for o, g in zip(outs, gb) if g is not None]
        r = torch.autograd.grad([o for o, _ in pairs], [x] + [t for wb in leaves for t in wb], [g for _, g in pairs], allow_unused=True)
        r = [t.cuda() if t is not None else None for t in r]
        gx_ref = r[0]
        assert bool(torch.isnan(gx0)[torch.isnan(gx_ref)].all()), l
        for li in range(7):
            rw, rb = r[1 + 2 * li], r[2 + 2 * li]
            if rw is None or dw[li] is None:
                assert (rw is None or not bool(torch.isnan(rw).any())) and dw[li] is None or rw is not None, (l, li)
                continue
            assert torch.equal(torch.isnan(dw[li]), torch.isnan(rw)), (l, li, int(torch.isnan(dw[li]).sum()), int(torch.isnan(rw).sum()))
            assert torch.equal(torch.isnan(db[li]), torch.isnan(rb)), (l, li)


# ------------------------------------------------------------------------------------------------------------------
# losses and Adam
# ------------------------------------------------------------------------------------------------------------------
CHUNK = 16384  # kLossChunk: elements per CTA of the loss kernels


@gpu
@pytest.mark.parametrize("fn", ["feature", "discriminator", "generator"])
def test_loss_rows(fn):
    """A NaN in one row (at the start of its last CTA's chunk) makes that row's mean NaN and no other; backward: L1
    elements at NaN get 0 (torch's sign), LSGAN elements NaN, the other rows' gradients bit for bit the clean call's.
    The clean means are held to float64."""
    rng = torch.Generator().manual_seed(7)
    sizes = [(2, 3, 2 * CHUNK // 6 + 5), (2, 1, CHUNK), (1, 2, CHUNK // 2 + 1), (3, 1, 100)]
    a = [torch.randn(s, generator=rng).cuda() for s in sizes]
    b = [torch.randn(s, generator=rng).cuda() for s in sizes]

    def run(aa, bb):
        aa = [t.clone().requires_grad_(True) for t in aa]
        bb = [t.clone().requires_grad_(True) for t in bb]
        if fn == "feature":
            rows = models._row_means(aa, bb, [engine.LOSS_L1] * len(aa))
        elif fn == "discriminator":
            rows = models._row_means(aa + bb, [None] * 8, [engine.LOSS_ONE_MINUS_SQ] * 4 + [engine.LOSS_SQ] * 4)
        else:
            rows = models._row_means(aa, [None] * 4, [engine.LOSS_ONE_MINUS_SQ] * 4)
        grads = torch.autograd.grad(rows, aa + bb, torch.ones_like(rows), allow_unused=True)
        return rows.detach(), grads
    # the public functions' values are these row sums
    fl = models.feature_loss([a], [b])
    dl = models.discriminator_loss(a, b)
    gl = models.generator_loss(a)
    rows_c, grads_c = run(a, b)
    ref = {"feature": [float((x.double() - y.double()).abs().mean()) for x, y in zip(a, b)],
           "discriminator": [float(((1 - x.double()) ** 2).mean()) for x in a] + [float((y.double() ** 2).mean()) for y in b],
           "generator": [float(((1 - x.double()) ** 2).mean()) for x in a]}[fn]
    assert np.allclose(rows_c.cpu().numpy(), ref, rtol=1e-5, atol=0), (rows_c.tolist(), ref)
    assert math.isclose(float(fl), 10 * sum(ref if fn == "feature" else [float((x.double() - y.double()).abs().mean()) for x, y in zip(a, b)]), rel_tol=1e-5)
    assert math.isfinite(float(dl[0])) and math.isfinite(float(gl))
    for r in range(4):
        n = a[r].numel()
        for e in sorted({(n - 1) // CHUNK * CHUNK, n - 1, 0}):
            ab = [t.clone() for t in a]
            ab[r].view(-1)[e] = NAN
            rows, grads = run(ab, b)
            for j in range(rows.numel()):
                assert math.isnan(float(rows[j])) == (j == r), (fn, r, e, rows.tolist())
            for j, (g, gc) in enumerate(zip(grads, grads_c)):
                if g is None:
                    continue
                if j != r and j != 4 + r:
                    assert bool(same_bits(g, gc).all()), (fn, r, e, j)
                    continue
                # float64 torch: d mean |a - b| = sign(a - b) / n (0 at NaN); d mean (1 - a)^2 = -2 (1 - a) / n (NaN)
                x = (ab[r] if j == r else b[r]).double().cpu().requires_grad_(True)
                other = (b[r] if j == r else ab[r]).double().cpu()
                if fn == "feature":
                    val = ((x - other) if j == r else (other - x)).abs().mean()
                elif fn == "discriminator" or fn == "generator":
                    val = ((1 - x) ** 2).mean() if j < 4 else (x ** 2).mean()
                (gr,) = torch.autograd.grad(val, x)
                assert torch.equal(torch.isnan(g).cpu(), torch.isnan(gr)), (fn, r, e, j)
                assert bool(same_bits(g, gc).view(-1)[torch.arange(g.numel(), device=g.device) != e].all()), (fn, r, e, j)


@gpu
def test_adam_nan_gradient():
    """optim.Adam with a NaN in one tensor's gradient, at a 4096-element chunk border and inside: only that element of
    that tensor's p, m and v changes from the clean step (to NaN, as float64 Adam gives)."""
    sizes = [5000, 4096 + 3, 100, 8192]
    rng = torch.Generator().manual_seed(8)
    p0 = [torch.randn(n, generator=rng).cuda() for n in sizes]
    g0 = [torch.randn(n, generator=rng).cuda() for n in sizes]

    def step(grads):
        ps = [torch.nn.Parameter(p.clone()) for p in p0]
        opt = optim.Adam(ps, lr=1e-3, betas=(0.8, 0.99))
        for _ in range(2):
            for p, g in zip(ps, grads):
                p.grad = g.clone()
            opt.step()
        return [(p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]) for p in ps]
    clean = step(g0)
    for t, e in ((1, 4095), (1, 4096), (3, 4096), (0, 17)):
        gb = [g.clone() for g in g0]
        gb[t][e] = NAN
        got = step(gb)
        for j in range(len(sizes)):
            for k in range(3):
                eq = same_bits(got[j][k], clean[j][k])
                if j != t:
                    assert bool(eq.all()), (t, e, j, k)
                else:
                    assert bool(torch.isnan(got[j][k][e])) and bool(eq[torch.arange(sizes[j], device=eq.device) != e].all()), (t, e, k)
