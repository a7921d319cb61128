"""CPU checks of the streaming denoiser (mg_denoise_stream_*): the finality rule restated and checked in float64 on the
denoiser's own definition (denoise_model.denoise64), the left context a session keeps for its END frames, the host
bookkeeping over seeded push schedules, and argument errors reported before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import denoise_model as dm
from melgan_multi_b200 import denoiser, engine

END, RESET = engine.STREAM_END, engine.STREAM_RESET
# (n_fft, hop, win_length): hop <= N/2 and hop > N/2, windows shorter than n_fft
ANALYSES = [(128, 32, 128), (256, 64, 200), (512, 384, 512), (1024, 256, 1024), (1024, 600, 800), (2048, 512, 1536)]


def emitted(n, h, R):
    """E(R): the samples an open session has emitted after receiving R."""
    if R <= n // 2:
        return 0
    q = (R - n // 2) // h
    return min(max((q + 1) * h - n // 2, 0), R)


def frames_open(n, h, R):
    return 0 if R <= n // 2 else (R - n // 2) // h + 1


def first_read(n, h, F):
    """The first sample a frame >= F can read: the tail an open session keeps starts there."""
    return max(0, F * h - n // 2 - 1)


def _lens_above(n, h, R):
    """Utterance lengths > R with L mod h = 0, 1 and h - 1 (the END residue classes), all NOLA-clean."""
    out = []
    for r in (0, 1, h - 1):
        L = (R // h + 2) * h + r
        out.append(L)
    return out


def _rs(n, h, rng):
    return sorted({n // 2, n // 2 + 1, n // 2 + h, n + 3 * h - 1, n + 3 * h} | {int(v) for v in rng.integers(n // 2 + 2, 4 * n, 5)})


@pytest.mark.parametrize("n,h,w", ANALYSES)
def test_samples_below_e_are_final(n, h, w):
    """Exactness: the samples below E(R) of denoise64 do not change when the signal after R, or its length, changes."""
    rng = np.random.default_rng(n + h)
    bias = torch.from_numpy(np.abs(rng.standard_normal(n // 2 + 1)) * 0.3)
    for R in _rs(n, h, rng):
        base = torch.from_numpy(rng.standard_normal(R))
        e = emitted(n, h, R)
        ref = None
        for L in _lens_above(n, h, R):
            if not dm.nola_ok(n, h, w, L):
                continue
            a = torch.cat([base, torch.from_numpy(rng.standard_normal(L - R))])
            y = dm.denoise64(a, n, h, w, bias, 0.5)[:e]
            if ref is None:
                ref = y
            assert torch.equal(y, ref), (n, h, w, R, L)
        # and at END: an utterance of exactly R samples (the END step emits the rest, but the first E(R) are the same)
        if R > n // 2 and dm.nola_ok(n, h, w, R) and ref is not None:
            assert torch.equal(dm.denoise64(base, n, h, w, bias, 0.5)[:e], ref), (n, h, w, R)


@pytest.mark.parametrize("n,h,w", ANALYSES)
def test_a_nan_at_r_first_reaches_sample_e(n, h, w):
    """Tightness: a NaN at sample R makes sample E(R) the first NaN output, so no sample at or past E(R) is final."""
    rng = np.random.default_rng(7 * n + h)
    bias = torch.from_numpy(np.abs(rng.standard_normal(n // 2 + 1)) * 0.3)
    cases = 0
    for R in _rs(n, h, rng):
        for L in _lens_above(n, h, R):
            if not dm.nola_ok(n, h, w, L):
                continue
            a = torch.from_numpy(rng.standard_normal(L))
            a[R] = float("nan")
            y = dm.denoise64(a, n, h, w, bias, 0.5)
            bad = torch.nonzero(torch.isnan(y)).flatten()
            assert int(bad[0]) == emitted(n, h, R), (n, h, w, R, L)
            cases += 1
    assert cases >= 10


@pytest.mark.parametrize("n,h,w", ANALYSES)
def test_end_frames_read_no_sample_left_of_the_tail(n, h, w):
    """The left context at END: with F frames computed, no frame >= F of any utterance reads a sample below
    first_read(F); frame L / h reads exactly that sample when h divides L (reflecting back to L - n/2 - 1, one left of
    its own window)."""
    rng = np.random.default_rng(n * 3 + h)
    for L in [n // 2 + 1, n, 3 * n + 1] + [(k * h) for k in range(n // (2 * h) + 1, n // (2 * h) + 6)] + [5 * h + 1, 5 * h + h - 1]:
        if L <= n // 2:
            continue
        T = 1 + L // h
        x = torch.nn.functional.pad(torch.arange(L, dtype=torch.float64)[None, None], (n // 2, n // 2), mode="reflect")[0, 0]
        lowest = [int(x[t * h:t * h + n].min()) for t in range(T)]  # the lowest sample each frame reads
        for F in range(T):
            assert min(lowest[F:]) >= first_read(n, h, F), (n, h, L, F)
        if L % h == 0 and L // h * h - n // 2 - 1 >= 0:
            assert lowest[L // h] == L - n // 2 - 1 == first_read(n, h, L // h)
    del rng


def _handle(n=1024, h=256, w=1024, S=4, P=700, strength=0.1):
    L = denoiser._lib()
    nbytes = L.mg_denoise_stream_state_bytes(n, h, S, P)
    assert nbytes > 0
    hd = ctypes.c_void_p()
    rc = L.mg_denoise_stream_create(ctypes.byref(hd), n, h, w, S, P, strength, ctypes.c_void_p(1 << 20), nbytes)
    assert rc == 0, L.mg_last_error_string()
    return hd


def _ints(v):
    return (ctypes.c_int * max(len(v), 1))(*v)


def _dry(hd, counts, flags=None, voice=None, n_voices=1):
    n = len(counts)
    out = (ctypes.c_int * max(n, 1))()
    nf = ctypes.c_int()
    rc = denoiser._lib().mg_denoise_stream_dry_step(hd, n_voices, None if voice is None else _ints(voice), _ints(counts),
                                                    None if flags is None else _ints(flags), n, out, ctypes.byref(nf))
    return rc, [out[i] for i in range(n)], nf.value


@pytest.mark.parametrize("n,h,w", ANALYSES)
@pytest.mark.parametrize("seed", [0, 1])
def test_bookkeeping_follows_the_contract(n, h, w, seed):
    """Seeded schedules of 0-, 1-, random and max_push_samples pushes with END and RESET: while open a slot has emitted
    E(R), after END all L; slots are reused; the frames computed follow F(R); max_out is never exceeded."""
    rng = np.random.default_rng(seed * 101 + n + h)
    S, P = 5, int(rng.choice([37, h, 3 * n]))
    L = denoiser._lib()
    hd = _handle(n, h, w, S, P)
    max_out = L.mg_denoise_stream_max_out(n, h, P)
    R = [0] * S
    got = [0] * S
    frames = [0] * S
    done = 0
    try:
        for _ in range(300):
            counts = [int(rng.choice([0, 1, P, rng.integers(0, P + 1)])) for _ in range(S)]
            flags = [0] * S
            for i in range(S):
                r = rng.random()
                L1 = R[i] + counts[i]
                if r < 0.03:
                    flags[i] = RESET
                elif r < 0.25 and L1 > n // 2 and dm.nola_ok(n, h, w, L1):
                    flags[i] = END
            rc, out, nf = _dry(hd, counts, flags)
            assert rc == 0, L.mg_last_error_string()
            want_frames = 0
            for i in range(S):
                if flags[i] & RESET:
                    R[i], got[i], frames[i] = 0, 0, 0
                R[i] += counts[i]
                got[i] += out[i]
                assert 0 <= out[i] <= max_out
                if flags[i] & END:
                    assert got[i] == R[i]
                    want_frames += 1 + R[i] // h - frames[i]
                    R[i], got[i], frames[i] = 0, 0, 0
                    done += 1
                else:
                    assert got[i] == emitted(n, h, R[i]), (i, R[i])
                    assert 0 <= R[i] - got[i] <= n - 1
                    f = frames_open(n, h, R[i])
                    want_frames += f - frames[i]
                    frames[i] = f
            assert nf == want_frames
    finally:
        L.mg_denoise_stream_destroy(hd)
    assert done > 10


@pytest.mark.parametrize("n,h", [(128, 32), (1024, 256), (1024, 600), (2048, 512)])
def test_max_out_is_tight(n, h):
    """max_out = P + n - 1, reached by an END push of P samples when R - E(R) = n - 1; open steps stay below it."""
    L = denoiser._lib()
    P = 3 * n
    assert L.mg_denoise_stream_max_out(n, h, P) == P + n - 1
    # R - E(R) = n - 1 exactly when (R - n/2) mod h = h - 1 and E(R) > 0
    R = n // 2 + 2 * h + h - 1
    assert R - emitted(n, h, R) == n - 1
    hd = _handle(n, h, n, 1, P)
    try:
        assert _dry(hd, [R])[0] == 0
        rc, out, _ = _dry(hd, [P], [END])
        assert rc == 0 and out == [P + n - 1]
    finally:
        L.mg_denoise_stream_destroy(hd)
    # an open push emits at most P + h - 1
    best = max(emitted(n, h, R + P) - emitted(n, h, R) for R in range(0, 4 * n))
    assert best <= P + h - 1 < P + n - 1


def test_steady_state_lookahead():
    """At n_fft 1024, hop 256 an open session holds back 768 .. 1023 samples once warmed up."""
    back = {R - emitted(1024, 256, R) for R in range(2048, 4096)}
    assert min(back) == 768 and max(back) == 1023


def test_voices_bind_and_release_like_the_generator_stream():
    L = denoiser._lib()
    hd = _handle(S=3)
    try:
        assert _dry(hd, [600, 600, 0], voice=[1, 0, 2], n_voices=3)[0] == 0
        rc = _dry(hd, [10, 0, 0], voice=[2, 0, 2], n_voices=3)[0]
        assert rc == -1
        msg = L.mg_last_error_string()
        assert b"voice[0] = 2" in msg and b"bound to voice 1" in msg and b"MG_GEN_STREAM_RESET" in msg
        # slot 2 has no open utterance: any id; RESET rebinds slot 0; END releases slot 1
        assert _dry(hd, [10, 10, 0], [RESET, END, 0], voice=[2, 0, 1], n_voices=3)[0] == 0
        assert _dry(hd, [5, 600, 0], voice=[2, 1, 0], n_voices=3)[0] == 0
        assert _dry(hd, [5, 5, 0], voice=[0, 1, 0], n_voices=3)[0] == -1
        assert _dry(hd, [5, 5, 0], voice=[2, 1, 0], n_voices=3)[0] == 0
        assert _dry(hd, [0, 0, 0], voice=[3, 1, 0], n_voices=3)[0] == -1 and b"voice[0] = 3" in L.mg_last_error_string()
    finally:
        L.mg_denoise_stream_destroy(hd)


def test_stream_argument_errors_are_reported_before_any_cuda_call():
    """Every refusal names its argument and leaves the counters as they were (the next accepted step continues them).
    The pointers are never dereferenced: each call is refused before any CUDA call."""
    L = denoiser._lib()
    p = ctypes.c_void_p(1 << 20)
    nbytes = L.mg_denoise_stream_state_bytes(1024, 256, 4, 700)
    hd = ctypes.c_void_p()

    def create(*args, state=p, size=nbytes):
        return L.mg_denoise_stream_create(ctypes.byref(hd), *args, state, size)

    def err():
        return L.mg_last_error_string()
    assert create(1000, 256, 1024, 4, 700, 0.1) == -1 and b"n_fft" in err()
    assert create(1024, 0, 1024, 4, 700, 0.1) == -1 and b"hop" in err()
    assert create(1024, 512, 256, 4, 700, 0.1) == -1 and b"hop=512" in err()
    assert create(1024, 256, 2048, 4, 700, 0.1) == -1 and b"win_length" in err()
    assert create(1024, 256, 1024, 0, 700, 0.1) == -1 and b"max_sessions" in err()
    assert create(1024, 256, 1024, 257, 700, 0.1) == -1 and b"max_sessions" in err()
    assert create(1024, 256, 1024, 4, 0, 0.1) == -1 and b"max_push_samples" in err()
    assert create(1024, 256, 1024, 4, 700, float("inf")) == -1 and b"strength" in err()
    assert create(1024, 1024, 1024, 4, 700, 0.1) == -1 and b"NOLA" in err()  # hop = n_fft: residue 0 has w[0]^2 = 0
    assert create(1024, 256, 1024, 4, 700, 0.1, state=ctypes.c_void_p((1 << 20) + 16)) == -1 and b"state" in err()
    assert create(1024, 256, 1024, 4, 700, 0.1, state=None) == -1 and b"state" in err()
    assert create(1024, 256, 1024, 4, 700, 0.1, size=nbytes - 1) == -4 and b"state" in err()
    assert L.mg_denoise_stream_state_bytes(1024, 256, 0, 700) == 0 and L.mg_denoise_stream_max_out(1024, 256, 0) == 0
    assert create(1024, 256, 1024, 4, 700, 0.1) == 0
    try:
        out = (ctypes.c_int * 4)()

        def step(counts, flags=None, voice=None, n_voices=1, tables=p, bias=p, audio=p, stride=700, o=p, pcm=False):
            fn = L.mg_denoise_stream_step_pcm16 if pcm else L.mg_denoise_stream_step
            return fn(hd, tables, bias, n_voices, None if voice is None else _ints(voice), audio, stride, _ints(counts),
                      None if flags is None else _ints(flags), len(counts), o, out, None)
        assert step([701]) == -1 and b"in_samples[0] = 701" in err()
        assert step([-1]) == -1 and b"in_samples[0]" in err()
        assert step([5], stride=4) == -1 and b"in_stride" in err()
        assert step([0] * 5) == -1 and b"max_sessions" in err()
        assert step([0], [END]) == -1 and b"no samples" in err()
        assert step([512], [END]) == -1 and b"L = 512" in err()
        assert step([0], [4]) == -1 and b"flags" in err()
        assert step([1], n_voices=0) == -1 and b"n_voices" in err()
        assert step([1], voice=[1]) == -1 and b"voice[0]" in err()
        assert step([1], tables=None) == -1 and b"tables" in err()
        assert step([1], tables=ctypes.c_void_p((1 << 20) + 4)) == -1 and b"tables" in err()
        assert step([1], bias=None) == -1 and b"bias" in err()
        assert step([1], audio=None) == -1 and b"audio_in" in err()
        assert step([1], o=None) == -1 and b"out" in err()
        assert step([1], o=ctypes.c_void_p((1 << 20) + 2)) == -1 and b"out" in err()
        assert step([1], o=ctypes.c_void_p((1 << 20) + 1), pcm=True) == -1 and b"out" in err()
        # nothing moved: a dry step from here sees a fresh handle
        rc, got, nf = _dry(hd, [600, 0, 0, 0])
        assert rc == 0 and got[0] == emitted(1024, 256, 600) and nf == frames_open(1024, 256, 600)
        assert step([1]) == -1 and b"dry_step" in err()
    finally:
        L.mg_denoise_stream_destroy(hd)


def test_end_nola_refusal_leaves_the_counters():
    """A window whose residue sums pass (create accepts it) can still fail torch.istft's NOLA condition at the edge of
    some lengths: the END step at such a length is refused, and the session continues to a length that passes."""
    n, h, w = 1024, 256, 300
    bad = next(L for L in range(n // 2 + 1, 4 * n) if not dm.nola_ok(n, h, w, L))
    good = next(L for L in range(bad + 1, 8 * n) if dm.nola_ok(n, h, w, L))
    lib = denoiser._lib()
    hd = _handle(n, h, w, 1, 8 * n)
    try:
        assert _dry(hd, [bad - 1])[0] == 0
        rc = _dry(hd, [1], [END])[0]
        msg = lib.mg_last_error_string()
        assert rc == -1 and b"NOLA" in msg and b"slot 0" in msg and (b"%d-sample" % bad) in msg
        rc, out, _ = _dry(hd, [good - bad + 1], [END])
        assert rc == 0 and out[0] == good - emitted(n, h, bad - 1)
    finally:
        lib.mg_denoise_stream_destroy(hd)
