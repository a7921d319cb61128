"""Concurrent inference calls on distinct CUDA streams and host threads give exactly their serial results.

The Python objects that drive the kernels keep device scratch between calls: the generator's workspace (activations and
status word), the discriminator's status word and backward workspace, the pinned slot each status word is copied to.
Each is kept per CUDA stream (engine._PerStream).  Every case here first computes each call's serial result on one
stream (held to float64 by the rest of the suite), then issues the calls unordered on separate streams and requires each
result to be bit-identical to its serial one.

Overlap is made by construction, not left to luck: every participating stream first waits on one event, recorded on a
separate gate stream after ``torch.cuda._sleep`` of about 200 ms (a call's first use of a fresh stream allocates
its buffers from the driver, which took the discriminator forward close to 50 ms).  The host enqueues every call while the gate is shut
(each case asserts it still is afterwards), so all queued chains are released at the same instant.  Batches are at
BASELINE config 2 (B = 64, T = 32: one forward is about 1.7 ms on an H100) or the training batch for the
discriminators.  Each case runs once; nothing calls ``torch.cuda.empty_cache``.

Measured on an H100 (700 W) with one workspace per module, as before per-stream scratch: the two-stream and two-thread
generator cases differed from their serial audio by up to 0.0086 (fp32, bf16, forward), 0.012 (ragged) and 0.0086
(threads), with |audio| about 0.06; the regrowth case kept S1's audio but wrote into the sentinel; a code injected into
the first (gated) call was never reported; scale_backward's gx0 differed by 4.3.  The discriminator forwards and the
streaming handles, whose scratch was already per call or per handle, passed there too."""
import threading
import warnings

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth
from kernel_model import gen, gstate, ddev, dstate  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu

GATE_CYCLES = 400_000_000  # torch.cuda._sleep cycles: about 200 ms at the H100's 1.98 GHz boost clock
B, T = 64, 32              # BASELINE config 2


class Gate:
    """An event recorded after a sleep on its own stream: streams that wait on it start together once it fires."""

    def __init__(self):
        torch.cuda.synchronize()  # (the serial references and inputs are complete before anything waits)
        self.stream = torch.cuda.Stream()
        self.event = torch.cuda.Event()
        with torch.cuda.stream(self.stream):
            torch.cuda._sleep(GATE_CYCLES)
            self.event.record()

    def stream_behind(self):
        s = torch.cuda.Stream()
        s.wait_event(self.event)
        return s

    def assert_shut(self):
        assert not self.event.query(), ("the gate opened before every call was enqueued: the enqueue outlasted the sleep, or "
                                        "it synchronised (a kernel's first launch in the process loads its module, which "
                                        "may wait for the device: run each kernel once before the gate)")


def concurrently(calls):
    """Runs each call on its own stream behind one gate; returns their results once all are done."""
    gate = Gate()
    outs = []
    for f in calls:
        with torch.cuda.stream(gate.stream_behind()):
            outs.append(f())
    gate.assert_shut()
    torch.cuda.synchronize()
    return outs


def same(got, ref, what):
    """Bit-identical tensors, or nested lists / tuples of them (None where None)."""
    if isinstance(ref, (list, tuple)):
        assert isinstance(got, (list, tuple)) and len(got) == len(ref), what
        for i, (g, r) in enumerate(zip(got, ref)):
            same(g, r, (what, i))
        return
    assert (got is None) == (ref is None), what
    if ref is not None:
        assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
        assert torch.equal(got, ref), (what, float((got.double() - ref.double()).abs().nan_to_num(float("inf")).max()))


def clone(tree):
    return [clone(t) for t in tree] if isinstance(tree, (list, tuple)) else tree.clone()


def mel(seed, b=B, t=T):
    return torch.from_numpy(synth.mel_input(b, t, seed)).cuda()


LENGTHS = ([int(v) for v in np.random.default_rng(3).integers(1, T + 1, B - 1)] + [T],
           [T] + [int(v) for v in np.random.default_rng(4).integers(1, T + 1, B - 1)])


def generator_call(gen, kind, i, x):  # noqa: F811
    if kind == "forward":
        with torch.no_grad():
            return gen(x)
    if kind == "ragged":
        return gen.generate(x, LENGTHS[i])
    return gen.generate(x, precision=kind)


# ------------------------------------------------------------------------------------------------------------------
# generator
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["fp32", "bf16", "ragged", "forward"])
def test_generator_two_streams_one_module(gen, kind):  # noqa: F811
    """generate (uniform at fp32 and bf16, ragged) and forward under no_grad: two calls of one module with different inputs
    of one shape, unordered on two streams."""
    xs = [mel(11), mel(12)]
    ref = [generator_call(gen, kind, i, x).clone() for i, x in enumerate(xs)]
    assert not torch.equal(ref[0], ref[1])  # (a shared buffer would show)
    got = concurrently([lambda i=i, x=x: generator_call(gen, kind, i, x) for i, x in enumerate(xs)])
    same(got, ref, kind)
    engine.poll_status(wait=True)


def test_generator_two_host_threads(gen):  # noqa: F811
    """Two host threads share one module; each enqueues a forward on its own stream behind the same gate."""
    xs = [mel(21), mel(22)]
    ref = [gen.generate(x).clone() for x in xs]
    gate = Gate()
    ready = threading.Barrier(len(xs))
    got, errors = [None] * len(xs), []

    def serve(i):
        try:
            with torch.cuda.stream(gate.stream_behind()):
                ready.wait()
                got[i] = gen.generate(xs[i])
        except BaseException as e:  # (re-raised on the main thread)
            errors.append(e)

    threads = [threading.Thread(target=serve, args=(i,)) for i in range(len(xs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    gate.assert_shut()
    torch.cuda.synchronize()
    same(got, ref, "threads")
    engine.poll_status(wait=True)


def test_workspace_regrowth_under_queued_work(gen):  # noqa: F811
    """A forward on S0 sizes a module's workspace for a small batch.  A small forward is queued on S1 behind the gate;
    then, on S0, a large forward regrows the workspace and a NaN-filled sentinel of the old workspace's size is
    allocated.  S1's audio must equal its serial result and the sentinel must stay all-NaN: no memory a queued call
    writes may be handed to another tensor."""
    dev = engine.GeneratorDevice("cuda:0")
    dev.packed.copy_(gen._ensure_packed().packed)
    small, small2, large = mel(31, 8), mel(32, 8), mel(33)
    ref_small2, ref_large = gen.generate(small2).clone(), gen.generate(large).clone()
    torch.full((1,), float("nan"), device="cuda")  # (the sentinel's fill kernel, loaded before the gate)
    s0 = torch.cuda.Stream()
    with torch.cuda.stream(s0):
        dev.forward(small)
        old = dev._ws
        old_ptr, old_numel = old.data_ptr(), old.numel()
        del old
    gate = Gate()
    with torch.cuda.stream(gate.stream_behind()):
        y1 = dev.forward(small2)
    with torch.cuda.stream(s0):
        y0 = dev.forward(large)
        assert dev._ws.numel() > old_numel  # regrown
        sentinel = torch.full((old_numel,), float("nan"), device="cuda")
        reused = sentinel.data_ptr() == old_ptr
    gate.assert_shut()
    torch.cuda.synchronize()
    print("regrowth: the sentinel %s the old workspace's block" % ("received" if reused else "did NOT receive"))
    if not reused:
        warnings.warn("the sentinel did not receive the old workspace's block: this run proved nothing about the reuse "
                      "of a freed workspace")
    same([y1, y0], [ref_small2, ref_large], "regrowth")
    assert bool(torch.isnan(sentinel).all()), "a queued forward wrote into memory handed to another tensor"
    engine.poll_status(wait=True)


@pytest.mark.parametrize("codes", [(3, 0), (0, 5)], ids=["first", "second"])
def test_status_of_either_call_in_flight_is_reported(gen, monkeypatch, codes):  # noqa: F811
    """Two forwards in flight on two streams, a timed-out pipeline wait injected into one of them: its status word is
    set on the call's own stream just before the copy to the host is armed (as test_stalled_pipeline_status_is_not_silent
    does by hand).  The first call waits behind the gate, so the second call's copy lands first.  The next
    poll_status(wait=True) must raise exactly once, whichever call carried the code."""
    xs = [mel(41), mel(42)]
    for x in xs:
        gen.generate(x)
    torch.cuda.synchronize()
    engine.poll_status(wait=True)
    pending = list(codes)
    arm = engine._StatusWatch.arm

    def arm_with_code(self, status_word):
        status_word.fill_(pending.pop(0))  # what a timed-out MMA issuer would have left behind (or a healthy 0)
        arm(self, status_word)

    monkeypatch.setattr(engine._StatusWatch, "arm", arm_with_code)
    gate = Gate()
    with torch.cuda.stream(gate.stream_behind()):
        gen.generate(xs[0])
    with torch.cuda.stream(torch.cuda.Stream()):
        gen.generate(xs[1])
    gate.assert_shut()
    assert not pending
    monkeypatch.undo()
    with pytest.raises(engine.EngineError, match="role code %d" % max(codes)):
        engine.poll_status(wait=True)
    engine.poll_status(wait=True)  # the healthy call's copy raises nothing; the error was reported once
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------
# discriminators
# ------------------------------------------------------------------------------------------------------------------
TRAIN_B, SEGMENT = 16, 8192  # BASELINE config 4's batch per GPU and segment length


@pytest.fixture(scope="module")
def msd(dstate):  # noqa: F811
    m = models.MultiScaleDiscriminator()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in dstate.items()})
    return m.cuda().eval()


@pytest.fixture(scope="module")
def disc(dstate):  # noqa: F811
    d = models.Discriminator()
    d.load_state_dict({k[len("discriminators.0."):]: torch.from_numpy(v) for k, v in dstate.items()
                       if k.startswith("discriminators.0.")})
    return d.cuda().eval()


def audio(seed, b=TRAIN_B):
    return torch.from_numpy(synth.audio_input(b, SEGMENT, seed)).cuda()


def test_discriminator_forwards_two_streams(msd, disc):
    """MultiScaleDiscriminator (real and generated batches) and the stand-alone Discriminator, each called twice with
    different audio, unordered on two streams: every logit and feature map as in the serial calls."""
    pairs = [(audio(51), audio(52)), (audio(53), audio(54))]
    singles = [audio(55, 2 * TRAIN_B), audio(56, 2 * TRAIN_B)]
    with torch.no_grad():
        ref_msd = [clone(msd(y, y_hat)) for y, y_hat in pairs]  # (y_d_rs, y_d_gs, fmap_rs, fmap_gs)
        ref_disc = [clone(disc(x)) for x in singles]            # (logits, fmap)
        same(concurrently([lambda p=p: msd(*p) for p in pairs]), ref_msd, "MultiScaleDiscriminator")
        same(concurrently([lambda x=x: disc(x) for x in singles]), ref_disc, "Discriminator")
    msd._dev.check_status()
    disc._dev.check_status()
    engine.poll_status(wait=True)


def test_scale_backward_two_streams(ddev):  # noqa: F811
    """DiscriminatorDevice.scale_backward of every scale on one forward's maps with two different upstream gradients,
    unordered on two streams: every dW, db and gx0 as in the serial calls."""
    Bt = 2 * TRAIN_B
    y = audio(61, Bt)
    fm = ddev.forward(y)
    x0 = [y]
    for k in range(2):  # the scales' inputs: MultiScaleDiscriminator's AvgPool chain
        x0.append(torch.nn.functional.avg_pool1d(x0[-1], 4, 2 if k == 0 else 4, padding=2))
    gens = [torch.Generator(device="cuda").manual_seed(70 + i) for i in range(2)]
    grads = [[[torch.randn(f.shape, device="cuda", generator=g) for f in fm[s]] for s in range(3)] for g in gens]

    def backward(i):
        return [ddev.scale_backward(s, x0[s], fm[s], grads[i][s], True) for s in range(3)]
    ref = [backward(i) for i in range(2)]
    assert not torch.equal(ref[0][0][1][5], ref[1][0][1][5])
    got = concurrently([lambda i=i: backward(i) for i in range(2)])
    same(got, ref, "scale_backward")
    ddev.check_status()


# ------------------------------------------------------------------------------------------------------------------
# streaming handles
# ------------------------------------------------------------------------------------------------------------------
def test_stream_handles_two_streams(gen):  # noqa: F811
    """Two GeneratorStream handles of one module step on two gated streams, steps interleaved on the host and never
    synchronised: each session's concatenated output equals its whole forward.  (The schedule is drawn up front, like
    test_gen_stream_gpu's, but without its per-step read-backs, which would order the streams.)"""
    P, S = 16, 4
    rng = np.random.default_rng(81)
    lens = [[int(v) for v in rng.integers(1, 6 * P, S)] for _ in range(2)]
    mels = [[mel(900 + 10 * h + i, 1, L) for i, L in enumerate(lens[h])] for h in range(2)]
    ref = [[gen.generate(m)[0, 0].clone() for m in mels[h]] for h in range(2)]
    handles = [gen.stream(S, P) for _ in range(2)]
    warm = gen.stream(S, P)  # the stream's own kernels, loaded before the gate
    warm.step([mels[0][0][0, :, :P]], end=[True])
    warm.check_status()
    pushes = [[[int(v) for v in rng.integers(0, P + 1, 64)] for _ in range(S)] for _ in range(2)]
    gate = Gate()
    streams = [gate.stream_behind() for _ in range(2)]
    pos = [[0] * S for _ in range(2)]
    out = [[[] for _ in range(S)] for _ in range(2)]
    done = [[False] * S for _ in range(2)]
    k = 0
    while not all(all(d) for d in done):
        for h in range(2):
            chunks, end = [], []
            for i in range(S):
                if done[h][i]:
                    chunks.append(None)
                    end.append(False)
                    continue
                n = min(pushes[h][i][k], lens[h][i] - pos[h][i])
                chunks.append(mels[h][i][0, :, pos[h][i]:pos[h][i] + n])
                pos[h][i] += n
                end.append(pos[h][i] == lens[h][i])
            with torch.cuda.stream(streams[h]):
                got = handles[h].step(chunks, end=end)
            for i in range(S):
                if not done[h][i]:
                    out[h][i].append(got[i][0])
                    done[h][i] = end[i]
        k += 1
    gate.assert_shut()
    torch.cuda.synchronize()
    for h in range(2):
        for i in range(S):
            same(torch.cat(out[h][i]), ref[h][i], ("handle", h, "session", i, "frames", lens[h][i]))
        with torch.cuda.stream(streams[h]):
            handles[h].check_status()


# ------------------------------------------------------------------------------------------------------------------
# the lazy pack of a module's first call
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["Generator", "MultiScaleDiscriminator"])
def test_first_call_on_another_stream_reads_the_packed_weights(gen, msd, gstate, dstate, which):  # noqa: F811
    """A module's first call packs its weights on its own stream.  That call waits behind the gate; a second call on
    another stream, not gated, must still read the packed weights, not the blob as it was before the pack (NaN here)."""
    if which == "Generator":
        m = models.Generator()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in gstate.items()})
        m._dev = engine.GeneratorDevice("cuda:0")
        xs = [mel(91), mel(92)]
        run, serial = (lambda mod, x: mod.generate(x)), gen
    else:
        m = models.MultiScaleDiscriminator()
        m.load_state_dict({k: torch.from_numpy(v) for k, v in dstate.items()})
        m._dev = engine.DiscriminatorDevice("cuda:0")
        xs = [(audio(93), audio(94)), (audio(95), audio(96))]
        run, serial = (lambda mod, x: mod(*x)), msd
    m = m.cuda().eval()
    m._dev.packed.fill_(float("nan"))
    with torch.no_grad():
        ref = [clone(run(serial, x)) for x in xs]
        gate = Gate()
        with torch.cuda.stream(gate.stream_behind()):
            first = run(m, xs[0])  # packs, then runs, behind the gate
        with torch.cuda.stream(torch.cuda.Stream()):
            second = run(m, xs[1])
        gate.assert_shut()
        torch.cuda.synchronize()
    same([first, second], ref, which)
    engine.poll_status(wait=True)
