"""Every forward runs on its parameters' current values, however they were changed.

The modules fold weight norm into a packed blob once and fold again only when some parameter's (data_ptr, _version)
changed (models.Generator._ensure_packed and the discriminators' _engine_forward).  Each case here packs a module, changes
its weights by one route, and compares the next output with that of a new module loaded with the same state_dict.  Both
run the same kernels on the same packed values, so they must agree bit for bit; each case also requires that the
output changed, or a route that did nothing would pass.

Three routes leave the key as it was: in-place writes through p.data, a replayed CUDA graph of an optimizer step (the
capture bumped the versions once, the replays write without the host), and AveragedModel's EMA update, whose
torch._foreach_lerp_ with a scalar weight bumps no version counter on CUDA.  For those the routes call repack(), and the
same comparison holds after it.  torch's fused Adam bumps no version counter either; models bumps them after every
fused optimizer step, so that route needs no repack()."""
import functools

import pytest
import torch
from torch.nn.utils import parameters_to_vector, remove_weight_norm, vector_to_parameters
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

from melgan_multi_b200 import models, synth
from melgan_multi_b200.optim import Adam as MultiTensorAdam

pytestmark = pytest.mark.gpu
VOICE_SEEDS = (1234, 2718, 3141)


@functools.lru_cache(maxsize=None)
def _gstate(seed):
    return {k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()}


@functools.lru_cache(maxsize=None)
def _dstate(seed):
    return {k: torch.from_numpy(v) for k, v in synth.discriminator_state(seed).items()}


def _new(cls, state):
    # built under no_grad: weight_norm's initial `weight` attribute then has no autograd history, which copy.deepcopy
    # (AveragedModel) refuses
    with torch.no_grad():
        m = cls()
    if state is not None:
        m.load_state_dict(state)
    return m.cuda()


def new_generator(seed=1234):
    return _new(models.Generator, _gstate(seed))


def new_msd(seed=4321):
    return _new(models.MultiScaleDiscriminator, _dstate(seed))


def fresh(m):
    """A new module of m's class loaded with m's state_dict: it packs those values at its first call."""
    f = _new(type(m), None)
    f.load_state_dict(m.state_dict())
    return f


def mel(B, T, seed):
    return torch.from_numpy(synth.mel_input(B, T, seed)).cuda()


def audio(B, L, seed):
    return torch.from_numpy(synth.audio_input(B, L, seed)).cuda()


def check_updated(before, after, ref):
    """after changed from before, and equals ref bit for bit (tensors or lists of tensors)."""
    before, after, ref = ([t] if torch.is_tensor(t) else list(t) for t in (before, after, ref))
    assert any(not torch.equal(a, b) for a, b in zip(after, before)), "the update did not change the output"
    for i, (a, r) in enumerate(zip(after, ref)):
        assert torch.equal(a, r), (i, float((a.double() - r.double()).abs().max()))


# -- update routes ---------------------------------------------------------------------------------------------------
# ROUTES[name](m, seed) -> (module, apply): set-up that may precede the first pack, then the module to call (m, or the
# averaged copy of the EMA route) and apply(), which changes that module's weights.

def ratios(m, seed):
    """1 + 0.02 n per parameter of m, n seeded standard normal: a nearby state that moves every layer's fold (a scalar
    factor on weight_v would leave the fold as it was)."""
    gen = torch.Generator().manual_seed(seed)
    return [(1 + 0.02 * torch.randn(p.shape, generator=gen)).to(p.device) for p in m.parameters()]


def grads(m, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(p.shape, generator=gen).to(p.device) for p in m.parameters()]


def _no_grad_op(op):
    def route(m, seed):
        rs = ratios(m, seed)

        def apply():
            with torch.no_grad():
                for p, r in zip(m.parameters(), rs):
                    op(p, r)
        return m, apply
    return route


def _foreach(m, seed):
    rs = ratios(m, seed)

    def apply():
        with torch.no_grad():
            torch._foreach_mul_(list(m.parameters()), rs)
    return m, apply


def _load_state_dict(assign):
    def route(m, seed):
        rs = ratios(m, seed)

        def apply():
            m.load_state_dict({k: p.detach() * r for (k, p), r in zip(m.named_parameters(), rs)}, assign=assign)
        return m, apply
    return route


def _assign(p, r):
    p.data = p.detach() * r


def _data_assign(m, seed):
    rs = ratios(m, seed)

    def apply():
        for p, r in zip(m.parameters(), rs):
            _assign(p, r)
    return m, apply


def _vector_to_parameters(m, seed):
    rs = torch.cat([r.reshape(-1) for r in ratios(m, seed)])

    def apply():
        vector_to_parameters(parameters_to_vector(m.parameters()).detach() * rs, m.parameters())
    return m, apply


def report_addresses(what, before, m):
    same = sum(a == p.data_ptr() for a, p in zip(before, m.parameters()))
    print("%s: %d of %d parameters came back at the address of the last pack" % (what, same, len(before)))


def _data_assign_twice(m, seed):
    """Two rounds of p.data = t with no call between: the second round's storage may land where the packed one was."""
    r1, r2 = ratios(m, seed), ratios(m, seed + 1)

    def apply():
        before = [p.data_ptr() for p in m.parameters()]
        for rs in (r1, r2):
            for p, r in zip(m.parameters(), rs):
                _assign(p, r)
        report_addresses("two rounds of p.data = t", before, m)
    return m, apply


def _vector_to_parameters_twice(m, seed):
    """The module packs while its parameters are views of one vector; two more vectors follow with no call between.
    Each vector is one allocation, and when the last one is made the packed vector is the only free block of its size,
    so the caching allocator is likely to put the parameters back at the packed addresses."""
    rs = [torch.cat([r.reshape(-1) for r in ratios(m, seed + k)]) for k in range(3)]

    def new_vector(r):
        vec = parameters_to_vector(m.parameters()).detach()
        vec.mul_(r)
        vector_to_parameters(vec, m.parameters())
    new_vector(rs[0])

    def apply():
        before = [p.data_ptr() for p in m.parameters()]
        new_vector(rs[1])
        new_vector(rs[2])
        report_addresses("two vector_to_parameters", before, m)
    return m, apply


def _optimizer(make):
    def route(m, seed):
        opt = make(m.parameters())
        gs = grads(m, seed)

        def apply():
            for p, g in zip(m.parameters(), gs):
                p.grad = g
            opt.step()
        return m, apply
    return route


def _ema(src, seed):
    ema = AveragedModel(src, multi_avg_fn=get_ema_multi_avg_fn(0.5))
    ema.update_parameters(src)  # the first update copies
    m = ema.module
    rs = ratios(src, seed)

    def apply():
        with torch.no_grad():
            torch._foreach_mul_(list(src.parameters()), rs)
        ema.update_parameters(src)  # _foreach_lerp_ with a scalar weight: on CUDA no version counter moves
        m.repack()
    return m, apply


def _cpu_round_trip(write):
    def route(m, seed):
        rs = ratios(m, seed)

        def apply():
            before = [p.data_ptr() for p in m.parameters()]
            m.cpu()
            with torch.no_grad():
                for p, r in zip(m.parameters(), rs):
                    write(p, r.cpu())
            m.cuda()
            report_addresses("CPU round trip", before, m)
        return m, apply
    return route


def _data_inplace(m, seed):
    rs = ratios(m, seed)

    def apply():
        for p, r in zip(m.parameters(), rs):
            p.data.mul_(r)  # leaves p._version as it was
        m.repack()
    return m, apply


def _graph_adam(m, seed):
    ps = list(m.parameters())
    static = grads(m, seed)
    for p, g in zip(ps, static):
        p.grad = g
    opt = torch.optim.Adam(ps, lr=1e-3, capturable=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        opt.step()  # warm-up: the optimizer's state is created outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()

    def apply():
        for p, g in zip(ps, static):  # the gradients the graph reads
            p.grad = g
        graph.replay()  # writes the parameters; no version counter moves
        m.repack()
    return m, apply


ROUTES = {
    "add_": _no_grad_op(lambda p, r: p.add_(p * (r - 1))),
    "copy_": _no_grad_op(lambda p, r: p.copy_(p * r)),
    "mul_": _no_grad_op(lambda p, r: p.mul_(r)),
    "foreach_mul_": _foreach,
    "load_state_dict": _load_state_dict(False),
    "load_state_dict_assign": _load_state_dict(True),
    "data_assign": _data_assign,
    "data_assign_twice": _data_assign_twice,
    "vector_to_parameters": _vector_to_parameters,
    "vector_to_parameters_twice": _vector_to_parameters_twice,
    "adam_for_loop": _optimizer(lambda ps: torch.optim.Adam(ps, lr=1e-3, foreach=False)),
    "adam_foreach": _optimizer(lambda ps: torch.optim.Adam(ps, lr=1e-3, foreach=True)),
    "adam_fused": _optimizer(lambda ps: torch.optim.Adam(ps, lr=1e-3, fused=True)),
    "adam_multi_tensor": _optimizer(lambda ps: MultiTensorAdam(ps, lr=1e-3)),
    "ema": _ema,
    "cpu_round_trip_mul_": _cpu_round_trip(lambda p, r: p.mul_(r)),
    "cpu_round_trip_data_assign": _cpu_round_trip(_assign),
    "data_inplace": _data_inplace,
    "graph_adam": _graph_adam,
}
INVISIBLE = ("data_inplace", "graph_adam", "ema")  # the routes that call repack()


# -- Generator ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("route", sorted(ROUTES))
def test_generator_forward(route):
    m, apply = ROUTES[route](new_generator(), 11)
    x = mel(2, 12, 12)
    with torch.no_grad():
        y0 = m(x)
        apply()
        y1 = m(x)
        check_updated(y0, y1, fresh(m)(x))


LENGTHS = [16, 5, 1, 11]
PATHS = {
    "generate": lambda g, x: g.generate(x),
    "ragged": lambda g, x: g.generate(x, LENGTHS),
    "bf16": lambda g, x: g.generate(x, precision="bf16"),
    "int16": lambda g, x: g.generate(x, dtype=torch.int16),
}
PATH_ROUTE = {"generate": "load_state_dict", "ragged": "vector_to_parameters", "bf16": "add_", "int16": "adam_foreach"}


@pytest.mark.parametrize("path,route", [(p, r) for p in sorted(PATHS) for r in (PATH_ROUTE[p], "data_inplace")])
def test_generator_inference_paths(path, route):
    m, apply = ROUTES[route](new_generator(), 21)
    x = mel(4, 16, 22)
    run = PATHS[path]
    y0 = run(m, x)
    apply()
    check_updated(y0, run(m, x), run(fresh(m), x))


@pytest.mark.parametrize("update", ["adam", "data_sgd"])
def test_generator_training_step(update):
    """The autograd forward after a training step: forward, loss, backward, then an optimizer step or a sign-SGD step
    written through p.data (followed by repack())."""
    g = new_generator().train()
    x = mel(2, 8, 31)
    y0 = g(x)
    y0.square().mean().backward()
    if update == "adam":
        torch.optim.Adam(g.parameters(), lr=1e-3).step()
    else:
        for p in g.parameters():
            p.data.add_(p.grad.sign(), alpha=-1e-3)
        g.repack()
    y1 = g(x)
    assert y1.requires_grad
    check_updated(y0.detach(), y1.detach(), fresh(g)(x).detach())


def stream_utterances(st, mels, voice=None):
    """Each mel [1, 80, T] through its own slot of st, max_push_frames a step, END with its last frames: the audio
    [1, 1, 256 T] of each."""
    P = st.max_push_frames
    pos, outs, done = [0] * len(mels), [[] for _ in mels], [False] * len(mels)
    while not all(done):
        chunks, end = [], []
        for i, x in enumerate(mels):
            if done[i]:
                chunks.append(None)
                end.append(False)
                continue
            n = min(P, x.shape[2] - pos[i])
            chunks.append(x[0, :, pos[i]:pos[i] + n])
            pos[i] += n
            end.append(pos[i] == x.shape[2])
        for i, a in enumerate(st.step(chunks, end=end, voice=voice)):
            outs[i].append(a)
        done = [d or e for d, e in zip(done, end)]
    return [torch.cat(o, dim=1).view(1, 1, -1) for o in outs]


@pytest.mark.parametrize("route", ["add_", "data_inplace"])
def test_stream_sessions_opened_after_a_change(route):
    """Weights changed between two steps of one handle: sessions opened after the change equal the new weights' whole
    forward.  (No session is open across the change.)"""
    g = new_generator()
    _, apply = ROUTES[route](g, 41)
    st = g.stream(max_sessions=2, max_push_frames=4)
    a, b, c = mel(1, 13, 42), mel(1, 9, 43), mel(1, 16, 44)
    (out_a,) = stream_utterances(st, [a])
    assert torch.equal(out_a, g.generate(a))
    old_b = g.generate(b)
    apply()
    out_b, out_c = stream_utterances(st, [b, c])
    f = fresh(g)
    check_updated(old_b, out_b, f.generate(b))
    assert torch.equal(out_c, f.generate(c))


@pytest.mark.parametrize("route", ["copy_", "data_inplace"])
def test_generate_voices_one_voice_updated(route):
    """Only voice 1 changes: its items follow it, the other voices' items stay bit-identical."""
    voices = [new_generator(s) for s in VOICE_SEEDS]
    _, apply = ROUTES[route](voices[1], 51)
    lens, voice = [12, 5, 9, 12], [0, 1, 2, 1]
    x = mel(4, 12, 52)
    y0 = models.generate_voices(voices, x, voice, lens)
    apply()
    y1 = models.generate_voices(voices, x, voice, lens)
    assert torch.equal(y1, models.generate_voices([voices[0], fresh(voices[1]), voices[2]], x, voice, lens))
    for i, v in enumerate(voice):
        assert torch.equal(y1[i], y0[i]) == (v != 1), (i, v)


@pytest.mark.parametrize("route", ["mul_", "data_inplace"])
def test_stream_voices_one_voice_updated(route):
    voices = [new_generator(s) for s in VOICE_SEEDS]
    _, apply = ROUTES[route](voices[1], 61)
    st = models.stream_voices(voices, max_sessions=3, max_push_frames=4)
    mels = [mel(1, T, 62 + i) for i, T in enumerate((11, 14, 7))]
    before = stream_utterances(st, mels, voice=[0, 1, 2])
    for v in range(3):
        assert torch.equal(before[v], voices[v].generate(mels[v])), v
    apply()
    after = stream_utterances(st, mels, voice=[0, 1, 2])
    assert torch.equal(after[0], before[0]) and torch.equal(after[2], before[2])
    check_updated(before[1], after[1], fresh(voices[1]).generate(mels[1]))


@pytest.mark.parametrize("route", ["add_", "data_inplace"])
def test_repack_on_one_stream_forward_on_another(route):
    """The update and the re-pack run on stream s1, held back by a device sleep; the next forward runs on s2 after
    s2.wait_stream(s1) and reads the new pack (engine._PackedBlob orders every read of the blob after its pack)."""
    g = new_generator()
    _, apply = ROUTES[route](g, 71)
    x = mel(2, 12, 72)
    with torch.no_grad():
        y0 = g(x)
        s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
        s1.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s1):
            torch.cuda._sleep(100_000_000)
            apply()
            g(x)  # re-packs on s1
        s2.wait_stream(s1)
        with torch.cuda.stream(s2):
            y1 = g(x)
        torch.cuda.current_stream().wait_stream(s2)
        check_updated(y0, y1, fresh(g)(x))


def test_remove_weight_norm_fails_loudly():
    """The modules read weight_g / weight_v (tests/golden/module_abi.json); without them a call raises."""
    g = new_generator()
    remove_weight_norm(g.ups[0])
    with pytest.raises(AttributeError, match="weight_v"):
        g(mel(1, 4, 1))


# -- discriminators ----------------------------------------------------------------------------------------------------

def msd_step(m, y, y_hat):
    """Forward on (y, y_hat), discriminator_loss, backward: every feature map, then every parameter's gradient (the
    backward reads the folded weights the forward packed)."""
    m.zero_grad(set_to_none=True)
    dr, dg, fr, fg = m(y, y_hat)
    loss, _, _ = models.discriminator_loss(dr, dg)
    loss.backward()
    return [f.detach() for maps in fr + fg for f in maps] + [p.grad for p in m.parameters()]


@pytest.mark.parametrize("route", ["add_", "load_state_dict_assign", "vector_to_parameters_twice", "adam_fused",
                                   "adam_multi_tensor", "data_inplace", "graph_adam"])
def test_msd_forward_and_gradients(route):
    m, apply = ROUTES[route](new_msd(), 81)
    y, y_hat = audio(2, 2048, 82), audio(2, 2048, 83)
    before = msd_step(m, y, y_hat)
    apply()
    check_updated(before, msd_step(m, y, y_hat), msd_step(fresh(m), y, y_hat))


def disc_outputs(d, x):
    logits, fmap = d(x)
    return [logits] + fmap


def msd_outputs(m, y, y_hat):
    _, _, fr, fg = m(y, y_hat)
    return [f for maps in fr + fg for f in maps]


@pytest.mark.parametrize("via", ["msd", "disc"])
@pytest.mark.parametrize("route", ["adam_foreach", "data_inplace"])
def test_discriminator_shared_with_msd(via, route):
    """A stand-alone Discriminator that is also scale 0 of an MSD: the two pack separately, keyed on the same
    parameters.  Update through one, then call the other first."""
    msd = new_msd()
    d = msd.discriminators[0]
    _, apply = ROUTES[route](msd if via == "msd" else d, 91)
    y, y_hat, x = audio(2, 2048, 92), audio(2, 2048, 93), audio(2, 2048, 94)
    with torch.no_grad():
        d0, m0 = disc_outputs(d, x), msd_outputs(msd, y, y_hat)
        apply()
        if route in INVISIBLE:
            msd.repack()  # covers its Discriminators too
        if via == "msd":
            d1 = disc_outputs(d, x)
            m1 = msd_outputs(msd, y, y_hat)
        else:
            m1 = msd_outputs(msd, y, y_hat)
            d1 = disc_outputs(d, x)
        check_updated(d0, d1, disc_outputs(fresh(d), x))
        check_updated(m0, m1, msd_outputs(fresh(msd), y, y_hat))
