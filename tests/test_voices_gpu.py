"""Many voices in one forward on the GPU (models.generate_voices / mg_gen_forward_voices): every item equals its own
single-voice forward bit for bit, whatever the order of the voices, wherever a voice change falls against the tiles.

Every voice comes from a different seed, so a tile that read its neighbour's blob would show in its items' audio.  At a
voice change the conv_pre and ConvT launchers start the new voice at a tile border; the border tests put the previous
voice's last row one before, at and one after a border of each of those kernels (tile sizes parsed from the
configurations the library reports), and one batch has more stride-2 ConvT tiles than SMs, so persistent CTAs walk from
one voice into another and reload the layer's weights."""
import re

import numpy as np
import pytest
import torch

from melgan_multi_b200 import engine, models, synth
from kernel_model import FILL, fill_faults, guard_ok, nan_buffer, ragged_batch

pytestmark = pytest.mark.gpu
SEEDS = (1234, 2718, 3141, 5772)


@pytest.fixture(scope="module")
def voices():
    out = []
    for seed in SEEDS:
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(seed).items()})
        out.append(g.cuda().eval())
    return out


def check_voices(voices, mel, lens, voice, precision="fp32"):
    audio = models.generate_voices(voices, mel, voice, lens, precision=precision)
    assert audio.shape == (len(lens), 1, 256 * mel.shape[2])
    voices[0]._dev.check_status(len(lens), mel.shape[2])
    for i, (L, v) in enumerate(zip(lens, voice)):
        own = voices[v].generate(mel[i:i + 1, :, :L].contiguous(), precision=precision)
        assert torch.equal(audio[i:i + 1, :, :256 * L], own), (i, L, v, precision)
        assert bool((audio[i, :, 256 * L:] == 0).all()), (i, L, v)
    return audio


BATCHES = {
    "sorted": ([9, 3, 33, 1, 20, 7, 64, 2], [0, 0, 0, 1, 1, 2, 2, 3]),
    "interleaved": ([9, 3, 33, 1, 20, 7, 64, 2], [0, 1, 0, 1, 0, 1, 0, 1]),
    "own_voice": ([17, 5, 40, 1], [0, 1, 2, 3]),
    "equal_lengths": ([24] * 8, [0, 0, 1, 1, 1, 2, 3, 3]),
}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("kind", sorted(BATCHES))
def test_per_item_bit_identity(voices, kind, precision):
    lens, voice = BATCHES[kind]
    mel = ragged_batch(lens, 40)
    check_voices(voices, mel, lens, voice, precision)


def _tiles():
    """{kernel: (tile rows, units of an item of L mel frames)} of conv_pre and the three ConvT kernels of the default chain."""
    L = engine.lib()
    m = re.fullmatch(r"conv_rows_tc_kernel<ConvCfg<80,512,(\d+),(\d+),\d+>>", L.mg_gen_conv_pre_config().decode())
    pad, rows = int(m.group(1)) // 2, int(m.group(2))
    out = {"pre": (rows, lambda T, pad=pad: T + pad)}
    for s, scale in ((0, 1), (1, 8), (2, 64)):
        name = L.mg_gen_convt_config(s).decode()
        rows = int(re.fullmatch(r"\w+<(?:Up|Stream)Cfg<%d,(\d+)(?:,\d+)+>>" % s, name).group(1))
        out["up%d" % s] = (rows, lambda T, scale=scale: scale * T + 1)  # Lin + 1 virtual rows per item
    return out


def _segment(rows, units, d):
    """Mel lengths of one voice's items (n - 1 of one frame, then one of L; the fewest items) whose units end d rows past
    a tile border."""
    for n in range(1, 2 * rows + 2):
        for L in range(1, 160):
            if ((n - 1) * units(1) + units(L) - d) % rows == 0:
                return [1] * (n - 1) + [L]
    raise AssertionError((rows, d))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("kernel", ["pre", "up0", "up1", "up2"])
def test_voice_change_at_tile_borders(voices, kernel, precision):
    rows, units = _tiles()[kernel]
    lens, voice = [], []
    for k, d in enumerate((-1, 0, 1)):  # each voice starts a tile: the next change is placed from 0 again
        seg = _segment(rows, units, d)
        lens += seg
        voice += [k] * len(seg)
    lens += [3, 11]
    voice += [3, 3]
    assert sum(lens) < 1024  # one batch slice (generator_tc_slices): unit offsets count from the batch's start
    mel = ragged_batch(lens, 60)
    check_voices(voices, mel, lens, voice, precision)


def test_persistent_convt_crosses_voices(voices):
    rng = np.random.default_rng(5)
    lens = [int(v) for v in rng.integers(1, 40, 40)]
    voice = [int(v) for v in rng.integers(0, len(SEEDS), 40)]
    rows, units = _tiles()["up2"]
    assert sum(lens) < 1024 and sum(units(L) for L in lens) > 2 * 132 * rows  # one slice, over two tiles per SM
    mel = ragged_batch(lens, 80)
    check_voices(voices, mel, lens, voice)


@pytest.mark.parametrize("lengths", [None, [5, 32, 1, 17]])
def test_one_voice_equals_generate(voices, lengths):
    g = voices[0]
    B, T = 4, 32
    mel = torch.from_numpy(synth.mel_input(B, T, 3)).cuda()
    ref = g.generate(mel, lengths)
    assert torch.equal(models.generate_voices([g], mel, [0] * B, lengths), ref)
    assert torch.equal(models.generate_voices(voices, mel, [2] * B, lengths), voices[2].generate(mel, lengths))


def test_outputs_written_and_guarded(voices):
    lens, voice = [9, 130, 1, 64, 33], [1, 0, 3, 3, 2]
    B, T = len(lens), max(lens)
    mel = ragged_batch(lens, 90)
    n = B * 256 * T
    buf = nan_buffer(n)
    devs = [g._ensure_packed() for g in voices]
    y = devs[0].forward_voices(devs, mel, voice, lens, out=buf[:n].view(B, 1, 256 * T))
    devs[0].check_status(B, T)
    assert guard_ok(buf, n)
    assert fill_faults(y, buf, lens, 256, zero_tail=True) == set()
    assert not bool((y.view(torch.int32) == FILL).any())
    ref = models.generate_voices(voices, mel, voice, lens)
    assert torch.equal(y, ref)


def test_refusals(voices):
    mel = ragged_batch([4, 2], 10)
    with pytest.raises(engine.EngineError, match="voice ids"):
        models.generate_voices(voices[:2], mel, [0, 2])
    with pytest.raises(engine.EngineError, match="CUDA"):
        models.generate_voices(voices[:2], mel.cpu(), [0, 1])
    cpu = models.Generator()
    with pytest.raises(engine.EngineError):
        models.generate_voices([voices[0], cpu], mel, [0, 1])


def test_streams_equal_serial(voices):
    calls = [(([30, 4, 12, 1, 50], [0, 2, 2, 1, 3]), 100), (([7, 7, 64, 2], [3, 1, 0, 0]), 200)]
    mels = [ragged_batch(lens, seed) for (lens, _v), seed in calls]
    serial = [models.generate_voices(voices, m, v, lens) for m, ((lens, v), _s) in zip(mels, calls)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in calls]
    outs = [None] * len(calls)
    cur = torch.cuda.current_stream()
    for k, (m, ((lens, v), _s)) in enumerate(zip(mels, calls)):
        streams[k].wait_stream(cur)
        with torch.cuda.stream(streams[k]):
            outs[k] = models.generate_voices(voices, m, v, lens)
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for a, b in zip(outs, serial):
        assert torch.equal(a, b)
