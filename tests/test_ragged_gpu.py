"""Ragged batches on the GPU (Generator.generate / mg_gen_forward_ragged): every item of one forward over utterances of
different lengths equals that utterance's own forward bit for bit, and the audio past its end is exactly 0.

The kernels place their tiles per item and apply each item's zero padding at the item's own end, so the per-item
arithmetic of a ragged batch is the single-item forward's.  The lengths include the stage-0 and stage-1 ResBlock
cluster and CTA-rank borders (kernel_model.lengths) mapped back to mel frames, so a border sits at or next
to an item's end; the mel past every length is NaN, which any read would carry into the audio."""
import numpy as np
import pytest
import torch

import cases
from conftest import rel_errors
from melgan_multi_b200 import engine, synth
from kernel_model import gen, gstate  # noqa: F401 (fixtures)
from kernel_model import check_items, cluster_border_frames, ragged_batch

pytestmark = pytest.mark.gpu
TOL = 1e-4  # test_generator_gpu's bound against the reference


def test_per_item_bit_identity(gen):
    lens = sorted({1, 2, 3, 7, 31, 32, 33, 1000} | set(cluster_border_frames()))
    assert len(lens) <= 256  # MG_GEN_RAGGED_MAX_B
    rng = np.random.default_rng(7)
    lens = [int(v) for v in rng.permutation(lens)]
    mel = ragged_batch(lens, 100)
    audio = gen.generate(mel, lens)
    check_items(gen, mel, lens, audio)
    assert not bool(torch.isnan(audio).any())


def test_several_slices(gen):
    rng = np.random.default_rng(11)
    lens = [int(v) for v in rng.integers(20, 201, 48)]
    assert sum(lens) >= 4 * 512  # generator_tc_slices: four chains (>= 512 frames each)
    mel = ragged_batch(lens, 300)
    check_items(gen, mel, lens, gen.generate(mel, torch.tensor(lens)))


@pytest.mark.parametrize("mask", [0, 2, 4, 6, 8, 10, 12, 14])
def test_every_chain(gen, mask):
    lens = [5, 1, 33, 12, 2]
    mel = ragged_batch(lens, 500 + mask)
    engine.check(engine.lib().mg_gen_set_pipeline(mask))
    try:
        check_items(gen, mel, lens, gen.generate(mel, lens))
    finally:
        engine.check(engine.lib().mg_gen_set_pipeline(-1))


@pytest.mark.parametrize("B,T", [(64, 32), (3, 33)])
def test_uniform_lengths_equal_forward(gen, B, T):
    mel = torch.from_numpy(synth.mel_input(B, T, 9)).cuda()
    with torch.no_grad():
        ref = gen(mel)
    assert torch.equal(gen.generate(mel, [T] * B), ref)
    gen._dev.check_status(B, T)


def test_goldens_in_one_batch(gen, golden):
    items = []
    for case in cases.GEN_CASES:
        B, T, seed, realistic = case
        x = synth.mel_input(B, T, seed, realistic)
        items += [(x[b], case, b) for b in range(B)]
    items.append((synth.mel_input(1, 1000, 0)[0], None, 0))
    lens = [x.shape[1] for x, _c, _b in items]
    mel = np.full((len(items), 80, max(lens)), np.nan, np.float32)
    for i, (x, _c, _b) in enumerate(items):
        mel[i, :, :x.shape[1]] = x
    y = gen.generate(torch.from_numpy(mel).cuda(), lens).cpu().numpy()
    gen._dev.check_status(len(lens), max(lens))
    for i, (x, case, b) in enumerate(items):
        got = y[i, 0, :256 * lens[i]]
        if case is None:
            scale = np.abs(golden["gen_T1000_mid"]).max()
            assert np.abs(got[:4096] - golden["gen_T1000_head"]).max() < TOL * scale
            assert np.abs(got[128000 - 2048:128000 + 2048] - golden["gen_T1000_mid"]).max() < TOL * scale
            assert np.abs(got[-4096:] - golden["gen_T1000_tail"]).max() < TOL * scale
        else:
            m, l2 = rel_errors(got, golden[cases.gen_key(*case)][b, 0])
            assert m < TOL and l2 < TOL, (case, b, m, l2)


def test_stage_taps(gen):
    lens = [3, 17, 1, 9]
    T = max(lens)
    mel = ragged_batch(lens, 700)
    engine.check(engine.lib().mg_gen_set_pipeline(0))
    try:
        gen.generate(mel, lens)
        taps = [gen._dev.stage_output(w, len(lens), T) for w in range(4)]
        gen._dev.check_status(len(lens), T)
        with torch.no_grad():
            for i, L in enumerate(lens):
                gen(mel[i:i + 1, :, :L].contiguous())
                for w, scale in enumerate((1, 8, 64, 128)):
                    own = gen._dev.stage_output(w, 1, L)
                    assert torch.equal(taps[w][i:i + 1, :, :scale * L], own), (i, L, w)
    finally:
        engine.check(engine.lib().mg_gen_set_pipeline(-1))


def test_host_engine_equals_device_path(gen, gstate):
    lens = [40, 7, 1, 64, 33]
    mel = ragged_batch(lens, 900)
    ref = gen.generate(mel, lens).cpu().numpy()
    gen._dev.check_status(len(lens), max(lens))
    host = engine.GeneratorHost(2, 8)
    host.load_state(gstate)
    try:
        mel_np = mel.cpu().numpy()
        assert np.array_equal(host.forward_ragged(mel_np, lens), ref)  # pageable buffers
        mel_pin = torch.from_numpy(mel_np).pin_memory()
        out_pin = torch.empty((len(lens), 1, 256 * max(lens)), dtype=torch.float32).pin_memory()
        host.forward_ragged(mel_pin.numpy(), lens, out=out_pin.numpy())  # pinned buffers, used in place
        assert np.array_equal(out_pin.numpy(), ref)
    finally:
        host.close()
