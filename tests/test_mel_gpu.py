"""GPU parity of the mel-spectrogram front end (csrc/mg_mel.cu through melgan_multi_b200.meldataset.mel_spectrogram, the
drop-in for /root/reference/meldataset.py:44-55) against oracle/mel_oracle.py on the same seeded waveforms.  Tolerance: the
oracle computes as librosa does -- the float64 window times the float32 frames, the FFT in float64, magnitudes stored as
complex64 / float32, then a float32 filter bank; the kernel is fp32 throughout (table twiddles), so linear mel energies agree
to ~1e-6 of the frame's largest band and log-mels to 1e-4 wherever they are above the clip floor.  The element-wise float64
bound of every option, length and batch layout is tests/test_mel_isolation_gpu.py."""
import numpy as np
import pytest
import torch

from melgan_multi_b200 import meldataset
from oracle import mel_oracle as mo

pytestmark = pytest.mark.gpu
ARGS = (1024, 80, 22050, 256, 1024, 55, 9000)


def _signals():
    rs = np.random.RandomState(11)
    t = np.arange(24000) / 22050.0
    yield "noise_segment", (rs.uniform(-1, 1, 8192) * 0.9).astype(np.float32)
    yield "harmonics", (0.3 * np.sin(2 * np.pi * 220 * t) + 0.2 * np.sin(2 * np.pi * 3520 * t + 1) + 0.01 * rs.standard_normal(t.size)).astype(np.float32)
    yield "chirp_odd_length", (0.8 * np.sin(2 * np.pi * (100 + 4000 * t[:23457]) * t[:23457])).astype(np.float32)
    yield "full_scale_square", np.sign(np.sin(2 * np.pi * 441 * t[:4096])).astype(np.float32)
    yield "one_frame", (rs.uniform(-1, 1, 256) * 0.5).astype(np.float32)
    yield "quiet", (rs.standard_normal(8192) * 1e-4).astype(np.float32)


@pytest.mark.parametrize("name,y", list(_signals()))
def test_mel_spectrogram_matches_oracle(name, y):
    ref = mo.mel_spectrogram(y)
    got = meldataset.mel_spectrogram(torch.from_numpy(y).cuda(), *ARGS).cpu().numpy()
    assert got.shape == ref.shape == (80, 1 + (len(y) + 768 - 1024) // 256)
    lin_ref, lin_got = np.exp(ref.astype(np.float64)), np.exp(got.astype(np.float64))
    scale = lin_ref.max(axis=0, keepdims=True)  # per frame
    assert (np.abs(lin_got - lin_ref) <= 2e-6 * scale + 1e-4 * lin_ref).all(), (name, np.abs(lin_got - lin_ref).max())
    above = ref > np.log(1e-4)
    assert np.abs(got - ref)[above].max(initial=0) < 1e-4 * max(1.0, np.abs(ref[above]).max(initial=1.0)), name


def test_mel_spectrogram_batch_silence_and_asserts():
    rs = np.random.RandomState(3)
    yb = (rs.uniform(-1, 1, (5, 8192)) * 0.6).astype(np.float32)
    yb[2] = 0
    got = meldataset.mel_spectrogram(torch.from_numpy(yb).cuda(), *ARGS).cpu().numpy()
    assert got.shape == (5, 80, 32)
    for i in range(5):
        assert np.abs(got[i] - mo.mel_spectrogram(yb[i])).max() < 2e-4
    assert np.allclose(got[2], np.log(1e-5), atol=1e-6)  # silence sits on the clip floor (meldataset.py:25)
    with pytest.raises(AssertionError):  # meldataset.py:45-46
        meldataset.mel_spectrogram(torch.full((1024,), 1.5).cuda(), *ARGS)
    with pytest.raises(Exception):
        meldataset.mel_spectrogram(torch.zeros(8192).cuda(), 2048, 80, 22050, 256, 1024, 55, 9000)


def test_vocoder_round_trip_shapes():
    """mel(audio) feeds the generator and the generator's audio feeds mel again (train.py:157,164): lengths line up."""
    from melgan_multi_b200 import models, synth
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    y = torch.from_numpy(synth.audio_input(2, 8192, 1)[:, 0]).cuda()
    m = meldataset.mel_spectrogram(y, *ARGS)
    with torch.no_grad():
        y_hat = g(m)
    assert m.shape == (2, 80, 32) and y_hat.shape == (2, 1, 8192)
    m2 = meldataset.mel_spectrogram(y_hat[:, 0].clamp(-1, 1), *ARGS)
    assert m2.shape == m.shape and torch.isfinite(m2).all()
