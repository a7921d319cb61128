"""CPU restatement of the reference's mel-spectrogram front end -- TEST INFRASTRUCTURE.

Follows /root/reference/meldataset.py:44-55 (`mel_spectrogram`: constant-pad by (n_fft - hop) / 2 on both sides, then
`librosa.feature.melspectrogram(y, hop_length, win_length, center=False, power=1, sr, n_fft, n_mels, fmin, fmax, norm=1)`,
then :19-25,34-36 `log(clip(x, 1e-5))`).

PARITY UNPINNED.  The arithmetic lives in a third-party dependency that is absent from /root/reference and from this
image: **librosa, unpinned** in /root/reference/requirements.txt:3.  The call site's API -- `y` passed positionally and
`norm=1` -- is that of librosa 0.6 / 0.7 (contemporary with the pinned torch==1.2.0, Aug 2019), where `filters.mel(norm=1)`
means *Slaney area normalisation* (each triangle scaled by 2 / (f[m+2] - f[m]); spelled `norm='slaney'` since 0.8, where
the integer 1 became an L1 normalisation instead).  This file restates the published algorithm of that API:
  stft            librosa.core.spectrum.stft: periodic Hann (scipy.signal.get_window('hann', win_length, fftbins=True)),
                  zero-padded/centred to n_fft, frames y[t*hop : t*hop + n_fft], the float64 window times the
                  frames and rfft in float64, complex64 result
  melspectrogram  |stft| ** power, then `filters.mel(...) @ S`
  filters.mel     Slaney mel scale (htk=False): linear below 1 kHz (200/3 Hz per mel), logarithmic above (step ln(6.4)/27);
                  n_mels + 2 band edges from fmin to fmax, triangular weights on the rfft bin frequencies
                  linspace(0, sr/2, 1 + n_fft/2), float32
With no librosa and no golden vectors in the reference, the restatement is anchored only by independent pieces available
here (tests/test_oracle.py: scipy.signal.stft for the STFT magnitudes, closed-form properties of the filter bank).
"""
import numpy as np


def hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz, logstep = 1000.0, np.log(6.4) / 27.0
    min_log_mel = min_log_hz / f_sp
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hz) / logstep, mels)


def mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp = 200.0 / 3
    min_log_hz, logstep = 1000.0, np.log(6.4) / 27.0
    min_log_mel = min_log_hz / f_sp
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_filterbank(sr, n_fft, n_mels, fmin, fmax, norm=1):
    """librosa.filters.mel of the 0.6/0.7 API.  norm: None, 1 (Slaney area normalisation), or "l1" (what the integer 1 means
    from librosa 0.8 on: every filter divided by its L1 norm)."""
    return mel_filterbank64(sr, n_fft, n_mels, fmin, fmax, norm).astype(np.float32)


def mel_filterbank64(sr, n_fft, n_mels, fmin, fmax, norm=1):
    """mel_filterbank before its float32 cast: [n_mels, 1 + n_fft/2] float64."""
    fftfreqs = np.linspace(0, float(sr) / 2, 1 + n_fft // 2, endpoint=True)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    if norm == 1:
        w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    elif norm == "l1":
        w /= np.maximum(np.abs(w).sum(axis=1, keepdims=True), 1e-30)
    return w


def stft_magnitude(y, n_fft, hop, win_length):
    """|librosa.stft(y, n_fft, hop, win_length, window='hann', center=False)|: [1 + n_fft/2, frames] float32.
    As librosa does it: the float64 window times the float32 frames, the FFT in float64, the result stored as complex64."""
    n = np.arange(win_length)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * n / win_length)  # periodic Hann, float64
    if win_length < n_fft:
        lpad = (n_fft - win_length) // 2
        win = np.pad(win, (lpad, n_fft - win_length - lpad))
    y = np.asarray(y, np.float32)
    frames = 1 + (len(y) - n_fft) // hop
    idx = np.arange(n_fft)[:, None] + hop * np.arange(frames)[None, :]
    spec = np.fft.rfft(win[:, None] * y[idx].astype(np.float64), axis=0).astype(np.complex64)
    return np.abs(spec).astype(np.float32)


def mel_spectrogram(y, n_fft=1024, num_mels=80, sampling_rate=22050, hop_size=256, win_size=1024, fmin=55, fmax=9000, norm=1):
    """meldataset.py:44-55 for one waveform y [L] in [-1, 1]: log-mel [num_mels, frames] float32."""
    y = np.asarray(y, np.float32)
    assert y.min() >= -1.0 and y.max() <= 1.0
    p = int((n_fft - hop_size) / 2)
    y = np.pad(y, (p, p), "constant", constant_values=(0, 0))
    S = stft_magnitude(y, n_fft, hop_size, win_size)
    mel = np.dot(mel_filterbank(sampling_rate, n_fft, num_mels, fmin, fmax, norm), S)
    return np.log(np.clip(mel, 1e-5, None)).astype(np.float32)
