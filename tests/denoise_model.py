"""The denoiser's float64 model (csrc/mg_denoise.cu), stated once for both of its test modules: the definition through
torch.stft / torch.istft, torch.istft's window-square envelope, and a step-by-step restatement with one step switchable
to a mutation, which the GPU tests' error bound has to reject."""
import torch
import torch.nn.functional as F


def hann64(w, n):
    """Periodic Hann of length w centred in n (torch.stft's padding of a shorter window), float64."""
    left = (n - w) // 2
    return F.pad(torch.hann_window(w, dtype=torch.float64), (left, n - w - left))


def denoise64(a, n, h, w, bias_row, strength):
    """The definition for one item: a the item's own float64 samples [L], bias_row [n/2 + 1]."""
    win = torch.hann_window(w, dtype=torch.float64)
    S = torch.stft(a, n, h, w, win, center=True, pad_mode="reflect", return_complex=True)
    M = S.abs()
    Mp = M - strength * bias_row.double()[:, None]
    Mp = torch.where(Mp < 0, torch.zeros_like(Mp), Mp)  # `x < 0 ? 0 : x`: NaN stays NaN
    P = torch.where(M > 0, S / M, torch.ones_like(S))
    return torch.istft(Mp * P, n, h, w, win, center=True, length=a.shape[-1])


def denoise64_batch(audio, n, h, w, bias, strength, lengths=None, voice=None):
    """[B, L_max] float64 of the definition applied to each item's first lengths[i] samples with bias row voice[i]."""
    a = torch.as_tensor(audio).double().cpu()
    B, L = a.shape
    bias = torch.as_tensor(bias).double().cpu()
    out = torch.zeros(B, L, dtype=torch.float64)
    for i in range(B):
        Li = L if lengths is None else int(lengths[i])
        out[i, :Li] = denoise64(a[i, :Li], n, h, w, bias[0 if voice is None else int(voice[i])], strength)
    return out


def envelope64(n, h, w, L):
    """torch.istft's float64 window-square envelope at the output samples of an L-sample item that some frame reaches."""
    T = 1 + L // h
    w2 = hann64(w, n) ** 2
    env = torch.zeros(n + h * (T - 1), dtype=torch.float64)
    for t in range(T):
        env[t * h:t * h + n] += w2
    return env[n // 2:n // 2 + L]


def nola_ok(n, h, w, L):
    return bool(envelope64(n, h, w, L).min() >= 1e-11)


DENOISE_MUTANTS = ("no_synthesis_window", "no_edge_envelope", "bias_on_power", "reflect_at_l_max", "voice0_bias", "frame_shift")


def denoise64_parts(audio, n, h, w, bias, strength, lengths=None, voice=None, mutant=None):
    """The definition restated step by step in float64 (frames, rfft, the bin rule, irfft, window, overlap-add, envelope),
    with one step changed when `mutant` names one of DENOISE_MUTANTS.  Also returns, per item, what the GPU bound needs:
    (out [B, L_max], per-item dict of windowed frames xw [T, n], spectra X and Y [T, n/2+1], synthesis frames yw [T, n],
    envelope env [L_i], window win [n])."""
    a = torch.as_tensor(audio).double().cpu()
    B, Lmax = a.shape
    bias = torch.as_tensor(bias).double().cpu()
    win = hann64(w, n)
    out = torch.zeros(B, Lmax, dtype=torch.float64)
    parts = []
    for i in range(B):
        Li = Lmax if lengths is None else int(lengths[i])
        Lr = Lmax if mutant == "reflect_at_l_max" else Li
        T = 1 + Li // h
        x = F.pad(a[i, :Lr][None, None], (n // 2, n // 2), mode="reflect")[0, 0]
        off = 1 if mutant == "frame_shift" else 0
        x = torch.cat([x, torch.zeros(1, dtype=torch.float64)])
        fr = torch.stack([x[t * h + off:t * h + off + n] for t in range(T)])
        xw = fr * win
        X = torch.fft.rfft(xw)
        m = X.abs()
        row = bias[0 if (voice is None or mutant == "voice0_bias") else int(voice[i])]
        mp = (m ** 2 - strength * row) if mutant == "bias_on_power" else (m - strength * row)
        mp = torch.where(mp < 0, torch.zeros_like(mp), mp)
        if mutant == "bias_on_power":
            mp = torch.sqrt(mp)
        Y = mp * torch.where(m > 0, X / m, torch.ones_like(X))
        y = torch.fft.irfft(Y, n)
        yw = y if mutant == "no_synthesis_window" else y * win
        ola = torch.zeros(n + h * (T - 1), dtype=torch.float64)
        env = torch.zeros_like(ola)
        for t in range(T):
            ola[t * h:t * h + n] += yw[t]
            env[t * h:t * h + n] += win ** 2
        if mutant == "no_edge_envelope":  # every sample divided by the interior (periodic) envelope
            full = torch.zeros(h, dtype=torch.float64)
            for k in range(n):
                full[k % h] += win[k] ** 2
            env = full[torch.arange(env.shape[0]) % h]
        seg = ola[n // 2:n // 2 + Li] / env[n // 2:n // 2 + Li]
        out[i, :seg.shape[0]] = seg
        parts.append(dict(xw=xw, X=X, Y=Y, yw=yw, y=y, env=env[n // 2:n // 2 + Li], win=win, T=T, L=Li))
    return out, parts
