// Per-frame mel arithmetic shared by the mel front end (mg_mel.cu, n_fft 1024) and the multi-resolution mel loss
// (mg_mel_loss.cu, every power-of-two n_fft from 128 to 2048): a zero-padded windowed frame through the N/2-point
// Stockham FFT and the real split to |X[k]|, k = 0..N/2; the sparse Slaney filter bank's band sums; log(clip(., 1e-5));
// and the band adjoint of the backward.  One body for both, so the loss's bands carry exactly the front end's bits.
#pragma once

#include "mg_fft.cuh"

namespace mg {

constexpr int kMelLossMaxMels = 512;  // the most bands a mel-loss table holds (the front end's MelTables holds 128)

// sparse filter bank: filter m = weights[woff[m] .. + kcount[m]) on bins kstart[m] ..
struct MelBank {
    const int *kstart, *kcount, *woff;
    const float *weights;
};

// Frame of signal xb whose first sample is xb[i0] (i0 = t hop - pad; samples outside [0, L) are the zero padding),
// by 128 threads (lt = 0..127) of a CTA that calls this together (it holds __syncthreads): the windowed N/2-point
// complex Stockham FFT in A / Bf, split into the N/2 + 1 bins of the real transform; mg[k] = |X[k]|, and X[k] itself
// when Xk is given.  win[N] is the window, tw[N/2] = e^{-2 pi i k / N}.
template <int N>
__device__ __forceinline__ void mel_frame_bins(const float *win, const float2 *tw, const float *xb, int L, int i0, bool live, int lt,
                                               float2 *A, float2 *Bf, float *mg, float2 *Xk) {
    constexpr int M = N / 2;
    // windowed frame, even samples -> real part, odd -> imaginary
    for (int n = lt; n < M; n += 128) {
        const int i = i0 + 2 * n;
        const float x0 = (live && i >= 0 && i < L) ? __ldg(xb + i) : 0.f;
        const float x1 = (live && i + 1 >= 0 && i + 1 < L) ? __ldg(xb + i + 1) : 0.f;
        A[n] = make_float2(win[2 * n] * x0, win[2 * n + 1] * x1);
    }
    __syncthreads();
    float2 *in = stockham<M, 128, false>(A, Bf, tw, lt);
    // X[k] = E[k] + e^{-2 pi i k / N} O[k], E = (Z[k] + conj Z[M-k]) / 2, O = (Z[k] - conj Z[M-k]) / 2i
    for (int k = lt; k <= M; k += 128) {
        const float2 X = real_split(in[k & (M - 1)], in[(M - k) & (M - 1)], k < M ? tw[k] : make_float2(-1.f, 0.f));
        mg[k] = sqrtf(X.x * X.x + X.y * X.y);  // power = 1 (meldataset.py:50)
        if (Xk) Xk[k] = X;
    }
    __syncthreads();
}

// mel band m before the log: the fma dot product of its sparse filter run with the magnitudes
__device__ __forceinline__ float mel_band_sum(const MelBank &bk, const float *mg, int m) {
    const int ks = bk.kstart[m], kc = bk.kcount[m];
    const float *w = bk.weights + bk.woff[m];
    float s = 0.f;
    for (int i = 0; i < kc; ++i) s = fmaf(w[i], mg[ks + i], s);
    return s;
}

// meldataset.py:19-25: log(clip(s, 1e-5) * 1).  Not fmaxf, which returns 1e-5 for a NaN s: np.clip and torch.clamp keep
// NaN, and a NaN (or Inf) sample must not reach a mel loss as log(1e-5) silence.  Equal to fmaxf otherwise.
__device__ __forceinline__ float mel_log(float s) { return logf(s < 1e-5f ? 1e-5f : s); }

// Band adjoint, by NT threads (lt = 0..NT-1) of a CTA that calls this together: dm = M^T gs over the bins (dm zeroed and
// synchronised by the caller; thread lt owns bands lt, lt + NT, ..., whose d loss / d s gs(m) gives), then
// Xk[k] = dm[k] X[k] / |X[k]| (abs' = X / |X|, 0 at X = 0) for k = 0..N/2, mg[k] = |X[k]|.  Filters of one parity never
// share a bin -- each triangle ends where the next-but-one starts -- so two passes, even then odd, accumulate without
// atomics and every bin sums its terms in the same order.  The caller synchronises before reading Xk.
template <int N, int NT, class GS>
__device__ __forceinline__ void mel_band_adjoint(const MelBank &bk, int n_mels, int lt, GS gs, float *dm, const float *mg, float2 *Xk) {
#pragma unroll 1
    for (int parity = 0; parity < 2; ++parity) {
        for (int m = lt; m < n_mels; m += NT) {
            if ((m & 1) == parity) {
                const int ks = bk.kstart[m], kc = bk.kcount[m];
                const float *w = bk.weights + bk.woff[m];
                const float g = gs(m);
                for (int i = 0; i < kc; ++i) dm[ks + i] = fmaf(w[i], g, dm[ks + i]);
            }
        }
        __syncthreads();
    }
    for (int k = lt; k <= N / 2; k += NT) {
        const float m = mg[k], r = m > 0.f ? dm[k] / m : 0.f;
        Xk[k] = make_float2(r * Xk[k].x, r * Xk[k].y);
    }
}

// host: the sparse Slaney filter bank of librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=False, norm) into
// kstart / kcount / woff [n_mels] and weights [2 (n_fft / 2 + 1)] (a bin lies under at most two triangles); norm 0 = none,
// 1 = Slaney area normalisation, 2 = L1.  The arguments are checked by the caller; fn names it in the one error this
// reports (a bank denser than two triangles per bin).
int mel_filters_build(const char *fn, int n_fft, int sr, int n_mels, float fmin, float fmax, int norm, int *kstart, int *kcount,
                      int *woff, float *weights);

}  // namespace mg
