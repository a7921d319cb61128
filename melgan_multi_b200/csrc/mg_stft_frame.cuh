// torch.stft's framing (center=True, pad_mode="reflect") on the fly, shared by the multi-resolution STFT loss
// (mg_stft_loss.cu) and the denoiser (mg_denoise.cu): a frame reads its N samples straight from the unpadded signal,
// the reflection done in the index math, times the window (the STFT-loss table: win[N], then tw[N / 2]).
#pragma once

#include "mg_fft.cuh"

namespace mg {

// reflect padding by N / 2, in the index math: padded position p reads sample p - N/2 reflected into [0, L)
__device__ __forceinline__ int stft_reflect(int i, int L) { return i < 0 ? -i : (i >= L ? 2 * (L - 1) - i : i); }

// one windowed frame (padded positions [p0, p0 + N)) of signal s through the N/2-point FFT, by the 128 threads of a
// group; returns the buffer (A or Bf) holding Z
template <int N>
__device__ __forceinline__ float2 *stft_frame(const float *__restrict__ win, const float2 *__restrict__ tw, const float *__restrict__ s,
                                              int L, int p0, int lt, float2 *A, float2 *Bf) {
    for (int n = lt; n < N / 2; n += 128) {
        const int i = p0 + 2 * n - N / 2;
        const float x0 = __ldg(s + stft_reflect(i, L)), x1 = __ldg(s + stft_reflect(i + 1, L));
        A[n] = make_float2(__ldg(win + 2 * n) * x0, __ldg(win + 2 * n + 1) * x1);
    }
    __syncthreads();
    return stockham<N / 2, 128, false>(A, Bf, tw, lt);
}

template <int N>
__device__ __forceinline__ float2 stft_bin(const float2 *Z, const float2 *__restrict__ tw, int k) {
    constexpr int M = N / 2;
    return real_split(Z[k & (M - 1)], Z[(M - k) & (M - 1)], k < M ? __ldg(tw + k) : make_float2(-1.f, 0.f));
}

}  // namespace mg
