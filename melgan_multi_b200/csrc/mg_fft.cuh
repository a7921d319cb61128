// Radix-2 Stockham FFT pieces shared by the mel front end (mg_mel.cu) and the multi-resolution STFT loss
// (mg_stft_loss.cu), the mel loss (mg_mel_loss.cu) and the denoiser (mg_denoise.cu).  A real frame of N = 2M samples is
// transformed as the M-point complex sequence z[n] = x[2n] + i x[2n+1]; real_split turns its transform Z into the bins
// X[0..M] of the real transform, real_unsplit is its inverse and split_adjoint_pass its adjoint.  Twiddle tables hold tw[k] = e^{-2 pi i k / N} for k < M.
// Every function is called by all NT threads of a group together (they hold __syncthreads).
#pragma once

namespace mg {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// M-point Stockham autosort FFT, radix 2: log2(M) passes of M/2 butterflies between in and out.  Forward twiddles
// e^{-2 pi i k / (2 ns)} = tw[k M / ns]; kInverse conjugates them (unnormalised).  Returns the buffer holding the result.
template <int M, int NT, bool kInverse>
__device__ __forceinline__ float2 *stockham(float2 *in, float2 *out, const float2 *tw, int lt) {
#pragma unroll 1
    for (int ns = 1; ns < M; ns <<= 1) {
#pragma unroll
        for (int r = 0; r < (M / 2 + NT - 1) / NT; ++r) {
            const int j = lt + NT * r;
            if ((M / 2) % NT == 0 || j < M / 2) {
                const int k = j & (ns - 1);
                float2 v0, v1;  // each direction keeps the load order the mel kernels were written with
                if (kInverse) {
                    const float2 w = tw[k * (M / ns)];
                    v0 = in[j];
                    v1 = cmul(in[j + M / 2], make_float2(w.x, -w.y));
                } else {
                    v0 = in[j];
                    v1 = cmul(in[j + M / 2], tw[k * (M / ns)]);
                }
                const int j0 = ((j - k) << 1) + k;
                out[j0] = make_float2(v0.x + v1.x, v0.y + v1.y);
                out[j0 + ns] = make_float2(v0.x - v1.x, v0.y - v1.y);
            }
        }
        __syncthreads();
        float2 *tmp = in; in = out; out = tmp;
    }
    return in;
}

// X[k] = E[k] + W^k O[k], E = (Z[k] + conj Z[M-k]) / 2, O = (Z[k] - conj Z[M-k]) / 2i, from zk = Z[k mod M],
// zc = Z[(M - k) mod M] and w = W^k (W^M = -1)
__device__ __forceinline__ float2 real_split(const float2 zk, const float2 zc, const float2 w) {
    const float2 E = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
    const float2 O = make_float2(0.5f * (zk.y + zc.y), -0.5f * (zk.x - zc.x));
    return make_float2(E.x + w.x * O.x - w.y * O.y, E.y + w.x * O.y + w.y * O.x);
}

// Inverse of the split: Z[k] = E + i O with E = (X[k] + conj X[M-k]) / 2, O = (X[k] - conj X[M-k]) conj(W^k) / 2, from
// xk = X[k], xc = X[M - k] and w = W^k, k = 0..M-1; the M-point inverse pass of Z gives M (x[2n] + i x[2n+1]).  At k = 0
// (xc = X[M]) the imaginary parts of X[0] and X[M] are dropped, as irfft drops them.
__device__ __forceinline__ float2 real_unsplit(float2 xk, float2 xc, const float2 w, bool k0) {
    if (k0) xk.y = xc.y = 0.f;
    const float2 E = make_float2(0.5f * (xk.x + xc.x), 0.5f * (xk.y - xc.y));
    const float2 D = make_float2(0.5f * (xk.x - xc.x), 0.5f * (xk.y + xc.y));  // (X[k] - conj X[M-k]) / 2
    const float2 O = make_float2(D.x * w.x + D.y * w.y, D.y * w.x - D.x * w.y);  // D conj(w)
    return make_float2(E.x - O.y, E.y + O.x);
}

// Adjoint of the split, with a_k = (1 - i W^k) / 2, b_k = (1 + i W^k) / 2, X[k] = a_k Z[k mod M] + b_k conj Z[(M - k) mod M]:
// dZ[j] = P(j) + Q((M - j) mod M), P(k) = conj(a_k) G[k], Q(k) = b_k conj G[k]; dZ[0] also takes P(M) + Q(M), the Nyquist
// bin's share.  G[k] = d loss / d Re X[k] + i d loss / d Im X[k], k = 0..M.
__device__ __forceinline__ float2 split_adjoint(const float2 G, const float2 w) {  // conj(a) G, w = W^k
    return make_float2(0.5f * (G.x + w.y * G.x - w.x * G.y), 0.5f * (G.y + w.x * G.x + w.y * G.y));
}
__device__ __forceinline__ float2 split_adjoint_conj(const float2 G, const float2 w) {  // b conj(G)
    return make_float2(0.5f * (G.x - w.y * G.x + w.x * G.y), 0.5f * (-G.y + w.x * G.x + w.y * G.y));
}

template <int M, int NT>
__device__ __forceinline__ void split_adjoint_pass(const float2 *G, float2 *dZ, const float2 *tw, int lt) {
    for (int j = lt; j < M; j += NT) {
        const int jc = (M - j) & (M - 1);
        const float2 p = split_adjoint(G[j], tw[j]), q = split_adjoint_conj(G[jc], tw[jc]);
        float2 d = make_float2(p.x + q.x, p.y + q.y);
        if (j == 0) {  // the Nyquist bin reads Z[0] as well: P(M) + Q(M), W^M = -1
            const float2 pn = split_adjoint(G[M], make_float2(-1.f, 0.f)), qn = split_adjoint_conj(G[M], make_float2(-1.f, 0.f));
            d = make_float2(d.x + (pn.x + qn.x), d.y + (pn.y + qn.y));
        }
        dZ[j] = d;
    }
}

}  // namespace mg
