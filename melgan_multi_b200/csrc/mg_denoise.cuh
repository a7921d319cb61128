// What the batch denoiser (mg_denoise.cu) and the streaming denoiser (mg_denoise_stream.cu) share: the device code of one
// frame, so both compute every frame from the same source, and the host's analysis limits and NOLA check.
#pragma once

#include <vector>

#include "mg_common.cuh"
#include "mg_fft.cuh"
#include "mg_stft_frame.cuh"

namespace mg {

constexpr int kDnMinN = 128, kDnMaxN = 2048;
constexpr int kDnMaxL = 1 << 30;   // keeps every sample, padded position and 2 (L - 1) inside int
constexpr double kDnNola = 1e-11;  // torch.istft's least window-square envelope

inline bool dn_n_ok(int n) { return n >= kDnMinN && n <= kDnMaxN && (n & (n - 1)) == 0; }
inline int dn_frames(int hop, int L) { return 1 + L / hop; }

// w2[n_fft]: the squared periodic Hann of win_length centred in n_fft; full[min(hop, n_fft)]: its per-residue sums
// sum_{n = q mod hop} w2[n], the envelope at every interior output position of residue q
void dn_window_sq(int n_fft, int hop, int win_length, std::vector<double> &w2, std::vector<double> &full);
// the first output sample of an L-sample item whose envelope is below 1e-11, or -1 (torch.istft's NOLA check)
long long dn_nola_fail(const std::vector<double> &w2, const std::vector<double> &full, int N, int hop, int L);
int dn_check_pointer(const char *fn, const char *name, const void *p, unsigned align);

// One frame of the denoiser by a 128-thread CTA: padded positions [p0, p0 + N) of signal s (L samples, reflected at 0
// and at L) through the forward FFT and split, the bin rule with bias row b, real_unsplit, the inverse Stockham pass, the
// 1 / M scale (exact: M = N / 2 is a power of two) and the window, stored to frame[0 .. N).  lt: the thread (0 .. 127);
// buf [N] and Y [N / 2 + 1]: the CTA's shared memory.  A statement macro rather than a function, so that each kernel
// compiles the loops in its own body: as a separate function the compiler unrolls them before inlining, which changes
// denoise_frame_kernel's instructions.  Its arguments must not name its locals (M, win, tw, Z, k, X, m, d, mc, r, A, z,
// inv, out, n): pass such values in variables of other names.
#define MG_DENOISE_FRAME(N, tab, s, L, p0, strength, b, frame, lt, buf, Y)                                                        \
    {                                                                                                                           \
        constexpr int M = (N) / 2;                                                                                              \
        const float *win = (tab);                                                                                               \
        const float2 *tw = reinterpret_cast<const float2 *>((tab) + (N));                                                       \
        const float2 *Z = stft_frame<N>(win, tw, (s), (L), (p0), (lt), (buf), (buf) + M);                                       \
        for (int k = (lt); k <= M; k += 128) {                                                                                  \
            const float2 X = stft_bin<N>(Z, tw, k);                                                                             \
            const float m = sqrtf(X.x * X.x + X.y * X.y), d = m - (strength) * __ldg((b) + k);                                  \
            const float mc = d < 0.f ? 0.f : d; /* NaN stays NaN */                                                             \
            const float r = mc / m;                                                                                             \
            (Y)[k] = m > 0.f ? make_float2(r * X.x, r * X.y) : make_float2(mc, 0.f); /* |X| = 0: phase 0 */                     \
        }                                                                                                                       \
        __syncthreads();                                                                                                        \
        float2 *A = Z == (buf) ? (buf) + M : (buf); /* the buffer Z is not in (Z is read no more) */                            \
        for (int k = (lt); k < M; k += 128)                                                                                     \
            A[k] = real_unsplit((Y)[k], (Y)[M - k], k ? __ldg(tw + k) : make_float2(1.f, 0.f), k == 0);                         \
        __syncthreads();                                                                                                        \
        const float2 *z = stockham<M, 128, true>(A, A == (buf) ? (buf) + M : (buf), tw, (lt));                                  \
        constexpr float inv = 1.f / M;                                                                                          \
        float2 *out = reinterpret_cast<float2 *>(frame);                                                                        \
        for (int n = (lt); n < M; n += 128)                                                                                     \
            out[n] = make_float2(__ldg(win + 2 * n) * (z[n].x * inv), __ldg(win + 2 * n + 1) * (z[n].y * inv));                \
    }

}  // namespace mg
