// Multi-resolution STFT loss (Parallel WaveGAN's MultiResolutionSTFTLoss), forward and gradient with respect to the
// predicted audio x, for target audio y.  Per resolution (n_fft N, hop h, window length w, periodic Hann):
//   X = stft(x, N, h, w, hann(w), center=True, pad_mode="reflect"), one-sided, T = 1 + L / h frames (torch.stft);
//   x_mag = sqrt(clamp(|X|^2, min=1e-7)), y_mag likewise;
//   sc = ||y_mag - x_mag||_F / ||y_mag||_F,  mag = mean |log y_mag - log x_mag|;
// the call returns the means of sc and mag over the resolutions.
//
// stft_loss_fwd_kernel<N>: one CTA per (item, frame), 256 threads: threads 0..127 transform x's frame, 128..255 y's.  Each
//   frame reads its N samples straight from the unpadded signal, the reflection done in the index math, times the window
//   (zero-padded to N, centred), as z[n] = s[2n] + i s[2n+1] through the N/2-point Stockham FFT and the real split of
//   mg_fft.cuh.  The CTA writes three partial sums over its N/2 + 1 bins: sum (y_mag - x_mag)^2, sum y_mag^2 and
//   sum |log y_mag - log x_mag|, in a fixed tree order.
// stft_loss_finish_kernel: one CTA sums every partial of every resolution in float64, in a fixed order, and writes the two
//   losses and each resolution's norms ||y_mag - x_mag|| and ||y_mag|| (kept for the backward).  No atomics anywhere: the
//   result has the same bits on every run.
// stft_loss_bwd_frame_kernel<N>: same geometry; recomputes X and Y with the forward's arithmetic, forms
//   G[k] = d loss / d Re X[k] + i d loss / d Im X[k] = (d loss / d x_mag[k]) X[k] / x_mag[k] (0 where |X|^2 < 1e-7),
//   runs the split's adjoint and the inverse N/2-point Stockham pass with all 256 threads, and writes the windowed frame
//   gradient (N floats) to the workspace.
// stft_loss_bwd_gather_kernel: grad_x[i] = sum over the frames reading padded position i + N/2, then N/2 - i (its left
//   reflection, 1 <= i <= N/2), then N/2 + 2(L - 1) - i (its right reflection, L - 1 - N/2 <= i <= L - 2), ascending t
//   within each; resolution r > 0 adds to resolution r - 1's result, so the frame workspace is reused across resolutions.
//
// Non-finite samples are not clamped away: the clamps are written `v < 1e-7f ? 1e-7f : v`, which keeps NaN, and a NaN
// or Inf sample reaches the losses and the gradient as float64 autograd of the definition carries it.
#include <math.h>

#include "mg_common.cuh"
#include "mg_fft.cuh"
#include "mg_frame_loss.cuh"
#include "mg_stft_frame.cuh"

namespace mg {

constexpr int kStftMinN = 128, kStftMaxN = 2048, kStftMaxRes = 8, kStftStatsBytes = 256;
constexpr int kStftMaxL = 1 << 30;  // keeps every sample and padded position, and 2 (L - 1), inside int
constexpr float kStftFloor = 1e-7f;

static bool stft_n_ok(int n) { return n >= kStftMinN && n <= kStftMaxN && (n & (n - 1)) == 0; }
static size_t round256(size_t v) { return (v + 255) / 256 * 256; }

size_t stft_tables_bytes(int n_fft) { return stft_n_ok(n_fft) ? (size_t)n_fft * 8 : 0; }

// host table of one resolution: win[N] (periodic Hann of length w, (N - w) / 2 zeros on the left, as torch.stft pads it),
// then tw[N / 2] = e^{-2 pi i k / N}; every value computed in double and rounded once
int stft_tables_build(int n_fft, int win_length, void *tables_host) {
    const char *fn = "mg_stft_loss_tables_build";
    if (!tables_host) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables_host is NULL", fn);
    if (!stft_n_ok(n_fft))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft=%d is not a power of two in [%d, %d]", fn, n_fft, kStftMinN, kStftMaxN);
    if (win_length < 1 || win_length > n_fft)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: win_length=%d is outside [1, n_fft=%d]", fn, win_length, n_fft);
    stft_tables_fill(n_fft, win_length, reinterpret_cast<float *>(tables_host));
    return MG_OK;
}

void stft_tables_fill(int n_fft, int win_length, float *win) {
    const double pi = 3.14159265358979323846;
    float2 *tw = reinterpret_cast<float2 *>(win + n_fft);
    const int left = (n_fft - win_length) / 2;
    for (int n = 0; n < n_fft; ++n) {
        const int j = n - left;
        // torch.hann_window(1) is [1]
        win[n] = (j >= 0 && j < win_length) ? (win_length == 1 ? 1.f : (float)(0.5 - 0.5 * cos(2 * pi * j / win_length))) : 0.f;
    }
    for (int k = 0; k < n_fft / 2; ++k) tw[k] = make_float2((float)cos(2 * pi * k / n_fft), (float)-sin(2 * pi * k / n_fft));
}

int stft_frames(int n_fft, int hop, int L) {
    if (!stft_n_ok(n_fft) || hop < 1 || L <= n_fft / 2 || L > kStftMaxL) return 0;
    return 1 + L / hop;
}

__device__ __forceinline__ float stft_clamp(float m2) { return m2 < kStftFloor ? kStftFloor : m2; }

template <int N>
__global__ void __launch_bounds__(256) stft_loss_fwd_kernel(const float *__restrict__ tab, const float *__restrict__ x,
                                                            const float *__restrict__ y, float *__restrict__ part, int L, int hop,
                                                            int T, int BT) {
    constexpr int M = N / 2;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);  // [x, y][2 buffers][M]
    float *mag = reinterpret_cast<float *>(buf + 4 * M);  // [x, y][M + 1]
    __shared__ float red[8];
    const int tid = threadIdx.x, g = tid >> 7, lt = tid & 127;
    const int f = (int)blockIdx.x, b = f / T, t = f - b * T;
    const float *win = tab;
    const float2 *tw = reinterpret_cast<const float2 *>(tab + N);
    float2 *A = buf + g * 2 * M;
    const float2 *Z = stft_frame<N>(win, tw, (g ? y : x) + (size_t)b * L, L, t * hop, lt, A, A + M);
    for (int k = lt; k <= M; k += 128) {
        const float2 X = stft_bin<N>(Z, tw, k);
        mag[g * (M + 1) + k] = sqrtf(stft_clamp(X.x * X.x + X.y * X.y));
    }
    __syncthreads();
    float s_diff = 0.f, s_y = 0.f, s_log = 0.f;
    for (int k = tid; k <= M; k += 256) {
        const float xm = mag[k], ym = mag[M + 1 + k], d = ym - xm;
        s_diff = fmaf(d, d, s_diff);
        s_y = fmaf(ym, ym, s_y);
        s_log += fabsf(logf(ym) - logf(xm));
    }
    s_diff = block_sum256(s_diff, red);
    s_y = block_sum256(s_y, red);
    s_log = block_sum256(s_log, red);
    if (tid == 0) {
        part[f] = s_diff;  // 3 B T can pass 2^31: index in 64 bits
        part[(size_t)BT + f] = s_y;
        part[(size_t)2 * BT + f] = s_log;
    }
}

struct StftFinishArgs {
    const float *part[kStftMaxRes];
    int bt[kStftMaxRes];
    double nel[kStftMaxRes];  // B * T * (N / 2 + 1)
    int n_res;
};

__global__ void __launch_bounds__(1024) stft_loss_finish_kernel(StftFinishArgs a, float *__restrict__ sc, float *__restrict__ mag,
                                                                float *__restrict__ stats) {
    __shared__ double red[32];
    double sc_acc = 0.0, mag_acc = 0.0;
    for (int r = 0; r < a.n_res; ++r) {
        const int bt = a.bt[r];
        const double s_diff = sum64_1024(a.part[r], bt, red);
        const double s_y = sum64_1024(a.part[r] + bt, bt, red);
        const double s_log = sum64_1024(a.part[r] + (size_t)2 * bt, bt, red);
        if (threadIdx.x == 0) {
            const double num = sqrt(s_diff), den = sqrt(s_y);
            stats[2 * r] = (float)num;
            stats[2 * r + 1] = (float)den;
            sc_acc += num / den;
            mag_acc += s_log / a.nel[r];
        }
    }
    if (threadIdx.x == 0) {
        *sc = (float)(sc_acc / a.n_res);
        *mag = (float)(mag_acc / a.n_res);
    }
}

template <int N>
__global__ void __launch_bounds__(256) stft_loss_bwd_frame_kernel(const float *__restrict__ tab, const float *__restrict__ x,
                                                                  const float *__restrict__ y, const float *__restrict__ grad_sc,
                                                                  const float *__restrict__ grad_mag, const float *__restrict__ stats,
                                                                  float inv_res, float inv_nel, float *__restrict__ dframe, int L,
                                                                  int hop, int T) {
    constexpr int M = N / 2;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);  // [x, y][2 buffers][M]
    float2 *G = buf + 4 * M;                              // [M + 1]
    const int tid = threadIdx.x, g = tid >> 7, lt = tid & 127;
    const int f = (int)blockIdx.x, b = f / T, t = f - b * T;
    const float *win = tab;
    const float2 *tw = reinterpret_cast<const float2 *>(tab + N);
    float2 *A = buf + g * 2 * M;
    const float2 *Zx = stft_frame<N>(win, tw, (g ? y : x) + (size_t)b * L, L, t * hop, lt, A, A + M) - g * 2 * M;
    const float2 *Zy = Zx + 2 * M;
    // d sc / d x_mag = -(y_mag - x_mag) / (||y_mag - x_mag|| ||y_mag||), 0 where the numerator's norm is 0 (torch's norm
    // backward); d mag / d x_mag = -sign(log y_mag - log x_mag) / (B T (N/2 + 1) x_mag), sign(0) = 0
    const float num = __ldg(stats), den = __ldg(stats + 1);
    const float a = num == 0.f ? 0.f : __ldg(grad_sc) * inv_res / den / num;
    const float cm = __ldg(grad_mag) * inv_res * inv_nel;
    for (int k = tid; k <= M; k += 256) {
        const float2 X = stft_bin<N>(Zx, tw, k), Y = stft_bin<N>(Zy, tw, k);
        const float xm2 = X.x * X.x + X.y * X.y;
        const float xm = sqrtf(stft_clamp(xm2)), ym = sqrtf(stft_clamp(Y.x * Y.x + Y.y * Y.y));
        const float d = logf(ym) - logf(xm), sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : d * 0.f);  // NaN stays NaN
        const float dxm = -(a * (ym - xm)) - cm * sg / xm;
        const float r = xm2 >= kStftFloor ? dxm / xm : 0.f;  // clamp(min=)' = [|X|^2 >= 1e-7]; sqrt' and |.|^2' give X / x_mag
        G[k] = make_float2(r * X.x, r * X.y);
    }
    __syncthreads();
    split_adjoint_pass<M, 256>(G, buf, tw, tid);
    __syncthreads();
    const float2 *dz = stockham<M, 256, true>(buf, buf + M, tw, tid);
    // d/dRe z[n] + i d/dIm z[n], z[n] = win[2n] s[2n] + i win[2n+1] s[2n+1]
    float2 *df = reinterpret_cast<float2 *>(dframe + (size_t)f * N);
    for (int n = tid; n < M; n += 256) df[n] = make_float2(__ldg(win + 2 * n) * dz[n].x, __ldg(win + 2 * n + 1) * dz[n].y);
}

__global__ void __launch_bounds__(256) stft_loss_bwd_gather_kernel(const float *__restrict__ dframe, float *__restrict__ grad_x, int L,
                                                                   int N, int hop, int T, int accumulate) {
    const int chunks = (L + 255) >> 8;
    const int b = (int)blockIdx.x / chunks, i = (((int)blockIdx.x - b * chunks) << 8) + (int)threadIdx.x;
    if (i >= L) return;
    const float *db = dframe + (size_t)b * T * N;
    const int h = N / 2;
    float acc = frame_gather(db, i + h, N, hop, T);
    if (i >= 1 && i <= h) acc += frame_gather(db, h - i, N, hop, T);
    if (i >= L - 1 - h && i <= L - 2) acc += frame_gather(db, h + (L - 1) + (L - 1 - i), N, hop, T);
    float *out = grad_x + (size_t)b * L + i;
    *out = accumulate ? *out + acc : acc;
}

template <int N>
static constexpr int stft_fwd_smem() { return 4 * (N / 2) * 8 + 2 * (N / 2 + 1) * 4; }
template <int N>
static constexpr int stft_bwd_smem() { return 4 * (N / 2) * 8 + (N / 2 + 1) * 8; }
static_assert(stft_fwd_smem<kStftMaxN>() <= 48 * 1024 && stft_bwd_smem<kStftMaxN>() <= 48 * 1024, "no opt-in needed");

// every argument of a forward or backward call that the kernels rely on; *T gets each resolution's frame count
int stft_check(const char *fn, int n_res, const void *const *tables, const int *n_fft, const int *hop, int B, int L, int *T) {
    if (n_res < 1 || n_res > kStftMaxRes)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_res=%d resolutions, 1 to %d supported", fn, n_res, kStftMaxRes);
    if (!n_fft || !hop) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, !n_fft ? "n_fft" : "hop");
    if (B < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d, at least 1 item needed", fn, B);
    if (L > kStftMaxL) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L=%d samples, at most 2^30 supported", fn, L);
    for (int r = 0; r < n_res; ++r) {
        if (!stft_n_ok(n_fft[r]))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft[%d]=%d is not a power of two in [%d, %d]", fn, r, n_fft[r], kStftMinN,
                             kStftMaxN);
        if (hop[r] < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: hop[%d]=%d, at least 1 needed", fn, r, hop[r]);
        if (L <= n_fft[r] / 2)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L=%d samples, reflect padding by n_fft[%d]/2=%d needs more", fn, L, r,
                             n_fft[r] / 2);
        if (tables) {
            if (!tables[r]) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables[%d] is NULL", fn, r);
            if ((uintptr_t)tables[r] % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables[%d] must be 16-byte aligned", fn, r);
        }
        T[r] = stft_frames(n_fft[r], hop[r], L);
        if ((long long)B * T[r] > 0x7fffffffll)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d x %d frames of resolution %d exceed 2^31 - 1 CTAs", fn, B, T[r], r);
    }
    if ((long long)B * ((L + 255) / 256) > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d x %d sample blocks exceed 2^31 - 1 CTAs", fn, B, (L + 255) / 256);
    return MG_OK;
}

void stft_workspace(int n_res, const int *n_fft, int B, const int *T, size_t *fwd, size_t *bwd) {
    size_t f = kStftStatsBytes, w = 0;
    for (int r = 0; r < n_res; ++r) {
        f += round256((size_t)3 * B * T[r] * sizeof(float));
        const size_t d = (size_t)B * T[r] * n_fft[r] * sizeof(float);
        w = d > w ? d : w;
    }
    *fwd = f;
    *bwd = w;
}

int launch_stft_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                             int B, int L, const int *T, float *sc, float *mag, void *workspace, cudaStream_t s) {
    StftFinishArgs a{};
    a.n_res = n_res;
    char *ws = reinterpret_cast<char *>(workspace);
    float *stats = reinterpret_cast<float *>(ws);
    size_t off = kStftStatsBytes;
    for (int r = 0; r < n_res; ++r) {
        const int BT = B * T[r];
        float *part = reinterpret_cast<float *>(ws + off);
        off += round256((size_t)3 * BT * sizeof(float));
        a.part[r] = part;
        a.bt[r] = BT;
        a.nel[r] = (double)BT * (n_fft[r] / 2 + 1);
        const float *tab = reinterpret_cast<const float *>(tables[r]);
        switch (n_fft[r]) {
#define MG_STFT_FWD(NN)                                                                                                    \
    case NN: stft_loss_fwd_kernel<NN><<<(unsigned)BT, 256, stft_fwd_smem<NN>(), s>>>(tab, x, y, part, L, hop[r], T[r], BT); break;
            MG_STFT_FWD(128) MG_STFT_FWD(256) MG_STFT_FWD(512) MG_STFT_FWD(1024) MG_STFT_FWD(2048)
#undef MG_STFT_FWD
        }
        MG_CUDA_TRY(cudaGetLastError());
    }
    stft_loss_finish_kernel<<<1, 1024, 0, s>>>(a, sc, mag, stats);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

int launch_stft_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                              int B, int L, const int *T, const float *grad_sc, const float *grad_mag, const void *fwd_workspace,
                              float *grad_x, void *workspace, cudaStream_t s) {
    const float *stats = reinterpret_cast<const float *>(fwd_workspace);
    float *dframe = reinterpret_cast<float *>(workspace);
    for (int r = 0; r < n_res; ++r) {
        const float *tab = reinterpret_cast<const float *>(tables[r]);
        const float inv_res = 1.f / n_res, inv_nel = (float)(1.0 / ((double)B * T[r] * (n_fft[r] / 2 + 1)));
        const unsigned BT = (unsigned)(B * T[r]);
        switch (n_fft[r]) {
#define MG_STFT_BWD(NN)                                                                                                          \
    case NN:                                                                                                                     \
        stft_loss_bwd_frame_kernel<NN><<<BT, 256, stft_bwd_smem<NN>(), s>>>(tab, x, y, grad_sc, grad_mag, stats + 2 * r, inv_res, \
                                                                          inv_nel, dframe, L, hop[r], T[r]);                      \
        break;
            MG_STFT_BWD(128) MG_STFT_BWD(256) MG_STFT_BWD(512) MG_STFT_BWD(1024) MG_STFT_BWD(2048)
#undef MG_STFT_BWD
        }
        MG_CUDA_TRY(cudaGetLastError());
        stft_loss_bwd_gather_kernel<<<(unsigned)((long long)B * ((L + 255) / 256)), 256, 0, s>>>(dframe, grad_x, L, n_fft[r], hop[r],
                                                                                                 T[r], r > 0);
        MG_CUDA_TRY(cudaGetLastError());
    }
    return MG_OK;
}

}  // namespace mg
