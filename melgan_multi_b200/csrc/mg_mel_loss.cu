// Multi-resolution log-mel L1 loss (HiFi-GAN's `l1(mel(y_hat), mel(y))`, summed over several analyses as later GAN
// vocoders do), forward and gradient with respect to the predicted audio x, for target audio y.  Per resolution r
// (n_fft N, hop H, window length W, n_mels M; sampling rate, fmin and fmax shared), p = (N - H) / 2:
//   frames t of x zero-padded by p on each side, T = 1 + (L + 2p - N) / H; X_t = rfft(w . frame_t), w a periodic Hann of
//   length W centred in N; S_t = F |X_t| (F the Slaney filter bank of mg_mel_bank.cuh); mel = log(clip(S, 1e-5));
//   l_r = mean over (b, m, t) of |mel_x - mel_y|;
// the call returns (1 / R) sum_r l_r.  At (1024, 256, 1024, 80) this is F.l1_loss of meldataset.mel_spectrogram's two
// outputs: the frame, band and log code is the front end's own (mel_frame_bins, mel_band_sum, mel_log).
//
// mel_loss_fwd_kernel<N>: one CTA per (item, frame), 256 threads: threads 0..127 transform x's frame, 128..255 y's.  The
//   CTA writes one partial sum_m |mel_x - mel_y| in a fixed tree order.
// mel_loss_finish_kernel: one CTA sums every partial of every resolution in float64, in a fixed order: no atomics, the
//   same bits on every run.
// mel_loss_bwd_frame_kernel<N>: same geometry; recomputes X and Y with the forward's arithmetic, forms
//   gs_m = sign(mel_x - mel_y) grad / (R B M T_r) / S_x,m (0 where S_x,m < 1e-5; sign(0) = sign(NaN) = 0 as torch.sign),
//   runs the band adjoint and the phasor X / |X| (mel_band_adjoint), the split's adjoint and the inverse N/2-point
//   Stockham pass with all 256 threads, and writes the windowed frame gradient (N floats) to the workspace.
// mel_loss_bwd_gather_kernel: grad_x[i] = sum over the frames reading padded position i + p, ascending t; resolution
//   r > 0 adds to resolution r - 1's result, so the frame workspace is one resolution's.
//
// Table of one resolution (16-byte aligned, mel_loss_tables_bytes(N)): the STFT loss's window and twiddles
// (stft_tables_fill: win[N], tw[N/2]), then MelLossBank and the filter weights [2 (N/2 + 1)].
#include <math.h>
#include <string.h>

#include "mg_common.cuh"
#include "mg_frame_loss.cuh"
#include "mg_mel_bank.cuh"

namespace mg {

constexpr int kMelLossMinN = 128, kMelLossMaxN = 2048, kMelLossMaxRes = 8;
constexpr int kMelLossMaxL = 1 << 30;  // keeps every sample and padded position inside int

struct MelLossBank {
    int n_mels, pad_[3];
    int kstart[kMelLossMaxMels], kcount[kMelLossMaxMels], woff[kMelLossMaxMels];
};

static bool mel_loss_n_ok(int n) { return n >= kMelLossMinN && n <= kMelLossMaxN && (n & (n - 1)) == 0; }
static size_t round256(size_t v) { return (v + 255) / 256 * 256; }

size_t mel_loss_tables_bytes(int n_fft) {
    if (!mel_loss_n_ok(n_fft)) return 0;
    return (size_t)n_fft * 8 + sizeof(MelLossBank) + ((size_t)2 * (n_fft / 2 + 1) * 4 + 15) / 16 * 16;
}

int mel_loss_tables_build(int n_fft, int win_length, int sr, int n_mels, float fmin, float fmax, void *tables_host) {
    const char *fn = "mg_mel_loss_tables_build";
    if (!tables_host) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables_host is NULL", fn);
    if (!mel_loss_n_ok(n_fft))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft=%d is not a power of two in [%d, %d]", fn, n_fft, kMelLossMinN, kMelLossMaxN);
    if (win_length < 1 || win_length > n_fft)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: win_length=%d is outside [1, n_fft=%d]", fn, win_length, n_fft);
    if (sr < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: sampling_rate=%d, at least 1 needed", fn, sr);
    if (n_mels < 1 || n_mels > kMelLossMaxMels)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_mels=%d is outside [1, %d]", fn, n_mels, kMelLossMaxMels);
    if (!(fmin >= 0.f) || !(fmax > fmin) || !((double)fmax <= sr / 2.0))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: fmin=%g fmax=%g, 0 <= fmin < fmax <= sampling_rate / 2 = %g needed", fn, fmin,
                         fmax, sr / 2.0);
    float *tab = reinterpret_cast<float *>(tables_host);
    memset(tab, 0, mel_loss_tables_bytes(n_fft));
    stft_tables_fill(n_fft, win_length, tab);
    MelLossBank *bk = reinterpret_cast<MelLossBank *>(tab + 2 * n_fft);
    bk->n_mels = n_mels;
    return mel_filters_build(fn, n_fft, sr, n_mels, fmin, fmax, 1, bk->kstart, bk->kcount, bk->woff, reinterpret_cast<float *>(bk + 1));
}

int mel_loss_frames(int n_fft, int hop, int L) {
    if (!mel_loss_n_ok(n_fft) || hop < 1 || hop > n_fft || L < 1 || L > kMelLossMaxL) return 0;
    const int span = L + 2 * ((n_fft - hop) / 2);
    return span < n_fft ? 0 : 1 + (span - n_fft) / hop;
}

__device__ __forceinline__ MelBank mel_loss_bank(const float *tab, int N, int *n_mels) {
    const MelLossBank *h = reinterpret_cast<const MelLossBank *>(tab + 2 * N);
    *n_mels = h->n_mels;
    return MelBank{h->kstart, h->kcount, h->woff, reinterpret_cast<const float *>(h + 1)};
}

constexpr int ilog2(int v) { return v > 1 ? 1 + ilog2(v >> 1) : 0; }
template <int N>
constexpr int mag_stride() { return (N / 2 + 4) & ~3; }  // N/2 + 1 magnitudes, 16-byte rows

template <int N>
__global__ void __launch_bounds__(256) mel_loss_fwd_kernel(const float *__restrict__ tab, const float *__restrict__ x,
                                                           const float *__restrict__ y, float *__restrict__ part, int L, int hop,
                                                           int pad, int T) {
    constexpr int M = N / 2;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);  // [x, y][2 buffers][M]
    float *mag = reinterpret_cast<float *>(buf + 4 * M);  // [x, y][mag_stride]
    __shared__ float red[8];
    const int tid = threadIdx.x, g = tid >> 7, lt = tid & 127;
    const int f = (int)blockIdx.x, b = f / T, t = f - b * T;
    int n_mels;
    const MelBank bk = mel_loss_bank(tab, N, &n_mels);
    float2 *A = buf + g * 2 * M;
    mel_frame_bins<N>(tab, reinterpret_cast<const float2 *>(tab + N), (g ? y : x) + (size_t)b * L, L, t * hop - pad, true, lt, A, A + M,
                      mag + g * mag_stride<N>(), nullptr);
    float s = 0.f;
    for (int m = tid; m < n_mels; m += 256) s += fabsf(mel_log(mel_band_sum(bk, mag, m)) - mel_log(mel_band_sum(bk, mag + mag_stride<N>(), m)));
    s = block_sum256(s, red);
    if (tid == 0) part[f] = s;
}

struct MelLossFinishArgs {
    const float *part[kMelLossMaxRes];
    const int *n_mels[kMelLossMaxRes];  // in each resolution's device table
    int bt[kMelLossMaxRes];
    int n_res;
};

__global__ void __launch_bounds__(1024) mel_loss_finish_kernel(MelLossFinishArgs a, float *__restrict__ loss) {
    __shared__ double red[32];
    double acc = 0.0;
    for (int r = 0; r < a.n_res; ++r) {
        const double s = sum64_1024(a.part[r], a.bt[r], red);
        if (threadIdx.x == 0) acc += s / ((double)a.bt[r] * __ldg(a.n_mels[r]));
    }
    if (threadIdx.x == 0) *loss = (float)(acc / a.n_res);
}

template <int N>
__global__ void __launch_bounds__(256) mel_loss_bwd_frame_kernel(const float *__restrict__ tab, const float *__restrict__ x,
                                                                 const float *__restrict__ y, const float *__restrict__ grad, int n_res,
                                                                 float *__restrict__ dframe, int L, int hop, int pad, int T) {
    constexpr int M = N / 2;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // [x, y][2 buffers][M]; y's magnitudes go to whichever of its buffers the FFT's result is not in, and the bins'
    // gradient dm replaces them once the bands' gradients are formed, which keeps the largest N under 48 KB
    float2 *buf = reinterpret_cast<float2 *>(smem_raw);
    float *mgx = reinterpret_cast<float *>(buf + 4 * M);                    // [mag_stride]
    float2 *Xk = reinterpret_cast<float2 *>(mgx + mag_stride<N>());         // [mag_stride]
    float *gsm = reinterpret_cast<float *>(Xk + mag_stride<N>());           // [kMelLossMaxMels]
    float *mgy = reinterpret_cast<float *>(buf + 2 * M + (ilog2(M) % 2 == 0 ? M : 0));
    float *dm = mgy;
    const int tid = threadIdx.x, g = tid >> 7, lt = tid & 127;
    const int f = (int)blockIdx.x, b = f / T, t = f - b * T;
    int n_mels;
    const MelBank bk = mel_loss_bank(tab, N, &n_mels);
    const float2 *tw = reinterpret_cast<const float2 *>(tab + N);
    float2 *A = buf + g * 2 * M;
    mel_frame_bins<N>(tab, tw, (g ? y : x) + (size_t)b * L, L, t * hop - pad, true, lt, A, A + M, g ? mgy : mgx, g ? nullptr : Xk);
    // d loss / d mel_x = sign(mel_x - mel_y) c, c = grad / (R B M T); log' = 1 / s; clamp(min=)' = [s >= 1e-5]
    const float c = __ldg(grad) * (float)(1.0 / ((double)n_res * (double)(gridDim.x) * n_mels));
    for (int m = tid; m < n_mels; m += 256) {
        const float sx = mel_band_sum(bk, mgx, m);
        const float d = mel_log(sx) - mel_log(mel_band_sum(bk, mgy, m));
        const float gm = d > 0.f ? c : (d < 0.f ? -c : 0.f);
        gsm[m] = sx >= 1e-5f ? gm / sx : 0.f;
    }
    __syncthreads();
    for (int k = tid; k <= M; k += 256) dm[k] = 0.f;
    __syncthreads();
    mel_band_adjoint<N, 256>(bk, n_mels, tid, [&](int m) { return gsm[m]; }, dm, mgx, Xk);
    __syncthreads();
    split_adjoint_pass<M, 256>(Xk, buf, tw, tid);
    __syncthreads();
    // inverse transform: the forward's Stockham passes with conjugate twiddles, unnormalised
    const float2 *dz = stockham<M, 256, true>(buf, buf + M, tw, tid);
    // dz[n] = d/dRe z[n] + i d/dIm z[n], z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1]
    float2 *df = reinterpret_cast<float2 *>(dframe + (size_t)f * N);
    for (int n = tid; n < M; n += 256) df[n] = make_float2(__ldg(tab + 2 * n) * dz[n].x, __ldg(tab + 2 * n + 1) * dz[n].y);
}

__global__ void __launch_bounds__(256) mel_loss_bwd_gather_kernel(const float *__restrict__ dframe, float *__restrict__ grad_x, int L,
                                                                  int N, int hop, int pad, int T, int accumulate) {
    const int chunks = (L + 255) >> 8;
    const int b = (int)blockIdx.x / chunks, i = (((int)blockIdx.x - b * chunks) << 8) + (int)threadIdx.x;
    if (i >= L) return;
    const float acc = frame_gather(dframe + (size_t)b * T * N, i + pad, N, hop, T);
    float *out = grad_x + (size_t)b * L + i;
    *out = accumulate ? *out + acc : acc;
}

template <int N>
static constexpr int mel_loss_fwd_smem() { return 4 * (N / 2) * 8 + 2 * mag_stride<N>() * 4; }
template <int N>
static constexpr int mel_loss_bwd_smem() { return 4 * (N / 2) * 8 + mag_stride<N>() * 4 + mag_stride<N>() * 8 + kMelLossMaxMels * 4; }
static_assert(mel_loss_fwd_smem<kMelLossMaxN>() <= 48 * 1024 && mel_loss_bwd_smem<kMelLossMaxN>() <= 48 * 1024, "no opt-in needed");
static_assert(mag_stride<kMelLossMinN>() <= kMelLossMinN, "y's magnitudes fit in one of its FFT buffers");

// every argument of a forward or backward call that the kernels rely on; *T gets each resolution's frame count
int mel_loss_check(const char *fn, int n_res, const void *const *tables, const int *n_fft, const int *hop, int B, int L, int *T) {
    if (n_res < 1 || n_res > kMelLossMaxRes)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_res=%d resolutions, 1 to %d supported", fn, n_res, kMelLossMaxRes);
    if (!n_fft || !hop) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, !n_fft ? "n_fft" : "hop");
    if (B < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d, at least 1 item needed", fn, B);
    if (L < 1 || L > kMelLossMaxL) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L=%d samples, 1 to 2^30 supported", fn, L);
    for (int r = 0; r < n_res; ++r) {
        if (!mel_loss_n_ok(n_fft[r]))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft[%d]=%d is not a power of two in [%d, %d]", fn, r, n_fft[r], kMelLossMinN,
                             kMelLossMaxN);
        if (hop[r] < 1 || hop[r] > n_fft[r])
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: hop[%d]=%d is outside [1, n_fft=%d]", fn, r, hop[r], n_fft[r]);
        T[r] = mel_loss_frames(n_fft[r], hop[r], L);
        if (T[r] < 1)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L=%d samples are fewer than one frame of resolution %d (n_fft=%d, hop=%d)", fn,
                             L, r, n_fft[r], hop[r]);
        if (tables) {
            if (!tables[r]) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables[%d] is NULL", fn, r);
            if ((uintptr_t)tables[r] % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables[%d] must be 16-byte aligned", fn, r);
        }
        if ((long long)B * T[r] > 0x7fffffffll)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d x %d frames of resolution %d exceed 2^31 - 1 CTAs", fn, B, T[r], r);
    }
    if ((long long)B * ((L + 255) / 256) > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d x %d sample blocks exceed 2^31 - 1 CTAs", fn, B, (L + 255) / 256);
    return MG_OK;
}

void mel_loss_workspace(int n_res, const int *n_fft, int B, const int *T, size_t *fwd, size_t *bwd) {
    size_t f = 0, w = 0;
    for (int r = 0; r < n_res; ++r) {
        f += round256((size_t)B * T[r] * sizeof(float));
        const size_t d = (size_t)B * T[r] * n_fft[r] * sizeof(float);
        w = d > w ? d : w;
    }
    *fwd = f;
    *bwd = w;
}

int launch_mel_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                            int B, int L, const int *T, float *loss, void *workspace, cudaStream_t s) {
    MelLossFinishArgs a{};
    a.n_res = n_res;
    char *ws = reinterpret_cast<char *>(workspace);
    size_t off = 0;
    for (int r = 0; r < n_res; ++r) {
        const int BT = B * T[r], pad = (n_fft[r] - hop[r]) / 2;
        float *part = reinterpret_cast<float *>(ws + off);
        off += round256((size_t)BT * sizeof(float));
        const float *tab = reinterpret_cast<const float *>(tables[r]);
        a.part[r] = part;
        a.n_mels[r] = reinterpret_cast<const int *>(tab + 2 * n_fft[r]);
        a.bt[r] = BT;
        switch (n_fft[r]) {
#define MG_MEL_LOSS_FWD(NN)                                                                                                       \
    case NN: mel_loss_fwd_kernel<NN><<<(unsigned)BT, 256, mel_loss_fwd_smem<NN>(), s>>>(tab, x, y, part, L, hop[r], pad, T[r]); break;
            MG_MEL_LOSS_FWD(128) MG_MEL_LOSS_FWD(256) MG_MEL_LOSS_FWD(512) MG_MEL_LOSS_FWD(1024) MG_MEL_LOSS_FWD(2048)
#undef MG_MEL_LOSS_FWD
        }
        MG_CUDA_TRY(cudaGetLastError());
    }
    mel_loss_finish_kernel<<<1, 1024, 0, s>>>(a, loss);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

int launch_mel_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                             int B, int L, const int *T, const float *grad, float *grad_x, void *workspace, cudaStream_t s) {
    float *dframe = reinterpret_cast<float *>(workspace);
    for (int r = 0; r < n_res; ++r) {
        const float *tab = reinterpret_cast<const float *>(tables[r]);
        const int pad = (n_fft[r] - hop[r]) / 2;
        const unsigned BT = (unsigned)(B * T[r]);
        switch (n_fft[r]) {
#define MG_MEL_LOSS_BWD(NN)                                                                                                      \
    case NN:                                                                                                                     \
        mel_loss_bwd_frame_kernel<NN><<<BT, 256, mel_loss_bwd_smem<NN>(), s>>>(tab, x, y, grad, n_res, dframe, L, hop[r], pad, T[r]); \
        break;
            MG_MEL_LOSS_BWD(128) MG_MEL_LOSS_BWD(256) MG_MEL_LOSS_BWD(512) MG_MEL_LOSS_BWD(1024) MG_MEL_LOSS_BWD(2048)
#undef MG_MEL_LOSS_BWD
        }
        MG_CUDA_TRY(cudaGetLastError());
        mel_loss_bwd_gather_kernel<<<(unsigned)((long long)B * ((L + 255) / 256)), 256, 0, s>>>(dframe, grad_x, L, n_fft[r], hop[r], pad,
                                                                                                T[r], r > 0);
        MG_CUDA_TRY(cudaGetLastError());
    }
    return MG_OK;
}

}  // namespace mg
