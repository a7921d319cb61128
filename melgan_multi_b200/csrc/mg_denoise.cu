// Denoiser (WaveGlow's Denoiser): subtract a vocoder's bias spectrum from its audio.  Per item i (its first L_i samples),
// analysis (n_fft N, hop H, the periodic Hann window of the STFT-loss table) and bias row b = bias[voice[i]]:
//   S = torch.stft(a_i, N, H, W, hann(W), center=True, pad_mode="reflect"), T_i = 1 + L_i / H frames;
//   Y = max(|S| - strength b, 0) S / |S|  (S / |S| := 1 where |S| = 0);  out_i = torch.istft(Y, ..., length=L_i), 0 after.
//
// denoise_bias_kernel<N>: one CTA (128 threads) per audio row: |X[k]|, k = 0..N/2, of the row's frame 0.
// denoise_frame_kernel<N>: one CTA (128 threads) per (item, frame), the frames of all items numbered consecutively
//   through a RunTable (units: frames; len: the item's samples; blob: the run's bias row), so frame f's N floats sit at
//   f N in the workspace.  The frame is read reflecting at the item's own length, through the forward FFT and split of
//   mg_stft_frame.cuh; each bin becomes Y; real_unsplit and the inverse Stockham pass give the real frame, which is
//   scaled by 1 / M (M = N / 2: the pass returns M times the samples; exact, M is a power of two) and multiplied by the
//   window.  The frame's code is MG_DENOISE_FRAME (mg_denoise.cuh), which the streaming denoiser's frame kernel expands too.
// denoise_ola_kernel<S>: one thread per output sample: the frames covering its padded position and the window-square
//   envelope, both summed in ascending frame order (frame_gather_env), then their quotient stored as audio_sample<S>
//   (S float or int16_t); 0 from L_i to L_max, and 0 where no frame reaches (torch.istft's zero fill past the last frame
//   when hop > N / 2).
// No atomics: the same inputs give the same bits on every run.  NaN and Inf are not clamped away: the clamp is written
// `x < 0 ? 0 : x`, so a NaN bin stays NaN and spreads over its frame and the samples that frame reaches.
#include <math.h>

#include <vector>

#include "mg_common.cuh"
#include "mg_denoise.cuh"
#include "mg_fft.cuh"
#include "mg_frame_loss.cuh"
#include "mg_stft_frame.cuh"

namespace mg {

template <int N>
__global__ void __launch_bounds__(128) denoise_bias_kernel(const float *__restrict__ tab, const float *__restrict__ audio, int L,
                                                           float *__restrict__ bias) {
    constexpr int M = N / 2;
    __shared__ __align__(16) float2 buf[2 * M];
    const int lt = threadIdx.x;
    const float2 *tw = reinterpret_cast<const float2 *>(tab + N);
    const float2 *Z = stft_frame<N>(tab, tw, audio + (size_t)blockIdx.x * L, L, 0, lt, buf, buf + M);
    for (int k = lt; k <= M; k += 128) {
        const float2 X = stft_bin<N>(Z, tw, k);
        bias[(size_t)blockIdx.x * (M + 1) + k] = sqrtf(X.x * X.x + X.y * X.y);
    }
}

template <int N>
__global__ void __launch_bounds__(128) denoise_frame_kernel(const float *__restrict__ tab, const float *__restrict__ audio, int hop,
                                                            float strength, float *__restrict__ frames,
                                                            const __grid_constant__ RunTable run) {
    __shared__ __align__(16) float2 buf[N];
    __shared__ __align__(16) float2 Y[N / 2 + 1];
    const int lt = threadIdx.x, f = blockIdx.x;
    const RunPos at = run.find(f);  // the grid is first[n] frames, with no gaps: every frame belongs to an item
    const float *__restrict__ b = run.blob_at(f);
    MG_DENOISE_FRAME(N, tab, audio + (size_t)at.item * run.stride, at.len, at.unit * hop, strength, b, frames + (size_t)f * N, lt, buf, Y)
}

template <class S>
__global__ void __launch_bounds__(256) denoise_ola_kernel(const float *__restrict__ tab, const float *__restrict__ frames, int N, int hop,
                                                          S *__restrict__ out, const __grid_constant__ RunTable run) {
    const int chunks = (run.stride + 255) >> 8;
    const int b = (int)blockIdx.x / chunks, i = (((int)blockIdx.x - b * chunks) << 8) + (int)threadIdx.x;
    if (i >= run.stride) return;
    int r = 0, hi = run.n;  // the run of item b: item0[r] <= b < item0[r + 1]
    while (hi - r > 1) {
        const int m = (r + hi) >> 1;
        if (run.item0[m] <= b) r = m;
        else hi = m;
    }
    float v = 0.f;
    if (i < run.len[r]) {
        const int T = run.per[r];
        const float *db = frames + ((size_t)run.first[r] + (size_t)(b - run.item0[r]) * T) * N;
        float acc, env;
        if (frame_gather_env(db, tab, i + N / 2, N, hop, T, acc, env)) v = acc / env;
    }
    out[(size_t)b * run.stride + i] = audio_sample<S>(v);
}

// ---- host side -------------------------------------------------------------------------------------------------------

void dn_window_sq(int n_fft, int hop, int win_length, std::vector<double> &w2, std::vector<double> &full) {
    const double pi = 3.14159265358979323846;
    const int left = (n_fft - win_length) / 2;
    w2.assign(n_fft, 0.0);
    for (int j = 0; j < win_length; ++j) {
        const double w = win_length == 1 ? 1.0 : 0.5 - 0.5 * cos(2 * pi * j / win_length);
        w2[left + j] = w * w;
    }
    full.assign(std::min(hop, n_fft), 0.0);
    for (int n = 0; n < n_fft; ++n) full[n % hop] += w2[n];
}

// float64 window-square envelope of torch.istft at padded position p of a T-frame signal, w2 = the squared window
static double dn_env_at(const std::vector<double> &w2, int N, int hop, int T, long long p) {
    const long long t1 = std::min<long long>(p / hop, T - 1), t0 = p >= N ? (p - N) / hop + 1 : 0;
    double e = 0.0;
    for (long long t = t0; t <= t1; ++t) e += w2[(size_t)(p - t * hop)];
    return e;
}

// the first output sample (of an L-sample item) whose envelope is below 1e-11, or -1: torch.istft's NOLA check, over the
// output positions some frame reaches.  Interior positions (every frame position n = p mod hop present) read the
// per-residue sums `full`, so the cost is O(N^2 / hop + N), not O(L).
long long dn_nola_fail(const std::vector<double> &w2, const std::vector<double> &full, int N, int hop, int L) {
    const int T = dn_frames(hop, L);
    const long long start = N / 2, end = std::min<long long>((long long)N / 2 + L, (long long)N + (long long)hop * (T - 1));
    const long long i0 = std::max<long long>(start, N - 1), i1 = std::min<long long>(end, (long long)hop * T);  // interior
    auto full_at = [&](long long q) { return q < N ? full[(size_t)q] : 0.0; };  // (residues past N: no frame position)
    for (long long p = start; p < end; ++p) {
        if (p < i0 || p >= i1) {
            if (dn_env_at(w2, N, hop, T, p) < kDnNola) return p - start;
            continue;
        }
        if (i1 - i0 >= hop) {  // a whole period: every residue occurs (the scan stops at the first residue >= N)
            for (long long q = 0; q < hop; ++q)
                if (full_at(q) < kDnNola) return i0 + ((q - i0 % hop) % hop + hop) % hop - start;
        } else {
            for (long long c = i0; c < i1; ++c)
                if (full_at(c % hop) < kDnNola) return c - start;
        }
        p = i1 - 1;
    }
    return -1;
}

int dn_check_pointer(const char *fn, const char *name, const void *p, unsigned align) {
    if (!p) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, name);
    if ((uintptr_t)p % align) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s must be %u-byte aligned", fn, name, align);
    return MG_OK;
}

// the analysis and batch geometry; *bytes gets the frame workspace, sum_i (1 + L_i / hop) n_fft floats
static int dn_check_batch(const char *fn, int n_fft, int hop, int B, int L_max, const int *lengths, bool voiced, size_t *bytes) {
    if (!dn_n_ok(n_fft))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft=%d is not a power of two in [%d, %d]", fn, n_fft, kDnMinN, kDnMaxN);
    if (hop < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: hop=%d, at least 1 needed", fn, hop);
    if (B < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d, at least 1 item needed", fn, B);
    if (L_max > kDnMaxL) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L_max=%d samples, at most 2^30 supported", fn, L_max);
    if (L_max <= n_fft / 2)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L_max=%d samples, reflect padding by n_fft/2=%d needs more", fn, L_max, n_fft / 2);
    if ((lengths || voiced) && B > MG_GEN_RAGGED_MAX_B)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d exceeds MG_GEN_RAGGED_MAX_B=%d for a ragged or voiced batch", fn, B,
                         MG_GEN_RAGGED_MAX_B);
    long long frames = 0;
    for (int i = 0; i < B; ++i) {
        const int L = lengths ? lengths[i] : L_max;
        if (L <= n_fft / 2 || L > L_max)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: lengths[%d]=%d is outside (n_fft/2=%d, L_max=%d]", fn, i, L, n_fft / 2, L_max);
        frames += dn_frames(hop, L);
    }
    if (frames > 0x7fffffffll) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %lld frames exceed 2^31 - 1 CTAs", fn, frames);
    if ((long long)B * ((L_max + 255) / 256) > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B=%d x %d sample blocks exceed 2^31 - 1 CTAs", fn, B, (L_max + 255) / 256);
    *bytes = (size_t)frames * n_fft * sizeof(float);
    return MG_OK;
}

static int denoise_forward(const char *fn, const void *tables, int n_fft, int hop, int win_length, const float *audio, int B, int L_max,
                           const int *lengths, const float *bias, int n_voices, const int *voice, float strength, void *out, bool pcm,
                           void *workspace, size_t workspace_bytes, cudaStream_t s) {
    size_t need;
    int rc;
    if ((rc = dn_check_batch(fn, n_fft, hop, B, L_max, lengths, voice != nullptr, &need))) return rc;
    if (win_length < 1 || win_length > n_fft)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: win_length=%d is outside [1, n_fft=%d]", fn, win_length, n_fft);
    if (hop > win_length)  // torch.istft's own refusal
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: hop=%d exceeds win_length=%d (torch.istft needs hop <= win_length)", fn, hop,
                         win_length);
    if (n_voices < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_voices=%d, at least 1 needed", fn, n_voices);
    if (voice)
        for (int i = 0; i < B; ++i)
            if (voice[i] < 0 || voice[i] >= n_voices)
                return set_error(MG_ERR_INVALID_ARGUMENT, "%s: voice[%d]=%d is outside [0, n_voices=%d)", fn, i, voice[i], n_voices);
    if (!isfinite(strength)) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: strength=%g is not finite", fn, (double)strength);
    // torch.istft's NOLA refusal, in float64, once per distinct length
    std::vector<double> w2, full;
    dn_window_sq(n_fft, hop, win_length, w2, full);
    std::vector<int> seen;
    for (int i = 0; i < B; ++i) {
        const int L = lengths ? lengths[i] : L_max;
        bool dup = false;
        for (int v : seen) dup = dup || v == L;
        if (dup) continue;
        seen.push_back(L);
        const long long at = dn_nola_fail(w2, full, n_fft, hop, L);
        if (at >= 0)
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: (n_fft=%d, hop=%d, win_length=%d) leaves the window-square envelope below 1e-11 at sample %lld of a "
                             "%d-sample item (torch.istft's NOLA condition)",
                             fn, n_fft, hop, win_length, at, L);
        if (!lengths) break;
    }
    if ((rc = dn_check_pointer(fn, "tables", tables, 16)) || (rc = dn_check_pointer(fn, "audio", audio, 4)) ||
        (rc = dn_check_pointer(fn, "bias", bias, 4)) || (rc = dn_check_pointer(fn, "out", out, pcm ? 2 : 4)) ||
        (rc = dn_check_pointer(fn, "workspace", workspace, 16)))
        return rc;
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);

    const int M1 = n_fft / 2 + 1;
    RunTable run;
    if (!lengths && !voice) {
        run = RunTable::uniform(B, L_max, bias);
    } else {
        std::vector<const float *> rows(n_voices);
        for (int v = 0; v < n_voices; ++v) rows[v] = bias + (size_t)v * M1;
        run = RunTable::voices(lengths, B, L_max, rows.data(), voice);
    }
    run.set_units([hop](int L) { return dn_frames(hop, L); });
    const float *tab = reinterpret_cast<const float *>(tables);
    float *frames = reinterpret_cast<float *>(workspace);
    switch (n_fft) {
#define MG_DN_FRAME(NN) \
    case NN: denoise_frame_kernel<NN><<<(unsigned)run.first[run.n], 128, 0, s>>>(tab, audio, hop, strength, frames, run); break;
        MG_DN_FRAME(128) MG_DN_FRAME(256) MG_DN_FRAME(512) MG_DN_FRAME(1024) MG_DN_FRAME(2048)
#undef MG_DN_FRAME
    }
    MG_CUDA_TRY(cudaGetLastError());
    const unsigned blocks = (unsigned)((long long)B * ((L_max + 255) / 256));
    if (pcm) denoise_ola_kernel<int16_t><<<blocks, 256, 0, s>>>(tab, frames, n_fft, hop, (int16_t *)out, run);
    else denoise_ola_kernel<float><<<blocks, 256, 0, s>>>(tab, frames, n_fft, hop, (float *)out, run);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

}  // namespace mg

using namespace mg;

int mg_denoise_workspace_bytes(int n_fft, int hop, int B, int L_max, const int *lengths, size_t *bytes) {
    const char *fn = "mg_denoise_workspace_bytes";
    if (!bytes) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: bytes is NULL", fn);
    *bytes = 0;
    return dn_check_batch(fn, n_fft, hop, B, L_max, lengths, false, bytes);
}

int mg_denoise_bias(const void *tables, int n_fft, const float *audio, int n_rows, int L, float *bias, void *stream) {
    const char *fn = "mg_denoise_bias";
    int rc;
    if (!dn_n_ok(n_fft))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft=%d is not a power of two in [%d, %d]", fn, n_fft, kDnMinN, kDnMaxN);
    if (n_rows < 1 || n_rows > 65535) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_rows=%d is outside [1, 65535]", fn, n_rows);
    if (L <= n_fft / 2 || L > kDnMaxL)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: L=%d is outside (n_fft/2=%d, 2^30]", fn, L, n_fft / 2);
    if ((rc = dn_check_pointer(fn, "tables", tables, 16)) || (rc = dn_check_pointer(fn, "audio", audio, 4)) ||
        (rc = dn_check_pointer(fn, "bias", bias, 4)))
        return rc;
    const float *tab = reinterpret_cast<const float *>(tables);
    cudaStream_t s = (cudaStream_t)stream;
    switch (n_fft) {
#define MG_DN_BIAS(NN) \
    case NN: denoise_bias_kernel<NN><<<(unsigned)n_rows, 128, 0, s>>>(tab, audio, L, bias); break;
        MG_DN_BIAS(128) MG_DN_BIAS(256) MG_DN_BIAS(512) MG_DN_BIAS(1024) MG_DN_BIAS(2048)
#undef MG_DN_BIAS
    }
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

int mg_denoise_forward(const void *tables, int n_fft, int hop, int win_length, const float *audio, int B, int L_max, const int *lengths,
                       const float *bias, int n_voices, const int *voice, float strength, float *out, void *workspace,
                       size_t workspace_bytes, void *stream) {
    return denoise_forward("mg_denoise_forward", tables, n_fft, hop, win_length, audio, B, L_max, lengths, bias, n_voices, voice,
                           strength, out, false, workspace, workspace_bytes, (cudaStream_t)stream);
}

int mg_denoise_forward_pcm16(const void *tables, int n_fft, int hop, int win_length, const float *audio, int B, int L_max,
                             const int *lengths, const float *bias, int n_voices, const int *voice, float strength, int16_t *out,
                             void *workspace, size_t workspace_bytes, void *stream) {
    return denoise_forward("mg_denoise_forward_pcm16", tables, n_fft, hop, win_length, audio, B, L_max, lengths, bias, n_voices, voice,
                           strength, out, true, workspace, workspace_bytes, (cudaStream_t)stream);
}
