// Streaming denoiser (mg_denoise_stream_*, contract in include/melgan_b200.h): the batch denoiser of mg_denoise.cu applied
// to live audio, many sessions per step, each denoised sample emitted once final.
//
// With N = n_fft, H = hop and R the samples a session has received, frame t reads samples [t H - N/2, t H + N/2)
// reflected at 0 (frame 0 reads 0 .. N/2), so an open session can compute frames 0 .. q, q = floor((R - N/2) / H), once
// R > N/2.  Output sample j sums frames t0(j) .. floor((j + N/2) / H), so the samples below
//   E(R) = 0 if R <= N/2, else clamp((q + 1) H - N/2, 0, R)
// are final: neither the utterance's length nor the envelope's edge enters them.  At END (length L) the frames up to
// floor(L / H) are computed reflecting at L and every sample is emitted.  The host derives everything from R alone:
// frames computed F(R) = q + 1, samples emitted E(R), and the first sample a later frame can read, lo = max(0, F H - N/2 - 1)
// (frame floor(L / H) reflects back to sample L - N/2 - 1 when H divides L, one left of its own window).
//
// A step is three launches on the caller's stream, each skipped when it has no work:
//   denoise_stream_window_kernel: per session, its tail [lo, R) then its new samples into a contiguous window, and the
//     next tail [lo', R') into the other half of a two-slot store (no launch reads what it writes);
//   denoise_stream_frame_kernel<N>: one CTA per newly computable frame, numbered through RunTable::voices (units: frames,
//     blob: the session's bias row), computed by denoise_frame (mg_denoise.cuh), the batch kernel's own code, reading the
//     window at offset t H - lo (with lo > 0 no new frame reaches below sample 1, so the reflection at 0 never applies
//     there, and the reflection at L is the same in window coordinates), into slot t mod K of the session's frame ring;
//   denoise_stream_ola_kernel<S>: one thread per newly final sample, frame_gather_env over the ring (FramesRing), the
//     quotient stored as audio_sample<S> into the caller's row.
// The ring holds the frames pending samples still need, at most ceil(N / H) - 1, plus one step's new frames.
#include <math.h>

#include <algorithm>
#include <new>
#include <string.h>

#include "mg_common.cuh"
#include "mg_denoise.cuh"
#include "mg_frame_loss.cuh"

namespace mg {
namespace {

constexpr int kMaxPush = 1 << 20;

struct WinJob {
    int slot, tin, tout, tlen, nnew, keep;  // keep >= 0: window positions [keep, tlen + nnew) become the tail (half tout)
};
struct WinTable {
    WinJob job[MG_GEN_RAGGED_MAX_B];
};
struct FrameJob {
    int slot, t0, L, lo;  // frames t0 .. of the slot, its window starting at sample lo, reflected at sample lo + L
};
struct FrameTable {
    FrameJob job[MG_GEN_RAGGED_MAX_B];
};
struct OlaJob {
    int slot, e0, count, T;  // samples [e0, e0 + count) of the slot, frames computed so far T
};
struct OlaTable {
    OlaJob job[MG_GEN_RAGGED_MAX_B];
};

// memory-bound: one CTA row (blockIdx.y) per session, grid-stride over its window
__global__ void __launch_bounds__(256) denoise_stream_window_kernel(float *tails, int S, int N, const float *__restrict__ in,
                                                                    long long in_stride, float *__restrict__ win, int wcap,
                                                                    const __grid_constant__ WinTable t) {
    const WinJob j = t.job[blockIdx.y];
    const float *tin = tails + (size_t)(j.tin * S + j.slot) * N;
    float *tout = tails + (size_t)(j.tout * S + j.slot) * N;
    const float *s = in + (size_t)j.slot * in_stride - j.tlen;
    float *w = win + (size_t)j.slot * wcap;
    const int len = j.tlen + j.nnew;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < len; p += gridDim.x * blockDim.x) {
        const float v = p < j.tlen ? tin[p] : s[p];
        w[p] = v;
        if (j.keep >= 0 && p >= j.keep) tout[p - j.keep] = v;
    }
}

template <int N>
__global__ void __launch_bounds__(128) denoise_stream_frame_kernel(const float *__restrict__ tab, const float *__restrict__ windows,
                                                                   int wcap, int hop, float strength, float *__restrict__ ring, int K,
                                                                   const __grid_constant__ RunTable run,
                                                                   const __grid_constant__ FrameTable ft) {
    __shared__ __align__(16) float2 buf[N];
    __shared__ __align__(16) float2 Y[N / 2 + 1];
    const int lt = threadIdx.x, f = blockIdx.x;
    const RunPos at = run.find(f);  // no gaps: every CTA is a frame of some session
    const FrameJob j = ft.job[at.item];
    const int t = j.t0 + at.unit;
    const float *__restrict__ b = run.blob_at(f);
    const float *src = windows + (size_t)j.slot * wcap;  // (the macro's own names, e.g. win, must not appear in its arguments)
    float *dst = ring + ((size_t)j.slot * K + t % K) * N;
    MG_DENOISE_FRAME(N, tab, src, j.L, t * hop - j.lo, strength, b, dst, lt, buf, Y)
}

template <class S>
__global__ void __launch_bounds__(256) denoise_stream_ola_kernel(const float *__restrict__ tab, const float *__restrict__ ring, int N,
                                                                 int hop, int K, S *__restrict__ out, long long out_stride,
                                                                 const __grid_constant__ OlaTable t) {
    const OlaJob j = t.job[blockIdx.y];
    const FramesRing frame{ring + (size_t)j.slot * K * N, N, K};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < j.count; i += gridDim.x * blockDim.x) {
        float acc, env, v = 0.f;
        if (frame_gather_env(frame, tab, j.e0 + i + N / 2, N, hop, j.T, acc, env)) v = acc / env;
        out[(size_t)j.slot * out_stride + i] = audio_sample<S>(v);
    }
}

long long align256(long long v) { return (v + 255) / 256 * 256; }

struct Layout {
    long long tails, win, ring, total;
    int wcap, K;
};

// frame ring slots: the ceil(N / H) - 1 frames pending samples can still need, plus the most one step can add
// (floor((P + N/2) / H) + 1, at END)
Layout layout(int N, int H, int S, int P) {
    Layout L;
    L.wcap = (N + P + 63) / 64 * 64;  // a window: a tail of at most N samples plus one push
    L.K = (N + H - 1) / H + (P + N / 2) / H + 1;
    L.tails = 0;
    L.win = align256(L.tails + 4ll * 2 * S * N);
    L.ring = align256(L.win + 4ll * S * L.wcap);
    L.total = align256(L.ring + 4ll * S * L.K * N);
    return L;
}

bool geometry_ok(int N, int H, int S, int P) {
    return dn_n_ok(N) && H >= 1 && H <= N && S >= 1 && S <= MG_GEN_RAGGED_MAX_B && P >= 1 && P <= kMaxPush;
}

// an open session's counters after R samples
long long frames_open(int N, int H, long long R) { return R > N / 2 ? (R - N / 2) / H + 1 : 0; }
long long emitted_open(int N, int H, long long R) {
    if (R <= N / 2) return 0;
    const long long e = frames_open(N, H, R) * H - N / 2;
    return e < 0 ? 0 : e > R ? R : e;
}
// the first sample a frame >= F can read (F H - N/2, one less for the END frame that reflects at L = F H)
long long first_read(int N, int H, long long F) { return F * H - N / 2 - 1 > 0 ? F * H - N / 2 - 1 : 0; }
// the first frame output sample e sums
long long first_frame(int N, int H, long long e) { return e + N / 2 >= N ? (e + N / 2 - N) / H + 1 : 0; }

struct Plan {
    int n_win, n_frame, n_ola, frames;
    WinTable win;
    FrameTable fr;
    OlaTable ola;
    int lens[MG_GEN_RAGGED_MAX_B], voice[MG_GEN_RAGGED_MAX_B];  // per frame item: new frames, bias row
    int max_win, max_out;
    long long R[MG_GEN_RAGGED_MAX_B];
    unsigned char par[MG_GEN_RAGGED_MAX_B];
    int bound[MG_GEN_RAGGED_MAX_B];
};

}  // namespace
}  // namespace mg

using namespace mg;

struct mg_denoise_stream {
    int N, H, W, S, P;
    float strength;
    char *state;
    Layout L;
    std::vector<double> w2, full;  // the window's squares and per-residue sums (the NOLA check at END)
    long long R[MG_GEN_RAGGED_MAX_B];  // per slot: samples received by its open utterance (0: none open)
    unsigned char par[MG_GEN_RAGGED_MAX_B];  // which half of the tail store holds the slot's tail
    int voice[MG_GEN_RAGGED_MAX_B];  // per slot: the bias row its open utterance is bound to (-1: none open)
    bool dry;
    Plan plan;
};

namespace mg {
namespace {

// Argument checks of a step (no CUDA call), then the plan: the launches, the new counters and the slots' voices.
int plan_step(const char *fn, const mg_denoise_stream *s, int n_voices, const int *voice, const int *in_samples, long long in_stride,
              const int *flags, int n, int *out_samples, Plan &p) {
    if (!s || !in_samples || !out_samples) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if (n < 0 || n > s->S) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n = %d is outside [0, max_sessions = %d]", fn, n, s->S);
    if (n_voices < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_voices = %d, need at least 1", fn, n_voices);
    const int N = s->N, H = s->H;
    for (int i = 0; i < n; ++i) {
        const int fl = flags ? flags[i] : 0;
        const int v = voice ? voice[i] : 0;
        if (v < 0 || v >= n_voices)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: voice[%d] = %d is outside [0, n_voices = %d)", fn, i, v, n_voices);
        if (!(fl & MG_GEN_STREAM_RESET) && s->R[i] > 0 && v != s->voice[i])
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: voice[%d] = %d, but slot %d's open utterance is bound to voice %d (a slot changes voice only "
                             "with MG_GEN_STREAM_RESET or after MG_GEN_STREAM_END)",
                             fn, i, v, i, s->voice[i]);
        const int m = in_samples[i];
        if (m < 0 || m > s->P)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: in_samples[%d] = %d is outside [0, max_push_samples = %d]", fn, i, m, s->P);
        if (m > in_stride)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: in_samples[%d] = %d exceeds in_stride = %lld", fn, i, m, in_stride);
        if (fl & ~(MG_GEN_STREAM_END | MG_GEN_STREAM_RESET))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: flags[%d] = %d has bits other than MG_GEN_STREAM_END | MG_GEN_STREAM_RESET", fn, i, fl);
        const long long R1 = ((fl & MG_GEN_STREAM_RESET) ? 0 : s->R[i]) + m;
        if (R1 > kDnMaxL)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: slot %d's utterance reaches %lld samples, at most 2^30 supported", fn, i, R1);
        if (!(fl & MG_GEN_STREAM_END)) continue;
        if (R1 == 0) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: MG_GEN_STREAM_END on slot %d, which has no samples", fn, i);
        if (R1 <= N / 2)
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: slot %d's utterance ends at L = %lld samples; reflect padding by n_fft/2 = %d needs more", fn, i, R1,
                             N / 2);
        const long long at = dn_nola_fail(s->w2, s->full, N, H, (int)R1);
        if (at >= 0)
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: (n_fft=%d, hop=%d, win_length=%d) leaves the window-square envelope below 1e-11 at sample %lld of "
                             "slot %d's %lld-sample utterance (torch.istft's NOLA condition)",
                             fn, N, H, s->W, at, i, R1);
    }
    p.n_win = p.n_frame = p.n_ola = p.frames = p.max_win = p.max_out = 0;
    memcpy(p.R, s->R, sizeof(p.R));
    memcpy(p.par, s->par, sizeof(p.par));
    memcpy(p.bound, s->voice, sizeof(p.bound));
    for (int i = 0; i < n; ++i) {
        const int fl = flags ? flags[i] : 0, v = voice ? voice[i] : 0, m = in_samples[i];
        const bool end = fl & MG_GEN_STREAM_END;
        const long long R0 = (fl & MG_GEN_STREAM_RESET) ? 0 : s->R[i], R1 = R0 + m;
        const long long F0 = frames_open(N, H, R0), E0 = emitted_open(N, H, R0), lo = first_read(N, H, F0);
        const long long F1 = end ? dn_frames(H, (int)R1) : frames_open(N, H, R1), E1 = end ? R1 : emitted_open(N, H, R1);
        const long long lo1 = first_read(N, H, F1);
        if (R0 - lo > N || R1 - lo > s->L.wcap || (!end && R1 - lo1 > N) || F1 - first_frame(N, H, E0) > s->L.K)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: internal: window or frame ring exceeded at slot %d", fn, i);
        if (m > 0 || F1 > F0) {
            const int par = p.par[i];
            p.win.job[p.n_win++] = WinJob{i, par, 1 - par, (int)(R0 - lo), m, end ? -1 : (int)(lo1 - lo)};
            if (!end) p.par[i] = (unsigned char)(1 - par);
            p.max_win = std::max(p.max_win, (int)(R1 - lo));
        }
        if (F1 > F0) {
            p.lens[p.n_frame] = (int)(F1 - F0);
            p.voice[p.n_frame] = v;
            p.fr.job[p.n_frame++] = FrameJob{i, (int)F0, (int)(R1 - lo), (int)lo};
            p.frames += (int)(F1 - F0);
        }
        out_samples[i] = (int)(E1 - E0);
        if (E1 > E0) {
            p.ola.job[p.n_ola++] = OlaJob{i, (int)E0, (int)(E1 - E0), (int)F1};
            p.max_out = std::max(p.max_out, (int)(E1 - E0));
        }
        p.R[i] = end ? 0 : R1;
        p.bound[i] = p.R[i] > 0 ? v : -1;  // bound by the step that opens the utterance, free once it ends
    }
    return MG_OK;
}

void commit(mg_denoise_stream *s, const Plan &p) {
    memcpy(s->R, p.R, sizeof(s->R));
    memcpy(s->par, p.par, sizeof(s->par));
    memcpy(s->voice, p.bound, sizeof(s->voice));
}

int grid_x(int elems) { return std::max(1, std::min(64, (elems + 1023) / 1024)); }

int step(const char *fn, mg_denoise_stream *s, const void *tables, const float *bias, int n_voices, const int *voice, const float *audio_in,
         long long in_stride, const int *in_samples, const int *flags, int n, void *out, int *out_samples, cudaStream_t st, bool pcm) {
    if (!s) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if (s->dry) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: this handle was advanced by mg_denoise_stream_dry_step", fn);
    int rc;
    if ((rc = dn_check_pointer(fn, "tables", tables, 16)) || (rc = dn_check_pointer(fn, "bias", bias, 4)) ||
        (rc = dn_check_pointer(fn, "out", out, pcm ? 2 : 4)))
        return rc;
    bool any = false;
    for (int i = 0; in_samples && i < n && i < s->S; ++i) any |= in_samples[i] > 0;
    if (any && (rc = dn_check_pointer(fn, "audio_in", audio_in, 4))) return rc;
    if (in_stride < 0) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: in_stride = %lld is negative", fn, in_stride);
    Plan &p = s->plan;
    if ((rc = plan_step(fn, s, n_voices, voice, in_samples, in_stride, flags, n, out_samples, p))) return rc;

    const int N = s->N;
    float *tails = reinterpret_cast<float *>(s->state + s->L.tails), *win = reinterpret_cast<float *>(s->state + s->L.win);
    float *ring = reinterpret_cast<float *>(s->state + s->L.ring);
    const float *tab = reinterpret_cast<const float *>(tables);
    if (p.n_win) {
        denoise_stream_window_kernel<<<dim3(grid_x(p.max_win), p.n_win), 256, 0, st>>>(tails, s->S, N, audio_in, in_stride, win,
                                                                                         s->L.wcap, p.win);
        MG_CUDA_TRY(cudaGetLastError());
    }
    if (p.n_frame) {
        const int M1 = N / 2 + 1;
        std::vector<const float *> rows(n_voices);
        for (int v = 0; v < n_voices; ++v) rows[v] = bias + (size_t)v * M1;
        RunTable run = RunTable::voices(p.lens, p.n_frame, 0, rows.data(), p.voice);
        run.set_units([](int frames) { return frames; });
        switch (N) {
#define MG_DNS_FRAME(NN)                                                                                                    \
    case NN:                                                                                                                \
        denoise_stream_frame_kernel<NN><<<(unsigned)p.frames, 128, 0, st>>>(tab, win, s->L.wcap, s->H, s->strength, ring, s->L.K, \
                                                                            run, p.fr);                                     \
        break;
            MG_DNS_FRAME(128) MG_DNS_FRAME(256) MG_DNS_FRAME(512) MG_DNS_FRAME(1024) MG_DNS_FRAME(2048)
#undef MG_DNS_FRAME
        }
        MG_CUDA_TRY(cudaGetLastError());
    }
    if (p.n_ola) {
        const dim3 grid(std::min(256, (p.max_out + 255) / 256), p.n_ola);
        const long long stride = mg_denoise_stream_max_out(N, s->H, s->P);
        if (pcm)
            denoise_stream_ola_kernel<int16_t><<<grid, 256, 0, st>>>(tab, ring, N, s->H, s->L.K, (int16_t *)out, stride, p.ola);
        else
            denoise_stream_ola_kernel<float><<<grid, 256, 0, st>>>(tab, ring, N, s->H, s->L.K, (float *)out, stride, p.ola);
        MG_CUDA_TRY(cudaGetLastError());
    }
    commit(s, p);
    return MG_OK;
}

}  // namespace
}  // namespace mg

extern "C" {

int mg_denoise_stream_max_out(int n_fft, int hop, int max_push_samples) {
    if (!geometry_ok(n_fft, hop, 1, max_push_samples)) return 0;
    return max_push_samples + n_fft - 1;
}

size_t mg_denoise_stream_state_bytes(int n_fft, int hop, int max_sessions, int max_push_samples) {
    if (!geometry_ok(n_fft, hop, max_sessions, max_push_samples)) return 0;
    return (size_t)layout(n_fft, hop, max_sessions, max_push_samples).total;
}

int mg_denoise_stream_create(mg_denoise_stream **out, int n_fft, int hop, int win_length, int max_sessions, int max_push_samples,
                             float strength, void *state, size_t state_bytes) {
    const char *fn = "mg_denoise_stream_create";
    if (!out) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: out is NULL", fn);
    *out = nullptr;
    if (!dn_n_ok(n_fft))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_fft=%d is not a power of two in [%d, %d]", fn, n_fft, kDnMinN, kDnMaxN);
    if (win_length < 1 || win_length > n_fft)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: win_length=%d is outside [1, n_fft=%d]", fn, win_length, n_fft);
    if (hop < 1 || hop > win_length)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: hop=%d is outside [1, win_length=%d] (torch.istft needs hop <= win_length)", fn,
                         hop, win_length);
    if (max_sessions < 1 || max_sessions > MG_GEN_RAGGED_MAX_B)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: max_sessions = %d is outside [1, MG_GEN_RAGGED_MAX_B = %d]", fn, max_sessions,
                         MG_GEN_RAGGED_MAX_B);
    if (max_push_samples < 1 || max_push_samples > kMaxPush)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: max_push_samples = %d is outside [1, 2^20]", fn, max_push_samples);
    if (!isfinite(strength)) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: strength=%g is not finite", fn, (double)strength);
    std::vector<double> w2, full;
    dn_window_sq(n_fft, hop, win_length, w2, full);
    for (int q = 0; q < (int)full.size(); ++q)
        if (full[q] < kDnNola)
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: (n_fft=%d, hop=%d, win_length=%d) leaves the window-square envelope below 1e-11 at every sample "
                             "%d mod %d inside an utterance (torch.istft's NOLA condition)",
                             fn, n_fft, hop, win_length, q, hop);
    int rc;
    if ((rc = dn_check_pointer(fn, "state", state, 256))) return rc;
    const size_t need = mg_denoise_stream_state_bytes(n_fft, hop, max_sessions, max_push_samples);
    if (state_bytes < need) return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: state of %zu bytes, %zu needed", fn, state_bytes, need);
    mg_denoise_stream *s = new (std::nothrow) mg_denoise_stream();
    if (!s) return set_error(MG_ERR_OUT_OF_MEMORY, "%s: host allocation failed", fn);
    s->N = n_fft;
    s->H = hop;
    s->W = win_length;
    s->S = max_sessions;
    s->P = max_push_samples;
    s->strength = strength;
    s->state = (char *)state;
    s->L = layout(n_fft, hop, max_sessions, max_push_samples);
    s->w2 = w2;
    s->full = full;
    for (int i = 0; i < MG_GEN_RAGGED_MAX_B; ++i) s->voice[i] = -1;
    *out = s;
    return MG_OK;
}

void mg_denoise_stream_destroy(mg_denoise_stream *s) { delete s; }

int mg_denoise_stream_step(mg_denoise_stream *s, const void *tables, const float *bias, int n_voices, const int *voice,
                           const float *audio_in, long long in_stride, const int *in_samples, const int *flags, int n, float *out,
                           int *out_samples, void *stream) {
    return step("mg_denoise_stream_step", s, tables, bias, n_voices, voice, audio_in, in_stride, in_samples, flags, n, out, out_samples,
                (cudaStream_t)stream, false);
}

int mg_denoise_stream_step_pcm16(mg_denoise_stream *s, const void *tables, const float *bias, int n_voices, const int *voice,
                                 const float *audio_in, long long in_stride, const int *in_samples, const int *flags, int n, int16_t *out,
                                 int *out_samples, void *stream) {
    return step("mg_denoise_stream_step_pcm16", s, tables, bias, n_voices, voice, audio_in, in_stride, in_samples, flags, n, out,
                out_samples, (cudaStream_t)stream, true);
}

int mg_denoise_stream_dry_step(mg_denoise_stream *s, int n_voices, const int *voice, const int *in_samples, const int *flags, int n,
                               int *out_samples, int *new_frames) {
    const char *fn = "mg_denoise_stream_dry_step";
    if (!s) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    int rc = plan_step(fn, s, n_voices, voice, in_samples, (long long)s->P, flags, n, out_samples, s->plan);
    if (rc) return rc;
    s->dry = true;
    if (new_frames) *new_frames = s->plan.frames;
    commit(s, s->plan);
    return MG_OK;
}

}  // extern "C"
