// Incremental vocoding of live mel streams (mg_gen_stream_*, contract in include/melgan_b200.h).
//
// A step runs the default chain's eight kernels through their own launchers, each on a ragged RunTable whose items are the
// sessions that have new exact outputs at that kernel.  An item is a WINDOW [lo, hi) of the kernel's input: the input tail
// the session keeps at that boundary (its left context) followed by the inputs that became final in this step.  A kernel
// zero-pads outside its items, so of the outputs of a window only these are exact (DESIGN.md §3.4, checked in float64 by
// tests/test_gen_stream.py):
//
//   kernel k              output/input   exact outputs of [lo, hi)      left reach in inputs
//   0 conv_pre            1              [lo + 3,  hi - 3)              3
//   1, 3 up0, up1         8              [8 lo + 4, 8 hi - 4)           (F - 4) / 8
//   2, 4, 6 res0..res2    1              [lo + 16, hi - 16)             16
//   5 up2                 2              [2 lo + 1, 2 hi - 1)           (F - 1) / 2
//   7 up3+res3+post       2              [2 lo + 20, 2 hi - 20)         (F - 20) / 2
//
// except at lo = 0 (exact from 0) and, once the session has ended, at hi = its full length (exact to the end): there the
// zero padding is the whole forward's.  Composed, audio sample j is final once 256 t - 1542 > j (t frames pushed).
//
// The host keeps, per session and boundary b (the input of kernel b; b = 8 is the audio), F[b] = the number of final
// positions, and derives every window, offset and count from them: a step never reads the device.  One window-assembly
// launch per boundary builds the windows of the kernel that follows it in the padded [item][C][stride] layout the kernel
// reads, and stores each session's next tail; the same kernel copies the newly final audio to the caller.
//
// Voices (mg_gen_stream_step_voices): each slot runs on the blob of the voice its utterance was opened with.  The planner
// walks the sessions by ascending voice, slot order within a voice, so every kernel's items come in voice runs and its
// RunTable::voices starts a new tile at each change of voice, as in mg_gen_forward_voices.  Tails, mel rows and audio
// rows stay indexed by slot: only the item numbering follows the walk.  With one voice the walk is slot order.
#include <algorithm>
#include <new>
#include <string.h>

#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {

namespace {

constexpr int kKernels = 8;
constexpr int kLookahead = 1542;  // 256 * t - F[8] for an open session with t >= 7 frames
// per boundary b = 0..8: channels, positions per mel frame, and positions not yet final in an open session (S t - F)
constexpr int kC[9] = {80, 512, 256, 256, 128, 128, 64, 64, 1};
constexpr int kScale[9] = {1, 1, 8, 8, 64, 64, 128, 128, 256};
constexpr int kReach[9] = {0, 3, 28, 44, 356, 372, 745, 761, 1542};
// per kernel: output positions per input position; the longest input tail an open session keeps at its input boundary
constexpr int kRatio[kKernels] = {1, 8, 1, 8, 1, 2, 1, 2};
constexpr int kTail[kKernels] = {6, 1, 32, 1, 32, 1, 32, 20};

long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// final outputs of kernel k from F final inputs of an open session
long long exact_hi(int k, long long F) {
    long long v = 0;
    switch (k) {
        case 0: v = F - 3; break;
        case 1: case 3: v = 8 * F - 4; break;
        case 2: case 4: case 6: v = F - 16; break;
        case 5: v = 2 * F - 1; break;
        case 7: v = 2 * F - 20; break;
    }
    return v > 0 ? v : 0;
}

// the largest window start lo whose outputs are exact from output position Fout on
long long need_lo(int k, long long Fout) {
    long long v = 0;
    switch (k) {
        case 0: v = Fout - 3; break;
        case 1: case 3: v = floor_div(Fout - 4, 8); break;
        case 2: case 4: case 6: v = Fout - 16; break;
        case 5: v = floor_div(Fout - 1, 2); break;
        case 7: v = floor_div(Fout - 20, 2); break;
    }
    return v > 0 ? v : 0;
}

int round16(long long v) { return (int)((v + 15) / 16 * 16); }

// window capacity (positions) at the input of kernel k for pushes of at most P frames: the tail plus what one step can
// make final there (S P, plus the look-ahead when the session ends)
int window_cap(int k, int P) { return round16(kTail[k] + (long long)kScale[k] * P + kReach[k]); }

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// One session's share of a window-assembly launch: positions [0, tlen) of the window come from its tail (slot tin of the
// tail store), positions [tlen, tlen + nnew) from item `src_item` of the source at offset src_off.  dst_item >= 0: the
// window is written as that item of the next kernel's input; keep >= 0: positions [keep, tlen + nnew) become the new
// tail (slot tout).
struct AsmJob {
    int tin, tout, tlen, src_item, src_off, nnew, dst_item, keep;
};
struct AsmTable {
    int n;
    AsmJob job[MG_GEN_RAGGED_MAX_B];
};

// Memory-bound: one CTA row (blockIdx.y) per job, grid-stride over its C x (tlen + nnew) positions, consecutive threads on
// consecutive positions of a channel row.  Every thread waits for the previous launch (PDL) before its first access, so the
// chain's ordering stays transitive.
__global__ void __launch_bounds__(256) stream_window_kernel(const float *__restrict__ tail_in, float *__restrict__ tail_out, int tail_cap,
                                                            const float *__restrict__ src, long long src_item_stride, int src_row,
                                                            float *__restrict__ dst, long long dst_item_stride, int dst_row, int C,
                                                            const __grid_constant__ AsmTable t) {
    tc::pdl_wait();
    tc::pdl_trigger();
    const AsmJob j = t.job[blockIdx.y];
    const int len = j.tlen + j.nnew, total = C * len;
    const float *tin = tail_in + (size_t)j.tin * C * tail_cap;
    float *tout = tail_out + (size_t)j.tout * C * tail_cap;
    const float *s = src + (size_t)j.src_item * src_item_stride + j.src_off - j.tlen;
    float *d = dst + (size_t)(j.dst_item > 0 ? j.dst_item : 0) * dst_item_stride;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int c = e / len, p = e - c * len;
        const float v = p < j.tlen ? tin[c * tail_cap + p] : s[(size_t)c * src_row + p];
        if (j.dst_item >= 0) d[(size_t)c * dst_row + p] = v;
        if (j.keep >= 0 && p >= j.keep) tout[c * tail_cap + p - j.keep] = v;
    }
}

// The audio copy of an int16 step (mg_gen_stream_step_pcm16): the last window-assembly launch's jobs (no tail, no
// kept positions, dst_row unused: one channel), storing pcm16 of each newly final sample into the caller's int16 row.
__global__ void __launch_bounds__(256) stream_audio_pcm16_kernel(const float *__restrict__ src, long long src_item_stride,
                                                                 int16_t *__restrict__ dst, long long dst_item_stride,
                                                                 const __grid_constant__ AsmTable t) {
    tc::pdl_wait();
    tc::pdl_trigger();
    const AsmJob j = t.job[blockIdx.y];
    const float *s = src + (size_t)j.src_item * src_item_stride + j.src_off;
    int16_t *d = dst + (size_t)j.dst_item * dst_item_stride;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < j.nnew; p += gridDim.x * blockDim.x) d[p] = pcm16(s[p]);
}

struct Copy {
    const float *tail_in = nullptr;
    float *tail_out = nullptr;
    int tail_cap = 1;
    const float *src = nullptr;
    long long src_item_stride = 0;
    int src_row = 0;
    float *dst = nullptr;
    long long dst_item_stride = 0;
    int dst_row = 0, C = 1;
};

int launch_window(const Copy &c, const AsmTable &t, long long max_elems, cudaStream_t s) {
    if (t.n == 0) return MG_OK;
    long long bx = (max_elems + 1023) / 1024;
    bx = bx < 1 ? 1 : bx > 64 ? 64 : bx;
    MG_CUDA_TRY(launch_ex(stream_window_kernel, dim3((unsigned)bx, (unsigned)t.n), dim3(256), 0, s, true, 1, c.tail_in, c.tail_out,
                          c.tail_cap, c.src, c.src_item_stride, c.src_row, c.dst, c.dst_item_stride, c.dst_row, c.C, t));
    return MG_OK;
}

int launch_audio_pcm16(const float *src, long long src_item_stride, int16_t *dst, long long dst_item_stride, const AsmTable &t,
                       long long max_elems, cudaStream_t s) {
    if (t.n == 0) return MG_OK;
    long long bx = (max_elems + 1023) / 1024;
    bx = bx < 1 ? 1 : bx > 64 ? 64 : bx;
    MG_CUDA_TRY(launch_ex(stream_audio_pcm16_kernel, dim3((unsigned)bx, (unsigned)t.n), dim3(256), 0, s, true, 1, src,
                          src_item_stride, dst, dst_item_stride, t));
    return MG_OK;
}

// Where each piece of a stream's device state lives, relative to the caller's `state` buffer.
struct StateLayout {
    size_t status, tail[kKernels], win, out, total;
    long long win_item, out_item;  // floats per item
    int wcap[kKernels];
};

StateLayout state_layout(int S, int P) {
    StateLayout L{};
    size_t off = 256;  // status word
    L.win_item = L.out_item = 0;
    for (int k = 0; k < kKernels; ++k) {
        L.tail[k] = off;
        off = align256(off + (size_t)2 * S * kC[k] * kTail[k] * sizeof(float));
        L.wcap[k] = window_cap(k, P);
        const long long w = (long long)kC[k] * L.wcap[k], o = (long long)kC[k + 1] * kRatio[k] * L.wcap[k];
        if (w > L.win_item) L.win_item = w;
        if (o > L.out_item) L.out_item = o;
    }
    L.win = off;
    off = align256(off + (size_t)S * L.win_item * sizeof(float));
    L.out = off;
    off = align256(off + (size_t)S * L.out_item * sizeof(float));
    L.total = off;
    return L;
}

// Everything one step launches, derived on the host from the frame counts.
struct Plan {
    AsmTable asm_[kKernels + 1];       // boundary b = 0..7: the windows of kernel b and the tails; [8]: audio to the caller
    long long asm_elems[kKernels + 1];  // the largest job of each launch (floats)
    int items[kKernels], lens[kKernels][MG_GEN_RAGGED_MAX_B], stride[kKernels];
    int voice[kKernels][MG_GEN_RAGGED_MAX_B];  // each item's voice
    long long F[MG_GEN_RAGGED_MAX_B][9];  // the counters after the step
    unsigned char par[MG_GEN_RAGGED_MAX_B][kKernels];
    int bound[MG_GEN_RAGGED_MAX_B];  // each slot's voice after the step (-1: no utterance open)
    long long bytes;  // bytes the window-assembly and audio copies read plus write
};

}  // namespace

// Kernel k of the default chain: x [B][kC[k]][stride] -> y [B][kC[k + 1]][kRatio[k] stride], t in kernel k's input units.
// What mg_gen_stream_step launches per kernel, and mg_gen_chain_kernel alone.
int launch_chain_kernel(int k, const float *x, float *y, const RunTable &t, int *status, cudaStream_t st,
                        int precision) {
    switch (k) {
        case 0: return launch_gen_pre_tc(x, y, t, status, st);
        case 1: return launch_convt_tc(x, y, 0, t, status, st, precision);
        case 2: return launch_resblock_tc(x, y, 0, t, status, st, nullptr, precision);
        case 3: return launch_convt_tc(x, y, 1, t, status, st, precision);
        case 4: return launch_resblock_tc(x, y, 1, t, status, st, nullptr, precision);
        case 5: return launch_convt_tc(x, y, 2, t, status, st, precision);
        case 6: return launch_resblock_tc(x, y, 2, t, status, st, nullptr, precision);
        case 7: return launch_resblock_tc(x, y, 14, t.scaled(2), status, st, nullptr, precision);
    }
    return set_error(MG_ERR_INVALID_ARGUMENT, "launch_chain_kernel: kernel %d", k);
}

}  // namespace mg

using namespace mg;

struct mg_gen_stream {
    int S, P, precision;
    char *state;
    size_t state_bytes;
    StateLayout L;
    long long F[MG_GEN_RAGGED_MAX_B][9];  // per slot: final positions at every boundary (all 0: no utterance open)
    unsigned char par[MG_GEN_RAGGED_MAX_B][kKernels];  // which half of the tail store holds the slot's current tail
    int voice[MG_GEN_RAGGED_MAX_B];  // per slot: the voice its open utterance is bound to (-1: none open)
    bool status_written, dry;
    Plan plan;
};

namespace mg {
namespace {

// Argument checks of a step (no CUDA call), then the plan.  On success p holds the launches, the new counters and the
// slots' voices.  voice: n ids in [0, n_voices) (NULL: all 0); an open slot keeps its voice unless this step resets it.
int plan_step(const char *fn, const mg_gen_stream *s, int n_voices, const int *voice, const int *frames, const int *flags, int n,
              int *out_samples, Plan &p) {
    if (!s || !frames || !out_samples) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if (n < 0 || n > s->S) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n = %d is outside [0, max_sessions = %d]", fn, n, s->S);
    if (n_voices < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_voices = %d, need at least 1", fn, n_voices);
    for (int i = 0; i < n; ++i) {
        const int fl = flags ? flags[i] : 0;
        const int v = voice ? voice[i] : 0;
        if (v < 0 || v >= n_voices)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: voice[%d] = %d is outside [0, n_voices = %d)", fn, i, v, n_voices);
        if (!(fl & MG_GEN_STREAM_RESET) && s->F[i][0] > 0 && v != s->voice[i])
            return set_error(MG_ERR_INVALID_ARGUMENT,
                             "%s: voice[%d] = %d, but slot %d's open utterance is bound to voice %d (a slot changes voice only "
                             "with MG_GEN_STREAM_RESET or after MG_GEN_STREAM_END)",
                             fn, i, v, i, s->voice[i]);
        if (frames[i] < 0 || frames[i] > s->P)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: frames[%d] = %d is outside [0, max_push_frames = %d]", fn, i, frames[i], s->P);
        if (fl & ~(MG_GEN_STREAM_END | MG_GEN_STREAM_RESET))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: flags[%d] = %d has bits other than MG_GEN_STREAM_END | MG_GEN_STREAM_RESET", fn, i, fl);
        const long long t0 = (fl & MG_GEN_STREAM_RESET) ? 0 : s->F[i][0];
        if ((fl & MG_GEN_STREAM_END) && t0 + frames[i] == 0)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: MG_GEN_STREAM_END on slot %d, which has no frames", fn, i);
        if (t0 + frames[i] > (1ll << 40) / 256) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: slot %d's utterance is too long", fn, i);
    }
    p.bytes = 0;
    for (int b = 0; b <= kKernels; ++b) { p.asm_[b].n = 0; p.asm_elems[b] = 0; }
    for (int k = 0; k < kKernels; ++k) { p.items[k] = 0; p.stride[k] = 0; }
    memcpy(p.F, s->F, sizeof(p.F));
    memcpy(p.par, s->par, sizeof(p.par));
    memcpy(p.bound, s->voice, sizeof(p.bound));
    // the walk: by ascending voice, slot order within a voice (stable), so each kernel's items come in voice runs
    int order[MG_GEN_RAGGED_MAX_B];
    for (int i = 0; i < n; ++i) order[i] = i;
    if (voice) std::stable_sort(order, order + n, [voice](int a, int b) { return voice[a] < voice[b]; });
    for (int q = 0; q < n; ++q) {
        const int i = order[q];
        const int fl = flags ? flags[i] : 0, v = voice ? voice[i] : 0;
        const bool end = fl & MG_GEN_STREAM_END;
        long long F[9], Fn[9];
        for (int b = 0; b <= kKernels; ++b) F[b] = (fl & MG_GEN_STREAM_RESET) ? 0 : s->F[i][b];
        const long long t = F[0] + frames[i];
        Fn[0] = t;
        for (int k = 0; k < kKernels; ++k) Fn[k + 1] = end ? kScale[k + 1] * t : exact_hi(k, Fn[k]);
        int item_prev = -1;  // the session's item in the previous kernel
        long long lo_prev = 0;
        for (int k = 0; k < kKernels; ++k) {
            const bool runs = Fn[k + 1] > F[k + 1], fresh = Fn[k] > F[k];
            if (Fn[k + 1] < F[k + 1] || (fresh && k > 0 && item_prev < 0))
                return set_error(MG_ERR_INVALID_ARGUMENT, "%s: internal: inconsistent counters at kernel %d, slot %d", fn, k, i);
            const long long lo = need_lo(k, F[k + 1]), lo_new = need_lo(k, Fn[k + 1]);
            int item = -1;
            if (runs || fresh) {
                AsmJob &j = p.asm_[k].job[p.asm_[k].n++];
                const int par = p.par[i][k];
                j.tin = par * s->S + i;
                j.tout = (1 - par) * s->S + i;
                j.tlen = (int)(F[k] - lo);
                j.nnew = (int)(Fn[k] - F[k]);
                j.src_item = k == 0 ? i : item_prev;
                j.src_off = k == 0 ? 0 : (int)(F[k] - kRatio[k - 1] * lo_prev);
                j.keep = end ? -1 : (int)(lo_new - lo);
                const int len = j.tlen + j.nnew;
                if (j.tlen > kTail[k] || len > s->L.wcap[k] || (!end && Fn[k] - lo_new > kTail[k]))
                    return set_error(MG_ERR_INVALID_ARGUMENT, "%s: internal: window of %d positions at kernel %d, slot %d", fn, len, k, i);
                if (runs) {
                    item = p.items[k]++;
                    p.lens[k][item] = len;
                    p.voice[k][item] = v;
                    if (len > p.stride[k]) p.stride[k] = len;
                }
                j.dst_item = item;
                if (!end) p.par[i][k] = (unsigned char)(1 - par);
                const long long elems = (long long)kC[k] * len;
                if (elems > p.asm_elems[k]) p.asm_elems[k] = elems;
                p.bytes += 4ll * kC[k] * ((long long)len + (runs ? len : 0) + (end ? 0 : Fn[k] - lo_new));
            }
            item_prev = item;
            lo_prev = lo;
        }
        out_samples[i] = (int)(Fn[8] - F[8]);
        if (Fn[8] > F[8]) {
            AsmJob &j = p.asm_[kKernels].job[p.asm_[kKernels].n++];
            j = AsmJob{0, 0, 0, item_prev, (int)(F[8] - kRatio[kKernels - 1] * lo_prev), out_samples[i], i, -1};
            if (out_samples[i] > p.asm_elems[kKernels]) p.asm_elems[kKernels] = out_samples[i];
            p.bytes += 8ll * out_samples[i];
        }
        for (int b = 0; b <= kKernels; ++b) p.F[i][b] = end ? 0 : Fn[b];
        p.bound[i] = p.F[i][0] > 0 ? v : -1;  // bound by the step that opens the utterance, free once it ends
    }
    for (int k = 0; k < kKernels; ++k) p.stride[k] = round16(p.stride[k]);
    return MG_OK;
}

}  // namespace
}  // namespace mg

extern "C" {

int mg_gen_stream_lookahead(void) { return kLookahead; }

int mg_gen_stream_max_out(int max_push_frames) { return max_push_frames >= 1 ? 256 * max_push_frames + kLookahead : 0; }

size_t mg_gen_stream_state_bytes(int max_sessions, int max_push_frames) {
    if (max_sessions < 1 || max_sessions > MG_GEN_RAGGED_MAX_B || max_push_frames < 1 || max_push_frames > (1 << 16)) return 0;
    return state_layout(max_sessions, max_push_frames).total;
}

int mg_gen_stream_create(mg_gen_stream **out, int max_sessions, int max_push_frames, int precision, void *state, size_t state_bytes) {
    const char *fn = "mg_gen_stream_create";
    if (!out || !state) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    *out = nullptr;
    if (max_sessions < 1 || max_sessions > MG_GEN_RAGGED_MAX_B)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: max_sessions = %d is outside [1, MG_GEN_RAGGED_MAX_B = %d]", fn, max_sessions,
                         MG_GEN_RAGGED_MAX_B);
    if (max_push_frames < 1 || max_push_frames > (1 << 16))
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: max_push_frames = %d is outside [1, 65536]", fn, max_push_frames);
    int rc = check_precision(fn, precision);
    if (!rc) rc = check_default_chain(fn, "streaming runs on the default chain");
    if (rc) return rc;
    const size_t need = mg_gen_stream_state_bytes(max_sessions, max_push_frames);
    if (state_bytes < need) return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: state %zu < %zu bytes", fn, state_bytes, need);
    if ((uintptr_t)state % 256) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: state must be 256-byte aligned", fn);
    mg_gen_stream *s = new (std::nothrow) mg_gen_stream();
    if (!s) return set_error(MG_ERR_OUT_OF_MEMORY, "%s: host allocation failed", fn);
    s->S = max_sessions;
    s->P = max_push_frames;
    s->precision = precision;
    s->state = (char *)state;
    s->state_bytes = state_bytes;
    s->L = state_layout(max_sessions, max_push_frames);
    for (int i = 0; i < MG_GEN_RAGGED_MAX_B; ++i) s->voice[i] = -1;
    *out = s;
    return MG_OK;
}

void mg_gen_stream_destroy(mg_gen_stream *s) { delete s; }

}  // extern "C"

namespace {

// mg_gen_stream_step_voices, and mg_gen_stream_step as its one-voice case (&packed, 1, NULL); pcm16: audio holds int16
// samples (mg_gen_stream_step_pcm16), written by the int16 form of the last copy -- the chain and the state are the same
int step_voices(const char *fn, mg_gen_stream *s, const void *const *packed, int n_voices, const int *voice, const float *mel,
                const int *frames, const int *flags, int n, void *audio, int *out_samples, void *stream, bool pcm16 = false) {
    if (!s || !packed || !audio) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if (s->dry) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: this handle was advanced by mg_gen_stream_dry_step", fn);
    if (n_voices < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_voices = %d, need at least 1", fn, n_voices);
    for (int v = 0; v < n_voices; ++v) {
        if (!packed[v]) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed[%d] is NULL", fn, v);
        if ((uintptr_t)packed[v] % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed[%d] must be 16-byte aligned", fn, v);
    }
    int rc = check_default_chain(fn, "streaming runs on the default chain");
    if (rc) return rc;
    bool any = false;
    for (int i = 0; frames && i < n && i < s->S; ++i) any |= frames[i] > 0;
    if (any && !mel) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null mel with frames to push", fn);
    Plan &p = s->plan;
    if ((rc = plan_step(fn, s, n_voices, voice, frames, flags, n, out_samples, p))) return rc;

    cudaStream_t st = (cudaStream_t)stream;
    const StateLayout &L = s->L;
    int *status = reinterpret_cast<int *>(s->state + L.status);
    float *win = reinterpret_cast<float *>(s->state + L.win), *out = reinterpret_cast<float *>(s->state + L.out);
    if (!s->status_written) {
        MG_CUDA_TRY(cudaMemsetAsync(status, 0, sizeof(int), st));
        s->status_written = true;
    }
    const float *const *blobs = reinterpret_cast<const float *const *>(packed);
    const float *prev = nullptr;  // the previous kernel's output windows
    long long prev_item = 0;
    int prev_row = 0;
    for (int k = 0; k < kKernels; ++k) {
        Copy c;
        float *tail = reinterpret_cast<float *>(s->state + L.tail[k]);
        c.tail_in = tail;
        c.tail_out = tail;  // (the halves differ per job: tin / tout)
        c.tail_cap = kTail[k];
        c.C = kC[k];
        if (k == 0) {
            c.src = mel;
            c.src_item_stride = (long long)kMelBins * s->P;
            c.src_row = s->P;
        } else {
            c.src = prev;
            c.src_item_stride = prev_item;
            c.src_row = prev_row;
        }
        const int stride = p.stride[k];
        c.dst = win;
        c.dst_item_stride = (long long)kC[k] * stride;
        c.dst_row = stride;
        if ((rc = launch_window(c, p.asm_[k], p.asm_elems[k], st))) return rc;
        if (p.items[k] == 0) continue;  // (no later kernel has items either: nothing was made final here)
        const RunTable t = RunTable::voices(p.lens[k], p.items[k], stride, blobs, p.voice[k]);
        if ((rc = launch_chain_kernel(k, win, out, t, status, st, s->precision))) return rc;
        prev = out;
        prev_row = kRatio[k] * stride;
        prev_item = (long long)kC[k + 1] * prev_row;
    }
    if (pcm16) {  // the newly final audio of every session, as pcm16, to its row of the caller's int16 buffer
        if ((rc = launch_audio_pcm16(prev, prev_item, static_cast<int16_t *>(audio), mg_gen_stream_max_out(s->P), p.asm_[kKernels],
                                     p.asm_elems[kKernels], st)))
            return rc;
    } else {
        Copy c;  // the newly final audio of every session to its row of the caller's buffer
        c.src = prev;
        c.src_item_stride = prev_item;
        c.src_row = prev_row;
        c.dst = static_cast<float *>(audio);
        c.dst_item_stride = mg_gen_stream_max_out(s->P);
        c.dst_row = 0;
        if ((rc = launch_window(c, p.asm_[kKernels], p.asm_elems[kKernels], st))) return rc;
    }
    memcpy(s->F, p.F, sizeof(p.F));
    memcpy(s->par, p.par, sizeof(p.par));
    memcpy(s->voice, p.bound, sizeof(p.bound));
    return MG_OK;
}

int dry_step_voices(const char *fn, mg_gen_stream *s, int n_voices, const int *voice, const int *frames, const int *flags, int n,
                    int *out_samples, int *kernel_items, long long *copy_bytes) {
    if (!s) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    int rc = plan_step(fn, s, n_voices, voice, frames, flags, n, out_samples, s->plan);
    if (rc) return rc;
    s->dry = true;
    for (int k = 0; kernel_items && k < kKernels; ++k) kernel_items[k] = s->plan.items[k];
    if (copy_bytes) *copy_bytes = s->plan.bytes;
    memcpy(s->F, s->plan.F, sizeof(s->F));
    memcpy(s->par, s->plan.par, sizeof(s->par));
    memcpy(s->voice, s->plan.bound, sizeof(s->voice));
    return MG_OK;
}

}  // namespace

extern "C" {

int mg_gen_stream_step_voices(mg_gen_stream *s, const void *const *packed, int n_voices, const int *voice, const float *mel,
                              const int *frames, const int *flags, int n, float *audio, int *out_samples, void *stream) {
    return step_voices("mg_gen_stream_step_voices", s, packed, n_voices, voice, mel, frames, flags, n, audio, out_samples, stream);
}

int mg_gen_stream_step_pcm16(mg_gen_stream *s, const void *const *packed, int n_voices, const int *voice, const float *mel,
                             const int *frames, const int *flags, int n, int16_t *audio, int *out_samples, void *stream) {
    return step_voices("mg_gen_stream_step_pcm16", s, packed, n_voices, voice, mel, frames, flags, n, audio, out_samples, stream,
                       true);
}

int mg_gen_stream_step(mg_gen_stream *s, const void *packed, const float *mel, const int *frames, const int *flags, int n, float *audio,
                       int *out_samples, void *stream) {
    if (!packed) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_stream_step: null argument");
    return step_voices("mg_gen_stream_step", s, &packed, 1, nullptr, mel, frames, flags, n, audio, out_samples, stream);
}

int mg_gen_stream_dry_step_voices(mg_gen_stream *s, int n_voices, const int *voice, const int *frames, const int *flags, int n,
                                  int *out_samples, int *kernel_items, long long *copy_bytes) {
    return dry_step_voices("mg_gen_stream_dry_step_voices", s, n_voices, voice, frames, flags, n, out_samples, kernel_items,
                           copy_bytes);
}

int mg_gen_stream_dry_step(mg_gen_stream *s, const int *frames, const int *flags, int n, int *out_samples, int *kernel_items,
                           long long *copy_bytes) {
    return dry_step_voices("mg_gen_stream_dry_step", s, 1, nullptr, frames, flags, n, out_samples, kernel_items, copy_bytes);
}

int mg_gen_stream_check_status(mg_gen_stream *s, void *stream) {
    if (!s) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_stream_check_status: null argument");
    if (!s->status_written) return MG_OK;  // no step has run: nothing to check
    MG_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    int st = 0;
    MG_CUDA_TRY(cudaMemcpy(&st, s->state + s->L.status, sizeof(int), cudaMemcpyDeviceToHost));
    if (st) return set_error(MG_ERR_CUDA, "mg_gen_stream: tensor-core pipeline wait timed out (role code %d)", st);
    return MG_OK;
}

}  // extern "C"
