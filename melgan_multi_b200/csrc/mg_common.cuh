// Shared helpers: error plumbing for the C ABI, cp.async wrappers, activation.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/melgan_b200.h"
#include "mg_layout.h"

namespace mg {

// streaming multiprocessors of the H100 SXM: grid sizes of the persistent-style kernels are multiples of it
constexpr int kNumSMs = 132;

// thread-local error string (the only mutable global state of the library)
char *error_buffer();
int set_error(int code, const char *fmt, ...);

#define MG_CUDA_TRY(expr)                                                                     \
    do {                                                                                      \
        cudaError_t err__ = (expr);                                                           \
        if (err__ != cudaSuccess)                                                             \
            return ::mg::set_error(MG_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,               \
                                   cudaGetErrorString(err__), __FILE__, __LINE__);            \
    } while (0)

__device__ __forceinline__ float lrelu(float x) { return fmaxf(x, x * kSlope); }

// 16-bit PCM of an audio sample (mg_gen_forward_pcm16, include/melgan_b200.h): 0 for NaN, else
// clamp(rint(32768 a), -32768, 32767) with rint rounding half to even.  32768 a is exact in fp32, so the result depends on
// the fp32 sample alone; tanh can return exactly +-1.0f, which is why the clamp is needed on the positive side.
__device__ __forceinline__ int16_t pcm16(float a) {
    const float s = fminf(fmaxf(rintf(32768.f * a), -32768.f), 32767.f);
    return a != a ? (int16_t)0 : (int16_t)__float2int_rz(s);
}
// the sample type an audio store writes: the fp32 sample itself, or its pcm16
template <class T>
__device__ __forceinline__ T audio_sample(float a);
template <>
__device__ __forceinline__ float audio_sample<float>(float a) { return a; }
template <>
__device__ __forceinline__ int16_t audio_sample<int16_t>(float a) { return pcm16(a); }

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// A generator batch as runs of consecutive items of equal length and voice: items [item0[r], item0[r+1]) hold len[r]
// positions each, stored `stride` positions apart (the longest item's length, at the tensor's scale), and take their
// weights from blob[r] (a blob of mg_gen_pack: the run's voice).  A uniform batch is one run, a ragged or multi-voice one
// (mg_gen_forward_ragged, mg_gen_forward_voices) at most MG_GEN_RAGGED_MAX_B.  Each generator kernel takes the table BY
// VALUE (__grid_constant__: read in place from the parameter bank; 6160 bytes with the blob pointers, under the 32764 bytes
// of kernel parameters sm_90a allows since CUDA 12.1) once its launcher has filled in the kernel's units -- ResBlock
// clusters, or virtual rows for conv_pre and the ConvTs: run r has per[r] units per item and starts at unit first[r].
// A grid of first[n] units covers every item and nothing past any item's end.  Where the voice changes, first[r] is
// rounded up to the kernel's tile (set_units): the units in between belong to no item, so no tile holds two voices.
struct RunPos {
    int item, unit, len;  // item -1: the unit lies past the last run, or in the gap before a voice's first tile
};
struct RunTable {
    int n, stride;
    int item0[MG_GEN_RAGGED_MAX_B + 1], len[MG_GEN_RAGGED_MAX_B];
    int first[MG_GEN_RAGGED_MAX_B + 1], per[MG_GEN_RAGGED_MAX_B];
    const float *blob[MG_GEN_RAGGED_MAX_B];

    static RunTable uniform(int B, int L, const float *packed) {
        RunTable t;
        t.n = 1;
        t.stride = L;
        t.item0[0] = 0;
        t.item0[1] = B;
        t.len[0] = L;
        t.blob[0] = packed;
        return t;
    }
    // lengths[0..B) (B <= MG_GEN_RAGGED_MAX_B, every length in [1, stride]), equal neighbours merged
    static RunTable ragged(const int *lengths, int B, int stride, const float *packed) {
        return voices(lengths, B, stride, &packed, nullptr);
    }
    // item i: lengths[i] positions (lengths nullptr: stride), weights blobs[voice[i]] (voice nullptr: blobs[0]); neighbours
    // of equal length and blob merged
    static RunTable voices(const int *lengths, int B, int stride, const float *const *blobs, const int *voice) {
        RunTable t;
        t.n = 0;
        t.stride = stride;
        for (int i = 0; i < B; ++i) {
            const int L = lengths ? lengths[i] : stride;
            const float *w = blobs[voice ? voice[i] : 0];
            if (i == 0 || L != t.len[t.n - 1] || w != t.blob[t.n - 1]) {
                t.item0[t.n] = i;
                t.blob[t.n] = w;
                t.len[t.n++] = L;
            }
        }
        t.item0[t.n] = B;
        return t;
    }
    int items() const { return item0[n]; }
    // items [i0, i1) as a batch of their own (item i0 becomes item 0)
    RunTable slice(int i0, int i1) const {
        RunTable t;
        t.n = 0;
        t.stride = stride;
        for (int r = 0; r < n; ++r) {
            const int a = item0[r] > i0 ? item0[r] : i0, b = item0[r + 1] < i1 ? item0[r + 1] : i1;
            if (a < b) {
                t.item0[t.n] = a - i0;
                t.blob[t.n] = blob[r];
                t.len[t.n++] = len[r];
            }
        }
        t.item0[t.n] = i1 - i0;
        return t;
    }
    // every length and the stride times k (the same batch at a later stage's scale)
    RunTable scaled(int k) const {
        RunTable t = *this;
        t.stride *= k;
        for (int r = 0; r < n; ++r) t.len[r] *= k;
        return t;
    }
    // per[r] = units(len[r]) units per item; first[] follows, rounded up to a multiple of `tile` where the voice changes
    // (with one voice the units are contiguous, whatever the tile)
    template <class F>
    void set_units(F units, int tile = 1) {
        int f = 0;
        for (int r = 0; r < n; ++r) {
            if (r > 0 && blob[r] != blob[r - 1]) f = (f + tile - 1) / tile * tile;
            first[r] = f;
            per[r] = units(len[r]);
            f += (item0[r + 1] - item0[r]) * per[r];
        }
        first[n] = f;
    }
    // the run of unit f, 0 <= f < first[n]
    __device__ __forceinline__ int run_of(int f) const {
        int lo = 0, hi = n;  // first[lo] <= f < first[hi]
        while (hi - lo > 1) {
            const int m = (lo + hi) >> 1;
            if (first[m] <= f) lo = m;
            else hi = m;
        }
        return lo;
    }
    // the weights of unit f's voice, 0 <= f < first[n] (a gap unit: the voice before it, which owns the rest of its tile)
    __device__ __forceinline__ const float *blob_at(int f) const { return blob[run_of(f)]; }
    // unit f -> (item, unit within the item, the item's length)
    __device__ __forceinline__ RunPos find(int f) const {
        if (f < 0 || f >= first[n]) return {-1, 0, 0};
        const int lo = run_of(f);
        const int u = f - first[lo], k = (int)((unsigned)u / (unsigned)per[lo]);  // (unsigned: the shorter division)
        if (k >= item0[lo + 1] - item0[lo]) return {-1, 0, 0};  // the gap before the next voice's first tile
        return {item0[lo] + k, u - k * per[lo], len[lo]};
    }
};
static_assert(sizeof(RunTable) == 6160 && sizeof(RunTable) + 256 <= 32764, "a kernel's parameters: the table and a few more");

// Launch helper of the tensor-core kernels: optional programmatic dependent launch
// (mg_tc.cuh pdl_*; MG_PDL=0 in the environment turns the attribute off for A/B runs); cluster > 1: thread-block clusters
// of `cluster` consecutive CTAs along x (grid.x must be a multiple of it).
bool pdl_enabled();
template <class... KArgs, class... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, bool pdl, int cluster,
                             Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (pdl && pdl_enabled()) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- launches implemented in the .cu files ------------------------------------------------
int launch_pack(const float *const *v, const float *const *g, const float *const *bias, float *packed,
                cudaStream_t s);
// (test-only library, csrc/testlib) ev: nullptr, or 6 events recorded before each of the 5 launches and after the last one
int launch_generator_simt(const float *packed, const float *mel, float *audio, int B, int T, float *ws,
                          cudaStream_t s, cudaEvent_t *ev = nullptr);
int generator_simt_num_launches();
int generator_tc_num_launches();
int generator_tc_fused_up();  // bit 0: stage 2, bit 1: stage 3 run their stride-2 ConvT at the FRONT of the ResBlock kernel
int generator_tc_tail();      // bit i: stage i's ConvT runs at the TAIL of ResBlock i-1's kernel
void generator_tc_set_tail(int mask);
bool generator_tc_default_chain();  // no tail fusion, stage 3's ConvT (only) at the front of the last kernel
// the refusals every generator entry point with a precision shares: an unknown precision, and a chain other than the
// default one ("<fn>: <role> only, but ...", role e.g. "bf16 runs on the default chain")
int check_precision(const char *fn, int precision);
int check_default_chain(const char *fn, const char *role);
const char *generator_tc_kernel_name(int i);
const char *generator_tc_kernel_config(int i, int T);
const char *resblock_config_name(int stage, int L);
int generator_tc_slices(int B, long long frames);  // batch slices (concurrent kernel chains) one forward is cut into
// batch: the items' mel lengths, stride T_max (the layout of mel, audio and every workspace buffer), each run's weights
// pcm16: audio (and audio_host) hold int16 samples, pcm16 of the fp32 audio, written by the last kernel (default chain only)
int launch_generator_tc(const float *mel, void *audio, const RunTable &batch, float *ws, int *status,
                        cudaStream_t s, cudaEvent_t *ev = nullptr, const float *mel_host = nullptr, void *audio_host = nullptr,
                        int precision = MG_GEN_PRECISION_FP32, bool pcm16 = false);
int launch_gen_pre_tc(const float *mel, float *y, const RunTable &batch, int *status, cudaStream_t s);
int launch_disc_post1_tc(const float *x, float *y, const uint8_t *wtc, const float *bias, int Bt, int L, int *status,
                         cudaStream_t s);
int launch_disc_post1_dgrad_tc(const float *dz, float *dx, const uint8_t *wtcT, const float *zero_bias, int Bt, int L, int *status,
                               cudaStream_t s);
int launch_disc_post1_wgrad_tc(const float *x, const float *dz, float *dw, float *db, int Bt, int L, int *status, cudaStream_t s);
size_t disc_scale_backward_workspace_bytes(int Bt, int L0);
int launch_disc_scale_backward(const void *blob, const float *x0, const float *const *fmap, const float *const *gfmap, float *gx0,
                               float *const *dw, float *const *db, int *reached, void *workspace, size_t workspace_bytes, int Bt,
                               int L0, int *status, cudaStream_t st);
size_t edge_bwd_workspace_bytes(int l, int Bt, int L);
int launch_disc_edge_backward(const void *blob, int l, const float *dz, const float *x, float *dx, float *dw, float *db, float *ws,
                              int Bt, int L, cudaStream_t s);
int launch_disc_group_tc(const float *x, float *out, const uint8_t *wtc, const float *bias, int Bt, int Cin, int Cout,
                         int Lin, int Lout, int *status, cudaStream_t s);
int launch_disc_group4_tc(const float *x, float *out, const uint8_t *wtc, const float *bias, int Bt, int L, int *status,
                          cudaStream_t s);
int launch_disc_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, cudaStream_t s, int ndisc = 3);
int launch_disc_forward(const void *packed, const float *x, int Bt, int L, float *const *fmaps, int *status, cudaStream_t s);
int launch_disc_layer_forward(const void *blob, int l, const float *x, float *out, int Bt, int Lin, int Lout, int *status,
                              cudaStream_t s);
void msd_lengths(int L, int *lens);
int launch_lrelu_grad(const float *g1, const float *g2, const float *out, float *dz, long long n, cudaStream_t s);
size_t grouped_bwd_workspace_bytes(int l, int Bt, int Lout);
int launch_disc_grouped_backward(const void *blob, int l, const float *dz, const float *x, float *dx, float *dw, float *db,
                                 float *ws, int Bt, int Lin, int Lout, cudaStream_t s);
int launch_disc_wn_backward(const float *const *v, const float *const *g, const float *const *dw, float *const *dv,
                            float *const *dg, cudaStream_t s);
int launch_adam(float *const *p, const float *const *g, float *const *m, float *const *v, const long long *n, const int *first,
                int count, int total_ctas, float lr, float b1, float b2, float eps, float wd, long long step, cudaStream_t s);
long long loss_num_ctas(const long long *n, int count);
int launch_loss_forward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count, float *out,
                        float *partial, cudaStream_t s);
int launch_loss_backward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count,
                         const float *gout, float *const *ga, float *const *gb, cudaStream_t s);
struct MelTables;
size_t mel_tables_bytes();
int mel_tables_build(int sr, int n_mels, float fmin, float fmax, int norm, MelTables *t);
int mel_frames(int L);
int launch_mel(const void *tables, const float *audio, float *mel, int B, int L, cudaStream_t s);
size_t mel_backward_workspace_bytes(int B, int L);
int launch_mel_backward(const void *tables, const float *audio, const float *grad_mel, float *grad_audio, int B, int L,
                        void *workspace, size_t workspace_bytes, cudaStream_t s);
size_t stft_tables_bytes(int n_fft);
int stft_tables_build(int n_fft, int win_length, void *tables_host);
// the window and twiddles of one resolution (the STFT-loss table layout, win[n_fft] then tw[n_fft / 2]), arguments checked
void stft_tables_fill(int n_fft, int win_length, float *win);
int stft_frames(int n_fft, int hop, int L);
int stft_check(const char *fn, int n_res, const void *const *tables, const int *n_fft, const int *hop, int B, int L, int *T);
void stft_workspace(int n_res, const int *n_fft, int B, const int *T, size_t *fwd, size_t *bwd);
int launch_stft_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                             int B, int L, const int *T, float *sc, float *mag, void *workspace, cudaStream_t s);
int launch_stft_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                              int B, int L, const int *T, const float *grad_sc, const float *grad_mag, const void *fwd_workspace,
                              float *grad_x, void *workspace, cudaStream_t s);
size_t mel_loss_tables_bytes(int n_fft);
int mel_loss_tables_build(int n_fft, int win_length, int sr, int n_mels, float fmin, float fmax, void *tables_host);
int mel_loss_frames(int n_fft, int hop, int L);
int mel_loss_check(const char *fn, int n_res, const void *const *tables, const int *n_fft, const int *hop, int B, int L, int *T);
void mel_loss_workspace(int n_res, const int *n_fft, int B, const int *T, size_t *fwd, size_t *bwd);
int launch_mel_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                            int B, int L, const int *T, float *loss, void *workspace, cudaStream_t s);
int launch_mel_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                             int B, int L, const int *T, const float *grad, float *grad_x, void *workspace, cudaStream_t s);
int launch_msd_forward(const void *packed, const float *y, int Bt, int L, float *const *fmaps, int *status, cudaStream_t s);
// batch: lengths and stride of the kernel's input (ConvT) / of the ResBlock itself (the output length for codes 12..14)
// precision: MG_GEN_PRECISION_FP32 (3-pass split bf16) or MG_GEN_PRECISION_BF16 (one pass; only the default chain's kernels)
int launch_convt_tc(const float *x, float *y, int stage, const RunTable &batch, int *status, cudaStream_t s,
                    int precision = MG_GEN_PRECISION_FP32);
const char *convt_config_name(int stage);
const char *gen_pre_config_name();
// kernel k (0..7) of the default chain; batch in kernel k's input units (mg_gen_stream.cu)
int launch_chain_kernel(int k, const float *x, float *y, const RunTable &t, int *status, cudaStream_t st,
                        int precision);
int launch_resblock_tc(const float *x, float *y, int stage, const RunTable &batch, int *status, cudaStream_t s,
                       long long *trace = nullptr, int precision = MG_GEN_PRECISION_FP32);
// stage code 14 (the default chain's last kernel) storing pcm16 of its audio, at either precision
int launch_resblock_tc_pcm16(const float *x, int16_t *y, const RunTable &batch, int *status, cudaStream_t s, int precision);

}  // namespace mg
