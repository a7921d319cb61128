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

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src) {
    uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// A generator batch as runs of consecutive items of equal length: items [item0[r], item0[r+1]) hold len[r] positions
// each, stored `stride` positions apart (the longest item's length, at the tensor's scale).  A uniform batch is one run,
// a ragged one (mg_gen_forward_ragged) at most MG_GEN_RAGGED_MAX_B.  Each generator kernel takes the table BY VALUE
// (__grid_constant__: read in place from the parameter bank) once its launcher has filled in the kernel's units -- ResBlock
// clusters, or virtual rows for conv_pre and the ConvTs: run r has per[r] units per item and starts at unit first[r].
// A grid of first[n] units covers every item and nothing past any item's end.
struct RunPos {
    int item, unit, len;  // item -1: the unit lies past the last run
};
struct RunTable {
    int n, stride;
    int item0[MG_GEN_RAGGED_MAX_B + 1], len[MG_GEN_RAGGED_MAX_B];
    int first[MG_GEN_RAGGED_MAX_B + 1], per[MG_GEN_RAGGED_MAX_B];

    static RunTable uniform(int B, int L) {
        RunTable t;
        t.n = 1;
        t.stride = L;
        t.item0[0] = 0;
        t.item0[1] = B;
        t.len[0] = L;
        return t;
    }
    // lengths[0..B) (B <= MG_GEN_RAGGED_MAX_B, every length in [1, stride]), equal neighbours merged
    static RunTable ragged(const int *lengths, int B, int stride) {
        RunTable t;
        t.n = 0;
        t.stride = stride;
        for (int i = 0; i < B; ++i)
            if (i == 0 || lengths[i] != lengths[i - 1]) {
                t.item0[t.n] = i;
                t.len[t.n++] = lengths[i];
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
    // per[r] = units(len[r]) units per item; first[] follows
    template <class F>
    void set_units(F units) {
        first[0] = 0;
        for (int r = 0; r < n; ++r) {
            per[r] = units(len[r]);
            first[r + 1] = first[r] + (item0[r + 1] - item0[r]) * per[r];
        }
    }
    // unit f -> (item, unit within the item, the item's length)
    __device__ __forceinline__ RunPos find(int f) const {
        if (f < 0 || f >= first[n]) return {-1, 0, 0};
        int lo = 0, hi = n;  // first[lo] <= f < first[hi]
        while (hi - lo > 1) {
            const int m = (lo + hi) >> 1;
            if (first[m] <= f) lo = m;
            else hi = m;
        }
        const int u = f - first[lo], k = (int)((unsigned)u / (unsigned)per[lo]);  // (unsigned: the shorter division)
        return {item0[lo] + k, u - k * per[lo], len[lo]};
    }
};

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
const char *generator_tc_kernel_name(int i);
const char *generator_tc_kernel_config(int i, int T);
const char *resblock_config_name(int stage, int L);
int generator_tc_slices(int B, long long frames);  // batch slices (concurrent kernel chains) one forward is cut into
// batch: the items' mel lengths, stride T_max (the layout of mel, audio and every workspace buffer)
int launch_generator_tc(const float *packed, const float *mel, float *audio, const RunTable &batch, float *ws, int *status,
                        cudaStream_t s, cudaEvent_t *ev = nullptr, const float *mel_host = nullptr, float *audio_host = nullptr,
                        int precision = MG_GEN_PRECISION_FP32);
int launch_gen_pre_tc(const float *mel, float *y, const float *packed, const RunTable &batch, int *status, cudaStream_t s);
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
int launch_msd_forward(const void *packed, const float *y, int Bt, int L, float *const *fmaps, int *status, cudaStream_t s);
// batch: lengths and stride of the kernel's input (ConvT) / of the ResBlock itself (the output length for codes 12..14)
// precision: MG_GEN_PRECISION_FP32 (3-pass split bf16) or MG_GEN_PRECISION_BF16 (one pass; only the default chain's kernels)
int launch_convt_tc(const float *x, float *y, const float *packed, int stage, const RunTable &batch, int *status, cudaStream_t s,
                    int precision = MG_GEN_PRECISION_FP32);
const char *convt_config_name(int stage);
int launch_resblock_tc(const float *x, float *y, const float *packed, int stage, const RunTable &batch, int *status, cudaStream_t s,
                       long long *trace = nullptr, int precision = MG_GEN_PRECISION_FP32);

}  // namespace mg
