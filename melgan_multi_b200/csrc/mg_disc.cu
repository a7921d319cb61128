// Multi-scale discriminator forward (models.py:74-135): fold/pack of the 21 weight-normed convs in one launch, and the
// per-layer kernels of one Discriminator.  Real and generated batches are stacked (Bt = 2B) by the caller, so every
// weight is streamed once for both (the reference runs d(y) and d(y_hat) as separate calls, models.py:128-129).
//
//   conv_pre   1 -> 16, k15  (+ LeakyReLU), with the AvgPool1d chain of the scale fused into the input read
//              (models.py:114-117,125-127: scale 1 sees AvgPool1d(4,2,pad 2)(y), scale 2 AvgPool1d(4,4,pad 2) of that;
//              count_include_pad=True, so every window divides by 4)                                   fp32 SIMT
//   grouped    k41, 4 input channels per group, stride 4/4/4/1 (+ LeakyReLU)                           wgmma   (mg_disc_tc.cu;
//              the fp32 SIMT kernels below are the second implementation, MG_DISC_GROUP=simt)
//   conv_post1 1024 -> 1024, k5 (+ LeakyReLU): 88% of the FLOPs                                        wgmma   (mg_conv_tc.cu)
//   conv_post2 1024 -> 1, k3                                                                           fp32 SIMT
// Every layer writes its feature map (fp32 NCL) because Discriminator.forward returns all seven (models.py:87-103).
#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {

// ------------------------------------------------------------------------------------------------------------------
// fold + pack: one CTA per weight-norm row (3 * 3409 rows)
struct DiscPackArgs {
    const float *v[3 * kDiscLayers];
    const float *g[3 * kDiscLayers];
    const float *bias[3 * kDiscLayers];
};

__global__ void __launch_bounds__(128) disc_pack_kernel(DiscPackArgs a, uint8_t *__restrict__ packed) {
    int grow = blockIdx.x;
    const int d = grow / kDiscRows;
    grow -= d * kDiscRows;
    int l = 0;
#pragma unroll 1
    while (grow >= d_layer(l).cout) { grow -= d_layer(l).cout; ++l; }
    const int row = grow;  // output channel
    const DLayer sh = d_layer(l);
    const int cig = sh.cin / sh.groups, inner = cig * sh.k;
    const float *__restrict__ vr = a.v[d * kDiscLayers + l] + (size_t)row * inner;

    float ss = 0.f;
    for (int j = threadIdx.x; j < inner; j += blockDim.x) ss = fmaf(vr[j], vr[j], ss);
    __shared__ float red[4];
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    __syncthreads();
    const float scale = a.g[d * kDiscLayers + l][row] / sqrtf(red[0] + red[1] + red[2] + red[3]);

    uint8_t *blob = packed + (size_t)d * d_blob_bytes();
    float *fw = reinterpret_cast<float *>(blob) + d_weight_offset(l);
    if (l == 0) {
        for (int j = threadIdx.x; j < inner; j += blockDim.x) fw[j * 16 + row] = scale * vr[j];  // [tap][co]
    } else if (l <= 4) {
        const int cog = sh.cout / sh.groups, grp = row / cog, col = row % cog;
        for (int j = threadIdx.x; j < inner; j += blockDim.x)  // j = ci*41 + tap -> [grp][ci][tap][col]
            fw[((size_t)grp * inner + j) * cog + col] = scale * vr[j];
        if (l <= 3) {  // split-bf16 Toeplitz copy for the tensor-core kernel (layout: mg_layout.h d_gtc_index), zeros included
            __nv_bfloat16 *gt = reinterpret_cast<__nv_bfloat16 *>(blob + d_gtc_start() + d_gtc_offset(l) + (size_t)grp * d_gtc_group_bytes());
            for (int s = threadIdx.x; s < kDgPanels * 64; s += blockDim.x) {
                const int ci = s & 3, pos = (s >> 2) & 1, e = (s >> 3) & 1, r = (s >> 4) & 3, kp = s >> 6;
                const int q = 2 * kp + pos - 1 - e, k = 4 * q + r;
                const float wv = (q >= 0 && k <= 40) ? scale * vr[ci * 41 + k] : 0.f;
                __nv_bfloat16 hi, lo;
                tc::split_bf16(wv, hi, lo);
                gt[d_gtc_index(kp, r, e * 16 + col, pos, ci)] = hi;
                gt[d_gtc_index(kp, r, 32 + e * 16 + col, pos, ci)] = lo;
            }
        } else {  // layer 4 (stride 1): 8-outputs-per-lane Toeplitz copy, mg_layout.h d_g4tc_index
            __nv_bfloat16 *gt = reinterpret_cast<__nv_bfloat16 *>(blob + d_g4tc_start() + (size_t)grp * d_g4tc_group_bytes());
            for (int s = threadIdx.x; s < kDg4Panels * 4 * 64; s += blockDim.x) {
                const int i = s & 7, e = (s >> 3) & 7, ci = (s >> 6) & 3, kp = s >> 8;
                const int k = 8 * kp + i - e;
                const float wv = (k >= 0 && k <= 40) ? scale * vr[ci * 41 + k] : 0.f;
                __nv_bfloat16 hi, lo;
                tc::split_bf16(wv, hi, lo);
                gt[d_g4tc_index(kp, ci, e * 4 + col, i)] = hi;
                gt[d_g4tc_index(kp, ci, 32 + e * 4 + col, i)] = lo;
            }
        }
    } else if (l == 5) {
        __nv_bfloat16 *tcw = reinterpret_cast<__nv_bfloat16 *>(blob + d_tc_start());
        for (int j = threadIdx.x; j < inner; j += blockDim.x) {
            const int ci = j / 5, tap = j - 5 * ci;
            __nv_bfloat16 hi, lo;
            tc::split_bf16(scale * vr[j], hi, lo);
            tcw[conv_tc_weight_index(1024, 5, kPost1NG, row, ci, tap, 0)] = hi;
            tcw[conv_tc_weight_index(1024, 5, kPost1NG, row, ci, tap, 1)] = lo;
            __nv_bfloat16 *tct = reinterpret_cast<__nv_bfloat16 *>(blob + d_tcT_start());  // dgrad copy: [ci][co][4 - tap]
            tct[conv_tc_weight_index(1024, 5, kPost1NG, ci, row, 4 - tap, 0)] = hi;
            tct[conv_tc_weight_index(1024, 5, kPost1NG, ci, row, 4 - tap, 1)] = lo;
        }
    } else {
        for (int j = threadIdx.x; j < inner; j += blockDim.x) fw[j] = scale * vr[j];  // [ci][tap]
    }
    if (threadIdx.x == 0) reinterpret_cast<float *>(blob)[d_bias_offset(l) + row] = a.bias[d * kDiscLayers + l][row];
}

// ndisc = 3: the multi-scale stack (mg_msd_pack); ndisc = 1: one stand-alone Discriminator (mg_disc_pack), blob = d_blob_bytes()
int launch_disc_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, cudaStream_t s, int ndisc) {
    DiscPackArgs a = {};
    for (int i = 0; i < ndisc * kDiscLayers; ++i) {
        if (!v[i] || !g[i] || !bias[i]) return set_error(MG_ERR_INVALID_ARGUMENT, "discriminator pack: null tensor %d", i);
        a.v[i] = v[i]; a.g[i] = g[i]; a.bias[i] = bias[i];
    }
    for (int d = 0; d < ndisc; ++d)  // the dgrad launch's zero "bias"
        MG_CUDA_TRY(cudaMemsetAsync(reinterpret_cast<uint8_t *>(packed) + (size_t)d * d_blob_bytes() + d_zero_start(), 0, 4096, s));
    disc_pack_kernel<<<ndisc * kDiscRows, 128, 0, s>>>(a, reinterpret_cast<uint8_t *>(packed));
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// input of scale `sc` at position t (zero outside [0, L_sc)): the AvgPool1d chain evaluated on the fly
__device__ __forceinline__ float pool1_at(const float *__restrict__ y, int L0, int L1, int t) {  // AvgPool1d(4, 2, pad 2)
    if (t < 0 || t >= L1) return 0.f;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int i = 2 * t - 2 + j;
        if (i >= 0 && i < L0) s += __ldg(y + i);
    }
    return s * 0.25f;
}
template <int SC>
__device__ __forceinline__ float scale_input_at(const float *__restrict__ y, int L0, int L1, int L2, int t) {
    if (SC == 0) return (t >= 0 && t < L0) ? __ldg(y + t) : 0.f;
    if (SC == 1) return pool1_at(y, L0, L1, t);
    if (t < 0 || t >= L2) return 0.f;  // AvgPool1d(4, 4, pad 2) of the scale-1 signal
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += pool1_at(y, L0, L1, 4 * t - 2 + j);
    return s * 0.25f;
}

// conv_pre (1 -> 16, k15, pad 7) + LeakyReLU.  y [Bt][1][L0] -> out [Bt][16][Ls]
template <int SC>
__global__ void __launch_bounds__(256) disc_pre_kernel(const float *__restrict__ y, float *__restrict__ out,
                                                       const float *__restrict__ blob, int L0, int L1, int L2) {
    __shared__ float xs[256 + 16];
    __shared__ float ws[15 * 16];
    __shared__ float bs[16];
    const int Ls = SC == 0 ? L0 : SC == 1 ? L1 : L2;
    const int b = blockIdx.y, t0 = blockIdx.x * 256;
    const float *yb = y + (size_t)b * L0;
    for (int i = threadIdx.x; i < 256 + 14; i += 256) xs[i] = scale_input_at<SC>(yb, L0, L1, L2, t0 + i - 7);
    if (threadIdx.x < 240) ws[threadIdx.x] = blob[d_weight_offset(0) + threadIdx.x];
    if (threadIdx.x < 16) bs[threadIdx.x] = blob[d_bias_offset(0) + threadIdx.x];
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t >= Ls) return;
    float acc[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[c] = bs[c];
#pragma unroll
    for (int k = 0; k < 15; ++k) {
        const float xv = xs[threadIdx.x + k];
#pragma unroll
        for (int c = 0; c < 16; ++c) acc[c] = fmaf(ws[k * 16 + c], xv, acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) out[((size_t)b * 16 + c) * Ls + t] = lrelu(acc[c]);
}

// grouped conv k41 pad 20, 4 input channels per group, COG output channels per group, stride S, + LeakyReLU.
// CTA = 4 groups (one warp each) x 128 output positions; lane owns positions t0 + lane + 32 j.
template <int COG, int S>
__global__ void __launch_bounds__(128) disc_group_kernel(const float *__restrict__ x, float *__restrict__ out,
                                                         const float *__restrict__ w, const float *__restrict__ bias,
                                                         int Cin, int Cout, int Lin, int Lout) {
    constexpr int XT = (S == 4) ? 128 + 12 : 128 + 40;  // per phase
    constexpr int WG = 4 * 41 * COG;                     // weights per group
    extern __shared__ __align__(16) float dsm[];
    float *ws = dsm;                   // [4 groups][4 ci][41][COG]
    float *xs = dsm + 4 * WG;          // [4 groups][4 ci][S][XT]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t0 = blockIdx.x * 128, g0 = blockIdx.y * 4, b = blockIdx.z;
    // weights of the 4 groups are contiguous in the packed blob
    for (int i = threadIdx.x * 4; i < 4 * WG; i += 128 * 4)
        *reinterpret_cast<float4 *>(ws + i) = *reinterpret_cast<const float4 *>(w + (size_t)g0 * WG + i);
    // input windows: positions pos0 .. pos0 + S*XT of the 16 channels, de-interleaved by phase (pos - pos0) % S
    const int pos0 = (S == 4) ? 4 * (t0 - 5) : t0 - 20;
    const float *xb = x + ((size_t)b * Cin + g0 * 4) * Lin;
    for (int i = threadIdx.x; i < 16 * S * XT; i += 128) {
        const int c = i / (S * XT), r = i - c * (S * XT);  // r = offset from pos0
        const int pos = pos0 + r;
        const float v = (pos >= 0 && pos < Lin) ? __ldg(xb + (size_t)c * Lin + pos) : 0.f;
        xs[(c * S + (r % S)) * XT + r / S] = v;
    }
    __syncthreads();
    const float *wg = ws + warp * WG;
    const float *xg = xs + warp * 4 * S * XT;
    float acc[COG][4];
#pragma unroll
    for (int c = 0; c < COG; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[c][j] = 0.f;
#pragma unroll 1
    for (int ci = 0; ci < 4; ++ci) {
#pragma unroll
        for (int k = 0; k < 41; ++k) {
            // S == 4: position 4*(t0+tl) + k - 20 = pos0 + 4*tl + k  -> phase k%4, index tl + k/4
            // S == 1: position t0 + tl + k - 20 = pos0 + tl + k        -> phase 0, index tl + k
            const float *xr = xg + (ci * S + (S == 4 ? (k & 3) : 0)) * XT + (S == 4 ? (k >> 2) : k) + lane;
            float xv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) xv[j] = xr[32 * j];
            const float *wr = wg + (ci * 41 + k) * COG;
#pragma unroll
            for (int q = 0; q < COG / 4; ++q) {
                const float4 wv = *reinterpret_cast<const float4 *>(wr + 4 * q);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    acc[4 * q + 0][j] = fmaf(wv.x, xv[j], acc[4 * q + 0][j]);
                    acc[4 * q + 1][j] = fmaf(wv.y, xv[j], acc[4 * q + 1][j]);
                    acc[4 * q + 2][j] = fmaf(wv.z, xv[j], acc[4 * q + 2][j]);
                    acc[4 * q + 3][j] = fmaf(wv.w, xv[j], acc[4 * q + 3][j]);
                }
            }
        }
    }
    const int co0 = (g0 + warp) * COG;
#pragma unroll
    for (int c = 0; c < COG; ++c) {
        const float bv = __ldg(bias + co0 + c);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = t0 + lane + 32 * j;
            if (t < Lout) out[((size_t)b * Cout + co0 + c) * Lout + t] = lrelu(acc[c][j] + bv);
        }
    }
}

// conv_post2 (1024 -> 1, k3, pad 1), no activation.  x [Bt][1024][L] -> out [Bt][1][L]
// The op is a 16.8 MB read for 4 K outputs (scale 0), so the grid is cut fine: CTA = 8 positions of one item (one 32-byte
// sector per channel row); a warp load covers 4 channels x 8 positions, 8 warps split the 1024 channels.  The partial
// sums are combined in a fixed order (shuffles, then warp 0 over the 8 per-warp partials): bit-reproducible.
__global__ void __launch_bounds__(256) disc_post2_kernel(const float *__restrict__ x, float *__restrict__ out,
                                                         const float *__restrict__ w, const float *__restrict__ bias, int L) {
    __shared__ float part[8][8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cl = lane >> 3, pos = lane & 7;
    const int t = blockIdx.x * 8 + pos, b = blockIdx.y;
    const float *xb = x + (size_t)b * 1024 * L;
    float acc = 0.f;
    if (t < L) {
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const int ci = warp * 128 + j * 4 + cl;
            const float *xr = xb + (size_t)ci * L + t;
            const float xm = t >= 1 ? __ldg(xr - 1) : 0.f, xc = __ldg(xr), xp = t + 1 < L ? __ldg(xr + 1) : 0.f;
            acc = fmaf(__ldg(w + ci * 3), xm, fmaf(__ldg(w + ci * 3 + 1), xc, fmaf(__ldg(w + ci * 3 + 2), xp, acc)));
        }
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 8);
    acc += __shfl_xor_sync(0xffffffffu, acc, 16);
    if (lane < 8) part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && lane < 8 && t < L) {
        float s = __ldg(bias);
#pragma unroll
        for (int q = 0; q < 8; ++q) s += part[q][lane];
        out[(size_t)b * L + t] = s;
    }
}

// ------------------------------------------------------------------------------------------------------------------
static int conv_len(int L, int k, int s, int p) { return (L + 2 * p - (k - 1) - 1) / s + 1; }

void msd_lengths(int L, int *lens /* [3][7] */) {
    int Ls = L;
    for (int sc = 0; sc < 3; ++sc) {
        if (sc == 1) Ls = (L + 4 - 4) / 2 + 1;        // AvgPool1d(4, 2, pad 2)
        if (sc == 2) Ls = (Ls + 4 - 4) / 4 + 1;        // AvgPool1d(4, 4, pad 2) of the scale-1 signal
        int cur = Ls;
        for (int l = 0; l < kDiscLayers; ++l) {
            const DLayer d = d_layer(l);
            cur = conv_len(cur, d.k, d.stride, d.pad);
            lens[sc * kDiscLayers + l] = cur;
        }
    }
}

template <int COG, int S>
static int launch_group(const float *x, float *out, const float *w, const float *bias, int Bt, int Cin, int Cout, int Lin,
                        int Lout, cudaStream_t s) {
    constexpr int XT = (S == 4) ? 128 + 12 : 128 + 40;
    constexpr int smem = (4 * 4 * 41 * COG + 16 * S * XT) * (int)sizeof(float);
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(disc_group_kernel<COG, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    dim3 grid((Lout + 127) / 128, (Cin / 4) / 4, Bt);
    disc_group_kernel<COG, S><<<grid, 128, smem, s>>>(x, out, w, bias, Cin, Cout, Lin, Lout);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

// Side streams for the three scales (they are independent until the caller consumes the feature maps): forked from and
// joined back into the caller's stream with events, so the call stays asynchronous and stream-ordered for the caller.
// One pool per (host thread, device): streams and events belong to the device that was current at their creation.
constexpr int kMaxDevices = 64;
struct ScaleStreams {
    cudaStream_t st[2] = {nullptr, nullptr};
    cudaEvent_t fork = nullptr, join[2] = {nullptr, nullptr};
    bool ready = false;
    int init() {
        if (ready) return MG_OK;
        for (int i = 0; i < 2; ++i) {
            MG_CUDA_TRY(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
            MG_CUDA_TRY(cudaEventCreateWithFlags(&join[i], cudaEventDisableTiming));
        }
        MG_CUDA_TRY(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
        ready = true;
        return MG_OK;
    }
};

// Layer l (1..6) of one Discriminator: x [Bt][Cin][Lin] -> out [Bt][Cout][Lout], Lout = ln of layer l.  blob: that
// discriminator's packed weights.  group_tc: the grouped convs on the tensor cores (false: the fp32 SIMT second
// implementation, MG_DISC_GROUP=simt).  Enqueued on q.
static int disc_layer(const uint8_t *blob, int l, const float *x, float *out, int Bt, int Lin, int Lout, int *status, bool group_tc,
                      cudaStream_t q) {
    const float *fw = reinterpret_cast<const float *>(blob);
    const DLayer d = d_layer(l);
    if (l <= 3)
        return group_tc ? launch_disc_group_tc(x, out, blob + d_gtc_start() + d_gtc_offset(l), fw + d_bias_offset(l), Bt, d.cin,
                                               d.cout, Lin, Lout, status, q)
                        : launch_group<16, 4>(x, out, fw + d_weight_offset(l), fw + d_bias_offset(l), Bt, d.cin, d.cout, Lin, Lout, q);
    if (l == 4)
        return group_tc ? launch_disc_group4_tc(x, out, blob + d_g4tc_start(), fw + d_bias_offset(4), Bt, Lout, status, q)
                        : launch_group<4, 1>(x, out, fw + d_weight_offset(4), fw + d_bias_offset(4), Bt, 1024, 1024, Lin, Lout, q);
    if (l == 5) return launch_disc_post1_tc(x, out, blob + d_tc_start(), fw + d_bias_offset(5), Bt, Lout, status, q);
    dim3 gp2((Lin + 7) / 8, Bt);
    disc_post2_kernel<<<gp2, 256, 0, q>>>(x, out, fw + d_weight_offset(6), fw + d_bias_offset(6), Lin);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

// One Discriminator (models.py:87-103) on the input of scale `sc` of y [Bt][1][L] (sc = 0: y itself; 1, 2: the AvgPool1d chain
// of models.py:114-117, evaluated inside conv_pre).  blob: that discriminator's packed weights; f[0..6]: its feature maps;
// ln[0..6]: their lengths.  Everything is enqueued on q.
static int disc_chain(const uint8_t *blob, const float *y, int sc, int Bt, int L, int L1, int L2, const int *ln, float *const *f,
                      int *status, bool group_tc, cudaStream_t q) {
    const float *fw = reinterpret_cast<const float *>(blob);
    const int Ls = sc == 0 ? L : sc == 1 ? L1 : L2;
    dim3 gpre((Ls + 255) / 256, Bt);
    if (sc == 0) disc_pre_kernel<0><<<gpre, 256, 0, q>>>(y, f[0], fw, L, L1, L2);
    else if (sc == 1) disc_pre_kernel<1><<<gpre, 256, 0, q>>>(y, f[0], fw, L, L1, L2);
    else disc_pre_kernel<2><<<gpre, 256, 0, q>>>(y, f[0], fw, L, L1, L2);
    MG_CUDA_TRY(cudaGetLastError());
    for (int l = 1; l < kDiscLayers; ++l) {
        const int rc = disc_layer(blob, l, f[l - 1], f[l], Bt, ln[l - 1], ln[l], status, group_tc, q);
        if (rc) return rc;
    }
    return MG_OK;
}

static bool disc_group_tc() {
    const char *gp = getenv("MG_DISC_GROUP");
    return !(gp && strcmp(gp, "simt") == 0);
}

// one layer (1..6) of one discriminator on a caller-given input (mg_msd_layer_forward): blob = that discriminator's weights
int launch_disc_layer_forward(const void *blob, int l, const float *x, float *out, int Bt, int Lin, int Lout, int *status,
                              cudaStream_t s) {
    return disc_layer(reinterpret_cast<const uint8_t *>(blob), l, x, out, Bt, Lin, Lout, status, disc_group_tc(), s);
}

// stand-alone Discriminator.forward (models.py:87-103): x [Bt][1][L] -> fmaps[0..6] (lengths: the scale-0 row of msd_lengths)
int launch_disc_forward(const void *packed, const float *x, int Bt, int L, float *const *fmaps, int *status, cudaStream_t s) {
    int lens[3 * kDiscLayers];
    msd_lengths(L, lens);
    return disc_chain(reinterpret_cast<const uint8_t *>(packed), x, 0, Bt, L, 0, 0, lens, fmaps, status, disc_group_tc(), s);
}

// y [Bt][1][L] -> fmaps[sc*7 + l] (device pointers, fp32 NCL, lengths from msd_lengths); status: device int
int launch_msd_forward(const void *packed, const float *y, int Bt, int L, float *const *fmaps, int *status, cudaStream_t s) {
    static thread_local ScaleStreams pools[kMaxDevices];  // per host thread, like the rest of the library's state
    int dev = 0;
    MG_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kMaxDevices) return set_error(MG_ERR_INVALID_ARGUMENT, "launch_msd_forward: device ordinal %d", dev);
    ScaleStreams &ss = pools[dev];
    int rc = ss.init();
    if (rc) return rc;
    int lens[3 * kDiscLayers];
    msd_lengths(L, lens);
    const int L1 = (L + 4 - 4) / 2 + 1, L2 = (L1 + 4 - 4) / 4 + 1;
    const bool group_tc = disc_group_tc();
    MG_CUDA_TRY(cudaEventRecord(ss.fork, s));
    int forked = 0;
    for (int sc = 0; sc < 3 && rc == MG_OK; ++sc) {
        cudaStream_t q = sc == 0 ? s : ss.st[sc - 1];  // scale 0 (the largest) stays on the caller's stream
        if (sc > 0) {
            cudaError_t e = cudaStreamWaitEvent(q, ss.fork, 0);
            if (e != cudaSuccess) { rc = set_error(MG_ERR_CUDA, "launch_msd_forward: fork: %s", cudaGetErrorString(e)); break; }
            forked = sc;
        }
        rc = disc_chain(reinterpret_cast<const uint8_t *>(packed) + (size_t)sc * d_blob_bytes(), y, sc, Bt, L, L1, L2,
                        lens + sc * kDiscLayers, fmaps + sc * kDiscLayers, status, group_tc, q);
    }
    for (int sc = 1; sc <= forked; ++sc) {  // join every forked stream, also after an error
        cudaError_t e = cudaEventRecord(ss.join[sc - 1], ss.st[sc - 1]);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(s, ss.join[sc - 1], 0);
        if (e != cudaSuccess && rc == MG_OK) rc = set_error(MG_ERR_CUDA, "launch_msd_forward: join: %s", cudaGetErrorString(e));
    }
    return rc;
}

}  // namespace mg
