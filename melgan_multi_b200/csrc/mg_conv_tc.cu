// Stride-1 "same" Conv1d with a dense channel contraction on the tensor cores (wgmma, split-bf16).
//
// Used for   Generator.conv_pre      Conv1d(80 -> 512, k7, pad 3)                       models.py:46,62
//            Discriminator.conv_post1 Conv1d(1024 -> 1024, k5, pad 2) + LeakyReLU       models.py:84,96-97
//
// GEMM view: D[v, co] = sum_tap sum_pass X_pass[v + tap - PAD, :] * W_pass[tap][co, :]^T with M = 128 virtual positions
// (two warpgroups of 64 rows), N = 128 output channels, K = 16 per instruction.  Rows are VIRTUAL positions: the
// batch items are concatenated with PAD zero rows after each item (v = item*(L+PAD) + s), so every tap -- the same A
// buffer read `tap - PAD` rows further (row-linear operand layout, mg_tc.cuh) -- sees exactly the zero padding of the
// reference and short sequences (L = 17..128 in the discriminators, 32 in the generator) still fill the 128-row tile.
// One CTA = 128 virtual positions x one group of N output channels; K = Cin is streamed: A slots (KCA channels, hi/lo
// split of x) are produced by the converter warps straight from the fp32 NCL input, B slots (one tap of 16 input
// channels: [hi, lo][k-panel][N][8] bf16 = 64 N bytes) arrive by 1-D bulk TMA.
// Warp roles: converter warpgroup (A slots), two MMA warpgroups (rows 0..63 / 64..127; accumulators in registers, they
// also run the epilogue), one TMA producer warp.
#include <type_traits>

#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {
using namespace tc;

template <int CIN_, int COUT_, int NTAP_, int KCA_, bool LRELU_OUT_, int N_>
struct ConvCfg {
    static constexpr int CIN = CIN_, COUT = COUT_, NTAP = NTAP_, PAD = NTAP_ / 2, KCA = KCA_;
    static constexpr bool LRELU_OUT = LRELU_OUT_;
    static constexpr int N = N_;                            // output channels per CTA (MMA N)
    static constexpr int NCG = COUT / N;
    static constexpr int ROWS = 128;
    static constexpr int AROWS = ROWS + 2 * PAD + 2;        // row index i <-> virtual position r0 - PAD + i
    static constexpr int APITCH = AROWS * 16;
    static constexpr int ASLOT = 2 * (KCA / 8) * APITCH;    // [half][k-panel][AROWS][16 B]
    static constexpr int BSLOT = 2 * 2 * N * 16;            // [half][k-panel: 2][N][16 B]
    // B ring: a CTA streams CIN/16 * NTAP slots and each is consumed in 3 MMAs per warpgroup, far less than a bulk copy's
    // latency, so the ring depth (bytes in flight) sets the pace: 8 x 8 KB for the N = 128 tiles, 4 x 16 KB for N = 256
    static constexpr int NSA = (CIN == KCA) ? 1 : 2, NSB = (N_ == 128) ? 8 : 4;
    static constexpr int NCONV = 128, NMW = 2;              // converter threads, MMA warpgroups
    static constexpr int NT = NCONV + 128 * NMW + 32;
    static constexpr int SMEM_BYTES = NSA * ASLOT + NSB * BSLOT + (2 * NSA + 2 * NSB) * 8;
    static_assert(CIN % KCA == 0 && KCA % 16 == 0 && COUT % N == 0, "shape");
    static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
};

// packed weights for this kernel: conv_tc_weight_index() in mg_layout.h

// Virtual row -> (item, position, the item's length); item -1: no item.  The discriminators' batches are dense: B items of
// L positions, PAD zero rows after each.  The generator's conv_pre takes a RunTable instead (ragged batches; one unit
// per virtual row, L_i + PAD of them per item, items `stride` positions apart).
struct DenseRows {
    int stride, B, pad;
    __device__ __forceinline__ RunPos find(int v) const {
        const int Lv = stride + pad, item = v >= 0 ? v / Lv : 0;
        return (v >= 0 && item < B) ? RunPos{item, v - item * Lv, stride} : RunPos{-1, 0, 0};
    }
};

template <class Cfg, class Rows>
__global__ void __launch_bounds__(Cfg::NT, 1)
conv_rows_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const uint8_t *__restrict__ wtc,
                    const float *__restrict__ bias, const __grid_constant__ Rows rows, int *__restrict__ status) {
    constexpr int CIN = Cfg::CIN, COUT = Cfg::COUT, NTAP = Cfg::NTAP, PAD = Cfg::PAD, KCA = Cfg::KCA, N = Cfg::N;
    constexpr int ROWS = Cfg::ROWS, APITCH = Cfg::APITCH, ASLOT = Cfg::ASLOT, BSLOT = Cfg::BSLOT;
    constexpr int NSA = Cfg::NSA, NSB = Cfg::NSB, NCONV = Cfg::NCONV, NMW = Cfg::NMW;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *aring = smem, *bring = smem + NSA * ASLOT;
    uint64_t *fullA = reinterpret_cast<uint64_t *>(bring + NSB * BSLOT);
    uint64_t *emptyA = fullA + NSA, *fullB = emptyA + NSA, *emptyB = fullB + NSB;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = blockIdx.x * ROWS, cg = blockIdx.y;
    const int L = rows.stride;  // positions between items in x and y
    if constexpr (std::is_same<Rows, RunTable>::value) {  // conv_pre: the weights of the tile's voice (set_units keeps a
        const float *vb = rows.blob_at(r0);               // tile within one voice; rows of the gap are never stored)
        wtc = reinterpret_cast<const uint8_t *>(vb) + tc_region_start() + tc_pre_offset();
        bias = vb + bias_offset(0);
    }

    if (tid == 0) {
        for (int s = 0; s < NSA; ++s) { mbar_init(&fullA[s], NCONV); mbar_init(&emptyA[s], NMW); }
        for (int s = 0; s < NSB; ++s) { mbar_init(&fullB[s], 1); mbar_init(&emptyB[s], NMW); }  // one arrival per MMA warpgroup
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == (NCONV + 128 * NMW) / 32) {
        // ================= TMA producer: B slot = (16-channel chunk, tap) =================
        if (lane == 0) {
            const uint8_t *src = wtc + (size_t)cg * (CIN / 16) * NTAP * BSLOT;
            int s = 0, ph = 0;
            bool ok = true;
            for (int i = 0; i < (CIN / 16) * NTAP && ok; ++i) {
                if (!mbar_wait(&emptyB[s], ph ^ 1)) { ok = false; break; }
                mbar_arrive_expect_tx(&fullB[s], BSLOT);
                bulk_g2s(bring + s * BSLOT, src + (size_t)i * BSLOT, BSLOT, &fullB[s]);
                if (++s == NSB) { s = 0; ph ^= 1; }
            }
            if (!ok) atomicExch(status, 22);
        }
    } else if (warp >= NCONV / 32) {
        // ================= MMA warpgroups: rows [64 mw, 64 mw + 64) of the tile, all N columns =================
        const int mw = warp / 4 - NCONV / 128, t = tid & 127;
        const uint64_t adesc_t = desc_template(APITCH, 128), bdesc_t = desc_template(N * 16, 128);
        const uint32_t aring_addr = smem_u32(aring) + mw * 64 * 16, bring_addr = smem_u32(bring);
        float acc[N / 2];
        int sa = 0, pha = 0, sb = 0, phb = 0;
        int psb = -1, psa = -1;  // ring slots read by the MMA group still in flight (freed once it completes)
        bool ok = true;
#pragma unroll 1
        for (int ca = 0; ca < CIN / KCA; ++ca) {
            ok &= mbar_wait(&fullA[sa], pha);
            const uint64_t abase = desc_at(adesc_t, aring_addr + sa * ASLOT);
#pragma unroll 1
            for (int j = 0; j < KCA / 16; ++j) {
#pragma unroll 1
                for (int tap = 0; tap < NTAP; ++tap) {
                    ok &= mbar_wait(&fullB[sb], phb);
                    const uint64_t bbase = desc_at(bdesc_t, bring_addr + sb * BSLOT);
                    // A rows for this tap start at index `tap` (row i <-> v = r0 - PAD + i; the tap reads v + tap - PAD)
                    const uint64_t arow = abase + (uint64_t)tap + (uint64_t)(2 * j * (APITCH >> 4));
                    wgmma_fence();
#pragma unroll
                    for (int pass = 0; pass < 3; ++pass) {
                        const uint64_t adesc = arow + (uint64_t)(((pass == 1) * (KCA / 8) * APITCH) >> 4);
                        const uint64_t bdesc = bbase + (uint64_t)(((pass == 2) * 2 * N * 16) >> 4);
                        wgmma_bf16<N>(acc, adesc, bdesc, (ca | j | tap | pass) != 0);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();  // the previous slot's MMAs are complete: free its ring slots
                    if (t == 0 && psb >= 0) {
                        mbar_arrive(&emptyB[psb]);
                        if (psa >= 0) mbar_arrive(&emptyA[psa]);
                    }
                    psb = sb;
                    psa = (j == KCA / 16 - 1 && tap == NTAP - 1) ? sa : -1;
                    if (++sb == NSB) { sb = 0; phb ^= 1; }
                }
            }
            if (++sa == NSA) { sa = 0; pha ^= 1; }
        }
        wgmma_wait<0>();
        acc_fence<N / 2>(acc);
        if (!ok && t == 0) atomicExch(status, 23);
        pdl_trigger();  // MMAs done, only the output store is left: the next kernel of the chain may be scheduled
        pdl_wait();     // (y may still be read by the previous kernel of the chain)
        // ================= epilogue: D[v, co] + bias (-> LeakyReLU) -> y[item][co][s] =================
        const float *bp = bias + cg * N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const RunPos p = rows.find(r0 + 64 * mw + frag_row(t, h));
            if (p.item >= 0 && p.unit < p.len) {
                float *yp = y + ((size_t)p.item * COUT + cg * N) * L + p.unit;
#pragma unroll
                for (int k = 0; k < N / 8; ++k)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = frag_col(lane & 3, 4 * k + e);
                        float o = acc[4 * k + 2 * h + e] + __ldg(bp + col);
                        if (Cfg::LRELU_OUT) o = lrelu(o);
                        yp[(size_t)col * L] = o;
                    }
            }
        }
    } else {
        // ================= converter warps: A slots = split(x), KCA channels of every row =================
        // Thread tid owns row tid of every slot and keeps the NEXT chunk's KCA loads in flight while it converts the
        // current one (the chain of dependent memory round trips bounds a CTA: 32 chunks at K = 1024);
        // the 2 PAD rows beyond the first NCONV are picked up by the first threads without prefetch.
        pdl_wait();  // x: the previous kernel's output
        int sa = 0, pha = 0;
        bool ok = true;
        constexpr int NCH = CIN / KCA;
        const RunPos p0 = rows.find(r0 - PAD + tid);
        const bool inr0 = p0.item >= 0 && p0.unit < p0.len;
        const float *xrow = x + (size_t)(inr0 ? p0.item : 0) * CIN * L + (inr0 ? p0.unit : 0);
        auto store_row = [&](uint8_t *slot, int i, const float *f) {
#pragma unroll
            for (int kp = 0; kp < KCA / 8; ++kp) {
                uint32_t h[4], l[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) split2_bf16(f[8 * kp + 2 * e], f[8 * kp + 2 * e + 1], h[e], l[e]);
                *reinterpret_cast<uint4 *>(slot + kp * APITCH + i * 16) = make_uint4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<uint4 *>(slot + (KCA / 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
            }
        };
        auto tail_rows = [&](uint8_t *slot, int ca) {
#pragma unroll 1
            for (int i = NCONV + tid; i < ROWS + 2 * PAD; i += NCONV) {
                const RunPos p = rows.find(r0 - PAD + i);
                const bool inr = p.item >= 0 && p.unit < p.len;
                const float *xp = x + ((size_t)(inr ? p.item : 0) * CIN + ca * KCA) * L + (inr ? p.unit : 0);
                float f[KCA];
#pragma unroll
                for (int j = 0; j < KCA; ++j) f[j] = inr ? __ldg(xp + (size_t)j * L) : 0.f;
                store_row(slot, i, f);
            }
        };
        float fa[KCA], fb[KCA];  // chunk ca (even / odd) of this thread's row
#pragma unroll
        for (int j = 0; j < KCA; ++j) fa[j] = inr0 ? __ldg(xrow + (size_t)j * L) : 0.f;
#pragma unroll 1
        for (int ca = 0; ca < NCH; ca += 2) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int cc = ca + half;
                if (cc < NCH) {
                    float *cur = half ? fb : fa, *nxt = half ? fa : fb;
                    if (cc + 1 < NCH) {  // next chunk's loads go out before this chunk is converted
#pragma unroll
                        for (int j = 0; j < KCA; ++j) nxt[j] = inr0 ? __ldg(xrow + (size_t)((cc + 1) * KCA + j) * L) : 0.f;
                    }
                    if (ok && !mbar_wait(&emptyA[sa], pha ^ 1)) { ok = false; if (lane == 0) atomicExch(status, 24); }
                    uint8_t *slot = aring + sa * ASLOT;
                    store_row(slot, tid, cur);
                    tail_rows(slot, cc);
                    fence_proxy_async();
                    mbar_arrive(&fullA[sa]);
                    if (++sa == NSA) { sa = 0; pha ^= 1; }
                }
            }
        }
    }
}

// vrows: virtual rows of the batch (the grid covers them in 128-row tiles)
template <class Cfg, class Rows>
static int launch_conv_rows(const float *x, float *y, const uint8_t *wtc, const float *bias, const Rows &rows, long long vrows,
                            int *status, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(conv_rows_tc_kernel<Cfg, Rows>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES));
        configured = true;
    }
    const unsigned tiles = (unsigned)((vrows + Cfg::ROWS - 1) / Cfg::ROWS);
    MG_CUDA_TRY(launch_ex(conv_rows_tc_kernel<Cfg, Rows>, dim3(tiles, Cfg::NCG), dim3(Cfg::NT), Cfg::SMEM_BYTES, s, true, 1, x, y, wtc,
                          bias, rows, status));
    return MG_OK;
}

template <class Cfg>
static int launch_conv_dense(const float *x, float *y, const uint8_t *wtc, const float *bias, int B, int L, int *status,
                             cudaStream_t s) {
    return launch_conv_rows<Cfg>(x, y, wtc, bias, DenseRows{L, B, Cfg::PAD}, (long long)B * (L + Cfg::PAD), status, s);
}

using PreCfg = ConvCfg<80, 512, 7, 80, false, kPreNG>;  // generator conv_pre
// discriminator conv_post1 (+ LeakyReLU): N = 128 per CTA, 8 channel groups -> 8x the row tiles' CTAs (264 + 136 + 40 per
// group at 8192 samples over the three scales), so the grid spans several waves of the 132 SMs
using Post1Cfg = ConvCfg<1024, 1024, 5, 32, true, kPost1NG>;
using Post1DgradCfg = ConvCfg<1024, 1024, 5, 32, false, kPost1NG>;  // the same contraction on the transposed blob, no activation

// mel [B][80][T_max] -> y [B][512][T_max]   (Generator.conv_pre), item i's first len_i positions, on its run's blob
int launch_gen_pre_tc(const float *mel, float *y, const RunTable &batch, int *status, cudaStream_t s) {
    RunTable rows = batch;
    rows.set_units([](int L) { return L + PreCfg::PAD; }, PreCfg::ROWS);
    return launch_conv_rows<PreCfg>(mel, y, nullptr, nullptr, rows, rows.first[rows.n], status, s);  // (weights: rows.blob)
}

// conv_pre's tile geometry: ROWS virtual rows per CTA (each item's positions followed by PAD zero rows), N output channels
const char *gen_pre_config_name() {
    static char buf[80];
    snprintf(buf, sizeof(buf), "conv_rows_tc_kernel<ConvCfg<%d,%d,%d,%d,%d>>", PreCfg::CIN, PreCfg::COUT, PreCfg::NTAP, PreCfg::ROWS,
             PreCfg::N);
    return buf;
}

// x [Bt][1024][L] -> y [Bt][1024][L] = lrelu(conv_post1(x))   (Discriminator.conv_post1)
int launch_disc_post1_tc(const float *x, float *y, const uint8_t *wtc, const float *bias, int Bt, int L, int *status,
                         cudaStream_t s) {
    return launch_conv_dense<Post1Cfg>(x, y, wtc, bias, Bt, L, status, s);
}

// dz [Bt][1024][L] -> dx [Bt][1024][L]: data gradient of conv_post1 (autograd of models.py:96), wtcT = blob + d_tcT_start()
int launch_disc_post1_dgrad_tc(const float *dz, float *dx, const uint8_t *wtcT, const float *zero_bias, int Bt, int L, int *status,
                               cudaStream_t s) {
    return launch_conv_dense<Post1DgradCfg>(dz, dx, wtcT, zero_bias, Bt, L, status, s);
}

}  // namespace mg
