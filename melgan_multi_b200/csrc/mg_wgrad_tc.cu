// Weight gradient of Discriminator.conv_post1 (Conv1d 1024 -> 1024, k5, pad 2; models.py:84,96) on the tensor cores
// (wgmma, split-bf16: fp32-grade, not TF32), plus its bias gradient.
//
//     dW[co][ci][tap] = sum_b sum_l dz[b][co][l] * x[b][ci][l + tap - 2]        db[co] = sum_b sum_l dz[b][co][l]
//
// GEMM view: M = 64 output channels, N = 64 input channels per tap with the five taps side by side (5 x 64 = 320 columns,
// two warpgroups of N = 160 over the same A rows), K = the positions of all items (K-major operands: in the NCL layout a
// channel's positions ARE contiguous).  One CTA = one (64 co) x (64 ci) tile of all five taps: 16 x 16 = 256 CTAs, each
// streaming the whole K extent once.
// A tap shifts x along K, i.e. by one bf16 INSIDE a 16-byte operand row -- not expressible as a descriptor offset -- so the
// converter warps write five shifted copies of the x tile next to one copy of the dz tile; the zero padding of the
// reference at the two ends of every item is produced there, which is also what lets items follow each other along K.
//   stage (32 positions = 2 K16 steps): A = split(dz) [hi|lo][4 k-panels][64 rows][16 B]        =  8 KB  (+ 32 B per panel)
//                                       B = split(x)  [hi|lo][4 k-panels][tap 5][64 rows][16 B] = 40 KB     x 3 stages
// Positions are padded per item to a multiple of 8 (one k-panel never straddles two items), the K extent to a multiple of 32.
#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {
using namespace tc;

namespace wg {
constexpr int C = 1024, NTAP = 5, PAD = 2;
constexpr int MT = 64, NTILE = 64;             // co rows / ci rows of a CTA
constexpr int NPANEL = 4;                      // k-panels (8 positions) per stage
constexpr int NB = NTAP * NTILE;                // B rows of a stage: the five shifted copies stacked along N (row = tap * 64 + ci)
constexpr int NMW = 2, NW = NB / NMW;           // MMA warpgroups, N of each
// k-panel pitches: + 32 bytes, so the four panels of a stage start 8 banks apart and a half-warp's 8-byte stores (2 rows x 4
// panels x 2 halves of a 16-byte operand row) hit 16 different bank pairs
constexpr int APANEL = MT * 16 + 32, BPANEL = NB * 16 + 32;
constexpr int AHALF = NPANEL * APANEL, BHALF = NPANEL * BPANEL;
constexpr int ASTAGE = 2 * AHALF, BSTAGE = 2 * BHALF, STAGE = ASTAGE + BSTAGE;
constexpr int NSTAGE = 3;
constexpr int NCONV = 256;                     // converter threads: 512 dz units + 512 x units (row, half k-panel) per stage
constexpr int NT = NCONV + 128 * NMW;
constexpr int SMEM_BYTES = NSTAGE * STAGE + 2 * NSTAGE * 8 + 2 * NCONV * 4;
static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
}  // namespace wg

// 4 consecutive positions [p0, p0 + 4) of one channel row (length L, base `row`), zero outside [0, L)
__device__ __forceinline__ void load4(const float *__restrict__ row, int p0, int L, bool vec, bool live, float *f) {
    if (vec) {  // L % 4 == 0, p0 % 4 == 0 and the row base is 16-byte aligned: the float4 is wholly inside or wholly outside
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && p0 >= 0 && p0 < L) v = __ldg(reinterpret_cast<const float4 *>(row + p0));
        f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) f[j] = (live && p0 + j >= 0 && p0 + j < L) ? __ldg(row + p0 + j) : 0.f;
    }
}

// half of a 16-byte operand row: 4 consecutive K elements, hi and lo parts
__device__ __forceinline__ void store_split4(uint8_t *hi_dst, uint8_t *lo_dst, const float *f) {
    uint32_t h[2], l[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) split2_bf16(f[2 * e], f[2 * e + 1], h[e], l[e]);
    *reinterpret_cast<uint2 *>(hi_dst) = make_uint2(h[0], h[1]);
    *reinterpret_cast<uint2 *>(lo_dst) = make_uint2(l[0], l[1]);
}

__global__ void __launch_bounds__(wg::NT, 1)
post1_wgrad_tc_kernel(const float *__restrict__ x, const float *__restrict__ dz, float *__restrict__ dw, float *__restrict__ db,
                      int Bt, int L, int *__restrict__ status) {
    using namespace wg;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + NSTAGE * STAGE);
    uint64_t *empty = full + NSTAGE;
    float *dbsum = reinterpret_cast<float *>(empty + NSTAGE);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int co0 = blockIdx.x * MT, ci0 = blockIdx.y * NTILE;
    const int ppi = (L + 7) >> 3;                 // k-panels per item
    const int npanels = Bt * ppi;
    const int nstages = (npanels + NPANEL - 1) / NPANEL;

    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], NCONV / 32); mbar_init(&empty[s], NMW); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= NCONV / 32) {
        // ================= MMA warpgroup mw: columns [160 mw, 160 mw + 160) of [tap][ci] =================
        const int mw = warp / 4 - NCONV / 128, t = tid & 127;
        const uint64_t adesc_t = desc_template(APANEL, 128), bdesc_t = desc_template(BPANEL, 128);
        const uint32_t base = smem_u32(smem);
        float acc[NW / 2];
        int s = 0, ph = 0, ps = -1;
        bool ok = true;
#pragma unroll 1
        for (int st = 0; st < nstages; ++st) {
            ok &= mbar_wait(&full[s], ph);
            const uint32_t a0 = base + s * STAGE, b0 = a0 + ASTAGE + mw * NW * 16;
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < NPANEL / 2; ++j) {
#pragma unroll
                for (int pass = 0; pass < 3; ++pass) {
                    const uint64_t adesc = desc_at(adesc_t, a0 + (pass == 1) * AHALF + 2 * j * APANEL);
                    const uint64_t bdesc = desc_at(bdesc_t, b0 + (pass == 2) * BHALF + 2 * j * BPANEL);
                    wgmma_bf16<NW>(acc, adesc, bdesc, (st | j | pass) != 0);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (t == 0 && ps >= 0) mbar_arrive(&empty[ps]);
            ps = s;
            if (++s == NSTAGE) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        acc_fence<NW / 2>(acc);
        if (!ok && t == 0) atomicExch(status, 26);
        // ================= epilogue: D[co][tap * 64 + ci] -> dW [co][ci][tap] =================
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float *out = dw + ((size_t)(co0 + frag_row(t, h)) * C + ci0) * NTAP;
#pragma unroll
            for (int k = 0; k < NW / 8; ++k)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = mw * NW + frag_col(lane & 3, 4 * k + e), tap = n / NTILE, ci = n % NTILE;
                    out[ci * NTAP + tap] = acc[4 * k + 2 * h + e];
                }
        }
    } else {
        // ================= converter warps =================
        // Unit = (channel row, HALF a k-panel: 4 positions = one float4).  The 8 lanes of an octet are the 8 float4 of one
        // row's 32 positions of the stage, a warp is 4 rows: every load instruction reads 4 x 128 contiguous bytes (4 cache
        // lines, all sectors used).  Thread: rows rq and rq + 32 of dz and of x.
        const bool vec = (L & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dz)) & 15) == 0;
        const int l8 = tid & 7, rq = tid >> 3, pm = l8 >> 1, hf = l8 & 1;
        float acc_db[2] = {0.f, 0.f};
        int s = 0, ph = 0;
        bool ok = true;
        // fa[u]: positions p0 .. p0+3 of dz row rq + 32u; fb[u]: positions p0-4 .. p0+7 of x row rq + 32u (p0 = 8c + 4 hf)
        auto load_stage = [&](int st, float (&fa)[2][4], float (&fb)[2][12]) {
            const int q = st * NPANEL + pm;
            const bool live = q < npanels;
            const int b = live ? q / ppi : 0, c = q - b * ppi, p0 = 8 * c + 4 * hf;
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                load4(dz + ((size_t)b * C + co0 + rq + 32 * u) * L, p0, L, vec, live, fa[u]);
                const float *row = x + ((size_t)b * C + ci0 + rq + 32 * u) * L;
#pragma unroll
                for (int k = 0; k < 3; ++k) load4(row, p0 - 4 + 4 * k, L, vec, live, &fb[u][4 * k]);
            }
        };
        auto store_stage = [&](const float (&fa)[2][4], const float (&fb)[2][12]) {
            if (ok && !mbar_wait(&empty[s], ph ^ 1)) { ok = false; if (lane == 0) atomicExch(status, 27); }
            uint8_t *a = smem + s * STAGE + pm * APANEL + hf * 8, *bb = smem + s * STAGE + ASTAGE + pm * BPANEL + hf * 8;
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                uint8_t *dst = a + (rq + 32 * u) * 16;
                store_split4(dst, dst + AHALF, fa[u]);
                acc_db[u] += (fa[u][0] + fa[u][1]) + (fa[u][2] + fa[u][3]);
#pragma unroll
                for (int tap = 0; tap < NTAP; ++tap) {
                    // X_tap[ci][l] = x[ci][l + tap - PAD]; fb[u][j] holds position p0 - 4 + j
                    uint8_t *dstb = bb + (tap * NTILE + rq + 32 * u) * 16;
                    store_split4(dstb, dstb + BHALF, &fb[u][4 + tap - PAD]);
                }
            }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(&full[s]);
            if (++s == NSTAGE) { s = 0; ph ^= 1; }
        };
        // software pipeline: the NEXT stage's global loads are in flight while this one is split and stored
        float fa0[2][4], fb0[2][12], fa1[2][4], fb1[2][12];
        load_stage(0, fa0, fb0);
#pragma unroll 1
        for (int st = 0; st < nstages; st += 2) {
            if (st + 1 < nstages) load_stage(st + 1, fa1, fb1);
            store_stage(fa0, fb0);
            if (st + 1 < nstages) {
                if (st + 2 < nstages) load_stage(st + 2, fa0, fb0);
                store_stage(fa1, fb1);
            }
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) dbsum[u * NCONV + tid] = acc_db[u];
    }
    __syncthreads();
    if (blockIdx.y == 0 && tid < MT) {  // row tid = 32 u + rq: the eight float4 lanes of that row, in position order
        const float *p = dbsum + (tid >> 5) * NCONV + (tid & 31) * 8;
        db[co0 + tid] = ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
    }
}

// x, dz [Bt][1024][L] -> dw [1024][1024][5], db [1024]
int launch_disc_post1_wgrad_tc(const float *x, const float *dz, float *dw, float *db, int Bt, int L, int *status, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(post1_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, wg::SMEM_BYTES));
        configured = true;
    }
    MG_CUDA_TRY(launch_ex(post1_wgrad_tc_kernel, dim3(wg::C / wg::MT, wg::C / wg::NTILE), dim3(wg::NT), wg::SMEM_BYTES, s, false, 1, x, dz,
                          dw, db, Bt, L, status));
    return MG_OK;
}

}  // namespace mg
