// LeakyReLU -> ConvTranspose1d on the tensor cores (wgmma, split-bf16).
//
// Reference: Generator.forward, models.py:64-65 -- x = ups[i](F.leaky_relu(x)); ConvTranspose1d(Cin, Cout, K=2S, stride S,
// padding S/2), models.py:48-51.
//
// A transposed conv with K = 2S is, per output phase phi = (t + pad) mod S, a 2-tap conv over the INPUT positions:
//     out[co][S*s + phi - pad] = sum_ci  x[ci][s] * W[ci][co][phi]  +  x[ci][s-1] * W[ci][co][phi + S]
// All S phases of a tap read the same activation rows, so they are stacked along the MMA N dimension:
//     D[s, phi*NG + co] (+)= X[s - tap, :] * Wstack_tap[phi*NG + co, :]^T,   M = 64 input positions per warpgroup,
//     N = S*NG (256 for the stride-8 stages), K = 16 per instruction,
// i.e. 2 taps x 3 split-bf16 passes = 6 instructions per 16 input channels cover every phase.  The s-1 tap is the same
// A buffer read one row earlier (row-linear operand layout, mg_tc.cuh).  Because all S phases of a (row, channel) sit in
// the same thread's accumulator registers, the epilogue stores the S consecutive output samples [S*s - pad, S*s - pad + S)
// of a channel as contiguous vectors.
//
// Rows are VIRTUAL input positions: the batch items are concatenated with one zero row after each item (item i's rows
// s in [0, Lin_i], row s = Lin_i is zero; RunTable maps a row to its item), so that x[-1] = x[Lin_i] = 0 falls out of the
// layout, short sequences (stage 0: Lin = 32) still fill 64-row blocks, and no row lies past an item's end in a ragged
// batch.  In memory every item keeps the padded layout: items `stride` input positions apart.
// One CTA = NMW blocks of 64 virtual input positions x one group of NG output channels.  K (= Cin) is streamed: the A
// slots (KCA channels: LeakyReLU + hi/lo split of x) are produced in shared memory by the converter warps straight from
// the fp32 NCL input (all KCA loads of a row in flight at once), the B slots (16 channels: both taps, hi and lo, all
// phases) arrive by 1-D bulk TMA from the pre-packed blob (mg_layout.h).
// Warp roles: converter warpgroup, NMW MMA warpgroups (one per 64-row block; accumulators in registers, they also run
// the epilogue), TMA producer warp.  An N = 256 tile is 128 accumulator registers per thread, so the stride-8 stages run
// one MMA warpgroup per CTA.
#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {
using namespace tc;

template <int STAGE_>
struct UpCfg {
    static constexpr int STAGE = STAGE_;
    static constexpr int CIN = stage_cin(STAGE), COUT = stage_cout(STAGE), S = stage_stride(STAGE), PAD = stage_pad(STAGE);
    static constexpr int NG = up_ng(STAGE);
    static constexpr int NCG = COUT / NG;
    static constexpr int N = S * NG;                      // MMA N: every phase of the channel group
    static constexpr int NMW = (N > 128) ? 1 : 2;         // MMA warpgroups = 64-row blocks per CTA
    // channels per A slot = channels fetched per memory round trip of a converter thread
    static constexpr int KCA = (S == 8) ? 64 : 32;
    static constexpr int ROWS = 64 * NMW;
    static constexpr int AROWS = ROWS + 8;                // row index i <-> virtual position r0 - 1 + i, i in [0, ROWS]
    static constexpr int APITCH = AROWS * 16;             // bytes between k-panels
    static constexpr int ASLOT = 2 * (KCA / 8) * APITCH;  // [half: hi, lo][k-panel][AROWS][16 B]
    static constexpr int BSLOT = up_slot_bytes(STAGE);    // [tap][half][k-panel: 2][N][16 B]
    static constexpr int NSA = (CIN == KCA) ? 1 : 2, NSB = (S == 8) ? 4 : (CIN >= 128 ? 2 : 3);
    static constexpr int NCHUNK = CIN / 16;               // B slots per tile
    static constexpr int NCONV = 128;                     // converter threads
    static constexpr int NT = NCONV + 128 * NMW + 32;
    static constexpr int SMEM_BYTES = NSA * ASLOT + NSB * BSLOT + (2 * NSA + 2 * NSB) * 8;
    static_assert(N <= 256 && N % 16 == 0, "wgmma N");
    static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
    static_assert(CIN % KCA == 0, "A slot");
};

// D[s, phi*NG + co] + bias -> out[co][S*s + phi - pad] for the two accumulator rows of this thread (block-local rows
// m = 64 mw + frag_row(t, h)); row(m): the row's RunPos; Lout: output positions between items
template <class Cfg, class Row>
__device__ __forceinline__ void convt_store(const float *acc, float *__restrict__ y, const float *__restrict__ bias, int mw, int t,
                                            int cg, int Lout, Row row) {
    constexpr int S = Cfg::S, NG = Cfg::NG, N = Cfg::N, COUT = Cfg::COUT, PAD = Cfg::PAD;
    const int q = t & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        // one row's lookup at a time, after the previous row's stores: overlapped, the lookups would be live next to the
        // whole accumulator
        int m = 64 * mw + frag_row(t, h);
        asm volatile("" : "+r"(m) : : "memory");
        const RunPos p = row(m);
        const int s = p.unit;
        const bool row_ok = p.item >= 0;
        const bool lo_ok = row_ok && s >= 1, hi_ok = row_ok && s <= p.len - 1;
        float *yb = y + ((size_t)(row_ok ? p.item : 0) * COUT + cg * NG) * Lout + (S * s - PAD);
        if constexpr (S == 8) {
            // column 8k + 2q + e = phi * 32 + co: block k holds phase k / 4 of channels 8 (k % 4) + 2q + e
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int co = 8 * c + 2 * q + e;
                    const float bj = __ldg(bias + co);
                    float *yp = yb + (size_t)co * Lout;
                    if (lo_ok)
                        *reinterpret_cast<float4 *>(yp) =
                            make_float4(acc[4 * (0 + c) + 2 * h + e] + bj, acc[4 * (4 + c) + 2 * h + e] + bj,
                                        acc[4 * (8 + c) + 2 * h + e] + bj, acc[4 * (12 + c) + 2 * h + e] + bj);
                    if (hi_ok)
                        *reinterpret_cast<float4 *>(yp + 4) =
                            make_float4(acc[4 * (16 + c) + 2 * h + e] + bj, acc[4 * (20 + c) + 2 * h + e] + bj,
                                        acc[4 * (24 + c) + 2 * h + e] + bj, acc[4 * (28 + c) + 2 * h + e] + bj);
                }
        } else {  // S == 2: out[2s - 1] (phase 0) and out[2s] (phase 1)
#pragma unroll
            for (int k = 0; k < N / 8; ++k)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = frag_col(q, 4 * k + e), phi = col / NG, co = col % NG;
                    const float o = acc[4 * k + 2 * h + e] + __ldg(bias + co);
                    if (phi == 0 ? lo_ok : hi_ok) yb[(size_t)co * Lout + phi] = o;
                }
        }
    }
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NT, 1)
convt_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const float *__restrict__ packed,
                const __grid_constant__ RunTable rows, int *__restrict__ status) {
    constexpr int CIN = Cfg::CIN, N = Cfg::N, NG = Cfg::NG;
    constexpr int ROWS = Cfg::ROWS, APITCH = Cfg::APITCH, ASLOT = Cfg::ASLOT, BSLOT = Cfg::BSLOT, KCA = Cfg::KCA;
    constexpr int NSA = Cfg::NSA, NSB = Cfg::NSB, NCHUNK = Cfg::NCHUNK, NCONV = Cfg::NCONV, NMW = Cfg::NMW;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *aring = smem, *bring = smem + NSA * ASLOT;
    uint64_t *fullA = reinterpret_cast<uint64_t *>(bring + NSB * BSLOT);
    uint64_t *emptyA = fullA + NSA, *fullB = emptyA + NSA, *emptyB = fullB + NSB;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = blockIdx.x * ROWS;  // first virtual row of the tile
    const int cg = blockIdx.y;
    const int Lin = rows.stride;  // input positions between items

    if (tid == 0) {
        for (int s = 0; s < NSA; ++s) { mbar_init(&fullA[s], NCONV); mbar_init(&emptyA[s], NMW); }
        for (int s = 0; s < NSB; ++s) { mbar_init(&fullB[s], 1); mbar_init(&emptyB[s], NMW); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == (NCONV + 128 * NMW) / 32) {
        // ================= TMA producer: one B slot per 16 input channels =================
        if (lane == 0) {
            const uint8_t *src = reinterpret_cast<const uint8_t *>(packed) + tc_region_start() + tc_up_offset(Cfg::STAGE) +
                                 (size_t)cg * NCHUNK * BSLOT;
            int s = 0, ph = 0;
            bool ok = true;
            for (int i = 0; i < NCHUNK && ok; ++i) {
                if (!mbar_wait(&emptyB[s], ph ^ 1)) { ok = false; break; }
                mbar_arrive_expect_tx(&fullB[s], BSLOT);
                bulk_g2s(bring + s * BSLOT, src + (size_t)i * BSLOT, BSLOT, &fullB[s]);
                if (++s == NSB) { s = 0; ph ^= 1; }
            }
            if (!ok) atomicExch(status, 12);
        }
    } else if (warp >= NCONV / 32) {
        // ================= MMA warpgroup mw: rows [64 mw, 64 mw + 64) =================
        const int mw = warp / 4 - NCONV / 128, t = tid & 127;
        const uint64_t adesc_t = desc_template(APITCH, 128), bdesc_t = desc_template(N * 16, 128);
        const uint32_t aring_addr = smem_u32(aring) + mw * 64 * 16, bring_addr = smem_u32(bring);
        float acc[N / 2];
        int sa = 0, pha = 0, sb = 0, phb = 0, psb = -1, psa = -1;
        bool ok = true;  // a timed-out wait only raises the status word: control flow stays uniform
#pragma unroll 1
        for (int ca = 0; ca < CIN / KCA; ++ca) {
            ok &= mbar_wait(&fullA[sa], pha);
            const uint64_t abase = desc_at(adesc_t, aring_addr + sa * ASLOT);
#pragma unroll 1
            for (int j = 0; j < KCA / 16; ++j) {
                ok &= mbar_wait(&fullB[sb], phb);
                const uint64_t bbase = desc_at(bdesc_t, bring_addr + sb * BSLOT);
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 2; ++tap)
#pragma unroll
                    for (int pass = 0; pass < 3; ++pass) {
                        const int ahalf = (pass == 1), bhalf = (pass == 2);
                        const uint64_t bdesc = bbase + (uint64_t)((((tap * 2 + bhalf) * 2) * N * 16) >> 4);
                        const uint64_t adesc =
                            abase + (uint64_t)((ahalf * (KCA / 8) * APITCH + (1 - tap) * 16) >> 4) + (uint64_t)(2 * j * (APITCH >> 4));
                        wgmma_bf16<N>(acc, adesc, bdesc, (ca | j | tap | pass) != 0);
                    }
                wgmma_commit();
                wgmma_wait<1>();
                if (t == 0 && psb >= 0) {
                    mbar_arrive(&emptyB[psb]);
                    if (psa >= 0) mbar_arrive(&emptyA[psa]);
                }
                psb = sb;
                psa = (j == KCA / 16 - 1) ? sa : -1;
                if (++sb == NSB) { sb = 0; phb ^= 1; }
            }
            if (++sa == NSA) { sa = 0; pha ^= 1; }
        }
        wgmma_wait<0>();
        acc_fence<N / 2>(acc);
        if (!ok && t == 0) atomicExch(status, 13);
        pdl_trigger();  // MMAs done, only the output store is left: the next kernel of the chain may be scheduled
        pdl_wait();
        convt_store<Cfg>(acc, y, packed + bias_offset(1 + Cfg::STAGE) + cg * NG, mw, t, cg, Cfg::S * Lin,
                         [&](int m) { return rows.find(r0 + m); });
    } else {
        // ================= converter warps: A slots = split(lrelu(x)), KCA channels of every row =================
        pdl_wait();  // x: the previous kernel's output
        int sa = 0, pha = 0;
        bool ok = true;
#pragma unroll 1
        for (int ca = 0; ca < CIN / KCA; ++ca) {
            if (ok && !mbar_wait(&emptyA[sa], pha ^ 1)) { ok = false; if (lane == 0) atomicExch(status, 14); }
            uint8_t *slot = aring + sa * ASLOT;
#pragma unroll 1
            for (int i = tid; i <= ROWS; i += NCONV) {
                const RunPos p = rows.find(r0 - 1 + i);
                const bool inr = p.item >= 0 && p.unit < p.len;
                const float *xp = x + ((size_t)(inr ? p.item : 0) * CIN + ca * KCA) * Lin + (inr ? p.unit : 0);
                float f[KCA];
#pragma unroll
                for (int j = 0; j < KCA; ++j) f[j] = inr ? __ldg(xp + (size_t)j * Lin) : 0.f;  // all in flight together
#pragma unroll
                for (int kp = 0; kp < KCA / 8; ++kp) {
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) split2_bf16(lrelu(f[8 * kp + 2 * e]), lrelu(f[8 * kp + 2 * e + 1]), h[e], l[e]);
                    *reinterpret_cast<uint4 *>(slot + kp * APITCH + i * 16) = make_uint4(h[0], h[1], h[2], h[3]);
                    *reinterpret_cast<uint4 *>(slot + (KCA / 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
                }
            }
            fence_proxy_async();
            mbar_arrive(&fullA[sa]);
            if (++sa == NSA) { sa = 0; pha ^= 1; }
        }
    }
}

// Lin + 1 virtual rows per item: position s = Lin feeds the last `pad` outputs
static RunTable convt_rows(const RunTable &batch) {
    RunTable rows = batch;
    rows.set_units([](int Lin) { return Lin + 1; });
    return rows;
}

template <class Cfg>
static int launch_convt(const float *x, float *y, const float *packed, const RunTable &batch, int *status, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(convt_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        configured = true;
    }
    const RunTable rows = convt_rows(batch);
    dim3 grid((unsigned)((rows.first[rows.n] + Cfg::ROWS - 1) / Cfg::ROWS), Cfg::NCG);
    MG_CUDA_TRY(launch_ex(convt_tc_kernel<Cfg>, grid, dim3(Cfg::NT), Cfg::SMEM_BYTES, s, true, 1, x, y, packed, rows, status));
    return MG_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Variant for a stage whose whole activation tile fits in shared memory (stage 1: 65 rows x 256 channels, hi+lo =
// 72 KB): the A operand is converted ONCE per row tile and stays resident, and the CTA loops over the NCG output-channel
// groups, so no activation is loaded or converted twice.  One MMA warpgroup (64 rows, N = 256) per CTA.  The converter
// also parks the tile's 64 row lookups in shared memory for the epilogue, which runs once per channel group.
template <class Cfg>
__global__ void __launch_bounds__(Cfg::NCONV + 128 + 32, 1)
convt_resident_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const float *__restrict__ packed,
                         const __grid_constant__ RunTable rows, int *__restrict__ status) {
    constexpr int CIN = Cfg::CIN, NG = Cfg::NG, N = Cfg::N, NCG = Cfg::NCG;
    constexpr int ROWS = 64, APITCH = Cfg::APITCH, BSLOT = Cfg::BSLOT, NCHUNK = Cfg::NCHUNK;
    constexpr int KPT = CIN / 8;                    // k-panels of the resident A
    constexpr int AHALF = KPT * APITCH;             // bytes of one of {hi, lo}
    constexpr int NSB = 4, NCONV = Cfg::NCONV;
    static_assert(Cfg::S == 8 && N == 256 && Cfg::NMW == 1 && 2 * AHALF + NSB * BSLOT + 256 + ROWS * 12 <= 227 * 1024,
                  "resident ConvT shape");
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *abuf = smem, *bring = smem + 2 * AHALF;
    uint64_t *fullA = reinterpret_cast<uint64_t *>(bring + NSB * BSLOT);  // [CIN/64]: a 64-channel slice of A is written
    uint64_t *fullB = fullA + CIN / 64, *emptyB = fullB + NSB;
    RunPos *srow = reinterpret_cast<RunPos *>(emptyB + NSB);  // [ROWS]: virtual row r0 + m, written with A's first slice

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = blockIdx.x * ROWS;
    const int Lin = rows.stride;  // input positions between items

    if (tid == 0) {
        for (int s = 0; s < CIN / 64; ++s) mbar_init(&fullA[s], NCONV);
        for (int s = 0; s < NSB; ++s) { mbar_init(&fullB[s], 1); mbar_init(&emptyB[s], 1); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCONV / 32 + 4) {
        // ================= TMA producer: B slots of every channel group, in consumption order =================
        if (lane == 0) {
            const uint8_t *src = reinterpret_cast<const uint8_t *>(packed) + tc_region_start() + tc_up_offset(Cfg::STAGE);
            int s = 0, ph = 0;
            bool ok = true;
            for (int i = 0; i < NCG * NCHUNK && ok; ++i) {  // blob order is [cg][chunk]: exactly this loop
                if (!mbar_wait(&emptyB[s], ph ^ 1)) { ok = false; break; }
                mbar_arrive_expect_tx(&fullB[s], BSLOT);
                bulk_g2s(bring + s * BSLOT, src + (size_t)i * BSLOT, BSLOT, &fullB[s]);
                if (++s == NSB) { s = 0; ph ^= 1; }
            }
            if (!ok) atomicExch(status, 32);
        }
    } else if (warp >= NCONV / 32) {
        // ================= MMA warpgroup: one channel group after the other =================
        const int t = tid & 127;
        const uint64_t adesc_t = desc_template(APITCH, 128), bdesc_t = desc_template(N * 16, 128);
        const uint32_t a_addr = smem_u32(abuf), bring_addr = smem_u32(bring);
        float acc[N / 2];
        int sb = 0, phb = 0, psb = -1;
        bool ok = true;
#pragma unroll 1
        for (int cg = 0; cg < NCG; ++cg) {
#pragma unroll 1
            for (int ch = 0; ch < NCHUNK; ++ch) {
                if (cg == 0 && (ch & 3) == 0) ok &= mbar_wait(&fullA[ch >> 2], 0);  // first pass only: the 64-channel slice of A
                ok &= mbar_wait(&fullB[sb], phb);
                const uint64_t bbase = desc_at(bdesc_t, bring_addr + sb * BSLOT);
                const uint64_t abase = desc_at(adesc_t, a_addr + 2 * ch * APITCH);
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 2; ++tap)
#pragma unroll
                    for (int pass = 0; pass < 3; ++pass) {
                        const uint64_t bdesc = bbase + (uint64_t)((((tap * 2 + (pass == 2)) * 2) * N * 16) >> 4);
                        const uint64_t adesc = abase + (uint64_t)((((pass == 1) ? AHALF : 0) + (1 - tap) * 16) >> 4);
                        wgmma_bf16<N>(acc, adesc, bdesc, (ch | tap | pass) != 0);
                    }
                wgmma_commit();
                wgmma_wait<1>();
                if (t == 0 && psb >= 0) mbar_arrive(&emptyB[psb]);
                psb = sb;
                if (++sb == NSB) { sb = 0; phb ^= 1; }
            }
            wgmma_wait<0>();
            acc_fence<N / 2>(acc);
            if (t == 0) { mbar_arrive(&emptyB[psb]); psb = -1; }
            if (cg == NCG - 1) pdl_trigger();  // last channel group's MMAs done: the next kernel may be scheduled
            if (cg == 0) pdl_wait();
            convt_store<Cfg>(acc, y, packed + bias_offset(1 + Cfg::STAGE) + cg * NG, 0, t, cg, Cfg::S * Lin,
                             [&](int m) { return ok ? srow[m] : RunPos{-1, 0, 0}; });  // (after fullA[0]: srow is complete)
        }
        if (!ok && t == 0) atomicExch(status, 33);
    } else {
        // ================= converter: the whole A tile, once =================
        pdl_wait();  // x: the previous kernel's output
#pragma unroll 1
        for (int ca = 0; ca < CIN / 64; ++ca) {
#pragma unroll 1
            for (int i = tid; i <= ROWS; i += NCONV) {
                const RunPos p = rows.find(r0 - 1 + i);
                if (ca == 0 && i > 0) srow[i - 1] = p;
                const bool inr = p.item >= 0 && p.unit < p.len;
                const float *xp = x + ((size_t)(inr ? p.item : 0) * CIN + ca * 64) * Lin + (inr ? p.unit : 0);
                float f[64];
#pragma unroll
                for (int j = 0; j < 64; ++j) f[j] = inr ? __ldg(xp + (size_t)j * Lin) : 0.f;
#pragma unroll
                for (int kp = 0; kp < 8; ++kp) {
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) split2_bf16(lrelu(f[8 * kp + 2 * e]), lrelu(f[8 * kp + 2 * e + 1]), h[e], l[e]);
                    *reinterpret_cast<uint4 *>(abuf + (ca * 8 + kp) * APITCH + i * 16) = make_uint4(h[0], h[1], h[2], h[3]);
                    *reinterpret_cast<uint4 *>(abuf + AHALF + (ca * 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
                }
            }
            fence_proxy_async();
            mbar_arrive(&fullA[ca]);
        }
    }
}

template <class Cfg>
static int launch_convt_resident(const float *x, float *y, const float *packed, const RunTable &batch, int *status, cudaStream_t s) {
    constexpr int smem = 2 * (Cfg::CIN / 8) * Cfg::APITCH + 4 * Cfg::BSLOT + (Cfg::CIN / 64 + 2 * 4) * 8 + 64 * sizeof(RunPos);
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(convt_resident_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    const RunTable rows = convt_rows(batch);
    MG_CUDA_TRY(launch_ex(convt_resident_tc_kernel<Cfg>, dim3((unsigned)((rows.first[rows.n] + 63) / 64)), dim3(Cfg::NCONV + 128 + 32),
                          smem, s, true, 1, x, y, packed, rows, status));
    return MG_OK;
}

// x [B][Cin][Lin] -> y [B][Cout][S*Lin], fp32 NCL, (Cin, Cout, S) of generator stage `stage`; Lin = batch.stride, item i's
// first len_i input positions (and S len_i output positions) are its own.
int launch_convt_tc(const float *x, float *y, const float *packed, int stage, const RunTable &batch, int *status, cudaStream_t s) {
    switch (stage) {
        case 0: return launch_convt<UpCfg<0>>(x, y, packed, batch, status, s);
        case 1: return launch_convt_resident<UpCfg<1>>(x, y, packed, batch, status, s);
        case 2: return launch_convt<UpCfg<2>>(x, y, packed, batch, status, s);
        case 3: return launch_convt<UpCfg<3>>(x, y, packed, batch, status, s);
    }
    return set_error(MG_ERR_INVALID_ARGUMENT, "launch_convt_tc: stage %d", stage);
}

}  // namespace mg
