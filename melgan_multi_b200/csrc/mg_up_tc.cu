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
//
// The stride-2 stages (2, 3) move 4 bytes of input and 4 of output per 8 multiply-adds (x 3 passes): they are bound by
// memory, not by the tensor cores, so they run as a streaming kernel of their own (convt_stream_tc_kernel below): persistent
// CTAs, the weights resident in shared memory, each tile's input brought in by bulk copies several slots ahead of the
// converter, and an epilogue that stores pairs of neighbouring output samples.
//
// Bf16<UpCfg<0>> / Bf16<UpCfg<1>> (mg_tc.cuh): the stride-8 kernels with one pass (xh, wh) per product.  The converter
// writes the hi operand only, and each B slot is filled by two bulk copies, tap 0 hi and tap 1 hi (half the slot's bytes),
// at their usual offsets.  The streaming stride-2 kernel has no such variant: it is bound by memory, not by its MMAs.
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
    static constexpr bool ONEPASS = false;                // Bf16<UpCfg<..>>: one bf16 pass per product (mg_tc.cuh)
    static constexpr int N = S * NG;                      // MMA N: every phase of the channel group
    static constexpr int NMW = (N > 128) ? 1 : 2;         // MMA warpgroups = 64-row blocks per CTA
    // channels per A slot = channels fetched per memory round trip of a converter thread
    static constexpr int KCA = (S == 8) ? 64 : 32;
    static constexpr int ROWS = 64 * NMW;
    static constexpr int AROWS = ROWS + 8;                // row index i <-> virtual position r0 - 1 + i, i in [0, ROWS]
    static constexpr int APITCH = AROWS * 16;             // bytes between k-panels
    static constexpr int ASLOT = 2 * (KCA / 8) * APITCH;  // [half: hi, lo][k-panel][AROWS][16 B]
    static constexpr int BSLOT = up_slot_bytes(STAGE);    // [tap][half][k-panel: 2][N][16 B]
    static constexpr int NSA = (CIN == KCA) ? 1 : 2, NSB = 4;  // (convt_tc_kernel: stride 8)
    static constexpr int NCHUNK = CIN / 16;               // B slots per tile
    static constexpr int NCONV = 128;                     // converter threads
    static constexpr int NT = NCONV + 128 * NMW + 32;
    static constexpr int SMEM_BYTES = NSA * ASLOT + NSB * BSLOT + (2 * NSA + 2 * NSB + 1) * 8;  // (+ the tile's blob pointer)
    static_assert(N <= 256 && N % 16 == 0, "wgmma N");
    static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
    static_assert(CIN % KCA == 0, "A slot");
};

// D[s, phi*NG + co] + bias -> out[co][S*s + phi - pad] for the two accumulator rows of this thread (block-local rows
// m = 64 mw + frag_row(t, h)); row(m): the row's RunPos; Lout: output positions between items
template <class Cfg, class Row>
__device__ __forceinline__ void convt_store(const float *acc, float *__restrict__ y, const float *__restrict__ bias, int mw, int t,
                                            int cg, int Lout, Row row) {
    constexpr int S = Cfg::S, NG = Cfg::NG, COUT = Cfg::COUT, PAD = Cfg::PAD;
    static_assert(S == 8, "the stride-2 stages store through convt_stream_store");
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
    }
}

// B slot i of the blob ([tap][half: hi, lo][k-panel: 2][N][16 B]) into shared memory, completing on `bar`: the whole slot,
// or (single pass) its tap-0 hi and tap-1 hi quarters, at the same offsets
template <class Cfg>
__device__ __forceinline__ void load_bslot(uint8_t *dst, const uint8_t *src, uint64_t *bar) {
    constexpr uint32_t BSLOT = Cfg::BSLOT;
    if constexpr (Cfg::ONEPASS) {
        mbar_arrive_expect_tx(bar, BSLOT / 2);
        bulk_g2s(dst, src, BSLOT / 4, bar);
        bulk_g2s(dst + BSLOT / 2, src + BSLOT / 2, BSLOT / 4, bar);
    } else {
        mbar_arrive_expect_tx(bar, BSLOT);
        bulk_g2s(dst, src, BSLOT, bar);
    }
}

// The weights of the tile at virtual row r0: set_units keeps a tile within one voice.  Looked up where they are used
// (r0 opaque to the compiler), so that no pointer stays live next to the accumulators.
__device__ __forceinline__ const float *tile_blob(const RunTable &rows, int r0) {
    asm volatile("" : "+r"(r0));
    return rows.blob_at(r0);
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NT, 1)
convt_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const __grid_constant__ RunTable rows, int *__restrict__ status) {
    constexpr int CIN = Cfg::CIN, N = Cfg::N, NG = Cfg::NG;
    constexpr int ROWS = Cfg::ROWS, APITCH = Cfg::APITCH, ASLOT = Cfg::ASLOT, BSLOT = Cfg::BSLOT, KCA = Cfg::KCA;
    constexpr int NSA = Cfg::NSA, NSB = Cfg::NSB, NCHUNK = Cfg::NCHUNK, NCONV = Cfg::NCONV, NMW = Cfg::NMW;
    constexpr int NPASS = Cfg::ONEPASS ? 1 : 3;  // (xh, wh), (xl, wh), (xh, wl), or the first alone
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *aring = smem, *bring = smem + NSA * ASLOT;
    uint64_t *fullA = reinterpret_cast<uint64_t *>(bring + NSB * BSLOT);
    uint64_t *emptyA = fullA + NSA, *fullB = emptyA + NSA, *emptyB = fullB + NSB;
    // the tile's weights, looked up once: the epilogue reads the pointer back instead of searching the table while the
    // accumulators are live
    const float **vblob = reinterpret_cast<const float **>(emptyB + NSB);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = blockIdx.x * ROWS;  // first virtual row of the tile
    const int cg = blockIdx.y;
    const int Lin = rows.stride;  // input positions between items

    if (tid == 0) {
        *vblob = rows.blob_at(r0);  // set_units keeps a tile within one voice
        for (int s = 0; s < NSA; ++s) { mbar_init(&fullA[s], NCONV); mbar_init(&emptyA[s], NMW); }
        for (int s = 0; s < NSB; ++s) { mbar_init(&fullB[s], 1); mbar_init(&emptyB[s], NMW); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == (NCONV + 128 * NMW) / 32) {
        // ================= TMA producer: one B slot per 16 input channels =================
        if (lane == 0) {
            const uint8_t *src = reinterpret_cast<const uint8_t *>(*vblob) + tc_region_start() + tc_up_offset(Cfg::STAGE) +
                                 (size_t)cg * NCHUNK * BSLOT;
            int s = 0, ph = 0;
            bool ok = true;
            for (int i = 0; i < NCHUNK && ok; ++i) {
                if (!mbar_wait(&emptyB[s], ph ^ 1)) { ok = false; break; }
                load_bslot<Cfg>(bring + s * BSLOT, src + (size_t)i * BSLOT, &fullB[s]);
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
                    for (int pass = 0; pass < NPASS; ++pass) {
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
        const float *vb = *reinterpret_cast<const float *volatile *>(vblob);
        convt_store<Cfg>(acc, y, vb + bias_offset(1 + Cfg::STAGE) + cg * NG, mw, t, cg, Cfg::S * Lin,
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
                    if constexpr (!Cfg::ONEPASS)
                        *reinterpret_cast<uint4 *>(slot + (KCA / 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
                }
            }
            fence_proxy_async();
            mbar_arrive(&fullA[sa]);
            if (++sa == NSA) { sa = 0; pha ^= 1; }
        }
    }
}

// Lin + 1 virtual rows per item: position s = Lin feeds the last `pad` outputs; a voice starts at a multiple of `tile`
static RunTable convt_rows(const RunTable &batch, int tile) {
    RunTable rows = batch;
    rows.set_units([](int Lin) { return Lin + 1; }, tile);
    return rows;
}

template <class Cfg>
static int launch_convt(const float *x, float *y, const RunTable &batch, int *status, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(convt_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        configured = true;
    }
    const RunTable rows = convt_rows(batch, Cfg::ROWS);
    dim3 grid((unsigned)((rows.first[rows.n] + Cfg::ROWS - 1) / Cfg::ROWS), Cfg::NCG);
    MG_CUDA_TRY(launch_ex(convt_tc_kernel<Cfg>, grid, dim3(Cfg::NT), Cfg::SMEM_BYTES, s, true, 1, x, y, rows, status));
    return MG_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Streaming kernel of the stride-2 stages.  Per output element it computes exactly what convt_tc_kernel would (the same
// A and B operands, MMA order, 3 passes and bias add); only the data movement differs:
//  - persistent CTAs, one per SM (grid = min(tiles, SMs)), walk the row tiles blockIdx.x, + gridDim.x, ...  The layer's
//    whole B operand (NCHUNK slots: 128 KB at stage 2, one channel group) is loaded once per CTA and stays resident,
//    until the walk reaches a tile of another voice (multi-voice batches): then it is loaded again, see the kernel;
//  - a tile's input arrives by 1-D bulk copies, one per (channel, item segment) of the 16-byte-aligned superset of the
//    segment, into a ring of NSX fp32 staging slots of KCA channels.  The producer warp (lane c: channel c of the slot)
//    runs up to NSX slots ahead, across tiles, so the next tile's loads are in flight under this tile's MMAs and stores;
//  - the converter does LeakyReLU + split from the staging slot into the A ring (rows of items too short to be staged,
//    past the MAXSEG-th segment of a tile, it reads from global memory);
//  - the MMA warpgroups add the bias (registers, loaded once) and store, per channel, out[2s] (phase 1 of row s) and
//    out[2s + 1] (phase 0 of row s + 1, from the lane 4 up by shuffle) as one float2; meanwhile the converter already fills
//    the A ring with the next tile.
template <class Cfg>
struct StreamCfg {
    static_assert(Cfg::S == 2 && Cfg::NCG == 1 && Cfg::NMW == 2, "streaming ConvT: stride 2, one channel group");
    static constexpr int MAXSEG = 3;                          // staged item segments per tile: 3 when items have >= 64 positions
    static constexpr int AR = Cfg::ROWS + 1;                  // A rows of a tile (virtual rows r0 - 1 .. r0 + ROWS - 1)
    static constexpr int XPITCH = (AR + 6 * MAXSEG + 3) & ~3;  // floats per channel of a staging slot: each segment's
                                                               // aligned superset is at most 6 floats longer than it
    static constexpr int XSLOT = Cfg::KCA * XPITCH * 4;
    static constexpr int BRES = Cfg::NCHUNK * Cfg::BSLOT;     // resident B
    static constexpr int NSA = 2;
    static constexpr int FIXED = BRES + NSA * Cfg::ASLOT + 256;  // (+ the mbarriers)
    static constexpr int NSX = (227 * 1024 - 1024 - FIXED) / XSLOT < 4 ? (227 * 1024 - 1024 - FIXED) / XSLOT : 4;
    static constexpr int NT = Cfg::NCONV + 128 * Cfg::NMW + 32;
    static constexpr int SMEM_BYTES = BRES + NSA * Cfg::ASLOT + NSX * XSLOT + (2 + 2 * NSA + 2 * NSX) * 8;
    static_assert(NSX >= 2 && SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
    static_assert(XPITCH % 4 == 0 && Cfg::KCA == 32, "staging slot: 16-byte channel rows, one channel per producer lane");
};

// A rows [i0, i0 + n) of a tile are input positions [u0, u0 + n) of `item`, staged from float dst (+ the channel's
// alignment offset) of each channel's staging row
struct XSeg {
    int i0, n, item, u0, dst;
};
// The staged segments of the tile at virtual row r0 (A row i = virtual row r0 - 1 + i); producer and converter both call
// it.  Rows below `covered` outside every segment are zero rows (row -1, an item's zero row, a gap row before the first
// tile of a voice); rows from `covered` on (with items shorter than 64 positions, or a gap at the tile's end) are not
// staged.
template <class SC>
__device__ __forceinline__ void tile_segments(const RunTable &rows, int r0, XSeg (&seg)[SC::MAXSEG], int &covered) {
    int i = r0 == 0 ? 1 : 0, dst = 0;
#pragma unroll
    for (int k = 0; k < SC::MAXSEG; ++k) {
        RunPos p = rows.find(r0 - 1 + i);
        // skip an item's zero row, or the gap row before r0 (r0 itself always belongs to an item: see set_units)
        if (i < SC::AR && (p.item >= 0 ? p.unit == p.len : i == 0)) p = rows.find(r0 - 1 + ++i);
        const int n = (i < SC::AR && p.item >= 0) ? min(p.len - p.unit, SC::AR - i) : 0;
        seg[k] = {i, n, p.item, p.unit, dst};
        dst += (n + 6) & ~3;
        i += n;
    }
    covered = i;
}

// D[s, phi*NG + co] + bias -> out[co][2s - 1 + phi] for the two accumulator rows of this thread (stride 2, pad 1).  Row s
// with s < len owns the pair out[2s], out[2s + 1] = (its phase 1, row s + 1's phase 0); the last row of each warp (its
// successor is in the next warp) stores only out[2s], the first row of each warp also its own out[2s - 1].
template <class Cfg>
__device__ __forceinline__ void convt_stream_store(const float *acc, const float (&bj)[Cfg::NG / 8][2], float *__restrict__ y, int mw,
                                                   int t, int r0, const RunTable &rows) {
    constexpr int KB = Cfg::NG / 8, COUT = Cfg::COUT;
    const int lane = t & 31, q = t & 3, g = lane >> 2;
    const int Lout = 2 * rows.stride;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        int m = 64 * mw + frag_row(t, h);
        asm volatile("" : "+r"(m) : : "memory");  // one row's lookup at a time (see convt_store)
        const RunPos p = rows.find(r0 + m);
        const int s = p.unit;
        const bool pair_ok = p.item >= 0 && s < p.len, lo_ok = p.item >= 0 && s >= 1;
        float *yb = y + (size_t)(p.item >= 0 ? p.item : 0) * COUT * Lout + 2 * s;
#pragma unroll
        for (int k = 0; k < KB; ++k)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int co = 8 * k + 2 * q + e;
                const float p0 = acc[4 * k + 2 * h + e] + bj[k][e];         // phase 0: out[2s - 1]
                const float p1 = acc[4 * (KB + k) + 2 * h + e] + bj[k][e];  // phase 1: out[2s]
                // phase 0 of row m + 1: lane + 4, same h; for h = 0 and g = 7 it is lane - 28's h = 1 row
                const float nx = h == 0 ? __shfl_sync(0xffffffffu, g == 0 ? acc[4 * k + 2 + e] + bj[k][e] : p0, (lane + 4) & 31)
                                        : __shfl_down_sync(0xffffffffu, p0, 4);
                float *yp = yb + (size_t)co * Lout;
                if (h == 1 && g == 7) {
                    if (pair_ok) yp[0] = p1;
                } else if (pair_ok) {
                    *reinterpret_cast<float2 *>(yp) = make_float2(p1, nx);
                }
                if (h == 0 && g == 0 && lo_ok) yp[-1] = p0;
            }
    }
}

template <class Cfg>
__global__ void __launch_bounds__(StreamCfg<Cfg>::NT, 1)
convt_stream_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const __grid_constant__ RunTable rows, int ntiles,
                       int *__restrict__ status) {
    using SC = StreamCfg<Cfg>;
    constexpr int CIN = Cfg::CIN, N = Cfg::N, NG = Cfg::NG, KCA = Cfg::KCA, NCONV = Cfg::NCONV, NMW = Cfg::NMW;
    constexpr int ROWS = Cfg::ROWS, APITCH = Cfg::APITCH, ASLOT = Cfg::ASLOT, BSLOT = Cfg::BSLOT, NCHUNK = Cfg::NCHUNK;
    constexpr int AR = SC::AR, XPITCH = SC::XPITCH, XSLOT = SC::XSLOT, NSA = SC::NSA, NSX = SC::NSX, MAXSEG = SC::MAXSEG;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *bres = smem, *aring = smem + SC::BRES, *xring = aring + NSA * ASLOT;
    uint64_t *fullW = reinterpret_cast<uint64_t *>(xring + NSX * XSLOT), *emptyW = fullW + 1;
    uint64_t *fullA = emptyW + 1, *emptyA = fullA + NSA, *fullX = emptyA + NSA, *emptyX = fullX + NSX;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int Lin = rows.stride;  // input positions between items
    // Resident B per voice.  set_units keeps every tile within one voice, so tile r0's weights are rows.blob_at(r0).  Load
    // k of B (k = 0, 1, ...: one per voice change along this CTA's walk, the first before the first tile) completes phase k
    // of fullW; the MMA warpgroups wait for it (parity k & 1) before the first MMA of a tile of that voice.  B is
    // overwritten only by the producer's lane 0, and only after emptyW has completed phase k - 1: each MMA warpgroup's
    // thread 0 arrives there after wgmma_wait<0> of the last tile before the voice change, so every MMA that read the
    // old B has completed.  The producer has issued the staging loads of every earlier tile by then, so the wait cannot
    // close a cycle; it only holds back the new voice's staging loads until the old voice's MMAs are done.
    auto voice = [&](int tile) { return rows.blob_at(tile * ROWS); };
    auto load_b = [&](const float *vb) {
        const uint8_t *src = reinterpret_cast<const uint8_t *>(vb) + tc_region_start() + tc_up_offset(Cfg::STAGE);
        mbar_arrive_expect_tx(fullW, SC::BRES);
        for (int i = 0; i < NCHUNK; ++i) bulk_g2s(bres + i * BSLOT, src + (size_t)i * BSLOT, BSLOT, fullW);
    };

    if (tid == 0) {
        mbar_init(fullW, 1);
        mbar_init(emptyW, NMW);
        for (int s = 0; s < NSA; ++s) { mbar_init(&fullA[s], NCONV); mbar_init(&emptyA[s], NMW); }
        for (int s = 0; s < NSX; ++s) { mbar_init(&fullX[s], 1); mbar_init(&emptyX[s], NCONV); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == (NCONV + 128 * NMW) / 32) {
        // ================= producer warp: resident B (lane 0), then the input tiles (lane c: channel c of a slot) =========
        const float *wb = voice(blockIdx.x);  // the voice whose B is resident (or on its way)
        int nw = 0;                           // loads of B so far, minus one
        if (lane == 0) load_b(wb);
        pdl_wait();  // x: the previous kernel's output
        int sx = 0, phx = 0;
        bool ok = true;
#pragma unroll 1
        for (int tile = blockIdx.x; tile < ntiles && ok; tile += gridDim.x) {
            const int r0 = tile * ROWS;
            if (voice(tile) != wb) {
                wb = voice(tile);
                ok = __shfl_sync(0xffffffffu, lane == 0 ? mbar_wait(emptyW, nw & 1) : false, 0);
                if (!ok) break;
                if (lane == 0) load_b(wb);
                ++nw;
                __syncwarp();
            }
            XSeg seg[MAXSEG];
            int covered;
            tile_segments<SC>(rows, r0, seg, covered);
#pragma unroll 1
            for (int ca = 0; ca < CIN / KCA; ++ca) {
                ok = __shfl_sync(0xffffffffu, lane == 0 ? mbar_wait(&emptyX[sx], phx ^ 1) : false, 0);
                if (!ok) break;
                float *slot = reinterpret_cast<float *>(xring + sx * XSLOT) + lane * XPITCH;
                size_t g0[MAXSEG];
                uint32_t bytes = 0;
#pragma unroll
                for (int k = 0; k < MAXSEG; ++k) {
                    g0[k] = ((size_t)seg[k].item * CIN + ca * KCA + lane) * Lin + seg[k].u0;
                    if (seg[k].n > 0) bytes += (uint32_t)((((g0[k] + seg[k].n + 3) & ~(size_t)3) - (g0[k] & ~(size_t)3)) * 4);
                }
                const uint32_t total = __reduce_add_sync(0xffffffffu, bytes);
                if (lane == 0) mbar_arrive_expect_tx(&fullX[sx], total);
                __syncwarp();
#pragma unroll
                for (int k = 0; k < MAXSEG; ++k)
                    if (seg[k].n > 0) {
                        const size_t a = g0[k] & ~(size_t)3, e = (g0[k] + seg[k].n + 3) & ~(size_t)3;
                        bulk_g2s(slot + seg[k].dst, x + a, (uint32_t)((e - a) * 4), &fullX[sx]);
                    }
                if (++sx == NSX) { sx = 0; phx ^= 1; }
            }
        }
        if (!ok && lane == 0) atomicExch(status, 12);
    } else if (warp >= NCONV / 32) {
        // ================= MMA warpgroup mw: rows [64 mw, 64 mw + 64) of every tile =================
        const int mw = warp / 4 - NCONV / 128, t = tid & 127;
        const uint64_t adesc_t = desc_template(APITCH, 128), bdesc_t = desc_template(N * 16, 128);
        const uint32_t aring_addr = smem_u32(aring) + mw * 64 * 16, bres_addr = smem_u32(bres);
        float bj[NG / 8][2];  // bias of this thread's channels 8k + 2q + e, of the resident voice
        auto load_bias = [&](const float *vb) {
#pragma unroll
            for (int k = 0; k < NG / 8; ++k)
#pragma unroll
                for (int e = 0; e < 2; ++e) bj[k][e] = __ldg(vb + bias_offset(1 + Cfg::STAGE) + 8 * k + 2 * (t & 3) + e);
        };
        const float *wb = voice(blockIdx.x);
        int nw = 0;
        load_bias(wb);
        float acc[N / 2];
        int sa = 0, pha = 0;
        bool ok = mbar_wait(fullW, 0);  // a timed-out wait only raises the status word: control flow stays uniform
#pragma unroll 1
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            if (voice(tile) != wb) {  // B of this voice: load nw + 1
                wb = voice(tile);
                ++nw;
                load_bias(wb);
                ok &= mbar_wait(fullW, nw & 1);
            }
            int psa = -1;
#pragma unroll 1
            for (int ca = 0; ca < CIN / KCA; ++ca) {
                ok &= mbar_wait(&fullA[sa], pha);
                const uint64_t abase = desc_at(adesc_t, aring_addr + sa * ASLOT);
#pragma unroll 1
                for (int j = 0; j < KCA / 16; ++j) {
                    const uint64_t bbase = desc_at(bdesc_t, bres_addr + (ca * (KCA / 16) + j) * BSLOT);
                    wgmma_fence();
#pragma unroll
                    for (int tap = 0; tap < 2; ++tap)
#pragma unroll
                        for (int pass = 0; pass < 3; ++pass) {
                            const int ahalf = (pass == 1), bhalf = (pass == 2);
                            const uint64_t bdesc = bbase + (uint64_t)((((tap * 2 + bhalf) * 2) * N * 16) >> 4);
                            const uint64_t adesc = abase + (uint64_t)((ahalf * (KCA / 8) * APITCH + (1 - tap) * 16) >> 4) +
                                                   (uint64_t)(2 * j * (APITCH >> 4));
                            wgmma_bf16<N>(acc, adesc, bdesc, (ca | j | tap | pass) != 0);
                        }
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (t == 0 && psa >= 0) mbar_arrive(&emptyA[psa]);
                    psa = (j == KCA / 16 - 1) ? sa : -1;
                }
                if (++sa == NSA) { sa = 0; pha ^= 1; }
            }
            wgmma_wait<0>();
            acc_fence<N / 2>(acc);
            if (t == 0) mbar_arrive(&emptyA[psa]);
            const int next = tile + (int)gridDim.x;
            if (t == 0 && next < ntiles && voice(next) != wb) mbar_arrive(emptyW);  // every MMA on this B has completed
            if (next >= ntiles) pdl_trigger();  // last tile's MMAs done: the next kernel may be scheduled
            pdl_wait();
            convt_stream_store<Cfg>(acc, bj, y, mw, t, tile * ROWS, rows);
        }
        if (!ok && t == 0) atomicExch(status, 13);
    } else {
        // ================= converter warps: A slots = split(lrelu(x)) from the staging slots =================
        pdl_wait();  // (rows that are not staged are read from x)
        int sx = 0, phx = 0, sa = 0, pha = 0;
        bool ok = true;
#pragma unroll 1
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            const int r0 = tile * ROWS;
            XSeg seg[MAXSEG];
            int covered;
            tile_segments<SC>(rows, r0, seg, covered);
#pragma unroll 1
            for (int ca = 0; ca < CIN / KCA; ++ca) {
                if (ok && !(mbar_wait(&fullX[sx], phx) && mbar_wait(&emptyA[sa], pha ^ 1))) {
                    ok = false;
                    atomicExch(status, 14);
                }
                const float *xs = reinterpret_cast<const float *>(xring + sx * XSLOT);
                uint8_t *slot = aring + sa * ASLOT;
#pragma unroll 1
                for (int u = tid; u < AR * (KCA / 8); u += NCONV) {
                    const int i = u % AR, kp = u / AR;
                    int off = -1;
                    uint32_t gb = 0;  // low bits of the global float index of channel 8 kp's row: the staging alignment
#pragma unroll
                    for (int k = 0; k < MAXSEG; ++k)
                        if (i >= seg[k].i0 && i < seg[k].i0 + seg[k].n) {
                            off = seg[k].dst + i - seg[k].i0;
                            gb = ((uint32_t)seg[k].item * CIN + ca * KCA + 8 * kp) * (uint32_t)Lin + seg[k].u0;
                        }
                    float f[8];
                    if (off >= 0) {
#pragma unroll
                        for (int e = 0; e < 8; ++e) f[e] = xs[(8 * kp + e) * XPITCH + off + ((gb + e * Lin) & 3)];
                    } else {
                        const RunPos p = i >= covered ? rows.find(r0 - 1 + i) : RunPos{-1, 0, 0};
                        const bool inr = p.item >= 0 && p.unit < p.len;
                        const float *xp = x + ((size_t)(inr ? p.item : 0) * CIN + ca * KCA + 8 * kp) * Lin + (inr ? p.unit : 0);
#pragma unroll
                        for (int e = 0; e < 8; ++e) f[e] = inr ? __ldg(xp + (size_t)e * Lin) : 0.f;
                    }
                    uint32_t h[4], l[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) split2_bf16(lrelu(f[2 * e]), lrelu(f[2 * e + 1]), h[e], l[e]);
                    *reinterpret_cast<uint4 *>(slot + kp * APITCH + i * 16) = make_uint4(h[0], h[1], h[2], h[3]);
                    *reinterpret_cast<uint4 *>(slot + (KCA / 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
                }
                fence_proxy_async();
                mbar_arrive(&fullA[sa]);
                mbar_arrive(&emptyX[sx]);
                if (++sa == NSA) { sa = 0; pha ^= 1; }
                if (++sx == NSX) { sx = 0; phx ^= 1; }
            }
        }
    }
}

template <class Cfg>
static int launch_convt_stream(const float *x, float *y, const RunTable &batch, int *status, cudaStream_t s) {
    using SC = StreamCfg<Cfg>;
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(convt_stream_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, SC::SMEM_BYTES));
        configured = true;
    }
    if (reinterpret_cast<uintptr_t>(x) % 16 != 0)  // the bulk copies read 16-byte-aligned supersets of x's rows
        return set_error(MG_ERR_INVALID_ARGUMENT, "launch_convt_tc: stage %d input not 16-byte aligned", Cfg::STAGE);
    int dev = 0, sms = 0;
    MG_CUDA_TRY(cudaGetDevice(&dev));
    MG_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const RunTable rows = convt_rows(batch, Cfg::ROWS);
    const int ntiles = (rows.first[rows.n] + Cfg::ROWS - 1) / Cfg::ROWS;
    const unsigned grid = (unsigned)(ntiles < sms ? ntiles : sms);
    MG_CUDA_TRY(launch_ex(convt_stream_tc_kernel<Cfg>, dim3(grid), dim3(SC::NT), SC::SMEM_BYTES, s, true, 1, x, y, rows, ntiles, status));
    return MG_OK;
}

// the tile geometry of the streaming stride-2 ConvT (stage 2 or 3): rows per tile, staged item segments per tile, staging
// slots; its grid is min(tiles, SMs)
template <class Cfg>
static const char *stream_cfg_name() {
    static char buf[80];
    snprintf(buf, sizeof(buf), "convt_stream_tc_kernel<StreamCfg<%d,%d,%d,%d>>", Cfg::STAGE, Cfg::ROWS, StreamCfg<Cfg>::MAXSEG,
             StreamCfg<Cfg>::NSX);
    return buf;
}

// ---------------------------------------------------------------------------------------------------------------------
// Variant for a stage whose whole activation tile fits in shared memory (stage 1: 65 rows x 256 channels, hi+lo =
// 72 KB): the A operand is converted ONCE per row tile and stays resident, and the CTA loops over the NCG output-channel
// groups, so no activation is loaded or converted twice.  One MMA warpgroup (64 rows, N = 256) per CTA.  The converter
// also parks the tile's 64 row lookups in shared memory for the epilogue, which runs once per channel group.
template <class Cfg>
__global__ void __launch_bounds__(Cfg::NCONV + 128 + 32, 1)
convt_resident_tc_kernel(const float *__restrict__ x, float *__restrict__ y, const __grid_constant__ RunTable rows,
                         int *__restrict__ status) {
    constexpr int CIN = Cfg::CIN, NG = Cfg::NG, N = Cfg::N, NCG = Cfg::NCG;
    constexpr int ROWS = 64, APITCH = Cfg::APITCH, BSLOT = Cfg::BSLOT, NCHUNK = Cfg::NCHUNK;
    constexpr int KPT = CIN / 8;                    // k-panels of the resident A
    constexpr int AHALF = KPT * APITCH;             // bytes of one of {hi, lo}
    constexpr int NSB = 4, NCONV = Cfg::NCONV;
    constexpr int NPASS = Cfg::ONEPASS ? 1 : 3;  // (xh, wh), (xl, wh), (xh, wl), or the first alone
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
            const uint8_t *src = reinterpret_cast<const uint8_t *>(tile_blob(rows, r0)) + tc_region_start() + tc_up_offset(Cfg::STAGE);
            int s = 0, ph = 0;
            bool ok = true;
            for (int i = 0; i < NCG * NCHUNK && ok; ++i) {  // blob order is [cg][chunk]: exactly this loop
                if (!mbar_wait(&emptyB[s], ph ^ 1)) { ok = false; break; }
                load_bslot<Cfg>(bring + s * BSLOT, src + (size_t)i * BSLOT, &fullB[s]);
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
                    for (int pass = 0; pass < NPASS; ++pass) {
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
            convt_store<Cfg>(acc, y, tile_blob(rows, r0) + bias_offset(1 + Cfg::STAGE) + cg * NG, 0, t, cg, Cfg::S * Lin,
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
                    if constexpr (!Cfg::ONEPASS)
                        *reinterpret_cast<uint4 *>(abuf + AHALF + (ca * 8 + kp) * APITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
                }
            }
            fence_proxy_async();
            mbar_arrive(&fullA[ca]);
        }
    }
}

template <class Cfg>
static int launch_convt_resident(const float *x, float *y, const RunTable &batch, int *status, cudaStream_t s) {
    constexpr int smem = 2 * (Cfg::CIN / 8) * Cfg::APITCH + 4 * Cfg::BSLOT + (Cfg::CIN / 64 + 2 * 4) * 8 + 64 * sizeof(RunPos);
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(convt_resident_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    const RunTable rows = convt_rows(batch, 64);
    MG_CUDA_TRY(launch_ex(convt_resident_tc_kernel<Cfg>, dim3((unsigned)((rows.first[rows.n] + 63) / 64)), dim3(Cfg::NCONV + 128 + 32),
                          smem, s, true, 1, x, y, rows, status));
    return MG_OK;
}

// x [B][Cin][Lin] -> y [B][Cout][S*Lin], fp32 NCL, (Cin, Cout, S) of generator stage `stage`; Lin = batch.stride, item i's
// first len_i input positions (and S len_i output positions) are its own.  precision MG_GEN_PRECISION_BF16: stages 0 and 1
// run their single-pass variants; stages 2 and 3 keep the streaming kernel's three passes (it is bound by memory).
int launch_convt_tc(const float *x, float *y, int stage, const RunTable &batch, int *status, cudaStream_t s, int precision) {
    if (precision != MG_GEN_PRECISION_FP32 && precision != MG_GEN_PRECISION_BF16)
        return set_error(MG_ERR_INVALID_ARGUMENT, "launch_convt_tc: precision %d", precision);
    if (precision == MG_GEN_PRECISION_BF16 && stage == 0) return launch_convt<Bf16<UpCfg<0>>>(x, y, batch, status, s);
    if (precision == MG_GEN_PRECISION_BF16 && stage == 1) return launch_convt_resident<Bf16<UpCfg<1>>>(x, y, batch, status, s);
    switch (stage) {
        case 0: return launch_convt<UpCfg<0>>(x, y, batch, status, s);
        case 1: return launch_convt_resident<UpCfg<1>>(x, y, batch, status, s);
        case 2: return launch_convt_stream<UpCfg<2>>(x, y, batch, status, s);
        case 3: return launch_convt_stream<UpCfg<3>>(x, y, batch, status, s);
    }
    return set_error(MG_ERR_INVALID_ARGUMENT, "launch_convt_tc: stage %d", stage);
}

// the tile geometry of a stride-8 ConvT: ROWS input positions per CTA (the batch's items concatenated with one zero row
// after each), NG output channels per CTA (grid.y = COUT / NG for convt_tc_kernel; the resident kernel loops over them)
template <class Cfg>
static const char *up_cfg_name(const char *kernel) {
    static char buf[80];
    snprintf(buf, sizeof(buf), "%s<UpCfg<%d,%d,%d>>", kernel, Cfg::STAGE, Cfg::ROWS, Cfg::NG);
    return buf;
}

// the configuration launch_convt_tc runs for `stage` ("" for an unknown stage)
const char *convt_config_name(int stage) {
    switch (stage) {
        case 0: return up_cfg_name<UpCfg<0>>("convt_tc_kernel");
        case 1: return up_cfg_name<UpCfg<1>>("convt_resident_tc_kernel");
        case 2: return stream_cfg_name<UpCfg<2>>();
        case 3: return stream_cfg_name<UpCfg<3>>();
    }
    return "";
}

}  // namespace mg
