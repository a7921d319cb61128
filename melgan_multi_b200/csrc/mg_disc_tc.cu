// Discriminator grouped convs on the tensor cores: Conv1d(k41, stride 4, pad 20, 4 input / 16 output channels per group)
// + LeakyReLU, layers 1..3 of models.py:78-81,89-95 (groups 4 / 16 / 64), wgmma, split-bf16.
//
// Toeplitz view.  Tap k = 4q + r of output t reads input position 4(t + q - 5) + r, so with the input of one group
// de-interleaved by phase r into channels-last rows  U_r[u][ci] = x[ci][4u + r]  (8 B per u in bf16), one output is
//     out[co][t] = sum_r sum_q sum_ci  U_r[t + q - 5][ci] * w[co][ci][4q + r].
// A 16-byte unit of U_r holds two consecutive u (x 4 ci) = one 8-element k-panel, and rows of a wgmma operand are
// 16 B = 2 u apart, so accumulator row m of a tile is the output PAIR t = t0 + 2m + e (e = 0, 1) and both parities read the
// same A rows:  unit (m + kp) of U_r  x  weights of q = 2 kp + pos - 1 - e  (7 panels cover q = -2..11, zeros outside
// 0..10; mg_layout.h d_gtc_index).  One K = 16 instruction contracts panel kp of phases r and r + 1 (LBO = the pitch
// between phase buffers), with N = 64 columns = [w hi | w lo] x parity x 16 co:
//     pass 0:  A = hi(U),  B = [w hi | w lo]  (N = 64)        pass 1:  A = lo(U),  B = w hi  (N = 32, same columns)
// = 28 instructions per (group, 256 outputs); the epilogue adds the hi and lo column blocks (fp32-grade: ~4e-6).
// CTA = 2 groups x 256 outputs of one batch item, 93 KB of shared memory -> two CTAs per SM overlap each other's
// load / convert, MMA and epilogue phases.  Weights (28 KB per group, contiguous in the packed blob) arrive by bulk TMA.
// The two converter warpgroups then run the MMAs of rows 0..63 / 64..127 and the epilogue from their accumulator registers.
#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {
using namespace tc;

namespace dg {
constexpr int NGRP = 2;                       // groups per CTA
constexpr int TILE = 256;                     // outputs per CTA (128 accumulator rows x 2 parities)
constexpr int UNITS = 128 + kDgPanels - 1;    // 16-byte units per phase buffer
constexpr int XP = UNITS * 16;                // phase-buffer pitch: 536 words = 24 (mod 32) -> conflict-free 8-byte stores
constexpr int NPOS = UNITS * 8;               // input positions per channel per tile
constexpr int WBYTES = 28672;                 // d_gtc_group_bytes()
constexpr int XBYTES = NGRP * 2 * 4 * XP;     // [group][half][phase r][unit][pos 2][ci 4] bf16
constexpr int NCONV = 256, NT = NCONV + 32;
constexpr int SMEM_BYTES = NGRP * WBYTES + XBYTES + 8;
static_assert(WBYTES == (int)d_gtc_group_bytes(), "weight block");
}  // namespace dg

__global__ void __launch_bounds__(dg::NT, 2)
disc_group_tc_kernel(const float *__restrict__ x, float *__restrict__ out, const uint8_t *__restrict__ wtc,
                     const float *__restrict__ bias, int Bt, int Cin, int Cout, int Lin, int Lout, int rp, int ni,
                     int *__restrict__ status) {
    using namespace dg;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *wsm = smem, *xsm = smem + NGRP * WBYTES;
    uint64_t *wbar = reinterpret_cast<uint64_t *>(xsm + XBYTES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // rows are VIRTUAL when the sequence is short: ni items share the tile at a pitch of rp rows / units (an item's
    // ceil(Lout/2) output pairs + 6 halo units); ni == 1 (rp = 2^30): blockIdx.x walks the 256-output tiles of one item
    const int t0 = blockIdx.x * TILE, g0 = blockIdx.y * NGRP, b0 = blockIdx.z * ni;

    if (tid == 0) {
        mbar_init(wbar, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCONV / 32) {
        if (lane == 0) {
            mbar_arrive_expect_tx(wbar, NGRP * WBYTES);
            bulk_g2s(wsm, wtc + (size_t)g0 * WBYTES, NGRP * WBYTES, wbar);
        }
    } else {
        // U_r[u][ci] of both groups, hi / lo split: item = (group, offset pp from the first position 4 (t0 - 6))
        const int p0 = 4 * (t0 - 6);
        // (three items per trip: 12 independent loads in flight per thread)
#pragma unroll 1
        for (int i0 = tid; i0 < NGRP * NPOS; i0 += 3 * NCONV) {
            float f[3][4];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int i = i0 + k * NCONV, g = i >= NPOS, pp = i - g * NPOS;
                const int j = (pp >> 3) / rp, p = p0 + pp - 8 * j * rp, b = b0 + j;  // a unit = 8 consecutive positions
                const bool in = i < NGRP * NPOS && b < Bt && p >= 0 && p < Lin;
                const float *xp = x + ((size_t)(in ? b : 0) * Cin + (g0 + g) * 4) * Lin + (in ? p : 0);
#pragma unroll
                for (int ci = 0; ci < 4; ++ci) f[k][ci] = in ? __ldg(xp + (size_t)ci * Lin) : 0.f;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int i = i0 + k * NCONV, g = i >= NPOS, pp = i - g * NPOS;
                if (i < NGRP * NPOS) {
                    uint32_t h0, h1, l0, l1;
                    split2_bf16(f[k][0], f[k][1], h0, l0);
                    split2_bf16(f[k][2], f[k][3], h1, l1);
                    uint8_t *dst = xsm + ((g * 2) * 4 + (pp & 3)) * XP + (pp >> 2) * 8;
                    *reinterpret_cast<uint2 *>(dst) = make_uint2(h0, h1);
                    *reinterpret_cast<uint2 *>(dst + 4 * XP) = make_uint2(l0, l1);
                }
            }
        }
        fence_proxy_async();
    }
    __syncthreads();

    if (warp < NCONV / 32) {
        // ================= MMA: warpgroup mw owns accumulator rows [64 mw, 64 mw + 64), both groups =================
        const int mw = warp >> 2, t = tid & 127;
        bool ok = mbar_wait(wbar, 0);
        const uint64_t adesc_t = desc_template(XP, 128), bdesc_t = desc_template(64 * 16, 128);
        const uint32_t x_addr = smem_u32(xsm) + mw * 64 * 16, w_addr = smem_u32(wsm);
        float acc[NGRP][32];
        wgmma_fence();
#pragma unroll
        for (int g = 0; g < NGRP; ++g) {
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                const uint64_t a0 = desc_at(adesc_t, x_addr + (g * 2 + pass) * 4 * XP);
                const uint64_t b0 = desc_at(bdesc_t, w_addr + g * WBYTES);
#pragma unroll
                for (int kp = 0; kp < kDgPanels; ++kp) {
#pragma unroll
                    for (int rq = 0; rq < 2; ++rq) {  // phase pair (r = 2 rq, 2 rq + 1)
                        const uint64_t adesc = a0 + (uint64_t)((2 * rq * XP + 16 * kp) >> 4);
                        const uint64_t bdesc = b0 + (uint64_t)(((kp * 2 + rq) * 2048) >> 4);
                        if (pass) wgmma_bf16<32>(acc[g], adesc, bdesc, 1);
                        else wgmma_bf16<64>(acc[g], adesc, bdesc, (kp | rq) != 0);
                    }
                }
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence<32>(acc[0]);
        acc_fence<32>(acc[1]);
        if (!ok && t == 0) atomicExch(status, 31);
        // ================= epilogue: row m <-> outputs t0 + 2m, t0 + 2m + 1 =================
        // column 8k + 2q + e = [hi | lo] (k / 4) x parity ((k / 2) % 2) x co 8 (k % 2) + 2q + e
        const bool pair = (Lout & 1) == 0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = 64 * mw + frag_row(t, h), jm = m / rp, b = b0 + jm;
            const int tt = (jm < ni && b < Bt) ? t0 + 2 * (m - jm * rp) : Lout;  // rows of the inter-item gap store nothing
            if (tt >= Lout) continue;
#pragma unroll
            for (int g = 0; g < NGRP; ++g)
#pragma unroll
                for (int c8 = 0; c8 < 2; ++c8)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int co = (g0 + g) * 16 + 8 * c8 + 2 * (lane & 3) + e;
                        const float bv = __ldg(bias + co);
                        const int i0 = 2 * h + e;
                        const float v0 = lrelu(acc[g][4 * c8 + i0] + acc[g][4 * (4 + c8) + i0] + bv);
                        const float v1 = lrelu(acc[g][4 * (2 + c8) + i0] + acc[g][4 * (6 + c8) + i0] + bv);
                        float *o = out + ((size_t)b * Cout + co) * Lout + tt;
                        if (pair && tt + 1 < Lout) {
                            *reinterpret_cast<float2 *>(o) = make_float2(v0, v1);
                        } else {
                            o[0] = v0;
                            if (tt + 1 < Lout) o[1] = v1;
                        }
                    }
        }
    }
}

// x [Bt][Cin][Lin] -> out [Bt][Cout][Lout] = lrelu(grouped conv), layer l in 1..3;  wtc = blob + d_gtc_start() + d_gtc_offset(l)
int launch_disc_group_tc(const float *x, float *out, const uint8_t *wtc, const float *bias, int Bt, int Cin, int Cout,
                         int Lin, int Lout, int *status, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(disc_group_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dg::SMEM_BYTES));
        configured = true;
    }
    int rp = (Lout + 1) / 2 + kDgPanels - 1, ni = dg::UNITS / rp;
    if (ni <= 1) { ni = 1; rp = 1 << 30; }
    const int zb = (Bt + ni - 1) / ni;
    if (zb > 65535) return set_error(MG_ERR_INVALID_ARGUMENT, "discriminator batch %d exceeds the grid", Bt);
    dim3 grid(ni > 1 ? 1 : (Lout + dg::TILE - 1) / dg::TILE, (Cin / 4) / dg::NGRP, zb);
    disc_group_tc_kernel<<<grid, dg::NT, dg::SMEM_BYTES, s>>>(x, out, wtc, bias, Bt, Cin, Cout, Lin, Lout, rp, ni, status);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Layer 4: Conv1d(1024 -> 1024, k41, stride 1, pad 20, groups 256: 4 -> 4 channels per group) + LeakyReLU, models.py:82.
// With only 4 outputs per group the contraction is made dense along TIME instead: accumulator row m owns the 8 consecutive
// outputs t = 8 kb + e, the A operand of input channel ci is the plain bf16 signal cut into 16-byte units of 8 positions
// (unit u = positions 8u - 20 .. 8u - 13, so lane kb reads units kb .. kb + 5: 48 positions for 8 outputs x 41 taps),
// and B is the Toeplitz matrix  B[(e, co)][i of panel kp] = w[co][ci][8 kp + i - e]  (85 % dense; mg_layout.h).
// One K = 16 instruction contracts panel kp of channels ci and ci + 1 (LBO = pitch between the channel buffers):
// 12 instructions of N = 64 ([w hi | w lo] x 8 e x 4 co) for A = hi(x) + 12 of N = 32 for A = lo(x) per (group, 128 lanes).
// Lanes are VIRTUAL: with Lout = 128 / 65 / 17 (the three scales at 8192 samples) an item needs only nb = ceil(L/8)
// lanes, so a tile packs NI = floor(133 / (nb + 5)) batch items at a pitch of nb + 5 units (the 5 extra units are the
// item's right halo; the lanes in that gap compute garbage that is never stored).  Longer items take ceil(nb / 128)
// tiles of one item each.
namespace dg4 {
constexpr int NGRP = 2;
constexpr int UNITS = 128 + kDg4Panels - 1;   // 133 units of 8 positions per channel buffer
constexpr int XP = UNITS * 16;                // channel-buffer pitch
constexpr int WBYTES = 24576;                 // d_g4tc_group_bytes()
constexpr int XBYTES = NGRP * 2 * 4 * XP;     // [group][half][ci][unit][8 positions] bf16
constexpr int NCONV = 256, NT = NCONV + 32;
constexpr int SMEM_BYTES = NGRP * WBYTES + XBYTES + 8;
static_assert(WBYTES == (int)d_g4tc_group_bytes(), "weight block");
}  // namespace dg4

__global__ void __launch_bounds__(dg4::NT, 2)
disc_group4_tc_kernel(const float *__restrict__ x, float *__restrict__ out, const uint8_t *__restrict__ wtc,
                      const float *__restrict__ bias, int Bt, int C, int L, int nb, int rp, int ni, int segs,
                      int *__restrict__ status) {
    using namespace dg4;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *wsm = smem, *xsm = smem + NGRP * WBYTES;
    uint64_t *wbar = reinterpret_cast<uint64_t *>(xsm + XBYTES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int item0 = (blockIdx.x / segs) * ni, kb0 = (blockIdx.x % segs) * 128, g0 = blockIdx.y * NGRP;

    if (tid == 0) {
        mbar_init(wbar, 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCONV / 32) {
        if (lane == 0) {
            mbar_arrive_expect_tx(wbar, NGRP * WBYTES);
            bulk_g2s(wsm, wtc + (size_t)g0 * WBYTES, NGRP * WBYTES, wbar);
        }
    } else {
        // channel c of the CTA's 8 (= group, ci), virtual position vp = 8 * unit + i: consecutive threads read consecutive
        // positions of one channel and write consecutive bf16 of its buffer
        // (the 8 channel loads of one position are independent: all in flight together, index math paid once)
#pragma unroll 1
        for (int vp = tid; vp < UNITS * 8; vp += NCONV) {
            const int ui = vp >> 3, j = ui / rp, item = item0 + j;
            const int p = 8 * (kb0 + ui - j * rp) - 20 + (vp & 7);
            const bool in = item < Bt && p >= 0 && p < L;
            const float *xp = x + ((size_t)(in ? item : 0) * C + g0 * 4) * L + (in ? p : 0);
            float v[NGRP * 4];
#pragma unroll
            for (int c = 0; c < NGRP * 4; ++c) v[c] = in ? __ldg(xp + (size_t)c * L) : 0.f;
#pragma unroll
            for (int c = 0; c < NGRP * 4; ++c) {
                uint8_t *dst = xsm + (((c >> 2) * 2) * 4 + (c & 3)) * XP + vp * 2;
                __nv_bfloat16 hi, lo;
                split_bf16(v[c], hi, lo);
                *reinterpret_cast<__nv_bfloat16 *>(dst) = hi;
                *reinterpret_cast<__nv_bfloat16 *>(dst + 4 * XP) = lo;
            }
        }
        fence_proxy_async();
    }
    __syncthreads();

    if (warp < NCONV / 32) {
        // ================= MMA: warpgroup mw owns accumulator rows [64 mw, 64 mw + 64), both groups =================
        const int mw = warp >> 2, t = tid & 127;
        bool ok = mbar_wait(wbar, 0);
        const uint64_t adesc_t = desc_template(XP, 128), bdesc_t = desc_template(64 * 16, 128);
        const uint32_t x_addr = smem_u32(xsm) + mw * 64 * 16, w_addr = smem_u32(wsm);
        float acc[NGRP][32];
        wgmma_fence();
#pragma unroll
        for (int g = 0; g < NGRP; ++g) {
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                const uint64_t a0 = desc_at(adesc_t, x_addr + (g * 2 + pass) * 4 * XP);
                const uint64_t b0 = desc_at(bdesc_t, w_addr + g * WBYTES);
#pragma unroll
                for (int kp = 0; kp < kDg4Panels; ++kp) {
#pragma unroll
                    for (int cp = 0; cp < 2; ++cp) {
                        const uint64_t adesc = a0 + (uint64_t)((2 * cp * XP + 16 * kp) >> 4);
                        const uint64_t bdesc = b0 + (uint64_t)(((kp * 2 + cp) * 2048) >> 4);
                        if (pass) wgmma_bf16<32>(acc[g], adesc, bdesc, 1);
                        else wgmma_bf16<64>(acc[g], adesc, bdesc, (kp | cp) != 0);
                    }
                }
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence<32>(acc[0]);
        acc_fence<32>(acc[1]);
        if (!ok && t == 0) atomicExch(status, 33);
        // ================= epilogue: row m <-> the 8 outputs t = 8 kb + e =================
        // column 8k + 2q + e' = [hi | lo] (k / 4) x e (2 (k % 4) + q / 2) x co (2 (q % 2) + e'): this thread holds the
        // outputs e = 2 kk + q / 2 (kk = 0..3) of channels co = 2 (q % 2) + e'
        const int q = lane & 3;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = 64 * mw + frag_row(t, h), j = m / rp, item = item0 + j, kb = kb0 + m - j * rp;
            if (!(item < Bt && j < ni && kb < nb)) continue;
#pragma unroll
            for (int g = 0; g < NGRP; ++g)
#pragma unroll
                for (int ep = 0; ep < 2; ++ep) {
                    const int co = (g0 + g) * 4 + 2 * (q & 1) + ep;
                    const float bv = __ldg(bias + co);
                    float *o = out + ((size_t)item * C + co) * L + 8 * kb + (q >> 1);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const int i0 = 4 * kk + 2 * h + ep;
                        if (8 * kb + 2 * kk + (q >> 1) < L) o[2 * kk] = lrelu(acc[g][i0] + acc[g][16 + i0] + bv);
                    }
                }
        }
    }
}

// x [Bt][1024][L] -> out [Bt][1024][L] = lrelu(grouped conv, layer 4);  wtc = blob + d_g4tc_start()
int launch_disc_group4_tc(const float *x, float *out, const uint8_t *wtc, const float *bias, int Bt, int L, int *status,
                          cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(disc_group4_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dg4::SMEM_BYTES));
        configured = true;
    }
    const int C = d_layer(4).cin, nb = (L + 7) / 8;
    int rp = nb + dg4::UNITS - 128, ni = dg4::UNITS / rp, segs = 1;
    if (ni < 1) { ni = 1; segs = (nb + 127) / 128; rp = 1 << 30; }
    const long long tiles = (long long)((Bt + ni - 1) / ni) * segs;
    if (tiles > 0x7fffffffll) return set_error(MG_ERR_INVALID_ARGUMENT, "discriminator layer 4: %lld tiles", tiles);
    dim3 grid((unsigned)tiles, (C / 4) / dg4::NGRP);
    disc_group4_tc_kernel<<<grid, dg4::NT, dg4::SMEM_BYTES, s>>>(x, out, wtc, bias, Bt, C, L, nb, rp, ni, segs, status);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

}  // namespace mg
