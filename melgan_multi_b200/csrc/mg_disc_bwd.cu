// Backward of the discriminators' grouped convs (layers 1..4 of models.py:78-82: k41, pad 20, 4 input channels per group,
// stride 4/4/4/1) and of weight-norm for all 21 discriminator layers.  cuDNN runs a grouped conv's backward as one small
// kernel per group (thousands of launches per step at BASELINE config 3); here each
// gradient is one launch.  fp32 SIMT: the FLOPs are small (1.4 GF per layer), the dense layers' backward stays on
// cuDNN (aten::convolution_backward) for now.
//
//   dz [Bt][Cout][Lout]  = upstream gradient already multiplied by LeakyReLU'(output)
//   dx [Bt][Cin][Lin]    = sum_co sum_{k: 4t + k - 20 = p} dz[co][t] w[co][ci][k]            (grouped_dx_kernel)
//   dw [Cout][4][41]     = sum_b sum_t dz[co][t] x[ci][S t + k - 20],  db[co] = sum dz       (grouped_dw_kernel + combine)
#include "mg_common.cuh"

namespace mg {

// ------------------------------------------------------------------------------------------------------------------
// dx.  CTA = (tile of 256 input positions, group, item); thread = 2 positions x 4 input channels.
// w: packed fp32 [group][ci 4][tap 41][co COG] (d_weight_offset(l)).
template <int COG, int S>
__global__ void __launch_bounds__(128) grouped_dx_kernel(const float *__restrict__ dz, float *__restrict__ dx,
                                                         const float *__restrict__ w, int Cin, int Cout, int Lin, int Lout) {
    constexpr int TP = 256, NT_ = TP / S + 41 / S + 2;  // dz positions a tile can touch
    __shared__ float ws[4 * 41 * COG];
    __shared__ float zs[COG * NT_];
    const int p0 = blockIdx.x * TP, g = blockIdx.y, b = blockIdx.z;
    for (int i = threadIdx.x; i < 4 * 41 * COG; i += 128) ws[i] = w[(size_t)g * 4 * 41 * COG + i];
    // t of position p, tap k: (p + 20 - k) / S; over the tile t ranges from floor((p0 + 20 - 40) / S) upwards
    const int tb = (p0 - 20) >= 0 ? (p0 - 20) / S : -((20 - p0 + S - 1) / S);
    for (int i = threadIdx.x; i < COG * NT_; i += 128) {
        const int co = i / NT_, t = tb + i % NT_;
        zs[i] = (t >= 0 && t < Lout) ? dz[((size_t)b * Cout + g * COG + co) * Lout + t] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int p = p0 + threadIdx.x + 128 * h;
        if (p >= Lin) continue;
        const int k0 = (p + 20) % S, tq = (p + 20) / S;  // tap k0 + S q reads t = tq - q
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int co = 0; co < COG; ++co) {
            const float *zr = zs + co * NT_ + (tq - tb);
#pragma unroll
            for (int q = 0; q < (40 / S) + 1; ++q) {
                const int k = k0 + S * q;
                if (k <= 40) {
                    const float z = zr[-q];
#pragma unroll
                    for (int ci = 0; ci < 4; ++ci) acc[ci] = fmaf(z, ws[(ci * 41 + k) * COG + co], acc[ci]);
                }
            }
        }
#pragma unroll
        for (int ci = 0; ci < 4; ++ci) dx[((size_t)b * Cin + g * 4 + ci) * Lin + p] = acc[ci];
    }
}

// Stride-4 specialisation (layers 1..3: 16 output channels per group).  The four positions p = 4j .. 4j+3 read the same dz
// values (t = j + 5 - q) through taps k = 4q + (p & 3), so a thread owns a quad of positions x 4 input channels and one
// float4 of four consecutive taps feeds 4 FMAs per dz load: 16 FMAs per 5 shared-memory loads (the generic kernel: 4).
__global__ void __launch_bounds__(128) grouped_dx4_kernel(const float *__restrict__ dz, float *__restrict__ dx,
                                                          const float *__restrict__ w, int Cin, int Cout, int Lin, int Lout) {
    constexpr int COG = 16, TP = 512, NT_ = TP / 4 + 12, KP = 44;  // taps padded to 44 per (co, ci)
    __shared__ __align__(16) float ws[COG * 4 * KP];               // [co][ci][k]
    __shared__ float zs[COG * NT_];
    const int p0 = blockIdx.x * TP, g = blockIdx.y, b = blockIdx.z;
    // staging: loads in global order (coalesced), loops unrolled so that a thread's ~40 loads are in flight together -- a CTA's
    // 2.8 k FMAs per thread are cheaper than 40 exposed L2 round trips
    if (threadIdx.x < COG * 4) {  // zero padding of taps 41..43
        float *pz = ws + threadIdx.x * KP + 41;
        pz[0] = 0.f; pz[1] = 0.f; pz[2] = 0.f;
    }
    const float *wg = w + (size_t)g * 4 * 41 * COG;
#pragma unroll 7
    for (int i = threadIdx.x; i < COG * 4 * 41; i += 128) {
        const int cik = i / COG, co = i - cik * COG, ci = cik / 41, k = cik - ci * 41;
        ws[(co * 4 + ci) * KP + k] = wg[i];
    }
    const int tb = p0 / 4 - 5;  // dz position of zs column 0: t = j + 5 - q >= p0/4 - 5
#pragma unroll 6
    for (int i = threadIdx.x; i < COG * NT_; i += 128) {
        const int co = i / NT_, t = tb + i % NT_;
        zs[i] = (t >= 0 && t < Lout) ? dz[((size_t)b * Cout + g * COG + co) * Lout + t] : 0.f;
    }
    __syncthreads();
    const int j = threadIdx.x, p = p0 + 4 * j;  // quad of positions p .. p + 3
    if (p >= Lin) return;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int ci = 0; ci < 4; ++ci) acc[r][ci] = 0.f;
#pragma unroll 1
    for (int co = 0; co < COG; ++co) {
        const float *zr = zs + co * NT_ + j + 10;  // column of t = j + 5 (tb = p0/4 - 5): j + 5 - tb + ... = j + 10
        const float *wr = ws + co * 4 * KP;
#pragma unroll
        for (int q = 0; q < 11; ++q) {  // q = 10: only tap 40 is real (41..43 are zero padding)
            const float z = zr[-q];
#pragma unroll
            for (int ci = 0; ci < 4; ++ci) {
                const float4 wv = *reinterpret_cast<const float4 *>(wr + ci * KP + 4 * q);
                acc[0][ci] = fmaf(z, wv.x, acc[0][ci]);
                acc[1][ci] = fmaf(z, wv.y, acc[1][ci]);
                acc[2][ci] = fmaf(z, wv.z, acc[2][ci]);
                acc[3][ci] = fmaf(z, wv.w, acc[3][ci]);
            }
        }
    }
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
        float *o = dx + ((size_t)b * Cin + g * 4 + ci) * Lin + p;
        if ((Lin & 3) == 0) {
            *reinterpret_cast<float4 *>(o) = make_float4(acc[0][ci], acc[1][ci], acc[2][ci], acc[3][ci]);
        } else {
#pragma unroll
            for (int r = 0; r < 4; ++r)
                if (p + r < Lin) o[r] = acc[r][ci];
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// dw, db partial sums, generic form (the model's four grouped layers all take the specialisations below -- grouped_dw4_kernel,
// grouped_dw1_kernel -- this is the readable statement of the same sums for any COG / stride).
// CTA = (chunk of (item, 128-output tile) pairs, group); thread (ci, k) owns the COG outputs
// dw[.][ci][k]; threads 164 .. 164 + COG - 1 own db.  partial: [chunk][group][164 * COG + COG].
template <int COG, int S>
__global__ void __launch_bounds__(192) grouped_dw_kernel(const float *__restrict__ dz, const float *__restrict__ x,
                                                         float *__restrict__ partial, int Bt, int Cin, int Cout, int Lin, int Lout,
                                                         int tiles_per_item, int tiles_per_chunk) {
    constexpr int TT = 128, XW = S * TT + 40;
    __shared__ __align__(16) float zs[TT * COG];  // [t][co]
    __shared__ float xs[4 * XW];                   // [ci][position - (S t0 - 20)]
    const int g = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
    const int ci = tid / 41, k = tid - 41 * ci;    // valid for tid < 164
    float acc[COG];
#pragma unroll
    for (int c = 0; c < COG; ++c) acc[c] = 0.f;
    float bacc = 0.f;
    const int total = Bt * tiles_per_item;
    const int first = chunk * tiles_per_chunk, last = min(total, first + tiles_per_chunk);
#pragma unroll 1
    for (int tile = first; tile < last; ++tile) {
        const int b = tile / tiles_per_item, t0 = (tile - b * tiles_per_item) * TT;
        __syncthreads();
        for (int i = tid; i < TT * COG; i += 192) {
            const int co = i / TT, t = i - co * TT;  // coalesced along t
            zs[t * COG + co] = (t0 + t < Lout) ? dz[((size_t)b * Cout + g * COG + co) * Lout + t0 + t] : 0.f;
        }
        for (int i = tid; i < 4 * XW; i += 192) {
            const int c = i / XW, p = S * t0 - 20 + (i - c * XW);
            xs[i] = (p >= 0 && p < Lin) ? x[((size_t)b * Cin + g * 4 + c) * Lin + p] : 0.f;
        }
        __syncthreads();
        if (tid < 164) {
            const float *xr = xs + ci * XW + k;
#pragma unroll 4
            for (int t = 0; t < TT; ++t) {
                const float xv = xr[S * t];
#pragma unroll
                for (int c4 = 0; c4 < COG / 4; ++c4) {
                    const float4 z = *reinterpret_cast<const float4 *>(zs + t * COG + 4 * c4);
                    acc[4 * c4 + 0] = fmaf(z.x, xv, acc[4 * c4 + 0]);
                    acc[4 * c4 + 1] = fmaf(z.y, xv, acc[4 * c4 + 1]);
                    acc[4 * c4 + 2] = fmaf(z.z, xv, acc[4 * c4 + 2]);
                    acc[4 * c4 + 3] = fmaf(z.w, xv, acc[4 * c4 + 3]);
                }
            }
        } else if (tid < 164 + COG) {
            for (int t = 0; t < TT; ++t) bacc += zs[t * COG + (tid - 164)];
        }
    }
    float *out = partial + ((size_t)chunk * gridDim.y + g) * (165 * COG);
    if (tid < 164) {
#pragma unroll
        for (int c = 0; c < COG; ++c) out[tid * COG + c] = acc[c];
    } else if (tid < 164 + COG) {
        out[164 * COG + (tid - 164)] = bacc;
    }
}

// Stride-4 specialisation of dw (layers 1..3: 16 output channels per group).  With k = 4 j + r the input index of output t is
// 4 (t + j) + r - 20: the 11 taps of one residue r read ONE phase signal x[4 u + r] at u = t + j, so a thread that owns
// (ci, r, six consecutive j, eight output channels) keeps a six-value sliding window of that signal in registers and does
// 48 FMAs per output position for 3 shared-memory loads (two float4 of dz, one new x value); the generic kernel: 16 per 5,
// i.e. bound by shared-memory loads.  64 threads = 4 ci x 4 r x 2 tap halves x 2 channel halves; partial layout as above.
__global__ void __launch_bounds__(64) grouped_dw4_kernel(const float *__restrict__ dz, const float *__restrict__ x,
                                                        float *__restrict__ partial, int Bt, int Cin, int Cout, int Lin, int Lout,
                                                        int tiles_per_item, int tiles_per_chunk) {
    constexpr int COG = 16, TT = 128, XW = 4 * TT + 44;  // (XW % 32 = 12: the two ci of a warp read different banks)
    __shared__ __align__(16) float zs[TT * COG];         // [t][co]
    __shared__ float xs[4 * XW];                          // [ci][position - (4 t0 - 20)]
    const int g = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
    const int ch = tid & 1, jh = (tid >> 1) & 1, r = (tid >> 2) & 3, ci = tid >> 4;
    const int j0 = 6 * jh;
    float acc[6][8];
#pragma unroll
    for (int jj = 0; jj < 6; ++jj)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[jj][c] = 0.f;
    float bacc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) bacc[c] = 0.f;
    const int total = Bt * tiles_per_item;
    const int first = chunk * tiles_per_chunk, last = min(total, first + tiles_per_chunk);
    const float *xr = xs + ci * XW + 4 * j0 + r;  // window element (t, jj) = xr[4 (t + jj)]
#pragma unroll 1
    for (int tile = first; tile < last; ++tile) {
        const int b = tile / tiles_per_item, t0 = (tile - b * tiles_per_item) * TT;
        __syncthreads();
        // (staging loops unrolled: with 64 threads a tile is ~70 loads per thread, and one exposed L2 round trip per load would
        //  cost more than the tile's FMAs)
#pragma unroll 8
        for (int i = tid; i < TT * COG; i += 64) {
            const int co = i / TT, t = i - co * TT;  // coalesced along t
            zs[t * COG + co] = (t0 + t < Lout) ? dz[((size_t)b * Cout + g * COG + co) * Lout + t0 + t] : 0.f;
        }
#pragma unroll 7
        for (int i = tid; i < 4 * XW; i += 64) {
            const int c = i / XW, p = 4 * t0 - 20 + (i - c * XW);
            xs[i] = (p >= 0 && p < Lin && i - c * XW < 4 * TT + 40) ? x[((size_t)b * Cin + g * 4 + c) * Lin + p] : 0.f;
        }
        __syncthreads();
        float w[6];  // slot (t + jj) % 6 holds the window element (t, jj)
#pragma unroll
        for (int jj = 0; jj < 5; ++jj) w[jj] = xr[4 * jj];
        const int nt = min(TT, Lout - t0);  // (a short sequence's last tile is mostly padding: 33 of 128 positions at scale 2)
#pragma unroll 1
        for (int t = 0; t < nt; t += 6) {
#pragma unroll
            for (int tt = 0; tt < 6; ++tt) {
                if (t + tt < nt) {
                    w[(tt + 5) % 6] = xr[4 * (t + tt + 5)];
                    const float4 za = *reinterpret_cast<const float4 *>(zs + (t + tt) * COG + 8 * ch);
                    const float4 zb = *reinterpret_cast<const float4 *>(zs + (t + tt) * COG + 8 * ch + 4);
                    const float z[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
#pragma unroll
                    for (int jj = 0; jj < 6; ++jj)
#pragma unroll
                        for (int c = 0; c < 8; ++c) acc[jj][c] = fmaf(z[c], w[(tt + jj) % 6], acc[jj][c]);
                    if (tid < 2) {
#pragma unroll
                        for (int c = 0; c < 8; ++c) bacc[c] += z[c];
                    }
                }
            }
        }
    }
    float *out = partial + ((size_t)chunk * gridDim.y + g) * (165 * COG);
#pragma unroll
    for (int jj = 0; jj < 6; ++jj) {
        const int k = 4 * (j0 + jj) + r;
        if (k <= 40) {
#pragma unroll
            for (int c = 0; c < 8; ++c) out[(ci * 41 + k) * COG + 8 * ch + c] = acc[jj][c];
        }
    }
    if (tid < 2) {
#pragma unroll
        for (int c = 0; c < 8; ++c) out[164 * COG + 8 * tid + c] = bacc[c];
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Layer 4 (stride 1, 4 -> 4 channels per group, 256 groups): with only 4 output channels per group the generic kernels
// spend one shared-memory load per 2-4 FMAs.  Register-tiled along TIME instead:
//   dx: a thread owns 8 consecutive positions x 4 ci of one group; per co it keeps the 48 dz values those positions touch
//       (p + 20 - k, k = 0..40) in registers and streams the 164 weights: 1312 FMAs per 12 float4 + 164 scalar loads.
//   dw: a thread owns (group, ci, block of 8 taps) x 4 co = 32 accumulators and slides an 8-value window of x over t:
//       32 FMAs per 5 shared-memory loads.
constexpr int kG1Groups = 8;  // groups per CTA of both kernels

__global__ void __launch_bounds__(128) grouped_dx1_kernel(const float *__restrict__ dz, float *__restrict__ dx,
                                                          const float *__restrict__ w, int Lin) {
    constexpr int NG = kG1Groups, TP = 128, ZW = TP + 40, KP = 44, C = 1024;
    __shared__ __align__(16) float zs[NG * 4 * ZW];   // [group, co][position - (p0 - 20)]
    __shared__ float ws[NG * 16 * KP];                 // [group][co][ci][k]
    const int p0 = blockIdx.x * TP, g0 = blockIdx.y * NG, b = blockIdx.z;
    // staging (see grouped_dx4_kernel): the CTA's 8 groups are one contiguous run of the packed [group][ci][k][co] weights
    {
        float *pz = ws + threadIdx.x * KP + 41;  // 128 (group, co, ci) rows: zero padding of taps 41..43
        pz[0] = 0.f; pz[1] = 0.f; pz[2] = 0.f;
    }
    const float *wg = w + (size_t)g0 * 656;
#pragma unroll 8
    for (int i = threadIdx.x; i < NG * 656; i += 128) {
        const int g = i / 656, rem = i - g * 656, cik = rem >> 2, co = rem & 3, ci = cik / 41, k = cik - ci * 41;
        ws[((g * 4 + co) * 4 + ci) * KP + k] = wg[i];
    }
#pragma unroll 7
    for (int i = threadIdx.x; i < NG * 4 * ZW; i += 128) {
        const int c = i / ZW, t = p0 - 20 + i % ZW;  // stride 1: Lout == Lin
        zs[i] = (t >= 0 && t < Lin) ? dz[((size_t)b * C + g0 * 4 + c) * Lin + t] : 0.f;
    }
    __syncthreads();
    const int g = threadIdx.x >> 4, pb = threadIdx.x & 15, p = p0 + 8 * pb;
    if (p >= Lin) return;  // (a 65- or 33-position sequence fills half / a quarter of its last tile)
    float acc[4][8];
#pragma unroll
    for (int ci = 0; ci < 4; ++ci)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[ci][j] = 0.f;
#pragma unroll 1
    for (int co = 0; co < 4; ++co) {
        float zw[48];  // dz[co][p + j - 20], j = 0..47: position p + jj with tap k reads index jj + 40 - k
        const float4 *zr = reinterpret_cast<const float4 *>(zs + (g * 4 + co) * ZW + 8 * pb);
#pragma unroll
        for (int q = 0; q < 12; ++q) {
            const float4 v = zr[q];
            zw[4 * q] = v.x; zw[4 * q + 1] = v.y; zw[4 * q + 2] = v.z; zw[4 * q + 3] = v.w;
        }
#pragma unroll 1
        for (int ci = 0; ci < 4; ++ci) {
            const float *wr = ws + ((g * 4 + co) * 4 + ci) * KP;
#pragma unroll
            for (int k = 0; k < 41; ++k) {
                const float wv = wr[k];
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[ci][j] = fmaf(wv, zw[j + 40 - k], acc[ci][j]);
            }
        }
    }
#pragma unroll
    for (int ci = 0; ci < 4; ++ci) {
        float *o = dx + ((size_t)b * C + (g0 + g) * 4 + ci) * Lin + p;
        if ((Lin & 3) == 0 && p + 8 <= Lin) {
            *reinterpret_cast<float4 *>(o) = make_float4(acc[ci][0], acc[ci][1], acc[ci][2], acc[ci][3]);
            *reinterpret_cast<float4 *>(o + 4) = make_float4(acc[ci][4], acc[ci][5], acc[ci][6], acc[ci][7]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (p + j < Lin) o[j] = acc[ci][j];
        }
    }
}

// partial layout per (chunk, group) as in grouped_dw_kernel<4, 1>: [(ci * 41 + k) * 4 + co] then 4 bias sums
__global__ void __launch_bounds__(192) grouped_dw1_kernel(const float *__restrict__ dz, const float *__restrict__ x,
                                                          float *__restrict__ partial, int Bt, int L, int tiles_per_item,
                                                          int tiles_per_chunk) {
    constexpr int NG = kG1Groups, TT = 128, XW = TT + 48, C = 1024;
    __shared__ float zs[NG * 4 * TT];  // [group, co][t]
    __shared__ float xs[NG * 4 * XW];  // [group, ci][position - (t0 - 20)]
    const int chunk = blockIdx.x, g0 = blockIdx.y * NG, tid = threadIdx.x;
    const int g = tid / 24, ci = (tid / 6) & 3, tb = tid % 6;  // taps 8 tb .. 8 tb + 7
    float acc[4][8];
#pragma unroll
    for (int co = 0; co < 4; ++co)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[co][j] = 0.f;
    float bacc[4] = {0.f, 0.f, 0.f, 0.f};
    const int total = Bt * tiles_per_item;
    const int first = chunk * tiles_per_chunk, last = min(total, first + tiles_per_chunk);
#pragma unroll 1
    for (int tile = first; tile < last; ++tile) {
        const int b = tile / tiles_per_item, t0 = (tile - b * tiles_per_item) * TT;
        __syncthreads();
#pragma unroll 6
        for (int i = tid; i < NG * 4 * TT; i += 192) {
            const int c = i / TT, t = t0 + i % TT;
            zs[i] = t < L ? dz[((size_t)b * C + g0 * 4 + c) * L + t] : 0.f;
        }
#pragma unroll 6
        for (int i = tid; i < NG * 4 * XW; i += 192) {
            const int c = i / XW, p = t0 - 20 + i % XW;
            xs[i] = (p >= 0 && p < L) ? x[((size_t)b * C + g0 * 4 + c) * L + p] : 0.f;
        }
        __syncthreads();
        const int nt = min(TT, L - t0);  // positions of this tile that exist
        const float *zr = zs + g * 4 * TT, *xr = xs + (g * 4 + ci) * XW + 8 * tb;
        float xw[8];  // x[ci][t + 8 tb + j - 20], slid along t
#pragma unroll
        for (int j = 0; j < 8; ++j) xw[j] = xr[j];
#pragma unroll 8
        for (int t = 0; t < nt; ++t) {
            const float z0 = zr[t], z1 = zr[TT + t], z2 = zr[2 * TT + t], z3 = zr[3 * TT + t];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                acc[0][j] = fmaf(z0, xw[j], acc[0][j]);
                acc[1][j] = fmaf(z1, xw[j], acc[1][j]);
                acc[2][j] = fmaf(z2, xw[j], acc[2][j]);
                acc[3][j] = fmaf(z3, xw[j], acc[3][j]);
            }
            if (ci == 0 && tb == 0) { bacc[0] += z0; bacc[1] += z1; bacc[2] += z2; bacc[3] += z3; }
#pragma unroll
            for (int j = 0; j < 7; ++j) xw[j] = xw[j + 1];
            xw[7] = xr[t + 8];
        }
    }
    float *out = partial + ((size_t)chunk * 256 + g0 + g) * (165 * 4);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int k = 8 * tb + j;
        if (k < 41) {
#pragma unroll
            for (int co = 0; co < 4; ++co) out[(ci * 41 + k) * 4 + co] = acc[co][j];
        }
    }
    if (ci == 0 && tb == 0) {
#pragma unroll
        for (int co = 0; co < 4; ++co) out[164 * 4 + co] = bacc[co];
    }
}

// fixed-order combination of the chunk partials -> dw [Cout][4][41] (the weight_v layout), db [Cout]
template <int COG>
__global__ void __launch_bounds__(256) grouped_dw_combine_kernel(const float *__restrict__ partial, float *__restrict__ dw,
                                                                 float *__restrict__ db, int groups, int chunks) {
    const int per_group = 165 * COG;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= groups * per_group) return;
    const int g = i / per_group, r = i - g * per_group;
    float s = 0.f;
    for (int c = 0; c < chunks; ++c) s += partial[((size_t)c * groups + g) * per_group + r];
    if (r < 164 * COG) {
        const int cik = r / COG, co = r - cik * COG;  // cik = ci * 41 + k
        dw[((size_t)(g * COG + co)) * 164 + cik] = s;
    } else {
        db[g * COG + (r - 164 * COG)] = s;
    }
}

// dz = (g1 + g2) * LeakyReLU'(out): the gradient that reaches a layer's pre-activation from the next layer (g1) and from
// the feature-map loss (g2, may be null) -- one launch instead of add + compare + scale + select
__global__ void __launch_bounds__(256) lrelu_grad_kernel(const float *__restrict__ g1, const float *__restrict__ g2,
                                                         const float *__restrict__ out, float *__restrict__ dz, long long n) {
    const long long n4 = n >> 2;
    const bool vec = ((reinterpret_cast<uintptr_t>(g1) | reinterpret_cast<uintptr_t>(g2) | reinterpret_cast<uintptr_t>(out) |
                       reinterpret_cast<uintptr_t>(dz)) & 15) == 0;
    const long long stride = (long long)gridDim.x * 256, i0 = (long long)blockIdx.x * 256 + threadIdx.x;
    if (vec) {
        for (long long i = i0; i < n4; i += stride) {
            float4 a = reinterpret_cast<const float4 *>(g1)[i];
            if (g2) {
                const float4 b = reinterpret_cast<const float4 *>(g2)[i];
                a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
            }
            const float4 o = reinterpret_cast<const float4 *>(out)[i];
            reinterpret_cast<float4 *>(dz)[i] = make_float4(o.x > 0.f ? a.x : a.x * kSlope, o.y > 0.f ? a.y : a.y * kSlope,
                                                            o.z > 0.f ? a.z : a.z * kSlope, o.w > 0.f ? a.w : a.w * kSlope);
        }
    }
    for (long long i = (vec ? 4 * n4 : 0) + i0; i < n; i += stride) {
        const float a = g1[i] + (g2 ? g2[i] : 0.f);
        dz[i] = out[i] > 0.f ? a : a * kSlope;
    }
}

int launch_lrelu_grad(const float *g1, const float *g2, const float *out, float *dz, long long n, cudaStream_t s) {
    if (!g1 || !out || !dz || n < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_lrelu_backward: bad argument");
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    if (blocks < 1) blocks = 1;
    lrelu_grad_kernel<<<(unsigned)blocks, 256, 0, s>>>(g1, g2, out, dz, n);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

constexpr int kDw4Ctas = 8 * kNumSMs;  // grouped_dw4_kernel: 64 threads and 17 KB of shared memory per CTA -> 8 per SM
constexpr int kDwCtas = 4 * kNumSMs;   // the 192-thread weight-gradient kernels: 4 per SM
struct GroupedBwdPlan {
    int tiles_per_item, tiles_per_chunk, chunks;
};
static GroupedBwdPlan grouped_plan(int groups, int Bt, int Lout, int ctas = kDwCtas) {
    GroupedBwdPlan p;
    p.tiles_per_item = (Lout + 127) / 128;
    const int total = Bt * p.tiles_per_item;
    int want = (ctas + groups - 1) / groups;  // ~4 CTAs per SM over all groups (192-thread kernels), ~8 for the 64-thread one
    if (want > total) want = total;
    if (want < 1) want = 1;
    p.tiles_per_chunk = (total + want - 1) / want;
    p.chunks = (total + p.tiles_per_chunk - 1) / p.tiles_per_chunk;
    return p;
}

// CTAs along the group axis: the layer-4 kernels take kG1Groups groups each
static int group_blocks(int groups, int cog, int stride) { return (stride == 1 && cog == 4 && groups == 256) ? groups / kG1Groups : groups; }

size_t grouped_bwd_workspace_bytes(int l, int Bt, int Lout) {
    const DLayer d = d_layer(l);
    const int cog = d.cout / d.groups;
    return (size_t)grouped_plan(group_blocks(d.groups, cog, d.stride), Bt, Lout, d.stride == 4 ? kDw4Ctas : kDwCtas).chunks * d.groups * 165 * cog *
           sizeof(float);
}

template <int COG, int S>
static int grouped_backward(const float *w, const float *dz, const float *x, float *dx, float *dw, float *db, float *ws, int Bt,
                            int Cin, int Cout, int Lin, int Lout, cudaStream_t s) {
    const int groups = Cin / 4;
    if (dx) {
        if (S == 4 && COG == 16) {
            dim3 grid((Lin + 511) / 512, groups, Bt);
            grouped_dx4_kernel<<<grid, 128, 0, s>>>(dz, dx, w, Cin, Cout, Lin, Lout);
        } else if (S == 1 && COG == 4 && Cin == 1024) {
            dim3 grid((Lin + 127) / 128, groups / kG1Groups, Bt);
            grouped_dx1_kernel<<<grid, 128, 0, s>>>(dz, dx, w, Lin);
        } else {
            dim3 grid((Lin + 255) / 256, groups, Bt);
            grouped_dx_kernel<COG, S><<<grid, 128, 0, s>>>(dz, dx, w, Cin, Cout, Lin, Lout);
        }
        MG_CUDA_TRY(cudaGetLastError());
    }
    if (dw) {
        const GroupedBwdPlan p = grouped_plan(group_blocks(groups, COG, S), Bt, Lout, S == 4 ? kDw4Ctas : kDwCtas);
        if (S == 4 && COG == 16) {
            dim3 grid(p.chunks, groups);
            grouped_dw4_kernel<<<grid, 64, 0, s>>>(dz, x, ws, Bt, Cin, Cout, Lin, Lout, p.tiles_per_item, p.tiles_per_chunk);
        } else if (S == 1 && COG == 4 && Cin == 1024) {
            dim3 grid(p.chunks, groups / kG1Groups);
            grouped_dw1_kernel<<<grid, 192, 0, s>>>(dz, x, ws, Bt, Lin, p.tiles_per_item, p.tiles_per_chunk);
        } else {
            dim3 grid(p.chunks, groups);
            grouped_dw_kernel<COG, S><<<grid, 192, 0, s>>>(dz, x, ws, Bt, Cin, Cout, Lin, Lout, p.tiles_per_item, p.tiles_per_chunk);
        }
        MG_CUDA_TRY(cudaGetLastError());
        const int n = groups * 165 * COG;
        grouped_dw_combine_kernel<COG><<<(n + 255) / 256, 256, 0, s>>>(ws, dw, db, groups, p.chunks);
        MG_CUDA_TRY(cudaGetLastError());
    }
    return MG_OK;
}

// blob: one discriminator's packed weights (scale sc of the MSD blob); layer l in 1..4
int launch_disc_grouped_backward(const void *blob, int l, const float *dz, const float *x, float *dx, float *dw, float *db,
                                 float *ws, int Bt, int Lin, int Lout, cudaStream_t s) {
    const DLayer d = d_layer(l);
    const float *w = reinterpret_cast<const float *>(blob) + d_weight_offset(l);
    if (Bt > 65535) return set_error(MG_ERR_INVALID_ARGUMENT, "discriminator batch %d exceeds 65535", Bt);
    if (l == 4) return grouped_backward<4, 1>(w, dz, x, dx, dw, db, ws, Bt, d.cin, d.cout, Lin, Lout, s);
    return grouped_backward<16, 4>(w, dz, x, dx, dw, db, ws, Bt, d.cin, d.cout, Lin, Lout, s);
}

// ------------------------------------------------------------------------------------------------------------------
// weight-norm backward for all 21 layers in one launch (one CTA per norm row, like disc_pack_kernel):
//   w = g v / |v|   =>   dg = <dw, v> / |v|,   dv = (g / |v|) (dw - <dw, v> v / |v|^2)
struct DiscWnArgs {
    const float *v[3 * kDiscLayers];
    const float *g[3 * kDiscLayers];
    const float *dw[3 * kDiscLayers];
    float *dv[3 * kDiscLayers];
    float *dg[3 * kDiscLayers];
};

__global__ void __launch_bounds__(128) disc_wn_backward_kernel(const __grid_constant__ DiscWnArgs a) {
    int grow = blockIdx.x;
    const int d = grow / kDiscRows;
    grow -= d * kDiscRows;
    int l = 0;
#pragma unroll 1
    while (grow >= d_layer(l).cout) { grow -= d_layer(l).cout; ++l; }
    const DLayer sh = d_layer(l);
    const int inner = (sh.cin / sh.groups) * sh.k, idx = d * kDiscLayers + l;
    if (!a.dw[idx]) return;
    const float *vr = a.v[idx] + (size_t)grow * inner, *dwr = a.dw[idx] + (size_t)grow * inner;
    float ss = 0.f, dot = 0.f;
    for (int j = threadIdx.x; j < inner; j += 128) {
        ss = fmaf(vr[j], vr[j], ss);
        dot = fmaf(dwr[j], vr[j], dot);
    }
    __shared__ float red[2][4];
    for (int o = 16; o > 0; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        dot += __shfl_xor_sync(0xffffffffu, dot, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ss; red[1][threadIdx.x >> 5] = dot; }
    __syncthreads();
    ss = (red[0][0] + red[0][1]) + (red[0][2] + red[0][3]);
    dot = (red[1][0] + red[1][1]) + (red[1][2] + red[1][3]);
    const float inv = rsqrtf(ss), gv = a.g[idx][grow];
    const float sc = gv * inv, proj = dot / ss;
    float *dvr = a.dv[idx] + (size_t)grow * inner;
    for (int j = threadIdx.x; j < inner; j += 128) dvr[j] = sc * (dwr[j] - proj * vr[j]);
    if (threadIdx.x == 0) a.dg[idx][grow] = dot * inv;
}

int launch_disc_wn_backward(const float *const *v, const float *const *g, const float *const *dw, float *const *dv,
                            float *const *dg, cudaStream_t s) {
    DiscWnArgs a;
    for (int i = 0; i < 3 * kDiscLayers; ++i) {
        if (!v[i] || !g[i] || (dw[i] && (!dv[i] || !dg[i]))) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_wn_backward: null tensor %d", i);
        a.v[i] = v[i]; a.g[i] = g[i]; a.dw[i] = dw[i]; a.dv[i] = dv[i]; a.dg[i] = dg[i];
    }
    disc_wn_backward_kernel<<<3 * kDiscRows, 128, 0, s>>>(a);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

}  // namespace mg
