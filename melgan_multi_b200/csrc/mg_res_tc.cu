// ResBlock on the tensor cores (wgmma), split-bf16 (3 MMAs per product) for fp32-grade results.
//
// Reference semantics: ResBlock.forward, models.py:32-40 -- three times  x = c2(lrelu(c1(lrelu(x)))) + x  with
// c1 dilations 1/3/9 and c2 dilation 1, all k=3 "same" convs on C channels.
//
// One CTA owns P = 64*NRB consecutive positions of one batch item (16-position halo per side, recomputed by the
// neighbours; in a cluster of CS CTAs only at the cluster's outer edges) and keeps the whole block on chip:
//   registers  every consumer warpgroup owns RPW 64-position blocks x NCW = C/NCP channels of
//                R   fp32 residual stream                     D   fp32 c1 accumulator
//              (wgmma accumulator layout, mg_tc.cuh).  R + D are 2 * P * C floats per CTA: that product is what sizes the
//              tiles -- 64 x 256, 128 x 128, 256 x 64, 512 x 32 -- against the 64 K registers of an SM.
//   smem   X  = lrelu(current conv input) as split-bf16 (hi, lo), "row-linear K-major" (mg_tc.cuh): row = position,
//               k-panels of 8 channels.  A conv tap at dilation d is the same buffer with the start address
//               moved by 16*d bytes -- there is no im2col and no per-tap restaging.
//   smem   ring of weight chunks (one (tap, K-slice) of [Cout x KC] hi+lo per chunk), filled by 1-D bulk TMA
//               copies from the pre-packed blob (mg_layout.h), released by the consumers once their MMAs have read it.
// GEMM view of one conv: D[pos, co] (+)= sum_tap sum_pass X_pass[pos + (tap-1)*d, :] * W_pass[tap][co, :]^T with
// M = 64 positions per instruction, N = NCW, K = 16; passes (xh,wh), (xl,wh), (xh,wl).  At C <= 64 an instruction of
// N = NCW reads more operand bytes per clock than shared memory delivers, so there the weights are stacked [wh | wl]
// along N: xh * [wh | wl] is one MMA of N = 2 NCW and the activations are read twice per k-step, not three times.
// c2 accumulates straight onto R, so the residual add costs nothing; conv biases are added when the accumulator
// is read back (b2 is carried in `pend`).  Positions outside [0, L) are written as zeros into X after every conv,
// which is the per-layer zero padding of the reference.
//
// Warp roles: NWG consumer warpgroups (input load, MMAs, X hand-off between convs, output), one TMA producer warp.
// UPF (stride-2 stages): the stage's LeakyReLU -> ConvTranspose1d(2C -> C, k4, s2, p1) runs inside this kernel first, so
// the CTA reads the PREVIOUS stage's output [B][2C][L/2] and the ConvT output never goes to HBM.  Accumulator row m of a
// "ConvT block" owns the output pair (t = o + 2m, o + 2m + 1):
//     out[2s]     = x[s] W1 + x[s-1] W3        out[2s+1] = x[s+1] W0 + x[s] W2        (s = o/2 + m; taps of models.py:50-51)
// i.e. two MMA chains of N = C over the 2C input channels, whose A operand is the same (input-position) buffer read at
// row offsets 1, 0 / 2, 1.  The pairs are then de-interleaved through shared memory (fp32, in the X region that is not
// in use yet) so that row = output position can fill R, and from there on the kernel is the plain ResBlock.
// UPT = S (2 or 8): the NEXT stage's LeakyReLU -> ConvTranspose1d(C -> C/2, k = 2S, stride S) runs at the TAIL of this kernel
// (models.py:64-65 of the following loop iteration): after the sixth conv the consumers write X = split(lrelu(x)) exactly as
// they do between convs, and the ConvT is two more "taps" on that operand -- out[S s + phi - pad] = x[s] W[phi] + x[s-1] W[phi+S],
// all S phases stacked along N like mg_up_tc.cu (N = S * NG = C in every stage), accumulated in the registers of D, which the
// ResBlock no longer needs.  The kernel then stores the ConvT output [B][C/2][S L] instead of the ResBlock output: the
// ResBlock output never goes to HBM, and the separate ConvT kernel (its activation re-read, operand conversion and launch)
// disappears.  An input position s owns the outputs [S s - pad, S s - pad + S) and needs x[s - 1]: tiles overlap by one
// more row on the left (HL = HALO + 1).  Position L (x[L] = 0) would own the last `pad` outputs; those pad * C/2 outputs --
// dot products of x[L-1] with the tap-1 weights -- are computed in fp32 by the CTA that owns position L - 1.
// Bf16<Cfg> (mg_tc.cuh; the default chain's Rb0, Rb1, Rb2 and Up3Rb3Post): the same kernel with one pass (xh, wh) per
// product -- in the convs and the front ConvT's taps --, X and the front ConvT operand written as hi only, the weight
// ring filled with the hi half of each chunk (C <= 64: the whole stacked chunk, of which only the hi rows are read) and the cluster halo exchange sending the hi k-panels only.  The fp32 parts
// (residual stream, biases, conv_post epilogue) are unchanged.
// Pcm16<Cfg> (Up3Rb3Post and Bf16<Up3Rb3Post>): the audio is stored as 16-bit PCM, pcm16(tanhf(acc)), see below.
#include <stdlib.h>
#include <string.h>

#include "mg_common.cuh"
#include "mg_tc.cuh"

namespace mg {
using namespace tc;

// C channels; NRB 64-position blocks per CTA, RPW of them per consumer warpgroup; NCP column parts (warpgroups that share
// the same rows, each with C / NCP accumulator columns); NSTAGE weight-ring slots.  POST / UPF / UPT: see above.
// CS > 1: thread-block clusters of CS CTAs (see the kernel).
template <int C_, int NRB_, int RPW_, int NCP_, int NSTAGE_, bool POST_ = false, bool UPF_ = false, int UPT_ = 0, int CS_ = 1>
struct RbCfg {
    static constexpr int C = C_, NRB = NRB_, RPW = RPW_, NCP = NCP_, NSTAGE = NSTAGE_, UPT = UPT_, CS = CS_;
    static constexpr bool POST = POST_;  // fuse LeakyReLU -> conv_post -> tanh into the final epilogue (last stage)
    static constexpr bool UPF = UPF_;
    static constexpr bool ONEPASS = false;  // Bf16<RbCfg<..>>: one bf16 pass per product (mg_tc.cuh)
    using Out = float;                      // element type of y; Pcm16<Cfg>: int16 audio
    static constexpr int P = 64 * NRB;
    static constexpr int NWG = NRB / RPW * NCP;  // consumer warpgroups
    static constexpr int NCONS = 128 * NWG;
    static constexpr int NT = NCONS + 32;
    static constexpr int NCW = C / NCP;          // accumulator columns per warpgroup = MMA N
    static constexpr int SLACK = 16;             // zero rows either side of X (dilation-9 taps reach 9 rows out)
    static constexpr int HALO = 16 + (POST ? 3 : 0);  // 1+1+3+1+9+1 (+3 for the fused k7 conv_post)
    static constexpr int HL = HALO + (UPT_ ? 1 : 0);  // left halo: a fused tail ConvT also reads x[s - 1]
    static constexpr int ROWS = P + 2 * SLACK;
    static constexpr int XPITCH = ROWS * 16;  // bytes between k-panels
    static constexpr int KP = C / 8;
    static constexpr int XBYTES = KP * XPITCH;  // one of {hi, lo}
    static constexpr int KC = tc_kc(C);
    static constexpr int CHUNK = tc_chunk_bytes(C);
    static constexpr int HALF = CHUNK / 2;
    static constexpr int NCHUNK = tc_chunks_per_conv(C);
    static constexpr int KSL = C / KC;
    // tail ConvT: TNG output channels per group (mg_layout.h up_ng of the next stage), TN = MMA N over all column parts, TNCG
    // groups, ring slots of TSLOT bytes (stride 8: one tap of a 16-channel chunk; stride 2: both taps), TNSLOT of them
    static constexpr int TNG = UPT == 8 ? 32 : C / 2, TN = (UPT ? UPT : 1) * TNG, TNCG = (C / 2) / TNG;
    static constexpr int TSLOT = UPT == 8 ? 16384 : 128 * UPT * TNG, TNSLOT = UPT ? TNCG * (C / 16) * (UPT == 8 ? 2 : 1) : 0;
    static_assert(UPT == 0 || ((UPT == 2 || UPT == 8) && TN == C && TSLOT <= CHUNK && !POST_ && !UPF_), "tail ConvT shape");
    static_assert(UPT != 8 || NCW == 128, "stride-8 tail: each column part stores four phases of a channel as one float4");
    // fused ConvT: input rows s = o/2 - 1 .. o/2 + P/2 of 2C channels (2 KP k-panels), NPB blocks of 64 output pairs
    static constexpr int UROWS = P / 2 + 2, UPITCH = UROWS * 16, NPB = NRB / 2, UKSL = 2 * C / KC, NUPCH = UPF ? 4 * UKSL : 0;
    static constexpr int SPITCH = P + 4;  // floats between channels of the fp32 staging buffer [C][P]
    static_assert(!UPF || (NCP == 1 && NPB <= NWG && 2 * KP * UPITCH <= XBYTES && C * SPITCH * 4 <= 2 * XBYTES),
                  "fused ConvT must fit the X region");
    static_assert(!POST || (C == 32 && NCP == 1), "conv_post fusion is for the 32-channel stage");
    // clusters: CS * P positions per cluster, halos only at the cluster's outer edges (PVB outputs kept by a cluster with
    // more sequence on both sides); XCH rows (the largest dilation) of each cluster-internal border are copied into the
    // neighbour's slack rows at every X hand-off
    static constexpr int PVB = CS * P - HALO - HL, XCH = 9;
    static_assert(CS == 1 || ((CS == 2 || CS == 4) && !POST_ && !UPF_ && UPT_ == 0 && XCH <= SLACK && 2 * XCH <= P),
                  "clusters are for the plain ResBlock");
    // per-CTA constants, copied into shared memory before griddepcontrol.wait: the six conv biases [conv][C] (c1[0..2],
    // c2[0..2]: layers l0 .. l0 + 5), then the front ConvT's bias (C), the tail ConvT's bias (C / 2), conv_post's weights
    // [ci][8] and bias
    static constexpr int CB_UPF = 6 * C, CB_UPT = CB_UPF + (UPF_ ? C : 0), CB_POST = CB_UPT + (UPT_ ? C / 2 : 0);
    static constexpr int NCONST = CB_POST + (POST_ ? 32 * 8 + 4 : 0);
    static_assert(CB_POST % 4 == 0 && NCONST % 2 == 0, "conv_post weights are read as float4, the mbarriers follow");
    static constexpr int SMEM_BYTES = 2 * XBYTES + NSTAGE * CHUNK + (2 * C + NCONST) * 4 + (2 * NSTAGE + (CS > 1 ? 2 : 0) + 1) * 8;
    static_assert(SMEM_BYTES + 1024 <= 227 * 1024, "shared memory budget");
    static_assert(XPITCH / 16 < 16384, "LBO field");
    static_assert(NRB % RPW == 0 && C % NCP == 0 && NCW % 32 == 0, "warpgroup split");
};

// 16-bit PCM output of a conv_post configuration (mg_gen_forward_pcm16): the same kernel, whose epilogue stores
// pcm16(tanhf(acc)) (mg_common.cuh) as int16 instead of tanhf(acc); everything before the store is unchanged, so the
// samples are pcm16 of the float kernel's bit for bit.  A distinct type, so the instantiation has a symbol of its own.
template <class Cfg>
struct Pcm16 : Cfg {
    using Out = int16_t;
    static_assert(Cfg::POST, "int16 output is the audio of a conv_post configuration");
};

template <int RPW, int R>
__device__ __forceinline__ void acc_fence2(float (&a)[RPW][R]) {
#pragma unroll
    for (int r = 0; r < RPW; ++r) acc_fence<R>(a[r]);
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NT, 1)
resblock_tc_kernel(const float *__restrict__ x, float *__restrict__ y_, int stage, const __grid_constant__ RunTable clusters,
                   int *__restrict__ status, long long *__restrict__ trace) {
    constexpr int C = Cfg::C, P = Cfg::P, SLACK = Cfg::SLACK, HALO = Cfg::HALO, HL = Cfg::HL;
    constexpr int XPITCH = Cfg::XPITCH, XBYTES = Cfg::XBYTES, KC = Cfg::KC, CHUNK = Cfg::CHUNK, NSTAGE = Cfg::NSTAGE;
    constexpr int NCONS = Cfg::NCONS, NCP = Cfg::NCP, NCW = Cfg::NCW, RPW = Cfg::RPW, KSL = Cfg::KSL, NA = NCW / 2;
    constexpr int CS = Cfg::CS, XCH = Cfg::XCH;
    // passes per product: (xh, wh), (xl, wh), (xh, wl), or (xh, wh) alone in the single-pass variant, which then never
    // writes or reads Xl nor the lo half of a weight chunk
    constexpr bool ONE = Cfg::ONEPASS;
    constexpr int NPASS = ONE ? 1 : 3;
    // C <= 64: a weight chunk holds [hi | lo] rows per k-panel (mg_layout.h, tc_stacked).  Where a second accumulator is
    // free the three passes become two MMAs per k-step -- xh * [wh | wl] as one instruction of N = 2 NCW into an
    // accumulator pair (main, lo), then xl * wh of N = NCW onto main -- so the A operand is read from shared memory twice
    // instead of three times; the pair is added when the accumulator is read back.  That is every c2 (lo = D, dead between
    // its hand-off and the next c1) and the front ConvT's taps at RPW >= 2 (lo = row block 1 of R / D).  A c1 has R and D
    // live and would need a third accumulator: 3 * RPW * NA = 96 registers, which is all a thread of these 17-warp CTAs
    // can have (ptxas spills 1.6 - 2.8 KB per thread), so the c1 convs keep three passes, on the same chunks.
    // WLO: bytes from a k-panel's hi rows to its lo rows, WKP: k-panel pitch.
    constexpr bool STK = tc_stacked(C), PAIR = STK && !ONE;
    constexpr uint32_t WLO = STK ? C * 16 : Cfg::HALF, WKP = STK ? 2 * C * 16 : C * 16;
    static_assert(!STK || NCP == 1, "stacked weights: one column part");
    // bytes of a ResBlock / front-ConvT weight chunk brought in (single pass: the hi half where it is contiguous)
    constexpr uint32_t WBYTES = ONE && !STK ? Cfg::HALF : CHUNK;
    static_assert(!ONE || Cfg::UPT == 0, "the single-pass variant has no tail ConvT");
    // y is declared float * for every configuration, so that the float instantiations keep their signature and symbol;
    // Pcm16<Cfg> stores int16 audio through it
    typename Cfg::Out *__restrict__ y = reinterpret_cast<typename Cfg::Out *>(y_);
    static_assert(Cfg::POST || sizeof(typename Cfg::Out) == sizeof(float), "int16 output is for the conv_post epilogue only");
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t *Xh = smem, *Xl = smem + XBYTES, *ring = smem + 2 * XBYTES;
    float *pend = reinterpret_cast<float *>(ring + NSTAGE * CHUNK);  // sum of the c2 biases folded so far
    float *b1s = pend + C;                                            // (tail ConvT: lrelu(x[L-1]) for its fix-up)
    float *cst = b1s + C;                                             // [NCONST]: the per-CTA constants (RbCfg)
    uint64_t *full = reinterpret_cast<uint64_t *>(cst + Cfg::NCONST);
    uint64_t *empty = full + NSTAGE;
    // clusters: hfull completes once every cluster neighbour's border rows have landed in this CTA's slack rows (one phase
    // per X hand-off), hfree once every neighbour's MMAs have finished reading its X (one phase per conv): then the copies
    // of this CTA's border rows have been read, and the neighbours' slack rows may be refilled
    uint64_t *hfull = empty + NSTAGE, *hfree = hfull + 1;
    // (item, its length), read back by each phase: held in registers they would stay live across every MMA loop, and the
    // stage-0 configuration is at its register cap
    int *item_len = reinterpret_cast<int *>(empty + NSTAGE + (CS > 1 ? 2 : 0));

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // a cluster is CS consecutive CTAs along x (launch_resblock): rank crank of cluster clus of item b owns the cluster's
    // rows [crank P, (crank + 1) P).  The grid is item-major; an item's clusters never reach into the next item.  L: the
    // item's own length (every edge decision), Ls: positions between items in x and y.
    const int crank = blockIdx.x % CS;
    const RunPos cp = clusters.find(blockIdx.x / CS);
    const int clus = cp.unit, Ls = clusters.stride;
    // the weights of the item's voice: a cluster never spans two items, so every CTA of a cluster reads the same blob and
    // the chunk one rank multicasts is the one each of them expects.  Looked up where it is used (the index opaque to the
    // compiler): a pointer held across the MMA loops would cost registers the tiles need.
    auto voice_blob = [&]() {
        int c = blockIdx.x / CS;
        asm volatile("" : "+r"(c));
        return clusters.blob_at(c);
    };
    auto item = [&]() { return *reinterpret_cast<volatile int *>(&item_len[0]); };
    auto len = [&]() { return *reinterpret_cast<volatile int *>(&item_len[1]); };
    // Edge-aware tiling: a halo is only needed where the cluster (one CTA for CS = 1) borders MORE sequence.  Cluster 0
    // starts at position 0 (its left edge is the real zero padding) and keeps CS P - HALO outputs; later clusters keep
    // CS P - HALO - HL, and a cluster that reaches the end of the sequence keeps its right HALO rows too.  Cluster-internal
    // borders need no halo: the neighbours exchange their border rows of X.  A CTA whose rows all lie past the end still
    // runs the whole protocol (its neighbours write into its shared memory).
    const int oc = clus == 0 ? 0 : (CS * P - HALO) + (clus - 1) * Cfg::PVB - HL;  // position of the cluster's row 0
    const int o = oc + crank * P;                                                 // position of tile row 0
    const int p_lo = (clus == 0 || crank > 0) ? 0 : HL, p_hi = (crank < CS - 1 || oc + CS * P >= cp.len) ? P : P - HALO;
    const bool interior = (o >= 0 && o + P <= cp.len);  // every row of the tile is a real position
    // consumption order of the six convs of ResBlock `stage`: c1[0], c2[0], c1[1], c2[1], c1[2], c2[2]
    const int l0 = 5 + 6 * stage;

    if (tid == 0) {
        item_len[0] = cp.item;
        item_len[1] = cp.len;
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], Cfg::NWG * CS);  // one arrival per consumer warpgroup of every CTA of the cluster
        }
        if constexpr (CS > 1) {
            mbar_init(hfull, 1);                                     // + the bytes of the neighbours' copies
            mbar_init(hfree, (crank > 0) + (crank < CS - 1));        // one arrival per cluster neighbour
        }
        fence_mbar_init();
    }
    // (fused ConvT: the X region first holds the ConvT operand and the staging buffer; its slack rows are zeroed later)
    for (int i = Cfg::UPF ? 1 << 30 : tid; i < 2 * Cfg::KP * 2 * SLACK; i += Cfg::NT) {  // zero the slack rows of Xh and Xl
        const int r = i % (2 * SLACK), kp = (i / (2 * SLACK)) % Cfg::KP, hl = i / (2 * SLACK * Cfg::KP);
        const int row = r < SLACK ? r : P + r;  // r in [SLACK, 2*SLACK) -> rows P+SLACK .. P+2*SLACK-1
        *reinterpret_cast<uint4 *>((hl ? Xl : Xh) + kp * XPITCH + row * 16) = make_uint4(0, 0, 0, 0);
    }
    for (int i = tid; i < C; i += Cfg::NT) pend[i] = 0.f;
    // the constants come from the packed blob, not from the previous kernel: read before pdl_wait(), like the weight stream,
    // so that no global load sits between a hand-off and the next conv
    const float *packed = voice_blob();
    for (int i = tid; i < Cfg::NCONST; i += Cfg::NT) {
        float v = 0.f;
        if (i < Cfg::CB_UPF) v = __ldg(packed + bias_offset(l0) + i);  // layers l0 .. l0 + 5 have C biases each
        else if (i < Cfg::CB_UPT) v = __ldg(packed + bias_offset(1 + stage) + (i - Cfg::CB_UPF));
        else if (i < Cfg::CB_POST) v = __ldg(packed + bias_offset(1 + stage + 1) + (i - Cfg::CB_UPT));
        else if (i < Cfg::CB_POST + 32 * 8) {
            const int j = i - Cfg::CB_POST;
            if ((j & 7) < kPostK) v = __ldg(packed + weight_offset(29) + (j >> 3) * kPostK + (j & 7));
        } else if (i == Cfg::CB_POST + 32 * 8) {
            v = __ldg(packed + bias_offset(29));
        }
        cst[i] = v;
    }
    fence_proxy_async();
    __syncthreads();
    if constexpr (CS > 1) cluster_sync();  // every CTA's barriers are initialised before any remote access
    // optional timeline of one interior CTA (clock64 stamps of thread 0; see mg_gen_resblock_trace); per conv c = 0..5 the
    // slots 2 + 3c (X handed over), 3 + 3c (accumulator ready), 4 + 3c (next X written) are 2 + 6j .. 7 + 6j of conv pair j;
    // front ConvT: 21 (operand in shared memory), 22 (its MMAs done), 23 (R read back from the staging buffer); conv_post
    // epilogue: 24 (start), 26 (per-tap sums parked), 25 (audio stored)
    const bool tr = trace && blockIdx.x == (gridDim.x > 1 ? 1u : 0u) && tid == 0;
#define MG_TR(slot) do { if (tr) trace[slot] = clock64(); } while (0)

    if (warp == NCONS / 32) {
        // ================= TMA producer: streams the weight chunks through the ring in consumption order =================
        // (clusters: chunk j is read from L2 once, by rank j % CS, and multicast into the same slot of every CTA; each
        // producer still posts its own CTA's expected bytes, after its empty[s] has seen every consumer of the cluster.
        // Single pass: only the first WBYTES = HALF bytes of a chunk, its hi half, are sent and expected; of a stacked chunk,
        // whose hi rows are not contiguous, all of it.)
        if (lane == 0) {
            const uint8_t *tc_base = reinterpret_cast<const uint8_t *>(voice_blob()) + tc_region_start();
            int s = 0, ph = 0, j = 0;
            bool ok = true;
            auto put = [&](const uint8_t *src, uint32_t bytes) {
                if (!ok || !mbar_wait(&empty[s], ph ^ 1)) { ok = false; return; }
                mbar_arrive_expect_tx(&full[s], bytes);
                if constexpr (CS == 1) bulk_g2s(ring + s * CHUNK, src, bytes, &full[s]);
                else if (j % CS == crank) bulk_g2s_multicast(ring + s * CHUNK, src, bytes, &full[s], (1 << CS) - 1);
                ++j;
                if (++s == NSTAGE) { s = 0; ph ^= 1; }
            };
            if constexpr (Cfg::UPF) {  // the fused ConvT's 4 taps x UKSL K-slices, in blob order
                const uint8_t *src = tc_base + tc_upf_offset(stage);
                for (int i = 0; i < Cfg::NUPCH; ++i) put(src + (size_t)i * CHUNK, WBYTES);
            }
            for (int conv = 0; conv < 6; ++conv) {  // chunk (tap, K-slice) sits at blob index tap * KSL + ks: consumption order
                const uint8_t *src = tc_base + tc_res_offset(l0 + (conv >> 1) + 3 * (conv & 1));
                for (int i = 0; i < Cfg::NCHUNK; ++i) put(src + (size_t)i * CHUNK, WBYTES);
            }
            if constexpr (Cfg::UPT != 0) {  // the tail ConvT's B slots, in blob order [group][16-channel chunk][tap]
                const uint8_t *src = tc_base + tc_up_offset(stage + 1);
                for (int i = 0; i < Cfg::TNSLOT; ++i) put(src + (size_t)i * Cfg::TSLOT, Cfg::TSLOT);
            }
            if (!ok) atomicExch(status, 2);
        }
        if constexpr (CS > 1) cluster_sync();  // no CTA leaves while a peer may still access its shared memory
        return;
    }

    // ================= consumer warpgroups: rows of blocks [rb0, rb0 + RPW), columns [c0, c0 + NCW) =================
    const int wgi = warp >> 2, t = tid & 127, q = lane & 3;
    const int rb0 = (wgi / NCP) * RPW, c0 = (wgi % NCP) * NCW;
    const uint64_t adesc_t = desc_template(XPITCH, 128), bdesc_t = desc_template(WKP, 128);
    const uint32_t xh_addr = smem_u32(Xh), xl_addr = smem_u32(Xl), ring_addr = smem_u32(ring);
    float R[RPW][NA], D[RPW][NA];
    int s = 0, ph = 0, ps = -1;
    bool ok = true;  // a timed-out wait only raises the status word: control flow stays warpgroup-uniform
    // a slot is free once every consumer warpgroup of every CTA of the cluster has released it (thread t < CS of the
    // warpgroup arrives on CTA t's empty[], all of them in one instruction)
    auto release = [&](int slot) {
        if constexpr (CS == 1) {
            if (t == 0) mbar_arrive(&empty[slot]);
        } else if (t < CS) {
            mbar_arrive_remote(&empty[slot], t);
        }
    };
    // ring protocol: chunk_begin() waits for the next slot; chunk_end() commits its MMAs and frees the slot of the previous
    // chunk once those have completed (one group stays in flight); drain() waits for everything and frees the last slot
    auto chunk_begin = [&]() -> uint32_t {
        ok &= mbar_wait(&full[s], ph);
        acc_fence2(R);
        acc_fence2(D);
        wgmma_fence();
        return ring_addr + s * CHUNK;
    };
    auto chunk_end = [&]() {
        wgmma_commit();
        wgmma_wait<1>();
        if (ps >= 0) release(ps);
        ps = s;
        if (++s == NSTAGE) { s = 0; ph ^= 1; }
    };
    auto drain = [&]() {
        wgmma_wait<0>();
        acc_fence2(R);
        acc_fence2(D);
        if (ps >= 0) release(ps);
        ps = -1;
    };
    auto sync_cons = [&]() { named_bar_sync(1, NCONS); };
    // after a conv: every warpgroup's MMAs have read X (its slack rows included, which the neighbours may now refill);
    // thread 0 / 1 tells the left / right neighbour
    const int nbr = tid == 0 ? crank - 1 : crank + 1;
    const bool tells = tid < 2 && nbr >= 0 && nbr < CS;
    auto x_read = [&]() {
        sync_cons();
        if constexpr (CS > 1)
            if (tells) mbar_arrive_remote(hfree, nbr);
    };
    // X <- split(lrelu(A + bias)) for this warpgroup's rows and columns, zero outside [0, L); keep_last: also park the
    // fp32 lrelu(x[L-1]) in b1s (the tail ConvT's fix-up)
    auto write_x = [&](float (&A)[RPW][NA], const float *bsrc, bool keep_last) {
        const int L = len();
        // KB k-panels at a time, both rows of a fragment: their bias pairs are read before their stores.  A bias read after
        // a store to X may alias it, so one k-panel at a time ran each (load, lrelu, split, store) strictly after the
        // previous one, at shared-memory latency.  All NCW / 8 pairs at once do not fit the register budget (ptxas spills
        // in every configuration), nor do 4 in the stage-0 tile (NCP = 2), which is at its register cap
        constexpr int KB = NCP > 1 ? 2 : NCW / 8 < 4 ? NCW / 8 : 4;
#pragma unroll
        for (int r = 0; r < RPW; ++r)
#pragma unroll
            for (int k0 = 0; k0 < NCW / 8; k0 += KB) {
                float2 bb[KB];
#pragma unroll
                for (int j = 0; j < KB; ++j) bb[j] = *reinterpret_cast<const float2 *>(bsrc + c0 + 8 * (k0 + j) + 2 * q);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int p = (rb0 + r) * 64 + frag_row(t, h), tp = o + p;
                    const bool inr = interior || (tp >= 0 && tp < L);
                    uint8_t *xh = Xh + (c0 >> 3) * XPITCH + (p + SLACK) * 16 + q * 4, *xl = xh + XBYTES;
#pragma unroll
                    for (int j = 0; j < KB; ++j) {
                        const int k = k0 + j, col = c0 + 8 * k + 2 * q;
                        const float f0 = inr ? lrelu(A[r][4 * k + 2 * h] + bb[j].x) : 0.f;
                        const float f1 = inr ? lrelu(A[r][4 * k + 2 * h + 1] + bb[j].y) : 0.f;
                        uint32_t hi, lo;
                        split2_bf16(f0, f1, hi, lo);
                        *reinterpret_cast<uint32_t *>(xh + k * XPITCH) = hi;
                        if constexpr (!ONE) *reinterpret_cast<uint32_t *>(xl + k * XPITCH) = lo;
                        if (keep_last && tp == L - 1) *reinterpret_cast<float2 *>(b1s + col) = make_float2(f0, f1);
                    }
                }
            }
    };
    // clusters: the XCH rows next to a cluster-internal border (all k-panels of hi and lo; of hi only in the single-pass
    // variant) are bulk-copied into the neighbour's slack rows after every hand-off.  A thread that writes such a row first
    // waits until the neighbours' MMAs of the previous conv are done, which also means the previous copies out of this X
    // have landed.
    bool border = false;
#pragma unroll
    for (int r = 0; r < RPW; ++r)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int p = (rb0 + r) * 64 + frag_row(t, h);
            border |= (crank > 0 && p < XCH) || (crank < CS - 1 && p >= P - XCH);
        }
    constexpr int NXC = (ONE ? 1 : 2) * Cfg::KP;  // copies per border: one per k-panel of hi and lo (hi: single pass)
    constexpr uint32_t XCB = XCH * 16;      // bytes per copy
    // (a warp issues bulk copies one lane at a time: they are spread over every consumer warp, copy i by warp i % NW)
    constexpr int NW = NCONS / 32;
    auto send_halo = [&]() {
        for (int i = warp + NW * lane; i < 2 * NXC; i += NCONS) {
            const int side = i / NXC, nb = side ? crank + 1 : crank - 1;
            if (nb < 0 || nb >= CS) continue;
            const uint32_t panel = xh_addr + (i % NXC) * XPITCH;  // k-panel i % NXC of Xh, continuing into Xl
            const int src = side ? P - XCH : 0, dst = side ? -XCH : P;  // rows: mine, and the same positions in nb's tile
            bulk_s2s_cluster(mapa(panel + (SLACK + dst) * 16, nb), panel + (SLACK + src) * 16, XCB, mapa(smem_u32(hfull), nb));
        }
    };
    // X hand-off: X <- split(lrelu(A + bias)), visible to every warpgroup's MMAs (and, clusters, the neighbours')
    int hand = 0;
    auto hand_off = [&](float (&A)[RPW][NA], const float *bsrc, bool keep_last) {
        if constexpr (CS > 1) {
            if (border && hand > 0) {
                MG_TR(100 + 2 * hand);
                ok &= mbar_wait(hfree, (hand - 1) & 1);
                MG_TR(101 + 2 * hand);
            }
            if (tid == 0) mbar_arrive_expect_tx(hfull, ((crank > 0) + (crank < CS - 1)) * NXC * XCB);  // this hand-off's rows in
        }
        write_x(A, bsrc, keep_last);
        fence_proxy_async();
        sync_cons();
        if constexpr (CS > 1) send_halo();
        ++hand;
    };
    // one conv: every chunk (tap, K-slice) x NPASS passes x KC/16 k-steps x RPW row blocks.  Stacked weights, c2
    // (!fresh; a literal at both call sites): the accumulator pair is (D, R) -- D, started from zero, takes the wh
    // products and R, on top of the residual, the xh * wl^T ones -- and D is added to R once the MMAs are done.  D comes
    // first in the pair because a c1 and the xl * wh pass use it alone: ptxas keeps MMAs asynchronous only if such an
    // accumulator is the leading part of every wider one it belongs to.
    auto conv_mma = [&](float (&A)[RPW][NA], int dil, bool fresh, int conv) {
        float (&Hi)[RPW][NA] = D;
        const bool pair = PAIR && !fresh;
        if constexpr (CS > 1) {  // the neighbours' border rows of this conv's input are in the slack rows
            MG_TR(88 + 2 * conv);
            ok &= mbar_wait(hfull, conv & 1);
            MG_TR(89 + 2 * conv);
        }
        MG_TR(64 + 3 * conv);
        if (pair) {
#pragma unroll
            for (int r = 0; r < RPW; ++r)
#pragma unroll
                for (int j = 0; j < NA; ++j) Hi[r][j] = 0.f;
        }
#pragma unroll 1
        for (int ch = 0; ch < Cfg::NCHUNK; ++ch) {
            const int tap = ch / KSL, ks = ch % KSL;
            const uint64_t bbase = desc_at(bdesc_t, chunk_begin() + c0 * 16);
            if (ch == 0) MG_TR(65 + 3 * conv);
            const uint32_t arow = (SLACK + rb0 * 64 + (tap - 1) * dil) * 16 + ks * (KC / 8) * XPITCH;
            if (pair) {
#pragma unroll
                for (int k16 = 0; k16 < KC / 16; ++k16) {
                    const uint64_t bdesc = bbase + (uint64_t)((2 * k16 * WKP) >> 4);
                    const uint64_t ah = desc_at(adesc_t, xh_addr + arow + 2 * k16 * XPITCH);
                    const uint64_t al = desc_at(adesc_t, xl_addr + arow + 2 * k16 * XPITCH);
#pragma unroll
                    for (int r = 0; r < RPW; ++r)
                        wgmma_bf16_pair<PAIR ? 2 * NCW : 64>(Hi[r], A[r], ah + (uint64_t)(r * 64), bdesc, 1);
#pragma unroll
                    for (int r = 0; r < RPW; ++r) wgmma_bf16<NCW>(Hi[r], al + (uint64_t)(r * 64), bdesc, 1);
                }
            } else {
#pragma unroll
                for (int pass = 0; pass < NPASS; ++pass)
#pragma unroll
                    for (int k16 = 0; k16 < KC / 16; ++k16) {
                        const uint64_t bdesc = bbase + (uint64_t)(((pass == 2 ? WLO : 0) + 2 * k16 * WKP) >> 4);
                        const uint64_t adesc = desc_at(adesc_t, (pass == 1 ? xl_addr : xh_addr) + arow + 2 * k16 * XPITCH);
#pragma unroll
                        for (int r = 0; r < RPW; ++r)
                            wgmma_bf16<NCW>(A[r], adesc + (uint64_t)(r * 64), bdesc, !(fresh && ch == 0 && pass == 0 && k16 == 0));
                    }
            }
            chunk_end();
        }
        MG_TR(66 + 3 * conv);
        drain();
        if (pair) {
#pragma unroll
            for (int r = 0; r < RPW; ++r)
#pragma unroll
                for (int j = 0; j < NA; ++j) A[r][j] += Hi[r][j];
            acc_fence2(A);  // folded here: D is free again from this point on
        }
    };

    pdl_wait();  // x is the previous kernel's output (and y may still be read by it): every global access of this kernel is below
    MG_TR(0);
    if constexpr (Cfg::UPF) {
        constexpr int UROWS = Cfg::UROWS, UPITCH = Cfg::UPITCH, SPITCH = Cfg::SPITCH, UKSL = Cfg::UKSL;
        const int b = item(), L = len();
        const int Lin = L >> 1, Lins = Ls >> 1, s0 = (o >> 1) - 1;  // A row i <-> input position s0 + i (o is even)
        // ---- ConvT operand: A <- split(lrelu(x_in)), 2C channels of UROWS input positions; consecutive threads take
        // consecutive positions of one 8-channel k-panel.  A thread's UNR rounds of 8 loads are all issued before the
        // first is split and stored (no accumulator is live yet, so the registers are there): the loop pays one memory
        // latency, not one per round
        constexpr int UNIT = UROWS * 2 * Cfg::KP, UNR = (UNIT + NCONS - 1) / NCONS;
        static_assert(UNR * 8 <= 48, "front ConvT operand: rounds held in registers");
        float f[UNR][8];
#pragma unroll
        for (int rd = 0; rd < UNR; ++rd) {
            const int idx = tid + rd * NCONS, i = idx % UROWS, kp = idx / UROWS, sp = s0 + i;
            const bool inr = (idx < UNIT && sp >= 0 && sp < Lin);
            const float *xp = x + ((size_t)b * 2 * C + 8 * kp) * Lins + (inr ? sp : 0);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[rd][j] = inr ? __ldg(xp + (size_t)j * Lins) : 0.f;
        }
#pragma unroll
        for (int rd = 0; rd < UNR; ++rd) {
            const int idx = tid + rd * NCONS, i = idx % UROWS, kp = idx / UROWS;
            uint32_t h[4], l[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) split2_bf16(lrelu(f[rd][2 * e]), lrelu(f[rd][2 * e + 1]), h[e], l[e]);
            if (idx < UNIT) {
                *reinterpret_cast<uint4 *>(Xh + kp * UPITCH + i * 16) = make_uint4(h[0], h[1], h[2], h[3]);
                if constexpr (!ONE) *reinterpret_cast<uint4 *>(Xl + kp * UPITCH + i * 16) = make_uint4(l[0], l[1], l[2], l[3]);
            }
        }
        fence_proxy_async();
        sync_cons();
        MG_TR(21);
        // ---- ConvT MMAs: pair block wgi % NPB (warpgroups beyond NPB repeat a block and discard it: the MMA stream stays
        // free of divergent branches); odd taps feed the even outputs (R), even taps the odd ones (D)
        const uint64_t udesc_t = desc_template(UPITCH, 128);
        const bool mine = wgi < Cfg::NPB;
        const int pb = wgi % Cfg::NPB;
        auto upf_tap = [&](float (&A)[RPW][NA], int k) {
            const int rowoff = (k == 0) ? 2 : (k == 3) ? 0 : 1;  // A row i <-> input position o/2 - 1 + i
#pragma unroll 1
            for (int ks = 0; ks < UKSL; ++ks) {
                const uint64_t bbase = desc_at(bdesc_t, chunk_begin());
                const uint32_t arow = (rowoff + pb * 64) * 16 + ks * (KC / 8) * UPITCH;
#pragma unroll
                for (int pass = 0; pass < NPASS; ++pass)
#pragma unroll
                    for (int k16 = 0; k16 < KC / 16; ++k16) {
                        const uint64_t bdesc = bbase + (uint64_t)(((pass == 2 ? WLO : 0) + 2 * k16 * WKP) >> 4);
                        const uint64_t adesc = desc_at(udesc_t, (pass == 1 ? xl_addr : xh_addr) + arow + 2 * k16 * UPITCH);
                        wgmma_bf16<NCW>(A[0], adesc, bdesc, !(k < 2 && ks == 0 && pass == 0 && k16 == 0));
                    }
                chunk_end();
            }
        };
        upf_tap(D, 0);  // blob order: tap 0, 1, 2, 3, each over its UKSL K-slices
        upf_tap(R, 1);
        upf_tap(D, 2);
        upf_tap(R, 3);
        drain();
        MG_TR(22);
        sync_cons();  // every ConvT MMA has read the operand: the region becomes the fp32 staging buffer [c][p]
        float *stg = reinterpret_cast<float *>(Xh);
        const float *ubias = cst + Cfg::CB_UPF;
        if (mine) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = wgi * 64 + frag_row(t, h);
#pragma unroll
                for (int j = 0; j < NA; ++j) {
                    const int col = frag_col(q, (j & ~3) | (j & 1));
                    if ((j & 2) == 2 * h) {
                        const float bj = ubias[col];
                        *reinterpret_cast<float2 *>(stg + (size_t)col * SPITCH + 2 * m) = make_float2(R[0][j] + bj, D[0][j] + bj);
                    }
                }
            }
        }
        sync_cons();
        // ---- R <- ConvT output (row = output position), then X <- split(lrelu(x)) exactly like after a c2 (pend = 0)
#pragma unroll
        for (int r = 0; r < RPW; ++r)
#pragma unroll
            for (int j = 0; j < NA; ++j) {
                const int p = (rb0 + r) * 64 + frag_row(t, (j >> 1) & 1);
                R[r][j] = stg[(size_t)frag_col(q, (j & ~3) | (j & 1)) * SPITCH + p];
            }
        sync_cons();  // every staging read is done: the region becomes X
        MG_TR(23);
        for (int i = tid; i < 2 * Cfg::KP * 2 * SLACK; i += NCONS) {  // zero the slack rows of Xh and Xl
            const int r = i % (2 * SLACK), kp = (i / (2 * SLACK)) % Cfg::KP, hl = i / (2 * SLACK * Cfg::KP);
            const int row = r < SLACK ? r : P + r;
            *reinterpret_cast<uint4 *>((hl ? Xl : Xh) + kp * XPITCH + row * 16) = make_uint4(0, 0, 0, 0);
        }
    } else {
        // ---- load the input tile: R <- x (fp32, exact), X <- split(lrelu(x))
        const int b = item(), L = len();
#pragma unroll
        for (int r = 0; r < RPW; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = (rb0 + r) * 64 + frag_row(t, h), tp = o + p;
                const bool inr = (tp >= 0 && tp < L);
                const float *xp = x + (size_t)b * C * Ls + (inr ? tp : 0);
#pragma unroll
                for (int k = 0; k < NCW / 8; ++k)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        R[r][4 * k + 2 * h + e] = inr ? __ldg(xp + (size_t)(c0 + frag_col(q, 4 * k + e)) * Ls) : 0.f;
            }
    }
    hand_off(R, pend, false);  // (pend is still all zeros)
    MG_TR(1);

#pragma unroll 1
    for (int pr = 0; pr < 3; ++pr) {
        // ---- c1 (dilation 1, 3, 9) into D, then X <- split(lrelu(D + b1))
        MG_TR(2 + 6 * pr);
        conv_mma(D, pr == 0 ? 1 : pr == 1 ? 3 : 9, true, 2 * pr);
        MG_TR(3 + 6 * pr);
        x_read();
        hand_off(D, cst + pr * C, false);
        MG_TR(4 + 6 * pr);
        // ---- c2 (dilation 1) accumulating onto R, then X <- split(lrelu(R + pend)) for the next c1 (or the tail ConvT)
        for (int c = tid; c < C; c += NCONS) pend[c] += cst[(3 + pr) * C + c];
        MG_TR(5 + 6 * pr);
        conv_mma(R, 1, false, 2 * pr + 1);
        MG_TR(6 + 6 * pr);
        x_read();
        if (pr < 2 || Cfg::UPT != 0) hand_off(R, pend, Cfg::UPT != 0 && pr == 2);
        MG_TR(7 + 6 * pr);
    }

    if constexpr (Cfg::POST) {
        // ---- fused LeakyReLU -> conv_post (32 -> 1, k7, pad 3) -> tanh (models.py:67-69); y is audio [B][1][L].
        // Each position turns its 32 channels into the 7 per-tap partial sums q_k[p] = sum_ci w[ci][k] * lrelu(x[ci][p])
        // (the four threads that share a row add their columns' parts), parks them in shared memory (the X buffer is dead
        // now), then audio[p] = tanh(b + sum_k q_k[p + k - 3]).
        pdl_trigger();
        MG_TR(24);
        float *Q = reinterpret_cast<float *>(Xh);      // [7][P]
        const float *wpost = cst + Cfg::CB_POST;        // [32][8]
        // A thread holds 8 channels of NR = 4 rows.  Channel outermost: its 7 weights and its bias are read once and
        // applied to the four rows (per row the sum runs over the channels in the same order as row by row).
        constexpr int NR = 2 * RPW;
        static_assert(NR == 4, "conv_post epilogue: four rows per thread, one per lane of a quad after the reduction");
        float qk[NR][kPostK];
        bool inr[NR];
        {
            const int L = len();
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                const int tp = o + (rb0 + (i >> 1)) * 64 + frag_row(t, i & 1);
                inr[i] = (tp >= 0 && tp < L);
#pragma unroll
                for (int k = 0; k < kPostK; ++k) qk[i][k] = 0.f;
            }
        }
#pragma unroll
        for (int k = 0; k < NCW / 8; ++k)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int ci = frag_col(q, 4 * k + e);
                const float pe = pend[ci];
                const float4 w0 = *reinterpret_cast<const float4 *>(wpost + ci * 8);
                const float4 w1 = *reinterpret_cast<const float4 *>(wpost + ci * 8 + 4);
#pragma unroll
                for (int i = 0; i < NR; ++i) {
                    const float a = inr[i] ? lrelu(R[i >> 1][4 * k + 2 * (i & 1) + e] + pe) : 0.f;
                    qk[i][0] = fmaf(w0.x, a, qk[i][0]); qk[i][1] = fmaf(w0.y, a, qk[i][1]); qk[i][2] = fmaf(w0.z, a, qk[i][2]);
                    qk[i][3] = fmaf(w0.w, a, qk[i][3]); qk[i][4] = fmaf(w1.x, a, qk[i][4]); qk[i][5] = fmaf(w1.y, a, qk[i][5]);
                    qk[i][6] = fmaf(w1.z, a, qk[i][6]);
                }
            }
        // The four lanes of a quad add their parts, (q0 + q1) + (q2 + q3) per row and tap.  Each step hands half of the
        // values to the partner lane instead of exchanging all of them: after lane ^ 1 the odd lanes keep rows 2, 3 and
        // the even ones rows 0, 1; after lane ^ 2 lane q holds the finished sums of row 2 (q & 1) + (q >> 1) -- 21
        // shuffles per thread instead of 56, and every lane stores one row.
        const bool odd = q & 1, up = q & 2;
        float s1[2][kPostK], s2[kPostK];
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int k = 0; k < kPostK; ++k) {
                const float keep = odd ? qk[j + 2][k] : qk[j][k], send = odd ? qk[j][k] : qk[j + 2][k];
                s1[j][k] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
            }
#pragma unroll
        for (int k = 0; k < kPostK; ++k) {
            const float keep = up ? s1[1][k] : s1[0][k], send = up ? s1[0][k] : s1[1][k];
            s2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        {
            const int i = 2 * (q & 1) + (q >> 1), p = (rb0 + (i >> 1)) * 64 + frag_row(t, i & 1);
#pragma unroll
            for (int k = 0; k < kPostK; ++k) Q[k * P + p] = s2[k];
        }
        MG_TR(26);
        sync_cons();
        const int b = item(), L = len();
        const float bpost = cst[Cfg::CB_POST + 32 * 8];
#pragma unroll 1
        for (int p = tid; p < P; p += NCONS) {
            const int tp = o + p;
            if (p >= p_lo && p < p_hi && tp < L) {
                float acc = bpost;
#pragma unroll
                for (int k = 0; k < kPostK; ++k) {
                    const int pp = p + k - 3;  // outside the tile only where it is outside the sequence too (zero padding)
                    if (pp >= 0 && pp < P) acc += Q[k * P + pp];
                }
                y[(size_t)b * Ls + tp] = audio_sample<typename Cfg::Out>(tanhf(acc));
            }
        }
        if (oc + P >= L)  // the item's last CTA: the audio past the item's end reads 0 (ragged batches)
            for (int p = L + tid; p < Ls; p += NCONS) y[(size_t)b * Ls + p] = 0;
        MG_TR(25);
    } else if constexpr (Cfg::UPT != 0) {
        // ---- tail ConvT: D[s, phi*TNG + co] (+)= X[s - tap, :] * Wstack_tap^T over the C channels of X = split(lrelu(x_out))
        constexpr int S = Cfg::UPT, TNG = Cfg::TNG, TN = Cfg::TN, PADT = S / 2, COT = C / 2;
        const int b = item(), L = len();
        const int Lout = S * Ls;  // output positions between items
        const float *tbias = cst + Cfg::CB_UPT;
        // ---- fix-up first (it only needs b1s[]): out[co][S L - pad + j] = bias + sum_ci lrelu(x[ci][L-1]) * W[ci][co][j + S],
        // j < pad (the outputs position L would own: x[L] = 0 leaves only the x[L-1] tap), by the CTA whose owned rows include
        // position L - 1.  fp32 FFMA on the fp32 copy of the ConvT weights ([Cin][Cout][S][2], mg_layout.h).
        {
            const int pl = L - 1 - o;  // tile-local row of position L - 1
            if (pl >= p_lo && pl < p_hi) {  // CTA-uniform; b1s[] was written before the last hand-off's barrier
                const float *wf = voice_blob() + weight_offset(1 + stage + 1);
                for (int i = tid; i < PADT * COT; i += NCONS) {
                    const int co = i / PADT, j = i - co * PADT;
                    const float *wp = wf + ((size_t)co * S + j) * 2 + 1;  // + ci * COT * S * 2
                    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
#pragma unroll 1
                    for (int cc = 0; cc < C; cc += 32) {  // 32 weights in flight per round trip
                        float wv[32];
#pragma unroll
                        for (int k = 0; k < 32; ++k) wv[k] = __ldg(wp + (size_t)(cc + k) * COT * S * 2);
#pragma unroll
                        for (int k = 0; k < 32; k += 4) {
                            acc0 = fmaf(b1s[cc + k], wv[k], acc0);
                            acc1 = fmaf(b1s[cc + k + 1], wv[k + 1], acc1);
                            acc2 = fmaf(b1s[cc + k + 2], wv[k + 2], acc2);
                            acc3 = fmaf(b1s[cc + k + 3], wv[k + 3], acc3);
                        }
                    }
                    y[((size_t)b * COT + co) * Lout + (size_t)S * L - PADT + j] = (acc0 + acc1) + (acc2 + acc3) + tbias[co];
                }
            }
        }
        const uint64_t tbdesc_t = desc_template(TN * 16, 128);
#pragma unroll 1
        for (int cg = 0; cg < Cfg::TNCG; ++cg) {
#pragma unroll 1
            for (int ch = 0; ch < C / 16; ++ch) {
#pragma unroll 1
                for (int ts = 0; ts < (S == 8 ? 2 : 1); ++ts) {  // stride 8: one ring slot per tap
                    const uint64_t bbase = desc_at(tbdesc_t, chunk_begin() + c0 * 16);
#pragma unroll
                    for (int tp = 0; tp < (S == 8 ? 1 : 2); ++tp) {
                        const int tap = S == 8 ? ts : tp;  // tap 0 reads x[s], tap 1 x[s - 1]: the same buffer one row earlier
#pragma unroll
                        for (int pass = 0; pass < 3; ++pass) {
                            const uint32_t boff = (uint32_t)((((S == 8 ? 0 : tp * 2) + (pass == 2 ? 1 : 0)) * 2) * TN * 16);
                            const uint64_t bdesc = bbase + (uint64_t)(boff >> 4);
                            const uint32_t arow = (uint32_t)((SLACK + rb0 * 64 - tap) * 16 + 2 * ch * XPITCH);
                            const uint64_t adesc = desc_at(adesc_t, (pass == 1 ? xl_addr : xh_addr) + arow);
#pragma unroll
                            for (int r = 0; r < RPW; ++r)
                                wgmma_bf16<NCW>(D[r], adesc + (uint64_t)(r * 64), bdesc, !(ch == 0 && tap == 0 && pass == 0));
                        }
                    }
                    chunk_end();
                }
            }
            drain();
            if (cg == Cfg::TNCG - 1) pdl_trigger();
            // ---- this group's outputs: the thread of input position s stores [S s - pad, S s - pad + S) of its channels
#pragma unroll
            for (int r = 0; r < RPW; ++r)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int p = (rb0 + r) * 64 + frag_row(t, h), sg = o + p;  // sg: global input position
                    const bool own = (p >= p_lo && p < p_hi && sg < L);
                    const bool lo_ok = own && sg >= 1, hi_ok = own;
                    if constexpr (S == 8) {
                        // column c0 + 8k + 2q + e = phi * 32 + co: this column part holds phases 4 (c0 / 128) .. + 3
                        const bool ok8 = c0 == 0 ? lo_ok : hi_ok;
                        float *yb = y + ((size_t)b * COT + cg * TNG) * Lout + (own ? 8 * sg - PADT + (c0 >> 5) : 0);
#pragma unroll
                        for (int c = 0; c < 4; ++c)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int co = 8 * c + 2 * q + e;
                                const float bj = tbias[cg * TNG + co];
                                if (ok8)
                                    *reinterpret_cast<float4 *>(yb + (size_t)co * Lout) =
                                        make_float4(D[r][4 * c + 2 * h + e] + bj, D[r][4 * (4 + c) + 2 * h + e] + bj,
                                                    D[r][4 * (8 + c) + 2 * h + e] + bj, D[r][4 * (12 + c) + 2 * h + e] + bj);
                            }
                    } else {
                        float *yb = y + (size_t)b * COT * Lout + (own ? 2 * sg - PADT : 0);
#pragma unroll
                        for (int k = 0; k < NCW / 8; ++k)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int col = c0 + frag_col(q, 4 * k + e), phi = col / TNG, co = col % TNG;
                                if (phi == 0 ? lo_ok : hi_ok) yb[(size_t)co * Lout + phi] = D[r][4 * k + 2 * h + e] + tbias[co];
                            }
                    }
                }
        }
    } else {
        // ---- store the valid part of R + pend
        pdl_trigger();
        const int b = item(), L = len();
#pragma unroll
        for (int r = 0; r < RPW; ++r)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = (rb0 + r) * 64 + frag_row(t, h), tp = o + p;
                if (p >= p_lo && p < p_hi && tp < L) {
                    float *yp = y + (size_t)b * C * Ls + tp;
#pragma unroll
                    for (int k = 0; k < NCW / 8; ++k)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = c0 + frag_col(q, 4 * k + e);
                            yp[(size_t)col * Ls] = R[r][4 * k + 2 * h + e] + pend[col];
                        }
                }
            }
    }
    if (!ok && t == 0) atomicExch(status, 3);
    if constexpr (CS > 1) cluster_sync();  // no CTA leaves while a peer may still access its shared memory
    MG_TR(20);
#undef MG_TR
}

template <class Cfg>
static int launch_resblock(const float *x, typename Cfg::Out *y, int stage, const RunTable &batch, int *status,
                           long long *trace, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(resblock_tc_kernel<Cfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        configured = true;
    }
    constexpr int CS = Cfg::CS, PC = CS * Cfg::P, PVB = Cfg::PVB;  // edge-aware tiling of CS * P-position clusters, see the kernel
    RunTable clusters = batch;
    clusters.set_units([](int L) { return 1 + (L > PC ? (L - PC + PVB - 1) / PVB : 0); });
    const dim3 grid(CS * clusters.first[clusters.n]);
    if (trace && CS > 1) {  // diagnostic: clusters resident at once (GPC boundaries can leave SMs idle), into trace[127]
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = grid;
        cfg.blockDim = dim3(Cfg::NT);
        cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = CS;
        attr.val.clusterDim.y = attr.val.clusterDim.z = 1;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        int n = 0;
        MG_CUDA_TRY(cudaOccupancyMaxActiveClusters(&n, resblock_tc_kernel<Cfg>, &cfg));
        const long long v = n;
        MG_CUDA_TRY(cudaMemcpy(trace + 127, &v, sizeof(v), cudaMemcpyHostToDevice));
    }
    MG_CUDA_TRY(launch_ex(resblock_tc_kernel<Cfg>, grid, dim3(Cfg::NT), Cfg::SMEM_BYTES, s, true, CS, x, reinterpret_cast<float *>(y),
                          stage, clusters, status, trace));
    return MG_OK;
}

template <class Cfg>
static const char *cfg_name() {
    static char buf[96];
    snprintf(buf, sizeof(buf), "resblock_tc_kernel<RbCfg<%d,%d,%d,%d,%d,%d,%d,%d,%d>>", Cfg::C, Cfg::NRB, Cfg::RPW, Cfg::NCP,
             Cfg::NSTAGE, (int)Cfg::POST, (int)Cfg::UPF, Cfg::UPT, Cfg::CS);
    return buf;
}

// Configurations per stage code (C, 64-row blocks, blocks per warpgroup, column parts, ring slots): the tile is as long as
// the register file allows (R and D of every position and channel: 2 * P * C floats), at one CTA per SM.  Stages 0 and 1
// run as clusters (the last parameter; H100 80GB HBM3, config 2): stage 0 as 4 CTAs = 256 positions, one cluster per item
// at L = 256 instead of 7 halo-overlapped tiles; stage 1 as pairs, 18 CTAs per item at L = 2048 instead of 21 (4-CTA
// clusters would need 20).
// stage 0..3: ResBlock `stage`; 4: ResBlock 3 with LeakyReLU -> conv_post -> tanh fused (y is the audio [B][1][L]);
// 12 / 13 / 14 = stages 2 / 3 / 3+post with the stage's stride-2 ConvT fused in front (x is the PREVIOUS stage's output
// [B][2C][L/2], L stays the output length); 20 / 21 / 22 = ResBlock 0 / 1 / 2 with the NEXT stage's LeakyReLU -> ConvT
// at its tail (y is [B][C/2][S L]).
using Rb0 = RbCfg<256, 1, 1, 2, 4, false, false, 0, 4>;
using Rb1 = RbCfg<128, 2, 1, 1, 4, false, false, 0, 2>;
using Rb2 = RbCfg<64, 4, 1, 1, 3>;
using Rb3 = RbCfg<32, 8, 2, 1, 4>;
using Rb3Post = RbCfg<32, 8, 2, 1, 4, true>;
using Up2Rb2 = RbCfg<64, 4, 1, 1, 3, false, true>;
using Up3Rb3 = RbCfg<32, 8, 2, 1, 4, false, true>;
using Up3Rb3Post = RbCfg<32, 8, 2, 1, 4, true, true>;
using Rb0Up1 = RbCfg<256, 1, 1, 2, 4, false, false, 8>;
using Rb1Up2 = RbCfg<128, 2, 1, 1, 4, false, false, 2>;
using Rb2Up3 = RbCfg<64, 4, 1, 1, 3, false, false, 2>;

// x, y: [B][C][L] fp32 NCL with C = 256 >> stage, L = batch.stride, item i's first len_i positions its own; status: device
// int, set non-zero if a pipeline wait timed out.  precision MG_GEN_PRECISION_BF16: the single-pass variant, which exists
// for the default chain's stage codes 0, 1, 2 and 14.
int launch_resblock_tc(const float *x, float *y, int stage, const RunTable &batch, int *status, cudaStream_t s,
                       long long *trace, int precision) {
    if (precision == MG_GEN_PRECISION_BF16) {
        switch (stage) {
            case 0: return launch_resblock<Bf16<Rb0>>(x, y, 0, batch, status, trace, s);
            case 1: return launch_resblock<Bf16<Rb1>>(x, y, 1, batch, status, trace, s);
            case 2: return launch_resblock<Bf16<Rb2>>(x, y, 2, batch, status, trace, s);
            case 14: return launch_resblock<Bf16<Up3Rb3Post>>(x, y, 3, batch, status, trace, s);
        }
        return set_error(MG_ERR_INVALID_ARGUMENT, "launch_resblock_tc: stage code %d has no bf16 variant", stage);
    }
    if (precision != MG_GEN_PRECISION_FP32)
        return set_error(MG_ERR_INVALID_ARGUMENT, "launch_resblock_tc: precision %d", precision);
    switch (stage) {
        case 0: return launch_resblock<Rb0>(x, y, 0, batch, status, trace, s);
        case 1: return launch_resblock<Rb1>(x, y, 1, batch, status, trace, s);
        case 2: return launch_resblock<Rb2>(x, y, 2, batch, status, trace, s);
        case 3: return launch_resblock<Rb3>(x, y, 3, batch, status, trace, s);
        case 4: return launch_resblock<Rb3Post>(x, y, 3, batch, status, trace, s);
        case 12: return launch_resblock<Up2Rb2>(x, y, 2, batch, status, trace, s);
        case 13: return launch_resblock<Up3Rb3>(x, y, 3, batch, status, trace, s);
        case 14: return launch_resblock<Up3Rb3Post>(x, y, 3, batch, status, trace, s);
        case 20: return launch_resblock<Rb0Up1>(x, y, 0, batch, status, trace, s);
        case 21: return launch_resblock<Rb1Up2>(x, y, 1, batch, status, trace, s);
        case 22: return launch_resblock<Rb2Up3>(x, y, 2, batch, status, trace, s);
    }
    return set_error(MG_ERR_INVALID_ARGUMENT, "launch_resblock_tc: stage %d", stage);
}

// the default chain's last kernel (stage code 14) with int16 audio y [B][1][L]: pcm16 of what launch_resblock_tc(.., 14, ..)
// stores at the same precision
int launch_resblock_tc_pcm16(const float *x, int16_t *y, const RunTable &batch, int *status, cudaStream_t s, int precision) {
    if (precision == MG_GEN_PRECISION_FP32) return launch_resblock<Pcm16<Up3Rb3Post>>(x, y, 3, batch, status, nullptr, s);
    if (precision == MG_GEN_PRECISION_BF16) return launch_resblock<Pcm16<Bf16<Up3Rb3Post>>>(x, y, 3, batch, status, nullptr, s);
    return set_error(MG_ERR_INVALID_ARGUMENT, "launch_resblock_tc_pcm16: precision %d", precision);
}

// the configuration launch_resblock_tc runs for a stage code (evidence files record it)
const char *resblock_config_name(int stage, int L) {
    (void)L;
    switch (stage) {
        case 0: return cfg_name<Rb0>();
        case 1: return cfg_name<Rb1>();
        case 2: return cfg_name<Rb2>();
        case 3: return cfg_name<Rb3>();
        case 4: return cfg_name<Rb3Post>();
        case 12: return cfg_name<Up2Rb2>();
        case 13: return cfg_name<Up3Rb3>();
        case 14: return cfg_name<Up3Rb3Post>();
        case 20: return cfg_name<Rb0Up1>();
        case 21: return cfg_name<Rb1Up2>();
        case 22: return cfg_name<Rb2Up3>();
    }
    return "";
}

}  // namespace mg
