// Generator layer table and the packed-weight layout (host + device).
//
// Layer order is the reference's registration order (models.py:46-59):
//   0 conv_pre | 1..4 ups[0..3] | 5+6i+j resblocks[i].convs1[j] | 5+6i+3+j resblocks[i].convs2[j] | 29 conv_post
//
// Packed layouts (what the kernels stream; all fp32, folded w = g*v/||v||):
//   Conv1d  [Cout][Cin][K]  ->  [Cin][K][Cout]      (Cout contiguous: a chunk of input channels is
//                                                    one contiguous block, co-vectors are float4-loadable)
//   ConvT1d [Cin][Cout][K]  ->  [Cin][Cout][S][2]   (K = 2S; the two taps (phase, phase+S) that reach one
//                                                    output phase sit side by side)
//   conv_post [1][32][7]    ->  [32][7]             (same as raw; Cout = 1)
//   biases: concatenated in layer order after the weights.
#pragma once
#include <stddef.h>

#ifndef MG_HD
#ifdef __CUDACC__
#define MG_HD __host__ __device__
#else
#define MG_HD
#endif
#endif

namespace mg {

constexpr int kNumLayers = 30;
constexpr int kMelBins = 80;
constexpr int kPreCout = 512;
constexpr int kPreK = 7;
constexpr int kPostK = 7;
constexpr float kSlope = 0.01f;  // F.leaky_relu default (models.py:35,37,64,67)

struct LayerShape {
    int kind;  // 0 = Conv1d, 1 = ConvTranspose1d
    int cin, cout, k;
    int stride;  // ConvT only
};

MG_HD constexpr int stage_cin(int i) { return 512 >> i; }
MG_HD constexpr int stage_cout(int i) { return 256 >> i; }
MG_HD constexpr int stage_stride(int i) { return i < 2 ? 8 : 2; }
MG_HD constexpr int stage_kup(int i) { return i < 2 ? 16 : 4; }
MG_HD constexpr int stage_pad(int i) { return i < 2 ? 4 : 1; }
// cumulative upsampling factor after stage i: 8, 64, 128, 256
MG_HD constexpr int stage_upfactor(int i) { return i == 0 ? 8 : i == 1 ? 64 : i == 2 ? 128 : 256; }

MG_HD constexpr LayerShape layer_shape(int l) {
    if (l == 0) return {0, kMelBins, kPreCout, kPreK, 1};
    if (l <= 4) return {1, stage_cin(l - 1), stage_cout(l - 1), stage_kup(l - 1), stage_stride(l - 1)};
    if (l <= 28) return {0, stage_cout((l - 5) / 6), stage_cout((l - 5) / 6), 3, 1};
    return {0, 32, 1, kPostK, 1};
}
MG_HD constexpr int layer_dilation(int l) {  // only meaningful for resblock convs
    return (l >= 5 && l <= 28 && ((l - 5) % 6) < 3) ? (((l - 5) % 6) == 0 ? 1 : ((l - 5) % 6) == 1 ? 3 : 9) : 1;
}
MG_HD constexpr size_t layer_weight_count(int l) {
    return (size_t)layer_shape(l).cin * layer_shape(l).cout * layer_shape(l).k;
}
// rows of the weight-norm (dim 0 of weight_v): Cout for Conv1d, Cin for ConvTranspose1d
MG_HD constexpr int layer_norm_rows(int l) { return layer_shape(l).kind == 0 ? layer_shape(l).cout : layer_shape(l).cin; }

MG_HD constexpr size_t weight_offset(int l) {  // in floats
    size_t o = 0;
    for (int i = 0; i < l; ++i) o += layer_weight_count(i);
    return o;
}
MG_HD constexpr size_t total_weight_count() { return weight_offset(kNumLayers); }
MG_HD constexpr size_t bias_offset(int l) {  // in floats, from the start of the blob
    size_t o = total_weight_count();
    for (int i = 0; i < l; ++i) o += (size_t)layer_shape(i).cout;
    return o;
}
MG_HD constexpr size_t packed_float_count() { return bias_offset(kNumLayers); }

static_assert(packed_float_count() == 4524290 - 4353, "packed blob = all G params minus the weight_g scalars");

// ---- tensor-core (split-bf16) blob for the 24 ResBlock convs -------------------------------------------
// Appended to the fp32 blob.  Per conv (C channels, 3 taps): chunks of KC input channels in consumption order
//   [tap][kslice = ci/KC][half: hi, lo][k-panel = (ci%KC)/8][co][ci%8]   (bf16)
// so one (tap, kslice) chunk -- hi and lo halves back to back -- is one contiguous bulk copy, and inside a
// half the layout is the "row-linear K-major" operand layout of mg_tc.cuh with rows = output channels.
// C <= 64 (tc_stacked; stages 2 and 3 and their fused front ConvT below): the halves are interleaved per k-panel,
//   [tap][kslice][k-panel][half: hi, lo][co][ci%8]
// so the 2 C rows of a k-panel -- hi rows [0, C), lo rows [C, 2 C) -- are one operand of N = 2 C with a panel pitch
// (LBO) of 2 C * 16 bytes: one MMA multiplies the activations by [wh | wl], and the same descriptor at N = C reads wh
// alone.  Chunk size, chunk order and every offset below are the same for both layouts.
MG_HD constexpr int tc_kc(int C) { return C >= 128 ? 4096 / C : C; }          // 256:16, 128:32, 64:64, 32:32
MG_HD constexpr bool tc_stacked(int C) { return C <= 64; }
// bf16 element index inside a chunk of KC input channels x C output rows
MG_HD constexpr size_t tc_in_chunk_index(int C, int co, int cik, int h) {  // cik = ci % KC
    const int KC = tc_kc(C);
    return tc_stacked(C) ? (((size_t)(cik / 8) * 2 + h) * C + co) * 8 + (cik % 8)
                         : (((size_t)h * (KC / 8) + cik / 8) * C + co) * 8 + (cik % 8);
}
MG_HD constexpr int tc_chunk_bytes(int C) { return 4 * C * tc_kc(C); }          // hi + lo halves
MG_HD constexpr int tc_chunks_per_conv(int C) { return 3 * C / tc_kc(C); }
MG_HD constexpr size_t tc_conv_bytes(int C) { return (size_t)12 * C * C; }
MG_HD constexpr size_t tc_res_offset(int l) {  // bytes from the start of the TC region, l in [5, 28]
    size_t o = 0;
    for (int i = 5; i < l; ++i) o += tc_conv_bytes(layer_shape(i).cout);
    return o;
}
// ---- tensor-core blob for the 4 ConvTranspose1d layers (after the ResBlock convs) -----------------------
// out[t] = sum_ci x[s]*W[ci][co][phi] + x[s-1]*W[ci][co][phi+S], phi = (t+pad) mod S: per output phase a
// 2-tap conv on the INPUT positions.  All S phases of a tap read the SAME activation rows, so they are stacked along
// the MMA N dimension (N = S*NG <= 256: one instruction per (tap, pass) covers every phase).  One ring slot =
// (co-group, 16-channel K chunk):
//   [cg][chunk = ci/16][tap][half: hi, lo][k-panel = (ci%16)/8][row = phi*NG + co%NG][ci % 8]   (bf16), 128*S*NG bytes
MG_HD constexpr int up_ng(int stage) { return stage == 2 ? 64 : 32; }  // output channels per CTA (S*NG = 256,256,128,64)
MG_HD constexpr int up_slot_bytes(int stage) { return 128 * stage_stride(stage) * up_ng(stage); }
MG_HD constexpr size_t up_tc_bytes(int stage) {  // = Cin*Cout*K*4 (hi + lo)
    return (size_t)stage_cin(stage) * stage_cout(stage) * stage_kup(stage) * 4;
}
MG_HD constexpr size_t tc_up_offset(int stage) {  // bytes from the start of the TC region
    size_t o = tc_res_offset(29);
    for (int i = 0; i < stage; ++i) o += up_tc_bytes(i);
    return o;
}
MG_HD constexpr size_t up_weight_index(int stage, int ci, int co, int k, int h) {  // bf16 element index in the layer's block
    const int S = stage_stride(stage), NG = up_ng(stage), CIN = stage_cin(stage);
    const int phi = k % S, tap = k / S;
    return (((((size_t)(co / NG) * (CIN / 16) + ci / 16) * 2 + tap) * 2 + h) * 2 + (ci % 16) / 8) * (S * NG) * 8 +
           (size_t)(phi * NG + co % NG) * 8 + (ci % 8);
}
// ---- tensor-core blob for stride-1 dense convs run by conv_rows_tc_kernel (mg_conv_tc.cu): conv_pre here, the
// discriminators' conv_post1 in their own blob.  One ring slot = (NG-channel output group, 16-channel K chunk, tap):
//   [cg = co/NG][chunk = ci/16][tap][half: hi, lo][k-panel = (ci%16)/8][co%NG][ci%8]   (bf16), 64 NG bytes per slot
constexpr int kPreNG = 128;    // conv_pre: 512 output channels = 4 groups (an N = 256 register tile does not fit beside the converter)
constexpr int kPost1NG = 128;  // conv_post1: 8 groups of 128 -> twice the CTAs of a 256-wide split at the same MMA efficiency
MG_HD constexpr size_t conv_tc_weight_index(int CIN, int NTAP, int NG, int co, int ci, int tap, int h) {
    return (((((size_t)(co / NG) * (CIN / 16) + ci / 16) * NTAP + tap) * 2 + h) * 2 + (ci % 16) / 8) * NG * 8 +
           (size_t)(co % NG) * 8 + (ci % 8);
}
MG_HD constexpr size_t tc_pre_offset() { return tc_up_offset(4); }
MG_HD constexpr size_t tc_pre_bytes() { return (size_t)kMelBins * kPreCout * kPreK * 4; }
// ---- stride-2 ConvT fused into the ResBlock kernel (stages 2, 3; mg_res_tc.cu, UPF): the four taps W_k[co][ci] are four
// "conv taps" over the 2C input channels, chunked exactly like a ResBlock conv of C output channels:
//   [tap k][kslice = ci/KC][k-panel = (ci%KC)/8][half: hi, lo][co][ci%8]   (bf16), chunk = tc_chunk_bytes(C)
// (C = 64 and 32: the stacked in-chunk order of tc_in_chunk_index)
MG_HD constexpr int upf_chunks(int C) { return 4 * (2 * C / tc_kc(C)); }
MG_HD constexpr size_t upf_bytes(int stage) { return (size_t)upf_chunks(stage_cout(stage)) * tc_chunk_bytes(stage_cout(stage)); }
MG_HD constexpr size_t tc_upf_offset(int stage) {  // stage 2 or 3; bytes from the start of the TC region
    return tc_pre_offset() + tc_pre_bytes() + (stage == 3 ? upf_bytes(2) : 0);
}
MG_HD constexpr size_t upf_weight_index(int C, int ci, int co, int k, int h) {  // bf16 element index in the stage's block
    const int KC = tc_kc(C);
    return (size_t)(k * (2 * C / KC) + ci / KC) * (2 * KC * C) + tc_in_chunk_index(C, co, ci % KC, h);
}
MG_HD constexpr size_t tc_region_bytes() { return tc_upf_offset(3) + upf_bytes(3); }
MG_HD constexpr size_t packed_total_bytes() { return ((packed_float_count() * 4 + 255) / 256) * 256 + tc_region_bytes(); }
MG_HD constexpr size_t tc_region_start() { return ((packed_float_count() * 4 + 255) / 256) * 256; }  // bytes
// element (bf16) index of w[co][ci][tap] (half h) inside its conv's TC block
MG_HD constexpr size_t tc_weight_index(int C, int co, int ci, int tap, int h) {
    const int KC = tc_kc(C);
    return (size_t)(tap * (C / KC) + ci / KC) * (2 * KC * C) + tc_in_chunk_index(C, co, ci % KC, h);
}

// =========================================================================================================
// Discriminator (models.py:74-103) layer table and packed layout.  7 layers per Discriminator, 3 per MSD:
//   0 conv_pre 1->16 k15 | 1..4 grouped k41 (groups 4,16,64,256; stride 4,4,4,1) | 5 conv_post1 1024->1024 k5 | 6 conv_post2 1024->1 k3
struct DLayer {
    int cin, cout, k, stride, groups, pad;
};
MG_HD constexpr DLayer d_layer(int l) {
    return l == 0 ? DLayer{1, 16, 15, 1, 1, 7}
         : l == 1 ? DLayer{16, 64, 41, 4, 4, 20}
         : l == 2 ? DLayer{64, 256, 41, 4, 16, 20}
         : l == 3 ? DLayer{256, 1024, 41, 4, 64, 20}
         : l == 4 ? DLayer{1024, 1024, 41, 1, 256, 20}
         : l == 5 ? DLayer{1024, 1024, 5, 1, 1, 2}
                  : DLayer{1024, 1, 3, 1, 1, 1};
}
constexpr int kDiscLayers = 7;
constexpr int kDiscRows = 16 + 64 + 256 + 1024 + 1024 + 1024 + 1;  // weight-norm rows (= biases) per Discriminator
// fp32 part of one Discriminator's blob (floats).  Layouts:
//   conv_pre   [tap 15][co 16]            grouped l=1..4  [group][ci 4][tap 41][co within group]      conv_post2 [ci 1024][tap 3]
MG_HD constexpr size_t d_weight_count(int l) {
    return l == 5 ? 0 : (size_t)d_layer(l).cout * (d_layer(l).cin / d_layer(l).groups) * d_layer(l).k;
}
MG_HD constexpr size_t d_weight_offset(int l) {
    size_t o = 0;
    for (int i = 0; i < l; ++i) o += d_weight_count(i);
    return o;
}
MG_HD constexpr size_t d_bias_offset(int l) {
    size_t o = d_weight_offset(kDiscLayers);
    for (int i = 0; i < l; ++i) o += (size_t)d_layer(i).cout;
    return o;
}
MG_HD constexpr size_t d_fp32_floats() { return d_bias_offset(kDiscLayers); }
MG_HD constexpr size_t d_tc_start() { return ((d_fp32_floats() * 4 + 255) / 256) * 256; }  // conv_post1, conv_tc_weight_index layout
MG_HD constexpr size_t d_tc_bytes() { return (size_t)1024 * 1024 * 5 * 4; }
// Tensor-core copy of the stride-4 grouped convs (layers 1..3), one 28 KB block per group (mg_disc_tc.cu):
//   tap k = 4q + r reads input position 4(t + q - 5) + r, so per input phase r the conv is a Toeplitz contraction over
//   (q, ci).  K is cut into 7 panels of 8 = 2 consecutive q x 4 ci; one block row n = [hi/lo half][output parity e][co 16]
//   holds w[co][ci][4q + r] with q = 2*kp + pos - 1 - e (zero outside 0 <= k <= 40): both output parities of a tile read
//   the same A operand.  Order [kp 7][r pair 2][r & 1][n 64][8 bf16] = one B operand (N = 64, K = 16) per (kp, r pair).
constexpr int kDgPanels = 7;
MG_HD constexpr size_t d_gtc_group_bytes() { return (size_t)kDgPanels * 2 * 2 * 64 * 16; }
MG_HD constexpr size_t d_gtc_index(int kp, int r, int n, int pos, int ci) {  // bf16 element index inside a group block
    return ((((size_t)(kp * 2 + (r >> 1)) * 2 + (r & 1)) * 64 + n) * 8) + pos * 4 + ci;
}
MG_HD constexpr size_t d_gtc_start() { return d_tc_start() + d_tc_bytes(); }
MG_HD constexpr size_t d_gtc_offset(int l) {  // bytes from d_gtc_start(), l = 1..3
    size_t o = 0;
    for (int i = 1; i < l; ++i) o += (size_t)d_layer(i).groups * d_gtc_group_bytes();
    return o;
}
MG_HD constexpr size_t d_gtc_bytes() { return d_gtc_offset(4); }
// Tensor-core copy of the stride-1 grouped conv (layer 4: 256 groups of 4 -> 4 channels), 24 KB per group: one accumulator row
// owns a block of 8 consecutive outputs t = 8 m + e, a 16-byte unit of the A operand is 8 consecutive positions of ONE
// input channel, and element i of k-panel kp (of channel ci) multiplies w[co][ci][tap = 8 kp + i - e] (zero outside 0..40):
//   [kp 6][ci pair 2][ci & 1][n 64 = half 2 x e 8 x co 4][8 bf16] = one B operand (N = 64, K = 16) per (kp, ci pair).
constexpr int kDg4Panels = 6;
MG_HD constexpr size_t d_g4tc_group_bytes() { return (size_t)kDg4Panels * 2 * 2 * 64 * 16; }
MG_HD constexpr size_t d_g4tc_index(int kp, int ci, int n, int i) {  // bf16 element index inside a group block
    return ((((size_t)(kp * 2 + (ci >> 1)) * 2 + (ci & 1)) * 64 + n) * 8) + i;
}
MG_HD constexpr size_t d_g4tc_start() { return d_gtc_start() + d_gtc_bytes(); }
MG_HD constexpr size_t d_g4tc_bytes() { return (size_t)d_layer(4).groups * d_g4tc_group_bytes(); }
// conv_post1 once more, TRANSPOSED and tap-flipped, for its data gradient: dx = conv1d(dz, W'), W'[ci][co][k] = W[co][ci][4 - k] (a
// stride-1 "same" conv's dgrad is the same conv on flipped, transposed weights), same conv_tc_weight_index layout (mg_conv_tc.cu
// streams it unchanged); then 1024 zero floats: the dgrad launch's "bias"
MG_HD constexpr size_t d_tcT_start() { return d_g4tc_start() + d_g4tc_bytes(); }
MG_HD constexpr size_t d_zero_start() { return d_tcT_start() + d_tc_bytes(); }
MG_HD constexpr size_t d_blob_bytes() { return d_zero_start() + 4096; }
MG_HD constexpr size_t msd_packed_bytes() { return 3 * d_blob_bytes(); }

// Activation workspace (floats per batch item per mel frame): conv_pre out, stage 0..2 outs.
MG_HD constexpr size_t ws_offset(int which, size_t B, size_t T) {  // which: 0 pre, 1..3 stage 0..2
    size_t o = 0;
    if (which >= 1) o += B * 512 * T;
    if (which >= 2) o += B * 256 * 8 * T;
    if (which >= 3) o += B * 128 * 64 * T;
    if (which >= 4) o += B * 64 * 128 * T;
    if (which >= 5) o += B * 32 * 256 * T;   // stage 3 output (tensor-core pipeline only)
    if (which >= 6) o += B * 32 * 256 * T;   // ConvT scratch (tensor-core pipeline only)
    return o;
}

}  // namespace mg
