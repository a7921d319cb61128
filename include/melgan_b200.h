/*
 * melgan_b200.h -- C ABI of the native (sm_90a, H100) MelGAN engine (libmelgan_b200.so).
 *
 * The reference (diver-j/melgan-multi) has no FFI or operator registry: its boundary for the
 * hot path is the torch.nn.Module protocol of models.py, imported by name at train.py:13
 * (`from models import Generator, MultiScaleDiscriminator, ...`).  This library sits directly
 * underneath a drop-in `models` module (melgan_multi_b200/models.py); each entry point below
 * names the reference code it replaces.  Plain pointers and sizes only, no torch types.
 *
 * Conventions
 *   - Every function returns 0 on success or a negative MG_ERR_* code; the message for the
 *     calling thread is available from mg_last_error_string().  Nothing throws or exits.
 *   - "device pointer" arguments are CUDA device addresses owned by the caller (PyTorch
 *     storage in practice); the library never frees or retains them past the call.
 *   - Tensors are fp32, contiguous, NCL ([batch][channel][length]) exactly like the
 *     reference's (models.py:61-71 takes [B,80,T], returns [B,1,256*T]).
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued asynchronously on it and
 *     the library never synchronises the device in the device-pointer entry points.
 *   - Re-entrant: no mutable global state except the thread-local error string.
 */
#ifndef MELGAN_B200_H_
#define MELGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MG_OK 0
#define MG_ERR_INVALID_ARGUMENT (-1)
#define MG_ERR_CUDA (-2)
#define MG_ERR_UNSUPPORTED_DEVICE (-3)
#define MG_ERR_WORKSPACE_TOO_SMALL (-4)
#define MG_ERR_OUT_OF_MEMORY (-5)

#define MG_GEN_NUM_LAYERS 30 /* conv_pre, ups[0..3], 4 x (convs1[0..2], convs2[0..2]), conv_post */

/* ABI version of this header (bumped on any signature change). */
int mg_abi_version(void);

/* Message describing the last failure on the calling thread ("" if none). */
const char *mg_last_error_string(void);

/* 0 if the current CUDA device can run the sm_90a kernels (an H100), MG_ERR_UNSUPPORTED_DEVICE /
 * MG_ERR_CUDA otherwise.  There is no CPU fallback anywhere in this library. */
int mg_device_check(void);

/* ---------------------------------------------------------------------------------------
 * Weight-norm fold + packing.   Replaces: the weight_norm pre-forward hooks that recompute
 * w = g * v / ||v|| on every forward of every layer (models.py:16-28,46-59; 30 launches of
 * aten::_weight_norm_interface per Generator.forward, SURVEY 2.2) with ONE launch that folds
 * all 30 layers and writes them in the layouts the fused kernels stream from.
 *
 * v, g, bias: HOST arrays of MG_GEN_NUM_LAYERS DEVICE pointers in reference registration
 * order (conv_pre, ups.0-3, resblocks.0.convs1.0-2, resblocks.0.convs2.0-2, ..., conv_post);
 * shapes as in the reference state_dict (Conv1d weight_v [Cout,Cin,K], weight_g [Cout,1,1];
 * ConvTranspose1d weight_v [Cin,Cout,K], weight_g [Cin,1,1] -- the norm is per dim 0).
 * packed: device buffer of mg_gen_packed_bytes() bytes, 256-byte aligned.
 */
size_t mg_gen_packed_bytes(void);
int mg_gen_pack(const float *const *v, const float *const *g, const float *const *bias,
                void *packed, void *stream);

/* ---------------------------------------------------------------------------------------
 * Generator forward.   Replaces: models.Generator.forward (models.py:61-71): conv_pre, four
 * fused (LeakyReLU -> ConvTranspose1d -> ResBlock) stages (ResBlock.forward, models.py:32-40),
 * LeakyReLU -> conv_post -> tanh fused into the last stage.
 *
 * mel   [B, 80, T]     device, fp32
 * audio [B, 1, 256*T]  device, fp32
 * workspace: device scratch of at least mg_gen_workspace_bytes(B, T) bytes, 256-byte aligned.
 * Any B >= 1, T >= 1 (train.py:157 feeds whole utterances).
 */
size_t mg_gen_workspace_bytes(int B, int T);
int mg_gen_forward(const void *packed, const float *mel, float *audio, int B, int T,
                   void *workspace, size_t workspace_bytes, void *stream);

/* Ragged batch: B utterances of different lengths in one forward (inference only).
 *   mel   [B, 80, T_max]        device, fp32; item i's frames t >= lengths[i] are never read (they may hold NaN)
 *   audio [B, 1, 256*T_max]     device, fp32; audio[i, 0, :256*lengths[i]] is bit-identical to the mg_gen_forward of
 *                               mel[i:i+1, :, :lengths[i]] alone under the same chain (mg_gen_set_pipeline), the rest 0.0
 *   lengths: HOST array of B ints, 1 <= lengths[i] <= T_max (the grids depend on them: no device read, no sync)
 *   workspace: mg_gen_workspace_bytes(B, T_max) bytes, so mg_gen_check_status(workspace, B, T_max, ...) and
 *   mg_gen_stage_output(workspace, which, out, B, T_max, ...) work as after mg_gen_forward (a tap's values past each item's
 *   valid prefix are unspecified).
 * Every activation keeps the padded [B][C][T_max * scale] layout; the kernels run tiles only inside each item, with the
 * item's own zero padding at its own end.  1 <= B <= MG_GEN_RAGGED_MAX_B (the per-launch tables travel as kernel
 * parameters).  mg_gen_forward is this call with every length equal to T.  Asynchronous on `stream`, no allocation. */
#define MG_GEN_RAGGED_MAX_B 256
int mg_gen_forward_ragged(const void *packed, const float *mel, float *audio, int B, int T_max, const int *lengths,
                          void *workspace, size_t workspace_bytes, void *stream);

/* Inference precision of a generator forward.
 *   MG_GEN_PRECISION_FP32: what mg_gen_forward computes -- every tensor-core product as three bf16 passes on a hi + lo
 *     split of both operands, fp32-equivalent audio (~1e-5 from a float64 forward).
 *   MG_GEN_PRECISION_BF16: one bf16 pass per product, fp32 accumulation, in the ConvTranspose of stages 0, 1 and 3 and in
 *     all 24 ResBlock convs: LeakyReLU(x) and the folded weights are each rounded to bf16 (round to nearest even) before
 *     they are multiplied.  conv_pre and the stride-2 ConvTranspose of stage 2 keep their three passes; the residual
 *     stream, the biases and LeakyReLU -> conv_post -> tanh stay fp32.  Same packed weights, same workspace, no extra
 *     memory.  Measured with the seeded random weights of the tests at B = 64, T = 32 (tests/test_bf16_inference_gpu.py):
 *     relative L2 from float64 9.8e-4 / 1.6e-3, SNR 60 / 56 dB, max |d| 1.8e-4 / 3.1e-4 for N(0,1) / log-mel-like input,
 *     within 1.12x of a float64 emulation of the same rounding.  Trained weights may behave differently.
 * Only the default chain has bf16 kernels: after mg_gen_set_pipeline / MG_GEN_TAIL / MG_GEN_FUSE_UP selected another one,
 * a bf16 forward returns MG_ERR_INVALID_ARGUMENT. */
#define MG_GEN_PRECISION_FP32 0
#define MG_GEN_PRECISION_BF16 1
/* mg_gen_forward (lengths NULL: every item T_max frames) or mg_gen_forward_ragged (lengths as there) with a precision;
 * MG_GEN_PRECISION_FP32 gives exactly their audio.  Ragged batches, batch slices, mg_gen_check_status and
 * mg_gen_stage_output work as after those calls.  Every argument is checked before any CUDA call; an unknown precision is
 * MG_ERR_INVALID_ARGUMENT. */
int mg_gen_forward_precision(const void *packed, const float *mel, float *audio, int B, int T_max, const int *lengths,
                             int precision, void *workspace, size_t workspace_bytes, void *stream);

/* Many voices in one forward: generators of the same architecture with different weights (a vocoder fine-tuned per
 * speaker), each item on its own voice's weights, in one launch of the default chain's eight kernels (inference only).
 *   packed: HOST array of n_voices >= 1 device pointers, each a blob of mg_gen_pack (16-byte aligned, none NULL)
 *   voice:  HOST array of B ints in [0, n_voices): item i runs on packed[voice[i]]
 *   mel, audio, T_max, lengths (NULL: every item T_max frames), precision (MG_GEN_PRECISION_*), workspace
 *   (mg_gen_workspace_bytes(B, T_max)), stream: as for mg_gen_forward_precision.
 * audio[i, 0, :256 L_i] is bit-identical to mg_gen_forward_precision of item i alone (mel[i:i+1, :, :L_i]) on
 * packed[voice[i]] at the same precision, and 0.0 past it.  Limits: at most MG_GEN_RAGGED_MAX_B runs, a run being
 * consecutive items of the same length and the same voice (B itself may exceed it when few runs remain).  Items need not
 * be sorted by voice, but the call is fastest when they are: at every change of voice the conv_pre and ConvT grids start
 * a new tile (a tile never holds two voices), and each persistent stride-2 ConvT CTA that walks into another voice
 * reloads that layer's weights.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call: n_voices < 1, a NULL or
 * misaligned blob, a voice id out of range, any argument mg_gen_forward_precision refuses, and a chain other than the
 * default one (mg_gen_set_pipeline, MG_GEN_TAIL, MG_GEN_FUSE_UP) at either precision.  mg_gen_check_status and
 * mg_gen_stage_output work as after mg_gen_forward_precision.  Asynchronous on `stream`, no allocation; concurrent calls
 * on different streams need different workspaces. */
int mg_gen_forward_voices(const void *const *packed, int n_voices, const int *voice, const float *mel, float *audio, int B,
                          int T_max, const int *lengths, int precision, void *workspace, size_t workspace_bytes, void *stream);

/* 16-bit PCM audio straight from the last kernel: int16 samples instead of fp32, for servers that send WAV / raw LPCM.
 * For the fp32 audio a that the matching float call returns at the same precision, every sample is
 *     pcm16(a) = 0                                      if a is NaN
 *              = clamp(rint(32768 a), -32768, 32767)    otherwise (rint rounds half to even)
 * 32768 (the reference's MAX_WAV_VALUE) times a is exact in fp32, so pcm16 depends on the fp32 sample alone; tanh returns
 * exactly +-1.0 for large arguments, so full scale saturates to 32767 / -32768 instead of wrapping.  The int16 audio is
 * bit-identical to pcm16 of the float call's audio on every path below, at both precisions, and 0 past 256 L_i samples.
 *
 * mg_gen_forward_pcm16: one entry point for uniform, ragged, precision and voices forwards.  audio [B][1][256 T_max] int16
 * device memory; everything else as for mg_gen_forward_voices, except that voice may be NULL (every item on packed[0]).
 * The matching float call is mg_gen_forward_voices when voice is given, else mg_gen_forward_precision on packed[0] (same
 * lengths, same limits: a ragged batch then has at most MG_GEN_RAGGED_MAX_B items).  Workspace, batch slices,
 * mg_gen_check_status and mg_gen_stage_output work as after mg_gen_forward_voices.  Refused with MG_ERR_INVALID_ARGUMENT
 * (MG_ERR_WORKSPACE_TOO_SMALL for a short workspace) before any CUDA call: everything the matching float call refuses,
 * n_voices < 1 or a NULL or misaligned blob among packed[0 .. n_voices), and any chain other than the default one
 * (mg_gen_set_pipeline, MG_GEN_TAIL, MG_GEN_FUSE_UP) at either precision.  Asynchronous on `stream`, no allocation. */
int mg_gen_forward_pcm16(const void *const *packed, int n_voices, const int *voice, const float *mel, int16_t *audio, int B,
                         int T_max, const int *lengths, int precision, void *workspace, size_t workspace_bytes, void *stream);

/* Streaming vocoder: many live sessions, mel frames pushed a few at a time, each audio sample emitted once it is final.
 * A handle serves up to max_sessions (<= MG_GEN_RAGGED_MAX_B) slots at one precision.  Each mg_gen_stream_step gives slot i
 * (i < n) a push of frames[i] in [0, max_push_frames] new mel frames and flags[i] (flags NULL: all 0):
 *   MG_GEN_STREAM_RESET  drop the slot's unfinished utterance before these frames;
 *   MG_GEN_STREAM_END    the utterance ends after these frames (END on a slot with no frames is MG_ERR_INVALID_ARGUMENT).
 * and writes the slot's newly final audio samples to audio[i][0 .. out_samples[i]):
 *   - open utterance of t frames in total: exactly max(0, 256 t - mg_gen_stream_lookahead()) samples have been emitted
 *     over all its steps (the look-ahead, 1542 samples = 70 ms at 22.05 kHz, is the default chain's right-hand receptive
 *     field; sample j depends on no frame past (j + 1542) / 256);
 *   - after the END step all 256 t samples have been emitted; the slot is then free and its next push starts a new
 *     utterance;
 *   - the concatenation of an utterance's outputs is bit-identical to mg_gen_forward_precision of its whole mel (T = t,
 *     same precision, default chain) for any push schedule, 0- and 1-frame pushes included.
 * out_samples is a HOST array filled before the call returns: the step derives every count and launch shape from frame
 * counts alone, enqueues its work asynchronously on `stream` and never synchronises or reads the device.
 * Arguments:
 *   mel   [n][80][max_push_frames] device fp32; slot i's frames are mel[i][:][0 .. frames[i]) (the rest is never read);
 *         may be NULL when every frames[i] is 0
 *   audio [n][mg_gen_stream_max_out(max_push_frames)] device fp32; only audio[i][0 .. out_samples[i]) is written
 *   packed: the weights of mg_gen_pack (may be re-packed between steps: each step reads them anew)
 *   state: caller-owned device memory of mg_gen_stream_state_bytes(max_sessions, max_push_frames) bytes, 256-byte aligned,
 *          for the lifetime of the handle and not shared with another handle.  It holds each session's cached left context
 *          at every kernel boundary, the kernels' windows and the status word.  No step lets a byte that an earlier step
 *          has not written reach an output, so its initial contents do not matter.
 * Every argument is checked before any CUDA call.  On a chain other than the default one (mg_gen_set_pipeline,
 * MG_GEN_TAIL, MG_GEN_FUSE_UP) create and step return MG_ERR_INVALID_ARGUMENT.  One thread drives a handle at a time;
 * steps of one handle must be enqueued on one stream (or otherwise ordered).  mg_gen_stream_check_status waits for `stream`
 * and reports a timed-out tensor-core pipeline wait of any step so far. */
#define MG_GEN_STREAM_END 1
#define MG_GEN_STREAM_RESET 2
typedef struct mg_gen_stream mg_gen_stream; /* host-side counters only */
int mg_gen_stream_lookahead(void);
size_t mg_gen_stream_state_bytes(int max_sessions, int max_push_frames);
int mg_gen_stream_max_out(int max_push_frames); /* 256 max_push_frames + mg_gen_stream_lookahead() */
int mg_gen_stream_create(mg_gen_stream **out, int max_sessions, int max_push_frames, int precision, void *state, size_t state_bytes);
void mg_gen_stream_destroy(mg_gen_stream *s);
int mg_gen_stream_step(mg_gen_stream *s, const void *packed, const float *mel, const int *frames, const int *flags, int n, float *audio,
                       int *out_samples, void *stream);
int mg_gen_stream_check_status(mg_gen_stream *s, void *stream);
/* Many voices in one stream step: slot i runs on the weights of packed[voice[i]], in the same launches as one voice.
 *   packed: HOST array of n_voices >= 1 blobs of mg_gen_pack (16-byte aligned, none NULL; each read anew every step)
 *   voice:  HOST array of n ids in [0, n_voices) (NULL: every slot uses voice 0)
 *   everything else as for mg_gen_stream_step (same handle, precision, state and mg_gen_stream_state_bytes).
 * A slot's voice binds on the step that opens its utterance (its first frames after create, MG_GEN_STREAM_END or
 * MG_GEN_STREAM_RESET).  While the utterance is open every step must pass the same id for the slot, or set
 * MG_GEN_STREAM_RESET on it; a slot with no open utterance accepts any id.  n_voices may change between steps as long as
 * the ids passed stay in range.  The concatenation of a session's outputs is bit-identical to mg_gen_forward_precision of
 * its whole mel on packed[its voice] at the handle's precision, for any push schedule.  Each kernel's items are planned
 * by ascending voice, slot order within a voice, so each voice is one run and (as in mg_gen_forward_voices) the conv_pre
 * and ConvT grids start a new tile at each change of voice.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call:
 * n_voices < 1, a NULL or misaligned blob, an id out of range, a changed id on an open slot without RESET, and
 * everything mg_gen_stream_step refuses.  mg_gen_stream_step(s, packed, ...) is this call with (&packed, 1, NULL). */
int mg_gen_stream_step_voices(mg_gen_stream *s, const void *const *packed, int n_voices, const int *voice, const float *mel,
                              const int *frames, const int *flags, int n, float *audio, int *out_samples, void *stream);
/* mg_gen_stream_step_voices with int16 audio [n][mg_gen_stream_max_out(max_push_frames)]: slot i's newly final samples are
 * pcm16 (see mg_gen_forward_pcm16) of what the float step would write, so an utterance's concatenated output is pcm16 of
 * mg_gen_forward_precision of its whole mel.  The format is chosen per step: float and int16 steps may alternate on one
 * handle, which does not change (same state, same mg_gen_stream_state_bytes).  Refused as mg_gen_stream_step_voices;
 * mg_gen_stream_dry_step* and their copy_bytes describe the float step. */
int mg_gen_stream_step_pcm16(mg_gen_stream *s, const void *const *packed, int n_voices, const int *voice, const float *mel,
                             const int *frames, const int *flags, int n, int16_t *audio, int *out_samples, void *stream);
/* Planning without a device: advances the handle's counters exactly as mg_gen_stream_step would and reports out_samples,
 * the items each of the 8 chain kernels would run (kernel_items[8], may be NULL) and the bytes the window-assembly and
 * audio copies would read and write (copy_bytes, may be NULL).  No CUDA call.  A handle advanced this way refuses later
 * real steps.  mg_gen_stream_dry_step_voices does the same for mg_gen_stream_step_voices (voices bound and refused as
 * there; no blob is needed); mg_gen_stream_dry_step is its case (1, NULL). */
int mg_gen_stream_dry_step(mg_gen_stream *s, const int *frames, const int *flags, int n, int *out_samples, int *kernel_items,
                           long long *copy_bytes);
int mg_gen_stream_dry_step_voices(mg_gen_stream *s, int n_voices, const int *voice, const int *frames, const int *flags, int n,
                                  int *out_samples, int *kernel_items, long long *copy_bytes);

/* Same as mg_gen_forward, but brackets each of the mg_gen_forward_launches() kernels with CUDA
 * events on `stream`, waits for the last one and returns the per-kernel device times in
 * kernel_ms[0 .. mg_gen_forward_launches()-1] (names: mg_gen_kernel_name(i)).  Used by bench.py for the
 * per-kernel roofline. */
int mg_gen_forward_timed(const void *packed, const float *mel, float *audio, int B, int T,
                         void *workspace, size_t workspace_bytes, void *stream, float *kernel_ms);

/* Waits for `stream` and reports whether the tensor-core pipeline of the last forward on `workspace`
 * completed (its producer/consumer waits are bounded so a logic error returns MG_ERR_CUDA here instead
 * of hanging the device). */
int mg_gen_check_status(const void *workspace, int B, int T, void *stream);

/* LeakyReLU -> ConvTranspose1d (models.py:64-65, ups[stage], models.py:48-51) on the tensor-core path:
 * x [B, 512>>stage, Lin] -> y [B, 256>>stage, S*Lin] (S = 8, 8, 2, 2), device fp32, x != y.  Synchronous;
 * parity-test entry point for the tensor-core ConvT kernel. */
int mg_gen_convt(const void *packed, int stage, const float *x, float *y, int B, int Lin, void *stream);

/* One ResBlock (models.py:32-40) of stage `stage` (C = 256 >> stage channels) on the tensor-core path:
 * x, y [B, C, L] device fp32, x != y.  Synchronous; parity-test entry point for the tensor-core kernel. */
int mg_gen_resblock(const void *packed, int stage, const float *x, float *y, int B, int L, void *stream);
/* Stage 2 or 3 as the pipeline runs it: LeakyReLU -> ConvTranspose1d(k4, s2) -> ResBlock in ONE kernel
 * (models.py:64-66); x [B][2C][Lin] is the previous stage's output, y [B][C][2 Lin] (C = 64 / 32).  Synchronous, like
 * mg_gen_resblock: a per-kernel parity entry point. */
int mg_gen_upres(const void *packed, int stage, const float *x, float *y, int B, int Lin, void *stream);
/* The default chain's last kernel: stage 3's LeakyReLU -> ConvTranspose1d(k4, s2), the ResBlock and LeakyReLU -> conv_post
 * -> tanh in ONE kernel (models.py:64-69); x [B][64][Lin] is stage 2's output, audio [B][1][2 Lin].  Synchronous parity
 * entry point. */
int mg_gen_upres_post(const void *packed, const float *x, float *audio, int B, int Lin, void *stream);
/* Template configuration of the ResBlock kernel behind a stage code (0..3 ResBlock, 4 + conv_post, 12 / 13 / 14 ConvT fused in
 * front, 20 / 21 / 22 next ConvT fused at the tail), "resblock_tc_kernel<RbCfg<C,NRB,RPW,NCP,NSTAGE,POST,UPF,UPT,CS>>";
 * "" for an unknown code.  Tests derive the tile and cluster borders from it. */
const char *mg_gen_resblock_config(int code);
/* Where the packed blob keeps the split-bf16 copy of one tensor-core weight: the byte offset of half h (0 hi, 1 lo) from the
 * start of the blob, or (size_t)-1 for an argument out of range.
 *   front = 0, layer 0: conv_pre, w[co][ci][tap], tap 0..6;
 *   front = 0, layer 1..4: ups[layer - 1], W[ci][co][tap] (the ConvTranspose1d layout), tap 0 .. 2 S - 1;
 *   front = 0, layer 5..28: a ResBlock conv, w[co][ci][tap], tap 0..2;
 *   front = 1, layer = stage 2 / 3: the stride-2 ConvT fused in front of that stage's ResBlock, W[ci][co][tap], tap 0..3.
 * Tests restate the layout the tensor-core descriptors expect against it. */
size_t mg_gen_tc_weight_offset(int front, int layer, int co, int ci, int tap, int h);
/* Tile geometry of the ConvT kernel launch_convt_tc runs for `stage`; tests derive tile borders from it.  A tile is ROWS
 * input positions of the batch's items concatenated with one zero row after each.
 *   stage 0: "convt_tc_kernel<UpCfg<0,ROWS,NG>>", one CTA per (tile, group of NG output channels);
 *   stage 1: "convt_resident_tc_kernel<UpCfg<1,ROWS,NG>>", one CTA per tile, looping over the groups of NG channels;
 *   stage 2 / 3: "convt_stream_tc_kernel<StreamCfg<STAGE,ROWS,MAXSEG,NSX>>": at most MAXSEG item segments of a tile staged
 *   by bulk copy, NSX staging slots; persistent grid of min(tiles, SMs) CTAs.
 * "" for any other stage. */
const char *mg_gen_convt_config(int stage);
/* conv_pre's tile geometry, "conv_rows_tc_kernel<ConvCfg<80,512,7,ROWS,N>>": ROWS virtual rows per CTA (each item's
 * positions followed by 3 zero rows), N output channels per CTA. */
const char *mg_gen_conv_pre_config(void);
/* Kernel k (0..7) of the default chain alone -- 0 conv_pre, 1 up0, 2 res0, 3 up1, 4 res1, 5 up2, 6 res2, 7 up3+res3+post --
 * as mg_gen_forward_precision and mg_gen_stream_step launch it, on a batch of B <= MG_GEN_RAGGED_MAX_B items:
 *   x [B][Cin][L_max] -> y [B][Cout][R L_max], device fp32, 16-byte aligned, x != y, where (Cin, Cout, R) is
 *   (80, 512, 1), (512, 256, 8), (256, 256, 1), (256, 128, 8), (128, 128, 1), (128, 64, 2), (64, 64, 1), (64, 1, 2) for k = 0..7;
 *   lengths: NULL (every item L_max positions) or a HOST array of B lengths in [1, L_max], in kernel k's input units.
 * Item i reads only x[i][:][0 .. lengths[i]) (the rest may hold NaN) and writes only y[i][:][0 .. R lengths[i]), except
 * kernel 7, which also writes 0.0 to y[i][0][R lengths[i] .. R L_max) (the ragged forward's zero audio tail).  precision:
 * MG_GEN_PRECISION_FP32 or _BF16 (kernels 0 and 5 run three passes at either).  Every argument is checked before any CUDA
 * call; on a chain other than the default one it returns MG_ERR_INVALID_ARGUMENT.  Synchronous, with its own status word
 * (a timed-out pipeline wait is MG_ERR_CUDA).  Test entry point: the same launcher the stream steps use. */
int mg_gen_chain_kernel(const void *packed, int k, const float *x, float *y, int B, int L_max, const int *lengths, int precision,
                        void *stream);

/* ResBlock `stage` (0..2) with the NEXT stage's LeakyReLU -> ConvTranspose1d fused at its tail, as the default pipeline runs it
 * (models.py:66 followed by :64-65 of the next loop iteration): x [B][C][L] is stage `stage`'s ConvT output, y
 * [B][C/2][S L] is stage+1's (S = 8 for stage 0, else 2).  Synchronous parity entry point. */
int mg_gen_resup(const void *packed, int stage, const float *x, float *y, int B, int L, void *stream);

/* conv_pre alone (models.py:46,62): mel [B,80,T] -> y [B,512,T], device fp32.  Synchronous parity-test entry point of
 * conv_rows_tc_kernel<80,512,k7>. */
int mg_gen_conv_pre(const void *packed, const float *mel, float *y, int B, int T, void *stream);
/* The last ResBlock with its fused epilogue (models.py:66-69 for stage 3: ResBlock -> LeakyReLU -> conv_post -> tanh):
 * x [B,32,L] (the stage-3 ConvT output) -> audio [B,1,L].  Synchronous parity-test entry point of the conv_post + tanh fusion. */
int mg_gen_resblock_post(const void *packed, const float *x, float *audio, int B, int L, void *stream);

/* Diagnostic twin of mg_gen_resblock: also returns 128 clock64 stamps (host buffer) of one interior CTA's
 * hand-off and MMA phases (slot meaning documented at the definition in csrc/mg_api.cu).  `stage` is any stage code of
 * mg_gen_resblock_config, with that kernel's shapes: L is the ResBlock's own length (codes 12..14: x [B][2C][L/2]). */
int mg_gen_resblock_trace(const void *packed, int stage, const float *x, float *y, int B, int L, long long *trace_host);

/* Debug/parity tap: copies the activation after stage `which` (0 = conv_pre output [B,512,T],
 * 1..3 = ResBlock 0..2 output [B,C,L]; the last stage is fused with conv_post and has no tap) of the LAST mg_gen_forward that used `workspace` into
 * `out` (device, NCL).  Only valid immediately after that call on the same stream. */
int mg_gen_stage_output(const void *workspace, int which, float *out, int B, int T, void *stream);

/* ---------------------------------------------------------------------------------------
 * Multi-scale discriminator forward.   Replaces: models.MultiScaleDiscriminator.forward (models.py:119-135) and
 * Discriminator.forward (models.py:87-103) for a batch in which the caller has stacked real and generated audio
 * (Bt = 2B: every weight is streamed once for both; the reference calls d(y) and d(y_hat) separately), with the
 * AvgPool1d chain (models.py:114-117) fused into each scale's first conv and the 21 weight-norm folds done by one
 * mg_msd_pack launch.
 *
 * v, g, bias: HOST arrays of 21 DEVICE pointers, discriminator-major, layers in reference registration order
 *   (conv_pre, grouped_convs.0-3, conv_post1, conv_post2).
 * y [Bt, 1, L] device fp32.  fmaps: HOST array of 21 DEVICE pointers (scale-major, 7 per scale) receiving the feature
 *   maps [Bt, C_l, len] with len = lens[scale*7 + l] from mg_msd_lengths(L, lens); the first six of a scale are
 *   post-LeakyReLU, the seventh is conv_post2's raw output, i.e. the flattened logits [Bt, len].
 * status_word: >= 4 bytes of device memory; check it with mg_msd_check_status after the call (bounded waits).
 * Bt <= 65535 (conv_pre, conv_post2 and the SIMT grouped convs put the items on grid.y / grid.z); a larger batch returns
 *   MG_ERR_INVALID_ARGUMENT before any CUDA call: split it into calls of at most 65535 items.
 */
size_t mg_msd_packed_bytes(void);
int mg_msd_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, void *stream);
int mg_msd_lengths(int L, int *lens);
int mg_msd_forward(const void *packed, const float *y, int Bt, int L, float *const *fmaps, void *status_word, void *stream);
int mg_msd_check_status(const void *status_word, void *stream);

/* One stand-alone Discriminator (models.py:74-103: Discriminator() called on its own, outside MultiScaleDiscriminator):
 * v, g, bias: HOST arrays of 7 DEVICE pointers (conv_pre, grouped_convs.0-3, conv_post1, conv_post2); packed: device buffer of
 * mg_disc_packed_bytes() bytes, 256-byte aligned.  x [Bt,1,L] -> fmaps: HOST array of 7 DEVICE pointers, lengths
 * lens[0..6] of mg_msd_lengths(L, lens) (the scale-0 row); fmaps[6] is the flattened logits.  status_word and the
 * Bt <= 65535 limit as above. */
size_t mg_disc_packed_bytes(void);
int mg_disc_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, void *stream);
int mg_disc_forward(const void *packed, const float *x, int Bt, int L, float *const *fmaps, void *status_word, void *stream);

/* Layer `layer` (1..6: grouped_convs.0-3, conv_post1, conv_post2) of discriminator `scale` (0..2; 0 for a stand-alone
 * Discriminator's blob) on a caller-given input, through the launcher mg_msd_forward runs for that layer:
 *   x [Bt][Cin][Lin] -> out [Bt][Cout][Lout] (device fp32, x != out), Lout = (Lin + 2 pad - k) / stride + 1 >= 1; the
 *   output is post-LeakyReLU except conv_post2's.  Writes out[:, :, 0 .. Lout) and nothing else.
 * Asynchronous on `stream`; status_word and the 1 <= Bt <= 65535 limit as for mg_msd_forward (the word is not cleared:
 * check it with mg_msd_check_status).  MG_DISC_GROUP=simt selects the SIMT grouped convs here too.  Every argument is checked
 * before any CUDA call.  Test entry point: a layer's kernel on inputs the caller chooses. */
int mg_msd_layer_forward(const void *packed, int scale, int layer, const float *x, float *out, int Bt, int Lin, void *status_word,
                         void *stream);
/* Which folded weight a bf16 element of one discriminator's blob holds in the four split-bf16 copies the tensor cores read:
 * `offset` is the element's byte offset from the start of that discriminator's blob.  Returns the half (0 hi, 1 lo) of weight
 * w[co][ci][tap] of the layer's torch layout [Cout][Cin / groups][k] (ci < 4 for the grouped convs), 2 for a structural zero
 * of a Toeplitz copy (co and ci are then the slot's, tap the out-of-range tap it stands for), or -1 for an offset outside
 * the copies.  *copy: 1..3 the Toeplitz copy of grouped_convs.0-2, 4 that of grouped_convs.3, 5 conv_post1's forward copy,
 * 6 its transposed, tap-flipped copy (the data gradient's; still reported as the forward weight w[co][ci][tap]).  One
 * weight sits in several Toeplitz slots, hence the map from slot to weight.  Tests restate the layouts against it. */
int mg_disc_tc_element(size_t offset, int *copy, int *co, int *ci, int *tap);

/* ---------------------------------------------------------------------------------------
 * Mel-spectrogram front end.   Replaces: mel_spectrogram (meldataset.py:44-55: zero-pad by (n_fft - hop)/2, librosa
 * melspectrogram with power 1 and Slaney-normalised triangles, log(clip(., 1e-5))) for the reference's analysis parameters
 * n_fft = 1024, hop = 256, win = 1024 (config.json:15-17), on the GPU: the loader's and the validation loop's librosa call
 * (train.py:164) without the host round trip.
 *   mg_mel_tables_build fills a HOST buffer of mg_mel_tables_bytes() bytes (window, twiddles, sparse filter bank);
 *     norm: 0 none, 1 Slaney area normalisation (= librosa 0.6/0.7 `norm=1`, today's `norm="slaney"`), 2 L1.  The caller
 *     copies it to device memory (16-byte aligned) once.
 *   mg_mel_spectrogram: audio [B][L] device fp32 in [-1, 1] -> mel [B][n_mels][T] device fp32, T = mg_mel_frames(L)
 *     (= L / 256 when L is a multiple of 256).  Asynchronous on `stream`.  One CTA per item and pair of frames, all on
 *     grid.x: any B works as long as B * ceil(T / 2) <= 2^31 - 1; beyond that MG_ERR_INVALID_ARGUMENT, before any launch.
 *   mg_mel_spectrogram_backward: the gradient of a loss with respect to the audio, grad_audio = d loss / d audio [B][L]
 *     device fp32, given grad_mel = d loss / d mel [B][n_mels][T] device fp32, for
 *       mel = log(clamp(M . |rfft(w . frame_t(pad(audio)))|, min=1e-5))
 *     (pad: 384 zeros each side; frame_t: padded samples [256 t, 256 t + 1024); w: periodic Hann; M: the tables' filter
 *     bank), under torch autograd's conventions: the gradient passes where the band's sum s >= 1e-5 and is 0 below it;
 *     a bin with |X| = 0 contributes 0; the rfft's adjoint runs over bins 0..512 as the forward has them (interior bins
 *     not doubled); gradients on padding are dropped; samples no frame reaches (the trailing L mod 256 past the last
 *     frame) get exactly 0.  Every element of grad_audio is written; it may be uninitialised.  The magnitudes and s are
 *     recomputed with the forward's arithmetic.  Deterministic: no floating-point atomics, each item bit-identical to its
 *     own B = 1 call.  Asynchronous on `stream`, no host synchronisation (capturable in a CUDA graph).
 *     workspace: caller-owned device memory, 16-byte aligned, of at least mg_mel_backward_workspace_bytes(B, L) =
 *     B * mg_mel_frames(L) * 1024 * 4 bytes (0 when B, L or the launch limit are invalid); it holds the per-frame
 *     gradients for one call, so concurrent calls need their own.  Same limit as the forward (B * ceil(T / 2) <= 2^31 - 1).
 *     NULL pointers, B < 1, T < 1, misaligned tables or workspace are refused with MG_ERR_INVALID_ARGUMENT, a short
 *     workspace with MG_ERR_WORKSPACE_TOO_SMALL, before any launch.
 */
size_t mg_mel_tables_bytes(void);
int mg_mel_tables_build(int sampling_rate, int n_mels, float fmin, float fmax, int norm, void *tables_host);
int mg_mel_frames(int L);
int mg_mel_spectrogram(const void *tables, const float *audio, float *mel, int B, int L, void *stream);
size_t mg_mel_backward_workspace_bytes(int B, int L);
int mg_mel_spectrogram_backward(const void *tables, const float *audio, const float *grad_mel, float *grad_audio, int B, int L,
                                void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Multi-resolution STFT loss (Parallel WaveGAN's MultiResolutionSTFTLoss) of predicted audio x against target audio y,
 * both [B][L] device fp32, and its gradient with respect to x.  For each of n_res resolutions (n_fft[r], hop[r], and the
 * window length given to the table build):
 *   X = torch.stft(x, n_fft, hop, win_length, periodic Hann(win_length), center=True, pad_mode="reflect"), one-sided,
 *   T = 1 + L / hop frames (mg_stft_loss_frames); x_mag = sqrt(clamp(|X|^2, min=1e-7)), y_mag likewise;
 *   sc = ||y_mag - x_mag||_F / ||y_mag||_F and mag = mean |log y_mag - log x_mag| over the whole [B][T][n_fft/2 + 1].
 * The losses are the means of sc and mag over the resolutions.  Supported: n_fft a power of two in [128, 2048],
 * 1 <= win_length <= n_fft, hop >= 1, n_fft / 2 < L <= 2^30 (reflect padding by n_fft / 2), 1 to 8 resolutions.
 *   mg_stft_loss_tables_build fills a HOST buffer of mg_stft_loss_tables_bytes(n_fft) bytes (0 for an unsupported n_fft)
 *     for one resolution: the window zero-padded to n_fft with (n_fft - win_length) / 2 zeros on the left, then the
 *     twiddles e^{-2 pi i k / n_fft}, k < n_fft / 2, each computed in double and rounded once.  The caller copies it to
 *     device memory, 16-byte aligned, once per device.
 *   mg_stft_loss_workspace_bytes: the forward workspace (each resolution's per-frame partial sums, and the norms the
 *     backward reads) and the backward workspace (the largest resolution's per-frame gradients, B T n_fft floats).
 *   mg_stft_loss_forward writes the two losses to the device scalars sc_loss and mag_loss.  The sums are reduced in a
 *     fixed order (no atomics): the same inputs give the same bits on every run.
 *   mg_stft_loss_backward writes grad_x = grad_sc d sc / dx + grad_mag d mag / dx [B][L], every element (it may be
 *     uninitialised), for device scalars grad_sc and grad_mag.  forward_workspace is the workspace of the forward call on
 *     the same x and y, which it reads; workspace is its own.  Torch autograd's conventions: the clamp passes gradient
 *     where |X|^2 >= 1e-7, a zero ||y_mag - x_mag|| gives the sc term gradient 0, sign(0) = 0, gradient on reflected
 *     positions is folded back onto the samples they copy.  The magnitudes are recomputed with the forward's arithmetic.
 *     Deterministic, no floating-point atomics.
 * Both are asynchronous on `stream`, with no host synchronisation (capturable in a CUDA graph); concurrent calls need
 * their own workspaces.  NaN and Inf samples are not clamped away: they make the losses and the gradient NaN or Inf
 * where float64 autograd of the definition does.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call, with a
 * message naming the argument: n_res outside [1, 8], a NULL array or pointer, misaligned tables or workspaces (16 bytes)
 * or float pointers (4 bytes), an unsupported n_fft, win_length outside [1, n_fft], hop < 1, L <= n_fft / 2,
 * L > 2^30, B < 1, a
 * grid past 2^31 - 1 CTAs (B T per resolution, B ceil(L / 256) for the gradient's gather); a short workspace with
 * MG_ERR_WORKSPACE_TOO_SMALL.
 */
size_t mg_stft_loss_tables_bytes(int n_fft);
int mg_stft_loss_tables_build(int n_fft, int win_length, void *tables_host);
int mg_stft_loss_frames(int n_fft, int hop, int L); /* 1 + L / hop, or 0 when the analysis or L is unsupported */
int mg_stft_loss_workspace_bytes(int n_res, const int *n_fft, const int *hop, int B, int L, size_t *forward_bytes,
                                 size_t *backward_bytes);
int mg_stft_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                         int B, int L, float *sc_loss, float *mag_loss, void *workspace, size_t workspace_bytes, void *stream);
int mg_stft_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                          int B, int L, const float *grad_sc, const float *grad_mag, const void *forward_workspace, float *grad_x,
                          void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Multi-resolution log-mel L1 loss of predicted audio x against target audio y, both [B][L] device fp32, and its
 * gradient with respect to x (HiFi-GAN's 45 * l1(mel(y_hat), mel(y)) without the 45, summed over several analyses).
 * For each of n_res resolutions r (n_fft[r] = N, hop[r] = H, and the window length W, sampling rate, n_mels M, fmin and
 * fmax given to the table build), p = (N - H) / 2:
 *   x~ = x with p zeros on each side; frames T = 1 + (L + 2p - N) / H (mg_mel_loss_frames; T < 1 is refused);
 *   w = periodic Hann of length W, zero-padded to N with (N - W) / 2 zeros on the left (librosa's pad_center);
 *   X_t[k] = sum_n w[n] x~[t H + n] e^{-2 pi i k n / N}, k = 0..N/2;  S_t[m] = sum_k F[m, k] |X_t[k]|, F the librosa
 *   Slaney filter bank (htk=False, Slaney area normalisation, bin frequencies k sr / N);  mel = ln(clip(S, min=1e-5));
 *   l_r = mean over (b, m, t) of |mel_x - mel_y|.
 * The loss is (1 / n_res) sum_r l_r, a device fp32 scalar.  At one resolution (1024, 256, 1024, 80) it is F.l1_loss of
 * mg_mel_spectrogram's two outputs.  Supported: N a power of two in [128, 2048], 1 <= W <= N, 1 <= H <= N,
 * 1 <= M <= 512 (empty filters allowed: their band is ln(1e-5) and gets no gradient), 0 <= fmin < fmax <= sr / 2,
 * 1 to 8 resolutions, T >= 1, L <= 2^30.
 *   mg_mel_loss_tables_build fills a HOST buffer of mg_mel_loss_tables_bytes(n_fft) bytes (0 for an unsupported n_fft):
 *     the STFT loss's window and twiddles for (n_fft, win_length), then n_mels and the sparse filter bank.  The caller
 *     copies it to device memory, 16-byte aligned, once per device.
 *   mg_mel_loss_workspace_bytes: the forward workspace (one partial sum per item and frame of each resolution) and the
 *     backward workspace (the largest resolution's per-frame gradients, B T n_fft floats).
 *   mg_mel_loss_forward writes the loss to the device scalar `loss`.  Per-frame fp32 partials are summed in float64 in a
 *     fixed order (no atomics): the same inputs give the same bits on every run.
 *   mg_mel_loss_backward writes grad_x = grad d loss / dx [B][L], every element (it may be uninitialised), for the
 *     device scalar grad.  It reads no forward workspace: the spectra and bands are recomputed with the forward's
 *     arithmetic.  Torch autograd's conventions: d|a - b| / da = sign(a - b) with sign(0) = sign(NaN) = 0, the clip
 *     passes the gradient where S >= 1e-5, a bin with |X| = 0 contributes 0, the rfft's adjoint runs over bins 0..N/2
 *     as the forward has them, gradients on padding are dropped.  Deterministic, no floating-point atomics.
 * Both are asynchronous on `stream`, with no host synchronisation (capturable in a CUDA graph); concurrent calls need
 * their own workspaces.  NaN and Inf samples are not clamped away: they make the loss and the gradient NaN or Inf where
 * float64 autograd of the definition does.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call, with a message
 * naming the argument: n_res outside [1, 8], a NULL array or pointer, misaligned tables or workspaces (16 bytes) or
 * float pointers (4 bytes), an unsupported n_fft, win_length, n_mels, fmin or fmax, hop outside [1, n_fft], L outside
 * [1, 2^30], fewer samples than one frame, B < 1, a grid past 2^31 - 1 CTAs (B T per resolution, B ceil(L / 256) for the
 * gradient's gather); a short workspace with MG_ERR_WORKSPACE_TOO_SMALL.
 */
size_t mg_mel_loss_tables_bytes(int n_fft);
int mg_mel_loss_tables_build(int n_fft, int win_length, int sampling_rate, int n_mels, float fmin, float fmax, void *tables_host);
int mg_mel_loss_frames(int n_fft, int hop, int L); /* 1 + (L + 2p - n_fft) / hop, or 0 when the analysis or L is unsupported */
int mg_mel_loss_workspace_bytes(int n_res, const int *n_fft, const int *hop, int B, int L, size_t *forward_bytes,
                                size_t *backward_bytes);
int mg_mel_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y, int B,
                        int L, float *loss, void *workspace, size_t workspace_bytes, void *stream);
int mg_mel_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y, int B,
                         int L, const float *grad, float *grad_x, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Denoiser (WaveGlow's Denoiser): subtract a vocoder's bias spectrum from its audio.  audio [B][L_max] device fp32; item i
 * owns its first L_i = lengths[i] samples (lengths NULL: every item L_max) and uses bias row voice[i] (voice NULL: row 0)
 * of bias [n_voices][n_fft/2 + 1] device fp32.  With N = n_fft, H = hop, W = win_length and, in float64 terms,
 *   S  = torch.stft(a_i[:L_i], N, H, W, periodic Hann(W), center=True, pad_mode="reflect"), 1 + L_i / H frames;
 *   M' = max(|S| - strength bias[voice[i]], 0)  (written `x < 0 ? 0 : x`: NaN stays NaN);
 *   P  = S / |S| where |S| > 0, else 1;
 *   out_i[:L_i] = torch.istft(M' P, N, H, W, periodic Hann(W), center=True, length=L_i), out_i[L_i:] = 0.
 * tables: the STFT loss's table for (n_fft, win_length) (mg_stft_loss_tables_build), on the device, 16-byte aligned.
 * Supported: N a power of two in [128, 2048], 1 <= H <= W <= N (torch.istft's limit), N/2 < L_i <= L_max <= 2^30, any (N, H, W, L_i) whose
 * window-square envelope stays >= 1e-11 at every output sample some frame reaches (torch.istft's NOLA condition, checked
 * on the host in float64 for each distinct length), B <= MG_GEN_RAGGED_MAX_B when lengths or voice is given.
 *   mg_denoise_workspace_bytes: the frame workspace, sum_i (1 + L_i / H) N floats (each frame resynthesised and windowed).
 *   mg_denoise_bias writes bias [n_rows][N/2 + 1] = |X[k]| of frame 0 of each row of audio [n_rows][L] (the same frame,
 *     FFT and bins as the forward): WaveGlow's bias spectrum of a generator's audio.  1 <= n_rows <= 65535.
 *   mg_denoise_forward writes out [B][L_max], every element; mg_denoise_forward_pcm16 writes int16 out, pcm16 of the
 *     float output (mg_gen_forward_pcm16's rounding, by the same kernel).  Each output sample sums its frames and the
 *     window-square envelope in ascending frame order: no atomics, the same inputs give the same bits on every run, and
 *     each item's samples are those of its own B = 1 call.  win_length must be the one the tables were built with.
 * Asynchronous on `stream`, no host synchronisation (capturable in a CUDA graph); concurrent calls need their own
 * workspaces.  NaN and Inf samples are not clamped away: a non-finite sample makes its frames non-finite, hence the output
 * samples those frames reach.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call, with a message naming the
 * argument: an unsupported n_fft, hop < 1, win_length outside [1, n_fft], hop > win_length, B < 1, L_max > 2^30, a length outside
 * (n_fft/2, L_max], a ragged or voiced batch of more than MG_GEN_RAGGED_MAX_B items, n_voices < 1, a voice outside
 * [0, n_voices), a non-finite strength, a NULL or misaligned pointer (tables and workspace 16 bytes, float 4, int16 2), a
 * grid past 2^31 - 1 CTAs, the NOLA condition; a short workspace with MG_ERR_WORKSPACE_TOO_SMALL.
 */
int mg_denoise_workspace_bytes(int n_fft, int hop, int B, int L_max, const int *lengths, size_t *bytes);
int mg_denoise_bias(const void *tables, int n_fft, const float *audio, int n_rows, int L, float *bias, void *stream);
int mg_denoise_forward(const void *tables, int n_fft, int hop, int win_length, const float *audio, int B, int L_max, const int *lengths,
                       const float *bias, int n_voices, const int *voice, float strength, float *out, void *workspace,
                       size_t workspace_bytes, void *stream);
int mg_denoise_forward_pcm16(const void *tables, int n_fft, int hop, int win_length, const float *audio, int B, int L_max,
                             const int *lengths, const float *bias, int n_voices, const int *voice, float strength, int16_t *out,
                             void *workspace, size_t workspace_bytes, void *stream);

/* Streaming denoiser: mg_denoise_forward applied to live audio.  A handle serves up to max_sessions (<= MG_GEN_RAGGED_MAX_B)
 * slots at one analysis (n_fft N, hop H, win_length W) and one strength.  Each mg_denoise_stream_step gives slot i (i < n)
 * in_samples[i] in [0, max_push_samples] new fp32 samples and flags[i] (flags NULL: all 0), with mg_gen_stream_step's
 * meaning: MG_GEN_STREAM_RESET drops the slot's unfinished utterance first, MG_GEN_STREAM_END ends it after these samples.
 * It writes the slot's newly final denoised samples to out[i][0 .. out_samples[i]).
 * The finality rule.  With R the samples an open utterance has received: frame t reads samples [t H - N/2, t H + N/2)
 * reflected at 0 (frame 0 reads 0 .. N/2), so frames 0 .. q, q = floor((R - N/2) / H), are computable once R > N/2.
 * Output sample j sums frames up to floor((j + N/2) / H) <= q, so exactly
 *     E(R) = 0 if R <= N/2, else clamp((q + 1) H - N/2, 0, R)
 * samples have been emitted over the utterance's steps; R - E(R) lies in [N - H, N - 1] in steady state (768 .. 1023
 * samples at N = 1024, H = 256).  The rule follows the frames the kernel sums, not the window's support: a later frame's
 * term is added even where the window is 0, so a NaN or Inf reaches exactly the samples it reaches in mg_denoise_forward.
 * After the END step, at length L, all L samples have been emitted (frames up to floor(L / H) reflect at L; samples no
 * frame reaches when H > N/2 are 0) and the slot is free.  The concatenation of an utterance's outputs is bit-identical to
 * mg_denoise_forward of its L samples (same tables, bias row, strength) for any push schedule, 0- and 1-sample pushes
 * included; mg_denoise_stream_step_pcm16 writes int16 out, pcm16 of what the float step writes (the format is chosen per
 * step and may alternate on one handle).
 * Arguments:
 *   tables: the STFT loss's table for (n_fft, win_length) on the device; bias [n_voices][N/2 + 1] device fp32
 *   voice: HOST array of n ids in [0, n_voices) (NULL: all 0).  A slot's bias row binds on the step that opens its
 *          utterance and is released at END or RESET; a changed id on an open slot without RESET is refused, as in
 *          mg_gen_stream_step_voices.
 *   audio_in [n][in_stride] device fp32: slot i's new samples are audio_in[i][0 .. in_samples[i]) (in_samples[i] <=
 *          in_stride); may be NULL when every in_samples[i] is 0.  mg_gen_stream_step's audio [n][mg_gen_stream_max_out(P)]
 *          with its out_samples is a valid (audio_in, in_stride, in_samples) as it is.
 *   in_samples, flags, out_samples: HOST arrays; out_samples is filled before the call returns.  The step derives every
 *          count and launch from sample counts alone, enqueues its work on `stream` and never synchronises or reads the
 *          device.
 *   out [n][mg_denoise_stream_max_out(N, H, max_push_samples)] device fp32 (int16 for _pcm16): only out[i][0 ..
 *          out_samples[i]) is written.  max_out = max_push_samples + N - 1, reached by an END push of max_push_samples
 *          when R - E(R) = N - 1.
 *   state: caller-owned device memory of mg_denoise_stream_state_bytes(N, H, max_sessions, max_push_samples) bytes,
 *          256-byte aligned, for the lifetime of the handle and not shared with another handle: each session's tail of
 *          at most N samples, its window and a ring of the frames its pending samples need.  No step lets a byte an
 *          earlier step has not written reach an output, so its initial contents do not matter.
 * Supported: N a power of two in [128, 2048], 1 <= H <= W <= N, max_push_samples in [1, 2^20], utterances of
 * N/2 < L <= 2^30 samples.  create refuses the length-independent part of torch.istft's NOLA condition (a residue mod H
 * whose window-square sum is below 1e-11), the END step the rest, at the utterance's length.  Refused with
 * MG_ERR_INVALID_ARGUMENT before any CUDA call, with a message naming the argument, and leaving the counters unchanged:
 * a bad analysis, max_sessions or max_push_samples, a non-finite strength, n outside [0, max_sessions], n_voices < 1, an
 * id out of range or changed on an open slot, in_samples outside [0, max_push_samples] or past in_stride, unknown flag
 * bits, END on a slot with no samples or at L <= N/2, an utterance past 2^30 samples, the NOLA condition, a NULL or
 * misaligned pointer (state 256 bytes, tables 16, float 4, int16 2); a short state with MG_ERR_WORKSPACE_TOO_SMALL.  One
 * thread drives a handle at a time; its steps must be enqueued on one stream (or otherwise ordered).
 * mg_denoise_stream_dry_step advances the counters exactly as a step would, with no device and no pointer, and reports
 * out_samples and the frames the step would compute (new_frames, may be NULL); a handle advanced this way refuses later
 * real steps. */
typedef struct mg_denoise_stream mg_denoise_stream; /* host-side counters only */
size_t mg_denoise_stream_state_bytes(int n_fft, int hop, int max_sessions, int max_push_samples);
int mg_denoise_stream_max_out(int n_fft, int hop, int max_push_samples);
int mg_denoise_stream_create(mg_denoise_stream **out, int n_fft, int hop, int win_length, int max_sessions, int max_push_samples,
                             float strength, void *state, size_t state_bytes);
void mg_denoise_stream_destroy(mg_denoise_stream *s);
int mg_denoise_stream_step(mg_denoise_stream *s, const void *tables, const float *bias, int n_voices, const int *voice,
                           const float *audio_in, long long in_stride, const int *in_samples, const int *flags, int n, float *out,
                           int *out_samples, void *stream);
int mg_denoise_stream_step_pcm16(mg_denoise_stream *s, const void *tables, const float *bias, int n_voices, const int *voice,
                                 const float *audio_in, long long in_stride, const int *in_samples, const int *flags, int n, int16_t *out,
                                 int *out_samples, void *stream);
int mg_denoise_stream_dry_step(mg_denoise_stream *s, int n_voices, const int *voice, const int *in_samples, const int *flags, int n,
                               int *out_samples, int *new_frames);

/* ---------------------------------------------------------------------------------------
 * Host-buffer engine.   The call a non-PyTorch host makes: owns its device buffers, takes and
 * returns HOST memory, and performs the host<->device copies itself (this is the path
 * bench.py times as "e2e").  One engine per host thread / CUDA stream.
 */
typedef struct mg_gen_engine mg_gen_engine;

/* Creates an engine able to run up to max_B x max_T (it grows on demand if exceeded). */
int mg_gen_engine_create(mg_gen_engine **out, int max_B, int max_T);
/* v/g/bias: HOST arrays of 30 HOST pointers (state_dict tensors, reference order). */
int mg_gen_engine_load_state(mg_gen_engine *e, const float *const *v, const float *const *g,
                             const float *const *bias);
/* mel_host [B,80,T] -> audio_host [B,1,256T]; synchronous (returns when audio_host is filled).
 * Pinned host memory is used as given; pageable memory is staged through an internal pinned
 * buffer.  The copies are cut with the batch slices (mg_gen_forward_slices): a slice's audio goes
 * back to the host while the other slices are still computing. */
int mg_gen_engine_forward(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T);
/* Ragged twin of mg_gen_engine_forward (semantics and limits of mg_gen_forward_ragged): mel_host [B,80,T_max] ->
 * audio_host [B,1,256 T_max].  Each slice uploads only its items' valid mel prefixes and downloads its audio rows (the
 * valid prefix and the zero tail). */
int mg_gen_engine_forward_ragged(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T_max,
                                 const int *lengths);
/* mg_gen_engine_forward (lengths NULL) / mg_gen_engine_forward_ragged with a precision (MG_GEN_PRECISION_*, contract at
 * mg_gen_forward_precision). */
int mg_gen_engine_forward_precision(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T_max,
                                    const int *lengths, int precision);
/* mg_gen_engine_forward_precision with int16 audio_host [B][1][256 T_max]: pcm16 of its audio (contract at
 * mg_gen_forward_pcm16).  The int16 samples are staged in pinned memory and downloaded per batch slice, half the bytes of
 * the float call.  Refused with MG_ERR_INVALID_ARGUMENT before any CUDA call: everything the float call refuses, and any
 * chain other than the default one. */
int mg_gen_engine_forward_pcm16(mg_gen_engine *e, const float *mel_host, int16_t *audio_host, int B, int T_max,
                                const int *lengths, int precision);
/* Device time of the last forward in milliseconds (CUDA events on the engine's stream around the sliced
 * upload -> kernels -> download sequence). */
int mg_gen_engine_last_kernel_ms(mg_gen_engine *e, float *ms);
void mg_gen_engine_destroy(mg_gen_engine *e);

/* ---- discriminator backward (autograd of Discriminator.forward, models.py:87-103): no aten / cuDNN call is left --------
 * Conventions: dz = gradient w.r.t. a layer's PRE-activation output (i.e. already multiplied by LeakyReLU'), x = the layer's
 * input, dw = gradient of the layer's FOLDED weight in torch layout, db = bias gradient; mg_msd_wn_backward turns the layers'
 * dw into (d weight_v, d weight_g). */

/* The whole backward of discriminator `scale` in ONE call: the host side walks the seven layers from the logits down and
 * enqueues the kernels of the per-layer entry points below itself (what models._MSDFunction.backward uses).
 *   x0 [Bt][1][L0]: the discriminator's input (the pooled audio for scale > 0); fmap[7]: the maps the forward returned;
 *   gfmap[7]: gradient w.r.t. each returned map (NULL entries: none); gx0 [Bt][1][L0] or NULL (input gradient not needed);
 *   dw[7] / db[7]: outputs -- layers the gradient does not reach are left untouched and reported in reached[7] (host ints,
 *   may be NULL); workspace: bytes from the helper. */
size_t mg_msd_scale_backward_workspace_bytes(int Bt, int L0);
int mg_msd_scale_backward(const void *packed, int scale, const float *x0, const float *const *fmap, const float *const *gfmap,
                          float *gx0, float *const *dw, float *const *db, int *reached, void *workspace, size_t workspace_bytes,
                          int Bt, int L0, void *status_word, void *stream);

/* dz = (g1 + g2) * LeakyReLU'(out) over n elements (g2 may be NULL): the gradient entering a layer's pre-activation from the
 * next layer and from the feature-map loss, in one launch (F.leaky_relu backward of models.py:91,94,97 + the add). */
int mg_lrelu_backward(const float *g1, const float *g2, const float *out, float *dz, long long n, void *stream);

/* Gradients of ONE grouped conv (layer 1..4: k41, pad 20, 4 input channels per group, stride 4/4/4/1) of discriminator
 * `scale` of the packed MSD blob, each a single launch (cuDNN runs one kernel per group):
 *   dz [Bt][Cout][Lout], x [Bt][Cin][Lin]; dx [Bt][Cin][Lin] (NULL: skip), dw [Cout][4][41] + db [Cout] (dw NULL: skip both). */
size_t mg_msd_grouped_backward_workspace_bytes(int layer, int Bt, int Lout);
int mg_msd_grouped_backward(const void *packed, int scale, int layer, const float *dz, const float *x, float *dx, float *dw,
                            float *db, void *workspace, size_t workspace_bytes, int Bt, int Lin, int Lout, void *stream);

/* Data gradient of conv_post1 (Conv1d 1024 -> 1024, k5, pad 2; models.py:84,96) of discriminator `scale`: dz [Bt][1024][L]
 * -> dx [Bt][1024][L], on the same tensor-core kernel as the forward, streaming the transposed, tap-flipped copy of the weights
 * that mg_msd_pack / mg_disc_pack keep for it. */
int mg_msd_post1_dgrad(const void *packed, int scale, const float *dz, float *dx, int Bt, int L, void *status_word, void *stream);
/* Weight and bias gradient of conv_post1 (no weights needed): x [Bt][1024][L], dz [Bt][1024][L] -> dw [1024][1024][5],
 * db [1024]; one tensor-core launch, split-bf16 (fp32-grade) with fp32 accumulation over all Bt * L positions. */
int mg_msd_post1_wgrad(const float *x, const float *dz, float *dw, float *db, int Bt, int L, void *status_word, void *stream);

/* Backward of conv_pre (layer 0: Conv1d 1 -> 16, k15; x [Bt][1][L], dz [Bt][16][L], dw [16][1][15]) or conv_post2 (layer 6:
 * Conv1d 1024 -> 1, k3; x [Bt][1024][L], dz [Bt][1][L], dw [1][1024][3]) of discriminator `scale` (autograd of models.py:90,99):
 * dx (same shape as x; NULL: skip -- conv_pre's is only needed when the audio requires a gradient), dw, db.  fp32, fixed
 * summation order.  Layer 0 needs a workspace (bytes from the helper), layer 6 none. */
size_t mg_msd_edge_backward_workspace_bytes(int layer, int Bt, int L);
int mg_msd_edge_backward(const void *packed, int scale, int layer, const float *dz, const float *x, float *dx, float *dw, float *db,
                         void *workspace, size_t workspace_bytes, int Bt, int L, void *stream);

/* weight-norm backward of the 21 layers of an MSD blob in one launch: v, g, dw, dv, dg are HOST arrays of 21 device pointers
 * (dw[i] NULL: layer skipped):  dg = <dw, v> / |v|,  dv = (g / |v|) (dw - <dw, v> v / |v|^2) per norm row. */
int mg_msd_wn_backward(const float *const *v, const float *const *g, const float *const *dw, float *const *dv,
                       float *const *dg, void *stream);

/* ---- multi-tensor Adam (the optimizer step either side of the path: train.py:51-52,118,129) -------------------------
 * One launch updates `count` parameter tensors.  p, g, m, v: DEVICE arrays of `count` device pointers (parameter,
 * gradient, exp_avg, exp_avg_sq); n: DEVICE array of element counts; first: DEVICE array of count + 1 ints with
 * first[i] = sum_{j<i} ceil(n[j] / mg_adam_chunk()), total_ctas = first[count].  `step` is the 1-based step number of
 * this update.  Arithmetic of torch.optim.Adam (L2 weight decay, no amsgrad). */
int mg_adam_chunk(void);
int mg_adam_step(float *const *p, const float *const *g, float *const *m, float *const *v, const long long *n,
                 const int *first, int count, int total_ctas, float lr, float beta1, float beta2, float eps,
                 float weight_decay, long long step, void *stream);

/* ---- fused loss reductions (reference: feature_loss / discriminator_loss / generator_loss, models.py:138-167) ----
 * A loss is a table of `count` (<= 24) rows; out[i] = mean over the n[i] elements of
 *   mode 0: |a[i] - b[i]|   (one feature-map pair of feature_loss, models.py:142)
 *   mode 1: (1 - a[i])^2    (real term of discriminator_loss :151, generator_loss :165)
 *   mode 2: a[i]^2          (generated term of discriminator_loss :152)
 * (b[i] is ignored for modes 1, 2).  All rows are reduced by one launch plus a fixed-order combine (bit-reproducible);
 * `workspace` holds the per-CTA partial sums.  The caller scales / sums the row means (x10 for feature_loss).
 * mg_loss_backward writes grad_a[i] (and grad_b[i] for mode 0; either may be NULL) = grad_out[i] * d out[i] / d input;
 * grad_out is a DEVICE array of `count` floats. */
size_t mg_loss_workspace_bytes(const long long *n, int count);
int mg_loss_forward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count,
                    float *out, void *workspace, size_t workspace_bytes, void *stream);
int mg_loss_backward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count,
                     const float *grad_out, float *const *grad_a, float *const *grad_b, void *stream);

/* Number of kernels in the generator's chain (at most 16) and the name of the i-th one.  mg_gen_forward cuts
 * the batch into mg_gen_forward_slices(B, T) contiguous slices whose chains run concurrently on forked streams
 * (joined back into `stream` before it returns), so one forward enqueues slices x launches kernels.  A ragged batch is cut
 * by the same rule applied to its total frames, into groups of about equal frames. */
int mg_gen_forward_launches(void);
int mg_gen_forward_slices(int B, int T);
/* Selects the generator chain for the calling thread: bit i (1..3) of tail_mask = stage i's ConvT fused at the tail of
 * ResBlock i-1's kernel; 0 = one kernel per ConvT / ResBlock (all stage outputs materialised: mg_gen_stage_output works for
 * which = 1..3); -1 = the default (environment MG_GEN_TAIL, else none).  For tests and A/B measurements. */
int mg_gen_set_pipeline(int tail_mask);
const char *mg_gen_kernel_name(int i);
/* Template configuration of the i-th chain kernel at T mel frames per item (e.g. "resblock_tc_kernel<RbCfg<128,2,4,4,1,0,0,1,0,1>>/NH4"):
 * profile evidence (profiles/ ncu captures) records it, and bench.py only quotes a capture taken with the configuration this
 * build actually runs. */
const char *mg_gen_kernel_config(int i, int T);

#ifdef __cplusplus
}
#endif
#endif /* MELGAN_B200_H_ */
