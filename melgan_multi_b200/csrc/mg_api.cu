// C ABI of libmelgan_b200.so (see include/melgan_b200.h for the contract of every entry point).
#include <new>
#include <stdlib.h>
#include <string.h>

#include "mg_common.cuh"

namespace mg {

// (error plumbing: mg_error.cu.  The first-generation fp32 SIMT generator is NOT part of this library: it builds into the
//  test-only libmelgan_b200_simt_test.so, csrc/testlib.)

static int *status_ptr(void *workspace, int B, int T) {
    return reinterpret_cast<int *>(reinterpret_cast<float *>(workspace) + ws_offset(6, (size_t)B, (size_t)T));
}

// batch: mel lengths (stride T); mel_host / audio_host: optional pinned host buffers (the engine entry point); the copies
// ride on the batch slices' streams; pcm16: audio and audio_host hold int16 samples
static int run_generator(const float *mel, void *audio, const RunTable &batch, float *ws, cudaStream_t s,
                         cudaEvent_t *ev, const float *mel_host = nullptr, void *audio_host = nullptr,
                         int precision = MG_GEN_PRECISION_FP32, bool pcm16 = false) {
    int *st = status_ptr(ws, batch.items(), batch.stride);
    MG_CUDA_TRY(cudaMemsetAsync(st, 0, sizeof(int), s));
    return launch_generator_tc(mel, audio, batch, ws, st, s, ev, mel_host, audio_host, precision, pcm16);
}

int check_precision(const char *fn, int precision) {
    if (precision != MG_GEN_PRECISION_FP32 && precision != MG_GEN_PRECISION_BF16)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: unknown precision %d (MG_GEN_PRECISION_FP32 = 0, MG_GEN_PRECISION_BF16 = 1)", fn,
                         precision);
    return MG_OK;
}

int check_default_chain(const char *fn, const char *role) {
    if (!generator_tc_default_chain())
        return set_error(MG_ERR_INVALID_ARGUMENT,
                         "%s: %s only, but mg_gen_set_pipeline / MG_GEN_TAIL / MG_GEN_FUSE_UP selected another (tail mask %d, "
                         "front mask %d); mg_gen_set_pipeline(-1) restores the default",
                         fn, role, generator_tc_tail(), generator_tc_fused_up());
    return MG_OK;
}

static int check_shape(const char *fn, int B, int T) {
    if (B < 1 || T < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: need B >= 1 and T >= 1 (got B=%d, T=%d)", fn, B, T);
    if ((long long)B * T > (1ll << 24)) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B*T = %lld too large", fn, (long long)B * T);
    return MG_OK;
}

// Parity-test entry points run ONE kernel synchronously with their own status word: launch, wait, report a timed-out pipeline.
template <class F>
static int run_one_kernel(const char *fn, cudaStream_t stream, F launch) {
    int *st = nullptr;
    MG_CUDA_TRY(cudaMalloc(&st, sizeof(int)));
    cudaMemsetAsync(st, 0, sizeof(int), stream);
    int rc = launch(st);
    int h = 0;
    if (rc == MG_OK) {
        cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) rc = set_error(MG_ERR_CUDA, "%s: %s", fn, cudaGetErrorString(e));
        else if (cudaMemcpy(&h, st, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess || h)
            rc = set_error(MG_ERR_CUDA, "%s: pipeline wait timed out (role code %d)", fn, h);
    }
    cudaFree(st);
    return rc;
}

}  // namespace mg

using namespace mg;

/* ------------------------------- multi-resolution STFT loss ------------------------------ */

size_t mg_stft_loss_tables_bytes(int n_fft) { return stft_tables_bytes(n_fft); }

int mg_stft_loss_tables_build(int n_fft, int win_length, void *tables_host) { return stft_tables_build(n_fft, win_length, tables_host); }

int mg_stft_loss_frames(int n_fft, int hop, int L) { return stft_frames(n_fft, hop, L); }

int mg_stft_loss_workspace_bytes(int n_res, const int *n_fft, const int *hop, int B, int L, size_t *forward_bytes,
                                 size_t *backward_bytes) {
    const char *fn = "mg_stft_loss_workspace_bytes";
    if (!forward_bytes || !backward_bytes)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, !forward_bytes ? "forward_bytes" : "backward_bytes");
    *forward_bytes = *backward_bytes = 0;
    int T[8];
    const int rc = stft_check(fn, n_res, nullptr, n_fft, hop, B, L, T);
    if (rc) return rc;
    stft_workspace(n_res, n_fft, B, T, forward_bytes, backward_bytes);
    return MG_OK;
}

static int stft_check_pointer(const char *fn, const char *name, const void *p, unsigned align) {
    if (!p) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, name);
    if ((uintptr_t)p % align) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s must be %u-byte aligned", fn, name, align);
    return MG_OK;
}

int mg_stft_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                         int B, int L, float *sc_loss, float *mag_loss, void *workspace, size_t workspace_bytes, void *stream) {
    const char *fn = "mg_stft_loss_forward";
    int rc, T[8];
    if (!tables && n_res >= 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables is NULL", fn);
    if ((rc = stft_check(fn, n_res, tables, n_fft, hop, B, L, T))) return rc;
    if ((rc = stft_check_pointer(fn, "x", x, 4)) || (rc = stft_check_pointer(fn, "y", y, 4)) ||
        (rc = stft_check_pointer(fn, "sc_loss", sc_loss, 4)) || (rc = stft_check_pointer(fn, "mag_loss", mag_loss, 4)) ||
        (rc = stft_check_pointer(fn, "workspace", workspace, 16)))
        return rc;
    size_t need, unused;
    stft_workspace(n_res, n_fft, B, T, &need, &unused);
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
    return launch_stft_loss_forward(n_res, tables, n_fft, hop, x, y, B, L, T, sc_loss, mag_loss, workspace, (cudaStream_t)stream);
}

int mg_stft_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y,
                          int B, int L, const float *grad_sc, const float *grad_mag, const void *forward_workspace, float *grad_x,
                          void *workspace, size_t workspace_bytes, void *stream) {
    const char *fn = "mg_stft_loss_backward";
    int rc, T[8];
    if (!tables && n_res >= 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables is NULL", fn);
    if ((rc = stft_check(fn, n_res, tables, n_fft, hop, B, L, T))) return rc;
    if ((rc = stft_check_pointer(fn, "x", x, 4)) || (rc = stft_check_pointer(fn, "y", y, 4)) ||
        (rc = stft_check_pointer(fn, "grad_sc", grad_sc, 4)) || (rc = stft_check_pointer(fn, "grad_mag", grad_mag, 4)) ||
        (rc = stft_check_pointer(fn, "forward_workspace", forward_workspace, 16)) ||
        (rc = stft_check_pointer(fn, "grad_x", grad_x, 4)) || (rc = stft_check_pointer(fn, "workspace", workspace, 16)))
        return rc;
    size_t unused, need;
    stft_workspace(n_res, n_fft, B, T, &unused, &need);
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
    return launch_stft_loss_backward(n_res, tables, n_fft, hop, x, y, B, L, T, grad_sc, grad_mag, forward_workspace, grad_x, workspace,
                                     (cudaStream_t)stream);
}

/* ------------------------------- multi-resolution mel loss ------------------------------- */

size_t mg_mel_loss_tables_bytes(int n_fft) { return mel_loss_tables_bytes(n_fft); }

int mg_mel_loss_tables_build(int n_fft, int win_length, int sampling_rate, int n_mels, float fmin, float fmax, void *tables_host) {
    return mel_loss_tables_build(n_fft, win_length, sampling_rate, n_mels, fmin, fmax, tables_host);
}

int mg_mel_loss_frames(int n_fft, int hop, int L) { return mel_loss_frames(n_fft, hop, L); }

int mg_mel_loss_workspace_bytes(int n_res, const int *n_fft, const int *hop, int B, int L, size_t *forward_bytes,
                                size_t *backward_bytes) {
    const char *fn = "mg_mel_loss_workspace_bytes";
    if (!forward_bytes || !backward_bytes)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %s is NULL", fn, !forward_bytes ? "forward_bytes" : "backward_bytes");
    *forward_bytes = *backward_bytes = 0;
    int T[8];
    const int rc = mel_loss_check(fn, n_res, nullptr, n_fft, hop, B, L, T);
    if (rc) return rc;
    mel_loss_workspace(n_res, n_fft, B, T, forward_bytes, backward_bytes);
    return MG_OK;
}

int mg_mel_loss_forward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y, int B,
                        int L, float *loss, void *workspace, size_t workspace_bytes, void *stream) {
    const char *fn = "mg_mel_loss_forward";
    int rc, T[8];
    if (!tables && n_res >= 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables is NULL", fn);
    if ((rc = mel_loss_check(fn, n_res, tables, n_fft, hop, B, L, T))) return rc;
    if ((rc = stft_check_pointer(fn, "x", x, 4)) || (rc = stft_check_pointer(fn, "y", y, 4)) ||
        (rc = stft_check_pointer(fn, "loss", loss, 4)) || (rc = stft_check_pointer(fn, "workspace", workspace, 16)))
        return rc;
    size_t need, unused;
    mel_loss_workspace(n_res, n_fft, B, T, &need, &unused);
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
    return launch_mel_loss_forward(n_res, tables, n_fft, hop, x, y, B, L, T, loss, workspace, (cudaStream_t)stream);
}

int mg_mel_loss_backward(int n_res, const void *const *tables, const int *n_fft, const int *hop, const float *x, const float *y, int B,
                         int L, const float *grad, float *grad_x, void *workspace, size_t workspace_bytes, void *stream) {
    const char *fn = "mg_mel_loss_backward";
    int rc, T[8];
    if (!tables && n_res >= 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables is NULL", fn);
    if ((rc = mel_loss_check(fn, n_res, tables, n_fft, hop, B, L, T))) return rc;
    if ((rc = stft_check_pointer(fn, "x", x, 4)) || (rc = stft_check_pointer(fn, "y", y, 4)) ||
        (rc = stft_check_pointer(fn, "grad", grad, 4)) || (rc = stft_check_pointer(fn, "grad_x", grad_x, 4)) ||
        (rc = stft_check_pointer(fn, "workspace", workspace, 16)))
        return rc;
    size_t unused, need;
    mel_loss_workspace(n_res, n_fft, B, T, &unused, &need);
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace of %zu bytes, %zu needed", fn, workspace_bytes, need);
    return launch_mel_loss_backward(n_res, tables, n_fft, hop, x, y, B, L, T, grad, grad_x, workspace, (cudaStream_t)stream);
}

/* ------------------------------- host-buffer engine ------------------------------------- */

struct mg_gen_engine {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float *packed = nullptr;
    float *raw = nullptr;  // device staging for raw v/g/bias
    float *mel = nullptr, *audio = nullptr, *ws = nullptr;
    float *pin_in = nullptr, *pin_out = nullptr;  // (audio and pin_out hold int16 samples after a pcm16 forward)
    int *pin_status = nullptr;
    size_t cap_frames = 0;  // B*T capacity
    bool loaded = false;
    float last_ms = 0.f;
};

static void engine_free_io(mg_gen_engine *e) {
    cudaFree(e->mel); cudaFree(e->audio); cudaFree(e->ws);
    cudaFreeHost(e->pin_in); cudaFreeHost(e->pin_out);
    e->mel = e->audio = e->ws = e->pin_in = e->pin_out = nullptr;
    e->cap_frames = 0;
}

static int engine_reserve(mg_gen_engine *e, size_t frames) {
    if (frames <= e->cap_frames) return MG_OK;
    engine_free_io(e);
    MG_CUDA_TRY(cudaMalloc(&e->mel, frames * kMelBins * sizeof(float)));
    MG_CUDA_TRY(cudaMalloc(&e->audio, frames * 256 * sizeof(float)));
    MG_CUDA_TRY(cudaMalloc(&e->ws, mg_gen_workspace_bytes(1, (int)frames)));
    MG_CUDA_TRY(cudaMallocHost(&e->pin_in, frames * kMelBins * sizeof(float)));
    MG_CUDA_TRY(cudaMallocHost(&e->pin_out, frames * 256 * sizeof(float)));
    e->cap_frames = frames;
    return MG_OK;
}

// pcm16: audio_host receives int16 samples; the device audio and the pinned staging are then read as int16, so the
// download moves half the bytes
static int engine_forward(mg_gen_engine *e, const float *mel_host, void *audio_host, const RunTable &batch,
                          int precision = MG_GEN_PRECISION_FP32, bool pcm16 = false) {
    const int B = batch.items(), T = batch.stride;
    const size_t frames = (size_t)B * T;
    int rc = engine_reserve(e, frames);
    if (rc) return rc;
    const size_t nin = frames * kMelBins * sizeof(float), nout = frames * 256 * (pcm16 ? sizeof(int16_t) : sizeof(float));
    cudaPointerAttributes at;
    const bool in_pinned = cudaPointerGetAttributes(&at, mel_host) == cudaSuccess && at.type == cudaMemoryTypeHost;
    const bool out_pinned = cudaPointerGetAttributes(&at, audio_host) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();  // clear "invalid value" some drivers raise for pageable pointers
    const float *src = mel_host;
    if (!in_pinned) { memcpy(e->pin_in, mel_host, nin); src = e->pin_in; }
    if (!e->pin_status) MG_CUDA_TRY(cudaMallocHost(&e->pin_status, sizeof(int)));
    MG_CUDA_TRY(cudaEventRecord(e->ev0, e->stream));
    // upload, kernels and download are enqueued per batch slice (launch_generator_tc); one synchronisation at the end
    rc = run_generator(e->mel, e->audio, batch, e->ws, e->stream, nullptr, src, out_pinned ? audio_host : (void *)e->pin_out,
                       precision, pcm16);
    if (rc) return rc;
    MG_CUDA_TRY(cudaEventRecord(e->ev1, e->stream));
    *e->pin_status = 0;
    MG_CUDA_TRY(cudaMemcpyAsync(e->pin_status, status_ptr(e->ws, B, T), sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    MG_CUDA_TRY(cudaStreamSynchronize(e->stream));
    if (!out_pinned) memcpy(audio_host, e->pin_out, nout);
    if (*e->pin_status)
        return set_error(MG_ERR_CUDA, "mg_gen_engine_forward: tensor-core pipeline wait timed out (code %d)", *e->pin_status);
    MG_CUDA_TRY(cudaEventElapsedTime(&e->last_ms, e->ev0, e->ev1));
    return MG_OK;
}

/* ------------------------------- generator forward -------------------------------------- */

namespace mg {

// What a forward entry point asks of the shared rules beyond those every one applies (ForwardCall::rules)
enum : unsigned {
    kBlobArray = 1,         // packed is the caller's array of n_voices blobs, each checked ("packed[i] is NULL")
    kNeedVoice = 2,         // voice must not be NULL
    kNeedLengths = 4,       // lengths must not be NULL
    kDefaultChainOnly = 8,  // any other chain is refused at fp32 too (the multi-voice and int16 kernels exist only there)
    kPcm16 = 16,            // audio holds int16 samples
    kHost = 32,             // mel and audio are host buffers; engine holds the weights and the workspace
};

// One generator forward as an entry point received it.  The device-pointer entry points pass packed, ws, ws_bytes and
// stream (a single-pointer one passes its pointer's address and n_voices = 1); the host-buffer ones pass engine.
struct ForwardCall {
    const char *fn;
    unsigned rules;
    const void *const *packed;
    int n_voices;
    const int *voice;
    const float *mel;
    void *audio;
    int B, T;
    const int *lengths;
    int precision;
    void *ws;
    size_t ws_bytes;
    void *stream;
    mg_gen_engine *engine;
};

// The rules of every generator forward in the order they are checked; the first one broken is reported, before any CUDA
// call:
//   1. precision is MG_GEN_PRECISION_FP32 or MG_GEN_PRECISION_BF16;
//   2. the chain is the default one, at bf16 or under kDefaultChainOnly;
//   3. kBlobArray: n_voices >= 1, packed (and voice, kNeedVoice) not NULL, every blob non-NULL and 16-byte aligned;
//   4. B >= 1, T >= 1, B*T <= 2^24;
//   5. lengths not NULL (kNeedLengths); without voice ids a ragged batch has at most MG_GEN_RAGGED_MAX_B items; item by
//      item, voice[i] in [0, n_voices) and lengths[i] in [1, T];
//   6. with voice ids, at most MG_GEN_RAGGED_MAX_B runs of equal length and voice;
//   7. device calls: packed, mel, audio and workspace not NULL, a workspace of mg_gen_workspace_bytes(B, T) bytes
//      (else MG_ERR_WORKSPACE_TOO_SMALL), packed and workspace 16-byte aligned; host-buffer calls: engine, mel and audio
//      not NULL, weights loaded.
static int check_forward(const ForwardCall &c) {
    const char *fn = c.fn;
    const bool bf16 = c.precision == MG_GEN_PRECISION_BF16;
    int rc = check_precision(fn, c.precision);
    if (!rc && (bf16 || (c.rules & kDefaultChainOnly)))
        rc = check_default_chain(fn, bf16 ? "bf16 runs on the default chain" : "runs the default chain");
    if (rc) return rc;
    if (c.rules & kBlobArray) {
        if (c.n_voices < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: n_voices = %d, need at least 1", fn, c.n_voices);
        if (!c.packed || ((c.rules & kNeedVoice) && !c.voice))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null packed%s array", fn, c.rules & kNeedVoice ? " or voice" : "");
        for (int v = 0; v < c.n_voices; ++v) {
            if (!c.packed[v]) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed[%d] is NULL", fn, v);
            if ((uintptr_t)c.packed[v] % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed[%d] must be 16-byte aligned", fn, v);
        }
    }
    if ((rc = check_shape(fn, c.B, c.T))) return rc;
    if ((c.rules & kNeedLengths) && !c.lengths) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null lengths", fn);
    if (c.lengths && !c.voice && c.B > MG_GEN_RAGGED_MAX_B)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B = %d exceeds MG_GEN_RAGGED_MAX_B = %d", fn, c.B, MG_GEN_RAGGED_MAX_B);
    for (int i = 0; (c.voice || c.lengths) && i < c.B; ++i) {
        if (c.voice && (c.voice[i] < 0 || c.voice[i] >= c.n_voices))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: voice[%d] = %d is outside [0, n_voices = %d)", fn, i, c.voice[i],
                             c.n_voices);
        if (c.lengths && (c.lengths[i] < 1 || c.lengths[i] > c.T))
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: lengths[%d] = %d is outside [1, T_max = %d]", fn, i, c.lengths[i], c.T);
    }
    if (c.voice) {
        int runs = 1;  // what RunTable::voices merges: neighbours of equal length and blob
        for (int i = 1; i < c.B; ++i)
            runs += (c.lengths && c.lengths[i] != c.lengths[i - 1]) || c.packed[c.voice[i]] != c.packed[c.voice[i - 1]];
        if (runs > MG_GEN_RAGGED_MAX_B)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: %d runs of equal length and voice exceed MG_GEN_RAGGED_MAX_B = %d", fn,
                             runs, MG_GEN_RAGGED_MAX_B);
    }
    if (c.rules & kHost) {
        if (!c.engine || !c.mel || !c.audio) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
        if (!c.engine->loaded) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: no weights loaded", fn);
        return MG_OK;
    }
    if (!c.packed[0] || !c.mel || !c.audio || !c.ws) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    const size_t need = mg_gen_workspace_bytes(c.B, c.T);
    if (c.ws_bytes < need) return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "%s: workspace %zu < %zu bytes", fn, c.ws_bytes, need);
    if ((uintptr_t)c.packed[0] % 16 || (uintptr_t)c.ws % 16)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed/workspace must be 16-byte aligned", fn);
    return MG_OK;
}

// the batch table of a call check_forward accepted
static RunTable batch_table(const ForwardCall &c) {
    const float *const *blobs = c.rules & kHost ? &c.engine->packed : reinterpret_cast<const float *const *>(c.packed);
    if (c.voice) return RunTable::voices(c.lengths, c.B, c.T, blobs, c.voice);
    return c.lengths ? RunTable::ragged(c.lengths, c.B, c.T, blobs[0]) : RunTable::uniform(c.B, c.T, blobs[0]);
}

static int forward(const ForwardCall &c) {
    int rc = check_forward(c);
    if (rc) return rc;
    const RunTable t = batch_table(c);
    const bool pcm16 = c.rules & kPcm16;
    if (c.rules & kHost) return engine_forward(c.engine, c.mel, c.audio, t, c.precision, pcm16);
    return run_generator(c.mel, c.audio, t, (float *)c.ws, (cudaStream_t)c.stream, nullptr, nullptr, nullptr, c.precision, pcm16);
}

}  // namespace mg

extern "C" {

int mg_abi_version(void) { return 2; }

const char *mg_last_error_string(void) { return error_buffer(); }

int mg_device_check(void) {
    int dev = 0;
    MG_CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp p;
    MG_CUDA_TRY(cudaGetDeviceProperties(&p, dev));
    if (p.major != 9 || p.minor != 0)
        return set_error(MG_ERR_UNSUPPORTED_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a (H100) only",
                         dev, p.major, p.minor);
    return MG_OK;
}

size_t mg_gen_packed_bytes(void) { return packed_total_bytes(); }

int mg_gen_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, void *stream) {
    if (!v || !g || !bias || !packed) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_pack: null argument");
    if ((uintptr_t)packed % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_pack: packed must be 16-byte aligned");
    return launch_pack(v, g, bias, (float *)packed, (cudaStream_t)stream);
}

size_t mg_gen_workspace_bytes(int B, int T) {
    if (B < 1 || T < 1) return 0;
    return ws_offset(6, (size_t)B, (size_t)T) * sizeof(float) + 256;  // + pipeline status word
}

int mg_gen_forward(const void *packed, const float *mel, float *audio, int B, int T, void *workspace,
                   size_t workspace_bytes, void *stream) {
    return forward({"mg_gen_forward", 0, &packed, 1, nullptr, mel, audio, B, T, nullptr, MG_GEN_PRECISION_FP32, workspace,
                    workspace_bytes, stream});
}

int mg_gen_forward_ragged(const void *packed, const float *mel, float *audio, int B, int T_max, const int *lengths,
                          void *workspace, size_t workspace_bytes, void *stream) {
    return forward({"mg_gen_forward_ragged", kNeedLengths, &packed, 1, nullptr, mel, audio, B, T_max, lengths,
                    MG_GEN_PRECISION_FP32, workspace, workspace_bytes, stream});
}

int mg_gen_forward_precision(const void *packed, const float *mel, float *audio, int B, int T_max, const int *lengths,
                             int precision, void *workspace, size_t workspace_bytes, void *stream) {
    return forward({"mg_gen_forward_precision", 0, &packed, 1, nullptr, mel, audio, B, T_max, lengths, precision, workspace,
                    workspace_bytes, stream});
}

int mg_gen_forward_voices(const void *const *packed, int n_voices, const int *voice, const float *mel, float *audio, int B,
                          int T_max, const int *lengths, int precision, void *workspace, size_t workspace_bytes, void *stream) {
    return forward({"mg_gen_forward_voices", kBlobArray | kNeedVoice | kDefaultChainOnly, packed, n_voices, voice, mel, audio, B,
                    T_max, lengths, precision, workspace, workspace_bytes, stream});
}

int mg_gen_forward_pcm16(const void *const *packed, int n_voices, const int *voice, const float *mel, int16_t *audio, int B,
                         int T_max, const int *lengths, int precision, void *workspace, size_t workspace_bytes, void *stream) {
    return forward({"mg_gen_forward_pcm16", kBlobArray | kDefaultChainOnly | kPcm16, packed, n_voices, voice, mel, audio, B,
                    T_max, lengths, precision, workspace, workspace_bytes, stream});
}

int mg_gen_forward_timed(const void *packed, const float *mel, float *audio, int B, int T, void *workspace,
                         size_t workspace_bytes, void *stream, float *kernel_ms) {
    const ForwardCall c{"mg_gen_forward_timed", 0, &packed, 1, nullptr, mel, audio, B, T, nullptr, MG_GEN_PRECISION_FP32,
                        workspace, workspace_bytes, stream};
    int rc = kernel_ms ? check_forward(c) : set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_forward_timed: null argument");
    if (rc) return rc;
    const int n = mg_gen_forward_launches();  // events: one before each launch + one after the last
    cudaEvent_t ev[17];  // at most 12 kernels
    for (int i = 0; i <= n; ++i) MG_CUDA_TRY(cudaEventCreate(&ev[i]));
    rc = run_generator(mel, audio, batch_table(c), (float *)workspace, (cudaStream_t)stream, ev);
    if (rc == MG_OK) {
        cudaError_t e = cudaEventSynchronize(ev[n]);
        if (e != cudaSuccess) rc = set_error(MG_ERR_CUDA, "mg_gen_forward_timed: %s", cudaGetErrorString(e));
        for (int i = 0; i < n && rc == MG_OK; ++i)
            if (cudaEventElapsedTime(&kernel_ms[i], ev[i], ev[i + 1]) != cudaSuccess)
                rc = set_error(MG_ERR_CUDA, "mg_gen_forward_timed: cudaEventElapsedTime failed");
    }
    for (int i = 0; i <= n; ++i) cudaEventDestroy(ev[i]);
    return rc;
}

const char *mg_gen_kernel_name(int i) { return generator_tc_kernel_name(i); }

const char *mg_gen_kernel_config(int i, int T) { return generator_tc_kernel_config(i, T); }

int mg_gen_set_pipeline(int tail_mask) {
    if (tail_mask < -1 || tail_mask > 15) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_set_pipeline: mask %d", tail_mask);
    generator_tc_set_tail(tail_mask);
    return MG_OK;
}

int mg_gen_stage_output(const void *workspace, int which, float *out, int B, int T, void *stream) {
    int rc = check_shape("mg_gen_stage_output", B, T);
    if (rc) return rc;
    if (which < 0 || which > 3 || !workspace || !out)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_stage_output: which must be 0..3 (the last stage is fused with conv_post)");
    if (which > 0 && generator_tc_tail() != 0)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_stage_output: ResBlock outputs are not materialised while the next stage's "
                         "ConvT is fused at their kernel's tail; select the unfused chain with mg_gen_set_pipeline(0) first");
    const size_t off = ws_offset(which, B, T), n = ws_offset(which + 1, B, T) - off;
    MG_CUDA_TRY(cudaMemcpyAsync(out, (const float *)workspace + off, n * sizeof(float), cudaMemcpyDeviceToDevice,
                                (cudaStream_t)stream));
    return MG_OK;
}

size_t mg_msd_grouped_backward_workspace_bytes(int layer, int Bt, int Lout) {
    if (layer < 1 || layer > 4 || Bt < 1 || Lout < 1) return 0;
    return grouped_bwd_workspace_bytes(layer, Bt, Lout);
}

int mg_msd_grouped_backward(const void *packed, int scale, int layer, const float *dz, const float *x, float *dx, float *dw,
                            float *db, void *workspace, size_t workspace_bytes, int Bt, int Lin, int Lout, void *stream) {
    if (!packed || !dz || scale < 0 || scale > 2 || layer < 1 || layer > 4 || Bt < 1 || Lin < 1 || Lout < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_grouped_backward: bad argument");
    const DLayer d = d_layer(layer);
    if (Lout != (Lin + 2 * d.pad - d.k) / d.stride + 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_grouped_backward: Lout %d does not follow from Lin %d", Lout, Lin);
    if (dw && (!x || !db || !workspace || workspace_bytes < grouped_bwd_workspace_bytes(layer, Bt, Lout)))
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "mg_msd_grouped_backward: dw needs x, db and a workspace of %zu bytes",
                         grouped_bwd_workspace_bytes(layer, Bt, Lout));
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(packed) + (size_t)scale * d_blob_bytes();
    return launch_disc_grouped_backward(blob, layer, dz, x, dx, dw, db, (float *)workspace, Bt, Lin, Lout, (cudaStream_t)stream);
}

int mg_msd_post1_dgrad(const void *packed, int scale, const float *dz, float *dx, int Bt, int L, void *status_word, void *stream) {
    if (!packed || !dz || !dx || dz == dx || !status_word || scale < 0 || scale > 2 || Bt < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_post1_dgrad: bad argument");
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(packed) + (size_t)scale * d_blob_bytes();
    return launch_disc_post1_dgrad_tc(dz, dx, blob + d_tcT_start(), reinterpret_cast<const float *>(blob + d_zero_start()), Bt, L,
                                      (int *)status_word, (cudaStream_t)stream);
}

int mg_msd_post1_wgrad(const float *x, const float *dz, float *dw, float *db, int Bt, int L, void *status_word, void *stream) {
    if (!x || !dz || !dw || !db || !status_word || Bt < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_post1_wgrad: bad argument");
    return launch_disc_post1_wgrad_tc(x, dz, dw, db, Bt, L, (int *)status_word, (cudaStream_t)stream);
}

size_t mg_msd_edge_backward_workspace_bytes(int layer, int Bt, int L) {
    return (layer == 0 && Bt > 0 && L > 0) ? edge_bwd_workspace_bytes(layer, Bt, L) : 0;
}

int mg_msd_edge_backward(const void *packed, int scale, int layer, const float *dz, const float *x, float *dx, float *dw, float *db,
                         void *workspace, size_t workspace_bytes, int Bt, int L, void *stream) {
    if (!packed || !dz || !x || !dw || !db || scale < 0 || scale > 2 || (layer != 0 && layer != 6) || Bt < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_edge_backward: bad argument (layer is 0 = conv_pre or 6 = conv_post2)");
    if (layer == 0 && (!workspace || workspace_bytes < edge_bwd_workspace_bytes(0, Bt, L)))
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "mg_msd_edge_backward: conv_pre needs a workspace of %zu bytes",
                         edge_bwd_workspace_bytes(0, Bt, L));
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(packed) + (size_t)scale * d_blob_bytes();
    return launch_disc_edge_backward(blob, layer, dz, x, dx, dw, db, (float *)workspace, Bt, L, (cudaStream_t)stream);
}

size_t mg_msd_scale_backward_workspace_bytes(int Bt, int L0) {
    return (Bt > 0 && L0 > 0) ? disc_scale_backward_workspace_bytes(Bt, L0) : 0;
}

int mg_msd_scale_backward(const void *packed, int scale, const float *x0, const float *const *fmap, const float *const *gfmap,
                          float *gx0, float *const *dw, float *const *db, int *reached, void *workspace, size_t workspace_bytes,
                          int Bt, int L0, void *status_word, void *stream) {
    if (!packed || !x0 || !fmap || !gfmap || !dw || !db || !workspace || !status_word || scale < 0 || scale > 2 || Bt < 1 || L0 < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_scale_backward: bad argument");
    for (int l = 0; l < kDiscLayers; ++l)
        if (!fmap[l]) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_scale_backward: fmap[%d] is NULL", l);
    if (Bt > 65535) return set_error(MG_ERR_INVALID_ARGUMENT, "discriminator batch %d exceeds 65535", Bt);
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(packed) + (size_t)scale * d_blob_bytes();
    return launch_disc_scale_backward(blob, x0, fmap, gfmap, gx0, dw, db, reached, workspace, workspace_bytes, Bt, L0,
                                      (int *)status_word, (cudaStream_t)stream);
}

int mg_lrelu_backward(const float *g1, const float *g2, const float *out, float *dz, long long n, void *stream) {
    return launch_lrelu_grad(g1, g2, out, dz, n, (cudaStream_t)stream);
}

int mg_msd_wn_backward(const float *const *v, const float *const *g, const float *const *dw, float *const *dv,
                       float *const *dg, void *stream) {
    if (!v || !g || !dw || !dv || !dg) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_wn_backward: null argument");
    return launch_disc_wn_backward(v, g, dw, dv, dg, (cudaStream_t)stream);
}

int mg_adam_chunk(void) { return 4096; }

int mg_adam_step(float *const *p, const float *const *g, float *const *m, float *const *v, const long long *n,
                 const int *first, int count, int total_ctas, float lr, float beta1, float beta2, float eps,
                 float weight_decay, long long step, void *stream) {
    return launch_adam(p, g, m, v, n, first, count, total_ctas, lr, beta1, beta2, eps, weight_decay, step, (cudaStream_t)stream);
}

size_t mg_loss_workspace_bytes(const long long *n, int count) {
    if (!n || count < 1) return 0;
    return (size_t)loss_num_ctas(n, count) * sizeof(float);
}

int mg_loss_forward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count,
                    float *out, void *workspace, size_t workspace_bytes, void *stream) {
    if (!out || !workspace) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_loss_forward: null argument");
    if (n && count >= 1 && workspace_bytes < mg_loss_workspace_bytes(n, count))
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "mg_loss_forward: workspace too small");
    return launch_loss_forward(a, b, n, mode, count, out, (float *)workspace, (cudaStream_t)stream);
}

int mg_loss_backward(const float *const *a, const float *const *b, const long long *n, const int *mode, int count,
                     const float *grad_out, float *const *grad_a, float *const *grad_b, void *stream) {
    if (!grad_out) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_loss_backward: null grad_out");
    return launch_loss_backward(a, b, n, mode, count, grad_out, grad_a, grad_b, (cudaStream_t)stream);
}

int mg_gen_forward_launches(void) { return generator_tc_num_launches(); }

int mg_gen_forward_slices(int B, int T) { return (B >= 1 && T >= 1) ? generator_tc_slices(B, (long long)B * T) : 1; }

int mg_gen_check_status(const void *workspace, int B, int T, void *stream) {
    int rc = check_shape("mg_gen_check_status", B, T);
    if (rc) return rc;
    if (!workspace) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_check_status: null workspace");
    MG_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    int st = 0;
    MG_CUDA_TRY(cudaMemcpy(&st, status_ptr(const_cast<void *>(workspace), B, T), sizeof(int), cudaMemcpyDeviceToHost));
    if (st) return set_error(MG_ERR_CUDA, "tensor-core pipeline wait timed out (role code %d)", st);
    return MG_OK;
}

int mg_gen_convt(const void *packed, int stage, const float *x, float *y, int B, int Lin, void *stream) {
    if (!packed || !x || !y || x == y || stage < 0 || stage > 3 || B < 1 || Lin < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_convt: bad argument");
    return run_one_kernel("mg_gen_convt", (cudaStream_t)stream, [&](int *st) {
        return launch_convt_tc(x, y, stage, RunTable::uniform(B, Lin, (const float *)packed), st, (cudaStream_t)stream);
    });
}

int mg_gen_conv_pre(const void *packed, const float *mel, float *y, int B, int T, void *stream) {
    if (!packed || !mel || !y || B < 1 || T < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_conv_pre: bad argument");
    return run_one_kernel("mg_gen_conv_pre", (cudaStream_t)stream, [&](int *st) {
        return launch_gen_pre_tc(mel, y, RunTable::uniform(B, T, (const float *)packed), st, (cudaStream_t)stream);
    });
}

int mg_gen_resblock_post(const void *packed, const float *x, float *audio, int B, int L, void *stream) {
    if (!packed || !x || !audio || B < 1 || L < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_resblock_post: bad argument");
    return run_one_kernel("mg_gen_resblock_post", (cudaStream_t)stream, [&](int *st) {
        return launch_resblock_tc(x, audio, 4, RunTable::uniform(B, L, (const float *)packed), st, (cudaStream_t)stream);
    });
}

/* Diagnostic: runs one tensor-core ResBlock and returns clock64 stamps of thread 0 of one interior CTA in trace[0..127]
 * (host buffer) for any stage code of resblock_config_name: [0] start, [1] input loaded, per conv c: [2+3c] X handed to the
 * MMAs (the interval from [1+3c] holds only shared-memory work: the conv biases are staged before griddepcontrol.wait),
 * [3+3c] accumulator ready,
 * [4+3c] next X written, [20] output stored; the same thread's MMA issue: [64+3c] X received, [65+3c] first weights
 * landed, [66+3c] last MMA issued.  Clustered stages (0, 1): [88+2c] / [89+2c] before / after the wait for the cluster
 * neighbours' border rows of conv c's input, [100+2k] / [101+2k] before / after the wait until the neighbours' MMAs of
 * conv k-1 have released their slack rows (hand-off k = 1..5), and [127] = cudaOccupancyMaxActiveClusters of the launch. */
int mg_gen_resblock_trace(const void *packed, int stage, const float *x, float *y, int B, int L, long long *trace_host) {
    if (!packed || !x || !y || x == y || !trace_host || !*resblock_config_name(stage, 0) || B < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_resblock_trace: bad argument");
    int *st = nullptr;
    long long *tr = nullptr;
    MG_CUDA_TRY(cudaMalloc(&st, sizeof(int)));
    MG_CUDA_TRY(cudaMalloc(&tr, 128 * sizeof(long long)));
    cudaMemset(st, 0, sizeof(int));
    cudaMemset(tr, 0, 128 * sizeof(long long));
    int rc = launch_resblock_tc(x, y, stage, RunTable::uniform(B, L, (const float *)packed), st, 0, tr);
    if (rc == MG_OK && cudaDeviceSynchronize() != cudaSuccess) rc = set_error(MG_ERR_CUDA, "mg_gen_resblock_trace: kernel failed");
    if (rc == MG_OK) cudaMemcpy(trace_host, tr, 128 * sizeof(long long), cudaMemcpyDeviceToHost);
    cudaFree(st);
    cudaFree(tr);
    return rc;
}

int mg_gen_resblock(const void *packed, int stage, const float *x, float *y, int B, int L, void *stream) {
    if (!packed || !x || !y || x == y || stage < 0 || stage > 3 || B < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_resblock: bad argument");
    return run_one_kernel("mg_gen_resblock", (cudaStream_t)stream, [&](int *st) {
        return launch_resblock_tc(x, y, stage, RunTable::uniform(B, L, (const float *)packed), st, (cudaStream_t)stream);
    });
}

int mg_gen_resup(const void *packed, int stage, const float *x, float *y, int B, int L, void *stream) {
    if (!packed || !x || !y || x == y || stage < 0 || stage > 2 || B < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_resup: bad argument");
    return run_one_kernel("mg_gen_resup", (cudaStream_t)stream, [&](int *st) {
        return launch_resblock_tc(x, y, 20 + stage, RunTable::uniform(B, L, (const float *)packed), st, (cudaStream_t)stream);
    });
}

int mg_gen_upres(const void *packed, int stage, const float *x, float *y, int B, int Lin, void *stream) {
    if (!packed || !x || !y || x == y || (stage != 2 && stage != 3) || B < 1 || Lin < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_upres: bad argument");
    return run_one_kernel("mg_gen_upres", (cudaStream_t)stream, [&](int *st) {
        return launch_resblock_tc(x, y, 10 + stage, RunTable::uniform(B, 2 * Lin, (const float *)packed), st, (cudaStream_t)stream);
    });
}

int mg_gen_upres_post(const void *packed, const float *x, float *audio, int B, int Lin, void *stream) {
    if (!packed || !x || !audio || (const void *)x == (const void *)audio || B < 1 || Lin < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_upres_post: bad argument");
    return run_one_kernel("mg_gen_upres_post", (cudaStream_t)stream, [&](int *st) {
        return launch_resblock_tc(x, audio, 14, RunTable::uniform(B, 2 * Lin, (const float *)packed), st, (cudaStream_t)stream);
    });
}

const char *mg_gen_resblock_config(int code) { return resblock_config_name(code, 0); }
size_t mg_gen_tc_weight_offset(int front, int layer, int co, int ci, int tap, int h) {
    if (h < 0 || h > 1 || co < 0 || ci < 0 || tap < 0) return (size_t)-1;
    if (front) {
        if (layer < 2 || layer > 3 || tap > 3) return (size_t)-1;
        const int C = stage_cout(layer);
        if (co >= C || ci >= 2 * C) return (size_t)-1;
        return tc_region_start() + tc_upf_offset(layer) + 2 * upf_weight_index(C, ci, co, tap, h);
    }
    if (layer < 0) return (size_t)-1;
    if (layer == 0) {  // conv_pre, w[co][ci][tap]
        if (co >= kPreCout || ci >= kMelBins || tap >= kPreK) return (size_t)-1;
        return tc_region_start() + tc_pre_offset() + 2 * conv_tc_weight_index(kMelBins, kPreK, kPreNG, co, ci, tap, h);
    }
    if (layer <= 4) {  // ups[layer - 1], W[ci][co][tap], tap < 2 S
        const int s = layer - 1;
        if (co >= stage_cout(s) || ci >= stage_cin(s) || tap >= stage_kup(s)) return (size_t)-1;
        return tc_region_start() + tc_up_offset(s) + 2 * up_weight_index(s, ci, co, tap, h);
    }
    if (layer > 28 || tap > 2) return (size_t)-1;
    const int C = layer_shape(layer).cout;
    if (co >= C || ci >= C) return (size_t)-1;
    return tc_region_start() + tc_res_offset(layer) + 2 * tc_weight_index(C, co, ci, tap, h);
}
const char *mg_gen_convt_config(int stage) { return convt_config_name(stage); }
const char *mg_gen_conv_pre_config(void) { return gen_pre_config_name(); }

int mg_gen_chain_kernel(const void *packed, int k, const float *x, float *y, int B, int L_max, const int *lengths, int precision,
                        void *stream) {
    const char *fn = "mg_gen_chain_kernel";
    if (!packed || !x || !y) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if (x == y) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: x and y must differ", fn);
    if ((uintptr_t)packed % 16 || (uintptr_t)x % 16 || (uintptr_t)y % 16)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: packed, x and y must be 16-byte aligned", fn);
    if (k < 0 || k > 7) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: kernel %d is outside [0, 7]", fn, k);
    if (B < 1 || B > MG_GEN_RAGGED_MAX_B || L_max < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: need 1 <= B <= MG_GEN_RAGGED_MAX_B = %d and L_max >= 1 (got B=%d, L_max=%d)", fn,
                         MG_GEN_RAGGED_MAX_B, B, L_max);
    if ((long long)B * L_max > (1ll << 28)) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: B*L_max too large", fn);
    for (int i = 0; lengths && i < B; ++i)
        if (lengths[i] < 1 || lengths[i] > L_max)
            return set_error(MG_ERR_INVALID_ARGUMENT, "%s: lengths[%d] = %d is outside [1, L_max = %d]", fn, i, lengths[i], L_max);
    int rc = check_precision(fn, precision);
    if (!rc) rc = check_default_chain(fn, "runs the default chain's kernels");
    if (rc) return rc;
    const float *w = (const float *)packed;
    const RunTable t = lengths ? RunTable::ragged(lengths, B, L_max, w) : RunTable::uniform(B, L_max, w);
    return run_one_kernel(fn, (cudaStream_t)stream, [&](int *st) {
        return launch_chain_kernel(k, x, y, t, st, (cudaStream_t)stream, precision);
    });
}

/* ------------------------------- multi-scale discriminator ------------------------------- */

size_t mg_msd_packed_bytes(void) { return msd_packed_bytes(); }

int mg_msd_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, void *stream) {
    if (!v || !g || !bias || !packed) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_pack: null argument");
    if ((uintptr_t)packed % 256) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_pack: packed must be 256-byte aligned");
    return launch_disc_pack(v, g, bias, packed, (cudaStream_t)stream);
}

int mg_msd_lengths(int L, int *lens) {
    if (L < 1 || !lens) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_lengths: bad argument");
    msd_lengths(L, lens);
    for (int i = 0; i < 21; ++i)
        if (lens[i] < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_lengths: L = %d is too short for the discriminators", L);
    return MG_OK;
}

int mg_msd_forward(const void *packed, const float *y, int Bt, int L, float *const *fmaps, void *status_word, void *stream) {
    if (!packed || !y || !fmaps || !status_word || Bt < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_forward: bad argument");
    if (Bt > 65535)  // conv_pre, conv_post2 and the SIMT grouped convs put the items on grid.y / grid.z
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_forward: batch %d exceeds 65535 items", Bt);
    int lens[21];
    int rc = mg_msd_lengths(L, lens);
    if (rc) return rc;
    for (int i = 0; i < 21; ++i)
        if (!fmaps[i]) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_forward: null feature-map pointer %d", i);
    MG_CUDA_TRY(cudaMemsetAsync(status_word, 0, sizeof(int), (cudaStream_t)stream));
    return launch_msd_forward(packed, y, Bt, L, fmaps, (int *)status_word, (cudaStream_t)stream);
}

size_t mg_disc_packed_bytes(void) { return d_blob_bytes(); }

int mg_disc_pack(const float *const *v, const float *const *g, const float *const *bias, void *packed, void *stream) {
    if (!v || !g || !bias || !packed) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_pack: null argument");
    if ((uintptr_t)packed % 256) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_pack: packed must be 256-byte aligned");
    return launch_disc_pack(v, g, bias, packed, (cudaStream_t)stream, 1);
}

int mg_disc_forward(const void *packed, const float *x, int Bt, int L, float *const *fmaps, void *status_word, void *stream) {
    if (!packed || !x || !fmaps || !status_word || Bt < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_forward: bad argument");
    if (Bt > 65535) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_forward: batch %d exceeds 65535 items", Bt);
    int lens[21];
    msd_lengths(L, lens);
    for (int i = 0; i < 7; ++i) {
        if (lens[i] < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_forward: L = %d is too short", L);
        if (!fmaps[i]) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_disc_forward: null feature-map pointer %d", i);
    }
    MG_CUDA_TRY(cudaMemsetAsync(status_word, 0, sizeof(int), (cudaStream_t)stream));
    return launch_disc_forward(packed, x, Bt, L, fmaps, (int *)status_word, (cudaStream_t)stream);
}

int mg_msd_layer_forward(const void *packed, int scale, int layer, const float *x, float *out, int Bt, int Lin, void *status_word,
                         void *stream) {
    const char *fn = "mg_msd_layer_forward";
    if (!packed || !x || !out || !status_word) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: null argument", fn);
    if ((const void *)x == (const void *)out) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: x and out must differ", fn);
    if (scale < 0 || scale > 2) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: scale %d is outside [0, 2]", fn, scale);
    if (layer < 1 || layer >= kDiscLayers)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: layer %d is outside [1, %d]", fn, layer, kDiscLayers - 1);
    if (Bt < 1 || Bt > 65535)  // conv_post2 and the SIMT grouped convs put the items on grid.y / grid.z, as in mg_msd_forward
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: batch %d is outside [1, 65535]", fn, Bt);
    const DLayer d = d_layer(layer);
    const int Lout = Lin < 1 ? 0 : (Lin + 2 * d.pad - d.k) / d.stride + 1;
    if (Lout < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: Lin = %d gives no output at layer %d", fn, Lin, layer);
    if ((long long)Bt * d.cin * Lin > 0x7fffffffll || (long long)Bt * d.cout * Lout > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: Bt * C * L exceeds 2^31 - 1 elements", fn);
    const uint8_t *blob = reinterpret_cast<const uint8_t *>(packed) + (size_t)scale * d_blob_bytes();
    return launch_disc_layer_forward(blob, layer, x, out, Bt, Lin, Lout, (int *)status_word, (cudaStream_t)stream);
}

int mg_disc_tc_element(size_t offset, int *copy, int *co, int *ci, int *tap) {
    if (!copy || !co || !ci || !tap || offset % 2) return -1;
    int h = 2;
    if (offset >= d_gtc_start() && offset < d_gtc_start() + d_gtc_bytes()) {  // layers 1..3: d_gtc_index
        size_t rel = offset - d_gtc_start();
        int l = 1;
        while (rel >= d_gtc_offset(l + 1)) ++l;
        rel -= d_gtc_offset(l);
        const int grp = (int)(rel / d_gtc_group_bytes()), i = (int)(rel % d_gtc_group_bytes()) / 2;
        const int c = i & 3, pos = (i >> 2) & 1, n = (i >> 3) & 63, r = ((i >> 9) & 1) | (((i >> 10) & 1) << 1), kp = i >> 11;
        const int half = n >> 5, e = (n >> 4) & 1, q = 2 * kp + pos - 1 - e, k = 4 * q + r;
        *copy = l; *co = grp * 16 + (n & 15); *ci = c; *tap = k;
        if (q >= 0 && k <= 40) h = half;
    } else if (offset >= d_g4tc_start() && offset < d_g4tc_start() + d_g4tc_bytes()) {  // layer 4: d_g4tc_index
        const size_t rel = offset - d_g4tc_start();
        const int grp = (int)(rel / d_g4tc_group_bytes()), i = (int)(rel % d_g4tc_group_bytes()) / 2;
        const int j = i & 7, n = (i >> 3) & 63, c = ((i >> 9) & 1) | (((i >> 10) & 1) << 1), kp = i >> 11;
        const int half = n >> 5, e = (n >> 2) & 7, k = 8 * kp + j - e;
        *copy = 4; *co = grp * 4 + (n & 3); *ci = c; *tap = k;
        if (k >= 0 && k <= 40) h = half;
    } else {  // conv_post1: the forward copy (5) and the transposed, tap-flipped copy (6), conv_tc_weight_index
        const bool fwd = offset >= d_tc_start() && offset < d_tc_start() + d_tc_bytes();
        if (!fwd && !(offset >= d_tcT_start() && offset < d_tcT_start() + d_tc_bytes())) return -1;
        const size_t i = (offset - (fwd ? d_tc_start() : d_tcT_start())) / 2;
        const int c8 = (int)(i % 8), row = (int)((i / 8) % kPost1NG);
        size_t rest = i / (8 * kPost1NG);
        const int kh = (int)(rest % 2), half = (int)((rest / 2) % 2), t = (int)((rest / 4) % 5), c16 = (int)((rest / 20) % 64);
        const int a = (int)(rest / 1280) * kPost1NG + row, b = c16 * 16 + kh * 8 + c8;  // [a][b][t]: W[co][ci][tap] / W'[ci][co][4 - tap]
        *copy = fwd ? 5 : 6; *co = fwd ? a : b; *ci = fwd ? b : a; *tap = fwd ? t : 4 - t;
        h = half;
    }
    return h;
}

int mg_msd_check_status(const void *status_word, void *stream) {
    if (!status_word) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_check_status: null argument");
    MG_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    int st = 0;
    MG_CUDA_TRY(cudaMemcpy(&st, status_word, sizeof(int), cudaMemcpyDeviceToHost));
    if (st) return set_error(MG_ERR_CUDA, "tensor-core pipeline wait timed out (role code %d)", st);
    return MG_OK;
}

/* ------------------------------- mel-spectrogram front end -------------------------------- */

size_t mg_mel_tables_bytes(void) { return mel_tables_bytes(); }

int mg_mel_tables_build(int sampling_rate, int n_mels, float fmin, float fmax, int norm, void *tables_host) {
    if (!tables_host) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_tables_build: null buffer");
    return mel_tables_build(sampling_rate, n_mels, fmin, fmax, norm, reinterpret_cast<MelTables *>(tables_host));
}

int mg_mel_frames(int L) { return L < 1 ? 0 : mel_frames(L); }

int mg_mel_spectrogram(const void *tables, const float *audio, float *mel, int B, int L, void *stream) {
    if (!tables || !audio || !mel || B < 1 || L < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram: bad argument");
    if ((uintptr_t)tables % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram: tables must be 16-byte aligned");
    return launch_mel(tables, audio, mel, B, L, (cudaStream_t)stream);
}

size_t mg_mel_backward_workspace_bytes(int B, int L) { return mel_backward_workspace_bytes(B, L); }

int mg_mel_spectrogram_backward(const void *tables, const float *audio, const float *grad_mel, float *grad_audio, int B, int L,
                                void *workspace, size_t workspace_bytes, void *stream) {
    const char *fn = "mg_mel_spectrogram_backward";
    if (!tables || !audio || !grad_mel || !grad_audio || !workspace || B < 1 || L < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "%s: bad argument", fn);
    if ((uintptr_t)tables % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: tables must be 16-byte aligned", fn);
    if ((uintptr_t)workspace % 16) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: workspace must be 16-byte aligned", fn);
    return launch_mel_backward(tables, audio, grad_mel, grad_audio, B, L, workspace, workspace_bytes, (cudaStream_t)stream);
}

/* ------------------------------- host-buffer engine ------------------------------------- */

int mg_gen_engine_create(mg_gen_engine **out, int max_B, int max_T) {
    if (!out) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_engine_create: null out");
    int rc = check_shape("mg_gen_engine_create", max_B, max_T);
    if (rc) return rc;
    if ((rc = mg_device_check())) return rc;
    mg_gen_engine *e = new (std::nothrow) mg_gen_engine();
    if (!e) return set_error(MG_ERR_OUT_OF_MEMORY, "mg_gen_engine_create: host allocation failed");
    *out = e;
    MG_CUDA_TRY(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    MG_CUDA_TRY(cudaEventCreate(&e->ev0));
    MG_CUDA_TRY(cudaEventCreate(&e->ev1));
    MG_CUDA_TRY(cudaMalloc((void **)&e->packed, mg_gen_packed_bytes()));
    MG_CUDA_TRY(cudaMalloc(&e->raw, (packed_float_count() + 4353) * sizeof(float)));
    return engine_reserve(e, (size_t)max_B * max_T);
}

int mg_gen_engine_load_state(mg_gen_engine *e, const float *const *v, const float *const *g, const float *const *bias) {
    if (!e || !v || !g || !bias) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_engine_load_state: null argument");
    const float *dv[kNumLayers], *dg[kNumLayers], *db[kNumLayers];
    float *p = e->raw;
    for (int l = 0; l < kNumLayers; ++l) {
        if (!v[l] || !g[l] || !bias[l]) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_engine_load_state: null tensor, layer %d", l);
        const size_t nv = layer_weight_count(l), ng = layer_norm_rows(l), nb = layer_shape(l).cout;
        MG_CUDA_TRY(cudaMemcpyAsync(p, v[l], nv * sizeof(float), cudaMemcpyHostToDevice, e->stream)); dv[l] = p; p += nv;
        MG_CUDA_TRY(cudaMemcpyAsync(p, g[l], ng * sizeof(float), cudaMemcpyHostToDevice, e->stream)); dg[l] = p; p += ng;
        MG_CUDA_TRY(cudaMemcpyAsync(p, bias[l], nb * sizeof(float), cudaMemcpyHostToDevice, e->stream)); db[l] = p; p += nb;
    }
    int rc = launch_pack(dv, dg, db, e->packed, e->stream);
    if (rc) return rc;
    MG_CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->loaded = true;
    return MG_OK;
}

int mg_gen_engine_forward(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T) {
    return forward({"mg_gen_engine_forward", kHost, nullptr, 1, nullptr, mel_host, audio_host, B, T, nullptr,
                    MG_GEN_PRECISION_FP32, nullptr, 0, nullptr, e});
}

int mg_gen_engine_forward_ragged(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T_max, const int *lengths) {
    return forward({"mg_gen_engine_forward_ragged", kHost | kNeedLengths, nullptr, 1, nullptr, mel_host, audio_host, B, T_max,
                    lengths, MG_GEN_PRECISION_FP32, nullptr, 0, nullptr, e});
}

int mg_gen_engine_forward_precision(mg_gen_engine *e, const float *mel_host, float *audio_host, int B, int T_max,
                                    const int *lengths, int precision) {
    return forward({"mg_gen_engine_forward_precision", kHost, nullptr, 1, nullptr, mel_host, audio_host, B, T_max, lengths,
                    precision, nullptr, 0, nullptr, e});
}

int mg_gen_engine_forward_pcm16(mg_gen_engine *e, const float *mel_host, int16_t *audio_host, int B, int T_max, const int *lengths,
                                int precision) {
    return forward({"mg_gen_engine_forward_pcm16", kHost | kDefaultChainOnly | kPcm16, nullptr, 1, nullptr, mel_host, audio_host,
                    B, T_max, lengths, precision, nullptr, 0, nullptr, e});
}

int mg_gen_engine_last_kernel_ms(mg_gen_engine *e, float *ms) {
    if (!e || !ms) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_gen_engine_last_kernel_ms: null argument");
    *ms = e->last_ms;
    return MG_OK;
}

void mg_gen_engine_destroy(mg_gen_engine *e) {
    if (!e) return;
    engine_free_io(e);
    cudaFree(e->packed); cudaFree(e->raw);
    if (e->pin_status) cudaFreeHost(e->pin_status);
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

}  // extern "C"
