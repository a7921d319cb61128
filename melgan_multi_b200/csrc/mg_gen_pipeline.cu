// The generator's tensor-core pipeline: which kernels run, in what order, on which streams.
//   conv_pre -> 4 x [LeakyReLU -> ConvTranspose1d -> ResBlock] (-> LeakyReLU -> conv_post -> tanh), models.py:61-71,
// as 8 kernels per chain (mg_conv_tc.cu, mg_up_tc.cu, mg_res_tc.cu), the batch cut into concurrent slices.
#include <stdlib.h>

#include "mg_common.cuh"

namespace mg {

// Pipeline shape.  TAIL mask: bit i (i = 1..3) set = ConvTranspose of stage i runs at the TAIL of ResBlock i-1's kernel
// (mg_res_tc.cu, UPT): the chain is then  conv_pre, up0, res0+up1, res1+up2, res2+up3, res3+post  -- six kernels, no ResBlock
// output ever written to HBM.  Default: none (H100 80GB HBM3 at 700 W, config 2, bench.py: 1.96 ms per forward with no tail
// fusion, 1.99 with stage 3's, 2.04 with stage 1's, 2.06 with both, 2.07 with all three -- a tail ConvT's extra halo row
// and its un-overlapped per-group stores cost more than the HBM round trip it saves).  MG_GEN_TAIL=<digits> ("123", "0"
// for none) / mg_gen_set_pipeline() override it.  Where stage 3's ConvT is not at res2's tail it runs at the FRONT of the last
// kernel (UPF, "up3+res3+post") unless MG_GEN_FUSE_UP says otherwise (bit 0: stage 2 front-fused, bit 1: stage 3).
static thread_local int g_tail_override = -1;
void generator_tc_set_tail(int mask) { g_tail_override = mask; }
int generator_tc_tail() {
    static const int env_mask = [] {
        const char *e = getenv("MG_GEN_TAIL");
        if (!e) return 0;
        int m = 0;
        for (; *e; ++e) m |= (*e >= '1' && *e <= '3') ? 1 << (*e - '0') : 0;
        return m;
    }();
    return g_tail_override >= 0 ? (g_tail_override & 0b1110) : env_mask;
}
bool generator_tc_default_chain() { return generator_tc_tail() == 0 && generator_tc_fused_up() == 2; }
int generator_tc_fused_up() {
    static const int mask = [] {
        const char *e = getenv("MG_GEN_FUSE_UP");
        if (!e) return 2;
        int m = 0;
        for (; *e; ++e) m |= (*e == '2') ? 1 : (*e == '3') ? 2 : 0;
        return m;
    }();
    return mask;
}

// The chain as a list of steps (shared by the launcher, the launch counter and the kernel-name table).
struct ChainStep {
    const char *name;
    int kind;  // 0 conv_pre, 1 ConvT (arg = stage), 2 ResBlock kernel (arg = launch_resblock_tc code)
    int arg;
};
static int build_chain(ChainStep *st) {
    const int tail = generator_tc_tail(), front = generator_tc_fused_up();
    int n = 0;
    st[n++] = {"conv_pre", 0, 0};
    st[n++] = {"up0", 1, 0};
    if (tail & 2) st[n++] = {"res0+up1", 2, 20};
    else { st[n++] = {"res0", 2, 0}; st[n++] = {"up1", 1, 1}; }
    if (tail & 4) st[n++] = {"res1+up2", 2, 21};
    else if (front & 1) st[n++] = {"res1", 2, 1};
    else { st[n++] = {"res1", 2, 1}; st[n++] = {"up2", 1, 2}; }
    const bool front2 = !(tail & 4) && (front & 1);
    if (tail & 8) { st[n++] = {front2 ? "up2+res2+up3" : "res2+up3", 2, front2 ? -1 : 22}; st[n++] = {"res3+post", 2, 4}; }
    else if (front & 2) { st[n++] = {front2 ? "up2+res2" : "res2", 2, front2 ? 12 : 2}; st[n++] = {"up3+res3+post", 2, 14}; }
    else { st[n++] = {front2 ? "up2+res2" : "res2", 2, front2 ? 12 : 2}; st[n++] = {"up3", 1, 3}; st[n++] = {"res3+post", 2, 4}; }
    return n;
}
int generator_tc_num_launches() {
    ChainStep st[12];
    return build_chain(st);
}
const char *generator_tc_kernel_name(int i) {
    ChainStep st[12];
    const int n = build_chain(st);
    return (i >= 0 && i < n) ? st[i].name : "";
}

// template configuration of chain kernel i at T mel frames (what evidence files record; "" for non-ResBlock kernels)
const char *generator_tc_kernel_config(int i, int T) {
    ChainStep st[12];
    const int n = build_chain(st);
    if (i < 0 || i >= n || T < 1) return "";
    int len = T;
    for (int k = 0; k <= i; ++k) {
        if (st[k].kind == 1) len *= stage_stride(st[k].arg);
        else if (st[k].kind == 2) {
            const int a = st[k].arg;
            const int Lk = (a >= 12 && a <= 14) ? 2 * len : len;
            if (k == i) return resblock_config_name(a, Lk);
            len = a >= 20 ? Lk * stage_stride(a - 20 + 1) : Lk;
        }
    }
    return st[i].kind == 0 ? "conv_rows_tc_kernel<ConvCfg<80,512,7>>" : "convt_tc_kernel";
}

// Tensor-core pipeline of one contiguous slice of the batch (mel lengths, stride T_max).  a0: conv_pre output; a[0]:
// ResBlock-0 output (unfused chains); a[1], a[2], u: three buffers of 8192 T_max floats per item that the stages rotate
// through (a kernel never writes its input).  Every kernel gets the batch at its own scale.  precision goes to the ConvT
// and ResBlock kernels (conv_pre always runs its three passes).
static int generator_tc_chain(const float *packed, const float *mel, float *audio, const RunTable &batch, float *a0,
                              float *const *a, float *u, int *status, cudaStream_t s, cudaEvent_t *ev, int precision) {
    ChainStep st[12];
    const int n = build_chain(st);
    int rc;
    float *big[3] = {a[1], a[2], u};
    auto other = [&](const float *x, const float *y) -> float * {  // a rotation buffer that is neither x nor y
        for (float *b : big)
            if (b != x && b != y) return b;
        return nullptr;
    };
    const float *cur = mel;
    int len = 1;  // positions of `cur` per mel frame
    for (int i = 0; i < n; ++i) {
        if (ev) MG_CUDA_TRY(cudaEventRecord(ev[i], s));
        const ChainStep &k = st[i];
        if (k.kind == 0) {
            if ((rc = launch_gen_pre_tc(cur, a0, packed, batch, status, s))) return rc;
            cur = a0;
        } else if (k.kind == 1) {
            float *out = cur != u ? u : other(cur, nullptr);  // (unfused chain: ConvT outputs live in u, ResBlock i's in a[i])
            if ((rc = launch_convt_tc(cur, out, packed, k.arg, batch.scaled(len), status, s, precision))) return rc;
            cur = out;
            len *= stage_stride(k.arg);
        } else {
            if (k.arg < 0) return set_error(MG_ERR_INVALID_ARGUMENT, "generator pipeline: MG_GEN_FUSE_UP=2 cannot be combined with a tail-fused up3");
            const bool last = k.arg == 4 || k.arg == 14;
            const bool front = k.arg >= 12 && k.arg <= 14, tailf = k.arg >= 20;
            float *out = last ? audio : (k.arg <= 2 && cur != a[k.arg]) ? a[k.arg] : other(cur, nullptr);
            const int Lk = front ? 2 * len : len;  // the ResBlock's own length
            if ((rc = launch_resblock_tc(cur, out, packed, k.arg, batch.scaled(Lk), status, s, nullptr, precision))) return rc;
            cur = out;
            len = tailf ? Lk * stage_stride(k.arg - 20 + 1) : Lk;
        }
    }
    if (ev) MG_CUDA_TRY(cudaEventRecord(ev[n], s));
    return MG_OK;
}

// Side streams for batch slices (forked from / joined into the caller's stream with events: the call stays asynchronous
// and stream-ordered for the caller).  Per host thread, like the rest of the library's state.
constexpr int kMaxDevices = 64;
struct SliceStreams {
    static constexpr int kMax = 8;
    cudaStream_t st[kMax - 1] = {};
    cudaEvent_t fork = nullptr, join[kMax - 1] = {};
    bool ready = false;
    int init() {
        if (ready) return MG_OK;
        for (int i = 0; i < kMax - 1; ++i) {
            MG_CUDA_TRY(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
            MG_CUDA_TRY(cudaEventCreateWithFlags(&join[i], cudaEventDisableTiming));
        }
        MG_CUDA_TRY(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
        ready = true;
        return MG_OK;
    }
};

// Whole generator.  The batch items are independent and every kernel's grid is a whole number of tiles per item (or per
// 128 virtual rows), so the batch is cut into `slices` contiguous parts whose nine-kernel chains run on forked streams:
// the block scheduler fills the SMs one chain's partial last wave leaves idle (stage 0 at config 2 is 512 one-per-SM
// tiles on 132 SMs) with the other chain's tiles.  Same kernels, same per-item arithmetic: results are bit-identical
// to the single-chain order.  ev != nullptr (per-kernel timing) keeps everything on one stream.
// frames: mel frames of the whole batch (B T for a uniform one); the parts hold about equal shares of them.
int generator_tc_slices(int B, long long frames) {
    static const int forced = [] {  // MG_GEN_SLICES=n pins the slice count (experiments); default: chosen from the shape
        const char *e = getenv("MG_GEN_SLICES");
        const int v = e ? atoi(e) : 0;
        return v < 0 ? 0 : v > SliceStreams::kMax ? SliceStreams::kMax : v;
    }();
    // slicing pays while a slice still fills the machine: >= 512 mel frames per slice (stage-0 tiles ~ frames / 11)
    int slices = forced ? forced : 4;
    while (slices > 1 && ((!forced && frames < 512ll * slices) || B < slices)) --slices;
    return slices;
}

// mel_host / audio_host (both or neither; pinned): the host-buffer entry point's copies, cut the same way -- each slice's
// stream uploads its items' valid mel prefixes before its chain and downloads its audio rows (valid prefix and zero tail)
// after it, so all but the last download overlap the other chains' kernels.  precision: MG_GEN_PRECISION_*; the caller
// has checked that a bf16 forward runs the default chain.
int launch_generator_tc(const float *packed, const float *mel, float *audio, const RunTable &batch, float *ws, int *status,
                        cudaStream_t s, cudaEvent_t *ev, const float *mel_host, float *audio_host, int precision) {
    const int B = batch.items(), T = batch.stride;
    long long frames = 0;
    for (int r = 0; r < batch.n; ++r) frames += (long long)(batch.item0[r + 1] - batch.item0[r]) * batch.len[r];
    int slices = ev ? 1 : generator_tc_slices(B, frames);
    // slice k = items [cut[k], cut[k + 1]): cut where the running frame count passes k / slices of the total, leaving at
    // least one item for every later slice
    int cut[SliceStreams::kMax + 1] = {0};
    {
        long long acc = 0;
        int k = 0;
        for (int r = 0; r < batch.n; ++r)
            for (int i = batch.item0[r]; i < batch.item0[r + 1]; ++i) {
                acc += batch.len[r];
                if (k < slices - 1 && acc * slices >= frames * (k + 1) && B - (i + 1) >= slices - 1 - k) cut[++k] = i + 1;
            }
        slices = k + 1;
        cut[slices] = B;
    }
    float *base[6];
    for (int i = 0; i < 6; ++i) base[i] = ws + ws_offset(i, B, T);
    const size_t per_item[6] = {(size_t)512 * T, (size_t)256 * 8 * T, (size_t)128 * 64 * T, (size_t)64 * 128 * T, 0, (size_t)8192 * T};
    const size_t mel_item = (size_t)kMelBins * T, audio_item = (size_t)256 * T;
    // one pool per (host thread, device): streams and events belong to the device that was current when they were created
    static thread_local SliceStreams pools[kMaxDevices];
    int dev = 0;
    MG_CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kMaxDevices) return set_error(MG_ERR_INVALID_ARGUMENT, "launch_generator_tc: device ordinal %d", dev);
    SliceStreams &ss = pools[dev];
    int rc = MG_OK;
    if (slices > 1) {
        if ((rc = ss.init())) return rc;
        MG_CUDA_TRY(cudaEventRecord(ss.fork, s));
    }
    int forked = 0;  // side streams that wait on `fork` so far: all of them are joined back, also on the error path
    for (int k = 0; k < slices && rc == MG_OK; ++k) {
        const int b0 = cut[k], nb = cut[k + 1] - b0;
        const RunTable part = batch.slice(b0, cut[k + 1]);
        cudaStream_t q = k == 0 ? s : ss.st[k - 1];
        auto slice = [&]() -> int {
            if (k > 0) {
                MG_CUDA_TRY(cudaStreamWaitEvent(q, ss.fork, 0));
                forked = k;
            }
            for (int r = 0; mel_host && r < part.n; ++r) {  // one copy per run: rows of len floats, T apart
                const size_t off = (b0 + part.item0[r]) * mel_item, rows = (size_t)(part.item0[r + 1] - part.item0[r]) * kMelBins;
                float *dst = const_cast<float *>(mel) + off;
                if (part.len[r] == T)
                    MG_CUDA_TRY(cudaMemcpyAsync(dst, mel_host + off, rows * T * sizeof(float), cudaMemcpyHostToDevice, q));
                else
                    MG_CUDA_TRY(cudaMemcpy2DAsync(dst, T * sizeof(float), mel_host + off, T * sizeof(float), part.len[r] * sizeof(float),
                                                  rows, cudaMemcpyHostToDevice, q));
            }
            float *a[3] = {base[1] + b0 * per_item[1], base[2] + b0 * per_item[2], base[3] + b0 * per_item[3]};
            int r = generator_tc_chain(packed, mel + b0 * mel_item, audio + b0 * audio_item, part, base[0] + b0 * per_item[0], a,
                                       base[5] + b0 * per_item[5], status, q, ev, precision);
            if (r) return r;
            if (audio_host)
                MG_CUDA_TRY(cudaMemcpyAsync(audio_host + b0 * audio_item, audio + b0 * audio_item, nb * audio_item * sizeof(float),
                                            cudaMemcpyDeviceToHost, q));
            return MG_OK;
        };
        rc = slice();
    }
    for (int k = 1; k <= forked; ++k) {  // join (best effort after an error: the caller's stream must not outrun a forked one)
        cudaError_t e = cudaEventRecord(ss.join[k - 1], ss.st[k - 1]);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(s, ss.join[k - 1], 0);
        if (e != cudaSuccess && rc == MG_OK) rc = set_error(MG_ERR_CUDA, "launch_generator_tc: joining slice %d: %s", k, cudaGetErrorString(e));
    }
    return rc;
}

}  // namespace mg
