// GPU mel-spectrogram front end (SURVEY 8f row 4): waveform -> |STFT| (n_fft 1024, hop 256, periodic Hann 1024, center=False on a
// signal padded by (n_fft - hop)/2 zeros) -> mel filter bank -> log(clip(., 1e-5)).
//
// Reference: mel_spectrogram, /root/reference/meldataset.py:44-55 (np.pad :48-49, librosa.feature.melspectrogram :50-52,
// spectral_normalize :54 -> dynamic_range_compression :19-25), with the parameters of /root/reference/config.json:14-22
// (n_fft 1024, hop 256, win 1024, 80 mels, 22050 Hz, fmin 55, fmax 9000).  Today it runs in librosa on the host, inside the
// DataLoader workers and once more per validation utterance (train.py:164).  librosa's published algorithm is restated
// here and in oracle/mel_oracle.py (its header says which API version the reference's call site implies, and that this row's
// parity is UNPINNED by any reference fixture).
//
// One CTA = 2 frames of one batch item, 128 threads each (CTA c: item c / ceil(T/2), frames 2 (c mod ceil(T/2)) + {0, 1}):
//   z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1]  ->  512-point complex Stockham FFT in shared memory (fp32, table twiddles)
//   ->  split into the 513 bins of the real 1024-point transform, magnitudes  ->  80 short dot products with the
//   triangular mel weights (stored sparse: each filter is a contiguous run of bins)  ->  log(max(., 1e-5)).
// A frame reads 1024 samples and writes 80 values: the kernel is bound by neither HBM nor the tensor cores (an 8192-sample
// segment is 32 frames, 1.1 MFLOP); what matters is that it no longer costs a host round trip.
#include <math.h>

#include "mg_common.cuh"
#include "mg_mel_bank.cuh"

namespace mg {

constexpr int kMelNfft = 1024, kMelHop = 256, kMelBinsFft = kMelNfft / 2 + 1, kMelMaxMels = 128;
constexpr int kMelPad = (kMelNfft - kMelHop) / 2;  // meldataset.py:48

// table buffer (host-built, caller uploads): everything a CTA needs, 15 KB
struct MelTables {
    float win[kMelNfft];       // periodic Hann, scipy.signal.get_window('hann', 1024, fftbins=True)
    float2 tw[kMelNfft / 2];   // e^{-2 pi i k / 1024}, k < 512
    int n_mels;
    int kstart[kMelMaxMels], kcount[kMelMaxMels], woff[kMelMaxMels];  // filter m = weights[woff[m] .. + kcount[m]) on bins kstart[m] ..
    float weights[2 * kMelBinsFft];  // a bin lies under at most two triangles
};

static double hz_to_mel(double f) {  // librosa.core.convert.hz_to_mel, htk=False (Slaney)
    const double f_sp = 200.0 / 3, min_log_hz = 1000.0, logstep = log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_hz / f_sp + log(f / min_log_hz) / logstep : f / f_sp;
}
static double mel_to_hz(double m) {
    const double f_sp = 200.0 / 3, min_log_hz = 1000.0, logstep = log(6.4) / 27.0, min_log_mel = min_log_hz / f_sp;
    return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}

// librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=False, norm): norm 0 = None, 1 = Slaney area normalisation (what
// `norm=1` means in the librosa 0.6/0.7 API the reference was written against), 2 = L1 (what the integer 1 means since 0.8)
int mel_filters_build(const char *fn, int n_fft, int sr, int n_mels, float fmin, float fmax, int norm, int *kstart, int *kcount,
                      int *woff, float *weights) {
    const int bins = n_fft / 2 + 1;
    double edge[kMelLossMaxMels + 2];
    const double m0 = hz_to_mel(fmin), m1 = hz_to_mel(fmax);
    for (int i = 0; i < n_mels + 2; ++i) edge[i] = mel_to_hz(m0 + (m1 - m0) * i / (n_mels + 1));
    int off = 0;
    for (int m = 0; m < n_mels; ++m) {
        const double lo = edge[m], mid = edge[m + 1], hi = edge[m + 2];
        const double scale = norm == 1 ? 2.0 / (hi - lo) : 1.0;
        int ks = -1, kc = 0;
        double l1 = 0;
        for (int k = 0; k < bins; ++k) {
            const double f = (double)k * (sr / 2.0) / (n_fft / 2);
            const double up = (f - lo) / (mid - lo), dn = (hi - f) / (hi - mid);
            const double w = up < dn ? (up > 0 ? up : 0.0) : (dn > 0 ? dn : 0.0);
            if (w > 0) {
                if (ks < 0) ks = k;
                if (off + (k - ks) >= 2 * bins) return set_error(MG_ERR_INVALID_ARGUMENT, "%s: filter bank too dense", fn);
                weights[off + (k - ks)] = (float)(w * scale);
                kc = k - ks + 1;
                l1 += w;
            }
        }
        if (norm == 2 && l1 > 0)
            for (int i = 0; i < kc; ++i) weights[off + i] = (float)(weights[off + i] / l1);
        kstart[m] = ks < 0 ? 0 : ks;
        kcount[m] = kc;
        woff[m] = off;
        off += kc;
    }
    return MG_OK;
}

int mel_tables_build(int sr, int n_mels, float fmin, float fmax, int norm, MelTables *t) {
    if (sr < 1 || n_mels < 1 || n_mels > kMelMaxMels || !(fmin >= 0.f) || !(fmax > fmin) || fmax > sr / 2.0f + 1e-3f || norm < 0 || norm > 2)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_tables_build: sr=%d n_mels=%d fmin=%g fmax=%g norm=%d", sr, n_mels, fmin, fmax, norm);
    const double pi = 3.14159265358979323846;
    for (int n = 0; n < kMelNfft; ++n) t->win[n] = (float)(0.5 - 0.5 * cos(2 * pi * n / kMelNfft));
    for (int k = 0; k < kMelNfft / 2; ++k) t->tw[k] = make_float2((float)cos(2 * pi * k / kMelNfft), (float)-sin(2 * pi * k / kMelNfft));
    t->n_mels = n_mels;
    return mel_filters_build("mg_mel_tables_build", kMelNfft, sr, n_mels, fmin, fmax, norm, t->kstart, t->kcount, t->woff, t->weights);
}

__device__ __forceinline__ MelBank mel_bank(const MelTables *st) { return MelBank{st->kstart, st->kcount, st->woff, st->weights}; }

__global__ void __launch_bounds__(256) mel_kernel(const MelTables *__restrict__ tab, const float *__restrict__ audio,
                                                  float *__restrict__ mel, int L, int T) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MelTables *st = reinterpret_cast<MelTables *>(smem_raw);
    float2 *buf = reinterpret_cast<float2 *>(smem_raw + ((sizeof(MelTables) + 15) / 16) * 16);  // [2 frames][2 buffers][512]
    float *mag = reinterpret_cast<float *>(buf + 2 * 2 * 512);                                     // [2 frames][513 (+3)]
    const int tid = threadIdx.x, fr = tid >> 7, lt = tid & 127;
    const int pairs = (T + 1) >> 1;  // grid.x = items x frame pairs: a batch is not limited by grid.y's 65535
    const int b = (int)blockIdx.x / pairs, t = 2 * ((int)blockIdx.x - b * pairs) + fr;
    for (int i = tid; i < (int)(sizeof(MelTables) / 4); i += 256) reinterpret_cast<uint32_t *>(st)[i] = reinterpret_cast<const uint32_t *>(tab)[i];
    __syncthreads();
    const bool live = t < T;
    float2 *A = buf + fr * 1024;
    float *mg = mag + fr * 516;
    // the forward and the backward both run mel_frame_bins, so the backward differentiates the very magnitudes the forward summed
    mel_frame_bins<kMelNfft>(st->win, st->tw, audio + (size_t)b * L, L, t * kMelHop - kMelPad, live, lt, A, A + 512, mg, nullptr);
    if (live && lt < st->n_mels) mel[((size_t)b * st->n_mels + lt) * T + t] = mel_log(mel_band_sum(mel_bank(st), mg, lt));
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward: grad_audio = d loss / d audio given grad_mel = d loss / d mel, torch autograd's conventions (clamp(min=)
// passes where s >= 1e-5, |0| has gradient 0, the rfft adjoint over bins 0..512 as the forward has them, padding dropped).
//
// mel_backward_frame_kernel, same CTA geometry as mel_kernel, per frame:
//   recompute X and s with the forward's arithmetic  ->  gs_m = g_m / s_m (0 below the clip)  ->  dmag = M^T gs and
//   G[k] = dmag_k X_k / |X_k| (mel_band_adjoint, mg_mel_bank.cuh)  ->  adjoint of the even/odd split into dZ[0..511]  ->
//   512-point inverse Stockham FFT (conjugate twiddles, unnormalised)  ->  times the window  ->  dframe[b][t][1024].
// mel_backward_ola_kernel: grad_audio[b][i] = sum over the <= 4 frames covering padded sample i + 384, ascending t.
//
// The split's adjoint (split_adjoint_pass) and the inverse pass (stockham<512, 128, true>) are in mg_fft.cuh.
// ---------------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) mel_backward_frame_kernel(const MelTables *__restrict__ tab, const float *__restrict__ audio,
                                                                 const float *__restrict__ grad_mel, float *__restrict__ dframe,
                                                                 int L, int T) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MelTables *st = reinterpret_cast<MelTables *>(smem_raw);
    float2 *buf = reinterpret_cast<float2 *>(smem_raw + ((sizeof(MelTables) + 15) / 16) * 16);  // [2 frames][2 buffers][512]
    float2 *Xall = buf + 2 * 2 * 512;                                                             // [2 frames][513 (+3)]
    float *mag = reinterpret_cast<float *>(Xall + 2 * 516);                                       // [2 frames][513 (+3)]
    float *dmag = mag + 2 * 516;                                                                  // [2 frames][513 (+3)]
    const int tid = threadIdx.x, fr = tid >> 7, lt = tid & 127;
    const int pairs = (T + 1) >> 1;
    const int b = (int)blockIdx.x / pairs, t = 2 * ((int)blockIdx.x - b * pairs) + fr;
    for (int i = tid; i < (int)(sizeof(MelTables) / 4); i += 256) reinterpret_cast<uint32_t *>(st)[i] = reinterpret_cast<const uint32_t *>(tab)[i];
    __syncthreads();
    const bool live = t < T;
    float2 *A = buf + fr * 1024, *Xk = Xall + fr * 516;
    float *mg = mag + fr * 516, *dm = dmag + fr * 516;
    mel_frame_bins<kMelNfft>(st->win, st->tw, audio + (size_t)b * L, L, t * kMelHop - kMelPad, live, lt, A, A + 512, mg, Xk);
    const int n_mels = st->n_mels;
    const MelBank bk = mel_bank(st);
    float gs = 0.f;
    if (live && lt < n_mels) {
        const float s = mel_band_sum(bk, mg, lt);
        gs = s >= 1e-5f ? __ldg(grad_mel + ((size_t)b * n_mels + lt) * T + t) / s : 0.f;  // log' = 1 / s; clamp(min=)' = [s >= min]
    }
    for (int k = lt; k <= 512; k += 128) dm[k] = 0.f;
    __syncthreads();
    mel_band_adjoint<kMelNfft, 128>(bk, n_mels, lt, [&](int) { return gs; }, dm, mg, Xk);  // band lt is this thread's
    __syncthreads();
    split_adjoint_pass<512, 128>(Xk, A, st->tw, lt);
    __syncthreads();
    // inverse transform: the forward's Stockham passes with conjugate twiddles, e^{+2 pi i k / (2 ns)}, no 1/512
    float2 *in = stockham<512, 128, true>(A, A + 512, st->tw, lt);
    if (!live) return;
    // dz[n] = d/dRe z[n] + i d/dIm z[n], z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1]
    float2 *df = reinterpret_cast<float2 *>(dframe + ((size_t)b * T + t) * kMelNfft);
    for (int n = lt; n < 512; n += 128) df[n] = make_float2(st->win[2 * n] * in[n].x, st->win[2 * n + 1] * in[n].y);
}

// one CTA = 1024 consecutive samples of one item; each sample gathers the frames that read it, ascending t, so the sum is
// the same bits in every run and for every batch layout.  Every sample in [0, L) is written (0 where no frame reaches).
__global__ void __launch_bounds__(256) mel_backward_ola_kernel(const float *__restrict__ dframe, float *__restrict__ grad_audio,
                                                               int L, int T) {
    const int chunks = (L + 1023) >> 10;
    const int b = (int)blockIdx.x / chunks, c = (int)blockIdx.x - b * chunks;
    const float *db = dframe + (size_t)b * T * kMelNfft;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int i = (c << 10) + 256 * r + (int)threadIdx.x;
        if (i >= L) break;
        const int p = i + kMelPad;                     // index in the padded signal; frame t covers [256 t, 256 t + 1024)
        const int t1 = min(p / kMelHop, T - 1), t0 = p >= kMelNfft ? (p - kMelNfft) / kMelHop + 1 : 0;
        float acc = 0.f;
        for (int t = t0; t <= t1; ++t) acc += __ldg(db + (size_t)t * kMelNfft + (p - t * kMelHop));
        grad_audio[(size_t)b * L + i] = acc;
    }
}

int mel_frames(int L) { return L + 2 * kMelPad < kMelNfft ? 0 : 1 + (L + 2 * kMelPad - kMelNfft) / kMelHop; }

int launch_mel(const void *tables, const float *audio, float *mel, int B, int L, cudaStream_t s) {
    const int T = mel_frames(L);
    if (T < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram: %d samples are fewer than one frame", L);
    const long long ctas = (long long)B * ((T + 1) / 2);
    if (ctas > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram: B=%d x %d frame pairs exceed 2^31 - 1 CTAs", B, (T + 1) / 2);
    constexpr int smem = ((sizeof(MelTables) + 15) / 16) * 16 + 2 * 2 * 512 * 8 + 2 * 516 * 4;
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    mel_kernel<<<(unsigned)ctas, 256, smem, s>>>(reinterpret_cast<const MelTables *>(tables), audio, mel, L, T);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

size_t mel_backward_workspace_bytes(int B, int L) {
    const int T = L < 1 ? 0 : mel_frames(L);
    if (B < 1 || T < 1 || (long long)B * ((T + 1) / 2) > 0x7fffffffll) return 0;
    return (size_t)B * T * kMelNfft * sizeof(float);
}

int launch_mel_backward(const void *tables, const float *audio, const float *grad_mel, float *grad_audio, int B, int L,
                        void *workspace, size_t workspace_bytes, cudaStream_t s) {
    const int T = mel_frames(L);
    if (T < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram_backward: %d samples are fewer than one frame", L);
    const long long ctas = (long long)B * ((T + 1) / 2);
    if (ctas > 0x7fffffffll)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_spectrogram_backward: B=%d x %d frame pairs exceed 2^31 - 1 CTAs", B, (T + 1) / 2);
    const size_t need = mel_backward_workspace_bytes(B, L);
    if (workspace_bytes < need)
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "mg_mel_spectrogram_backward: workspace of %zu bytes, %zu needed", workspace_bytes, need);
    constexpr int smem = ((sizeof(MelTables) + 15) / 16) * 16 + 2 * 2 * 512 * 8 + 2 * 516 * 8 + 2 * 2 * 516 * 4;
    static bool configured = false;
    if (!configured) {
        MG_CUDA_TRY(cudaFuncSetAttribute(mel_backward_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    float *dframe = reinterpret_cast<float *>(workspace);
    mel_backward_frame_kernel<<<(unsigned)ctas, 256, smem, s>>>(reinterpret_cast<const MelTables *>(tables), audio, grad_mel, dframe, L, T);
    MG_CUDA_TRY(cudaGetLastError());
    // B * ceil(L / 1024) <= B * ceil(T / 2) CTAs: L < 256 (T + 1) gives L / 1024 < (T + 1) / 4
    mel_backward_ola_kernel<<<(unsigned)((long long)B * ((L + 1023) / 1024)), 256, 0, s>>>(dframe, grad_audio, L, T);
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

size_t mel_tables_bytes() { return sizeof(MelTables); }

}  // namespace mg
