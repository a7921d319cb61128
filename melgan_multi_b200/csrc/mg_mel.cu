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

// librosa.filters.mel(sr, 1024, n_mels, fmin, fmax, htk=False, norm): norm 0 = None, 1 = Slaney area normalisation (what
// `norm=1` means in the librosa 0.6/0.7 API the reference was written against), 2 = L1 (what the integer 1 means since 0.8)
int mel_tables_build(int sr, int n_mels, float fmin, float fmax, int norm, MelTables *t) {
    if (sr < 1 || n_mels < 1 || n_mels > kMelMaxMels || !(fmin >= 0.f) || !(fmax > fmin) || fmax > sr / 2.0f + 1e-3f || norm < 0 || norm > 2)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_tables_build: sr=%d n_mels=%d fmin=%g fmax=%g norm=%d", sr, n_mels, fmin, fmax, norm);
    const double pi = 3.14159265358979323846;
    for (int n = 0; n < kMelNfft; ++n) t->win[n] = (float)(0.5 - 0.5 * cos(2 * pi * n / kMelNfft));
    for (int k = 0; k < kMelNfft / 2; ++k) t->tw[k] = make_float2((float)cos(2 * pi * k / kMelNfft), (float)-sin(2 * pi * k / kMelNfft));
    t->n_mels = n_mels;
    double edge[kMelMaxMels + 2];
    const double m0 = hz_to_mel(fmin), m1 = hz_to_mel(fmax);
    for (int i = 0; i < n_mels + 2; ++i) edge[i] = mel_to_hz(m0 + (m1 - m0) * i / (n_mels + 1));
    int off = 0;
    for (int m = 0; m < n_mels; ++m) {
        const double lo = edge[m], mid = edge[m + 1], hi = edge[m + 2];
        const double scale = norm == 1 ? 2.0 / (hi - lo) : 1.0;
        int ks = -1, kc = 0;
        double l1 = 0;
        for (int k = 0; k < kMelBinsFft; ++k) {
            const double f = (double)k * (sr / 2.0) / (kMelNfft / 2);
            const double up = (f - lo) / (mid - lo), dn = (hi - f) / (hi - mid);
            const double w = up < dn ? (up > 0 ? up : 0.0) : (dn > 0 ? dn : 0.0);
            if (w > 0) {
                if (ks < 0) ks = k;
                if (off + (k - ks) >= 2 * kMelBinsFft) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_mel_tables_build: filter bank too dense");
                t->weights[off + (k - ks)] = (float)(w * scale);
                kc = k - ks + 1;
                l1 += w;
            }
        }
        if (norm == 2 && l1 > 0)
            for (int i = 0; i < kc; ++i) t->weights[off + i] = (float)(t->weights[off + i] / l1);
        t->kstart[m] = ks < 0 ? 0 : ks;
        t->kcount[m] = kc;
        t->woff[m] = off;
        off += kc;
    }
    return MG_OK;
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

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
    float2 *A = buf + fr * 1024, *Bf = A + 512;
    // windowed frame, even samples -> real part, odd -> imaginary; sample index in the UNPADDED signal: t*hop - 384 + n
    const float *xb = audio + (size_t)b * L;
    for (int n = lt; n < 512; n += 128) {
        const int i0 = t * kMelHop - kMelPad + 2 * n;
        const float x0 = (live && i0 >= 0 && i0 < L) ? __ldg(xb + i0) : 0.f;
        const float x1 = (live && i0 + 1 >= 0 && i0 + 1 < L) ? __ldg(xb + i0 + 1) : 0.f;
        A[n] = make_float2(st->win[2 * n] * x0, st->win[2 * n + 1] * x1);
    }
    __syncthreads();
    // 512-point Stockham autosort FFT, radix 2: 9 passes, 256 butterflies each (2 per thread)
    float2 *in = A, *out = Bf;
#pragma unroll 1
    for (int ns = 1; ns < 512; ns <<= 1) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int j = lt + 128 * r;
            const int k = j & (ns - 1);
            const float2 v0 = in[j], v1 = cmul(in[j + 256], st->tw[k * (512 / ns)]);  // e^{-2 pi i k / (2 ns)}
            const int j0 = ((j - k) << 1) + k;
            out[j0] = make_float2(v0.x + v1.x, v0.y + v1.y);
            out[j0 + ns] = make_float2(v0.x - v1.x, v0.y - v1.y);
        }
        __syncthreads();
        float2 *tmp = in; in = out; out = tmp;
    }
    // Z = in: bins of the real transform, X[k] = E[k] + e^{-2 pi i k / 1024} O[k], E = (Z[k] + conj Z[512-k]) / 2, O = (Z[k] - conj Z[512-k]) / 2i
    float *mg = mag + fr * 516;
    for (int k = lt; k <= 512; k += 128) {
        const float2 zk = in[k & 511], zc = in[(512 - k) & 511];
        const float2 E = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y - zc.y));
        const float2 O = make_float2(0.5f * (zk.y + zc.y), -0.5f * (zk.x - zc.x));
        const float2 w = k < 512 ? st->tw[k] : make_float2(-1.f, 0.f);
        const float2 X = make_float2(E.x + w.x * O.x - w.y * O.y, E.y + w.x * O.y + w.y * O.x);
        mg[k] = sqrtf(X.x * X.x + X.y * X.y);  // power = 1 (meldataset.py:50)
    }
    __syncthreads();
    if (live && lt < st->n_mels) {
        const int ks = st->kstart[lt], kc = st->kcount[lt];
        const float *w = st->weights + st->woff[lt];
        float s = 0.f;
        for (int i = 0; i < kc; ++i) s = fmaf(w[i], mg[ks + i], s);
        mel[((size_t)b * st->n_mels + lt) * T + t] = logf(fmaxf(s, 1e-5f));  // meldataset.py:19-25: log(clip(x, 1e-5) * 1)
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

size_t mel_tables_bytes() { return sizeof(MelTables); }

}  // namespace mg
