// Fixed-order reductions and the frame-gradient gather shared by the multi-resolution STFT loss (mg_stft_loss.cu) and
// the multi-resolution mel loss (mg_mel_loss.cu), and the denoiser's overlap-add (mg_denoise.cu).  No atomics: every
// sum has the same bits on every run.
#pragma once

namespace mg {

// fixed-order sum of v over the CTA's 8 warps (256 threads); the total is valid in thread 0
__device__ __forceinline__ float block_sum256(float v, float *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < 8; ++w) s += red[w];
    __syncthreads();
    return s;
}

// float64 sum of p[0 .. n) over the CTA's 1024 threads in a fixed order; the total is valid in thread 0
__device__ __forceinline__ double sum64_1024(const float *__restrict__ p, int n, double *red) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += 1024) acc += (double)__ldg(p + i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < 32; ++w) s += red[w];
    __syncthreads();
    return s;
}

// sum of the frame gradients db[t][N] at padded position p over the frames t covering it, [t h, t h + N), ascending t
__device__ __forceinline__ float frame_gather(const float *__restrict__ db, int p, int N, int hop, int T) {
    const int t1 = min(p / hop, T - 1), t0 = p >= N ? (p - N) / hop + 1 : 0;
    float acc = 0.f;
    for (int t = t0; t <= t1; ++t) acc += __ldg(db + (size_t)t * N + (p - t * hop));
    return acc;
}

// where frame t of a frame_gather_env sum lives: frames stored one after another (the batch denoiser), or in a ring of
// K slots, frame t in slot t mod K (the streaming denoiser's per-session frames)
struct FramesLinear {
    const float *__restrict__ db;
    int N;
    __device__ __forceinline__ const float *operator()(int t) const { return db + (size_t)t * N; }
};
struct FramesRing {
    const float *__restrict__ db;
    int N, K;
    __device__ __forceinline__ const float *operator()(int t) const { return db + (size_t)(t % K) * N; }
};

// frame_gather's sum and, in the same loop and order, the window-square envelope sum win[p - t h]^2 (the overlap-add
// of an inverse STFT); false when no frame covers p.  frame(t): frame t's N floats
template <class Frames>
__device__ __forceinline__ bool frame_gather_env(Frames frame, const float *__restrict__ win, int p, int N, int hop, int T, float &acc,
                                                 float &env) {
    const int t1 = min(p / hop, T - 1), t0 = p >= N ? (p - N) / hop + 1 : 0;
    acc = 0.f;
    env = 0.f;
    for (int t = t0; t <= t1; ++t) {
        const int n = p - t * hop;
        const float w = __ldg(win + n);
        acc += __ldg(frame(t) + n);
        env = fmaf(w, w, env);
    }
    return t0 <= t1;
}
__device__ __forceinline__ bool frame_gather_env(const float *__restrict__ db, const float *__restrict__ win, int p, int N, int hop,
                                                 int T, float &acc, float &env) {
    return frame_gather_env(FramesLinear{db, N}, win, p, N, hop, T, acc, env);
}

}  // namespace mg
