// Multi-tensor Adam: one launch updates every parameter tensor of an optimizer group (SURVEY 8f rank 1; the reference
// calls torch.optim.Adam on 90 (G) / 63 (D) separate tensors, train.py:51-52,118,129 -- with torch's foreach path that is
// ~10 sequences of small launches per step).  Same arithmetic as torch.optim.Adam (no amsgrad):
//   g += wd p;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
#include "mg_common.cuh"

namespace mg {

constexpr int kAdamChunk = 4096;  // elements per CTA

// table (device memory, built by the caller): per tensor {p, g, m, v} pointers and element count; first[i] = first CTA
__global__ void __launch_bounds__(256) adam_kernel(float *const *__restrict__ p, const float *const *__restrict__ g,
                                                   float *const *__restrict__ m, float *const *__restrict__ v,
                                                   const long long *__restrict__ n, const int *__restrict__ first, int count,
                                                   float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt) {
    int lo = 0, hi = count - 1;  // last tensor whose first CTA <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const long long base = (long long)(blockIdx.x - first[lo]) * kAdamChunk;
    const long long end = base + kAdamChunk < n[lo] ? base + kAdamChunk : n[lo];
    float *pp = p[lo], *mm = m[lo], *vv = v[lo];
    const float *gg = g[lo];
    const float step = lr / bc1;
    for (long long j = base + threadIdx.x; j < end; j += 256) {
        float gr = gg[j];
        const float pv = pp[j];
        if (wd != 0.f) gr = fmaf(wd, pv, gr);
        const float mn = b1 * mm[j] + (1.f - b1) * gr;
        const float vn = b2 * vv[j] + (1.f - b2) * gr * gr;
        mm[j] = mn;
        vv[j] = vn;
        pp[j] = pv - step * mn / (sqrtf(vn) / bc2_sqrt + eps);
    }
}

int launch_adam(float *const *p, const float *const *g, float *const *m, float *const *v, const long long *n, const int *first,
                int count, int total_ctas, float lr, float b1, float b2, float eps, float wd, long long step, cudaStream_t s) {
    if (!p || !g || !m || !v || !n || !first || count < 1 || total_ctas < 1 || step < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_adam_step: bad argument");
    const double bc1 = 1.0 - pow((double)b1, (double)step), bc2 = 1.0 - pow((double)b2, (double)step);
    adam_kernel<<<total_ctas, 256, 0, s>>>(p, g, m, v, n, first, count, lr, b1, b2, eps, wd, (float)bc1, (float)sqrt(bc2));
    MG_CUDA_TRY(cudaGetLastError());
    return MG_OK;
}

}  // namespace mg
