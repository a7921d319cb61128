// The whole backward of ONE Discriminator (autograd of models.py:87-103 of the reference) behind a single call: the host walks
// the seven layers from the logits down and enqueues every kernel itself -- LeakyReLU', grouped-conv dx / dw / db, conv_post1
// dgrad + wgrad (wgmma), conv_pre / conv_post2 -- so a training step pays one host call per discriminator instead of ~25
// Python-level launches (host work that would otherwise bound the step, not the GPU).
// Gradients of the FOLDED weights come back per layer; mg_msd_wn_backward turns them into (d weight_v, d weight_g).
#include "mg_common.cuh"

#define MG_TRY(expr) do { const int rc_ = (expr); if (rc_ != MG_OK) return rc_; } while (0)

namespace mg {

namespace {
struct ScaleShapes {
    int L[kDiscLayers + 1];  // L[0] = input length, L[l + 1] = output length of layer l
    size_t act;              // floats of the largest activation [Bt][C][L]
};
ScaleShapes scale_shapes(int Bt, int L0) {
    ScaleShapes s;
    s.L[0] = L0;
    s.act = (size_t)Bt * L0;
    for (int l = 0; l < kDiscLayers; ++l) {
        const DLayer d = d_layer(l);
        s.L[l + 1] = (s.L[l] + 2 * d.pad - d.k) / d.stride + 1;
        const size_t n = (size_t)Bt * d.cout * s.L[l + 1];
        if (n > s.act) s.act = n;
    }
    return s;
}
size_t round256(size_t b) { return (b + 255) / 256 * 256; }
size_t kernel_ws_bytes(int Bt, const ScaleShapes &s) {
    size_t w = edge_bwd_workspace_bytes(0, Bt, s.L[0]);
    for (int l = 1; l <= 4; ++l) {
        const size_t b = grouped_bwd_workspace_bytes(l, Bt, s.L[l + 1]);
        if (b > w) w = b;
    }
    return w;
}
}  // namespace

// three activation-sized buffers (dz and two alternating dx) + the largest per-kernel workspace
size_t disc_scale_backward_workspace_bytes(int Bt, int L0) {
    const ScaleShapes s = scale_shapes(Bt, L0);
    return 3 * round256(s.act * sizeof(float)) + round256(kernel_ws_bytes(Bt, s));
}

// blob: this discriminator's packed weights.  x0 [Bt][1][L0]; fmap[l] = output of layer l as returned by the forward
// (post-LeakyReLU for l < 6); gfmap[l] = gradient w.r.t. that returned map or NULL; gx0 [Bt][1][L0] or NULL;
// dw[l] / db[l]: outputs (torch layout of the folded weight), written for every layer the gradient reaches.
// reached[l] (host int array, may be NULL) reports which layers were written.
int launch_disc_scale_backward(const void *blob, const float *x0, const float *const *fmap, const float *const *gfmap, float *gx0,
                               float *const *dw, float *const *db, int *reached, void *workspace, size_t workspace_bytes, int Bt,
                               int L0, int *status, cudaStream_t st) {
    const ScaleShapes s = scale_shapes(Bt, L0);
    if (s.L[kDiscLayers] < 1) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_scale_backward: sequence too short (%d samples)", L0);
    if (workspace_bytes < disc_scale_backward_workspace_bytes(Bt, L0))
        return set_error(MG_ERR_WORKSPACE_TOO_SMALL, "mg_msd_scale_backward: workspace of %zu bytes needed",
                         disc_scale_backward_workspace_bytes(Bt, L0));
    const size_t abytes = round256(s.act * sizeof(float));
    uint8_t *wsb = static_cast<uint8_t *>(workspace);
    float *dzbuf = reinterpret_cast<float *>(wsb), *dxbuf[2] = {reinterpret_cast<float *>(wsb + abytes), reinterpret_cast<float *>(wsb + 2 * abytes)};
    float *kws = reinterpret_cast<float *>(wsb + 3 * abytes);
    const float *g = nullptr;  // gradient w.r.t. the output of the layer being visited, from the layer above
    int flip = 0;
    for (int l = kDiscLayers - 1; l >= 0; --l) {
        if (reached) reached[l] = 0;
        const float *go = gfmap[l];
        if (!g && !go) continue;
        const DLayer d = d_layer(l);
        const int Lin = s.L[l], Lout = s.L[l + 1];
        const long long n = (long long)Bt * d.cout * Lout;
        const float *dz;
        if (l < kDiscLayers - 1) {  // (g + go) * LeakyReLU'(layer output)
            MG_TRY(launch_lrelu_grad(g ? g : go, g ? go : nullptr, fmap[l], dzbuf, n, st));
            dz = dzbuf;
        } else {
            dz = go;  // conv_post2 has no activation and no layer above
        }
        if (!dw[l] || !db[l]) return set_error(MG_ERR_INVALID_ARGUMENT, "mg_msd_scale_backward: dw[%d] / db[%d] missing", l, l);
        const float *x = l == 0 ? x0 : fmap[l - 1];
        float *dx = l == 0 ? gx0 : dxbuf[flip];
        if (d.groups > 1) {
            MG_TRY(launch_disc_grouped_backward(blob, l, dz, x, dx, dw[l], db[l], kws, Bt, Lin, Lout, st));
        } else if (l == 5) {
            const uint8_t *b8 = static_cast<const uint8_t *>(blob);
            MG_TRY(launch_disc_post1_dgrad_tc(dz, dx, b8 + d_tcT_start(), reinterpret_cast<const float *>(b8 + d_zero_start()), Bt, Lout, status, st));
            MG_TRY(launch_disc_post1_wgrad_tc(x, dz, dw[l], db[l], Bt, Lout, status, st));
        } else {
            MG_TRY(launch_disc_edge_backward(blob, l, dz, x, dx, dw[l], db[l], kws, Bt, Lin, st));
        }
        if (reached) reached[l] = 1;
        g = dx;
        flip ^= 1;
    }
    return MG_OK;
}

}  // namespace mg
