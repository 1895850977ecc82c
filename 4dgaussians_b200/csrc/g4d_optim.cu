// g4d_optim.cu -- the optimizer step of the data-parallel training harness (SURVEY.md 8f N1): ONE launch of Adam over
// the flat parameter / gradient / moment buffers (per-Gaussian SoA 59 x N + HexPlane planes + MLP, ~20 M floats at C3),
// with a per-segment learning rate (the reference's 8 param groups, scene/gaussian_model.py:165-183) and the 1 / world_size
// of the gradient all-reduce folded in.  Same update as torch.optim.Adam(eps=1e-15) without weight decay / amsgrad:
//     m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// Reference stage replaced: gaussians.optimizer.step() (train.py:290-292) -- 8 groups x multi-tensor launches.
// HBM-bound by construction: reads p, g, m, v and writes p, m, v = 28 B per parameter.
#include "g4d_internal.h"

namespace g4d {

namespace {
struct AdamSegs { int64_t begin[G4D_ADAM_MAX_SEGMENTS]; int64_t end[G4D_ADAM_MAX_SEGMENTS]; float lr[G4D_ADAM_MAX_SEGMENTS]; int n; };

// kDevice: the learning rates, bias corrections and grad scale come from *ds (device memory, read at run time) instead of
// segs.lr and the three scalar arguments
template <bool kDevice>
__global__ void __launch_bounds__(256) adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                        float* __restrict__ v, int64_t n4, AdamSegs segs, float b1, float b2, float eps,
                                                        float inv_bc1, float inv_sqrt_bc2, float grad_scale,
                                                        const G4DAdamScalars* __restrict__ ds) {
    if (kDevice) { inv_bc1 = ds->inv_bc1; inv_sqrt_bc2 = ds->inv_sqrt_bc2; grad_scale = ds->grad_scale; }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e0 = i * 4;
        int s = 0;
        while (s + 1 < segs.n && e0 >= segs.end[s]) ++s;
        float4 P = reinterpret_cast<float4*>(p)[i];
        const float4 G = reinterpret_cast<const float4*>(g)[i];
        float4 M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i];
        float* pp = &P.x; const float* gp = &G.x; float* mp = &M.x; float* vp = &V.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            int sk = s;
            while (sk + 1 < segs.n && e0 + k >= segs.end[sk]) ++sk;       // a float4 may straddle a segment boundary
            const bool live = e0 + k >= segs.begin[sk] && e0 + k < segs.end[sk];
            const float gr = gp[k] * grad_scale;
            const float mn = mp[k] + (gr - mp[k]) * (1.f - b1);           // lerp_, as torch
            const float vn = vp[k] * b2 + (1.f - b2) * gr * gr;
            const float denom = sqrtf(vn) * inv_sqrt_bc2 + eps;
            const float lr = kDevice ? ds->lr[sk] : segs.lr[sk];
            if (live) { mp[k] = mn; vp[k] = vn; pp[k] -= lr * inv_bc1 * (mn / denom); }
        }
        reinterpret_cast<float4*>(p)[i] = P;
        reinterpret_cast<float4*>(m)[i] = M;
        reinterpret_cast<float4*>(v)[i] = V;
    }
}
template <bool kDevice>
cudaError_t launch_adam(float* p, const float* g, float* m, float* v, int64_t numel, const G4DAdamSegment* segs, int nseg, float b1,
                        float b2, float eps, const G4DAdamScalars& hs, const G4DAdamScalars* ds, int sm_count, cudaStream_t st) {
    if (numel <= 0 || nseg <= 0) return cudaSuccess;
    if (nseg > G4D_ADAM_MAX_SEGMENTS || (numel & 3)) return cudaErrorInvalidValue;
    AdamSegs s{};
    s.n = nseg;
    for (int i = 0; i < nseg; ++i) { s.begin[i] = segs[i].begin; s.end[i] = segs[i].end; s.lr[i] = hs.lr[i]; }
    const int64_t n4 = numel / 4;
    int64_t blocks = (n4 + 255) / 256;
    if (blocks > (int64_t)sm_count * 16) blocks = (int64_t)sm_count * 16;
    return launch_k(adam_flat_kernel<kDevice>, (unsigned)blocks, 256, 0, st, kOrdinary, p, g, m, v, n4, s, b1, b2, eps, hs.inv_bc1,
                    hs.inv_sqrt_bc2, hs.grad_scale, ds);
}
}  // namespace

void adam_scalars(const G4DAdamSegment* segs, int nseg, float b1, float b2, int64_t step, float grad_scale, G4DAdamScalars* out) {
    *out = G4DAdamScalars{};
    for (int i = 0; i < nseg && i < G4D_ADAM_MAX_SEGMENTS; ++i) out->lr[i] = segs[i].lr;
    const double bc1 = 1.0 - pow((double)b1, (double)step), bc2 = 1.0 - pow((double)b2, (double)step);
    out->inv_bc1 = (float)(1.0 / bc1);
    out->inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    out->grad_scale = grad_scale;
}

cudaError_t launch_adam_flat(float* p, const float* g, float* m, float* v, int64_t numel, const G4DAdamSegment* segs, int nseg,
                             float b1, float b2, float eps, int64_t step, float grad_scale, int sm_count, cudaStream_t st) {
    G4DAdamScalars hs;
    adam_scalars(segs, nseg, b1, b2, step, grad_scale, &hs);
    return launch_adam<false>(p, g, m, v, numel, segs, nseg, b1, b2, eps, hs, nullptr, sm_count, st);
}

cudaError_t launch_adam_flat_device(float* p, const float* g, float* m, float* v, int64_t numel, const G4DAdamSegment* segs, int nseg,
                                    float b1, float b2, float eps, const G4DAdamScalars* d_scalars, int sm_count, cudaStream_t st) {
    return launch_adam<true>(p, g, m, v, numel, segs, nseg, b1, b2, eps, G4DAdamScalars{}, d_scalars, sm_count, st);
}

}  // namespace g4d
