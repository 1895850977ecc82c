// g4d_loss.cu -- the step either side of the path (SURVEY.md 8f N2): the image loss and the HexPlane regularisers, each as
// ONE kernel that produces the loss value AND the gradient the next stage consumes.
//
//   l1_loss_kernel / l1_grad_kernel   <- utils/loss_utils.py:20-21  l1_loss = |out - gt|.mean()        (train.py:201)
//   plane_regulation_kernel           <- scene/regulation.py:22-28 compute_plane_smoothness and
//                                        scene/gaussian_model.py:538-577 _plane_regulation / _time_regulation /
//                                        _l1_regulation / compute_regulation                            (train.py:207-210)
//   ssim_* kernels                    <- utils/loss_utils.py:37-66 ssim (11x11 Gaussian window, sigma 1.5, zero padding)
//
// The reference runs these as ~8 (L1), ~60 (regularisers: 12-18 planes x slices, squares, means) and ~25 (SSIM) ATen
// launches per step, each streaming the image / the 9.5-25 MB plane pyramid through HBM several times.
#include "g4d_internal.h"

namespace g4d {

namespace {

// ---- L1 -----------------------------------------------------------------------------------------------------------
// kVec: every pointer is 16-byte aligned, float4 loads + a scalar tail in block 0.  Otherwise (a view at an odd storage
// offset, e.g. batch[1] of a [B,3,H,W] batch with H*W odd) the same sum with scalar loads.
template <bool kVec>
__global__ void __launch_bounds__(256) l1_loss_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float scale,
                                                      float* __restrict__ loss) {
    float acc = 0.f;
    if (kVec) {
        const int64_t n4 = n >> 2;
        const float4* a4 = reinterpret_cast<const float4*>(a);
        const float4* b4 = reinterpret_cast<const float4*>(b);
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 x = a4[i], y = __ldg(b4 + i);
            acc += fabsf(x.x - y.x) + fabsf(x.y - y.y) + fabsf(x.z - y.z) + fabsf(x.w - y.w);
        }
        if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const int64_t i = (n4 << 2) + threadIdx.x; acc += fabsf(a[i] - b[i]); }
    } else {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
            acc += fabsf(a[i] - __ldg(b + i));
    }
    const float tot = block_sum_f(acc);
    if (threadIdx.x == 0) atomicAdd(loss, tot * scale);
}

// grad = sign(a - b) * scale * upstream[0]     (torch.abs backward: sign(0) = 0)
template <bool kVec>
__global__ void __launch_bounds__(256) l1_grad_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float scale,
                                                      const float* __restrict__ upstream, float* __restrict__ grad) {
    const float s = scale * (upstream ? __ldg(upstream) : 1.f);
    auto sg = [s](float d) { return d > 0.f ? s : (d < 0.f ? -s : 0.f); };
    if (kVec) {
        const int64_t n4 = n >> 2;
        const float4* a4 = reinterpret_cast<const float4*>(a);
        const float4* b4 = reinterpret_cast<const float4*>(b);
        float4* g4 = reinterpret_cast<float4*>(grad);
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
            const float4 x = a4[i], y = __ldg(b4 + i);
            g4[i] = make_float4(sg(x.x - y.x), sg(x.y - y.y), sg(x.z - y.z), sg(x.w - y.w));
        }
        if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const int64_t i = (n4 << 2) + threadIdx.x; grad[i] = sg(a[i] - b[i]); }
    } else {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
            grad[i] = sg(a[i] - __ldg(b + i));
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- HexPlane regularisers ----------------------------------------------------------------------------------------------
// plane k of a level, channel-last [H][W][C]; planes 0,1,3 are spatial (xy, xz, yz), planes 2,4,5 carry the time axis
// (H = time).  compute_plane_smoothness = mean over [C][H-2][W] of the squared second difference along H.
struct RegPlane { const float* p; float* g; int H, W, C; float w_smooth, w_l1; int64_t start; };
struct RegDesc { RegPlane pl[G4D_MAX_LEVELS * 6]; int count; int64_t total; };

__global__ void __launch_bounds__(256) plane_regulation_kernel(RegDesc d, float* __restrict__ loss, const float* __restrict__ upstream) {
    const float up = upstream ? __ldg(upstream) : 1.f;
    float acc = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < d.total; i += (int64_t)gridDim.x * blockDim.x) {
        int m = 0;
        while (m + 1 < d.count && i >= d.pl[m + 1].start) ++m;
        const RegPlane& P = d.pl[m];
        const int64_t e = i - P.start;
        const int64_t row = (int64_t)P.W * P.C;
        const int h = (int)(e / row);
        const float* q = P.p + e;                  // p[h] at this (w, c)
        const int H = P.H;
        const float c0 = __ldg(q);
        float g = 0.f;
        if (H >= 3) {
            const float inv = 1.f / ((float)P.C * (float)(H - 2) * (float)P.W);
            // d2[j] = p[j+2] - 2 p[j+1] + p[j], 0 <= j <= H-3
            const float pm2 = h >= 2 ? __ldg(q - 2 * row) : 0.f, pm1 = h >= 1 ? __ldg(q - row) : 0.f;
            const float pp1 = h + 1 < H ? __ldg(q + row) : 0.f, pp2 = h + 2 < H ? __ldg(q + 2 * row) : 0.f;
            const float d2_h = h <= H - 3 ? pp2 - 2.f * pp1 + c0 : 0.f;
            const float d2_hm1 = (h >= 1 && h <= H - 2) ? pp1 - 2.f * c0 + pm1 : 0.f;
            const float d2_hm2 = h >= 2 ? c0 - 2.f * pm1 + pm2 : 0.f;
            acc += P.w_smooth * inv * d2_h * d2_h;
            g += P.w_smooth * inv * 2.f * (d2_h - 2.f * d2_hm1 + d2_hm2);
        }
        if (P.w_l1 != 0.f) {
            const float inv = 1.f / ((float)P.C * (float)H * (float)P.W);
            const float r = 1.f - c0;
            acc += P.w_l1 * inv * fabsf(r);
            g += P.w_l1 * inv * (r > 0.f ? -1.f : (r < 0.f ? 1.f : 0.f));
        }
        if (P.g) P.g[e] += g * up;
    }
    const float tot = block_sum_f(acc);
    if (threadIdx.x == 0 && loss) atomicAdd(loss, tot);
}

// ---- SSIM (11 x 11 Gaussian window, sigma 1.5, zero padding; per channel) ---------------------------------------------------
constexpr int kSsimR = 5, kSsimT = 16, kSsimIn = kSsimT + 2 * kSsimR;   // 16x16 outputs from a 26x26 input patch
struct SsimWin { float w[11]; };
constexpr float kSsimC1 = 0.01f * 0.01f, kSsimC2 = 0.03f * 0.03f;

// forward: ssim map statistics per pixel -> loss accumulation (sum of the map * scale) and, for the backward, the three
// partial derivatives of the map w.r.t. (mu1, E[x^2], E[xy]) at every pixel
__global__ void __launch_bounds__(kSsimT * kSsimT) ssim_forward_kernel(SsimWin win, const float* __restrict__ x, const float* __restrict__ y,
                                                                       int H, int W, float scale, float* __restrict__ loss,
                                                                       float* __restrict__ dmu, float* __restrict__ dxx, float* __restrict__ dxy) {
    __shared__ float sx[kSsimIn][kSsimIn + 1], sy[kSsimIn][kSsimIn + 1];
    __shared__ float h1[kSsimIn][kSsimT], h2[kSsimIn][kSsimT], h3[kSsimIn][kSsimT], h4[kSsimIn][kSsimT], h5[kSsimIn][kSsimT];
    const int ch = blockIdx.z;
    const float* xc = x + (size_t)ch * H * W;
    const float* yc = y + (size_t)ch * H * W;
    const int tx = threadIdx.x % kSsimT, ty = threadIdx.x / kSsimT;
    const int ox = blockIdx.x * kSsimT, oy = blockIdx.y * kSsimT;
    for (int i = threadIdx.x; i < kSsimIn * kSsimIn; i += kSsimT * kSsimT) {
        const int r = i / kSsimIn, c = i % kSsimIn;
        const int gy = oy + r - kSsimR, gx = ox + c - kSsimR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        sx[r][c] = in ? xc[(size_t)gy * W + gx] : 0.f;
        sy[r][c] = in ? __ldg(yc + (size_t)gy * W + gx) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSsimIn * kSsimT; i += kSsimT * kSsimT) {     // horizontal pass
        const int r = i / kSsimT, c = i % kSsimT;
        float a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f, a5 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float u = sx[r][c + k], v = sy[r][c + k], w = win.w[k];
            a1 += w * u; a2 += w * v; a3 += w * u * u; a4 += w * v * v; a5 += w * u * v;
        }
        h1[r][c] = a1; h2[r][c] = a2; h3[r][c] = a3; h4[r][c] = a4; h5[r][c] = a5;
    }
    __syncthreads();
    float m1 = 0.f, m2 = 0.f, exx = 0.f, eyy = 0.f, exy = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {                                               // vertical pass
        const float w = win.w[k];
        m1 += w * h1[ty + k][tx]; m2 += w * h2[ty + k][tx]; exx += w * h3[ty + k][tx]; eyy += w * h4[ty + k][tx]; exy += w * h5[ty + k][tx];
    }
    const int gx = ox + tx, gy = oy + ty;
    float val = 0.f;
    if (gx < W && gy < H) {
        const float A1 = 2.f * m1 * m2 + kSsimC1, A2 = 2.f * (exy - m1 * m2) + kSsimC2;
        const float B1 = m1 * m1 + m2 * m2 + kSsimC1, B2 = (exx - m1 * m1) + (eyy - m2 * m2) + kSsimC2;
        const float inv = 1.f / (B1 * B2);
        val = A1 * A2 * inv;
        if (dmu) {
            const size_t o = (size_t)ch * H * W + (size_t)gy * W + gx;
            dmu[o] = (2.f * m2 * (A2 - A1)) * inv - val * (2.f * m1 / B1) + val * (2.f * m1 / B2);
            dxx[o] = -val / B2;
            dxy[o] = 2.f * A1 * inv;
        }
    }
    const float tot = block_sum_f(val);
    if (threadIdx.x == 0 && loss) atomicAdd(loss, tot * scale);
}

// backward: grad_x(p) = s * sum_q w(q - p) [dmu(q) + 2 x(p) dxx(q) + y(p) dxy(q)],  s = scale * upstream
__global__ void __launch_bounds__(kSsimT * kSsimT) ssim_backward_kernel(SsimWin win, const float* __restrict__ x, const float* __restrict__ y,
                                                                        int H, int W, float scale, const float* __restrict__ upstream,
                                                                        const float* __restrict__ dmu, const float* __restrict__ dxx,
                                                                        const float* __restrict__ dxy, float* __restrict__ grad) {
    __shared__ float s1[kSsimIn][kSsimIn + 1], s2[kSsimIn][kSsimIn + 1], s3[kSsimIn][kSsimIn + 1];
    __shared__ float h1[kSsimIn][kSsimT], h2[kSsimIn][kSsimT], h3[kSsimIn][kSsimT];
    const int ch = blockIdx.z;
    const size_t base = (size_t)ch * H * W;
    const int tx = threadIdx.x % kSsimT, ty = threadIdx.x / kSsimT;
    const int ox = blockIdx.x * kSsimT, oy = blockIdx.y * kSsimT;
    for (int i = threadIdx.x; i < kSsimIn * kSsimIn; i += kSsimT * kSsimT) {
        const int r = i / kSsimIn, c = i % kSsimIn;
        const int gy = oy + r - kSsimR, gx = ox + c - kSsimR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        const size_t o = base + (size_t)gy * W + gx;
        s1[r][c] = in ? dmu[o] : 0.f; s2[r][c] = in ? dxx[o] : 0.f; s3[r][c] = in ? dxy[o] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSsimIn * kSsimT; i += kSsimT * kSsimT) {
        const int r = i / kSsimT, c = i % kSsimT;
        float a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) { const float w = win.w[k]; a1 += w * s1[r][c + k]; a2 += w * s2[r][c + k]; a3 += w * s3[r][c + k]; }
        h1[r][c] = a1; h2[r][c] = a2; h3[r][c] = a3;
    }
    __syncthreads();
    float c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) { const float w = win.w[k]; c1 += w * h1[ty + k][tx]; c2 += w * h2[ty + k][tx]; c3 += w * h3[ty + k][tx]; }
    const int gx = ox + tx, gy = oy + ty;
    if (gx < W && gy < H) {
        const size_t o = base + (size_t)gy * W + gx;
        const float s = scale * (upstream ? __ldg(upstream) : 1.f);
        grad[o] = s * (c1 + 2.f * x[o] * c2 + __ldg(y + o) * c3);
    }
}

SsimWin make_ssim_window() {
    SsimWin w{};
    double g[11], sum = 0.0;
    for (int i = 0; i < 11; ++i) { g[i] = exp(-(double)((i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5)); sum += g[i]; }
    // loss_utils.py:26-28 builds the window in fp32: gauss / gauss.sum()
    float gf[11], sf = 0.f;
    for (int i = 0; i < 11; ++i) { gf[i] = (float)g[i]; sf += gf[i]; }
    (void)sum;
    for (int i = 0; i < 11; ++i) w.w[i] = gf[i] / sf;
    return w;
}

int grid_for(int64_t work, int sm_count) {
    int64_t b = (work + 255) / 256;
    const int64_t cap = (int64_t)sm_count * 8;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

cudaError_t launch_l1_loss(const float* a, const float* b, int64_t n, float scale, float* loss, int sm_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    if (aligned16(a) && aligned16(b))
        l1_loss_kernel<true><<<grid_for(n / 4, sm_count), 256, 0, st>>>(a, b, n, scale, loss);
    else
        l1_loss_kernel<false><<<grid_for(n, sm_count), 256, 0, st>>>(a, b, n, scale, loss);
    return cudaGetLastError();
}
cudaError_t launch_l1_grad(const float* a, const float* b, int64_t n, float scale, const float* upstream, float* grad, int sm_count,
                           cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    if (aligned16(a) && aligned16(b) && aligned16(grad))
        l1_grad_kernel<true><<<grid_for(n / 4, sm_count), 256, 0, st>>>(a, b, n, scale, upstream, grad);
    else
        l1_grad_kernel<false><<<grid_for(n, sm_count), 256, 0, st>>>(a, b, n, scale, upstream, grad);
    return cudaGetLastError();
}

cudaError_t launch_plane_regulation(const G4DDeformParams& prm, const G4DDeformGrads* grads, float w_plane_tv, float w_time_smooth,
                                    float w_l1_time, const float* upstream, float* loss, int sm_count, cudaStream_t st) {
    RegDesc d{};
    int64_t total = 0;
    for (int l = 0; l < prm.levels; ++l)
        for (int k = 0; k < 6; ++k) {
            const int c0 = plane_axis0(k), c1 = plane_axis1(k);
            const bool is_time = c1 == 3;                        // planes 2, 4, 5 (gaussian_model.py:557,570)
            RegPlane& P = d.pl[d.count++];
            P.p = prm.planes[l][k]; P.g = grads ? grads->planes[l][k] : nullptr;
            P.H = prm.res[l][c1]; P.W = prm.res[l][c0]; P.C = prm.channels;
            P.w_smooth = is_time ? w_time_smooth : w_plane_tv;   // compute_regulation: plane_tv * _plane + time_smooth * _time + l1 * _l1
            P.w_l1 = is_time ? w_l1_time : 0.f;
            P.start = total;
            total += (int64_t)P.H * P.W * P.C;
        }
    d.total = total;
    if (total == 0) return cudaSuccess;
    plane_regulation_kernel<<<grid_for(total, sm_count), 256, 0, st>>>(d, loss, upstream);
    return cudaGetLastError();
}

cudaError_t launch_ssim_forward(const float* x, const float* y, int C, int H, int W, float scale, float* loss, float* dmu, float* dxx,
                                float* dxy, cudaStream_t st) {
    if ((int64_t)C * H * W == 0) return cudaSuccess;
    const dim3 grid((W + kSsimT - 1) / kSsimT, (H + kSsimT - 1) / kSsimT, C);
    ssim_forward_kernel<<<grid, kSsimT * kSsimT, 0, st>>>(make_ssim_window(), x, y, H, W, scale, loss, dmu, dxx, dxy);
    return cudaGetLastError();
}
cudaError_t launch_ssim_backward(const float* x, const float* y, int C, int H, int W, float scale, const float* upstream,
                                 const float* dmu, const float* dxx, const float* dxy, float* grad, cudaStream_t st) {
    if ((int64_t)C * H * W == 0) return cudaSuccess;
    const dim3 grid((W + kSsimT - 1) / kSsimT, (H + kSsimT - 1) / kSsimT, C);
    ssim_backward_kernel<<<grid, kSsimT * kSsimT, 0, st>>>(make_ssim_window(), x, y, H, W, scale, upstream, dmu, dxx, dxy, grad);
    return cudaGetLastError();
}

}  // namespace g4d
