// g4d_geom_bwd.cu -- per-Gaussian backward of the projection stage (A.4): gradients w.r.t. the means, scales, rotations and
// SH coefficients of the Gaussians, and optionally w.r.t. each camera, for one camera (launch_preprocess_backward) or several
// cameras at one timestamp (launch_preprocess_backward_cameras), with or without a depth gradient.  Kept apart from the
// deformation network's backward (g4d_backward.cu): the code NVVM makes of a kernel can depend on the other kernels of its
// translation unit.  Compiled with the default FMA contraction.
#include "g4d_internal.h"
#include "g4d_math.cuh"

namespace g4d {

// Adds the camera terms of the warp's lanes [0, cnt) into acc[kCamGradFloats]: a shuffle tree to lane 0 per element the
// forward reads, then one atomic per such element.  Called by exactly the lanes [0, cnt) (cnt >= 1).
G4D_D void cam_grad_flush(const CamGrad& cg, int lane, int cnt, float* __restrict__ acc) {
    const unsigned mask = cnt == 32 ? 0xffffffffu : (1u << cnt) - 1u;
#pragma unroll
    for (int i = 0; i < kCamGradFloats; ++i) {
        if (!cam_grad_read(i)) continue;
        float s = cg.g[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float t = __shfl_down_sync(mask, s, o);
            if (lane + o < cnt) s = add_rn(s, t);
        }
        if (lane == 0) atomicAdd(acc + i, s);
    }
}

// FULL: M = 16 SH coefficients per Gaussian (ShIn), else M = in.sh.m = g_sh.m.  CAM: the camera's gradient is added into
// g_cam[kCamGradFloats] (zeroed by the caller).  DEPTH: g_depth [N] is dL/d(view-space depth) (not read otherwise).
template <bool FULL, bool CAM, bool DEPTH>
__global__ void __launch_bounds__(256)
preprocess_backward_kernel(const CameraDev* __restrict__ camp, int64_t n, RasterInputs in, GeomBuffers g,
                           const float* __restrict__ g_mean2D, const float* __restrict__ g_conic,
                           const float* __restrict__ g_rgb, float* __restrict__ g_means3D, float* __restrict__ g_means2D_out,
                           float* __restrict__ g_scales, float* __restrict__ g_rotations, ShOut g_sh, float* __restrict__ g_cam,
                           const float* __restrict__ g_depth) {
    // SH coefficients travel through shared memory: a warp reads / writes the 32 x 48 floats of its Gaussians as contiguous
    // 128-byte lines instead of 48 scalar accesses per thread at a 192-byte stride
    extern __shared__ float sh_smem[];             // [warps][2][32 * kShRow]
    __shared__ CameraDev cam;
    stage_cameras(&cam, &camp, 1);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* ld = sh_smem + (size_t)warp * 2 * 32 * kShRow;
    float* st = ld + 32 * kShRow;
    const int64_t g0 = (int64_t)blockIdx.x * blockDim.x + warp * 32;
    const int cnt = (int)(n - g0 < 32 ? (n - g0 > 0 ? n - g0 : 0) : 32);
    if (cnt == 0) return;                          // whole warp
    const int64_t gi = g0 + lane;
    const bool active = lane < cnt;
    in.sh.stage_warp<FULL>(g0, cnt, lane, ld);
    __syncwarp();
    auto sh_store = [&](int k, int ch, float v) { st[lane * kShRow + 3 * k + ch] = v; };
    if (active) {
        CamGrad cg;
        if constexpr (CAM)
#pragma unroll
            for (int i = 0; i < kCamGradFloats; ++i) cg.g[i] = 0.f;
        if (g_means2D_out) {
            const bool vis = g.radii[gi] > 0;
            g_means2D_out[3 * gi] = vis ? g_mean2D[2 * gi] : 0.f;
            g_means2D_out[3 * gi + 1] = vis ? g_mean2D[2 * gi + 1] : 0.f;
            g_means2D_out[3 * gi + 2] = 0.f;
        }
        if (!(g.radii[gi] > 0)) {
            for (int k = 0; k < 3; ++k) { g_means3D[3 * gi + k] = 0.f; g_scales[3 * gi + k] = 0.f; }
            for (int k = 0; k < 4; ++k) g_rotations[4 * gi + k] = 0.f;
            for (int k = 0; k < kShCoeffs; ++k)
                for (int ch = 0; ch < 3; ++ch) sh_store(k, ch, 0.f);
        } else {
            const Vec3 p{in.means3D[3 * gi], in.means3D[3 * gi + 1], in.means3D[3 * gi + 2]};
            const Vec3 sc{in.scales[3 * gi], in.scales[3 * gi + 1], in.scales[3 * gi + 2]};
            const float4 q4 = *reinterpret_cast<const float4*>(in.rotations + 4 * gi);
            const float gm2[2] = {g_mean2D[2 * gi], g_mean2D[2 * gi + 1]};
            const float gc[3] = {g_conic[3 * gi], g_conic[3 * gi + 1], g_conic[3 * gi + 2]};
            const float gr[3] = {g_rgb[3 * gi], g_rgb[3 * gi + 1], g_rgb[3 * gi + 2]};
            GaussGrad gg;
            const float* row = ld + lane * kShRow;
            gaussian_backward<CAM, DEPTH>(cam, p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, (uint32_t)g.clamped[gi], gm2, gc, gr,
                                          [&](int k, int ch) { return row[3 * k + ch]; }, sh_store, gg, &cg,
                                          DEPTH ? g_depth[gi] : 0.f);
            for (int k = 0; k < 3; ++k) { g_means3D[3 * gi + k] = gg.mean[k]; g_scales[3 * gi + k] = gg.scale[k]; }
            for (int k = 0; k < 4; ++k) g_rotations[4 * gi + k] = gg.rot[k];
        }
        if constexpr (CAM) cam_grad_flush(cg, lane, cnt, g_cam);
    }
    __syncwarp();
    g_sh.store_warp<FULL>(g0, cnt, lane, st);
}

// Per-Gaussian backward of several cameras at one timestamp (g4d_render_backward_cameras): the deformed state and the SH
// coefficients are loaded once, gaussian_backward runs for every camera that sees the Gaussian, and the sums -- mean,
// scale and rotation in registers, SH in the warp's shared-memory rows, opacity from the cameras' blend backward passes --
// are written once.  Each camera's screen-space gradient goes to its own sink.  CAM: camera c's gradient is added into
// cs.out[c][kCamGradFloats] (zeroed by the caller; NULL: not wanted), reduced over the warp inside the loop over the cameras.
// DEPTH: each camera's blend gradient has the depth block (BlendGradLayout::kDepth), its dL/d(view-space depth).
template <bool FULL, bool CAM, bool DEPTH>
__global__ void __launch_bounds__(128)
preprocess_backward_cameras_kernel(BackwardCameras bc, int64_t n, RasterInputs in, float* __restrict__ g_means3D,
                                   float* __restrict__ g_scales, float* __restrict__ g_rotations, float* __restrict__ g_opacities,
                                   ShOut g_sh, CamGradSinks cs) {
    extern __shared__ float sh_smem[];             // [warps][2][32 * kShRow]: SH coefficients, SH gradient sums
    __shared__ CameraDev cams[G4D_MAX_CAMERAS];
    stage_cameras(cams, bc.cam, bc.count);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* ld = sh_smem + (size_t)warp * 2 * 32 * kShRow;
    float* st = ld + 32 * kShRow;
    const int64_t g0 = (int64_t)blockIdx.x * blockDim.x + warp * 32;
    const int cnt = (int)(n - g0 < 32 ? (n - g0 > 0 ? n - g0 : 0) : 32);
    if (cnt == 0) return;
    const int64_t gi = g0 + lane;
    in.sh.stage_warp<FULL>(g0, cnt, lane, ld);
    for (int idx = lane; idx < cnt * 48; idx += 32) st[idx / 48 * kShRow + idx % 48] = 0.f;
    __syncwarp();
    if (lane < cnt) {
        const Vec3 p{in.means3D[3 * gi], in.means3D[3 * gi + 1], in.means3D[3 * gi + 2]};
        const Vec3 sc{in.scales[3 * gi], in.scales[3 * gi + 1], in.scales[3 * gi + 2]};
        const float4 q4 = *reinterpret_cast<const float4*>(in.rotations + 4 * gi);
        const float* row = ld + lane * kShRow;
        float* srow = st + lane * kShRow;
        float gm[3] = {0.f, 0.f, 0.f}, gs[3] = {0.f, 0.f, 0.f}, gr[4] = {0.f, 0.f, 0.f, 0.f}, gop = 0.f;
        using L = BlendGradLayout;
        for (int c = 0; c < bc.count; ++c) {
            const float* gb = bc.grad[c];
            const float* gmb = gb + L::kMean2D * n;
            const float* gcb = gb + L::kConic * n;
            const float* grb = gb + L::kRgb * n;
            gop += gb[L::kOpacity * n + gi];
            const bool vis = bc.radii[c][gi] > 0;
            if (bc.g_means2D[c]) {
                bc.g_means2D[c][3 * gi] = vis ? gmb[2 * gi] : 0.f;
                bc.g_means2D[c][3 * gi + 1] = vis ? gmb[2 * gi + 1] : 0.f;
                bc.g_means2D[c][3 * gi + 2] = 0.f;
            }
            CamGrad cg;
            if constexpr (CAM)
#pragma unroll
                for (int i = 0; i < kCamGradFloats; ++i) cg.g[i] = 0.f;
            if (vis) {
                const float gm2[2] = {gmb[2 * gi], gmb[2 * gi + 1]};
                const float gc[3] = {gcb[3 * gi], gcb[3 * gi + 1], gcb[3 * gi + 2]};
                const float grgb[3] = {grb[3 * gi], grb[3 * gi + 1], grb[3 * gi + 2]};
                GaussGrad gg;
                gaussian_backward<CAM, DEPTH>(cams[c], p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, (uint32_t)bc.clamped[c][gi], gm2, gc,
                                              grgb, [&](int k, int ch) { return row[3 * k + ch]; },
                                              [&](int k, int ch, float v) { srow[3 * k + ch] += v; }, gg, &cg,
                                              DEPTH ? gb[L::kDepth * n + gi] : 0.f);
                for (int k = 0; k < 3; ++k) { gm[k] += gg.mean[k]; gs[k] += gg.scale[k]; }
                for (int k = 0; k < 4; ++k) gr[k] += gg.rot[k];
            }
            if constexpr (CAM)
                if (cs.out[c]) cam_grad_flush(cg, lane, cnt, cs.out[c]);
        }
        for (int k = 0; k < 3; ++k) { g_means3D[3 * gi + k] = gm[k]; g_scales[3 * gi + k] = gs[k]; }
        for (int k = 0; k < 4; ++k) g_rotations[4 * gi + k] = gr[k];
        g_opacities[gi] = gop;
    }
    __syncwarp();
    g_sh.store_warp<FULL>(g0, cnt, lane, st);
}

// Both kernels run one Gaussian per thread in blocks of 128, with 50 KB of dynamic shared memory: each warp's
// [2][32 * kShRow] floats of SH staging.
constexpr int kBwdThreads = 128;
constexpr size_t kBwdSmem = (size_t)(kBwdThreads / 32) * 2 * 32 * kShRow * sizeof(float);

cudaError_t launch_preprocess_backward(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                       const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                       float* g_means2D_out, float* g_scales, float* g_rotations, const ShOut& g_sh,
                                       float* g_cam, const float* g_depth, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    using K = decltype(&preprocess_backward_kernel<false, false, false>);
    const K kernel[2][2][2] = {   // [FULL][CAM][DEPTH]
        {{preprocess_backward_kernel<false, false, false>, preprocess_backward_kernel<false, false, true>},
         {preprocess_backward_kernel<false, true, false>, preprocess_backward_kernel<false, true, true>}},
        {{preprocess_backward_kernel<true, false, false>, preprocess_backward_kernel<true, false, true>},
         {preprocess_backward_kernel<true, true, false>, preprocess_backward_kernel<true, true, true>}}};
    return launch_k(kernel[g_sh.m == kShCoeffs][g_cam != nullptr][g_depth != nullptr], (unsigned)((n + kBwdThreads - 1) / kBwdThreads),
                    kBwdThreads, kBwdSmem, st, kOrdinary, cam, n, in, g, g_mean2D, g_conic, g_rgb, g_means3D, g_means2D_out, g_scales,
                    g_rotations, g_sh, g_cam, g_depth);
}

cudaError_t launch_preprocess_backward_cameras(const BackwardCameras& bc, int64_t n, const RasterInputs& in, float* g_means3D,
                                               float* g_scales, float* g_rotations, float* g_opacities, const ShOut& g_sh,
                                               const CamGradSinks* cs, bool depth, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    using K = decltype(&preprocess_backward_cameras_kernel<false, false, false>);
    const K kernel[2][2][2] = {   // [FULL][CAM][DEPTH]
        {{preprocess_backward_cameras_kernel<false, false, false>, preprocess_backward_cameras_kernel<false, false, true>},
         {preprocess_backward_cameras_kernel<false, true, false>, preprocess_backward_cameras_kernel<false, true, true>}},
        {{preprocess_backward_cameras_kernel<true, false, false>, preprocess_backward_cameras_kernel<true, false, true>},
         {preprocess_backward_cameras_kernel<true, true, false>, preprocess_backward_cameras_kernel<true, true, true>}}};
    return launch_k(kernel[g_sh.m == kShCoeffs][cs != nullptr][depth], (unsigned)((n + kBwdThreads - 1) / kBwdThreads), kBwdThreads,
                    kBwdSmem, st, kOrdinary, bc, n, in, g_means3D, g_scales, g_rotations, g_opacities, g_sh, cs ? *cs : CamGradSinks{});
}

}  // namespace g4d
