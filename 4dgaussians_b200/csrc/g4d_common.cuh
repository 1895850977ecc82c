// g4d_common.cuh -- constants, device-side camera, small helpers shared by every kernel.
// Every behavioural constant of the rasterizer lives here (SURVEY.md Appendix A): changing one changes pixels.
#pragma once
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/g4d.h"

#if defined(__CUDACC__)
#define G4D_HD __host__ __device__ __forceinline__
#define G4D_D __device__ __forceinline__
#else
#define G4D_HD inline
#define G4D_D inline
#endif

namespace g4d {

constexpr int kTile = 16;                 // BLOCK_X = BLOCK_Y (A: 16x16 pixel tiles)
constexpr int kTilePixels = kTile * kTile;
constexpr int kShCoeffs = 16;             // coefficient slots per Gaussian ([N,16,3])
constexpr int kCamGradFloats = 35;        // a camera's gradient: view [16], proj [16], campos [3] (g4d_context_set_camera_grad)
constexpr float kNearCull = 0.2f;         // A.1 step 2
constexpr float kWEps = 0.0000001f;       // A.1 step 3
constexpr float kGuardBand = 1.3f;        // A.1 step 5
constexpr float kDilation = 0.3f;         // A.1 step 5
constexpr float kMinDiscriminant = 0.1f;  // A.1 step 7
constexpr float kAlphaMax = 0.99f;        // A.3
constexpr float kAlphaMin = 1.0f / 255.0f;
constexpr float kTransmittanceStop = 0.0001f;
constexpr float kDet2Eps = 0.0000001f;    // A.4 regularised 1/(det^2+eps)

constexpr float kSH0 = 0.28209479177387814f;
constexpr float kSH1 = 0.4886025119029199f;
// degree-2 / degree-3 constants: /root/reference/utils/sh_utils.py:26-43
#define G4D_SH2_0 1.0925484305920792f
#define G4D_SH2_1 -1.0925484305920792f
#define G4D_SH2_2 0.31539156525252005f
#define G4D_SH2_3 -1.0925484305920792f
#define G4D_SH2_4 0.5462742152960396f
#define G4D_SH3_0 -0.5900435899266435f
#define G4D_SH3_1 2.890611442640554f
#define G4D_SH3_2 -0.4570457994644658f
#define G4D_SH3_3 0.3731763325901154f
#define G4D_SH3_4 -0.4570457994644658f
#define G4D_SH3_5 1.445305721320277f
#define G4D_SH3_6 -0.5900435899266435f

// Device-resident camera, written once per forward by pack_camera_kernel and read (uniformly) by all stages.
struct CameraDev {
    int32_t H, W, sh_degree, grid_x;
    int32_t grid_y, num_tiles;
    uint32_t depth_min, depth_max;   // bits of the smallest / largest view-space depth among the visible Gaussians of this
                                     // forward (reset by pack_camera, RED.MIN / RED.MAX by the projection stage, read by bin_sort)
    float tanfovx, tanfovy, scale_modifier, time;
    float focal_x, focal_y;
    uint32_t grid_bar;               // arrival counter of bin_sort_kernel's grid-wide barriers (reset by pack_camera every forward)
    uint32_t pad3;
    float view[16];
    float proj[16];
    float campos[4];
    float bg[4];
};

#if defined(__CUDACC__)
#define G4D_CE __host__ __device__ constexpr
#else
#define G4D_CE constexpr
#endif
// plane-pair axes of combinations(range(4), 2)   (scene/hexplane.py:79): (0,1),(0,2),(0,3),(1,2),(1,3),(2,3)
G4D_CE int plane_axis0(int k) { return k < 3 ? 0 : (k < 5 ? 1 : 2); }
G4D_CE int plane_axis1(int k) { return k == 0 ? 1 : (k == 1 || k == 3) ? 2 : 3; }

// head output widths: pos, scales, rotations, opacity, shs
G4D_CE int head_out(int h) { return h == 0 ? 3 : h == 1 ? 3 : h == 2 ? 4 : h == 3 ? 1 : 48; }
// column offset of head h inside the per-Gaussian delta row (always the full 59-wide layout)
G4D_CE int head_col(int h) { return h == 0 ? 0 : h == 1 ? 3 : h == 2 ? 6 : h == 3 ? 10 : 11; }
constexpr int kDeltaCols = 59;

#if defined(__CUDACC__)
// ---- programmatic dependent launch (sm_90+): a kernel launched with the "programmatic stream serialization" attribute may
// become resident while the previous kernel of the stream is still draining; it must not touch anything that kernel (or the
// one before it) wrote, nor write anything they read, before pdl_wait().  Every kernel of the forward chain does
// `pdl_wait(); pdl_trigger();` in that order: a dependent can then only start once ALL CTAs of its predecessor are past
// their own wait, i.e. once the predecessor's predecessor has completed -- what a kernel does before its wait may therefore
// read anything older than its direct predecessor (parameters, weight images), and only that.  Both are no-ops in a kernel
// launched the ordinary way.
G4D_D void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
G4D_D void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

extern int g_pdl;   // process-wide switch (G4D_OPT_PDL / env G4D_PDL; g4d_api.cu)

// <<<grid, block, smem, st>>> with the programmatic-stream-serialization attribute when `pdl` is set
template <class... KArgs, class... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = (pdl && g_pdl) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

G4D_D float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// block-wide sum (any block size that is a multiple of 32, <= 1024); result valid in thread 0
G4D_D float block_sum_f(float v) {
    __shared__ float s_part[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum_f(v);
    __syncthreads();
    if (lane == 0) s_part[warp] = v;
    __syncthreads();
    float r = 0.f;
    if (warp == 0) {
        r = lane < (int)(blockDim.x >> 5) ? s_part[lane] : 0.f;
        r = warp_sum_f(r);
    }
    return r;
}
#endif

}  // namespace g4d
