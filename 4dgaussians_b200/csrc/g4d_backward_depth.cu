// g4d_backward_depth.cu -- the per-Gaussian backward kernels with a depth gradient (per_gaussian_bwd.cuh): dL/d(view-space
// depth) of the blend backward joins dL/d p_view.z.  Compiled with the default FMA contraction, as g4d_backward.cu.
#include "per_gaussian_bwd.cuh"

namespace g4d {

cudaError_t launch_preprocess_backward_depth(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                             const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                             float* g_means2D_out, float* g_scales, float* g_rotations, const ShOut& g_sh,
                                             float* g_cam, const float* g_depth, cudaStream_t st) {
    return launch_per_gaussian_backward(preprocess_backward_kernel<false, false, true>, preprocess_backward_kernel<false, true, true>,
                                        preprocess_backward_kernel<true, false, true>, preprocess_backward_kernel<true, true, true>,
                                        g_sh.m == kShCoeffs, g_cam != nullptr, n, st, cam, n, in, g, g_mean2D, g_conic, g_rgb,
                                        g_means3D, g_means2D_out, g_scales, g_rotations, g_sh, g_cam, g_depth);
}

cudaError_t launch_preprocess_backward_cameras_depth(const BackwardCameras& bc, int64_t n, const RasterInputs& in, float* g_means3D,
                                                     float* g_scales, float* g_rotations, float* g_opacities, const ShOut& g_sh,
                                                     const CamGradSinks* cs, cudaStream_t st) {
    return launch_per_gaussian_backward(
        preprocess_backward_cameras_kernel<false, false, true>, preprocess_backward_cameras_kernel<false, true, true>,
        preprocess_backward_cameras_kernel<true, false, true>, preprocess_backward_cameras_kernel<true, true, true>,
        g_sh.m == kShCoeffs, cs != nullptr, n, st, bc, n, in, g_means3D, g_scales, g_rotations, g_opacities, g_sh,
        cs ? *cs : CamGradSinks{});
}

}  // namespace g4d
