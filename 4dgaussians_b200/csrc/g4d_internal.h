// g4d_internal.h -- host-side declarations shared by the translation units of libg4d.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "deform_tile.cuh"
#include "g4d_common.cuh"

namespace g4d {

// per-Gaussian projected record kept by a forward (SoA; sizes in DESIGN.md §3)
struct GeomBuffers {
    float4* rec0;        // (px, py, conic.x, conic.y)
    float4* rec1;        // (conic.z, opacity, r, g)
    float2* rec2;        // (b, depth)
    int32_t* radii;
    uint2* rect;         // x = minx | miny<<16, y = maxx | maxy<<16   (tile units)
    uint32_t* tiles_touched;
    uint32_t* perm;      // the VISIBLE Gaussians' indices sorted by (depth bits, index)   (bin_sort_kernel)
    uint32_t* depth_range;   // -> CameraDev.depth_min / depth_max of this context
    uint8_t* clamped;    // bit ch set when the forward clamped colour channel ch at 0
};

struct BinBuffers {
    uint2* kbuf;            // [capacity] placement scratch: (depth rank, Gaussian index)
    uint32_t* ids_sorted;   // [capacity] Gaussian index of every (tile, Gaussian) instance, tile-major, depth-ordered per tile
    uint2* ranges;          // [tiles] (start, end) into ids_sorted
};

// ---- binning (g4d_bin.cu) ---------------------------------------------------------------------------------------
struct BinCtl { uint32_t n_visible, R, overflow, pad; long long phase_clk[16]; };   // device-resident results of one forward's binning (+ CTA 0's clock at every phase boundary)
struct BinSortArgs {
    int64_t n;
    const float2* rec2; const uint32_t* tiles_touched; const uint2* rect; const float4* rec0; const float4* rec1;
    const uint32_t* depth_range;   // [2] min / max depth bits of the visible Gaussians (written by the projection stage)
    uint32_t* grid_bar;            // arrival counter of the grid-wide barriers (CameraDev.grid_bar, zero at launch)
    uint32_t *kA, *vA, *kB, *vB;   // [N] ping-pong buffers of the depth sort
    uint32_t* perm;                // [N] out: visible Gaussians in depth order
    uint32_t* H;                   // [chunks][256] digit histograms of the current pass
    uint32_t* S;                   // [chunks] tiles_touched sums of equal-count slices
    uint32_t* chunk_start;         // [chunks + 1] positions in perm
    uint32_t* M;                   // [chunks][tiles] instance counts, then exclusive prefix over the chunks
    uint32_t* tile_total;          // [tiles] instances per tile
    BinCtl* ctl;
    int grid_x, grid_y, num_tiles, count_band_rows;
    int tight;
};
struct BinPlaceArgs {
    const uint32_t* perm; const uint2* rect; const float4* rec0; const float4* rec1;
    const uint32_t* chunk_start; const uint32_t* M; const uint32_t* tile_total;
    uint32_t* tile_start;          // [tiles] exclusive scan of tile_total (written by placement CTA 0, read by the fix-up)
    uint2* ranges;                 // [tiles] (start, end) clamped to the capacity; empty tiles (0, 0)
    uint32_t* ids;                 // [capacity] final instance list (Gaussian indices)
    uint2* kbuf;                   // [capacity] (depth rank, Gaussian index) as placed: unordered inside a (tile, chunk) sub-segment
    uint32_t capacity;
    int grid_x, grid_y, num_tiles, band_rows, tight;
};
struct BinLayout { uint32_t* chunk_start; uint32_t* M; uint32_t* tile_total; uint32_t* tile_start; BinCtl* ctl; int chunks; };
size_t bin_aux_bytes(int64_t n, int num_tiles, int sm_count);
// depth sort + chunking + per-(tile, chunk) counts + scan over the chunks: M, tile_total, ctl->R.  One cooperative launch.
cudaError_t launch_bin_sort(int64_t n, int grid_x, int grid_y, const GeomBuffers& g, void* aux, int tight, int sm_count,
                            BinLayout* out, cudaStream_t st);
// tile ranges + placement of every instance into its (tile, chunk) sub-segment + per-sub-segment ordering (2 launches)
cudaError_t launch_bin_place(int grid_x, int grid_y, const GeomBuffers& g, const BinLayout& lay, uint32_t* ids, uint2* kbuf,
                             uint2* ranges, uint32_t capacity, int tight, cudaStream_t st);

struct ImageBuffers {
    float* final_T;      // [H*W]
    uint32_t* n_contrib; // [H*W]
};

// inputs of the rasterizer stage in device memory (post-activation), either caller tensors or the
// tensors the fused path produced
struct RasterInputs {
    const float* means3D; const float* scales; const float* rotations; const float* opacities;
    const float* shs;       // fused [N,16,3] or NULL
    const float* sh_dc;     // used when shs == NULL: [N,1,3]
    const float* sh_rest;   //                        [N,15,3]
};

struct FusedOutputs {   // what the fused forward saves for its backward (may be NULL in deform-only mode)
    float* means3D; float* scales; float* rotations; float* opacities;
    float* shs;        // deformed SH coefficients, only when the SHS head is active
    float* rot_norm;   // |q| before F.normalize (needed by its backward)
};

// tensor-core weight images (g4d_deform_tc.cu): (hi | lo) parts in the canonical K-major shared-memory layout (tc_wgmma.cuh),
// FP16x2 (scaled f16) or 3xTF32 words
struct TcWeights {
    const float* w0;                   // packed (hi | lo), [128][F]
    const float* w1[G4D_NUM_HEADS];    // packed (hi | lo) K-parts, [128][128]
    const float* w2[G4D_NUM_HEADS];    // SH head only: packed (hi | lo), [48][128]
    long long* dbg;                    // optional [grid][12] per-phase cycle counters (debug)
    float* feat;                       // [N][F] fp32 staging of the HexPlane features (deform_features_kernel)
    uint32_t* relu_bits;               // optional [6][N][4]: ReLU sign bits saved for the backward (G4D_RELU_BITS_WORDS)
    int arith;                         // 1: 3xTF32, 2: FP16x2 (G4D_OPT_TENSOR_CORES)
    uint32_t* status;                  // host-mapped word: set to 1 by the FP16x2 kernel when a value left the f16 operand range
};

size_t tc_packed_floats(const G4DDeformParams& prm);
cudaError_t launch_tc_pack_weights(const G4DDeformParams& prm, int arith, float* blob, TcWeights* out, cudaStream_t st);
bool tc_deform_supported(const DeformDesc& d, int arith);

// tensor-core backward (g4d_deform_tc_bwd.cu): BF16 (hi | lo) weight images in the 8x8-core layout of tc_wgmma.cuh
struct TcBwdWeights {
    const uint8_t* w0;                    // image [128][F]
    const uint8_t* w1[G4D_NUM_HEADS];     // image [128][128]
    const uint8_t* w2sh;                  // SH head: image of W2^T [128][48]
};
size_t tc_bwd_weight_bytes(const G4DDeformParams& prm);
cudaError_t launch_tc_bwd_pack_weights(const G4DDeformParams& prm, uint8_t* blob, TcBwdWeights* out, cudaStream_t st);
bool tc_backward_supported(const DeformDesc& d);
size_t tc_deform_backward_scratch_bytes(const DeformDesc& d, int64_t n);
cudaError_t launch_deform_backward_tc(const DeformDesc& d, const G4DDeformParams& prm, const G4DDeformGrads& grads,
                                      const TcBwdWeights& w, float time, int64_t n, const float* xyz,
                                      const float* const go[G4D_NUM_HEADS], float* const gi[G4D_NUM_HEADS],
                                      const uint32_t* relu_bits, const float* saved_feat, uint8_t* scratch, int sm_count,
                                      cudaStream_t st);
// collapsed time-row gradients -> the two time rows of each (axis, t) plane (g4d_backward.cu)
cudaError_t launch_distribute_time_grad(const DeformDesc& d, float* const (*trow_grad)[3], float* const (*g_planes)[6], float time,
                                        cudaStream_t st);

// ---- launchers (defined in g4d_geom.cu / g4d_raster.cu / g4d_backward.cu) -----------------------------
cudaError_t launch_pack_camera(const G4DCamera& cam, CameraDev* dst, cudaStream_t st);
cudaError_t launch_pack_weights(const G4DDeformParams& p, float* w0t, float* const* w1t, cudaStream_t st);
cudaError_t launch_collapse_time_rows(const G4DDeformParams& p, const CameraDev* cam, float time, bool use_cam_time,
                                      float* const (*trow)[3], cudaStream_t st);
cudaError_t launch_preprocess(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g, int32_t* out_radii,
                              cudaStream_t st);
// mode 0: deform only (writes the five out_* tensors); mode 1: fused deform + preprocess
cudaError_t launch_deform(const DeformDesc& d, int mode, const CameraDev* cam, float time, bool use_cam_time, int64_t n,
                          const float* xyz, const float* scaling, const float* rotation, const float* opacity,
                          const float* shs, const float* sh_dc, const float* sh_rest, float* out_xyz, float* out_scaling,
                          float* out_rotation, float* out_opacity, float* out_shs, GeomBuffers g, FusedOutputs fo,
                          int32_t* out_radii, int sm_count, cudaStream_t st, const TcWeights* tw = nullptr);

cudaError_t launch_blend_forward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                 float* out_color, float* out_depth, int warp_cull, cudaStream_t st);
cudaError_t launch_blend_backward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                  const float* dL_dcolor, float* g_mean2D, float* g_conic, float* g_opacity, float* g_rgb,
                                  int warp_cull, cudaStream_t st);
// per-Gaussian backward; g_shs may alias separate dc/rest sinks through (g_sh_dc, g_sh_rest) when g_shs == NULL
cudaError_t launch_preprocess_backward(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                       const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                       float* g_means2D_out, float* g_scales, float* g_rotations, float* g_shs,
                                       float* g_sh_dc, float* g_sh_rest, cudaStream_t st);   // fused and split SH sinks may both be given

size_t deform_backward_scratch_bytes(const DeformDesc& d, int64_t n);
// go[h] / gi[h]: gradient w.r.t. the outputs / inputs of head h's residual tensor (xyz, scaling, rotation, opacity, shs)
cudaError_t launch_deform_backward(const DeformDesc& d, const G4DDeformParams& prm, const G4DDeformGrads& grads, float time,
                                   int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                                   float* const gi[G4D_NUM_HEADS], float* scratch, int sm_count, cudaStream_t st);
// coarse stage of render(): activations + projection without the deformation network
cudaError_t launch_activate_preprocess(const CameraDev* cam, int64_t n, const float* xyz, const float* scaling,
                                       const float* rotation, const float* opacity, const float* shs, const float* sh_dc,
                                       const float* sh_rest, GeomBuffers g, FusedOutputs fo, int32_t* out_radii,
                                       cudaStream_t st);
// chain rule through exp / normalize / sigmoid (gaussian_renderer/__init__.py:97-99); in-place on the gradient buffers
cudaError_t launch_activation_backward(int64_t n, const FusedOutputs& fo, float* g_scales, float* g_rotations,
                                       float* g_opacities, cudaStream_t st);

// ---- losses either side of the path (g4d_loss.cu) -------------------------------------------------------------------
cudaError_t launch_l1_loss(const float* a, const float* b, int64_t n, float scale, float* loss, int sm_count, cudaStream_t st);
cudaError_t launch_l1_grad(const float* a, const float* b, int64_t n, float scale, const float* upstream, float* grad, int sm_count,
                           cudaStream_t st);
cudaError_t launch_plane_regulation(const G4DDeformParams& prm, const G4DDeformGrads* grads, float w_plane_tv, float w_time_smooth,
                                    float w_l1_time, const float* upstream, float* loss, int sm_count, cudaStream_t st);
cudaError_t launch_ssim_forward(const float* x, const float* y, int C, int H, int W, float scale, float* loss, float* dmu, float* dxx,
                                float* dxy, cudaStream_t st);
cudaError_t launch_ssim_backward(const float* x, const float* y, int C, int H, int W, float scale, const float* upstream,
                                 const float* dmu, const float* dxx, const float* dxy, float* grad, cudaStream_t st);

// ---- flat Adam (g4d_optim.cu) ------------------------------------------------------------------------------------------
cudaError_t launch_adam_flat(float* p, const float* g, float* m, float* v, int64_t numel, const G4DAdamSegment* segs, int nseg,
                             float b1, float b2, float eps, int64_t step, float grad_scale, int sm_count, cudaStream_t st);

// ---- 3-nearest-neighbour mean squared distance (g4d_knn.cu) ---------------------------------------------------------
size_t knn_scratch_bytes(int64_t n);
cudaError_t launch_knn_dist2(int64_t n, const float* xyz, float* out, void* scratch, int sm_count, cudaStream_t st);


}  // namespace g4d
