// g4d_internal.h -- host-side declarations shared by the translation units of libg4d.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "deform_tile.cuh"
#include "g4d_common.cuh"

namespace g4d {

// Hands out consecutive sub-ranges of one buffer, each starting on a 256-byte boundary, in the order they are taken.
// Without a base it hands out null pointers and only counts bytes: one layout function then both sizes a buffer
// (Carve{}, then bytes()) and places its pointers (Carve{base}).
struct Carve {
    char* base;
    size_t off = 0;
    explicit Carve(void* b = nullptr) : base(static_cast<char*>(b)) {}
    template <class T> T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += (count * sizeof(T) + 255) / 256 * 256;
        return p;
    }
    size_t bytes() const { return off; }
};

// The collapsed time rows of a deformation network, level-major, time axis a = x, y, z within a level: row (l, a) holds
// res[l][a] * C floats from start[3 * l + a]; start[3 * levels] is the total.  The same layout holds their gradients.
struct TimeRows {
    int levels = 0;
    int start[G4D_MAX_LEVELS * 3 + 1] = {};
    TimeRows(int levels_, const int32_t (*res)[4], int C) : levels(levels_) {
        for (int m = 0; m < 3 * levels; ++m) start[m + 1] = start[m] + res[m / 3][m % 3] * C;
    }
    size_t total() const { return (size_t)start[3 * levels]; }
    void place(float* base, float* (*rows)[3]) const {
        for (int m = 0; m < 3 * levels; ++m) rows[m / 3][m % 3] = base + start[m];
    }
};

// the time planes among a level's six, for time axes a = x, y, z: (x,t), (y,t), (z,t)
constexpr int kTimePlane[3] = {2, 4, 5};

// A kernel with one thread per float of the collapsed time rows: segment (l, a) is element range [start[3l+a], start[3l+a+1])
// and moves data from src[l][a] to dst[l][a].  The time-row collapse reads the time planes and writes the rows; the
// backward reads the rows' gradients and adds into the time planes' gradients.  The caller sets src and dst.
struct TimeRowSegs : TimeRows {
    int C;
    int res[G4D_MAX_LEVELS][4];
    const float* src[G4D_MAX_LEVELS][3];
    float* dst[G4D_MAX_LEVELS][3];
    TimeRowSegs(int levels_, const int32_t (*res_)[4], int C_) : TimeRows(levels_, res_, C_), C(C_), res{}, src{}, dst{} {
        for (int l = 0; l < levels; ++l)
            for (int a = 0; a < 4; ++a) res[l][a] = res_[l][a];
    }
    // element i < total() is element e of segment (level l, time axis a)
    G4D_D void locate(int i, int& l, int& a, int& e) const {
        int m = 0;
        while (i >= start[m + 1]) ++m;
        l = m / 3; a = m % 3; e = i - start[m];
    }
};

// The timestamp of a forward or backward: read from src (device; g4d_context_set_time_source) when it is set, so that a
// replayed CUDA graph sees the value of the replay, else `value`.
struct TimeArg {
    float value;
    const float* src;
    G4D_D float get() const { return src ? *src : value; }
};

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
size_t bin_aux_bytes(int64_t n, int num_tiles, int sm_count);   // size of launch_bin_sort's aux area
// depth sort + chunking + per-(tile, chunk) counts + scan over the chunks: M, tile_total, ctl->R.  One cooperative launch.
cudaError_t launch_bin_sort(int64_t n, int grid_x, int grid_y, const GeomBuffers& g, void* aux, int tight, int sm_count,
                            BinLayout* out, cudaStream_t st);
// tile ranges + placement of every instance into its (tile, chunk) sub-segment + per-sub-segment ordering (2 launches)
cudaError_t launch_bin_place(int grid_x, int grid_y, const GeomBuffers& g, const BinLayout& lay, uint32_t* ids, uint2* kbuf,
                             uint2* ranges, uint32_t capacity, int tight, cudaStream_t st);
// the overflow record of a captured no-sync forward: when ctl->R exceeds the capacity, words[0] += 1 and
// words[1] = max(words[1], R) (host-mapped words, g4d_workspace_graph_status)
cudaError_t launch_record_overflow(const BinCtl* ctl, uint32_t capacity, uint32_t* words, cudaStream_t st);

struct ImageBuffers {
    float* final_T;      // [H*W]
    uint32_t* n_contrib; // [H*W]
};

// ---- SH coefficients: one source and one sink type for both layouts ----------------------------------------------
// The accessors only move data: they are shared by units compiled with and without FMA contraction.
constexpr int kShRow = 49;   // floats per Gaussian in a warp's shared-memory SH rows: lane i <-> row i is bank-conflict free

// A Gaussian's M x 3 coefficients (M = (max degree + 1)^2: 1, 4, 9 or 16), fused [N,M,3] in shs, or (shs == NULL) split into
// dc [N,1,3] + rest [N,M-1,3].  Only coefficients k < M exist; the colour reads k < (active degree + 1)^2 <= M.
// FULL (the accessors' template argument): M = 16 known at compile time, so that the degree-3 kernels keep constant strides;
// otherwise M = m at run time.  At M = 1 the two layouts are the same [N,1,3] tensor: rest is never read.
struct ShIn {
    const float *shs, *dc, *rest;
    int m = kShCoeffs;
    template <bool FULL> G4D_D int coeffs() const { return FULL ? kShCoeffs : m; }
    // coefficient e = 3 * k + ch of Gaussian gi, e < 3M
    template <bool FULL> G4D_D float at(int64_t gi, int e) const {
        const int s = 3 * coeffs<FULL>();
        return shs ? __ldg(shs + gi * s + e) : e < 3 ? __ldg(dc + gi * 3 + e) : __ldg(rest + gi * (s - 3) + (e - 3));
    }
    // f(load) with load(k, ch) -> coefficient k, channel ch of Gaussian gi; the layout is chosen once, outside f
    template <bool FULL, class F> G4D_D void with_coeffs(int64_t gi, F&& f) const {
        const int s = 3 * coeffs<FULL>();
        if (shs) f([=](int k, int ch) { return __ldg(shs + gi * s + 3 * k + ch); });
        else f([=](int k, int ch) { return k == 0 ? __ldg(dc + gi * 3 + ch) : __ldg(rest + gi * (s - 3) + 3 * (k - 1) + ch); });
    }
    // all 48 of a Gaussian with M = 16 into registers (float4 loads on the fused layout); v[3 * k + ch]
    G4D_D void load(int64_t gi, float (&v)[48]) const {
        if (shs) {
#pragma unroll
            for (int j = 0; j < 48; j += 4) {
                const float4 b = __ldg(reinterpret_cast<const float4*>(shs + gi * 48 + j));
                v[j] = b.x; v[j + 1] = b.y; v[j + 2] = b.z; v[j + 3] = b.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 3; ++j) v[j] = __ldg(dc + gi * 3 + j);
#pragma unroll
            for (int j = 0; j < 45; ++j) v[3 + j] = __ldg(rest + gi * 45 + j);
        }
    }
    // warp-wide: Gaussians g0 .. g0 + cnt - 1 into rows[i * kShRow + 3 * k + ch] for k < M, read as contiguous 128-byte lines
    template <bool FULL> G4D_D void stage_warp(int64_t g0, int cnt, int lane, float* rows) const {
        const int s = 3 * coeffs<FULL>();
        for (int idx = lane; idx < cnt * s; idx += 32) {
            const int i = idx / s, e = idx - i * s;
            rows[i * kShRow + e] = at<FULL>(g0 + i, e);
        }
    }
};

// gradient sinks of the M coefficients (layouts as ShIn's); each may be NULL, and the fused and the split sinks may both be given
struct ShOut {
    float *shs, *dc, *rest;
    int m = kShCoeffs;
    // warp-wide: the inverse of ShIn::stage_warp
    template <bool FULL> G4D_D void store_warp(int64_t g0, int cnt, int lane, const float* rows) const {
        const int s = 3 * (FULL ? kShCoeffs : m);
        for (int idx = lane; idx < cnt * s; idx += 32) {
            const int i = idx / s, e = idx - i * s;
            const float v = rows[i * kShRow + e];
            if (shs) shs[g0 * s + idx] = v;
            if (e < 3) { if (dc) dc[(g0 + i) * 3 + e] = v; }
            else if (rest) rest[(g0 + i) * (s - 3) + (e - 3)] = v;
        }
    }
};

// copies the `count` cameras *src[c] into dst[c] (shared memory), word by word across the block; the caller syncs.
// (P: a camera pointer type, __restrict__ or not)
template <class P>
G4D_D void stage_cameras(CameraDev* dst, const P* src, int count) {
    for (int c = 0; c < count; ++c)
        for (int i = threadIdx.x; i < (int)(sizeof(CameraDev) / 4); i += blockDim.x)
            reinterpret_cast<uint32_t*>(dst + c)[i] = reinterpret_cast<const uint32_t*>(src[c])[i];
}

// inputs of the rasterizer stage in device memory (post-activation), either caller tensors or the
// tensors the fused path produced
struct RasterInputs {
    const float* means3D; const float* scales; const float* rotations; const float* opacities;
    ShIn sh;
};

struct FusedOutputs {   // what the fused forward saves for its backward (may be NULL in deform-only mode)
    float* means3D; float* scales; float* rotations; float* opacities;
    float* shs;        // deformed SH coefficients, only when the SHS head is active
    float* rot_norm;   // |q| before F.normalize (needed by its backward)
};

// tensors of one deformation launch (mode 0 reads xyz .. sh, SH fused, and writes out_*; mode 1, and the coarse stage that
// has no network, read either SH layout and write g, fo and out_radii)
struct DeformIO {
    const float *xyz, *scaling, *rotation, *opacity;
    ShIn sh;
    float *out_xyz, *out_scaling, *out_rotation, *out_opacity, *out_shs;
    GeomBuffers g;
    FusedOutputs fo;
    int32_t* out_radii;
};

// tag word behind the ReLU sign bits (G4D_RELU_BITS_WORDS): the tensor-core forward that wrote the bits sets it (as the
// byte pattern of a memset), anything else clears it
constexpr uint32_t kReluBitsTag = 0x5A5A5A5Au;
constexpr int kReluBitsTagByte = 0x5A;
static_assert(kReluBitsTag == 0x01010101u * (uint32_t)kReluBitsTagByte, "the tag is one byte repeated");

// tensor-core weight images (g4d_deform_tc.cu): (hi | lo) pairs of scaled f16 words in the canonical K-major shared-memory
// layout (tc_wgmma.cuh)
struct TcWeights {
    const float* w0;                   // packed (hi | lo), [128][F]
    const float* w1[G4D_NUM_HEADS];    // packed (hi | lo), [128][128]
    const float* w2[G4D_NUM_HEADS];    // SH head only: packed (hi | lo), [48][128]
    long long* dbg;                    // optional [grid][12] per-phase cycle counters (debug)
    float* feat;                       // the HexPlane features [N][F] and the walk order that gathered them (launch_deform's
    const uint32_t* order;             // DeformGather)
    uint32_t* relu_bits;             // optional [6][N][4]: ReLU sign bits saved for the backward (G4D_RELU_BITS_WORDS)
    uint32_t* status;                  // host-mapped word: set to 1 by the FP16x2 kernel when a value left the f16 operand range
};

size_t tc_packed_floats(const G4DDeformParams& prm);
cudaError_t launch_tc_pack_weights(const G4DDeformParams& prm, float* blob, TcWeights* out, cudaStream_t st);
bool tc_deform_supported(const G4DDeformParams& prm);
// HexPlane gather xyz -> feat [N][F] fp32, Gaussians visited in `order` (NULL: index order; feat[g] stays at row g either
// way); pdl: launched dependent on the previous kernel of the forward chain (DESIGN.md §4.6)
cudaError_t launch_deform_features(const DeformDesc& d, int64_t n, const float* xyz, const uint32_t* order, float* feat, bool pdl,
                                   cudaStream_t st);
// The gather's spatial walk order (DESIGN.md §4.1): order [n] = a permutation of [0, n) in Z order of the Gaussians' cells on a
// 64^3 grid over the normalised HexPlane coordinates, and the scratch of the counting sort that builds it.
constexpr int kOrderCells = 1 << 18;
struct GatherOrderBuffers {
    uint32_t* order;         // [n]
    uint2* key;              // [n] (cell, rank inside the cell)
    uint32_t* cell_start;    // [kOrderCells] counts, then exclusive prefix inside each block of 1024 cells
    uint32_t* block_total;   // [kOrderCells / 1024]
};
// memset + 3 ordinary launches; aabb as in DeformDesc
cudaError_t launch_gather_order(const float* aabb, int64_t n, const float* xyz, const GatherOrderBuffers& b, cudaStream_t st);

// tensor-core backward (g4d_deform_tc_bwd.cu): BF16 (hi | lo) weight images in the 8x8-core layout of tc_wgmma.cuh
struct TcBwdWeights {
    const uint8_t* w0;                    // image [128][F]
    const uint8_t* w1[G4D_NUM_HEADS];     // image [128][128]
    const uint8_t* w2sh;                  // SH head: image of W2^T [128][48]
};
size_t tc_bwd_weight_bytes(const G4DDeformParams& prm);
cudaError_t launch_tc_bwd_pack_weights(const G4DDeformParams& prm, uint8_t* blob, TcBwdWeights* out, cudaStream_t st);
bool tc_backward_supported(const G4DDeformParams& prm);
// The tensor-core engine of the deformation backward (launch_deform_backward runs it): kernel A (dgrad) writes d(feat) [N][F]
// and the operand images of kernel B (wgrad), which writes the weight gradients.  `images`: tc_bwd_images_bytes of scratch.
size_t tc_bwd_images_bytes(const DeformDesc& d, int64_t n);
cudaError_t launch_tc_bwd_dgrad(const DeformDesc& d, const TcBwdWeights& w, int64_t n, const float* const go[G4D_NUM_HEADS],
                                const uint32_t* relu_bits, const float* feat, float* dfeat, uint8_t* images, int sm_count,
                                cudaStream_t st);
cudaError_t launch_tc_bwd_wgrad(const DeformDesc& d, const G4DDeformGrads& grads, int64_t n, uint8_t* images, int sm_count,
                                cudaStream_t st);

// ---- launchers (defined in g4d_geom.cu / g4d_raster.cu / g4d_geom_bwd.cu / g4d_backward.cu) -------------
// d_time: the camera's timestamp from device memory (NULL: cam.time)
cudaError_t launch_pack_camera(const G4DCamera& cam, const float* d_time, CameraDev* dst, cudaStream_t st);
cudaError_t launch_pack_weights(const G4DDeformParams& p, float* w0t, float* const* w1t, float* const* wtt, cudaStream_t st);
cudaError_t launch_collapse_time_rows(const G4DDeformParams& p, TimeArg time, float* const (*trow)[3], cudaStream_t st);
cudaError_t launch_preprocess(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g, int32_t* out_radii,
                              cudaStream_t st);
// The HexPlane gather of a forward: feat [N][F] fp32 receives the features, Gaussians visited in `order` (NULL: index order).
struct DeformGather {
    float* feat;
    const uint32_t* order;
};
// The gather (launch_deform_features, dependent on the time-row collapse before it), then the network: mode 0: deform only
// (writes the five out_* tensors; cam unused); mode 1: fused deform + preprocess (camera from cam).  tw: the network runs on
// the tensor cores with these weight images and buffers, else on the FFMA kernel (an ordinary launch).
cudaError_t launch_deform(const DeformDesc& d, int mode, const CameraDev* cam, int64_t n, const DeformIO& io, const DeformGather& gather,
                          int sm_count, cudaStream_t st, const TcWeights* tw = nullptr);

// The per-Gaussian gradients of one blend backward in one float buffer, as blocks of N floats: d(mean2D) [2N] from block
// kMean2D, d(conic) [3N] from kConic, d(rgb) [3N] from kRgb, d(opacity) [N] from kOpacity; kFloats blocks in all.  A
// backward with a depth gradient adds the block d(view-space depth) [N] at kDepth: kDepthFloats blocks in all.
struct BlendGradLayout {
    static constexpr int kMean2D = 0, kConic = 2, kRgb = 5, kOpacity = 8, kFloats = 9, kDepth = 9, kDepthFloats = 10;
};

cudaError_t launch_blend_forward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                 float* out_color, float* out_depth, int warp_cull, float* out_alpha, cudaStream_t st);
// dL_ddepth != NULL: the depth image's gradient [H,W] is added too, and dL/d(view-space depth) of every Gaussian is added
// into g_depth [N] (zeroed by the caller).  dL_dalpha != NULL: the alpha image's gradient [H,W] is added too.  dL_dcolor
// may be NULL (a zero colour gradient) when either is set.
cudaError_t launch_blend_backward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                  const float* dL_dcolor, float* g_mean2D, float* g_conic, float* g_opacity, float* g_rgb,
                                  int warp_cull, const float* dL_ddepth, float* g_depth, const float* dL_dalpha,
                                  cudaStream_t st);
// per-Gaussian backward; g_cam != NULL: the camera's gradient (view[16], proj[16], campos[3]) is also added into g_cam,
// which the caller zeroes first; g_depth != NULL: dL/d(view-space depth) [N] of the blend backward, carried to the mean
// (and to the view matrix's depth row)
cudaError_t launch_preprocess_backward(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                       const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                       float* g_means2D_out, float* g_scales, float* g_rotations, const ShOut& g_sh,
                                       float* g_cam, const float* g_depth, cudaStream_t st);

// Backward of the deformation network (g4d_backward.cu): the HexPlane gather (skipped when saved_feat holds the features
// the forward gathered; order: its walk order), an engine -- the tensor-core kernels with the images tc, or the FFMA kernels
// (tc NULL) -- the scatter and the time-row gradients.  go[h] / gi[h]: gradient w.r.t. the outputs / inputs of head h's
// residual tensor (xyz, scaling, rotation, opacity, shs).  relu_bits: the signs a tensor-core forward saved, or NULL.
// d.times set (per-row times; `time` unused): no time rows, and dL/d(times) into g_times [N] when it is not NULL.
// d.times NULL: dL/d(time) is added into g_time [1] (zeroed by the caller) when it is not NULL.
size_t deform_backward_scratch_bytes(const DeformDesc& d, int64_t n, bool tc);   // size of launch_deform_backward's scratch
cudaError_t launch_deform_backward(const DeformDesc& d, const G4DDeformParams& prm, const G4DDeformGrads& grads, const TcBwdWeights* tc,
                                   TimeArg time, int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                                   float* const gi[G4D_NUM_HEADS], float* g_times, float* g_time, const uint32_t* relu_bits,
                                   const float* saved_feat, const uint32_t* order, void* scratch, int sm_count, cudaStream_t st);
// ---- several cameras at one timestamp (g4d_render_forward_cameras / _backward_cameras) -----------------------------
constexpr int kMaxExtraCameras = G4D_MAX_CAMERAS - 1;
// cameras 1..k-1 of a multi-camera forward: camera c reads cam[c] and writes its own context's records g[c] and out_radii[c]
struct ExtraCameras {
    int count;
    const CameraDev* cam[kMaxExtraCameras];
    GeomBuffers g[kMaxExtraCameras];
    int32_t* out_radii[kMaxExtraCameras];
};
// one thread per Gaussian: the deformed, activated tensors `in` (camera 0's FusedOutputs) are read once and projected into
// every extra camera (g4d_geom.cu; launched dependent on its predecessor, DESIGN.md §4.6)
cudaError_t launch_project_cameras(const ExtraCameras& ec, int64_t n, const RasterInputs& in, cudaStream_t st);

// cameras of a multi-camera backward that are part of the loss
struct BackwardCameras {
    int count;
    const CameraDev* cam[G4D_MAX_CAMERAS];
    const int32_t* radii[G4D_MAX_CAMERAS];
    const uint8_t* clamped[G4D_MAX_CAMERAS];
    const float* grad[G4D_MAX_CAMERAS];    // the camera's blend backward, BlendGradLayout (with the depth block when the call has one)
    float* g_means2D[G4D_MAX_CAMERAS];     // [N,3] screen-space gradient of the camera, or NULL
};
// the camera-gradient accumulators of those cameras (out[j]: camera j of BackwardCameras, kCamGradFloats floats, zeroed
// before the launch)
struct CamGradSinks {
    float* out[G4D_MAX_CAMERAS];
};
// per-Gaussian backward of all those cameras in one pass: the gradients w.r.t. means3D, scales, rotations, opacity and the
// SH coefficients are summed over the cameras and written once (OVERWRITTEN); cs != NULL: each camera's gradient is also
// added into its sink; depth: every camera's grad[] has the depth block (zeros for a camera without a depth gradient)
cudaError_t launch_preprocess_backward_cameras(const BackwardCameras& bc, int64_t n, const RasterInputs& in, float* g_means3D,
                                               float* g_scales, float* g_rotations, float* g_opacities, const ShOut& g_sh,
                                               const CamGradSinks* cs, bool depth, cudaStream_t st);

// coarse stage of render(): the fused forward's tail without the deformation network (io as for launch_deform mode 1)
cudaError_t launch_activate_preprocess(const CameraDev* cam, int64_t n, const DeformIO& io, cudaStream_t st);
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
// the per-step scalars launch_adam_flat runs with (g4d_adam_scalars)
void adam_scalars(const G4DAdamSegment* segs, int nseg, float b1, float b2, int64_t step, float grad_scale, G4DAdamScalars* out);
// launch_adam_flat with the scalars read from device memory at run time (the segments' lr fields are not read)
cudaError_t launch_adam_flat_device(float* p, const float* g, float* m, float* v, int64_t numel, const G4DAdamSegment* segs, int nseg,
                                    float b1, float b2, float eps, const G4DAdamScalars* d_scalars, int sm_count, cudaStream_t st);

// ---- 3-nearest-neighbour mean squared distance (g4d_knn.cu) ---------------------------------------------------------
size_t knn_scratch_bytes(int64_t n);   // size of launch_knn_dist2's scratch
cudaError_t launch_knn_dist2(int64_t n, const float* xyz, float* out, void* scratch, int sm_count, cudaStream_t st);


}  // namespace g4d
