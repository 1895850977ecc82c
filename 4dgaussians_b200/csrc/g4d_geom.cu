// g4d_geom.cu -- per-Gaussian forward stages: parameter packing, time-row collapse, deformation network,
// activations and projection ("preprocess"), standalone and fused.
//
// COMPILED WITH -fmad=false: the projection expression trees must round exactly like SURVEY.md Appendix A.1
// evaluated in plain fp32 (depth bits, radii and tile rects are index data and are tested bit-exactly);
// every place where fusion is wanted (MLP, bilinear taps) calls fmaf() explicitly.
//
// Reference path replaced: /root/reference/gaussian_renderer/__init__.py:52 (time tensor), :87-89 (deform),
// :97-99 (activations) and the preprocess stage inside the rasterizer called at :120.
#include "geom_finish.cuh"

namespace g4d {

// ------------------------------------------------------------------------------------------------------
__global__ void pack_camera_kernel(G4DCamera c, const float* d_time, CameraDev* dst) {
    pdl_trigger();      // (ordinary launch: everything before it in the stream has completed)
    const int t = threadIdx.x;
    if (t < 16) {
        dst->view[t] = c.d_viewmatrix ? c.d_viewmatrix[t] : c.viewmatrix[t];
        dst->proj[t] = c.d_projmatrix ? c.d_projmatrix[t] : c.projmatrix[t];
    }
    if (t < 4) {
        dst->campos[t] = t < 3 ? (c.d_campos ? c.d_campos[t] : c.campos[t]) : 0.f;
        dst->bg[t] = t < 3 ? (c.d_bg ? c.d_bg[t] : c.bg[t]) : 0.f;
    }
    if (t == 0) {
        dst->H = c.image_height; dst->W = c.image_width; dst->sh_degree = c.sh_degree;
        dst->grid_x = (c.image_width + kTile - 1) / kTile;
        dst->grid_y = (c.image_height + kTile - 1) / kTile;
        dst->num_tiles = dst->grid_x * dst->grid_y;
        dst->depth_min = 0xFFFFFFFFu; dst->depth_max = 0u;
        dst->tanfovx = c.tanfovx; dst->tanfovy = c.tanfovy; dst->scale_modifier = c.scale_modifier;
        dst->time = d_time ? *d_time : c.time;
        dst->focal_x = (float)c.image_width / (2.f * c.tanfovx);
        dst->focal_y = (float)c.image_height / (2.f * c.tanfovy);
        dst->grid_bar = 0u; dst->pad3 = 0u;
    }
}

cudaError_t launch_pack_camera(const G4DCamera& cam, const float* d_time, CameraDev* dst, cudaStream_t st) {
    return launch_k(pack_camera_kernel, 1, 32, 0, st, kOrdinary, cam, d_time, dst);
}

// ------------------------------------------------------------------------------------------------------
constexpr int kPackMax = 1 + G4D_NUM_HEADS + G4D_MAX_DEPTH - 1;   // W0, the heads' W1, the trunk's W_j
struct PackDesc {
    const float* src[kPackMax];
    float* dst[kPackMax];
    int rows[kPackMax];            // src is [rows][cols] (torch [out][in]); dst is [cols][rows]
    int cols[kPackMax];
    int start[kPackMax + 1];       // prefix sums of element counts
    int count;
};

__global__ void pack_weights_kernel(PackDesc p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.start[p.count]) return;
    int m = 0;
    while (i >= p.start[m + 1]) ++m;
    const int e = i - p.start[m];
    const int r = e % p.rows[m], c = e / p.rows[m];   // dst index e = c*rows + r
    p.dst[m][e] = __ldg(p.src[m] + r * p.cols[m] + c);
}

cudaError_t launch_pack_weights(const G4DDeformParams& prm, float* w0t, float* const* w1t, float* const* wtt, cudaStream_t st) {
    PackDesc p{};
    const int F = prm.levels * prm.channels, WD = prm.net_width;
    int m = 0, total = 0;
    p.src[m] = prm.w0; p.dst[m] = w0t; p.rows[m] = WD; p.cols[m] = F; p.start[m] = total; total += WD * F; ++m;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(prm.head_mask & (1 << h))) continue;
        p.src[m] = prm.w1[h]; p.dst[m] = w1t[h]; p.rows[m] = WD; p.cols[m] = WD; p.start[m] = total; total += WD * WD; ++m;
    }
    for (int j = 1; j < prm.depth; ++j) {
        p.src[m] = prm.wt[j - 1]; p.dst[m] = wtt[j - 1]; p.rows[m] = WD; p.cols[m] = WD; p.start[m] = total; total += WD * WD; ++m;
    }
    p.start[m] = total; p.count = m;
    return launch_k(pack_weights_kernel, (total + 255) / 256, 256, 0, st, kOrdinary, p);
}

// ------------------------------------------------------------------------------------------------------
// Every Gaussian of a view shares t, so the time-axis interpolation of the three time planes is done once:
// row[x][c] = plane[y0][x][c]*(y1-y) + plane[y1][x][c]*(y-y0)  with t NOT normalised (hexplane.py:164).
// s.src: the time planes [T][res[a]][C]; s.dst: the rows [res[a]][C].
__global__ void collapse_time_rows_kernel(TimeRowSegs s, TimeArg time) {
    pdl_wait();         // the row buffer is reused: the previous view's kernels read it until they complete
    pdl_trigger();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.start[3 * s.levels]) return;
    int l, a, e;
    s.locate(i, l, a, e);
    const int T = s.res[l][3];
    const Tap1D ty = make_tap(time.get(), T);   // (after pdl_wait: a source written by the previous kernel is complete)
    const int rowlen = s.res[l][a] * s.C;
    const float v0 = __ldg(s.src[l][a] + (size_t)ty.i0 * rowlen + e), v1 = __ldg(s.src[l][a] + (size_t)ty.i1 * rowlen + e);
    s.dst[l][a][e] = fmaf(v1, ty.w1, v0 * ty.w0);
}

cudaError_t launch_collapse_time_rows(const G4DDeformParams& p, TimeArg time, float* const (*trow)[3], cudaStream_t st) {
    TimeRowSegs s(p.levels, p.res, p.channels);
    for (int l = 0; l < p.levels; ++l)
        for (int a = 0; a < 3; ++a) { s.src[l][a] = p.planes[l][kTimePlane[a]]; s.dst[l][a] = trow[l][a]; }
    const int total = (int)s.total();
    return launch_k(collapse_time_rows_kernel, dim3((total + 255) / 256), dim3(256), 0, st, kPdl, s, time);
}

// ------------------------------------------------------------------------------------------------------
// Standalone preprocess: one thread per Gaussian, inputs are post-activation (A.1).  FULL: M = 16 (ShIn).
template <bool FULL>
__global__ void __launch_bounds__(256) preprocess_kernel(const CameraDev* __restrict__ camp, int64_t n, RasterInputs in,
                                                         GeomBuffers g, int32_t* out_radii) {
    __shared__ CameraDev cam;
    stage_cameras(&cam, &camp, 1);
    __syncthreads();
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n) return;
    const Vec3 p{in.means3D[3 * gi], in.means3D[3 * gi + 1], in.means3D[3 * gi + 2]};
    const Vec3 sc{in.scales[3 * gi], in.scales[3 * gi + 1], in.scales[3 * gi + 2]};
    const float4 q4 = *reinterpret_cast<const float4*>(in.rotations + 4 * gi);
    Projected pr;
    const bool ok = project_gaussian(cam, p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, pr);
    float rgb[3] = {0.f, 0.f, 0.f};
    uint32_t bits = 0;
    if (ok) in.sh.with_coeffs<FULL>(gi, [&](auto sh) { sh_to_rgb(cam, p, sh, rgb, bits); });
    store_projected(g, gi, ok, pr, in.opacities[gi], rgb, bits, out_radii);
}

cudaError_t launch_preprocess(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g, int32_t* out_radii,
                              cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    return launch_k(in.sh.m == kShCoeffs ? preprocess_kernel<true> : preprocess_kernel<false>, blocks, 256, 0, st, kOrdinary, cam, n,
                    in, g, out_radii);
}

// ------------------------------------------------------------------------------------------------------
// Extra cameras of a multi-camera forward (g4d_render_forward_cameras): one thread per Gaussian reads the deformed,
// activated state camera 0's fused forward stored (44 B, plus 192 B of SH staged per warp through shared memory) ONCE and
// projects it into every other camera with the fused kernels' projection and colour code: the inputs are the very floats
// those kernels held in registers, so each camera's records equal its own render()'s bit for bit.
template <bool FULL>
__global__ void __launch_bounds__(256) project_cameras_kernel(ExtraCameras ec, int64_t n, RasterInputs in) {
    extern __shared__ float sh_smem[];             // [warps][32 * kShRow]
    __shared__ CameraDev cams[kMaxExtraCameras];
    pdl_wait();         // the cameras (pack_camera) and camera 0's stored tensors
    pdl_trigger();
    stage_cameras(cams, ec.cam, ec.count);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* ld = sh_smem + (size_t)warp * 32 * kShRow;
    const int64_t g0 = (int64_t)blockIdx.x * blockDim.x + warp * 32;
    const int cnt = (int)(n - g0 < 32 ? (n - g0 > 0 ? n - g0 : 0) : 32);
    if (cnt == 0) return;                          // whole warp
    in.sh.stage_warp<FULL>(g0, cnt, lane, ld);
    __syncwarp();
    if (lane >= cnt) return;
    const int64_t gi = g0 + lane;
    const Vec3 p{in.means3D[3 * gi], in.means3D[3 * gi + 1], in.means3D[3 * gi + 2]};
    const Vec3 sc{in.scales[3 * gi], in.scales[3 * gi + 1], in.scales[3 * gi + 2]};
    const float4 q4 = *reinterpret_cast<const float4*>(in.rotations + 4 * gi);
    const float op = in.opacities[gi];
    const float* row = ld + lane * kShRow;
    for (int c = 0; c < ec.count; ++c) {
        const CameraDev& cam = cams[c];
        Projected pr;
        const bool ok = project_gaussian(cam, p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, pr);
        float rgb[3] = {0.f, 0.f, 0.f};
        uint32_t bits = 0;
        if (ok) sh_to_rgb(cam, p, [&](int k, int ch) { return row[3 * k + ch]; }, rgb, bits);
        store_projected(ec.g[c], gi, ok, pr, op, rgb, bits, ec.out_radii[c]);
    }
}

cudaError_t launch_project_cameras(const ExtraCameras& ec, int64_t n, const RasterInputs& in, cudaStream_t st) {
    if (n == 0 || ec.count == 0) return cudaSuccess;
    constexpr int kThreads = 256;
    const size_t smem = (size_t)(kThreads / 32) * 32 * kShRow * sizeof(float);   // 49 KB: SH staging
    auto kernel = in.sh.m == kShCoeffs ? project_cameras_kernel<true> : project_cameras_kernel<false>;
    return launch_k(kernel, dim3((unsigned)((n + kThreads - 1) / kThreads)), dim3(kThreads), smem, st, kPdl, ec, n, in);
}

// ------------------------------------------------------------------------------------------------------
// Persistent kernel: one CTA per SM, each looping over tiles of TG Gaussians whose HexPlane features feat [N][F] the gather
// wrote (an ordinary launch: the gather has completed).
//   MODE 0: deformation network only (drop-in for deform_network.forward; outputs pre-activation tensors)
//   MODE 1: fused deformation + activations + projection (the render() hot path), M = 16 SH coefficients per Gaussian
//   MODE 2: MODE 1 for models with M = io.sh.m < 16 (no SHS head)
template <int TG, int WD, int MODE>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_kernel(DeformDesc d, DeformSmem L, const CameraDev* __restrict__ camp, int64_t n, const float* __restrict__ feat, DeformIO io) {
    extern __shared__ __align__(16) float smem[];
    __shared__ CameraDev cam;
    const int tid = threadIdx.x;
    const int64_t ntiles = (n + TG - 1) / TG;
    if (MODE != 0) stage_cameras(&cam, &camp, 1);
    stage_persistent_weights(d, L, smem);
    void* bar = smem + L.mbar;
    if (tid == 0) { mbar_init(bar, 1); fence_barrier_init(); }
    __syncthreads();
    if (tid == 0 && wslot_images(d) > 0 && (int64_t)blockIdx.x < ntiles) wslot_issue<WD>(d, L, smem, 0);   // deform_mlp_tile's PRE
    uint32_t phase = 0;
    float* in_xyz = smem + L.in;
    float* in_sc = in_xyz + TG * 3;
    float* in_rot = in_sc + TG * 3;
    float* in_op = in_rot + TG * 4;
    float* out = smem + L.out;
    const bool hp = d.head_mask & G4D_HEAD_POS, hs = d.head_mask & G4D_HEAD_SCALES, hr = d.head_mask & G4D_HEAD_ROT,
               ho = d.head_mask & G4D_HEAD_OPACITY, hsh = d.head_mask & G4D_HEAD_SHS;

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG;
        const int64_t rem = n - base;   // > 0
        for (int i = tid; i < TG * 3; i += kDeformThreads) {
            const bool v = i < rem * 3;
            in_xyz[i] = v ? io.xyz[base * 3 + i] : 0.f;
            in_sc[i] = (v && io.scaling) ? io.scaling[base * 3 + i] : 0.f;
        }
        for (int i = tid; i < TG * 4; i += kDeformThreads) in_rot[i] = (i < rem * 4 && io.rotation) ? io.rotation[base * 4 + i] : 0.f;
        for (int i = tid; i < TG; i += kDeformThreads) in_op[i] = (i < rem && io.opacity) ? io.opacity[base + i] : 0.f;
        load_feature_tile<TG>(feat, d.F, base, rem, smem + L.a0, L.lda0);
        __syncthreads();
        deform_mlp_tile<TG, WD>(d, L, smem, phase, tile + gridDim.x < ntiles);

        if (MODE == 0) {
            for (int i = tid; i < TG * 3; i += kDeformThreads) {
                if (i < rem * 3) {
                    const int g = i / 3, c = i - 3 * g;
                    io.out_xyz[base * 3 + i] = in_xyz[i] + (hp ? out[g * 60 + 0 + c] : 0.f);
                    if (io.out_scaling) io.out_scaling[base * 3 + i] = in_sc[i] + (hs ? out[g * 60 + 3 + c] : 0.f);
                }
            }
            if (io.out_rotation)
                for (int i = tid; i < TG * 4; i += kDeformThreads)
                    if (i < rem * 4) io.out_rotation[base * 4 + i] = in_rot[i] + (hr ? out[(i >> 2) * 60 + 6 + (i & 3)] : 0.f);
            if (io.out_opacity)
                for (int i = tid; i < TG; i += kDeformThreads)
                    if (i < rem) io.out_opacity[base + i] = in_op[i] + (ho ? out[i * 60 + 10] : 0.f);
            if (io.out_shs && hsh)
                for (int i = tid; i < TG * 48; i += kDeformThreads)
                    if (i < rem * 48) {
                        const int g = i / 48, c = i - 48 * g;
                        io.out_shs[base * 48 + i] = io.sh.shs[base * 48 + i] + out[g * 60 + 11 + c];
                    }
        } else {
            if (hsh && io.fo.shs) {   // deformed SH coefficients are needed again by the backward pass
                for (int i = tid; i < TG * 48; i += kDeformThreads)
                    if (i < rem * 48) {
                        const int g = i / 48, c = i - 48 * g;
                        io.fo.shs[base * 48 + i] = io.sh.at<true>(base + g, c) + out[g * 60 + 11 + c];   // (SHS head: M = 16)
                    }
            }
            if (tid < TG && tid < rem) {
                const int g = tid;
                const int64_t gi = base + g;
                const float* o = out + g * 60;
                Vec3 p{in_xyz[3 * g], in_xyz[3 * g + 1], in_xyz[3 * g + 2]};
                float sl[3] = {in_sc[3 * g], in_sc[3 * g + 1], in_sc[3 * g + 2]};
                float q[4] = {in_rot[4 * g], in_rot[4 * g + 1], in_rot[4 * g + 2], in_rot[4 * g + 3]};
                float ol = in_op[g];
                if (hp) { p.x += o[0]; p.y += o[1]; p.z += o[2]; }
                if (hs) { sl[0] += o[3]; sl[1] += o[4]; sl[2] += o[5]; }
                if (hr) { q[0] += o[6]; q[1] += o[7]; q[2] += o[8]; q[3] += o[9]; }
                if (ho) ol += o[10];
                const float* dsh = o + 11;
                fused_finish<MODE == 1>(cam, io, gi, p, sl, q, ol, [&](int i) { return hsh ? dsh[i] : 0.f; });
            }
        }
        __syncthreads();
    }
}

cudaError_t launch_deform_tc(const DeformDesc& d, const TcWeights& tw, int mode, const CameraDev* cam, int64_t n,
                             const DeformIO& io, int sm_count, cudaStream_t st);

template <int TG, int WD, int MODE>
static cudaError_t launch_deform_t(const DeformDesc& d, const DeformSmem& L, size_t bytes, const CameraDev* cam, int64_t n,
                                   const float* feat, const DeformIO& io, int sm_count, cudaStream_t st) {
    const int64_t ntiles = (n + TG - 1) / TG;
    const int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
    return launch_k(deform_kernel<TG, WD, MODE>, grid, kDeformThreads, bytes, st, kOrdinary, d, L, cam, n, feat, io);
}

// The FFMA network runs tiles of TG Gaussians when their shared memory (dynamic and static) fits in an SM, and of TG / 2
// otherwise: wide features with the SH head, or those plus the trunk biases, at net_width 128 (every configuration the C-ABI
// takes fits at TG / 2).  tile_gemm's sums run over K in the same order whatever the tile, so both tiles give the same bits.
template <int TG, int WD, int MODE>
static cudaError_t launch_deform_tiles(const DeformDesc& d, const CameraDev* cam, int64_t n, const float* feat, const DeformIO& io,
                                       int sm_count, cudaStream_t st) {
    constexpr size_t kMaxSmem = 227 * 1024;
    const DeformSmem L = deform_smem_layout(TG, d.F, WD, d.head_mask, d.ntrunk);
    const size_t bytes = (size_t)L.total_floats * sizeof(float);
    cudaFuncAttributes a{};
    cudaError_t e = cudaFuncGetAttributes(&a, deform_kernel<TG, WD, MODE>);
    if (e != cudaSuccess) return e;
    if (bytes + a.sharedSizeBytes <= kMaxSmem) return launch_deform_t<TG, WD, MODE>(d, L, bytes, cam, n, feat, io, sm_count, st);
    const DeformSmem H = deform_smem_layout(TG / 2, d.F, WD, d.head_mask, d.ntrunk);
    const size_t hbytes = (size_t)H.total_floats * sizeof(float);
    if ((e = cudaFuncGetAttributes(&a, deform_kernel<TG / 2, WD, MODE>)) != cudaSuccess) return e;
    if (hbytes + a.sharedSizeBytes > kMaxSmem) return cudaErrorInvalidConfiguration;
    return launch_deform_t<TG / 2, WD, MODE>(d, H, hbytes, cam, n, feat, io, sm_count, st);
}

cudaError_t launch_deform(const DeformDesc& d, int mode, const CameraDev* cam, int64_t n, const DeformIO& io, const DeformGather& gather,
                          int sm_count, cudaStream_t st, const TcWeights* tw) {
    if (n == 0) return cudaSuccess;
    // the HexPlane gather of every path, dependent on the time-row collapse before it (DESIGN.md §4.6)
    cudaError_t e = launch_deform_features(d, n, io.xyz, gather.order, gather.feat, true, st);
    if (e != cudaSuccess) return e;
    if (tw) {
        TcWeights t = *tw;
        t.feat = gather.feat; t.order = gather.order;
        return launch_deform_tc(d, t, mode, cam, n, io, sm_count, st);
    }
    const bool full = io.sh.m == kShCoeffs;
    if (d.WD == 128) {
        return mode == 0 ? launch_deform_tiles<64, 128, 0>(d, cam, n, gather.feat, io, sm_count, st)
             : full      ? launch_deform_tiles<64, 128, 1>(d, cam, n, gather.feat, io, sm_count, st)
                         : launch_deform_tiles<64, 128, 2>(d, cam, n, gather.feat, io, sm_count, st);
    } else if (d.WD == 64) {
        return mode == 0 ? launch_deform_tiles<128, 64, 0>(d, cam, n, gather.feat, io, sm_count, st)
             : full      ? launch_deform_tiles<128, 64, 1>(d, cam, n, gather.feat, io, sm_count, st)
                         : launch_deform_tiles<128, 64, 2>(d, cam, n, gather.feat, io, sm_count, st);
    }
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------------
// "coarse" stage of render() (gaussian_renderer/__init__.py:80-81): the fused tail with no network deltas.  FULL: M = 16.
template <bool FULL>
__global__ void __launch_bounds__(256) activate_preprocess_kernel(const CameraDev* __restrict__ camp, int64_t n, DeformIO io) {
    __shared__ CameraDev cam;
    stage_cameras(&cam, &camp, 1);
    __syncthreads();
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n) return;
    const Vec3 p{io.xyz[3 * gi], io.xyz[3 * gi + 1], io.xyz[3 * gi + 2]};
    const float sl[3] = {io.scaling[3 * gi], io.scaling[3 * gi + 1], io.scaling[3 * gi + 2]};
    const float4 q4 = *reinterpret_cast<const float4*>(io.rotation + 4 * gi);
    const float q[4] = {q4.x, q4.y, q4.z, q4.w};
    // a delta of -0.f leaves every coefficient as it is (x + -0 == x, also for x = +0), so the add compiles away
    fused_finish<FULL>(cam, io, gi, p, sl, q, io.opacity[gi], [](int) { return -0.f; });
}

cudaError_t launch_activate_preprocess(const CameraDev* cam, int64_t n, const DeformIO& io, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    return launch_k(io.sh.m == kShCoeffs ? activate_preprocess_kernel<true> : activate_preprocess_kernel<false>, blocks, 256, 0, st,
                    kOrdinary, cam, n, io);
}

}  // namespace g4d
