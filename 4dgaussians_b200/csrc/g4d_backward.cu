// g4d_backward.cu -- per-Gaussian backward of the projection stage (A.4) and backward of the deformation
// network (HexPlane scatter + MLP dgrad/wgrad).
// Reference autograd path replaced: loss.backward() at /root/reference/train.py:219 through
// _RasterizeGaussians.backward, F.normalize/exp/sigmoid, nn.Linear, F.grid_sample.
#include "g4d_internal.h"
#include "g4d_math.cuh"

namespace g4d {

__global__ void __launch_bounds__(256)
preprocess_backward_kernel(const CameraDev* __restrict__ camp, int64_t n, RasterInputs in, GeomBuffers g,
                           const float* __restrict__ g_mean2D, const float* __restrict__ g_conic,
                           const float* __restrict__ g_rgb, float* __restrict__ g_means3D, float* __restrict__ g_means2D_out,
                           float* __restrict__ g_scales, float* __restrict__ g_rotations, ShOut g_sh) {
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
    in.sh.stage_warp(g0, cnt, lane, ld);
    __syncwarp();
    auto sh_store = [&](int k, int ch, float v) { st[lane * kShRow + 3 * k + ch] = v; };
    if (active) {
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
            gaussian_backward(cam, p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, (uint32_t)g.clamped[gi], gm2, gc, gr,
                              [&](int k, int ch) { return row[3 * k + ch]; }, sh_store, gg);
            for (int k = 0; k < 3; ++k) { g_means3D[3 * gi + k] = gg.mean[k]; g_scales[3 * gi + k] = gg.scale[k]; }
            for (int k = 0; k < 4; ++k) g_rotations[4 * gi + k] = gg.rot[k];
        }
    }
    __syncwarp();
    g_sh.store_warp(g0, cnt, lane, st);
}

cudaError_t launch_preprocess_backward(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                       const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                       float* g_means2D_out, float* g_scales, float* g_rotations, const ShOut& g_sh,
                                       cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    constexpr int kThreads = 128;
    const size_t smem = (size_t)(kThreads / 32) * 2 * 32 * kShRow * sizeof(float);   // 50 KB: SH staging (see the kernel)
    {
        cudaError_t e = cudaFuncSetAttribute(preprocess_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    preprocess_backward_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, smem, st>>>(cam, n, in, g, g_mean2D, g_conic, g_rgb,
                                                                                                  g_means3D, g_means2D_out, g_scales,
                                                                                                  g_rotations, g_sh);
    return cudaGetLastError();
}

// Per-Gaussian backward of several cameras at one timestamp (g4d_render_backward_cameras): the deformed state and the SH
// coefficients are loaded once, gaussian_backward runs for every camera that sees the Gaussian, and the sums -- mean,
// scale and rotation in registers, SH in the warp's shared-memory rows, opacity from the cameras' blend backward passes --
// are written once.  Each camera's screen-space gradient goes to its own sink.
__global__ void __launch_bounds__(128)
preprocess_backward_cameras_kernel(BackwardCameras bc, int64_t n, RasterInputs in, float* __restrict__ g_means3D,
                                   float* __restrict__ g_scales, float* __restrict__ g_rotations, float* __restrict__ g_opacities,
                                   ShOut g_sh) {
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
    in.sh.stage_warp(g0, cnt, lane, ld);
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
            if (!vis) continue;
            const float gm2[2] = {gmb[2 * gi], gmb[2 * gi + 1]};
            const float gc[3] = {gcb[3 * gi], gcb[3 * gi + 1], gcb[3 * gi + 2]};
            const float grgb[3] = {grb[3 * gi], grb[3 * gi + 1], grb[3 * gi + 2]};
            GaussGrad gg;
            gaussian_backward(cams[c], p, sc, Quat{q4.x, q4.y, q4.z, q4.w}, (uint32_t)bc.clamped[c][gi], gm2, gc, grgb,
                              [&](int k, int ch) { return row[3 * k + ch]; },
                              [&](int k, int ch, float v) { srow[3 * k + ch] += v; }, gg);
            for (int k = 0; k < 3; ++k) { gm[k] += gg.mean[k]; gs[k] += gg.scale[k]; }
            for (int k = 0; k < 4; ++k) gr[k] += gg.rot[k];
        }
        for (int k = 0; k < 3; ++k) { g_means3D[3 * gi + k] = gm[k]; g_scales[3 * gi + k] = gs[k]; }
        for (int k = 0; k < 4; ++k) g_rotations[4 * gi + k] = gr[k];
        g_opacities[gi] = gop;
    }
    __syncwarp();
    g_sh.store_warp(g0, cnt, lane, st);
}

cudaError_t launch_preprocess_backward_cameras(const BackwardCameras& bc, int64_t n, const RasterInputs& in, float* g_means3D,
                                               float* g_scales, float* g_rotations, float* g_opacities, const ShOut& g_sh,
                                               cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    constexpr int kThreads = 128;
    const size_t smem = (size_t)(kThreads / 32) * 2 * 32 * kShRow * sizeof(float);   // 50 KB: SH staging and sums
    cudaError_t e = cudaFuncSetAttribute(preprocess_backward_cameras_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    preprocess_backward_cameras_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, smem, st>>>(
        bc, n, in, g_means3D, g_scales, g_rotations, g_opacities, g_sh);
    return cudaGetLastError();
}

// ======================================================================================================
// Backward of the deformation network.
//
// Three persistent kernels (DESIGN.md §4):
//   P  "prepass":  re-sample the HexPlane features and recompute a1 = relu(feat W0^T + b0) for every Gaussian
//                  -> FEAT [N][F], A1 [N][Wd] in HBM.
//   H  "heads":    CTA c owns ONE head (c mod #active) for its whole life: W1 (torch layout, padded) and W2 stay in
//                  shared memory, dW1 / dW2 / db accumulate in REGISTERS across all the CTA's tiles and are flushed
//                  once with atomics; per tile it recomputes z, a2, forms dz and writes da1_h = dz W1 -> DA1[h] in HBM.
//   Q  "final":    dh = (sum_h DA1[h]) * (a1 > 0); dW0, db0 in registers; dfeat = dh W0; scatter-add into the planes
//                  (vector RED; time planes through the collapsed rows), d(xyz) through the bilinear coordinates,
//                  residual-path input gradients.
//   T  distributes the collapsed time-row gradients onto the two time rows of each time plane.
// ======================================================================================================

struct DeformBwdBuffers {
    float* feat;                      // [N][F]
    float* a1;                        // [N][WD]
    float* da1[G4D_NUM_HEADS];        // [N][WD] per active head
    float* trow_grad[G4D_MAX_LEVELS][3];
};

struct DeformBwdDesc {
    DeformDesc d;
    const float* w0;                  // torch layout [WD][F]
    const float* w1[G4D_NUM_HEADS];   // torch layout [WD][WD]
    float* g_w0; float* g_b0;
    float* g_w1[G4D_NUM_HEADS]; float* g_b1[G4D_NUM_HEADS];
    float* g_w2[G4D_NUM_HEADS]; float* g_b2[G4D_NUM_HEADS];
    float* g_planes[G4D_MAX_LEVELS][6];
    const float* go[G4D_NUM_HEADS];   // dL/d(out) per head: xyz[N,3], scaling[N,3], rotation[N,4], opacity[N,1], shs[N,48] (NULL = 0)
    float* gi[G4D_NUM_HEADS];         // dL/d(in), same shapes (NULL = not wanted)
};

// acc[r][c] += sum_k A[ty*RM + r][k] * Bt[tx + 16*c][k]       (both operands K-contiguous in shared memory)
template <int RM, int CN>
G4D_D void tile_gemm_nt(const float* __restrict__ A, int lda, const float* __restrict__ Bt, int ldb, int K, int ty, int tx,
                        float (&acc)[RM][CN]) {
    const float* arow = A + ty * RM * lda;
    const float* brow = Bt + tx * ldb;
#pragma unroll 1
    for (int k = 0; k < K; k += 4) {
        float4 a[RM], b[CN];
#pragma unroll
        for (int r = 0; r < RM; ++r) a[r] = *reinterpret_cast<const float4*>(arow + r * lda + k);
#pragma unroll
        for (int c = 0; c < CN; ++c) b[c] = *reinterpret_cast<const float4*>(brow + 16 * c * ldb + k);
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < CN; ++c) {
                float s = acc[r][c];
                s = fmaf(a[r].x, b[c].x, s); s = fmaf(a[r].y, b[c].y, s);
                s = fmaf(a[r].z, b[c].z, s); s = fmaf(a[r].w, b[c].w, s);
                acc[r][c] = s;
            }
    }
}

// ---- kernel P ------------------------------------------------------------------------------------------
template <int TG, int WD>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_prepass_kernel(DeformDesc d, DeformSmem L, int64_t n, const float* __restrict__ xyz,
                          float* __restrict__ feat_out, float* __restrict__ a1_out) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RM = TG / 16, CG = WD / 64;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int64_t ntiles = (n + TG - 1) / TG;
    const int n0 = d.F * WD;
    for (int i = tid * 4; i < n0; i += kDeformThreads * 4)
        *reinterpret_cast<float4*>(smem + L.w0t + i) = __ldg(reinterpret_cast<const float4*>(d.w0t + i));
    for (int i = tid; i < WD; i += kDeformThreads) smem[L.b0 + i] = __ldg(d.b0 + i);
    const AabbNorm nrm(d.aabb);
    float* coord = smem + L.coord;
    __syncthreads();
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG, rem = n - base;
        if (tid < TG) {
            float4 c = make_float4(0.f, 0.f, 0.f, 0.f);   // (w unused: time enters through the collapsed time rows)
            if (tid < rem) {
                c.x = nrm(0, xyz[(base + tid) * 3 + 0]);
                c.y = nrm(1, xyz[(base + tid) * 3 + 1]);
                c.z = nrm(2, xyz[(base + tid) * 3 + 2]);
            }
            *reinterpret_cast<float4*>(coord + 4 * tid) = c;
        }
        __syncthreads();
        sample_features<TG>(d, coord, smem + L.a0, L.lda0);
        __syncthreads();
        for (int i = tid; i < TG * (d.F >> 2); i += kDeformThreads) {
            const int g = i / (d.F >> 2), v = i - g * (d.F >> 2);
            if (g < rem)
                *reinterpret_cast<float4*>(feat_out + (base + g) * d.F + 4 * v) = *reinterpret_cast<const float4*>(smem + L.a0 + g * L.lda0 + 4 * v);
        }
        float acc[RM][CG * 4];
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
        tile_gemm<RM, CG>(smem + L.a0, L.lda0, smem + L.w0t, WD, d.F, ty, tx, acc);
#pragma unroll
        for (int c = 0; c < CG; ++c) {
            const float4 bv = *reinterpret_cast<const float4*>(smem + L.b0 + c * 64 + tx * 4);
#pragma unroll
            for (int r = 0; r < RM; ++r) {
                const int g = ty * RM + r;
                if (g < rem) {
                    float4 v = make_float4(fmaxf(acc[r][c * 4 + 0] + bv.x, 0.f), fmaxf(acc[r][c * 4 + 1] + bv.y, 0.f),
                                           fmaxf(acc[r][c * 4 + 2] + bv.z, 0.f), fmaxf(acc[r][c * 4 + 3] + bv.w, 0.f));
                    *reinterpret_cast<float4*>(a1_out + (base + g) * WD + c * 64 + tx * 4) = v;
                }
            }
        }
        __syncthreads();
    }
}

// ---- kernel H ------------------------------------------------------------------------------------------
struct HeadSmem { int w1, w2, b1, a1, a2, dz, dout, total_floats, ldw, lda, ldo; };

inline HeadSmem head_smem_layout(int TG, int WD) {
    HeadSmem s{};
    int off = 0;
    auto take = [&](int n) { int o = off; off += (n + 3) & ~3; return o; };
    s.ldw = WD + 4; s.lda = WD + 4; s.ldo = 48;
    s.w1 = take(WD * s.ldw);
    s.w2 = take(48 * s.ldw);
    s.b1 = take(WD);
    s.a1 = take(TG * s.lda);
    s.a2 = take(TG * s.lda);
    s.dz = take(TG * s.lda);
    s.dout = take(TG * s.ldo);
    s.total_floats = off;
    return s;
}

template <int TG, int WD>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_heads_kernel(DeformBwdDesc bd, HeadSmem L, int64_t n, int num_active, DeformBwdBuffers buf) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RM = TG / 16, CG = WD / 64, CN = WD / 16, JR = WD / 16;
    constexpr int NG = kDeformThreads / WD;           // thread groups for the dW2 mapping (2 or 4)
    constexpr int MAXO = 48 / NG;                     // dW2 accumulators per thread (24 or 12)
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    // which head does this CTA own?
    int slot = blockIdx.x % num_active, h = -1;
    for (int hh = 0, s = 0; hh < G4D_NUM_HEADS; ++hh)
        if (bd.d.head_mask & (1 << hh)) { if (s == slot) h = hh; ++s; }
    const int cta_in_head = blockIdx.x / num_active;
    const int ctas_for_head = (gridDim.x - slot + num_active - 1) / num_active;
    const int kout = head_out(h), kp = (kout + 3) & ~3;
    const int64_t ntiles = (n + TG - 1) / TG;
    float* sW1 = smem + L.w1; float* sW2 = smem + L.w2; float* sB1 = smem + L.b1;
    float* sA1 = smem + L.a1; float* sA2 = smem + L.a2; float* sDZ = smem + L.dz; float* sDO = smem + L.dout;
    // persistent weights: W1 [j][i] and W2 [o][j] in torch layout, rows padded to ldw
    for (int i = tid; i < WD * (WD >> 2); i += kDeformThreads) {
        const int r = i / (WD >> 2), v = i - r * (WD >> 2);
        *reinterpret_cast<float4*>(sW1 + r * L.ldw + 4 * v) = __ldg(reinterpret_cast<const float4*>(bd.w1[h] + r * WD + 4 * v));
    }
    for (int i = tid; i < 48 * (WD >> 2); i += kDeformThreads) {
        const int r = i / (WD >> 2), v = i - r * (WD >> 2);
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < kout) val = __ldg(reinterpret_cast<const float4*>(bd.d.w2[h] + r * WD + 4 * v));
        *reinterpret_cast<float4*>(sW2 + r * L.ldw + 4 * v) = val;
    }
    for (int i = tid; i < WD; i += kDeformThreads) sB1[i] = __ldg(bd.d.b1[h] + i);
    // register accumulators that live across all tiles of this CTA
    float gW1[JR][CG * 4];
#pragma unroll
    for (int a = 0; a < JR; ++a)
#pragma unroll
        for (int b = 0; b < CG * 4; ++b) gW1[a][b] = 0.f;
    float gW2[MAXO];
#pragma unroll
    for (int a = 0; a < MAXO; ++a) gW2[a] = 0.f;
    float gB1 = 0.f, gB2 = 0.f;
    const int w2_j = tid % WD, w2_g = tid / WD;
    const float* go = bd.go[h];
    const int go_stride = kout;   // [N][kout] contiguous for every head (shs: 48)
    __syncthreads();

    for (int64_t tile = cta_in_head; tile < ntiles; tile += ctas_for_head) {
        const int64_t base = tile * TG, rem = n - base;
        for (int i = tid; i < TG * (WD >> 2); i += kDeformThreads) {
            const int g = i / (WD >> 2), v = i - g * (WD >> 2);
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g < rem) val = *reinterpret_cast<const float4*>(buf.a1 + (base + g) * WD + 4 * v);
            *reinterpret_cast<float4*>(sA1 + g * L.lda + 4 * v) = val;
        }
        for (int i = tid; i < TG * kp; i += kDeformThreads) {
            const int g = i / kp, o = i - g * kp;
            sDO[g * L.ldo + o] = (go && g < rem && o < kout) ? go[(base + g) * go_stride + o] : 0.f;
        }
        __syncthreads();
        {   // z = a1 W1^T + b1 ; a2 = relu(z)
            float acc[RM][CN];
#pragma unroll
            for (int r = 0; r < RM; ++r)
#pragma unroll
                for (int c = 0; c < CN; ++c) acc[r][c] = 0.f;
            tile_gemm_nt<RM, CN>(sA1, L.lda, sW1, L.ldw, WD, ty, tx, acc);
#pragma unroll
            for (int r = 0; r < RM; ++r)
#pragma unroll
                for (int c = 0; c < CN; ++c) sA2[(ty * RM + r) * L.lda + tx + 16 * c] = fmaxf(acc[r][c] + sB1[tx + 16 * c], 0.f);
        }
        __syncthreads();
        {   // da2 = dout W2 ; dz = da2 * (a2 > 0)
            float acc[RM][CG * 4];
#pragma unroll
            for (int r = 0; r < RM; ++r)
#pragma unroll
                for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
            tile_gemm<RM, CG>(sDO, L.ldo, sW2, L.ldw, kp, ty, tx, acc);
#pragma unroll
            for (int c = 0; c < CG; ++c)
#pragma unroll
                for (int r = 0; r < RM; ++r) {
                    const int g = ty * RM + r, col = c * 64 + tx * 4;
                    const float4 a2 = *reinterpret_cast<const float4*>(sA2 + g * L.lda + col);
                    float4 v = make_float4(a2.x > 0.f ? acc[r][c * 4 + 0] : 0.f, a2.y > 0.f ? acc[r][c * 4 + 1] : 0.f,
                                           a2.z > 0.f ? acc[r][c * 4 + 2] : 0.f, a2.w > 0.f ? acc[r][c * 4 + 3] : 0.f);
                    *reinterpret_cast<float4*>(sDZ + g * L.lda + col) = v;
                }
        }
        __syncthreads();
        // dW2[o][j] += sum_g dout[g][o] a2[g][j];  thread owns column j = w2_j and rows o = w2_g + NG*m
        for (int g = 0; g < TG; ++g) {
            const float a2 = sA2[g * L.lda + w2_j];
#pragma unroll
            for (int m = 0; m < MAXO; ++m) {
                const int o = w2_g + NG * m;
                if (o < kp) gW2[m] = fmaf(sDO[g * L.ldo + o], a2, gW2[m]);
            }
        }
        if (tid < WD) {
            float s = 0.f;
            for (int g = 0; g < TG; ++g) s += sDZ[g * L.lda + tid];
            gB1 += s;
        } else if (tid - WD < kout && tid >= WD) {
            float s = 0.f;
            for (int g = 0; g < TG; ++g) s += sDO[g * L.ldo + (tid - WD)];
            gB2 += s;
        }
        {   // dW1[j][i] += sum_g dz[g][j] a1[g][i];  thread (ty, tx): j = ty*JR + a, i = c*64 + tx*4 + b
            for (int g = 0; g < TG; ++g) {
                float dzv[JR];
#pragma unroll
                for (int a = 0; a < JR; a += 4) {
                    const float4 t4 = *reinterpret_cast<const float4*>(sDZ + g * L.lda + ty * JR + a);
                    dzv[a] = t4.x; dzv[a + 1] = t4.y; dzv[a + 2] = t4.z; dzv[a + 3] = t4.w;
                }
                float4 av[CG];
#pragma unroll
                for (int c = 0; c < CG; ++c) av[c] = *reinterpret_cast<const float4*>(sA1 + g * L.lda + c * 64 + tx * 4);
#pragma unroll
                for (int a = 0; a < JR; ++a)
#pragma unroll
                    for (int c = 0; c < CG; ++c) {
                        gW1[a][c * 4 + 0] = fmaf(dzv[a], av[c].x, gW1[a][c * 4 + 0]);
                        gW1[a][c * 4 + 1] = fmaf(dzv[a], av[c].y, gW1[a][c * 4 + 1]);
                        gW1[a][c * 4 + 2] = fmaf(dzv[a], av[c].z, gW1[a][c * 4 + 2]);
                        gW1[a][c * 4 + 3] = fmaf(dzv[a], av[c].w, gW1[a][c * 4 + 3]);
                    }
            }
        }
        {   // da1_h = dz W1  -> HBM
            float acc[RM][CG * 4];
#pragma unroll
            for (int r = 0; r < RM; ++r)
#pragma unroll
                for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
            tile_gemm<RM, CG>(sDZ, L.lda, sW1, L.ldw, WD, ty, tx, acc);
#pragma unroll
            for (int c = 0; c < CG; ++c)
#pragma unroll
                for (int r = 0; r < RM; ++r) {
                    const int g = ty * RM + r;
                    if (g < rem)
                        *reinterpret_cast<float4*>(buf.da1[h] + (base + g) * WD + c * 64 + tx * 4) =
                            make_float4(acc[r][c * 4 + 0], acc[r][c * 4 + 1], acc[r][c * 4 + 2], acc[r][c * 4 + 3]);
                }
        }
        __syncthreads();
    }
    // flush the register accumulators (one atomic per element per CTA)
#pragma unroll
    for (int a = 0; a < JR; ++a)
#pragma unroll
        for (int c = 0; c < CG; ++c)
#pragma unroll
            for (int b = 0; b < 4; ++b) atomicAdd(bd.g_w1[h] + (ty * JR + a) * WD + c * 64 + tx * 4 + b, gW1[a][c * 4 + b]);
#pragma unroll
    for (int m = 0; m < MAXO; ++m) {
        const int o = w2_g + NG * m;
        if (o < kout) atomicAdd(bd.g_w2[h] + o * WD + w2_j, gW2[m]);
    }
    if (tid < WD) atomicAdd(bd.g_b1[h] + tid, gB1);
    else if (tid - WD < kout) atomicAdd(bd.g_b2[h] + (tid - WD), gB2);
}

// ---- kernel Q ------------------------------------------------------------------------------------------
struct FinalSmem { int w0, feat, dh, df, coord, total_floats, ldw0, ldf, ldh; };

inline FinalSmem final_smem_layout(int TG, int F, int WD) {
    FinalSmem s{};
    int off = 0;
    auto take = [&](int n) { int o = off; off += (n + 3) & ~3; return o; };
    s.ldw0 = F + 4; s.ldf = F + 4; s.ldh = WD + 4;
    s.w0 = take(WD * s.ldw0);
    s.feat = take(TG * s.ldf);
    s.dh = take(TG * s.ldh);
    s.df = take(TG * s.ldf);
    s.coord = take(TG * 4);
    s.total_floats = off;
    return s;
}

template <int TG, int WD, int FM>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_final_kernel(DeformBwdDesc bd, FinalSmem L, int64_t n, const float* __restrict__ xyz,
                        DeformBwdBuffers buf) {
    extern __shared__ __align__(16) float smem[];
    const DeformDesc& d = bd.d;
    const int tid = threadIdx.x;
    const int F = d.F, F4 = F >> 2, C4 = d.C >> 2;
    constexpr int NG = kDeformThreads / WD;
    constexpr int MAXF = FM / NG;                   // dW0 accumulators per thread (F <= FM)
    float* sW0 = smem + L.w0; float* sF = smem + L.feat; float* sDH = smem + L.dh; float* sDF = smem + L.df;
    float* coord = smem + L.coord;
    for (int i = tid; i < WD * F4; i += kDeformThreads) {
        const int r = i / F4, v = i - r * F4;
        *reinterpret_cast<float4*>(sW0 + r * L.ldw0 + 4 * v) = __ldg(reinterpret_cast<const float4*>(bd.w0 + r * F + 4 * v));
    }
    float gW0[MAXF];
#pragma unroll
    for (int m = 0; m < MAXF; ++m) gW0[m] = 0.f;
    float gB0 = 0.f;
    const int w0_j = tid % WD, w0_g = tid / WD;
    const AabbNorm nrm(d.aabb);
    const int64_t ntiles = (n + TG - 1) / TG;
    constexpr int TPG = kDeformThreads / TG;
    __syncthreads();

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG, rem = n - base;
        for (int i = tid; i < TG * F4; i += kDeformThreads) {
            const int g = i / F4, v = i - g * F4;
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g < rem) val = *reinterpret_cast<const float4*>(buf.feat + (base + g) * F + 4 * v);
            *reinterpret_cast<float4*>(sF + g * L.ldf + 4 * v) = val;
        }
        for (int i = tid; i < TG * (WD >> 2); i += kDeformThreads) {
            const int g = i / (WD >> 2), v = i - g * (WD >> 2);
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g < rem) {
                for (int h = 0; h < G4D_NUM_HEADS; ++h) {
                    if (!(d.head_mask & (1 << h))) continue;
                    const float4 t = *reinterpret_cast<const float4*>(buf.da1[h] + (base + g) * WD + 4 * v);
                    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                }
                const float4 a1 = *reinterpret_cast<const float4*>(buf.a1 + (base + g) * WD + 4 * v);
                s.x = a1.x > 0.f ? s.x : 0.f; s.y = a1.y > 0.f ? s.y : 0.f;
                s.z = a1.z > 0.f ? s.z : 0.f; s.w = a1.w > 0.f ? s.w : 0.f;
            }
            *reinterpret_cast<float4*>(sDH + g * L.ldh + 4 * v) = s;
        }
        if (tid < TG) {
            float4 c = make_float4(0.f, 0.f, 0.f, 0.f);   // (w unused: time enters through the collapsed time rows)
            if (tid < rem) {
                c.x = nrm(0, xyz[(base + tid) * 3 + 0]);
                c.y = nrm(1, xyz[(base + tid) * 3 + 1]);
                c.z = nrm(2, xyz[(base + tid) * 3 + 2]);
            }
            *reinterpret_cast<float4*>(coord + 4 * tid) = c;
        }
        __syncthreads();
        // dW0[j][f] += sum_g dh[g][j] feat[g][f];  thread owns row j = w0_j and columns f = w0_g + NG*m
        for (int g = 0; g < TG; ++g) {
            const float dh = sDH[g * L.ldh + w0_j];
#pragma unroll
            for (int m = 0; m < MAXF; ++m) {
                const int f = w0_g + NG * m;
                if (f < F) gW0[m] = fmaf(dh, sF[g * L.ldf + f], gW0[m]);
            }
        }
        if (tid < WD) {
            float s = 0.f;
            for (int g = 0; g < TG; ++g) s += sDH[g * L.ldh + tid];
            gB0 += s;
        }
        // dfeat[g][f..f+3] = sum_j dh[g][j] W0[j][f..f+3]
        for (int i = tid; i < TG * F4; i += kDeformThreads) {
            const int g = i / F4, v = i - g * F4;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int j = 0; j < WD; ++j) {
                const float dh = sDH[g * L.ldh + j];
                const float4 w = *reinterpret_cast<const float4*>(sW0 + j * L.ldw0 + 4 * v);
                acc.x = fmaf(dh, w.x, acc.x); acc.y = fmaf(dh, w.y, acc.y); acc.z = fmaf(dh, w.z, acc.z); acc.w = fmaf(dh, w.w, acc.w);
            }
            *reinterpret_cast<float4*>(sDF + g * L.ldf + 4 * v) = acc;
        }
        __syncthreads();
        // scatter into the planes and d(xyz): thread (g, q) handles channel vectors v = q, q+TPG, ...
        {
            const int g = tid / TPG, q = tid % TPG;
            const float4 pc = *reinterpret_cast<const float4*>(coord + 4 * g);
            const float pcs[3] = {pc.x, pc.y, pc.z};
            float gpix[3] = {0.f, 0.f, 0.f};   // dL/d(normalised coordinate) per axis
            if (g < rem) {
                for (int l = 0; l < d.levels; ++l) {
                    Tap1D tx[3];
#pragma unroll
                    for (int a = 0; a < 3; ++a) tx[a] = make_tap(pcs[a], d.res[l][a]);
                    for (int v = q; v < C4; v += TPG) {
                        const float4 df = *reinterpret_cast<const float4*>(sDF + g * L.ldf + l * d.C + 4 * v);
                        scatter_vector(d.planes[l], d.trow[l], d.res[l], bd.g_planes[l], buf.trow_grad[l], tx, v, C4, df, gpix);
                    }
                }
            }
            // reduce the TPG partial coordinate gradients of one Gaussian (adjacent lanes)
#pragma unroll
            for (int a = 0; a < 3; ++a)
                for (int o = 1; o < TPG; o <<= 1) gpix[a] += __shfl_xor_sync(0xffffffffu, gpix[a], o);
            if (q == 0 && g < rem && bd.gi[0]) {
                const int64_t gi = base + g;
#pragma unroll
                for (int a = 0; a < 3; ++a)
                    bd.gi[0][gi * 3 + a] = (bd.go[0] ? bd.go[0][gi * 3 + a] : 0.f) + gpix[a] * nrm.scale[a];
            }
        }
        // residual path of the other inputs: d(out)/d(in) = identity
        for (int hh = 1; hh < G4D_NUM_HEADS; ++hh) {
            if (!bd.gi[hh]) continue;
            const int ko = head_out(hh);
            for (int i = tid; i < TG * ko; i += kDeformThreads)
                if (i < rem * ko) bd.gi[hh][base * ko + i] = bd.go[hh] ? bd.go[hh][base * ko + i] : 0.f;
        }
        __syncthreads();
    }
#pragma unroll
    for (int m = 0; m < MAXF; ++m) {
        const int f = w0_g + NG * m;
        if (f < F) atomicAdd(bd.g_w0 + w0_j * F + f, gW0[m]);
    }
    if (tid < WD) atomicAdd(bd.g_b0 + tid, gB0);
}

// ---- kernel T: collapsed time-row gradients -> the two time rows of each (axis, t) plane --------------------
struct TimeGradDesc {
    int levels, C;
    int res[G4D_MAX_LEVELS][4];
    const float* row_grad[G4D_MAX_LEVELS][3];
    float* plane_grad[G4D_MAX_LEVELS][3];
    int start[G4D_MAX_LEVELS * 3 + 1];
};

__global__ void distribute_time_grad_kernel(TimeGradDesc d, TimeArg time) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nseg = d.levels * 3;
    if (i >= d.start[nseg]) return;
    int m = 0;
    while (i >= d.start[m + 1]) ++m;
    const int l = m / 3, a = m % 3, e = i - d.start[m];
    const Tap1D ty = make_tap(time.get(), d.res[l][3]);
    const int rowlen = d.res[l][a] * d.C;
    const float gv = d.row_grad[l][a][e];
    atomicAdd(d.plane_grad[l][a] + (size_t)ty.i0 * rowlen + e, gv * ty.w0);
    atomicAdd(d.plane_grad[l][a] + (size_t)ty.i1 * rowlen + e, gv * ty.w1);
}

// ---- host side -------------------------------------------------------------------------------------------
cudaError_t launch_distribute_time_grad(const DeformDesc& d, float* const (*trow_grad)[3], float* const (*g_planes)[6], TimeArg time,
                                        cudaStream_t st) {
    TimeGradDesc t{};
    t.levels = d.levels; t.C = d.C;
    const TimeRows tr(d.levels, d.res, d.C);
    const int tk[3] = {2, 4, 5};
    for (int l = 0; l < d.levels; ++l) {
        for (int a = 0; a < 4; ++a) t.res[l][a] = d.res[l][a];
        for (int a = 0; a < 3; ++a) { t.row_grad[l][a] = trow_grad[l][a]; t.plane_grad[l][a] = g_planes[l][tk[a]]; }
    }
    for (int m = 0; m <= 3 * d.levels; ++m) t.start[m] = tr.start[m];
    const int total = (int)tr.total();
    distribute_time_grad_kernel<<<(total + 255) / 256, 256, 0, st>>>(t, time);
    return cudaGetLastError();
}

// the scratch of the FFMA backward: FEAT [N][F], A1 [N][WD], DA1 of every active head [N][WD], the time-row gradients;
// returns the number of active heads
static int carve_backward_scratch(Carve& m, const DeformDesc& d, const TimeRows& tr, int64_t n, DeformBwdBuffers& buf) {
    const size_t N = (size_t)(n > 0 ? n : 1);
    buf.feat = m.take<float>(N * d.F);
    buf.a1 = m.take<float>(N * d.WD);
    int active = 0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h)
        if (d.head_mask & (1 << h)) { buf.da1[h] = m.take<float>(N * d.WD); ++active; }
    float* rows = m.take<float>(tr.total());
    if (rows) tr.place(rows, buf.trow_grad);
    return active;
}

size_t deform_backward_scratch_bytes(const DeformDesc& d, int64_t n) {
    Carve m;
    DeformBwdBuffers buf{};
    carve_backward_scratch(m, d, TimeRows(d.levels, d.res, d.C), n, buf);
    return m.bytes();
}

template <int TG, int WD>
static cudaError_t launch_deform_backward_t(const DeformBwdDesc& bd, TimeArg time, int64_t n, const float* xyz, float* scratch,
                                            int sm_count, cudaStream_t st) {
    const DeformDesc& d = bd.d;
    DeformBwdBuffers buf{};
    const TimeRows tr(d.levels, d.res, d.C);
    Carve m(scratch);
    const int active = carve_backward_scratch(m, d, tr, n, buf);
    cudaError_t e = cudaMemsetAsync(buf.trow_grad[0][0], 0, tr.total() * sizeof(float), st);
    if (e != cudaSuccess) return e;
    const int64_t ntiles = (n + TG - 1) / TG;
    // P
    {
        const DeformSmem L = deform_smem_layout(TG, d.F, WD, 0);
        const size_t bytes = (size_t)L.total_floats * 4;
        e = cudaFuncSetAttribute(deform_bwd_prepass_kernel<TG, WD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return e;
        const int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
        deform_bwd_prepass_kernel<TG, WD><<<grid, kDeformThreads, bytes, st>>>(d, L, n, xyz, buf.feat, buf.a1);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    // H
    if (active > 0) {
        const HeadSmem L = head_smem_layout(TG, WD);
        const size_t bytes = (size_t)L.total_floats * 4;
        e = cudaFuncSetAttribute(deform_bwd_heads_kernel<TG, WD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return e;
        int grid = sm_count;
        if ((int64_t)grid > ntiles * active) grid = (int)(ntiles * active);
        if (grid < active) grid = active;
        deform_bwd_heads_kernel<TG, WD><<<grid, kDeformThreads, bytes, st>>>(bd, L, n, active, buf);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    // Q
    {
        const FinalSmem L = final_smem_layout(TG, d.F, WD);
        const size_t bytes = (size_t)L.total_floats * 4;
        const int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
#define G4D_LAUNCH_Q(FM)                                                                                                  \
        do {                                                                                                              \
            e = cudaFuncSetAttribute(deform_bwd_final_kernel<TG, WD, FM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes); \
            if (e != cudaSuccess) return e;                                                                               \
            deform_bwd_final_kernel<TG, WD, FM><<<grid, kDeformThreads, bytes, st>>>(bd, L, n, xyz, buf);            \
        } while (0)
        if (d.F <= 32) G4D_LAUNCH_Q(32);
        else if (d.F <= 64) G4D_LAUNCH_Q(64);
        else G4D_LAUNCH_Q(128);
#undef G4D_LAUNCH_Q
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    // T
    if ((e = launch_distribute_time_grad(d, buf.trow_grad, bd.g_planes, time, st)) != cudaSuccess) return e;
    return cudaSuccess;
}

cudaError_t launch_deform_backward(const DeformDesc& d, const G4DDeformParams& prm, const G4DDeformGrads& grads, TimeArg time,
                                   int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                                   float* const gi[G4D_NUM_HEADS], float* scratch, int sm_count, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    DeformBwdDesc bd{};
    bd.d = d;
    bd.w0 = prm.w0; bd.g_w0 = grads.w0; bd.g_b0 = grads.b0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        bd.w1[h] = prm.w1[h]; bd.g_w1[h] = grads.w1[h]; bd.g_b1[h] = grads.b1[h]; bd.g_w2[h] = grads.w2[h]; bd.g_b2[h] = grads.b2[h];
        bd.go[h] = go[h]; bd.gi[h] = gi[h];
    }
    for (int l = 0; l < d.levels; ++l)
        for (int k = 0; k < 6; ++k) bd.g_planes[l][k] = grads.planes[l][k];
    if (d.WD == 128) return launch_deform_backward_t<64, 128>(bd, time, n, xyz, scratch, sm_count, st);
    if (d.WD == 64) return launch_deform_backward_t<128, 64>(bd, time, n, xyz, scratch, sm_count, st);
    return cudaErrorInvalidValue;
}

// ------------------------------------------------------------------------------------------------------
// Chain rule through exp / F.normalize / sigmoid, in place: on entry the buffers hold gradients w.r.t. the
// activated tensors, on exit w.r.t. the pre-activation tensors.
__global__ void __launch_bounds__(256)
activation_backward_kernel(int64_t n, FusedOutputs fo, float* __restrict__ g_scales, float* __restrict__ g_rotations,
                           float* __restrict__ g_opacities) {
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= n) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) g_scales[3 * gi + k] *= fo.scales[3 * gi + k];
    const float4 y = *reinterpret_cast<const float4*>(fo.rotations + 4 * gi);
    float4 g = *reinterpret_cast<const float4*>(g_rotations + 4 * gi);
    const float dot = y.x * g.x + y.y * g.y + y.z * g.z + y.w * g.w;
    const float inv = 1.f / fo.rot_norm[gi];
    g.x = (g.x - y.x * dot) * inv; g.y = (g.y - y.y * dot) * inv; g.z = (g.z - y.z * dot) * inv; g.w = (g.w - y.w * dot) * inv;
    *reinterpret_cast<float4*>(g_rotations + 4 * gi) = g;
    const float op = fo.opacities[gi];
    g_opacities[gi] *= op * (1.f - op);
}

cudaError_t launch_activation_backward(int64_t n, const FusedOutputs& fo, float* g_scales, float* g_rotations,
                                       float* g_opacities, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    activation_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, fo, g_scales, g_rotations, g_opacities);
    return cudaGetLastError();
}

}  // namespace g4d
