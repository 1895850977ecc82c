// g4d_backward.cu -- per-Gaussian backward of the projection stage (A.4; kernels in per_gaussian_bwd.cuh, the instances with a
// depth gradient in g4d_backward_depth.cu) and the backward of the deformation network: the
// frame every backward runs (HexPlane gather, scatter, time-row distribution) around the FFMA engine here or the tensor-core
// engine of g4d_deform_tc_bwd.cu.  Compiled with the default FMA contraction: the coordinate normalisation of the scatter
// rounds explicitly, as the forward's gather does (hexplane.cuh).
// Reference autograd path replaced: loss.backward() at /root/reference/train.py:219 through
// _RasterizeGaussians.backward, F.normalize/exp/sigmoid, nn.Linear, F.grid_sample.
#include "g4d_internal.h"
#include "g4d_math.cuh"
#include "per_gaussian_bwd.cuh"

namespace g4d {

cudaError_t launch_preprocess_backward(const CameraDev* cam, int64_t n, const RasterInputs& in, GeomBuffers g,
                                       const float* g_mean2D, const float* g_conic, const float* g_rgb, float* g_means3D,
                                       float* g_means2D_out, float* g_scales, float* g_rotations, const ShOut& g_sh,
                                       float* g_cam, const float* g_depth, cudaStream_t st) {
    if (g_depth)
        return launch_preprocess_backward_depth(cam, n, in, g, g_mean2D, g_conic, g_rgb, g_means3D, g_means2D_out, g_scales,
                                                g_rotations, g_sh, g_cam, g_depth, st);
    return launch_per_gaussian_backward(preprocess_backward_kernel<false, false, false>, preprocess_backward_kernel<false, true, false>,
                                        preprocess_backward_kernel<true, false, false>, preprocess_backward_kernel<true, true, false>,
                                        g_sh.m == kShCoeffs, g_cam != nullptr, n, st, cam, n, in, g, g_mean2D, g_conic, g_rgb,
                                        g_means3D, g_means2D_out, g_scales, g_rotations, g_sh, g_cam, g_depth);
}

cudaError_t launch_preprocess_backward_cameras(const BackwardCameras& bc, int64_t n, const RasterInputs& in, float* g_means3D,
                                               float* g_scales, float* g_rotations, float* g_opacities, const ShOut& g_sh,
                                               const CamGradSinks* cs, bool depth, cudaStream_t st) {
    if (depth) return launch_preprocess_backward_cameras_depth(bc, n, in, g_means3D, g_scales, g_rotations, g_opacities, g_sh, cs, st);
    return launch_per_gaussian_backward(
        preprocess_backward_cameras_kernel<false, false, false>, preprocess_backward_cameras_kernel<false, true, false>,
        preprocess_backward_cameras_kernel<true, false, false>, preprocess_backward_cameras_kernel<true, true, false>,
        g_sh.m == kShCoeffs, cs != nullptr, n, st, bc, n, in, g_means3D, g_scales, g_rotations, g_opacities, g_sh,
        cs ? *cs : CamGradSinks{});
}

// ======================================================================================================
// Backward of the deformation network (DESIGN.md §4): one frame (launch_deform_backward) around one of two engines.
//
//   gather:   the forward's HexPlane gather, deform_features_kernel -> FEAT [N][F] (skipped when the forward kept its features)
//   engine:   d(feat) -> DFEAT [N][F] and the network's weight gradients, either
//             FFMA, persistent kernels:
//               P  "prepass":  a_0 = relu(feat W0^T + b0) for every Gaussian -> A[0] [N][Wd] in HBM; with a trunk
//                              (defor_depth D >= 2) launched once more per trunk layer j = 1 .. D-1: a_j = relu(a_{j-1} W_j^T
//                              + b_j) -> A[j], with the forward's tile_gemm order (the ReLU signs are recomputed, so only the
//                              forward's arithmetic makes the gradient the gradient of the forward that ran).  A1 = A[D-1].
//               H  "heads":    CTA c owns ONE head (c mod #active) for its whole life: W1 (torch layout, padded) and W2 stay in
//                              shared memory, dW1 / dW2 / db accumulate in REGISTERS across all the CTA's tiles and are
//                              flushed once with atomics; per tile it recomputes z, a2, forms dz and writes da1_h = dz W1
//                              -> DA1[h] in HBM.
//               T  "trunk":    D >= 2 only, once per trunk layer j = D-1 .. 1: dz_j = dA_j * (a_j > 0) with dA_{D-1} =
//                              sum_h DA1[h]; dW_j, db_j in registers; dA_{j-1} = dz_j W_j -> a ping-pong pair of [N][Wd].
//               Q  "final":    dh = dA_0 * (a_0 > 0), dA_0 = sum_h DA1[h] when D <= 1; dW0, db0 in registers;
//                              dfeat = dh W0 -> DFEAT.
//             or tensor-core, kernels A (dgrad, -> DFEAT) and B (wgrad), g4d_deform_tc_bwd.cu, with the scatter between them.
//   scatter:  bwd_scatter_kernel: DFEAT into the planes (vector RED; time planes through the collapsed rows), d(xyz) through
//             the bilinear coordinates, residual-path input gradients.
//   T         distributes the collapsed time-row gradients onto the two time rows of each time plane.
// ======================================================================================================

// The scratch of a backward: the engine's own -- the FFMA kernels' activations and DA1 of every active head (and with a trunk
// its dA ping-pong pair), or the tensor-core kernels' operand images -- then the features and their gradient and the time-row
// gradients (both engines).
struct DeformBwdBuffers {
    const float* feat;                // [N][F]: the gather's, or the features the forward kept
    float* a1;                        // FFMA: [N][WD] relu(h_{D-1}), the heads' input (= act[ntrunk])
    float* act[G4D_MAX_DEPTH];        // FFMA: [N][WD] a_j = relu(h_j), j = 0 .. ntrunk
    float* da1[G4D_NUM_HEADS];        // FFMA: [N][WD] per active head
    float* dact[2];                   // FFMA with a trunk: [N][WD] dA_j ping-pong
    float* dfeat;                     // [N][F]
    float* trow_grad[G4D_MAX_LEVELS][3];
    uint8_t* images;                  // tensor-core: tc_bwd_images_bytes
};

// Everything one backward's kernels read and write besides their plain arguments, built once by launch_deform_backward: the
// FFMA kernels read the network's, the scatter the planes' and the residual paths'.
struct DeformBwdArgs {
    DeformDesc d;
    G4DDeformGrads g;                     // the caller's gradient sinks (accumulated into)
    const float* w0;                      // torch layout [WD][F]
    const float* w1[G4D_NUM_HEADS];       // torch layout [WD][WD]
    const float* wt[G4D_MAX_DEPTH - 1];   // trunk, torch layout [WD][WD]
    const float* go[G4D_NUM_HEADS];   // dL/d(out) per head: xyz[N,3], scaling[N,3], rotation[N,4], opacity[N,1], shs[N,48] (NULL = 0)
    float* gi[G4D_NUM_HEADS];         // dL/d(in), same shapes (NULL = not wanted)
    float* g_times;                   // [N] dL/d(times) of the per-row mode (OVERWRITTEN), or NULL
    DeformBwdBuffers buf;
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

// ---- building blocks of the FFMA engine's H, T and Q ----------------------------------------------------
// dst[r][0 .. K) = src[r][0 .. K) for the WD rows of a torch-layout [WD][K] matrix, rows padded to ld floats in dst
template <int WD>
G4D_D void stage_rows(float* dst, int ld, const float* src, int K) {
    const int K4 = K >> 2;
    for (int i = threadIdx.x; i < WD * K4; i += kDeformThreads) {
        const int r = i / K4, v = i - r * K4;
        *reinterpret_cast<float4*>(dst + r * ld + 4 * v) = __ldg(reinterpret_cast<const float4*>(src + r * K + 4 * v));
    }
}

// The register tile of a [WD][WD] weight gradient dW that thread (ty, tx) accumulates over all its CTA's tiles:
// acc[a][c * 4 + b] = dW[ty * JR + a][c * 64 + tx * 4 + b], JR = WD / 16, c < WD / 64
template <int WD> using WGradTile = float[WD / 16][WD / 16];

template <int WD>
G4D_D void wgrad_zero(WGradTile<WD>& acc) {
#pragma unroll
    for (int a = 0; a < WD / 16; ++a)
#pragma unroll
        for (int b = 0; b < WD / 16; ++b) acc[a][b] = 0.f;
}

// dW[o][i] += sum_g dz[g][o] a[g][i] over the TG rows of a tile: dz and a [TG][WD] in shared memory, rows ld floats apart
template <int TG, int WD>
G4D_D void wgrad_accumulate(WGradTile<WD>& acc, const float* dz, const float* a, int ld, int ty, int tx) {
    constexpr int CG = WD / 64, JR = WD / 16;
    for (int g = 0; g < TG; ++g) {
        float dzv[JR];
#pragma unroll
        for (int j = 0; j < JR; j += 4) {
            const float4 t4 = *reinterpret_cast<const float4*>(dz + g * ld + ty * JR + j);
            dzv[j] = t4.x; dzv[j + 1] = t4.y; dzv[j + 2] = t4.z; dzv[j + 3] = t4.w;
        }
        float4 av[CG];
#pragma unroll
        for (int c = 0; c < CG; ++c) av[c] = *reinterpret_cast<const float4*>(a + g * ld + c * 64 + tx * 4);
#pragma unroll
        for (int j = 0; j < JR; ++j)
#pragma unroll
            for (int c = 0; c < CG; ++c) {
                acc[j][c * 4 + 0] = fmaf(dzv[j], av[c].x, acc[j][c * 4 + 0]);
                acc[j][c * 4 + 1] = fmaf(dzv[j], av[c].y, acc[j][c * 4 + 1]);
                acc[j][c * 4 + 2] = fmaf(dzv[j], av[c].z, acc[j][c * 4 + 2]);
                acc[j][c * 4 + 3] = fmaf(dzv[j], av[c].w, acc[j][c * 4 + 3]);
            }
    }
}

// adds the tile into the sink g [WD][WD]: one atomic per element per CTA
template <int WD>
G4D_D void wgrad_flush(const WGradTile<WD>& acc, float* const& g, int ty, int tx) {
    constexpr int CG = WD / 64, JR = WD / 16;
#pragma unroll
    for (int a = 0; a < JR; ++a)
#pragma unroll
        for (int c = 0; c < CG; ++c)
#pragma unroll
            for (int b = 0; b < 4; ++b) atomicAdd(g + (ty * JR + a) * WD + c * 64 + tx * 4 + b, acc[a][c * 4 + b]);
}

// out[base + g][0 .. WD) = (dz W)[g] for the tile's rows g < rem: dz [TG][WD] (rows ldz floats apart) and W [WD][WD] (torch
// layout, rows ldw floats apart) in shared memory.  (out, a float pointer, by reference: the kernel argument is read where it is
// stored to, not held in registers across the GEMM.)
template <int TG, int WD, class P>
G4D_D void store_dz_w(const float* dz, int ldz, const float* W, int ldw, const P& out,
                      int64_t base, int64_t rem, int ty, int tx) {
    constexpr int RM = TG / 16, CG = WD / 64;
    float acc[RM][CG * 4];
#pragma unroll
    for (int r = 0; r < RM; ++r)
#pragma unroll
        for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
    tile_gemm<RM, CG>(dz, ldz, W, ldw, WD, ty, tx, acc);
#pragma unroll
    for (int c = 0; c < CG; ++c)
#pragma unroll
        for (int r = 0; r < RM; ++r) {
            const int g = ty * RM + r;
            if (g < rem)
                *reinterpret_cast<float4*>(out + (base + g) * WD + c * 64 + tx * 4) =
                    make_float4(acc[r][c * 4 + 0], acc[r][c * 4 + 1], acc[r][c * 4 + 2], acc[r][c * 4 + 3]);
        }
}

// sum over the TG rows of a tile of column col: a bias gradient's share of the tile
template <int TG>
G4D_D float column_sum(const float* t, int ld, int col) {
    float s = 0.f;
    for (int g = 0; g < TG; ++g) s += t[g * ld + col];
    return s;
}

// ---- kernel P ------------------------------------------------------------------------------------------
struct PrepassSmem { int wt, bias, in, total_floats, ldin; };

inline PrepassSmem prepass_smem_layout(int TG, int K, int WD) {
    PrepassSmem s{};
    SmemFloats m;
    s.ldin = K + 4;
    s.wt = m.take(K * WD);
    s.bias = m.take(WD);
    s.in = m.take(TG * s.ldin);
    s.total_floats = m.off;
    return s;
}

// out = relu(in wt + bias) for one layer: in [N][K] (the features, K = F; or a trunk layer's input a_{j-1}, K = WD), wt the
// packed transpose [K][WD], staged at L.wt, the bias at L.bias, the input tile at L.in (prepass_smem_layout).
template <int TG, int WD>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_prepass_kernel(PrepassSmem L, int64_t n, int K, const float* __restrict__ in, const float* __restrict__ wt,
                          const float* __restrict__ bias, float* __restrict__ a1_out) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RM = TG / 16, CG = WD / 64;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int64_t ntiles = (n + TG - 1) / TG;
    const int n0 = K * WD;
    for (int i = tid * 4; i < n0; i += kDeformThreads * 4)
        *reinterpret_cast<float4*>(smem + L.wt + i) = __ldg(reinterpret_cast<const float4*>(wt + i));
    for (int i = tid; i < WD; i += kDeformThreads) smem[L.bias + i] = __ldg(bias + i);
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG, rem = n - base;
        load_feature_tile<TG>(in, K, base, rem, smem + L.in, L.ldin);
        __syncthreads();
        float acc[RM][CG * 4];
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
        tile_gemm<RM, CG>(smem + L.in, L.ldin, smem + L.wt, WD, K, ty, tx, acc);
#pragma unroll
        for (int c = 0; c < CG; ++c) {
            const float4 bv = *reinterpret_cast<const float4*>(smem + L.bias + c * 64 + tx * 4);
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
    SmemFloats m;
    s.ldw = WD + 4; s.lda = WD + 4; s.ldo = 48;
    s.w1 = m.take(WD * s.ldw);
    s.w2 = m.take(48 * s.ldw);
    s.b1 = m.take(WD);
    s.a1 = m.take(TG * s.lda);
    s.a2 = m.take(TG * s.lda);
    s.dz = m.take(TG * s.lda);
    s.dout = m.take(TG * s.ldo);
    s.total_floats = m.off;
    return s;
}

template <int TG, int WD>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_heads_kernel(DeformBwdArgs ba, HeadSmem L, int64_t n, int num_active) {
    extern __shared__ __align__(16) float smem[];
    constexpr int RM = TG / 16, CG = WD / 64, CN = WD / 16;
    constexpr int NG = kDeformThreads / WD;           // thread groups for the dW2 mapping (2 or 4)
    constexpr int MAXO = 48 / NG;                     // dW2 accumulators per thread (24 or 12)
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    // which head does this CTA own?
    int slot = blockIdx.x % num_active, h = -1;
    for (int hh = 0, s = 0; hh < G4D_NUM_HEADS; ++hh)
        if (ba.d.head_mask & (1 << hh)) { if (s == slot) h = hh; ++s; }
    const int cta_in_head = blockIdx.x / num_active;
    const int ctas_for_head = (gridDim.x - slot + num_active - 1) / num_active;
    const int kout = head_out(h), kp = (kout + 3) & ~3;
    const int64_t ntiles = (n + TG - 1) / TG;
    float* sW1 = smem + L.w1; float* sW2 = smem + L.w2; float* sB1 = smem + L.b1;
    float* sA1 = smem + L.a1; float* sA2 = smem + L.a2; float* sDZ = smem + L.dz; float* sDO = smem + L.dout;
    // persistent weights: W1 [j][i] and W2 [o][j] in torch layout, rows padded to ldw
    stage_rows<WD>(sW1, L.ldw, ba.w1[h], WD);
    for (int i = tid; i < 48 * (WD >> 2); i += kDeformThreads) {
        const int r = i / (WD >> 2), v = i - r * (WD >> 2);
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < kout) val = __ldg(reinterpret_cast<const float4*>(ba.d.w2[h] + r * WD + 4 * v));
        *reinterpret_cast<float4*>(sW2 + r * L.ldw + 4 * v) = val;
    }
    for (int i = tid; i < WD; i += kDeformThreads) sB1[i] = __ldg(ba.d.b1[h] + i);
    // register accumulators that live across all tiles of this CTA
    WGradTile<WD> gW1;
    wgrad_zero<WD>(gW1);
    float gW2[MAXO];
#pragma unroll
    for (int a = 0; a < MAXO; ++a) gW2[a] = 0.f;
    float gB1 = 0.f, gB2 = 0.f;
    const int w2_j = tid % WD, w2_g = tid / WD;
    const float* go = ba.go[h];
    const int go_stride = kout;   // [N][kout] contiguous for every head (shs: 48)
    __syncthreads();

    for (int64_t tile = cta_in_head; tile < ntiles; tile += ctas_for_head) {
        const int64_t base = tile * TG, rem = n - base;
        for (int i = tid; i < TG * (WD >> 2); i += kDeformThreads) {
            const int g = i / (WD >> 2), v = i - g * (WD >> 2);
            float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g < rem) val = *reinterpret_cast<const float4*>(ba.buf.a1 + (base + g) * WD + 4 * v);
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
        if (tid < WD) gB1 += column_sum<TG>(sDZ, L.lda, tid);
        else if (tid - WD < kout && tid >= WD) gB2 += column_sum<TG>(sDO, L.ldo, tid - WD);
        // dW1[j][i] += sum_g dz[g][j] a1[g][i]
        wgrad_accumulate<TG, WD>(gW1, sDZ, sA1, L.lda, ty, tx);
        store_dz_w<TG, WD>(sDZ, L.lda, sW1, L.ldw, ba.buf.da1[h], base, rem, ty, tx);   // da1_h = dz W1 -> HBM
        __syncthreads();
    }
    // flush the register accumulators (one atomic per element per CTA)
    wgrad_flush<WD>(gW1, ba.g.w1[h], ty, tx);
#pragma unroll
    for (int m = 0; m < MAXO; ++m) {
        const int o = w2_g + NG * m;
        if (o < kout) atomicAdd(ba.g.w2[h] + o * WD + w2_j, gW2[m]);
    }
    if (tid < WD) atomicAdd(ba.g.b1[h] + tid, gB1);
    else if (tid - WD < kout) atomicAdd(ba.g.b2[h] + (tid - WD), gB2);
}

// dst[g][0 .. WD) = dA[g] * (act[g] > 0) for the tile's rows g < rem, zero for the rows past n; dA is in [N][WD], or, when
// in == NULL, the sum of the active heads' DA1.  The caller syncs.
template <int TG, int WD>
G4D_D void load_masked_grad(const DeformDesc& d, const DeformBwdBuffers& buf, const float* __restrict__ in,
                            const float* __restrict__ act, int64_t base, int64_t rem, float* __restrict__ dst, int ld) {
    for (int i = threadIdx.x; i < TG * (WD >> 2); i += kDeformThreads) {
        const int g = i / (WD >> 2), v = i - g * (WD >> 2);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        if (g < rem) {
            if (in) {
                s = *reinterpret_cast<const float4*>(in + (base + g) * WD + 4 * v);
            } else {
                for (int h = 0; h < G4D_NUM_HEADS; ++h) {
                    if (!(d.head_mask & (1 << h))) continue;
                    const float4 t = *reinterpret_cast<const float4*>(buf.da1[h] + (base + g) * WD + 4 * v);
                    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                }
            }
            const float4 a = *reinterpret_cast<const float4*>(act + (base + g) * WD + 4 * v);
            s.x = a.x > 0.f ? s.x : 0.f; s.y = a.y > 0.f ? s.y : 0.f;
            s.z = a.z > 0.f ? s.z : 0.f; s.w = a.w > 0.f ? s.w : 0.f;
        }
        *reinterpret_cast<float4*>(dst + g * ld + 4 * v) = s;
    }
}

// ---- kernel T ------------------------------------------------------------------------------------------
// One trunk layer j (1 <= j <= ntrunk): dz = dA_j * (a_j > 0) with dA_j from `din` (NULL: the heads' DA1 sum, j = ntrunk);
// dW_j += dz^T a_{j-1} and db_j += sum dz in registers, flushed once per CTA; dA_{j-1} = dz W_j -> dout.
struct TrunkSmem { int w, a, dz, total_floats, ldw, lda; };

inline TrunkSmem trunk_smem_layout(int TG, int WD) {
    TrunkSmem s{};
    SmemFloats m;
    s.ldw = WD + 4; s.lda = WD + 4;
    s.w = m.take(WD * s.ldw);
    s.a = m.take(TG * s.lda);
    s.dz = m.take(TG * s.lda);
    s.total_floats = m.off;
    return s;
}

template <int TG, int WD>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_trunk_kernel(DeformBwdArgs ba, TrunkSmem L, int64_t n, int j, const float* __restrict__ din, float* __restrict__ dout) {
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    float* sW = smem + L.w; float* sA = smem + L.a; float* sDZ = smem + L.dz;
    const float* act_in = ba.buf.act[j - 1];
    stage_rows<WD>(sW, L.ldw, ba.wt[j - 1], WD);   // W_j [o][i] in torch layout, rows padded to ldw
    WGradTile<WD> gW;
    wgrad_zero<WD>(gW);
    float gB = 0.f;
    const int64_t ntiles = (n + TG - 1) / TG;
    __syncthreads();

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG, rem = n - base;
        load_feature_tile<TG>(act_in, WD, base, rem, sA, L.lda);
        load_masked_grad<TG, WD>(ba.d, ba.buf, din, ba.buf.act[j], base, rem, sDZ, L.lda);
        __syncthreads();
        if (tid < WD) gB += column_sum<TG>(sDZ, L.lda, tid);
        // dW_j[o][i] += sum_g dz[g][o] a_{j-1}[g][i]
        wgrad_accumulate<TG, WD>(gW, sDZ, sA, L.lda, ty, tx);
        store_dz_w<TG, WD>(sDZ, L.lda, sW, L.ldw, dout, base, rem, ty, tx);   // dA_{j-1} = dz W_j -> HBM
        __syncthreads();
    }
    wgrad_flush<WD>(gW, ba.g.wt[j - 1], ty, tx);
    if (tid < WD) atomicAdd(ba.g.bt[j - 1] + tid, gB);
}

// ---- kernel Q ------------------------------------------------------------------------------------------
struct FinalSmem { int w0, feat, dh, total_floats, ldw0, ldf, ldh; };

inline FinalSmem final_smem_layout(int TG, int F, int WD) {
    FinalSmem s{};
    SmemFloats m;
    s.ldw0 = F + 4; s.ldf = F + 4; s.ldh = WD + 4;
    s.w0 = m.take(WD * s.ldw0);
    s.feat = m.take(TG * s.ldf);
    s.dh = m.take(TG * s.ldh);
    s.total_floats = m.off;
    return s;
}

// din: dA_0 from the last T launch, or NULL (no trunk): the heads' DA1 sum
template <int TG, int WD, int FM>
__global__ void __launch_bounds__(kDeformThreads, 1)
deform_bwd_final_kernel(DeformBwdArgs ba, FinalSmem L, int64_t n, const float* __restrict__ din) {
    extern __shared__ __align__(16) float smem[];
    const DeformDesc& d = ba.d;
    const DeformBwdBuffers& buf = ba.buf;
    const int tid = threadIdx.x;
    const int F = d.F, F4 = F >> 2;
    constexpr int NG = kDeformThreads / WD;
    constexpr int MAXF = FM / NG;                   // dW0 accumulators per thread (F <= FM)
    float* sW0 = smem + L.w0; float* sF = smem + L.feat; float* sDH = smem + L.dh;
    stage_rows<WD>(sW0, L.ldw0, ba.w0, F);
    float gW0[MAXF];
#pragma unroll
    for (int m = 0; m < MAXF; ++m) gW0[m] = 0.f;
    float gB0 = 0.f;
    const int w0_j = tid % WD, w0_g = tid / WD;
    const int64_t ntiles = (n + TG - 1) / TG;
    __syncthreads();

    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t base = tile * TG, rem = n - base;
        load_feature_tile<TG>(buf.feat, F, base, rem, sF, L.ldf);
        load_masked_grad<TG, WD>(d, buf, din, buf.act[0], base, rem, sDH, L.ldh);
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
        if (tid < WD) gB0 += column_sum<TG>(sDH, L.ldh, tid);
        // dfeat[g][f..f+3] = sum_j dh[g][j] W0[j][f..f+3]  -> DFEAT (the scatter's input)
        for (int i = tid; i < TG * F4; i += kDeformThreads) {
            const int g = i / F4, v = i - g * F4;
            if (g >= rem) continue;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int j = 0; j < WD; ++j) {
                const float dh = sDH[g * L.ldh + j];
                const float4 w = *reinterpret_cast<const float4*>(sW0 + j * L.ldw0 + 4 * v);
                acc.x = fmaf(dh, w.x, acc.x); acc.y = fmaf(dh, w.y, acc.y); acc.z = fmaf(dh, w.z, acc.z); acc.w = fmaf(dh, w.w, acc.w);
            }
            *reinterpret_cast<float4*>(buf.dfeat + (base + g) * F + 4 * v) = acc;
        }
        __syncthreads();
    }
#pragma unroll
    for (int m = 0; m < MAXF; ++m) {
        const int f = w0_g + NG * m;
        if (f < F) atomicAdd(ba.g.w0 + w0_j * F + f, gW0[m]);
    }
    if (tid < WD) atomicAdd(ba.g.b0 + tid, gB0);
}

// ---- HexPlane scatter of every backward at full occupancy: LPG lanes per Gaussian, lane v < C/4 scatters channel vector v --
// LPG is C/4 rounded up to a power of two (the d(xyz) reduction shuffles over the lanes of one Gaussian); lanes v >= C/4 add
// nothing.
constexpr int scatter_lanes(int C4) { return C4 <= 1 ? 1 : C4 <= 2 ? 2 : C4 <= 4 ? 4 : 8; }

// PER_ROW: Gaussian g at its own time d.times[g]; the time planes' gradients go straight to the planes and dL/dt to g_times
template <int C4, bool PER_ROW>
__global__ void __launch_bounds__(256, 2) bwd_scatter_kernel(DeformBwdArgs ba, int64_t n, const float* __restrict__ xyz) {
    const DeformDesc& d = ba.d;
    constexpr int LPG = scatter_lanes(C4);
    constexpr int GPB = 256 / LPG;          // Gaussians per block
    const int64_t g0 = (int64_t)blockIdx.x * GPB;
    const int64_t g = g0 + threadIdx.x / LPG;
    const int v = threadIdx.x % LPG;
    // residual path: d(out)/d(in) = identity for scaling / rotation / opacity / shs (contiguous ranges, coalesced)
    for (int hh = 1; hh < G4D_NUM_HEADS; ++hh) {
        if (!ba.gi[hh]) continue;
        const int ko = head_out(hh);
        const int64_t lo = g0 * ko, hi = (g0 + GPB < n ? g0 + GPB : n) * ko;
        for (int64_t i = lo + threadIdx.x; i < hi; i += 256) ba.gi[hh][i] = ba.go[hh] ? ba.go[hh][i] : 0.f;
    }
    float gpix[3] = {0.f, 0.f, 0.f};
    float gt = 0.f;   // dL/d(times[g]) (PER_ROW): t enters the time planes unnormalised, so d(t_pix)/dt is the tap's gmul
    const AabbNorm nrm(d.aabb);
    if (g < n && (LPG == C4 || v < C4)) {
        float pcs[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) pcs[a] = nrm(a, xyz[3 * g + a]);
        const float tg = PER_ROW ? __ldg(d.times + g) : 0.f;
        for (int l = 0; l < d.levels; ++l) {
            Tap1D tx[PER_ROW ? 4 : 3];
#pragma unroll
            for (int a = 0; a < 3; ++a) tx[a] = make_tap(pcs[a], d.res[l][a]);
            if (PER_ROW) tx[PER_ROW ? 3 : 0] = make_tap(tg, d.res[l][3]);
            const float4 df = __ldg(reinterpret_cast<const float4*>(ba.buf.dfeat + g * d.F + l * d.C + 4 * v));
            scatter_vector<PER_ROW>(d.planes[l], d.trow[l], d.res[l], ba.g.planes[l], ba.buf.trow_grad[l], tx, v, C4, df, gpix, gt);
        }
    }
    // the LPG lanes of a Gaussian are adjacent
#pragma unroll
    for (int a = 0; a < 3; ++a)
        for (int o = 1; o < LPG; o <<= 1) gpix[a] += __shfl_xor_sync(0xffffffffu, gpix[a], o);
    if (PER_ROW)
        for (int o = 1; o < LPG; o <<= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
    if (g < n && v == 0 && ba.gi[0]) {
#pragma unroll
        for (int a = 0; a < 3; ++a) ba.gi[0][g * 3 + a] = (ba.go[0] ? ba.go[0][g * 3 + a] : 0.f) + gpix[a] * nrm.scale[a];
    }
    if (PER_ROW && g < n && v == 0 && ba.g_times) ba.g_times[g] = gt;
}

static cudaError_t launch_bwd_scatter(const DeformBwdArgs& ba, int64_t n, const float* xyz, cudaStream_t st) {
    const int C4 = ba.d.C / 4;
    const unsigned grid = (unsigned)((n * scatter_lanes(C4) + 255) / 256);
    switch (C4) {   // every channel width the C-ABI takes: C = 4 .. 32
#define G4D_SCATTER_CASE(K)                                                     \
        case K:                                                                 \
            if (ba.d.times) bwd_scatter_kernel<K, true><<<grid, 256, 0, st>>>(ba, n, xyz); \
            else bwd_scatter_kernel<K, false><<<grid, 256, 0, st>>>(ba, n, xyz);          \
            break;
        G4D_SCATTER_CASE(1) G4D_SCATTER_CASE(2) G4D_SCATTER_CASE(3) G4D_SCATTER_CASE(4)
        G4D_SCATTER_CASE(5) G4D_SCATTER_CASE(6) G4D_SCATTER_CASE(7) G4D_SCATTER_CASE(8)
#undef G4D_SCATTER_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// ---- kernel T: collapsed time-row gradients -> the two time rows of each (axis, t) plane --------------------
// s.src: the rows' gradients; s.dst: the time planes' gradients; s.plane: the time planes.
// SINK: also dL/dt into *sink (zeroed by the caller; DESIGN.md §4.11).  A row r = w0 P[i0] + w1 P[i1] of the time plane
// P = s.plane[l][a] has dr/dt = gmul (P[i1] - P[i0]), so element e adds gv gmul (P[i1][e] - P[i0][e]); the block sums its
// elements and adds the sum into *sink with one atomic.
// (The plane pointers are a member of the segments, not a parameter of their own: as one, ptxas copies them to the stack.)
struct TimeGradSegs : TimeRowSegs {
    const float* plane[G4D_MAX_LEVELS][3];
    TimeGradSegs(int levels_, const int32_t (*res_)[4], int C_) : TimeRowSegs(levels_, res_, C_), plane{} {}
};
template <bool SINK>
__global__ void distribute_time_grad_kernel(TimeGradSegs s, TimeArg time, float* sink) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float dt = 0.f;
    if (i < s.start[3 * s.levels]) {
        int l, a, e;
        s.locate(i, l, a, e);
        const Tap1D ty = make_tap(time.get(), s.res[l][3]);
        const int rowlen = s.res[l][a] * s.C;
        const float gv = s.src[l][a][e];
        atomicAdd(s.dst[l][a] + (size_t)ty.i0 * rowlen + e, gv * ty.w0);
        atomicAdd(s.dst[l][a] + (size_t)ty.i1 * rowlen + e, gv * ty.w1);
        if (SINK) {
            const float* p = s.plane[l][a];
            dt = gv * (__ldg(p + (size_t)ty.i1 * rowlen + e) - __ldg(p + (size_t)ty.i0 * rowlen + e)) * ty.gmul;
        }
    }
    if (SINK) {
        const float sum = block_sum_f(dt);
        if (threadIdx.x == 0) atomicAdd(sink, sum);
    }
}

// ---- host side -------------------------------------------------------------------------------------------
static cudaError_t launch_distribute_time_grad(const DeformBwdArgs& ba, TimeArg time, float* g_time, cudaStream_t st) {
    const DeformDesc& d = ba.d;
    TimeGradSegs s(d.levels, d.res, d.C);
    for (int l = 0; l < d.levels; ++l)
        for (int a = 0; a < 3; ++a) {
            s.src[l][a] = ba.buf.trow_grad[l][a]; s.dst[l][a] = ba.g.planes[l][kTimePlane[a]];
            s.plane[l][a] = d.planes[l][kTimePlane[a]];
        }
    const int total = (int)s.total();
    if (g_time) distribute_time_grad_kernel<true><<<(total + 255) / 256, 256, 0, st>>>(s, time, g_time);
    else distribute_time_grad_kernel<false><<<(total + 255) / 256, 256, 0, st>>>(s, time, nullptr);
    return cudaGetLastError();
}

// carves the scratch; *gathered: where the gather writes the features (buf.feat until the forward's replace them)
static DeformBwdBuffers carve_backward_scratch(Carve& m, const DeformDesc& d, int64_t n, bool tc, float** gathered) {
    const size_t N = (size_t)(n > 0 ? n : 1);
    const TimeRows tr(d.levels, d.res, d.C);
    DeformBwdBuffers b{};
    if (tc) {
        b.images = m.take<uint8_t>(tc_bwd_images_bytes(d, n));
    } else {
        b.a1 = b.act[d.ntrunk] = m.take<float>(N * d.WD);
        for (int h = 0; h < G4D_NUM_HEADS; ++h)
            if (d.head_mask & (1 << h)) b.da1[h] = m.take<float>(N * d.WD);
        if (d.ntrunk > 0) {   // a_0 .. a_{D-2} and the dA pair: N * WD * 4 B each
            for (int j = 0; j < d.ntrunk; ++j) b.act[j] = m.take<float>(N * d.WD);
            for (int k = 0; k < 2; ++k) b.dact[k] = m.take<float>(N * d.WD);
        }
    }
    const size_t rows128 = (N + 127) / 128 * 128;   // whole tiles of the tensor-core kernels
    b.feat = *gathered = m.take<float>(rows128 * d.F);
    b.dfeat = m.take<float>(rows128 * d.F);
    if (d.times) return b;   // per-row: the time planes' gradients go straight to the planes
    float* rows = m.take<float>(tr.total());
    if (rows) tr.place(rows, b.trow_grad);
    return b;
}

size_t deform_backward_scratch_bytes(const DeformDesc& d, int64_t n, bool tc) {
    Carve m;
    float* gathered;
    carve_backward_scratch(m, d, n, tc, &gathered);
    return m.bytes();
}

// FFMA engine: P (once per layer up to a_{D-1}), H, T (once per trunk layer), Q
template <int TG, int WD>
static cudaError_t launch_ffma_engine(const DeformBwdArgs& ba, int64_t n, int sm_count, cudaStream_t st) {
    const DeformDesc& d = ba.d;
    const DeformBwdBuffers& buf = ba.buf;
    int active = 0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) active += (d.head_mask >> h) & 1;
    const int64_t ntiles = (n + TG - 1) / TG;
    const unsigned grid = (unsigned)(ntiles < sm_count ? ntiles : sm_count);
    cudaError_t e;
    // P
    for (int j = 0; j <= d.ntrunk; ++j) {
        const int K = j == 0 ? d.F : WD;
        const PrepassSmem L = prepass_smem_layout(TG, K, WD);
        e = j == 0 ? launch_smem(deform_bwd_prepass_kernel<TG, WD>, grid, kDeformThreads, (size_t)L.total_floats * 4, st, L, n, K,
                                 buf.feat, d.w0t, d.b0, buf.act[0])
                   : launch_smem(deform_bwd_prepass_kernel<TG, WD>, grid, kDeformThreads, (size_t)L.total_floats * 4, st, L, n, K,
                                 buf.act[j - 1], d.wtt[j - 1], d.bt[j - 1], buf.act[j]);
        if (e != cudaSuccess) return e;
    }
    // H
    if (active > 0) {
        const HeadSmem L = head_smem_layout(TG, WD);
        int hgrid = sm_count;
        if ((int64_t)hgrid > ntiles * active) hgrid = (int)(ntiles * active);
        if (hgrid < active) hgrid = active;
        e = launch_smem(deform_bwd_heads_kernel<TG, WD>, hgrid, kDeformThreads, (size_t)L.total_floats * 4, st, ba, L, n, active);
        if (e != cudaSuccess) return e;
    }
    // T: dA_{j-1} from dA_j, j = ntrunk .. 1 (dA_ntrunk: the heads' DA1 sum)
    const float* din = nullptr;
    const TrunkSmem LT = trunk_smem_layout(TG, WD);
    for (int j = d.ntrunk, k = 0; j >= 1; --j, k ^= 1) {
        e = launch_smem(deform_bwd_trunk_kernel<TG, WD>, grid, kDeformThreads, (size_t)LT.total_floats * 4, st, ba, LT, n, j, din,
                        buf.dact[k]);
        if (e != cudaSuccess) return e;
        din = buf.dact[k];
    }
    // Q
    const FinalSmem L = final_smem_layout(TG, d.F, WD);
    auto final_kernel = d.F <= 32 ? deform_bwd_final_kernel<TG, WD, 32>
                      : d.F <= 64 ? deform_bwd_final_kernel<TG, WD, 64> : deform_bwd_final_kernel<TG, WD, 128>;
    return launch_smem(final_kernel, grid, kDeformThreads, (size_t)L.total_floats * 4, st, ba, L, n, din);
}

cudaError_t launch_deform_backward(const DeformDesc& d, const G4DDeformParams& prm, const G4DDeformGrads& grads, const TcBwdWeights* tc,
                                   TimeArg time, int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                                   float* const gi[G4D_NUM_HEADS], float* g_times, float* g_time, const uint32_t* relu_bits,
                                   const float* saved_feat, const uint32_t* order, void* scratch, int sm_count, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const TimeRows tr(d.levels, d.res, d.C);
    Carve m(scratch);
    float* gathered;
    DeformBwdArgs ba{};
    ba.d = d;
    ba.g = grads;
    ba.w0 = prm.w0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) { ba.w1[h] = prm.w1[h]; ba.go[h] = go[h]; ba.gi[h] = gi[h]; }
    for (int j = 0; j < d.ntrunk; ++j) ba.wt[j] = prm.wt[j];
    ba.g_times = g_times;
    ba.buf = carve_backward_scratch(m, d, n, tc != nullptr, &gathered);
    if (saved_feat) ba.buf.feat = saved_feat;   // the features the forward of this view gathered
    const DeformBwdBuffers& buf = ba.buf;
    cudaError_t e = d.times ? cudaSuccess : cudaMemsetAsync(buf.trow_grad[0][0], 0, tr.total() * 4, st);
    if (e != cudaSuccess) return e;
    if (!saved_feat && (e = launch_deform_features(d, n, xyz, order, gathered, false, st)) != cudaSuccess) return e;
    // the engine: d(feat) -> DFEAT and the weight gradients (the tensor-core wgrad kernel after the scatter)
    if (tc) e = launch_tc_bwd_dgrad(d, *tc, n, go, relu_bits, buf.feat, buf.dfeat, buf.images, sm_count, st);
    else if (d.WD == 128) e = launch_ffma_engine<64, 128>(ba, n, sm_count, st);
    else if (d.WD == 64) e = launch_ffma_engine<128, 64>(ba, n, sm_count, st);
    else e = cudaErrorInvalidValue;
    if (e != cudaSuccess) return e;
    if ((e = launch_bwd_scatter(ba, n, xyz, st)) != cudaSuccess) return e;
    if (tc && (e = launch_tc_bwd_wgrad(d, grads, n, buf.images, sm_count, st)) != cudaSuccess) return e;
    return d.times ? cudaSuccess : launch_distribute_time_grad(ba, time, g_time, st);
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
