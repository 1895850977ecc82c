// g4d_raster.cu -- the per-tile front-to-back alpha compositing forward / back-to-front backward.
// SURVEY.md Appendix A.3-A.4 (binning, A.2, lives in g4d_bin.cu).
// Reference stage replaced: the CUDA rasterizer behind /root/reference/gaussian_renderer/__init__.py:120-128.
#include <type_traits>

#include "g4d_internal.h"
#include "raster_cull.cuh"

namespace g4d {

// Two-lane float arithmetic of the blend kernels.  Hopper has no packed FP32 instructions, so each is two scalar
// round-to-nearest operations (never contracted, whatever -fmad says): the per-lane results are exactly those of the scalar
// expression tree.
G4D_D float2 f2_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
G4D_D float2 f2_mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
G4D_D float2 f2_fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// ------------------------------------------------------------------------------------------------------
// A.3 blend forward: one 16x16 CTA per tile, instances staged through shared memory in batches of 256.  A warp owns a compact
// 16 x 4 pixel strip of the tile and culls instances against it; two pixels per thread, evaluated as f32x2 lanes: the two
// pixels of a thread share their column, so dx, the dx^2 term and the instance record are scalar and computed once per
// instance, and only what depends on the row is evaluated per lane (f2_add / f2_mul / f2_fma).  The per-pixel decisions are
// selects, not branches.  power = fma(dy, -(conic.y dx), -0.5 (conic.z dy^2 + conic.x dx^2)) per lane.
// out_alpha (may be NULL): the accumulated opacity 1 - T of every pixel, T the transmittance final_T holds.
__global__ void __launch_bounds__(kTilePixels / 2)
blend_forward_kernel(const CameraDev* __restrict__ cam, GeomBuffers g, const uint32_t* __restrict__ ids,
                     const uint2* __restrict__ ranges, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                     float* __restrict__ out_color, float* __restrict__ out_depth, int warp_cull,
                     float* __restrict__ out_alpha) {
    constexpr int PPT = 2, NT = kTilePixels / PPT;
    __shared__ float4 s0[kTilePixels];
    __shared__ float4 s1[kTilePixels];
    __shared__ float2 s2[kTilePixels];
    pdl_wait();
    pdl_trigger();
    const int H = cam->H, W = cam->W;
    const int tile = blockIdx.y * gridDim.x + blockIdx.x;
    const uint2 range = ranges[tile];
    const int rounds = (int)((range.y - range.x + kTilePixels - 1) / kTilePixels);
    int todo = (int)(range.y - range.x);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // warp w owns pixel rows [4w, 4w + 4) of the tile: lane l -> column l & 15, rows 4w + (l >> 4) and 4w + (l >> 4) + 2
    const int px = blockIdx.x * kTile + (lane & 15), py0 = blockIdx.y * kTile + 2 * PPT * warp + (lane >> 4), py1 = py0 + 2;
    const bool in0 = px < W && py0 < H, in1 = px < W && py1 < H;
    const float pxf = (float)px;
    const float2 npy = make_float2(-(float)py0, -(float)py1);
    float2 T = make_float2(1.f, 1.f), C0 = make_float2(0.f, 0.f), C1 = C0, C2 = C0, D = C0;
    uint32_t last0 = 0, last1 = 0;
    bool done0 = !in0, done1 = !in1;
    bool all_done = done0 && done1;
    const float sx0 = (float)(blockIdx.x * kTile), sx1 = sx0 + (float)(kTile - 1);
    const float sy0 = (float)(blockIdx.y * kTile + 2 * PPT * warp), sy1 = sy0 + (float)(2 * PPT - 1);
    for (int i = 0; i < rounds; ++i, todo -= kTilePixels) {
        if (__syncthreads_count(all_done) == NT) break;
#pragma unroll
        for (int k = 0; k < PPT; ++k) {
            const int slot = threadIdx.x + k * NT;
            const int progress = i * kTilePixels + slot;
            if (range.x + progress < range.y) {
                const uint32_t id = ids[range.x + progress];
                s0[slot] = g.rec0[id];
                s1[slot] = g.rec1[id];
                s2[slot] = g.rec2[id];
            }
        }
        __syncthreads();
        const int cnt = min(kTilePixels, todo);
        for (int base = 0; base < cnt; base += 32) {
            if (__all_sync(0xffffffffu, all_done)) break;
            // lane l tests instance base + l against the warp's strip: instances that cannot reach alpha >= 1/255 on any
            // of its pixels are skipped by the whole warp (they would be skipped pixel by pixel anyway)
            const int jt = base + lane;
            bool hit = jt < cnt;
            if (hit && warp_cull) hit = rect_contributes(s0[jt], s1[jt], sx0, sx1, sy0, sy1);
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                const int j = base + __ffs(mask) - 1;
                mask &= mask - 1;
                const uint32_t contributor = (uint32_t)(i * kTilePixels + j + 1);
                const float4 a = s0[j];
                const float4 b = s1[j];
                const float2 c = s2[j];
                const float dx = a.x - pxf;
                const float2 dy = f2_add(make_float2(a.y, a.y), npy);
                const float q = a.z * dx * dx, nr = -(a.w * dx);
                const float2 s = f2_fma(make_float2(b.x, b.x), f2_mul(dy, dy), make_float2(q, q));
                const float2 pw = f2_fma(dy, make_float2(nr, nr), f2_mul(s, make_float2(-0.5f, -0.5f)));
                // exp(power) = ex2(power * log2 e); .ftz: a power below -87 flushes to 0 instead of a denormal (alpha < 1/255 either way)
                const float2 pl = f2_mul(pw, make_float2(1.4426950408889634f, 1.4426950408889634f));
                float ex0, ex1;
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex0) : "f"(pl.x));
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex1) : "f"(pl.y));
                float2 al = f2_mul(make_float2(b.y, b.y), make_float2(ex0, ex1));
                al.x = fminf(kAlphaMax, al.x); al.y = fminf(kAlphaMax, al.y);
                const bool c0 = !done0 && pw.x <= 0.f && al.x >= kAlphaMin, c1 = !done1 && pw.y <= 0.f && al.y >= kAlphaMin;
                const float2 tt = f2_mul(T, f2_add(make_float2(1.f, 1.f), make_float2(-al.x, -al.y)));
                const bool st0 = c0 && tt.x < kTransmittanceStop, st1 = c1 && tt.y < kTransmittanceStop;
                done0 = done0 || st0; done1 = done1 || st1;
                const bool k0 = c0 && !st0, k1 = c1 && !st1;
                float2 w = f2_mul(al, T);
                w.x = k0 ? w.x : 0.f; w.y = k1 ? w.y : 0.f;
                C0 = f2_fma(make_float2(b.z, b.z), w, C0);
                C1 = f2_fma(make_float2(b.w, b.w), w, C1);
                C2 = f2_fma(make_float2(c.x, c.x), w, C2);
                D = f2_fma(make_float2(c.y, c.y), w, D);
                T.x = k0 ? tt.x : T.x; T.y = k1 ? tt.y : T.y;
                last0 = k0 ? contributor : last0; last1 = k1 ? contributor : last1;
            }
            all_done = done0 && done1;
        }
    }
    const size_t hw = (size_t)H * W;
    if (in0) {
        const size_t pix = (size_t)py0 * W + (size_t)px;
        final_T[pix] = T.x; n_contrib[pix] = last0;
        out_color[pix] = fmaf(T.x, cam->bg[0], C0.x); out_color[hw + pix] = fmaf(T.x, cam->bg[1], C1.x);
        out_color[2 * hw + pix] = fmaf(T.x, cam->bg[2], C2.x);
        out_depth[pix] = D.x;
        if (out_alpha) out_alpha[pix] = 1.f - T.x;
    }
    if (in1) {
        const size_t pix = (size_t)py1 * W + (size_t)px;
        final_T[pix] = T.y; n_contrib[pix] = last1;
        out_color[pix] = fmaf(T.y, cam->bg[0], C0.y); out_color[hw + pix] = fmaf(T.y, cam->bg[1], C1.y);
        out_color[2 * hw + pix] = fmaf(T.y, cam->bg[2], C2.y);
        out_depth[pix] = D.y;
        if (out_alpha) out_alpha[pix] = 1.f - T.y;
    }
}

cudaError_t launch_blend_forward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                 float* out_color, float* out_depth, int warp_cull, float* out_alpha, cudaStream_t st) {
    if (grid_x * grid_y == 0) return cudaSuccess;
    return launch_k(blend_forward_kernel, dim3(grid_x, grid_y), dim3(kTilePixels / 2), 0, st, kPdl, cam, g, b.ids_sorted, b.ranges,
                    im.final_T, im.n_contrib, out_color, out_depth, warp_cull, out_alpha);
}

// ------------------------------------------------------------------------------------------------------
// A.4 blend backward: same tiling, instances traversed back to front.  Per instance the 9 partial gradients
// of a warp's 32 pixels are reduced with shuffles (only when some lane contributes) and lane 0 issues the
// atomics, so global RED traffic is <= 8 x 9 per (tile, instance) instead of 256 x 9.
// the colour b of a staged rec2 entry: the colour-only instance stages (b), the depth instance (b, depth)
G4D_D float staged_b(float v) { return v; }
G4D_D float staged_b(float2 v) { return v.x; }

// Two pixels per thread as f32x2 lanes, like the forward: the per-pixel gradient arithmetic is one f2_* operation per pixel
// PAIR, validity is a select instead of a branch, and power / alpha are formed exactly as the forward forms them (same
// threshold decisions).
// DEPTH: the depth image D = sum_i w_i z_i takes the gradient dL_ddepth [H,W] too: a depth accumulator beside the colour
// ones adds (z_i - aD') dL/dD to dL/dalpha, and dL/dz_i = w_i dL/dD is reduced per warp into g_depth [N].  dL_dcolor may
// then be NULL (a zero colour gradient).  With DEPTH off dL_ddepth and g_depth are not read.
// dL_dalpha (may be NULL): the gradient [H,W] of the alpha image A = 1 - T_final.  dA/dalpha_i = T_final / (1 - alpha_i) is
// the background term's derivative with the opposite sign, so dL/dA folds into the per-pixel bgdot (bgdot - dL/dA) and needs
// no per-Gaussian term.  dL_dcolor may then be NULL too.
template <bool DEPTH>
__global__ void __launch_bounds__(kTilePixels / 2)
blend_backward_kernel(const CameraDev* __restrict__ cam, GeomBuffers g, const uint32_t* __restrict__ ids,
                      const uint2* __restrict__ ranges, const float* __restrict__ final_T,
                      const uint32_t* __restrict__ n_contrib, const float* __restrict__ dL_dcolor,
                      float* __restrict__ g_mean2D, float* __restrict__ g_conic, float* __restrict__ g_opacity,
                      float* __restrict__ g_rgb, int warp_cull, const float* __restrict__ dL_ddepth,
                      float* __restrict__ g_depth, const float* __restrict__ dL_dalpha) {
    constexpr int PPT = 2, NT = kTilePixels / PPT;
    __shared__ float4 s0[kTilePixels];
    __shared__ float4 s1[kTilePixels];
    __shared__ std::conditional_t<DEPTH, float2, float> s2[kTilePixels];
    __shared__ uint32_t sid[kTilePixels];
    const int H = cam->H, W = cam->W;
    const int tile = blockIdx.y * gridDim.x + blockIdx.x;
    const uint2 range = ranges[tile];
    const int total = (int)(range.y - range.x);
    const int rounds = (total + kTilePixels - 1) / kTilePixels;
    const size_t hw = (size_t)H * W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float sx0 = (float)(blockIdx.x * kTile), sx1 = sx0 + (float)(kTile - 1);
    const float sy0 = (float)(blockIdx.y * kTile + 2 * PPT * warp), sy1 = sy0 + (float)(2 * PPT - 1);
    // warp w owns pixel rows [4w, 4w + 4) of the tile: lane l -> column l & 15, rows 4w + (l >> 4) and 4w + (l >> 4) + 2
    const int px = blockIdx.x * kTile + (lane & 15), py0 = blockIdx.y * kTile + 2 * PPT * warp + (lane >> 4), py1 = py0 + 2;
    const bool in0 = px < W && py0 < H, in1 = px < W && py1 < H;
    const size_t pix0 = (size_t)py0 * W + px, pix1 = (size_t)py1 * W + px;
    const float pxf = (float)px;
    const float2 npy = make_float2(-(float)py0, -(float)py1);
    const float2 Tfin = make_float2(in0 ? final_T[pix0] : 0.f, in1 ? final_T[pix1] : 0.f);
    float2 T = Tfin;
    const int last0 = in0 ? (int)n_contrib[pix0] : 0, last1 = in1 ? (int)n_contrib[pix1] : 0;
    const bool c0in = in0 && dL_dcolor, c1in = in1 && dL_dcolor;
    const float2 dp0 = make_float2(c0in ? dL_dcolor[pix0] : 0.f, c1in ? dL_dcolor[pix1] : 0.f);
    const float2 dp1 = make_float2(c0in ? dL_dcolor[hw + pix0] : 0.f, c1in ? dL_dcolor[hw + pix1] : 0.f);
    const float2 dp2 = make_float2(c0in ? dL_dcolor[2 * hw + pix0] : 0.f, c1in ? dL_dcolor[2 * hw + pix1] : 0.f);
    float2 dpD = make_float2(0.f, 0.f), aD = dpD, lD = dpD;      // DEPTH: dL/dD, depth accumulator, last depth
    if constexpr (DEPTH) dpD = make_float2(in0 ? dL_ddepth[pix0] : 0.f, in1 ? dL_ddepth[pix1] : 0.f);
    float2 bgdot = make_float2(cam->bg[0] * dp0.x + cam->bg[1] * dp1.x + cam->bg[2] * dp2.x,
                               cam->bg[0] * dp0.y + cam->bg[1] * dp1.y + cam->bg[2] * dp2.y);
    if (dL_dalpha) {
        if (in0) bgdot.x = __fsub_rn(bgdot.x, dL_dalpha[pix0]);
        if (in1) bgdot.y = __fsub_rn(bgdot.y, dL_dalpha[pix1]);
    }
    const float2 nTfin = make_float2(-Tfin.x, -Tfin.y);
    float2 ac0 = make_float2(0.f, 0.f), ac1 = ac0, ac2 = ac0, lc0 = ac0, lc1 = ac0, lc2 = ac0, la = ac0;
    const float ddx = 0.5f * (float)W, ddy = 0.5f * (float)H;
    // block-wide maximum of n_contrib: entries beyond it contribute to no pixel of the tile
    const int max_last = __reduce_max_sync(0xffffffffu, max(last0, last1));
    __shared__ int s_max[NT / 32];
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = max_last;
    __syncthreads();
    int tile_last = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) tile_last = max(tile_last, s_max[w]);
    // warp-level reduction plan: after the butterfly lane l holds value (l >> 2) of {mean2D.xy, conic.xyz, rgb}; lanes
    // 0,4,..,28 add one value each, lane 1 adds the opacity gradient -- one predicated RED instruction per Gaussian
    const bool hi16 = lane & 16, hi8 = lane & 8, hi4 = lane & 4;
    const int vidx = lane >> 2;
    const bool red_lane = (lane & 3) == 0 || lane == 1;
    float* red_base = lane == 1 ? g_opacity : vidx < 2 ? g_mean2D + vidx : vidx < 5 ? g_conic + (vidx - 2) : g_rgb + (vidx - 5);
    const uint32_t red_stride = lane == 1 ? 1u : vidx < 2 ? 2u : 3u;
    const float2 one2 = make_float2(1.f, 1.f);

    for (int i = 0; i < rounds; ++i) {
        // batch i covers list positions [total - (i+1)*256, total - i*256) traversed from the back; slot s stages position hi-1-s
        const int hi = total - i * kTilePixels;
        if (hi - kTilePixels >= tile_last) continue;      // whole batch behind every pixel's last contributor
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PPT; ++k) {
            const int slot = threadIdx.x + k * NT;
            const int pos = hi - 1 - slot;
            if (pos >= 0) {
                const uint32_t id = ids[range.x + pos];
                sid[slot] = id;
                s0[slot] = g.rec0[id];
                s1[slot] = g.rec1[id];
                if constexpr (DEPTH) s2[slot] = g.rec2[id];
                else s2[slot] = g.rec2[id].x;
            }
        }
        __syncthreads();
        const int cnt = min(kTilePixels, hi);
        for (int base = 0; base < cnt; base += 32) {
            // lane l tests instance base + l: behind every pixel of this warp's strip, or unable to reach alpha >= 1/255
            // anywhere on the strip (same predicate as the exact tile cull) -> skipped by the whole warp
            const int jt = base + lane;
            bool hit = jt < cnt && (hi - 1 - jt) < max_last;
            if (hit && warp_cull) hit = rect_contributes(s0[jt], s1[jt], sx0, sx1, sy0, sy1);
            uint32_t mask = __ballot_sync(0xffffffffu, hit);
            while (mask) {
                const int j = base + __ffs(mask) - 1;
                mask &= mask - 1;
                const int lpos = hi - 1 - j;
                const float4 a = s0[j];
                const float4 b = s1[j];
                const float dx = a.x - pxf;
                const float2 dy = f2_add(make_float2(a.y, a.y), npy);
                const float q = a.z * dx * dx, nr = -(a.w * dx);
                const float2 sq = f2_fma(make_float2(b.x, b.x), f2_mul(dy, dy), make_float2(q, q));
                const float2 pw = f2_fma(dy, make_float2(nr, nr), f2_mul(sq, make_float2(-0.5f, -0.5f)));
                const float2 pl = f2_mul(pw, make_float2(1.4426950408889634f, 1.4426950408889634f));
                float2 G;
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(G.x) : "f"(pl.x));
                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(G.y) : "f"(pl.y));
                float2 al = f2_mul(make_float2(b.y, b.y), G);
                al.x = fminf(kAlphaMax, al.x); al.y = fminf(kAlphaMax, al.y);
                const bool v0 = lpos < last0 && pw.x <= 0.f && al.x >= kAlphaMin, v1 = lpos < last1 && pw.y <= 0.f && al.y >= kAlphaMin;
                if (!__any_sync(0xffffffffu, v0 || v1)) continue;
                const float c0 = b.z, c1 = b.w, c2 = staged_b(s2[j]);
                const float2 om = f2_add(one2, make_float2(-al.x, -al.y));
                const float2 ra = make_float2(__fdividef(1.f, om.x), __fdividef(1.f, om.y));   // alpha <= 0.99
                const float2 Tn = f2_mul(T, ra);
                float2 w = f2_mul(al, Tn);
                const float2 oml = f2_add(one2, make_float2(-la.x, -la.y));
                const float2 a0n = f2_fma(la, lc0, f2_mul(oml, ac0));
                const float2 a1n = f2_fma(la, lc1, f2_mul(oml, ac1));
                const float2 a2n = f2_fma(la, lc2, f2_mul(oml, ac2));
                float2 dLa = f2_mul(f2_add(make_float2(c0, c0), make_float2(-a0n.x, -a0n.y)), dp0);
                dLa = f2_fma(f2_add(make_float2(c1, c1), make_float2(-a1n.x, -a1n.y)), dp1, dLa);
                dLa = f2_fma(f2_add(make_float2(c2, c2), make_float2(-a2n.x, -a2n.y)), dp2, dLa);
                float z = 0.f;
                float2 aDn = aD;
                if constexpr (DEPTH) {     // no background term: depth has no bgdot analogue
                    z = s2[j].y;
                    aDn = f2_fma(la, lD, f2_mul(oml, aD));
                    dLa = f2_fma(f2_add(make_float2(z, z), make_float2(-aDn.x, -aDn.y)), dpD, dLa);
                }
                dLa = f2_mul(dLa, Tn);
                dLa = f2_fma(f2_mul(nTfin, ra), bgdot, dLa);
                // commit the per-pixel state of the pixels this instance is valid for; mask the contributions of the others
                T.x = v0 ? Tn.x : T.x; T.y = v1 ? Tn.y : T.y;
                ac0.x = v0 ? a0n.x : ac0.x; ac0.y = v1 ? a0n.y : ac0.y;
                ac1.x = v0 ? a1n.x : ac1.x; ac1.y = v1 ? a1n.y : ac1.y;
                ac2.x = v0 ? a2n.x : ac2.x; ac2.y = v1 ? a2n.y : ac2.y;
                lc0.x = v0 ? c0 : lc0.x; lc0.y = v1 ? c0 : lc0.y;
                lc1.x = v0 ? c1 : lc1.x; lc1.y = v1 ? c1 : lc1.y;
                lc2.x = v0 ? c2 : lc2.x; lc2.y = v1 ? c2 : lc2.y;
                la.x = v0 ? al.x : la.x; la.y = v1 ? al.y : la.y;
                if constexpr (DEPTH) {
                    aD.x = v0 ? aDn.x : aD.x; aD.y = v1 ? aDn.y : aD.y;
                    lD.x = v0 ? z : lD.x; lD.y = v1 ? z : lD.y;
                }
                w.x = v0 ? w.x : 0.f; w.y = v1 ? w.y : 0.f;
                dLa.x = v0 ? dLa.x : 0.f; dLa.y = v1 ? dLa.y : 0.f;
                float v[8];
                {
                    const float2 p5 = f2_mul(w, dp0), p6 = f2_mul(w, dp1), p7 = f2_mul(w, dp2);
                    v[5] = p5.x + p5.y; v[6] = p6.x + p6.y; v[7] = p7.x + p7.y;
                }
                const float2 dLdG = f2_mul(make_float2(b.y, b.y), dLa);
                const float2 gdx = f2_mul(G, make_float2(dx, dx)), gdy = f2_mul(G, dy);
                {
                    const float2 t0 = f2_fma(gdy, make_float2(-a.w, -a.w), f2_mul(gdx, make_float2(-a.z, -a.z)));
                    const float2 t1 = f2_fma(gdx, make_float2(-a.w, -a.w), f2_mul(gdy, make_float2(-b.x, -b.x)));
                    const float2 u0 = f2_mul(dLdG, t0), u1 = f2_mul(dLdG, t1);
                    const float2 u2 = f2_mul(f2_mul(gdx, make_float2(dx, dx)), dLdG);
                    const float2 u3 = f2_mul(f2_mul(gdx, dy), dLdG);
                    const float2 u4 = f2_mul(f2_mul(gdy, dy), dLdG);
                    v[0] = (u0.x + u0.y) * ddx; v[1] = (u1.x + u1.y) * ddy;
                    v[2] = -0.5f * (u2.x + u2.y); v[3] = -(u3.x + u3.y); v[4] = -0.5f * (u4.x + u4.y);
                }
                const float2 po = f2_mul(G, dLa);
                float v_op = po.x + po.y;
                // transposing butterfly: 8 values x 32 lanes -> value (lane >> 2) summed over the warp in 9 shuffles
                float u[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float send = hi16 ? v[k] : v[k + 4];
                    u[k] = (hi16 ? v[k + 4] : v[k]) + __shfl_xor_sync(0xffffffffu, send, 16);
                }
                float x2[2];
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const float send = hi8 ? u[k] : u[k + 2];
                    x2[k] = (hi8 ? u[k + 2] : u[k]) + __shfl_xor_sync(0xffffffffu, send, 8);
                }
                float x = (hi4 ? x2[1] : x2[0]) + __shfl_xor_sync(0xffffffffu, hi4 ? x2[0] : x2[1], 4);
                x += __shfl_xor_sync(0xffffffffu, x, 2);
                x += __shfl_xor_sync(0xffffffffu, x, 1);
                v_op = warp_sum_f(v_op);
                if (red_lane) {
                    const uint32_t id = sid[j];
                    atomicAdd(red_base + red_stride * id, lane == 1 ? v_op : x);
                }
                if constexpr (DEPTH) {     // the tenth value: dL/dz of the instance, added by lane 2
                    const float2 pz = f2_mul(w, dpD);
                    const float v_z = warp_sum_f(pz.x + pz.y);
                    if (lane == 2) atomicAdd(g_depth + sid[j], v_z);
                }
            }
        }
    }
}

cudaError_t launch_blend_backward(const CameraDev* cam, int grid_x, int grid_y, GeomBuffers g, BinBuffers b, ImageBuffers im,
                                  const float* dL_dcolor, float* g_mean2D, float* g_conic, float* g_opacity, float* g_rgb,
                                  int warp_cull, const float* dL_ddepth, float* g_depth, const float* dL_dalpha,
                                  cudaStream_t st) {
    if (grid_x * grid_y == 0) return cudaSuccess;
    return launch_k(dL_ddepth ? blend_backward_kernel<true> : blend_backward_kernel<false>, dim3(grid_x, grid_y), kTilePixels / 2, 0,
                    st, kOrdinary, cam, g, b.ids_sorted, b.ranges, im.final_T, im.n_contrib, dL_dcolor, g_mean2D, g_conic, g_opacity,
                    g_rgb, warp_cull, dL_ddepth, g_depth, dL_dalpha);
}

}  // namespace g4d
