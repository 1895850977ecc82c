// hexplane.cuh -- the HexPlane field (scene/hexplane.py:19-20,73-106,160-183) for every deformation kernel, forward and backward,
// FFMA and tensor-core: coordinate normalisation, border-clamped taps, the forward sample of one channel vector and its backward.
//
// Planes are channel-last [H][W][C], so one bilinear tap of a channel vector (4 channels) is one float4.  When every Gaussian
// shares t, the three time planes are collapsed once per call into 1-D rows; in the per-row mode (PER_ROW, one time per
// Gaussian) each Gaussian forms the two texels of those rows it needs on the fly, with the same arithmetic, so both modes give
// the same bits at equal times.  The functions take one level's entries of DeformDesc (planes[l], trow[l], res[l]) and the
// taps of the normalised (x, y, z) at that level, and in the per-row mode the tap of the row's t as tx[3].  The normalisation and the
// forward sample are explicit roundings (__fmul_rn / __fadd_rn, fmaf()) and single multiplies only: they round the same in the
// -fmad=false translation units as in the others, so a backward taps the very cells its forward sampled.
#pragma once
#include "g4d_common.cuh"

namespace g4d {

#if defined(__CUDACC__)

// normalize_aabb, per axis: p = (x - xyz_max) * 2 / (xyz_min - xyz_max) - 1, aabb = [xyz_max | xyz_min].
// scale[a] = dp / dx of axis a: the factor that turns dL/dp into dL/d(xyz).
struct AabbNorm {
    float amax[3], scale[3];
    G4D_D explicit AabbNorm(const float* __restrict__ aabb) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { amax[a] = __ldg(aabb + a); scale[a] = 2.0f / (__ldg(aabb + 3 + a) - amax[a]); }
    }
    // (never contracted to an FMA: a coordinate one ulp off can fall into the neighbouring texel cell)
    G4D_D float operator()(int a, float x) const { return __fadd_rn(__fmul_rn(x - amax[a], scale[a]), -1.0f); }
};

// grid_sample unnormalise (align_corners=True) + border clamp + floor (ATen grid_sampler_2d semantics).  gmul is the
// coordinate-gradient multiplier ATen uses: d(pixel)/du, 0 where the coordinate was clamped.
struct Tap1D { int i0, i1; float w0, w1, gmul; };
G4D_D Tap1D make_tap(float u, int size) {
    const float hi = (float)(size - 1);
    float x = ((u + 1.f) / 2.f) * hi;
    Tap1D t;
    t.gmul = (x > 0.f && x < hi) ? 0.5f * hi : 0.f;
    x = fminf(fmaxf(x, 0.f), hi);
    const float x0 = floorf(x);
    t.i0 = (int)x0; t.i1 = min(t.i0 + 1, size - 1);
    t.w0 = (x0 + 1.f) - x; t.w1 = x - x0;
    return t;
}

// The collapsed time row's texel from the plane's two time rows a (at ty.i0) and b (at ty.i1): the arithmetic of
// collapse_time_rows_kernel
G4D_D float4 time_lerp(float4 a, float4 b, const Tap1D& ty) {
    return make_float4(fmaf(b.x, ty.w1, a.x * ty.w0), fmaf(b.y, ty.w1, a.y * ty.w0), fmaf(b.z, ty.w1, a.z * ty.w0),
                       fmaf(b.w, ty.w1, a.w * ty.w0));
}

// The two texels r0 / r1 of the collapsed time row of plane k at the c0 taps X; PER_ROW: formed from the plane at the time
// tap ty, also handing back the four plane texels (nw, ne at ty.i0; sw, se at ty.i1) for the backward
template <bool PER_ROW>
G4D_D void time_row_texels(const float* plane, const float* trow, int W, const Tap1D& X, const Tap1D& ty, int v, int C4,
                           float4& r0, float4& r1, float4 (&q)[4]) {
    if (PER_ROW) {
        const float4* pl = reinterpret_cast<const float4*>(plane);
        q[0] = __ldg(pl + (ty.i0 * W + X.i0) * C4 + v); q[1] = __ldg(pl + (ty.i0 * W + X.i1) * C4 + v);
        q[2] = __ldg(pl + (ty.i1 * W + X.i0) * C4 + v); q[3] = __ldg(pl + (ty.i1 * W + X.i1) * C4 + v);
        r0 = time_lerp(q[0], q[2], ty); r1 = time_lerp(q[1], q[3], ty);
    } else {
        const float4* row = reinterpret_cast<const float4*>(trow);
        r0 = __ldg(row + X.i0 * C4 + v); r1 = __ldg(row + X.i1 * C4 + v);
    }
}

// One channel vector v (channels 4v .. 4v+3) of one level: the product over the 6 planes of the bilinear samples.
template <bool PER_ROW>
G4D_D float4 sample_vector(const float* const planes[6], const float* const trow[3], const int res[4],
                           const Tap1D (&tx)[PER_ROW ? 4 : 3], int v, int C4) {
    float4 prod = make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const int c0 = plane_axis0(k), c1 = plane_axis1(k);
        float4 s;
        if (c1 == 3) {   // time plane: 1-D lerp along c0 of the collapsed row
            float4 r0, r1, q[4];
            time_row_texels<PER_ROW>(planes[k], trow[c0], res[c0], tx[c0], tx[PER_ROW ? 3 : 0], v, C4, r0, r1, q);
            const float w0 = tx[c0].w0, w1 = tx[c0].w1;
            s.x = fmaf(r1.x, w1, r0.x * w0); s.y = fmaf(r1.y, w1, r0.y * w0);
            s.z = fmaf(r1.z, w1, r0.z * w0); s.w = fmaf(r1.w, w1, r0.w * w0);
        } else {
            const int W = res[c0];
            const float4* pl = reinterpret_cast<const float4*>(planes[k]);
            const Tap1D &X = tx[c0], &Y = tx[c1];
            const float4 nw = __ldg(pl + (Y.i0 * W + X.i0) * C4 + v), ne = __ldg(pl + (Y.i0 * W + X.i1) * C4 + v);
            const float4 sw = __ldg(pl + (Y.i1 * W + X.i0) * C4 + v), se = __ldg(pl + (Y.i1 * W + X.i1) * C4 + v);
            const float wnw = X.w0 * Y.w0, wne = X.w1 * Y.w0, wsw = X.w0 * Y.w1, wse = X.w1 * Y.w1;
            s.x = fmaf(se.x, wse, fmaf(sw.x, wsw, fmaf(ne.x, wne, nw.x * wnw)));
            s.y = fmaf(se.y, wse, fmaf(sw.y, wsw, fmaf(ne.y, wne, nw.y * wnw)));
            s.z = fmaf(se.z, wse, fmaf(sw.z, wsw, fmaf(ne.z, wne, nw.z * wnw)));
            s.w = fmaf(se.w, wse, fmaf(sw.w, wsw, fmaf(ne.w, wne, nw.w * wnw)));
        }
        prod.x *= s.x; prod.y *= s.y; prod.z *= s.z; prod.w *= s.w;
    }
    return prod;
}

G4D_D void red_add_v4(float* addr, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Backward of sample_vector (autograd of F.grid_sample and the plane product): scatter df = dL/d(feat[l*C + 4v .. +3]) into
// the taps of every plane (vector RED) and accumulate dL/d(normalised coordinate) into gpix.  A time plane's gradient goes to
// the collapsed rows' gradient trow_grad (2 taps), or PER_ROW straight to the plane's 2 x 2 texels of (c0 tap, time tap), and
// then dL/d(t) is accumulated into gt.
template <bool PER_ROW>
G4D_D void scatter_vector(const float* const planes[6], const float* const trow[3], const int res[4], float* const g_planes[6],
                          float* const trow_grad[3], const Tap1D (&tx)[PER_ROW ? 4 : 3], int v, int C4, float4 df, float gpix[3],
                          float& gt) {
    float4 s[6], dsx[6], dsy[6];   // sample, d(sample)/d(x_pix of c0), d/d(y_pix of c1) (PER_ROW time planes: of t_pix)
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const int c0 = plane_axis0(k), c1 = plane_axis1(k);
        if (c1 == 3) {
            float4 r0, r1, q[4];
            time_row_texels<PER_ROW>(planes[k], trow[c0], res[c0], tx[c0], tx[PER_ROW ? 3 : 0], v, C4, r0, r1, q);
            const float w0 = tx[c0].w0, w1 = tx[c0].w1;
            s[k] = make_float4(fmaf(r1.x, w1, r0.x * w0), fmaf(r1.y, w1, r0.y * w0), fmaf(r1.z, w1, r0.z * w0), fmaf(r1.w, w1, r0.w * w0));
            dsx[k] = make_float4(r1.x - r0.x, r1.y - r0.y, r1.z - r0.z, r1.w - r0.w);
            if (PER_ROW) {   // q = nw, ne, sw, se of the (c0, t) plane
                dsy[k] = make_float4((q[2].x - q[0].x) * w0 + (q[3].x - q[1].x) * w1, (q[2].y - q[0].y) * w0 + (q[3].y - q[1].y) * w1,
                                     (q[2].z - q[0].z) * w0 + (q[3].z - q[1].z) * w1, (q[2].w - q[0].w) * w0 + (q[3].w - q[1].w) * w1);
            } else {
                dsy[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        } else {
            const int W = res[c0];
            const float4* pl = reinterpret_cast<const float4*>(planes[k]);
            const Tap1D &X = tx[c0], &Y = tx[c1];
            const float4 nw = __ldg(pl + (Y.i0 * W + X.i0) * C4 + v), ne = __ldg(pl + (Y.i0 * W + X.i1) * C4 + v);
            const float4 sw = __ldg(pl + (Y.i1 * W + X.i0) * C4 + v), se = __ldg(pl + (Y.i1 * W + X.i1) * C4 + v);
            const float wnw = X.w0 * Y.w0, wne = X.w1 * Y.w0, wsw = X.w0 * Y.w1, wse = X.w1 * Y.w1;
            s[k] = make_float4(fmaf(se.x, wse, fmaf(sw.x, wsw, fmaf(ne.x, wne, nw.x * wnw))),
                               fmaf(se.y, wse, fmaf(sw.y, wsw, fmaf(ne.y, wne, nw.y * wnw))),
                               fmaf(se.z, wse, fmaf(sw.z, wsw, fmaf(ne.z, wne, nw.z * wnw))),
                               fmaf(se.w, wse, fmaf(sw.w, wsw, fmaf(ne.w, wne, nw.w * wnw))));
            dsx[k] = make_float4((ne.x - nw.x) * Y.w0 + (se.x - sw.x) * Y.w1, (ne.y - nw.y) * Y.w0 + (se.y - sw.y) * Y.w1,
                                 (ne.z - nw.z) * Y.w0 + (se.z - sw.z) * Y.w1, (ne.w - nw.w) * Y.w0 + (se.w - sw.w) * Y.w1);
            dsy[k] = make_float4((sw.x - nw.x) * X.w0 + (se.x - ne.x) * X.w1, (sw.y - nw.y) * X.w0 + (se.y - ne.y) * X.w1,
                                 (sw.z - nw.z) * X.w0 + (se.z - ne.z) * X.w1, (sw.w - nw.w) * X.w0 + (se.w - ne.w) * X.w1);
        }
    }
    float4 pre[6], suf[6];   // prefix / suffix products so that a zero sample does not poison the others
    pre[0] = make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll
    for (int k = 1; k < 6; ++k) pre[k] = make_float4(pre[k - 1].x * s[k - 1].x, pre[k - 1].y * s[k - 1].y, pre[k - 1].z * s[k - 1].z, pre[k - 1].w * s[k - 1].w);
    suf[5] = make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll
    for (int k = 4; k >= 0; --k) suf[k] = make_float4(suf[k + 1].x * s[k + 1].x, suf[k + 1].y * s[k + 1].y, suf[k + 1].z * s[k + 1].z, suf[k + 1].w * s[k + 1].w);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const int c0 = plane_axis0(k), c1 = plane_axis1(k);
        const float4 gs = make_float4(df.x * pre[k].x * suf[k].x, df.y * pre[k].y * suf[k].y, df.z * pre[k].z * suf[k].z, df.w * pre[k].w * suf[k].w);
        gpix[c0] += (gs.x * dsx[k].x + gs.y * dsx[k].y + gs.z * dsx[k].z + gs.w * dsx[k].w) * tx[c0].gmul;
        if (c1 == 3 && !PER_ROW) {
            float* row = trow_grad[c0];
            const float w0 = tx[c0].w0, w1 = tx[c0].w1;
            red_add_v4(row + (tx[c0].i0 * C4 + v) * 4, make_float4(gs.x * w0, gs.y * w0, gs.z * w0, gs.w * w0));
            red_add_v4(row + (tx[c0].i1 * C4 + v) * 4, make_float4(gs.x * w1, gs.y * w1, gs.z * w1, gs.w * w1));
        } else {
            const float gy = (gs.x * dsy[k].x + gs.y * dsy[k].y + gs.z * dsy[k].z + gs.w * dsy[k].w) * tx[c1].gmul;
            if (c1 == 3) gt += gy;
            else gpix[c1] += gy;
            const int W = res[c0];
            float* pl = g_planes[k];
            const Tap1D &X = tx[c0], &Y = tx[c1];
            const float wnw = X.w0 * Y.w0, wne = X.w1 * Y.w0, wsw = X.w0 * Y.w1, wse = X.w1 * Y.w1;
            red_add_v4(pl + ((Y.i0 * W + X.i0) * C4 + v) * 4, make_float4(gs.x * wnw, gs.y * wnw, gs.z * wnw, gs.w * wnw));
            red_add_v4(pl + ((Y.i0 * W + X.i1) * C4 + v) * 4, make_float4(gs.x * wne, gs.y * wne, gs.z * wne, gs.w * wne));
            red_add_v4(pl + ((Y.i1 * W + X.i0) * C4 + v) * 4, make_float4(gs.x * wsw, gs.y * wsw, gs.z * wsw, gs.w * wsw));
            red_add_v4(pl + ((Y.i1 * W + X.i1) * C4 + v) * 4, make_float4(gs.x * wse, gs.y * wse, gs.z * wse, gs.w * wse));
        }
    }
}

#endif  // __CUDACC__

}  // namespace g4d
