// geom_finish.cuh -- the per-Gaussian tail of the fused forward, shared by the SIMT and the tensor-core kernels and the coarse
// stage: activations (gaussian_renderer/__init__.py:97-99) -> projection (A.1) -> SH colour -> record + saved tensors.
// Included only by translation units compiled with -fmad=false (see g4d_math.cuh).
#pragma once
#include "g4d_internal.h"
#include "g4d_math.cuh"

namespace g4d {

// depth range of the visible Gaussians for the binning sort (keys are sorted as bits - min: fewer radix passes).  One RED
// pair per warp: the lanes that reach this point reduce among themselves first.
G4D_D void note_depth_range(const GeomBuffers& g, uint32_t tiles, float depth) {
    const unsigned m = __activemask();
    const uint32_t k = __float_as_uint(depth);
    const uint32_t lo = __reduce_min_sync(m, tiles ? k : 0xFFFFFFFFu), hi = __reduce_max_sync(m, tiles ? k : 0u);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(m) - 1) && lo <= hi) { atomicMin(g.depth_range, lo); atomicMax(g.depth_range + 1, hi); }
}

// the colour-independent fields of the record: rec0, radii, rect, tiles_touched
G4D_D void store_geometry(const GeomBuffers& g, int64_t gi, const Projected& pr, int32_t* out_radii) {
    note_depth_range(g, pr.tiles, pr.depth);
    g.rec0[gi] = make_float4(pr.px, pr.py, pr.conx, pr.cony);
    g.radii[gi] = pr.radius;
    if (out_radii) out_radii[gi] = pr.radius;
    g.rect[gi] = make_uint2((uint32_t)pr.rminx | ((uint32_t)pr.rminy << 16), (uint32_t)pr.rmaxx | ((uint32_t)pr.rmaxy << 16));
    g.tiles_touched[gi] = pr.tiles;
}

G4D_D void store_projected(const GeomBuffers& g, int64_t gi, bool ok, const Projected& pr, float opacity, const float rgb[3],
                           uint32_t bits, int32_t* out_radii) {
    store_geometry(g, gi, pr, out_radii);
    g.rec1[gi] = make_float4(pr.conz, ok ? opacity : 0.f, rgb[0], rgb[1]);
    g.rec2[gi] = make_float2(rgb[2], pr.depth);
    g.clamped[gi] = (uint8_t)bits;
}

// exp / F.normalize / sigmoid of the log-scale sl, raw quaternion q and opacity logit ol; qn is |q| before the normalisation
struct Activated { Vec3 sc; Quat rq; float qn, op; };
G4D_D Activated activate(const float sl[3], const float q[4], float ol) {
    Activated a;
    a.sc = Vec3{expf(sl[0]), expf(sl[1]), expf(sl[2])};
    a.qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
    a.rq = Quat{q[0] / a.qn, q[1] / a.qn, q[2] / a.qn, q[3] / a.qn};
    a.op = 1.f / (1.f + expf(-ol));
    return a;
}

// the activated tensors the backward reads (not stored when fo.means3D is NULL: a no-grad forward)
G4D_D void store_saved(const FusedOutputs& fo, int64_t gi, Vec3 p, const Activated& a) {
    if (!fo.means3D) return;
    fo.means3D[3 * gi] = p.x; fo.means3D[3 * gi + 1] = p.y; fo.means3D[3 * gi + 2] = p.z;
    fo.scales[3 * gi] = a.sc.x; fo.scales[3 * gi + 1] = a.sc.y; fo.scales[3 * gi + 2] = a.sc.z;
    *reinterpret_cast<float4*>(fo.rotations + 4 * gi) = make_float4(a.rq.r, a.rq.x, a.rq.y, a.rq.z);
    fo.opacities[gi] = a.op;
    if (fo.rot_norm) fo.rot_norm[gi] = a.qn;
}

// p, sl (log-scale), q (raw quaternion), ol (opacity logit) already include the network's deltas.
// ShDelta: float operator()(int flat_index in [0,48)) -> delta of SH coefficient (0 when the SHS head is inactive).
// FULL: io.sh holds M = 16 coefficients, known at compile time (constant strides); else M = io.sh.m.
template <bool FULL, class ShDelta>
G4D_D void fused_finish(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, const float sl[3], const float q[4], float ol,
                        ShDelta dsh) {
    const Activated a = activate(sl, q, ol);
    Projected pr;
    const bool ok = project_gaussian(cam, p, a.sc, a.rq, pr);
    float rgb[3] = {0.f, 0.f, 0.f};
    uint32_t bits = 0;
    if (ok)
        io.sh.with_coeffs<FULL>(gi, [&](auto sh) {
            sh_to_rgb(cam, p, [&](int k, int ch) { return sh(k, ch) + dsh(3 * k + ch); }, rgb, bits);
        });
    store_projected(io.g, gi, ok, pr, a.op, rgb, bits, io.out_radii);
    store_saved(io.fo, gi, p, a);
}

// The same tail split over two threads of the tensor-core kernel: the M thread does activations + projection,
// the G thread the SH colour (it writes the rgb / clamp fields of the record and the deformed SH coefficients).
// The G thread does not know whether the Gaussian was culled: it writes the evaluated colour either way.
G4D_D void fused_finish_geometry(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, const float sl[3], const float q[4],
                                 float ol) {
    const Activated a = activate(sl, q, ol);
    Projected pr;
    const bool ok = project_gaussian(cam, p, a.sc, a.rq, pr);
    const GeomBuffers& g = io.g;
    store_geometry(g, gi, pr, io.out_radii);
    *reinterpret_cast<float2*>(&g.rec1[gi]) = make_float2(pr.conz, ok ? a.op : 0.f);
    g.rec2[gi].y = pr.depth;
    store_saved(io.fo, gi, p, a);
}

// the colour fields of the record (rec1.zw, rec2.x, clamped)
G4D_D void store_colour(const GeomBuffers& g, int64_t gi, const float rgb[3], uint32_t bits) {
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(&g.rec1[gi]) + 2) = make_float2(rgb[0], rgb[1]);
    g.rec2[gi].x = rgb[2];
    g.clamped[gi] = (uint8_t)bits;
}

// dsh[48]: deltas of the SH coefficients (zeros when the SHS head is inactive); indices are compile-time after
// unrolling, so dsh stays in registers.  M = 16 coefficients per Gaussian.
G4D_D void fused_finish_colour(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, bool hsh, const float (&dsh)[48]) {
    float sh[48];
    io.sh.load(gi, sh);
#pragma unroll
    for (int j = 0; j < 48; ++j) sh[j] = sh[j] + dsh[j];
    if (hsh && io.fo.shs) {
#pragma unroll
        for (int j = 0; j < 48; j += 4) *reinterpret_cast<float4*>(io.fo.shs + gi * 48 + j) = make_float4(sh[j], sh[j + 1], sh[j + 2], sh[j + 3]);
    }
    float rgb[3];
    uint32_t bits;
    sh_to_rgb<true>(cam, p, [&](int k, int ch) { return sh[3 * k + ch]; }, rgb, bits);
    store_colour(io.g, gi, rgb, bits);
}

// The same for a model with M = io.sh.m < 16 coefficients (no SHS head, so no deltas): read from memory, M at run time.
G4D_D void fused_finish_colour_reduced(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p) {
    float rgb[3];
    uint32_t bits;
    io.sh.with_coeffs<false>(gi, [&](auto sh) { sh_to_rgb(cam, p, sh, rgb, bits); });
    store_colour(io.g, gi, rgb, bits);
}

}  // namespace g4d
