// geom_finish.cuh -- the per-Gaussian tail of the fused forward, shared by the SIMT and the tensor-core kernels:
// activations (gaussian_renderer/__init__.py:97-99) -> projection (A.1) -> SH colour -> record + saved tensors.
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

G4D_D void store_projected(const GeomBuffers& g, int64_t gi, bool ok, const Projected& pr, float opacity, const float rgb[3],
                           uint32_t bits, int32_t* out_radii) {
    note_depth_range(g, pr.tiles, pr.depth);
    g.rec0[gi] = make_float4(pr.px, pr.py, pr.conx, pr.cony);
    g.rec1[gi] = make_float4(pr.conz, ok ? opacity : 0.f, rgb[0], rgb[1]);
    g.rec2[gi] = make_float2(rgb[2], pr.depth);
    g.radii[gi] = pr.radius;
    if (out_radii) out_radii[gi] = pr.radius;
    g.rect[gi] = make_uint2((uint32_t)pr.rminx | ((uint32_t)pr.rminy << 16), (uint32_t)pr.rmaxx | ((uint32_t)pr.rmaxy << 16));
    g.tiles_touched[gi] = pr.tiles;
    g.clamped[gi] = (uint8_t)bits;
}

// p, sl (log-scale), q (raw quaternion), ol (opacity logit) already include the network's deltas.
// ShDelta: float operator()(int flat_index in [0,48)) -> delta of SH coefficient (0 when the SHS head is inactive).
template <class ShDelta>
G4D_D void fused_finish(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, const float sl[3], const float q[4], float ol,
                        ShDelta dsh) {
    const Vec3 sc{expf(sl[0]), expf(sl[1]), expf(sl[2])};
    const float qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
    const Quat rq{q[0] / qn, q[1] / qn, q[2] / qn, q[3] / qn};
    const float op = 1.f / (1.f + expf(-ol));
    Projected pr;
    const bool ok = project_gaussian(cam, p, sc, rq, pr);
    float rgb[3] = {0.f, 0.f, 0.f};
    uint32_t bits = 0;
    if (ok) {
        if (io.shs) {
            const float* sh = io.shs + gi * 48;
            sh_to_rgb(cam, p, [&](int k, int ch) { return __ldg(sh + 3 * k + ch) + dsh(3 * k + ch); }, rgb, bits);
        } else {
            const float* dc = io.sh_dc + gi * 3;
            const float* rest = io.sh_rest + gi * 45;
            sh_to_rgb(cam, p, [&](int k, int ch) {
                return (k == 0 ? __ldg(dc + ch) : __ldg(rest + 3 * (k - 1) + ch)) + dsh(3 * k + ch);
            }, rgb, bits);
        }
    }
    store_projected(io.g, gi, ok, pr, op, rgb, bits, io.out_radii);
    if (io.fo.means3D) {
        io.fo.means3D[3 * gi] = p.x; io.fo.means3D[3 * gi + 1] = p.y; io.fo.means3D[3 * gi + 2] = p.z;
        io.fo.scales[3 * gi] = sc.x; io.fo.scales[3 * gi + 1] = sc.y; io.fo.scales[3 * gi + 2] = sc.z;
        *reinterpret_cast<float4*>(io.fo.rotations + 4 * gi) = make_float4(rq.r, rq.x, rq.y, rq.z);
        io.fo.opacities[gi] = op;
        if (io.fo.rot_norm) io.fo.rot_norm[gi] = qn;
    }
}

// The same tail split over two threads of the tensor-core kernel: the M thread does activations + projection,
// the G thread the SH colour (it writes the rgb / clamp fields of the record and the deformed SH coefficients).
G4D_D void fused_finish_geometry(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, const float sl[3], const float q[4],
                                 float ol) {
    const Vec3 sc{expf(sl[0]), expf(sl[1]), expf(sl[2])};
    const float qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
    const Quat rq{q[0] / qn, q[1] / qn, q[2] / qn, q[3] / qn};
    const float op = 1.f / (1.f + expf(-ol));
    Projected pr;
    const bool ok = project_gaussian(cam, p, sc, rq, pr);
    const GeomBuffers& g = io.g;
    g.rec0[gi] = make_float4(pr.px, pr.py, pr.conx, pr.cony);
    *reinterpret_cast<float2*>(&g.rec1[gi]) = make_float2(pr.conz, ok ? op : 0.f);
    g.rec2[gi].y = pr.depth;
    g.radii[gi] = pr.radius;
    if (io.out_radii) io.out_radii[gi] = pr.radius;
    g.rect[gi] = make_uint2((uint32_t)pr.rminx | ((uint32_t)pr.rminy << 16), (uint32_t)pr.rmaxx | ((uint32_t)pr.rmaxy << 16));
    g.tiles_touched[gi] = pr.tiles;
    note_depth_range(g, pr.tiles, pr.depth);
    if (io.fo.means3D) {
        io.fo.means3D[3 * gi] = p.x; io.fo.means3D[3 * gi + 1] = p.y; io.fo.means3D[3 * gi + 2] = p.z;
        io.fo.scales[3 * gi] = sc.x; io.fo.scales[3 * gi + 1] = sc.y; io.fo.scales[3 * gi + 2] = sc.z;
        *reinterpret_cast<float4*>(io.fo.rotations + 4 * gi) = make_float4(rq.r, rq.x, rq.y, rq.z);
        io.fo.opacities[gi] = op;
        if (io.fo.rot_norm) io.fo.rot_norm[gi] = qn;
    }
}

// dsh[48]: deltas of the SH coefficients (zeros when the SHS head is inactive); indices are compile-time after
// unrolling, so dsh stays in registers.
G4D_D void fused_finish_colour(const CameraDev& cam, const DeformIO& io, int64_t gi, Vec3 p, bool hsh, const float (&dsh)[48]) {
    float sh[48];
    if (io.shs) {
#pragma unroll
        for (int j = 0; j < 48; j += 4) {
            const float4 b = __ldg(reinterpret_cast<const float4*>(io.shs + gi * 48 + j));
            sh[j] = b.x + dsh[j]; sh[j + 1] = b.y + dsh[j + 1]; sh[j + 2] = b.z + dsh[j + 2]; sh[j + 3] = b.w + dsh[j + 3];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 3; ++j) sh[j] = __ldg(io.sh_dc + gi * 3 + j) + dsh[j];
#pragma unroll
        for (int j = 0; j < 45; ++j) sh[3 + j] = __ldg(io.sh_rest + gi * 45 + j) + dsh[3 + j];
    }
    if (hsh && io.fo.shs) {
#pragma unroll
        for (int j = 0; j < 48; j += 4) *reinterpret_cast<float4*>(io.fo.shs + gi * 48 + j) = make_float4(sh[j], sh[j + 1], sh[j + 2], sh[j + 3]);
    }
    // A.1 step 10 with every coefficient index resolved at compile time
    float dx = p.x - cam.campos[0], dy = p.y - cam.campos[1], dz = p.z - cam.campos[2];
    const float len = sqrtf(dx * dx + dy * dy + dz * dz);
    dx = dx / len; dy = dy / len; dz = dz / len;
    float bas[16];
    sh_basis(3, dx, dy, dz, bas);
    const int deg = cam.sh_degree;
    uint32_t bits = 0;
    float rgb[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float acc = bas[0] * sh[ch];
#pragma unroll
        for (int k = 1; k < 16; ++k)
            if (k < (deg + 1) * (deg + 1)) acc = acc + bas[k] * sh[3 * k + ch];
        acc = acc + 0.5f;
        if (acc < 0.f) bits |= (1u << ch);
        rgb[ch] = fmaxf_(acc, 0.f);
    }
    const GeomBuffers& g = io.g;
    *reinterpret_cast<float2*>(reinterpret_cast<float*>(&g.rec1[gi]) + 2) = make_float2(rgb[0], rgb[1]);
    g.rec2[gi].x = rgb[2];
    g.clamped[gi] = (uint8_t)bits;
}

}  // namespace g4d
