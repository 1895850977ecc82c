// g4d_math.cuh -- per-Gaussian projection math (forward and backward), host+device.
//
// Forward follows SURVEY.md Appendix A.1 operation by operation; the translation unit that includes this
// for the forward kernels is compiled with -fmad=false so that depth bits, radii and tile rects are
// reproducible bit-for-bit from the same fp32 expression trees (explicit fmaf() is used where fusion is
// wanted).  Reference call site: /root/reference/gaussian_renderer/__init__.py:120-128.
#pragma once
#include <math.h>

#include "g4d_common.cuh"

namespace g4d {

struct Vec3 { float x, y, z; };
struct Quat { float r, x, y, z; };

G4D_HD float fminf_(float a, float b) { return a < b ? a : b; }
G4D_HD float fmaxf_(float a, float b) { return a > b ? a : b; }
G4D_HD int imin_(int a, int b) { return a < b ? a : b; }
G4D_HD int imax_(int a, int b) { return a > b ? a : b; }

G4D_HD int f2i_sat(float f) {
#if defined(__CUDA_ARCH__)
    return __float2int_rz(f);  // saturating, NaN -> 0
#else
    if (!(f == f)) return 0;
    if (f >= 2147483520.f) return 2147483647;
    if (f <= -2147483648.f) return (-2147483647 - 1);
    return (int)f;
#endif
}

G4D_HD Vec3 xform4x3(const float* m, Vec3 p) {
    Vec3 o;
    o.x = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
    o.y = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
    o.z = m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14];
    return o;
}

G4D_HD void quat_to_rot(Quat q, float R[9]) {
    float r = q.r, x = q.x, y = q.y, z = q.z;
    R[0] = 1.f - 2.f * (y * y + z * z);
    R[1] = 2.f * (x * y - r * z);
    R[2] = 2.f * (x * z + r * y);
    R[3] = 2.f * (x * y + r * z);
    R[4] = 1.f - 2.f * (x * x + z * z);
    R[5] = 2.f * (y * z - r * x);
    R[6] = 2.f * (x * z - r * y);
    R[7] = 2.f * (y * z + r * x);
    R[8] = 1.f - 2.f * (x * x + y * y);
}

// Sigma = R S S^T R^T, output (xx, xy, xz, yy, yz, zz)   (general_utils.py:84-116, gaussian_model.py:30-34)
G4D_HD void cov3d_from_scale_rot(Vec3 scale, float mod, Quat q, float c[6]) {
    float R[9], M[9];
    quat_to_rot(q, R);
    float s[3] = {mod * scale.x, mod * scale.y, mod * scale.z};
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) M[k * 3 + j] = s[k] * R[j * 3 + k];
    c[0] = M[0] * M[0] + M[3] * M[3] + M[6] * M[6];
    c[1] = M[0] * M[1] + M[3] * M[4] + M[6] * M[7];
    c[2] = M[0] * M[2] + M[3] * M[5] + M[6] * M[8];
    c[3] = M[1] * M[1] + M[4] * M[4] + M[7] * M[7];
    c[4] = M[1] * M[2] + M[4] * M[5] + M[7] * M[8];
    c[5] = M[2] * M[2] + M[5] * M[5] + M[8] * M[8];
}

struct Cov2DAux {
    float T0[3], T1[3];   // rows of T = J W
    float cov2[3];        // (a, b, c) before dilation
    float tx, ty, tz;     // guard-band clamped view-space point
    bool clampx, clampy;
};

G4D_HD void cov2d_project(const CameraDev& cam, Vec3 pv, const float cov3[6], Cov2DAux& o) {
    const float* v = cam.view;
    float limx = kGuardBand * cam.tanfovx, limy = kGuardBand * cam.tanfovy;
    float tz = pv.z;
    float txtz = pv.x / tz, tytz = pv.y / tz;
    o.clampx = (txtz < -limx) || (txtz > limx);
    o.clampy = (tytz < -limy) || (tytz > limy);
    float tx = fminf_(limx, fmaxf_(-limx, txtz)) * tz;
    float ty = fminf_(limy, fmaxf_(-limy, tytz)) * tz;
    o.tx = tx; o.ty = ty; o.tz = tz;
    float fx = cam.focal_x, fy = cam.focal_y;
    float j00 = fx / tz, j02 = -(fx * tx) / (tz * tz);
    float j11 = fy / tz, j12 = -(fy * ty) / (tz * tz);
    o.T0[0] = j00 * v[0] + j02 * v[2];
    o.T0[1] = j00 * v[4] + j02 * v[6];
    o.T0[2] = j00 * v[8] + j02 * v[10];
    o.T1[0] = j11 * v[1] + j12 * v[2];
    o.T1[1] = j11 * v[5] + j12 * v[6];
    o.T1[2] = j11 * v[9] + j12 * v[10];
    const float* T0 = o.T0; const float* T1 = o.T1;
    float u0 = cov3[0] * T0[0] + cov3[1] * T0[1] + cov3[2] * T0[2];
    float u1 = cov3[1] * T0[0] + cov3[3] * T0[1] + cov3[4] * T0[2];
    float u2 = cov3[2] * T0[0] + cov3[4] * T0[1] + cov3[5] * T0[2];
    float w0 = cov3[0] * T1[0] + cov3[1] * T1[1] + cov3[2] * T1[2];
    float w1 = cov3[1] * T1[0] + cov3[3] * T1[1] + cov3[4] * T1[2];
    float w2 = cov3[2] * T1[0] + cov3[4] * T1[1] + cov3[5] * T1[2];
    o.cov2[0] = T0[0] * u0 + T0[1] * u1 + T0[2] * u2;
    o.cov2[1] = T0[0] * w0 + T0[1] * w1 + T0[2] * w2;
    o.cov2[2] = T1[0] * w0 + T1[1] * w1 + T1[2] * w2;
}

G4D_HD void sh_basis(int deg, float x, float y, float z, float b[16]) {
    b[0] = kSH0;
    if (deg > 0) {
        b[1] = -kSH1 * y; b[2] = kSH1 * z; b[3] = -kSH1 * x;
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            b[4] = G4D_SH2_0 * xy; b[5] = G4D_SH2_1 * yz; b[6] = G4D_SH2_2 * (2.f * zz - xx - yy);
            b[7] = G4D_SH2_3 * xz; b[8] = G4D_SH2_4 * (xx - yy);
            if (deg > 2) {
                b[9] = G4D_SH3_0 * y * (3.f * xx - yy);
                b[10] = G4D_SH3_1 * xy * z;
                b[11] = G4D_SH3_2 * y * (4.f * zz - xx - yy);
                b[12] = G4D_SH3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy);
                b[13] = G4D_SH3_4 * x * (4.f * zz - xx - yy);
                b[14] = G4D_SH3_5 * z * (xx - yy);
                b[15] = G4D_SH3_6 * x * (xx - 3.f * yy);
            }
        }
    }
}

struct Projected {
    float depth, px, py;
    float conx, cony, conz;
    int radius;
    int rminx, rminy, rmaxx, rmaxy;
    uint32_t tiles;
};

// A.1 steps 2-9 (everything except colour).  Returns false when the Gaussian is culled (all outputs zero).
G4D_HD bool project_gaussian(const CameraDev& cam, Vec3 p, Vec3 scale, Quat rot, Projected& o) {
    o.depth = 0.f; o.px = 0.f; o.py = 0.f; o.conx = o.cony = o.conz = 0.f; o.radius = 0;
    o.rminx = o.rminy = o.rmaxx = o.rmaxy = 0; o.tiles = 0;
    Vec3 pv = xform4x3(cam.view, p);
    if (pv.z <= kNearCull) return false;
    const float* m = cam.proj;
    float hx = m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12];
    float hy = m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13];
    float hw = m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15];
    float pw = 1.0f / (hw + kWEps);
    float ndcx = hx * pw, ndcy = hy * pw;
    float c3[6];
    cov3d_from_scale_rot(scale, cam.scale_modifier, rot, c3);
    Cov2DAux aux;
    cov2d_project(cam, pv, c3, aux);
    float a = aux.cov2[0] + kDilation, b = aux.cov2[1], c = aux.cov2[2] + kDilation;
    float det = a * c - b * b;
    if (det == 0.0f) return false;
    float det_inv = 1.f / det;
    float mid = 0.5f * (a + c);
    float root = sqrtf(fmaxf_(kMinDiscriminant, mid * mid - det));
    float lam1 = mid + root, lam2 = mid - root;
    float rad = ceilf(3.f * sqrtf(fmaxf_(lam1, lam2)));
    float px = ((ndcx + 1.0f) * (float)cam.W - 1.0f) * 0.5f;
    float py = ((ndcy + 1.0f) * (float)cam.H - 1.0f) * 0.5f;
    int rminx = imin_(cam.grid_x, imax_(0, f2i_sat((px - rad) / (float)kTile)));
    int rminy = imin_(cam.grid_y, imax_(0, f2i_sat((py - rad) / (float)kTile)));
    int rmaxx = imin_(cam.grid_x, imax_(0, f2i_sat((px + rad + (float)(kTile - 1)) / (float)kTile)));
    int rmaxy = imin_(cam.grid_y, imax_(0, f2i_sat((py + rad + (float)(kTile - 1)) / (float)kTile)));
    int area = (rmaxx - rminx) * (rmaxy - rminy);
    if (area == 0) return false;
    o.depth = pv.z; o.px = px; o.py = py;
    o.conx = c * det_inv; o.cony = -b * det_inv; o.conz = a * det_inv;
    o.radius = f2i_sat(rad);
    o.rminx = rminx; o.rminy = rminy; o.rmaxx = rmaxx; o.rmaxy = rmaxy;
    o.tiles = (uint32_t)area;
    return true;
}

// A.1 step 10.  ShLoad: float operator()(int coeff, int channel).  UNROLL, for a loader that reads a register array: the loop
// runs to the constant 16 under the degree mask, so the compiler unrolls it and every coefficient index is a compile-time
// constant (the full basis is computed, without branches).  Otherwise, for a loader that reads memory, the loop runs to the
// camera's coefficient count and keeps the basis in a local array: fewer live registers.  The sums are the same either way.
template <bool UNROLL = false, class ShLoad>
G4D_HD void sh_to_rgb(const CameraDev& cam, Vec3 p, ShLoad sh, float rgb[3], uint32_t& clamped_bits) {
    float dx = p.x - cam.campos[0], dy = p.y - cam.campos[1], dz = p.z - cam.campos[2];
    float len = sqrtf(dx * dx + dy * dy + dz * dz);
    dx = dx / len; dy = dy / len; dz = dz / len;
    float bas[16];
    sh_basis(UNROLL ? 3 : cam.sh_degree, dx, dy, dz, bas);
    const int ncoef = (cam.sh_degree + 1) * (cam.sh_degree + 1);
    clamped_bits = 0;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        float acc = bas[0] * sh(0, ch);
        for (int k = 1; k < (UNROLL ? 16 : ncoef); ++k)
            if (k < ncoef) acc = acc + bas[k] * sh(k, ch);
        acc = acc + 0.5f;
        if (acc < 0.f) clamped_bits |= (1u << ch);
        rgb[ch] = fmaxf_(acc, 0.f);
    }
}

// ------------------------------------------------------------------------------------------------
// Backward of the per-Gaussian stage (A.4): from (g_mean2D[NDC units], g_conic, g_rgb) to gradients of
// mean3D, scale (post-activation), quaternion (as given) and SH coefficients.
// g_conic holds TRUE derivatives w.r.t. (conic.x, conic.y, conic.z).
// ------------------------------------------------------------------------------------------------
struct GaussGrad {
    float mean[3];
    float scale[3];
    float rot[4];
};

// d(basis_k)/d(x,y,z) contracted with s_k = sum_ch sh(k,ch)*gc[ch]; returns dL/d(dir)
template <class ShLoad>
G4D_HD void sh_dir_grad(int deg, float x, float y, float z, ShLoad sh, const float gc[3], float gdir[3]) {
    gdir[0] = gdir[1] = gdir[2] = 0.f;
    if (deg < 1) return;
    auto S = [&](int k) { return sh(k, 0) * gc[0] + sh(k, 1) * gc[1] + sh(k, 2) * gc[2]; };
    float s;
    s = S(1); gdir[1] += -kSH1 * s;
    s = S(2); gdir[2] += kSH1 * s;
    s = S(3); gdir[0] += -kSH1 * s;
    if (deg < 2) return;
    s = S(4); gdir[0] += G4D_SH2_0 * y * s; gdir[1] += G4D_SH2_0 * x * s;
    s = S(5); gdir[1] += G4D_SH2_1 * z * s; gdir[2] += G4D_SH2_1 * y * s;
    s = S(6); gdir[0] += G4D_SH2_2 * -2.f * x * s; gdir[1] += G4D_SH2_2 * -2.f * y * s; gdir[2] += G4D_SH2_2 * 4.f * z * s;
    s = S(7); gdir[0] += G4D_SH2_3 * z * s; gdir[2] += G4D_SH2_3 * x * s;
    s = S(8); gdir[0] += G4D_SH2_4 * 2.f * x * s; gdir[1] += G4D_SH2_4 * -2.f * y * s;
    if (deg < 3) return;
    float xx = x * x, yy = y * y, zz = z * z;
    s = S(9); gdir[0] += G4D_SH3_0 * 6.f * x * y * s; gdir[1] += G4D_SH3_0 * (3.f * xx - 3.f * yy) * s;
    s = S(10); gdir[0] += G4D_SH3_1 * y * z * s; gdir[1] += G4D_SH3_1 * x * z * s; gdir[2] += G4D_SH3_1 * x * y * s;
    s = S(11); gdir[0] += G4D_SH3_2 * -2.f * x * y * s; gdir[1] += G4D_SH3_2 * (4.f * zz - xx - 3.f * yy) * s;
    gdir[2] += G4D_SH3_2 * 8.f * y * z * s;
    s = S(12); gdir[0] += G4D_SH3_3 * -6.f * x * z * s; gdir[1] += G4D_SH3_3 * -6.f * y * z * s;
    gdir[2] += G4D_SH3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * s;
    s = S(13); gdir[0] += G4D_SH3_4 * (4.f * zz - 3.f * xx - yy) * s; gdir[1] += G4D_SH3_4 * -2.f * x * y * s;
    gdir[2] += G4D_SH3_4 * 8.f * x * z * s;
    s = S(14); gdir[0] += G4D_SH3_5 * 2.f * x * z * s; gdir[1] += G4D_SH3_5 * -2.f * y * z * s;
    gdir[2] += G4D_SH3_5 * (xx - yy) * s;
    s = S(15); gdir[0] += G4D_SH3_6 * (3.f * xx - 3.f * yy) * s; gdir[1] += G4D_SH3_6 * -6.f * x * y * s;
}

// Rounded product and sum that the compiler may neither contract into an FMA nor merge with the contractable arithmetic
// around them (mul.rn / add.rn): the camera terms of gaussian_backward use only these, so that computing them adds no use
// to a product of the per-Gaussian gradients and leaves those gradients' own contractions -- and bits -- as they were.
G4D_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
G4D_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

// The camera side of one Gaussian's backward: dL/d view [16], proj [16], campos [3], each in the element order of the
// caller's tensor (cam.view[i] is element i of the flattened world_view_transform).  Elements the forward never reads --
// view 3, 7, 11, 15 (xform4x3 uses rows 0..2) and proj 2, 6, 10, 14 (the clip-space z row) -- are zero.
struct CamGrad { float g[kCamGradFloats]; };
G4D_HD constexpr bool cam_grad_read(int i) { return i < 16 ? (i & 3) != 3 : i < 32 ? (i & 3) != 2 : true; }

// ShLoad as above; ShStore: void operator()(int coeff, int channel, float grad).  CAM: also the camera terms, into *cg
// (every element written), in mul_rn / add_rn only: the GaussGrad outputs are those of CAM = false bit for bit.
template <bool CAM = false, class ShLoad, class ShStore>
G4D_HD void gaussian_backward(const CameraDev& cam, Vec3 p, Vec3 scale, Quat rot, uint32_t clamped_bits,
                              const float g_mean2D[2], const float g_conic[3], const float g_rgb[3], ShLoad sh,
                              ShStore sh_store, GaussGrad& out, CamGrad* cg = nullptr) {
    const float* v = cam.view;
    const float* pm = cam.proj;
    float gm[3] = {0.f, 0.f, 0.f};
    // (1) conic -> cov2D -> (Sigma, T)
    Vec3 pv = xform4x3(v, p);
    float c3[6];
    cov3d_from_scale_rot(scale, cam.scale_modifier, rot, c3);
    Cov2DAux ax;
    cov2d_project(cam, pv, c3, ax);
    float a = ax.cov2[0] + kDilation, b = ax.cov2[1], c = ax.cov2[2] + kDilation;
    float det = a * c - b * b;
    float d2inv = 1.f / (det * det + kDet2Eps);
    float gcx = g_conic[0], gcy = g_conic[1], gcz = g_conic[2];
    float dL_da = d2inv * (-c * c * gcx + b * c * gcy + (det - a * c) * gcz);
    float dL_dc = d2inv * (-a * a * gcz + a * b * gcy + (det - a * c) * gcx);
    float dL_db = d2inv * (2.f * b * c * gcx - (det + 2.f * b * b) * gcy + 2.f * a * b * gcz);
    const float* t0 = ax.T0; const float* t1 = ax.T1;
    float gS[3][3];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int k = 0; k < 3; ++k)
            gS[j][k] = dL_da * t0[j] * t0[k] + dL_dc * t1[j] * t1[k] + 0.5f * dL_db * (t0[j] * t1[k] + t1[j] * t0[k]);
    float S3[3][3] = {{c3[0], c3[1], c3[2]}, {c3[1], c3[3], c3[4]}, {c3[2], c3[4], c3[5]}};
    float gT0[3], gT1[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float s0 = S3[j][0] * t0[0] + S3[j][1] * t0[1] + S3[j][2] * t0[2];
        float s1 = S3[j][0] * t1[0] + S3[j][1] * t1[1] + S3[j][2] * t1[2];
        gT0[j] = 2.f * dL_da * s0 + dL_db * s1;
        gT1[j] = 2.f * dL_dc * s1 + dL_db * s0;
    }
    float Wr[3][3] = {{v[0], v[4], v[8]}, {v[1], v[5], v[9]}, {v[2], v[6], v[10]}};
    float gJ00 = 0.f, gJ02 = 0.f, gJ11 = 0.f, gJ12 = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        gJ00 += Wr[0][j] * gT0[j]; gJ02 += Wr[2][j] * gT0[j];
        gJ11 += Wr[1][j] * gT1[j]; gJ12 += Wr[2][j] * gT1[j];
    }
    float fx = cam.focal_x, fy = cam.focal_y;
    float itz = 1.f / ax.tz, itz2 = itz * itz, itz3 = itz2 * itz;
    float gtx = ax.clampx ? 0.f : -fx * itz2 * gJ02;
    float gty = ax.clampy ? 0.f : -fy * itz2 * gJ12;
    float gtz = -fx * itz2 * gJ00 - fy * itz2 * gJ11 + (2.f * fx * ax.tx) * itz3 * gJ02 + (2.f * fy * ax.ty) * itz3 * gJ12;
    gm[0] += Wr[0][0] * gtx + Wr[1][0] * gty + Wr[2][0] * gtz;
    gm[1] += Wr[0][1] * gtx + Wr[1][1] * gty + Wr[2][1] * gtz;
    gm[2] += Wr[0][2] * gtx + Wr[1][2] * gty + Wr[2][2] * gtz;
    if constexpr (CAM) {
        // view: p_view = W p + t, so dL/d view[4c + r] = dL/d p_view[r] * [p, 1][c]; and T = J W, so the rows of W get J^T gT
        // (J: cov2d_project's j00, j02, j11, j12 at the clamped point)
        float* gv = cg->g;
        const float gp[3] = {gtx, gty, gtz};
        const float j00 = mul_rn(fx, itz), j02 = -mul_rn(mul_rn(fx, ax.tx), itz2);
        const float j11 = mul_rn(fy, itz), j12 = -mul_rn(mul_rn(fy, ax.ty), itz2);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            gv[r] = mul_rn(gp[r], p.x); gv[4 + r] = mul_rn(gp[r], p.y); gv[8 + r] = mul_rn(gp[r], p.z); gv[12 + r] = gp[r];
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            gv[4 * j] = add_rn(gv[4 * j], mul_rn(j00, gT0[j]));
            gv[4 * j + 1] = add_rn(gv[4 * j + 1], mul_rn(j11, gT1[j]));
            gv[4 * j + 2] = add_rn(gv[4 * j + 2], add_rn(mul_rn(j02, gT0[j]), mul_rn(j12, gT1[j])));
            gv[4 * j + 3] = 0.f;
        }
        gv[15] = 0.f;
    }
    // (2) mean2D (NDC units) -> mean3D through the projective divide
    {
        float hx = pm[0] * p.x + pm[4] * p.y + pm[8] * p.z + pm[12];
        float hy = pm[1] * p.x + pm[5] * p.y + pm[9] * p.z + pm[13];
        float hw = pm[3] * p.x + pm[7] * p.y + pm[11] * p.z + pm[15];
        float mw = 1.f / (hw + kWEps);
        float mul1 = hx * mw * mw, mul2 = hy * mw * mw;
        float g0 = g_mean2D[0], g1 = g_mean2D[1];
        gm[0] += (pm[0] * mw - pm[3] * mul1) * g0 + (pm[1] * mw - pm[3] * mul2) * g1;
        gm[1] += (pm[4] * mw - pm[7] * mul1) * g0 + (pm[5] * mw - pm[7] * mul2) * g1;
        gm[2] += (pm[8] * mw - pm[11] * mul1) * g0 + (pm[9] * mw - pm[11] * mul2) * g1;
        if constexpr (CAM) {
            // ndc = (hx, hy) / (hw + eps) with h = proj [p, 1]: dL/d proj[4c + r] = dL/dh[r] * [p, 1][c], r = x, y, w
            float* gp = cg->g + 16;
            const float ghx = mul_rn(g0, mw), ghy = mul_rn(g1, mw), ghw = -add_rn(mul_rn(g0, mul1), mul_rn(g1, mul2));
            const float ph[3] = {p.x, p.y, p.z};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                gp[4 * c] = mul_rn(ghx, ph[c]); gp[4 * c + 1] = mul_rn(ghy, ph[c]); gp[4 * c + 2] = 0.f;
                gp[4 * c + 3] = mul_rn(ghw, ph[c]);
            }
            gp[12] = ghx; gp[13] = ghy; gp[14] = 0.f; gp[15] = ghw;
        }
    }
    // (3) colour -> SH coefficients and view direction
    {
        float d0 = p.x - cam.campos[0], d1 = p.y - cam.campos[1], d2 = p.z - cam.campos[2];
        float len = sqrtf(d0 * d0 + d1 * d1 + d2 * d2);
        float ilen = 1.f / len;
        float x = d0 * ilen, y = d1 * ilen, z = d2 * ilen;
        float bas[16];
        sh_basis(cam.sh_degree, x, y, z, bas);
        float gc[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) gc[ch] = ((clamped_bits >> ch) & 1u) ? 0.f : g_rgb[ch];
        const int ncoef = (cam.sh_degree + 1) * (cam.sh_degree + 1);
        for (int k = 0; k < kShCoeffs; ++k)
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) sh_store(k, ch, k < ncoef ? bas[k] * gc[ch] : 0.f);
        float gdir[3];
        sh_dir_grad(cam.sh_degree, x, y, z, sh, gc, gdir);
        float dot = x * gdir[0] + y * gdir[1] + z * gdir[2];
        gm[0] += (gdir[0] - x * dot) * ilen;
        gm[1] += (gdir[1] - y * dot) * ilen;
        gm[2] += (gdir[2] - z * dot) * ilen;
        if constexpr (CAM) {   // the direction is p - campos: campos gets the negated mean term, (dir * dot - gdir) / len
            cg->g[32] = mul_rn(add_rn(mul_rn(x, dot), -gdir[0]), ilen);
            cg->g[33] = mul_rn(add_rn(mul_rn(y, dot), -gdir[1]), ilen);
            cg->g[34] = mul_rn(add_rn(mul_rn(z, dot), -gdir[2]), ilen);
        }
    }
    out.mean[0] = gm[0]; out.mean[1] = gm[1]; out.mean[2] = gm[2];
    // (4) Sigma -> scale, quaternion
    {
        float Rf[9];
        quat_to_rot(rot, Rf);
        float mod = cam.scale_modifier;
        float s[3] = {mod * scale.x, mod * scale.y, mod * scale.z};
        float gR[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float q = 0.f;
#pragma unroll
            for (int a_ = 0; a_ < 3; ++a_)
#pragma unroll
                for (int b_ = 0; b_ < 3; ++b_) q += Rf[a_ * 3 + k] * gS[a_][b_] * Rf[b_ * 3 + k];
            out.scale[k] = 2.f * s[k] * q * mod;
        }
#pragma unroll
        for (int a_ = 0; a_ < 3; ++a_)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float q = 0.f;
#pragma unroll
                for (int b_ = 0; b_ < 3; ++b_) q += gS[a_][b_] * Rf[b_ * 3 + k];
                gR[a_][k] = 2.f * q * s[k] * s[k];
            }
        float r = rot.r, x = rot.x, y = rot.y, z = rot.z;
        out.rot[0] = 2.f * (-z * gR[0][1] + y * gR[0][2] + z * gR[1][0] - x * gR[1][2] - y * gR[2][0] + x * gR[2][1]);
        out.rot[1] = 2.f * (y * gR[0][1] + z * gR[0][2] + y * gR[1][0] - 2.f * x * gR[1][1] - r * gR[1][2] + z * gR[2][0] +
                            r * gR[2][1] - 2.f * x * gR[2][2]);
        out.rot[2] = 2.f * (-2.f * y * gR[0][0] + x * gR[0][1] + r * gR[0][2] + x * gR[1][0] + z * gR[1][2] - r * gR[2][0] +
                            z * gR[2][1] - 2.f * y * gR[2][2]);
        out.rot[3] = 2.f * (-2.f * z * gR[0][0] - r * gR[0][1] + x * gR[0][2] + r * gR[1][0] - 2.f * z * gR[1][1] +
                            y * gR[1][2] + x * gR[2][0] + y * gR[2][1]);
    }
}

}  // namespace g4d
