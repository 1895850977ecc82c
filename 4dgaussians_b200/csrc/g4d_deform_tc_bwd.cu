// g4d_deform_tc_bwd.cu -- tensor-core backward of the deformation network (net_width 128), two wgmma kernels (tc_wgmma.cuh):
//
//  A  "dgrad":  a CTA owns a tile of 128 Gaussians per pass, one warpgroup per 64 of them, persistent over tiles.
//               Recomputes the forward activations with BF16x2 MMAs (hi + lo parts, 3 products, fp32 accumulate: ~16
//               mantissa bits), forms dz per head in the epilogue (the <= 4-wide heads' layer-2 dgrad in fp32, the SH head's
//               as a GEMM with K = 48), accumulates d(a1) over the heads in registers with one GEMM per head (W1 read
//               MN-major), then d(feat) = dh W0 -> [N][F] fp32.  Every A operand is a register fragment built from the
//               previous accumulator (tc_wgmma.cuh); W1 images stream through a two-slot TMA ring, one head ahead.  The ReLU
//               signs come from the bits the forward saved (G4D_RELU_BITS_WORDS), so this is the gradient of the forward
//               that ran.  Everything the weight gradients need is written ONCE to global memory as ready-to-use MMA operand
//               images (8x8 bf16 core-matrix layout) so that kernel B is pure TMA + MMA.
//               The HexPlane gather before it and the scatter after it are the ones every backward runs
//               (launch_deform_backward, g4d_backward.cu).
//  B  "wgrad":  dW1_h = DZ_h^T A1, dW2_h^T = A2_h^T DOUT_h, db1_h = DZ_h^T 1, db2_h = 1^T DOUT_h, dW0 = DH^T FEAT, db0 = DH^T 1
//               as split-K GEMMs over the Gaussian index (operands MN-major straight from the images), accumulators in
//               registers across the CTA's tiles (warpgroup w: output rows [64 w, 64 w + 64)), one atomic flush per CTA;
//               two half-tile smem stages pipeline the TMA loads against the MMAs.
//
// Replaces the autograd backward of scene/deformation.py:67-148 + scene/hexplane.py:73-106 (loss.backward(), train.py:219).
// Compiled with the default FMA contraction (no index-producing math here).
#include "g4d_internal.h"
#include "tc_wgmma.cuh"

namespace g4d {

namespace {

constexpr uint32_t kImg128 = 128u * 128u * 2u;   // bytes of one 128x128 bf16 part (hi or lo)

// D[64 x N] (+)= A * B with A = (hi, lo) bf16 register fragments (NS K-slices) and B = (hi, lo) images described by bh / bl,
// `step` = descriptor advance (16-byte units) per K = 16; TB = 1: B is MN-major
template <int N, int NS, int TB>
__device__ __forceinline__ void gemm3_rs(float (&d)[N / 2], const wg::Frags<NS>& a, uint64_t bh, uint64_t bl, uint32_t step, bool accumulate) {
    wg::fence_regs(d);
    wg::fence();
#pragma unroll
    for (int p = 0; p < 3; ++p) {
#pragma unroll
        for (int s = 0; s < NS; ++s)
            wg::mma_bf16_rs<N, TB>(d, p == 0 ? a.lo[s] : a.hi[s], ((p == 1) ? bl : bh) + (uint64_t)(s * step),
                                   (accumulate || p > 0 || s > 0) ? 1u : 0u);
    }
    wg::commit();
    wg::wait_all();
    wg::fence_regs(d);
}

// D[64 x N] (+)= A * B, both operands from shared memory, K = 64 (4 steps); b_single: B has no lo part (all-ones operand)
template <int N, int TA, int TB>
__device__ __forceinline__ void gemm3_ss(float (&d)[N / 2], uint64_t ah, uint64_t al, uint32_t astep, uint64_t bh, uint64_t bl,
                                         uint32_t bstep, bool accumulate, bool a_single, bool b_single) {
    wg::fence_regs(d);
    wg::fence();
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        if ((p == 0 && a_single) || (p == 1 && b_single)) continue;
#pragma unroll
        for (int s = 0; s < 4; ++s)
            wg::mma_bf16_ss<N, TA, TB>(d, ((p == 0) ? al : ah) + (uint64_t)(s * astep), ((p == 1) ? bl : bh) + (uint64_t)(s * bstep),
                                       (accumulate || s > 0 || p > (a_single || b_single ? 1 : 0)) ? 1u : 0u);
    }
    wg::commit();
    wg::wait_all();
    wg::fence_regs(d);
}

// accumulator block j of rows (g, g + 8), columns (c, c + 1) -> bf16 (hi, lo) A fragment slots + the rows' image words
__device__ __forceinline__ void put16(wg::Frags<8>& a, int j, float x0, float x1, float y0, float y1, uint32_t (&w)[4]) {
    const int s = j >> 1, o = (j & 1) * 2;
    wg::bf16_split2(x0, x1, a.hi[s][o], a.lo[s][o]);
    wg::bf16_split2(y0, y1, a.hi[s][o + 1], a.lo[s][o + 1]);
    w[0] = a.hi[s][o]; w[1] = a.lo[s][o]; w[2] = a.hi[s][o + 1]; w[3] = a.lo[s][o + 1];
}
// (hi, lo) words of rows ra / rb at column c of a (hi | lo) image with `ncols` columns (lo part at +part_bytes)
__device__ __forceinline__ void store_words(uint8_t* img, uint32_t part_bytes, uint32_t ncols, uint32_t ra, uint32_t rb, uint32_t c,
                                            const uint32_t (&w)[4]) {
    *reinterpret_cast<uint32_t*>(img + wg::img16_off(ra, c, ncols)) = w[0];
    *reinterpret_cast<uint32_t*>(img + part_bytes + wg::img16_off(ra, c, ncols)) = w[1];
    *reinterpret_cast<uint32_t*>(img + wg::img16_off(rb, c, ncols)) = w[2];
    *reinterpret_cast<uint32_t*>(img + part_bytes + wg::img16_off(rb, c, ncols)) = w[3];
}
__device__ __forceinline__ bool bit_of(const uint32_t (&m)[4], int c) {
    const uint32_t w = (c >> 5) == 0 ? m[0] : (c >> 5) == 1 ? m[1] : (c >> 5) == 2 ? m[2] : m[3];
    return (w >> (c & 31)) & 1u;
}
__device__ __forceinline__ void mbar_arrive1(void* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

}  // namespace

// ---- global-memory layout of the operand images (per tile of 128 Gaussians, (hi | lo), row = Gaussian) ---------------------
struct BwdImages {
    uint8_t* a1;                    // [ntiles][2 * kImg128]
    uint8_t* dh;                    // [ntiles][2 * kImg128]
    uint8_t* feat;                  // [ntiles][2 * 128*F*2]
    uint8_t* dz[G4D_NUM_HEADS];     // [ntiles][2 * kImg128]
    uint8_t* a2[G4D_NUM_HEADS];
    uint8_t* dout[G4D_NUM_HEADS];   // [ntiles][2 * 128*kp16*2]
    uint32_t feat_bytes;            // bytes of one (hi | lo) feature image
};

struct BwdSmemA { uint32_t w0, w1, w2t, bias, w2s, bars, total; };
static BwdSmemA bwd_smem_a(int F, bool sh) {
    BwdSmemA s{};
    uint32_t off = 0;
    auto take = [&](uint32_t b) { uint32_t o = off; off += (b + 127u) & ~127u; return o; };
    s.w0 = take(2u * 128 * F * 2);
    s.w1 = take(2u * 2u * kImg128);          // ring of two (hi | lo) head images
    s.w2t = take(sh ? 2u * 128 * 48 * 2 : 128);
    s.bias = take((128 + G4D_NUM_HEADS * 128) * 4);
    s.w2s = take(4 * 128 * 16);
    s.bars = take(64);
    s.total = off;
    return s;
}

// ---- weight images (bf16 hi | lo), rebuilt when the parameter version changes --------------------------------------
// matrix m: [rows][K] source; trans: image of the transpose ([K][rows], the SH head's W2 as the K-major B of d(a2) = dout W2)
struct BwdPackDesc {
    const float* src[2 + G4D_NUM_HEADS];
    uint8_t* dst[2 + G4D_NUM_HEADS];
    int K[2 + G4D_NUM_HEADS], rows[2 + G4D_NUM_HEADS], trans[2 + G4D_NUM_HEADS];
    int start[3 + G4D_NUM_HEADS];
    int count;
};
__global__ void bwd_pack_weights_kernel(BwdPackDesc p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.start[p.count]) return;
    int m = 0;
    while (i >= p.start[m + 1]) ++m;
    const int e = i - p.start[m], K = p.K[m];
    const uint32_t n = e / K, k = e % K;
    uint16_t hi, lo;
    wg::bf16_split(__ldg(p.src[m] + e), hi, lo);
    const uint32_t off = p.trans[m] ? wg::img16_off(k, n, (uint32_t)p.rows[m]) : wg::img16_off(n, k, (uint32_t)K);
    *reinterpret_cast<uint16_t*>(p.dst[m] + off) = hi;
    *reinterpret_cast<uint16_t*>(p.dst[m] + (size_t)p.rows[m] * K * 2u + off) = lo;
}

size_t tc_bwd_weight_bytes(const G4DDeformParams& prm) {
    return (size_t)2 * 128 * (prm.levels * prm.channels) * 2 + (size_t)G4D_NUM_HEADS * 2 * kImg128 + (size_t)2 * 48 * 128 * 2 + 512;
}

cudaError_t launch_tc_bwd_pack_weights(const G4DDeformParams& prm, uint8_t* blob, TcBwdWeights* out, cudaStream_t st) {
    BwdPackDesc p{};
    const int F = prm.levels * prm.channels;
    int m = 0, total = 0;
    uint8_t* q = blob;
    auto add = [&](const float* src, int rows, int K, int trans) {
        p.src[m] = src; p.dst[m] = q; p.rows[m] = rows; p.K[m] = K; p.trans[m] = trans; p.start[m] = total;
        total += rows * K;
        uint8_t* r = q;
        q += (size_t)2 * rows * K * 2;
        ++m;
        return r;
    };
    out->w0 = add(prm.w0, 128, F, 0);
    out->w2sh = nullptr;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        out->w1[h] = nullptr;
        if (!(prm.head_mask & (1 << h))) continue;
        out->w1[h] = add(prm.w1[h], 128, 128, 0);
    }
    if (prm.head_mask & G4D_HEAD_SHS) out->w2sh = add(prm.w2[4], 48, 128, 1);
    p.start[m] = total; p.count = m;
    return launch_k(bwd_pack_weights_kernel, (total + 255) / 256, 256, 0, st, kOrdinary, p);
}

bool tc_backward_supported(const G4DDeformParams& prm) {
    const int C = prm.channels, L = prm.levels;
    if (prm.net_width != 128 || prm.depth > 1) return false;   // no trunk layers (deep trunks: the FFMA kernels)
    if (!((C == 16 && (L == 2 || L == 3)) || (C == 32 && L == 2))) return false;
    return bwd_smem_a(C * L, (prm.head_mask & G4D_HEAD_SHS) != 0).total + 1024 <= 227 * 1024;
}

// ======================================================================================================
// Kernel A
// ======================================================================================================
struct BwdADesc {
    DeformDesc d;
    TcBwdWeights w;
    BwdImages img;
    const float* go[G4D_NUM_HEADS];
    const float* feat;           // [N][F] fp32 (deform_features_kernel)
    float* dfeat;                // [N][F] fp32 -> the scatter (bwd_scatter_kernel)
    const uint32_t* relu_bits;   // [6][N][4] + tag (g4d.h G4D_RELU_BITS_WORDS) or NULL
};

template <int C, int L>
__global__ void __launch_bounds__(256, 1)
deform_tc_bwd_dgrad_kernel(BwdADesc bd, BwdSmemA Ls, int64_t n) {
    constexpr int F = C * L, NS0 = F / 16;
    extern __shared__ __align__(1024) uint8_t smem[];
    const DeformDesc& d = bd.d;
    const int tid = threadIdx.x, wgi = tid >> 7, t128 = tid & 127, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int r0 = ((t128 >> 5) << 4) + g, r1 = r0 + 8;          // rows of this lane inside the warpgroup's 64
    const uint32_t ra = (uint32_t)(wgi * 64 + r0), rb = (uint32_t)(wgi * 64 + r1);   // ... inside the tile's 128
    float* sBias = reinterpret_cast<float*>(smem + Ls.bias);           // b0[128] | b1[5][128]
    float4* sW2s = reinterpret_cast<float4*>(smem + Ls.w2s);           // small heads: (W2[0][j], W2[1][j], W2[2][j], W2[3][j])
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Ls.bars);
    uint64_t *bar_w = bars, *bar_full = bars + 1, *bar_empty = bars + 3;
    const bool hsh = d.head_mask & G4D_HEAD_SHS;
    for (int i = tid; i < 128; i += 256) sBias[i] = __ldg(d.b0 + i);
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        for (int i = tid; i < 128; i += 256) sBias[128 + h * 128 + i] = __ldg(d.b1[h] + i);
        if (h < 4) {
            const int ko = head_out(h);
            for (int j = tid; j < 128; j += 256)
                sW2s[h * 128 + j] = make_float4(__ldg(d.w2[h] + j), ko > 1 ? __ldg(d.w2[h] + 128 + j) : 0.f,
                                               ko > 2 ? __ldg(d.w2[h] + 256 + j) : 0.f, ko > 3 ? __ldg(d.w2[h] + 384 + j) : 0.f);
        }
    }
    if (tid == 0) {
        mbar_init(bar_w, 1); mbar_init(bar_full, 1); mbar_init(bar_full + 1, 1); mbar_init(bar_empty, 8); mbar_init(bar_empty + 1, 8);
        fence_barrier_init();
    }
    __syncthreads();
    const int nheads = __popc(d.head_mask & 31);
    uint32_t hseq = 0;
    {
        int k = 0;
        for (int h = 0; h < G4D_NUM_HEADS; ++h)
            if (d.head_mask & (1 << h)) hseq |= (uint32_t)h << (3 * k++);
    }
    // saved ReLU signs are used when the forward that produced them says so (tag word behind the bits)
    const bool use_bits = bd.relu_bits && __ldg(bd.relu_bits + (size_t)24 * (size_t)n) == kReluBitsTag;
    const int64_t ntiles = (n + 127) / 128;
    const int64_t my_tiles = (int64_t)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const uint32_t total_items = (uint32_t)(my_tiles * nheads);
    // W1 ring: item u = (tile, head) in consumption order, slot u & 1; thread 0 loads one item ahead
    auto issue = [&](uint32_t u) {
        const uint32_t s = u & 1u;
        if (u >= 2) mbar_wait(bar_empty + s, ((u >> 1) - 1u) & 1u);
        const int h = (int)((hseq >> (3 * (u % (uint32_t)nheads))) & 7u);
        mbar_expect_tx(bar_full + s, 2u * kImg128);
        tma_bulk_g2s(smem + Ls.w1 + s * 2u * kImg128, bd.w.w1[h], 2u * kImg128, bar_full + s);
    };
    if (tid == 0) {
        const uint32_t w0b = 2u * 128 * F * 2, w2b = hsh ? 2u * 128 * 48 * 2 : 0u;
        mbar_expect_tx(bar_w, w0b + w2b);
        tma_bulk_g2s(smem + Ls.w0, bd.w.w0, w0b, bar_w);
        if (hsh) tma_bulk_g2s(smem + Ls.w2t, bd.w.w2sh, w2b, bar_w);
        if (total_items) issue(0);
    }
    __syncwarp();
    mbar_wait(bar_w, 0);
    const uint32_t sW0 = wg::smem_addr(smem + Ls.w0), sW1 = wg::smem_addr(smem + Ls.w1), sW2t = wg::smem_addr(smem + Ls.w2t);
    auto load_bits = [&](int slot, int64_t gi, uint32_t (&m)[4]) {
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (gi < n) v = __ldg(reinterpret_cast<const uint4*>(bd.relu_bits + ((size_t)slot * (size_t)n + (size_t)gi) * 4));
        m[0] = v.x; m[1] = v.y; m[2] = v.z; m[3] = v.w;
    };
    uint32_t u = 0;

    for (int64_t it = 0; it < my_tiles; ++it) {
        const int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
        const int64_t g0 = tile * 128 + ra, g1 = tile * 128 + rb;
        float acc[64];
        // ---- features -> A fragments + FEAT image; layer 0 recompute: D = feat W0^T
        {
            wg::Frags<NS0> x;
            uint8_t* img = bd.img.feat + (size_t)tile * bd.img.feat_bytes;
#pragma unroll
            for (int s = 0; s < NS0; ++s) {
#pragma unroll
                for (int hlf = 0; hlf < 2; ++hlf) {
                    const int c = 16 * s + 8 * hlf + 2 * t;
                    const float2 p0 = g0 < n ? __ldg(reinterpret_cast<const float2*>(bd.feat + g0 * F + c)) : make_float2(0.f, 0.f);
                    const float2 p1 = g1 < n ? __ldg(reinterpret_cast<const float2*>(bd.feat + g1 * F + c)) : make_float2(0.f, 0.f);
                    wg::bf16_split2(p0.x, p0.y, x.hi[s][2 * hlf], x.lo[s][2 * hlf]);
                    wg::bf16_split2(p1.x, p1.y, x.hi[s][2 * hlf + 1], x.lo[s][2 * hlf + 1]);
                    const uint32_t w[4] = {x.hi[s][2 * hlf], x.lo[s][2 * hlf], x.hi[s][2 * hlf + 1], x.lo[s][2 * hlf + 1]};
                    store_words(img, 128u * F * 2u, F, ra, rb, (uint32_t)c, w);
                }
            }
            const uint64_t bh = wg::desc_kmajor(sW0, F, 8), bl = wg::desc_kmajor(sW0 + 128u * F * 2u, F, 8);
            gemm3_rs<128, NS0, 0>(acc, x, bh, bl, 16, false);
        }
        // ---- a1 = relu(h0) -> A fragments + A1 image; hm = sign bits of h0
        uint32_t hm0[4], hm1[4];
        wg::Frags<8> a1;
        {
            if (use_bits) { load_bits(0, g0, hm0); load_bits(0, g1, hm1); }
            else {
#pragma unroll
                for (int w = 0; w < 4; ++w) { hm0[w] = 0u; hm1[w] = 0u; }
            }
            uint8_t* img = bd.img.a1 + (size_t)tile * 2 * kImg128;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * t;
                const float x0 = acc[4 * j] + sBias[c], x1 = acc[4 * j + 1] + sBias[c + 1];
                const float y0 = acc[4 * j + 2] + sBias[c], y1 = acc[4 * j + 3] + sBias[c + 1];
                bool on[4];
                if (use_bits) {
                    on[0] = bit_of(hm0, c); on[1] = bit_of(hm0, c + 1); on[2] = bit_of(hm1, c); on[3] = bit_of(hm1, c + 1);
                } else {
                    on[0] = x0 > 0.f; on[1] = x1 > 0.f; on[2] = y0 > 0.f; on[3] = y1 > 0.f;
                    const int sh = c & 31;
                    hm0[j >> 2] |= ((on[0] ? 1u : 0u) | (on[1] ? 2u : 0u)) << sh;
                    hm1[j >> 2] |= ((on[2] ? 1u : 0u) | (on[3] ? 2u : 0u)) << sh;
                }
                uint32_t w[4];
                put16(a1, j, on[0] ? fmaxf(x0, 0.f) : 0.f, on[1] ? fmaxf(x1, 0.f) : 0.f, on[2] ? fmaxf(y0, 0.f) : 0.f,
                      on[3] ? fmaxf(y1, 0.f) : 0.f, w);
                store_words(img, kImg128, 128, ra, rb, (uint32_t)c, w);
            }
        }
        float da1[64];
#pragma unroll 1
        for (int k = 0; k < nheads; ++k, ++u) {
            const int h = (int)((hseq >> (3 * k)) & 7u);
            const float* b1 = sBias + 128 + h * 128;
            if (tid == 0 && u + 1 < total_items) issue(u + 1);
            __syncwarp();
            const uint32_t slot = u & 1u;
            mbar_wait(bar_full + slot, (u >> 1) & 1u);
            const uint32_t w1 = sW1 + slot * 2u * kImg128;
            // ---- z = a1 W1^T
            gemm3_rs<128, 8, 0>(acc, a1, wg::desc_kmajor(w1, 128, 8), wg::desc_kmajor(w1 + kImg128, 128, 8), 16, false);
            uint32_t zm0[4], zm1[4];
            if (use_bits) { load_bits(1 + h, g0, zm0); load_bits(1 + h, g1, zm1); }
            // ---- a2 = relu(z) (A2 image); masks; dL/d(out) rows (DOUT image)
            uint8_t* img_a2 = bd.img.a2[h] + (size_t)tile * 2 * kImg128;
            const float* go = bd.go[h];
            float dn0[4] = {0.f, 0.f, 0.f, 0.f}, dn1[4] = {0.f, 0.f, 0.f, 0.f};
            uint64_t onm = 0ull;   // bit 4 j + q: ReLU of value q (x0, x1, y0, y1) of accumulator block j is on
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * t;
                const float x0 = acc[4 * j] + b1[c], x1 = acc[4 * j + 1] + b1[c + 1];
                const float y0 = acc[4 * j + 2] + b1[c], y1 = acc[4 * j + 3] + b1[c + 1];
                bool on[4];
                if (use_bits) {
                    on[0] = bit_of(zm0, c); on[1] = bit_of(zm0, c + 1); on[2] = bit_of(zm1, c); on[3] = bit_of(zm1, c + 1);
                } else {
                    on[0] = x0 > 0.f; on[1] = x1 > 0.f; on[2] = y0 > 0.f; on[3] = y1 > 0.f;
                }
                onm |= (uint64_t)((on[0] ? 1u : 0u) | (on[1] ? 2u : 0u) | (on[2] ? 4u : 0u) | (on[3] ? 8u : 0u)) << (4 * j);
                uint32_t w[4];
                wg::bf16_split2(on[0] ? fmaxf(x0, 0.f) : 0.f, on[1] ? fmaxf(x1, 0.f) : 0.f, w[0], w[1]);
                wg::bf16_split2(on[2] ? fmaxf(y0, 0.f) : 0.f, on[3] ? fmaxf(y1, 0.f) : 0.f, w[2], w[3]);
                store_words(img_a2, kImg128, 128, ra, rb, (uint32_t)c, w);
            }
            auto on_bit = [&](int j, int q) { return ((onm >> (4 * j + q)) & 1ull) != 0ull; };
            uint8_t* img_do = bd.img.dout[h] + (size_t)tile * 2 * 128 * (h == 4 ? 48 : 16) * 2;
            if (h < 4) {
                const int ko = head_out(h);
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    if (o < ko && go) {
                        if (g0 < n) dn0[o] = __ldg(go + g0 * ko + o);
                        if (g1 < n) dn1[o] = __ldg(go + g1 * ko + o);
                    }
                }
                // DOUT image [128][16]: lane t writes columns 2t, 2t + 1 and 8 + 2t, 9 + 2t (zero beyond the head's outputs)
                {
                    uint32_t w[4];
                    const float e0 = t == 0 ? dn0[0] : t == 1 ? dn0[2] : 0.f, e1 = t == 0 ? dn0[1] : t == 1 ? dn0[3] : 0.f;
                    const float f0 = t == 0 ? dn1[0] : t == 1 ? dn1[2] : 0.f, f1 = t == 0 ? dn1[1] : t == 1 ? dn1[3] : 0.f;
                    wg::bf16_split2(e0, e1, w[0], w[1]);
                    wg::bf16_split2(f0, f1, w[2], w[3]);
                    store_words(img_do, 128u * 16u * 2u, 16, ra, rb, (uint32_t)(2 * t), w);
                    const uint32_t z[4] = {0u, 0u, 0u, 0u};
                    store_words(img_do, 128u * 16u * 2u, 16, ra, rb, (uint32_t)(8 + 2 * t), z);
                }
                // dz = (dout W2) * [z > 0], in place of z
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int c = 8 * j + 2 * t;
                    const float4 wa = sW2s[h * 128 + c], wb = sW2s[h * 128 + c + 1];
                    const float da_x0 = dn0[0] * wa.x + dn0[1] * wa.y + dn0[2] * wa.z + dn0[3] * wa.w;
                    const float da_x1 = dn0[0] * wb.x + dn0[1] * wb.y + dn0[2] * wb.z + dn0[3] * wb.w;
                    const float da_y0 = dn1[0] * wa.x + dn1[1] * wa.y + dn1[2] * wa.z + dn1[3] * wa.w;
                    const float da_y1 = dn1[0] * wb.x + dn1[1] * wb.y + dn1[2] * wb.z + dn1[3] * wb.w;
                    acc[4 * j] = on_bit(j, 0) ? da_x0 : 0.f; acc[4 * j + 1] = on_bit(j, 1) ? da_x1 : 0.f;
                    acc[4 * j + 2] = on_bit(j, 2) ? da_y0 : 0.f; acc[4 * j + 3] = on_bit(j, 3) ? da_y1 : 0.f;
                }
            } else {
                // SH head: d(a2) = dout W2 as a GEMM (K = 48: dout rows as A fragments, W2^T image as B), DOUT image on the way
                wg::Frags<3> x;
#pragma unroll
                for (int s = 0; s < 3; ++s) {
#pragma unroll
                    for (int hlf = 0; hlf < 2; ++hlf) {
                        const int c = 16 * s + 8 * hlf + 2 * t;
                        float2 p0 = make_float2(0.f, 0.f), p1 = p0;
                        if (go && g0 < n) p0 = __ldg(reinterpret_cast<const float2*>(go + g0 * 48 + c));
                        if (go && g1 < n) p1 = __ldg(reinterpret_cast<const float2*>(go + g1 * 48 + c));
                        wg::bf16_split2(p0.x, p0.y, x.hi[s][2 * hlf], x.lo[s][2 * hlf]);
                        wg::bf16_split2(p1.x, p1.y, x.hi[s][2 * hlf + 1], x.lo[s][2 * hlf + 1]);
                        const uint32_t w[4] = {x.hi[s][2 * hlf], x.lo[s][2 * hlf], x.hi[s][2 * hlf + 1], x.lo[s][2 * hlf + 1]};
                        store_words(img_do, 128u * 48u * 2u, 48, ra, rb, (uint32_t)c, w);
                    }
                }
                gemm3_rs<128, 3, 0>(acc, x, wg::desc_kmajor(sW2t, 48, 8), wg::desc_kmajor(sW2t + 128u * 48u * 2u, 48, 8), 16, false);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    acc[4 * j] = on_bit(j, 0) ? acc[4 * j] : 0.f; acc[4 * j + 1] = on_bit(j, 1) ? acc[4 * j + 1] : 0.f;
                    acc[4 * j + 2] = on_bit(j, 2) ? acc[4 * j + 2] : 0.f; acc[4 * j + 3] = on_bit(j, 3) ? acc[4 * j + 3] : 0.f;
                }
            }
            // ---- DZ image + A fragments; d(a1) += dz W1 (W1 image read MN-major)
            {
                wg::Frags<8> dz;
                uint8_t* img = bd.img.dz[h] + (size_t)tile * 2 * kImg128;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    uint32_t w[4];
                    put16(dz, j, acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], w);
                    store_words(img, kImg128, 128, ra, rb, (uint32_t)(8 * j + 2 * t), w);
                }
                gemm3_rs<128, 8, 1>(da1, dz, wg::desc_mnmajor(w1, 128), wg::desc_mnmajor(w1 + kImg128, 128), (2u * 16u * 128u) >> 4, k > 0);
            }
            if (lane == 0) mbar_arrive1(bar_empty + slot);      // this warp's MMAs on the slot have retired
        }

        // ---- dh = d(a1) * [h0 > 0] -> A fragments + DH image; d(feat) = dh W0 (W0 image read MN-major) -> [N][F] fp32
        {
            wg::Frags<8> dh;
            uint8_t* img = bd.img.dh + (size_t)tile * 2 * kImg128;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * t;
                uint32_t w[4];
                put16(dh, j, bit_of(hm0, c) ? da1[4 * j] : 0.f, bit_of(hm0, c + 1) ? da1[4 * j + 1] : 0.f,
                      bit_of(hm1, c) ? da1[4 * j + 2] : 0.f, bit_of(hm1, c + 1) ? da1[4 * j + 3] : 0.f, w);
                store_words(img, kImg128, 128, ra, rb, (uint32_t)c, w);
            }
            float df[F / 2];
            gemm3_rs<F, 8, 1>(df, dh, wg::desc_mnmajor(sW0, F), wg::desc_mnmajor(sW0 + 128u * F * 2u, F), (2u * (F / 8) * 128u) >> 4, false);
#pragma unroll
            for (int j = 0; j < F / 8; ++j) {
                const int c = 8 * j + 2 * t;
                if (g0 < n) *reinterpret_cast<float2*>(bd.dfeat + g0 * F + c) = make_float2(df[4 * j], df[4 * j + 1]);
                if (g1 < n) *reinterpret_cast<float2*>(bd.dfeat + g1 * F + c) = make_float2(df[4 * j + 2], df[4 * j + 3]);
            }
        }
    }
}

// ======================================================================================================
// Kernel B: weight gradients from the operand images.
//   CTA (group, chunk): group = an active head or layer 0.  Two warpgroups, warpgroup w accumulates output rows
//   [64 w, 64 w + 64) (hidden units j); thread 0 streams the stages.
// ======================================================================================================
struct BwdBDesc {
    BwdImages img;
    int head_mask, F, nheads, chunks_head, chunks_l0;
    int64_t ntiles;
    float* g_w0; float* g_b0;
    float* g_w1[G4D_NUM_HEADS]; float* g_b1[G4D_NUM_HEADS]; float* g_w2[G4D_NUM_HEADS]; float* g_b2[G4D_NUM_HEADS];
};

constexpr uint32_t kHalf128 = kImg128 / 2;                          // 16 KB: 64 rows x 128 cols bf16
constexpr uint32_t kStage = 3u * 2u * kHalf128 + 2u * 64 * 48 * 2;   // 108 KB: X | Y | A2 | DOUT, each (hi half | lo half)
constexpr uint32_t kOnes = 64u * 64u * 2u;                           // all-ones bf16 operand

// NW = columns of dW (128, or F for layer 0); KP = columns of the DOUT image (16 for the small heads, 48 for the SH head, 0 for
// layer 0)
template <int NW, int KP>
__device__ __forceinline__ void wgrad_group(const BwdBDesc& b, int h, int64_t t0, int64_t t1, uint8_t* smem, uint64_t* bar_ld) {
    constexpr bool layer0 = KP == 0;
    constexpr int NW2 = KP > 0 ? KP : 8;
    const int tid = threadIdx.x, wgi = tid >> 7, t128 = tid & 127, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int kp16 = KP;
    const uint32_t yp = layer0 ? 128u * NW * 2u : kImg128;             // bytes of one part (hi or lo) of Y
    const uint32_t dp = 128u * kp16 * 2u;                              // ... of DOUT
    const int64_t nwork = t1 > t0 ? 2 * (t1 - t0) : 0;
    // work item w = 2 (t - t0) + hf: rows [64 hf, 64 hf + 64) of tile t; the images are row-group major, so that half of a
    // part is one contiguous half of its bytes
    auto load = [&](int64_t w) {
        const int st = (int)(w & 1), hf = (int)(w & 1);
        const int64_t tl = t0 + (w >> 1);
        uint8_t* base = smem + st * kStage;
        uint8_t *dX = base, *dY = base + 2 * kHalf128, *dA2 = base + 4 * kHalf128, *dDO = base + 6 * kHalf128;
        const uint8_t* srcX = (layer0 ? b.img.dh : b.img.dz[h]) + (size_t)tl * 2 * kImg128;
        const uint8_t* srcY = layer0 ? b.img.feat + (size_t)tl * b.img.feat_bytes : b.img.a1 + (size_t)tl * 2 * kImg128;
        const uint32_t bytes = 2u * kHalf128 + yp + (layer0 ? 0u : 2u * kHalf128 + dp);
        mbar_expect_tx(&bar_ld[st], bytes);
        tma_bulk_g2s(dX, srcX + hf * kHalf128, kHalf128, &bar_ld[st]);
        tma_bulk_g2s(dX + kHalf128, srcX + kImg128 + hf * kHalf128, kHalf128, &bar_ld[st]);
        tma_bulk_g2s(dY, srcY + hf * (yp / 2), yp / 2, &bar_ld[st]);
        tma_bulk_g2s(dY + yp / 2, srcY + yp + hf * (yp / 2), yp / 2, &bar_ld[st]);
        if (!layer0) {
            const uint8_t* srcA = b.img.a2[h] + (size_t)tl * 2 * kImg128;
            const uint8_t* srcD = b.img.dout[h] + (size_t)tl * 2 * dp;
            tma_bulk_g2s(dA2, srcA + hf * kHalf128, kHalf128, &bar_ld[st]);
            tma_bulk_g2s(dA2 + kHalf128, srcA + kImg128 + hf * kHalf128, kHalf128, &bar_ld[st]);
            tma_bulk_g2s(dDO, srcD + hf * (dp / 2), dp / 2, &bar_ld[st]);
            tma_bulk_g2s(dDO + dp / 2, srcD + dp + hf * (dp / 2), dp / 2, &bar_ld[st]);
        }
    };
    float accW[NW / 2], accW2[NW2 / 2], accB[4], accB2[NW2 / 2];
    if (tid == 0) {
        if (nwork > 0) load(0);
        if (nwork > 1) load(1);
    }
    const uint32_t ones = wg::smem_addr(smem + 2 * kStage);
    // all-ones operands: B of the bias sums ([64 Gaussians][8], MN-major) and A of db2 ([64][64 Gaussians], K-major)
    const uint64_t ones_b = wg::desc_mnmajor(ones, 8), ones_a = wg::desc_kmajor(ones, 64, 8);
    // MN-major operand images of 64 rows (Gaussians = K): one K = 16 step is two rows of core matrices
    const uint32_t step128 = (2u * 16u * 128u) >> 4;
    const uint32_t a_off = (uint32_t)wgi * 64u * 16u;                  // this warpgroup's 64 output rows (M) inside X / A2
    for (int64_t w = 0; w < nwork; ++w) {
        const int st = (int)(w & 1);
        mbar_wait(&bar_ld[st], (uint32_t)(w >> 1) & 1u);
        const uint32_t base = wg::smem_addr(smem + st * kStage);
        const uint32_t x = base, y = base + 2 * kHalf128, a2 = base + 4 * kHalf128, dd = base + 6 * kHalf128;
        const bool acc = w > 0;
        const uint64_t xh = wg::desc_mnmajor(x + a_off, 128), xl = wg::desc_mnmajor(x + kHalf128 + a_off, 128);
        if constexpr (layer0) {
            gemm3_ss<NW, 1, 1>(accW, xh, xl, step128, wg::desc_mnmajor(y, NW), wg::desc_mnmajor(y + yp / 2, NW), (2u * (NW / 8) * 128u) >> 4,
                               acc, false, false);
        } else {
            gemm3_ss<NW, 1, 1>(accW, xh, xl, step128, wg::desc_mnmajor(y, 128), wg::desc_mnmajor(y + kHalf128, 128), step128, acc, false, false);
            const uint64_t ah = wg::desc_mnmajor(a2 + a_off, 128), al = wg::desc_mnmajor(a2 + kHalf128 + a_off, 128);
            const uint64_t dh = wg::desc_mnmajor(dd, (uint32_t)kp16), dl = wg::desc_mnmajor(dd + dp / 2, (uint32_t)kp16);
            const uint32_t dstep = (2u * (uint32_t)(kp16 / 8) * 128u) >> 4;
            gemm3_ss<NW2, 1, 1>(accW2, ah, al, step128, dh, dl, dstep, acc, false, false);
            if (wgi == 0) gemm3_ss<NW2, 0, 1>(accB2, ones_a, ones_a, 16, dh, dl, dstep, acc, true, false);
        }
        gemm3_ss<8, 1, 1>(accB, xh, xl, step128, ones_b, ones_b, 16, acc, false, true);
        __syncthreads();                                  // both warpgroups are done with stage st
        if (tid == 0 && w + 2 < nwork) load(w + 2);
    }
    if (nwork == 0) return;
    // ---- flush: thread rows j0 = 64 wgi + 16 warp + g and j0 + 8 of every accumulator
    const int j0 = wgi * 64 + ((t128 >> 5) << 4) + g, j1 = j0 + 8;
    float* gw = layer0 ? b.g_w0 : b.g_w1[h];
#pragma unroll
    for (int q = 0; q < NW / 8; ++q) {
        const int c = 8 * q + 2 * t;
        atomicAdd(gw + (size_t)j0 * NW + c, accW[4 * q]); atomicAdd(gw + (size_t)j0 * NW + c + 1, accW[4 * q + 1]);
        atomicAdd(gw + (size_t)j1 * NW + c, accW[4 * q + 2]); atomicAdd(gw + (size_t)j1 * NW + c + 1, accW[4 * q + 3]);
    }
    float* gb = layer0 ? b.g_b0 : b.g_b1[h];
    if (t == 0) { atomicAdd(gb + j0, accB[0]); atomicAdd(gb + j1, accB[2]); }    // (every column of the ones product is the sum)
    if constexpr (!layer0) {
        const int ko = head_out(h);
#pragma unroll
        for (int q = 0; q < NW2 / 8; ++q) {
            const int c = 8 * q + 2 * t;
            if (c < ko) { atomicAdd(b.g_w2[h] + (size_t)c * 128 + j0, accW2[4 * q]); atomicAdd(b.g_w2[h] + (size_t)c * 128 + j1, accW2[4 * q + 2]); }
            if (c + 1 < ko) { atomicAdd(b.g_w2[h] + (size_t)(c + 1) * 128 + j0, accW2[4 * q + 1]); atomicAdd(b.g_w2[h] + (size_t)(c + 1) * 128 + j1, accW2[4 * q + 3]); }
            // db2: every row of 1^T DOUT is the same sum -- warpgroup 0, row 0 (lanes 0-3 of warp 0) flushes it
            if (wgi == 0 && tid < 4) {
                if (c < ko) atomicAdd(b.g_b2[h] + c, accB2[4 * q]);
                if (c + 1 < ko) atomicAdd(b.g_b2[h] + c + 1, accB2[4 * q + 1]);
            }
        }
    }
}

__global__ void __launch_bounds__(256, 1) deform_tc_bwd_wgrad_kernel(BwdBDesc b) {
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar_ld[2];
    const int tid = threadIdx.x;
    // CTAs [0, nheads * chunks_head) serve the active heads, the rest layer 0 (CTA counts proportional to the bytes per tile)
    const bool layer0 = (int)blockIdx.x >= b.nheads * b.chunks_head;
    const int chunk = layer0 ? (int)blockIdx.x - b.nheads * b.chunks_head : (int)blockIdx.x % b.chunks_head;
    const int nch = layer0 ? b.chunks_l0 : b.chunks_head;
    int h = 5;
    if (!layer0) {
        int m = b.head_mask;
        for (int i = 0; i < (int)blockIdx.x / b.chunks_head; ++i) m &= m - 1;
        h = __ffs(m) - 1;
    }
    uint16_t* ones = reinterpret_cast<uint16_t*>(smem + 2 * kStage);
    for (int i = tid; i < (int)(kOnes / 2); i += 256) ones[i] = 0x3F80;     // bf16 1.0
    if (tid == 0) {
        mbar_init(&bar_ld[0], 1); mbar_init(&bar_ld[1], 1);
        fence_barrier_init();
    }
    wg::fence_proxy_async();                      // the ones image is read by the tensor cores
    __syncthreads();
    const int64_t per = (b.ntiles + nch - 1) / nch;
    const int64_t t0 = (int64_t)chunk * per, t1 = (t0 + per < b.ntiles) ? t0 + per : b.ntiles;
    if (!layer0) {
        if (h == 4) wgrad_group<128, 48>(b, h, t0, t1, smem, bar_ld);
        else wgrad_group<128, 16>(b, h, t0, t1, smem, bar_ld);
    } else if (b.F == 32) wgrad_group<32, 0>(b, 5, t0, t1, smem, bar_ld);
    else if (b.F == 48) wgrad_group<48, 0>(b, 5, t0, t1, smem, bar_ld);
    else wgrad_group<64, 0>(b, 5, t0, t1, smem, bar_ld);
}

// ======================================================================================================
// host side: the tensor-core engine of the deformation backward (launch_deform_backward, g4d_backward.cu, runs the gather,
// the scatter and the time-row distribution around it)
// ======================================================================================================
// the operand images kernel A writes for kernel B, per tile of 128 Gaussians
static BwdImages carve_images(Carve& m, const DeformDesc& d, int64_t n) {
    const size_t ntiles = (size_t)((n + 127) / 128);
    BwdImages img{};
    img.feat_bytes = 2u * 128 * d.F * 2;
    img.a1 = m.take<uint8_t>(ntiles * 2 * kImg128);
    img.dh = m.take<uint8_t>(ntiles * 2 * kImg128);
    img.feat = m.take<uint8_t>(ntiles * img.feat_bytes);
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        img.dz[h] = m.take<uint8_t>(ntiles * 2 * kImg128);
        img.a2[h] = m.take<uint8_t>(ntiles * 2 * kImg128);
        img.dout[h] = m.take<uint8_t>(ntiles * 2 * 128 * (h == 4 ? 48 : 16) * 2);
    }
    return img;
}

size_t tc_bwd_images_bytes(const DeformDesc& d, int64_t n) {
    Carve m;
    carve_images(m, d, n);
    return m.bytes();
}

template <int C, int L>
static cudaError_t launch_a(const BwdADesc& bd, int64_t n, int sm_count, cudaStream_t st) {
    const BwdSmemA Ls = bwd_smem_a(C * L, bd.d.head_mask & G4D_HEAD_SHS);
    const size_t bytes = Ls.total + 1024;
    const int64_t ntiles = (n + 127) / 128;
    const int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
    return launch_k(deform_tc_bwd_dgrad_kernel<C, L>, grid, 256, bytes, st, kOrdinary, bd, Ls, n);
}

cudaError_t launch_tc_bwd_dgrad(const DeformDesc& d, const TcBwdWeights& w, int64_t n, const float* const go[G4D_NUM_HEADS],
                                const uint32_t* relu_bits, const float* feat, float* dfeat, uint8_t* images, int sm_count,
                                cudaStream_t st) {
    Carve m(images);
    BwdADesc a{};
    a.d = d; a.w = w; a.relu_bits = relu_bits; a.img = carve_images(m, d, n);
    for (int h = 0; h < G4D_NUM_HEADS; ++h) a.go[h] = go[h];
    a.feat = feat; a.dfeat = dfeat;
    if (d.C == 16 && d.levels == 2) return launch_a<16, 2>(a, n, sm_count, st);
    if (d.C == 16 && d.levels == 3) return launch_a<16, 3>(a, n, sm_count, st);
    if (d.C == 32 && d.levels == 2) return launch_a<32, 2>(a, n, sm_count, st);
    return cudaErrorInvalidValue;
}

cudaError_t launch_tc_bwd_wgrad(const DeformDesc& d, const G4DDeformGrads& grads, int64_t n, uint8_t* images, int sm_count,
                                cudaStream_t st) {
    const int64_t ntiles = (n + 127) / 128;
    Carve m(images);
    BwdBDesc b{};
    b.img = carve_images(m, d, n); b.head_mask = d.head_mask; b.F = d.F; b.ntiles = ntiles;
    {
        int nheads = 0;
        for (int h = 0; h < G4D_NUM_HEADS; ++h) nheads += (d.head_mask >> h) & 1;
        // bytes per tile: a head streams DZ + A1 + A2 (+ DOUT), layer 0 streams DH + FEAT
        const double wh = 3.0 * 64 + 16, w0 = 64 + (double)(2 * 128 * d.F * 2) / 1024.0, tot = nheads * wh + w0;
        int ch = nheads ? (int)(sm_count * wh / tot) : 0;
        if (ch < 1) ch = 1;
        int c0 = sm_count - nheads * ch;
        if (c0 < 1) c0 = 1;
        if ((int64_t)ch > ntiles) ch = (int)ntiles;
        if ((int64_t)c0 > ntiles) c0 = (int)ntiles;
        b.nheads = nheads; b.chunks_head = ch; b.chunks_l0 = c0;
    }
    b.g_w0 = grads.w0; b.g_b0 = grads.b0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) { b.g_w1[h] = grads.w1[h]; b.g_b1[h] = grads.b1[h]; b.g_w2[h] = grads.w2[h]; b.g_b2[h] = grads.b2[h]; }
    const size_t smem_b = (size_t)2 * kStage + kOnes + 1024;   // two half-tile stages + the all-ones operand
    return launch_k(deform_tc_bwd_wgrad_kernel, b.nheads * b.chunks_head + b.chunks_l0, 256, smem_b, st, kOrdinary, b);
}

}  // namespace g4d
