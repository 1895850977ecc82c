// g4d_deform_tc.cu -- tensor-core version of the fused deform + activate + project forward (net_width 128).
//
// The deformation MLP (scene/deformation.py:67-148: 93.6 kMAC per Gaussian at the DyNeRF config) runs on the Hopper tensor
// cores with hand-written wgmma PTX (tc_wgmma.cuh), on FP16x2 operands (G4D_OPT_TENSOR_CORES = 2, the default):
// x = hi + lo with hi = rn_f16(s x), lo = rn_f16(s x - hi), s a fixed power of two per operand class (features 2^6,
// activations 2^3, weights 2^8; undone exactly by the epilogue's FMA).  |x - (hi + lo)/s| <= max(2^-22 |x|, 2^-25 / s): an
// absolute floor far below the fp32 accumulation noise of a K = 128 dot product.  The three products lo*hi + hi*lo + hi*hi
// with fp32 accumulation give fp32-level accuracy (single-pass F16 is ~1000x worse than the 1e-4 image tolerance allows).
// s |x| must stay below 65504 (activations < 8188, features < 1023, weights < 255): conversions saturate and the kernel
// raises a flag in host-mapped memory that the next call reports (G4D_ERR_OVERFLOW).  Networks beyond that range run on the
// FFMA kernels (G4D_OPT_TENSOR_CORES = 0), which have no range limit.
//
// Structure: a warpgroup (128 threads) owns 64 Gaussians (the M = 64 of wgmma) and carries them through every layer:
//   * the A operand of every GEMM lives in registers: the features are loaded straight into fragment layout, and each
//     epilogue (bias, ReLU, sign bits for the backward, hi / lo split) turns the fp32 accumulator fragment into the next
//     layer's A fragment in place (tc_wgmma.cuh) -- activations never touch shared memory or HBM;
//   * weights are the B operand in shared memory: packed once per parameter version into the no-swizzle canonical K-major
//     image (hi | lo), W0 and the SH head's W2 resident, W1 streamed head by head through a two-slot ring with TMA bulk
//     copies and mbarriers (full: transaction count; empty: one arrival per consumer warp), one load ahead;
//   * three warpgroups per CTA (192 Gaussians per W1 image load) where their shared memory fits, else two (F = 48 / 64
//     with the SH head);
//   * layer 2 of the <= 4-wide heads runs in exact fp32 in the epilogue (each lane sums its 32 hidden units, a quad shuffle
//     completes the row); the SH head's layer 2 (N = 48) is a fourth GEMM;
//   * the per-Gaussian tail (residual adds, activations, EWA projection, SH colour -- geom_finish.cuh) runs after a hand-over
//     through shared memory: threads 0-63 of the warpgroup finish the geometry, 64-127 the colour of one Gaussian each.
// The HexPlane gather runs BEFORE this kernel at full occupancy (deform_features_kernel, feat [N][F] stays in L2).
// Compiled with -fmad=false (it contains the projection, see g4d_math.cuh); the FMAs of the epilogues are explicit.
#include "geom_finish.cuh"
#include "tc_wgmma.cuh"

namespace g4d {

// FP16x2 operands: K per wgmma slice, bytes per element, elements per 16-byte core row; scales of features, activations, weights
struct TcArith {
    static constexpr int KS = 16, ES = 2, EPC = 8;
    static constexpr float SF = 64.f, SA = 8.f, SW = 256.f;
};
constexpr float kF16Max = 65504.f;
constexpr int kStageCols = 60;
// shared memory of one block: the dynamic layout below + the static camera copy (padded to the 128 B alignment of the dynamic
// array) must fit the 227 KB a block may use on sm_90
constexpr uint32_t kMaxSmemPerBlock = 227u * 1024u;
constexpr uint32_t kTcStaticSmem = (uint32_t)((sizeof(CameraDev) + 127) & ~(size_t)127);                 // per Gaussian: 11 geometry deltas | 48 SH deltas | pad

struct TcSmem { uint32_t w1, w0, w2, bias, w2s, stage, bars, slot_bytes, total; };

// slot_bytes: one ring slot = one head's W1 image, (hi | lo); one stage slab per consumer warpgroup
inline TcSmem tc_smem_layout(int nwg, int F, bool sh) {
    constexpr uint32_t es = TcArith::ES;
    TcSmem s{};
    uint32_t off = 0;
    auto take = [&](uint32_t bytes) { uint32_t o = off; off += (bytes + 127u) & ~127u; return o; };
    s.slot_bytes = 2u * 128u * 128u * es;
    s.w1 = take(2u * s.slot_bytes);
    s.w0 = take(2u * 128u * F * es);
    s.w2 = take(sh ? 2u * 48u * 128u * es : 128u);
    s.bias = take((128 + G4D_NUM_HEADS * 128 + 64) * 4);
    s.w2s = take(4 * 128 * 16);
    s.stage = take((uint32_t)nwg * 64u * kStageCols * 4u);
    s.bars = take(64);
    s.total = off;
    return s;
}

// consumer warpgroups per CTA: the most (3, else 2) whose layout fits a block; 0 when none fits.  More warpgroups share
// each W1 image load and keep the tensor pipe busy while others run epilogues; every Gaussian's arithmetic is the same at
// any count.
inline int tc_warpgroups(int F, bool sh) {
    for (int nwg = 3; nwg >= 2; --nwg)
        if (tc_smem_layout(nwg, F, sh).total + kTcStaticSmem <= kMaxSmemPerBlock) return nwg;
    return 0;
}

// ---- weight packing (once per parameter version) --------------------------------------------------------------
// Every matrix [rows][K] (torch Linear layout) becomes a (hi | lo) pair of canonical K-major images of scaled f16 words.
struct TcPackDesc {
    const float* src[1 + G4D_NUM_HEADS + 1];
    uint8_t* dst[1 + G4D_NUM_HEADS + 1];
    int rows[1 + G4D_NUM_HEADS + 1], K[1 + G4D_NUM_HEADS + 1];
    int start[2 + G4D_NUM_HEADS + 1];
    int count;
    uint32_t* status;                 // set to 1 when a scaled weight leaves the f16 range (TcWeights::status)
};

__global__ void tc_pack_weights_kernel(TcPackDesc p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.start[p.count]) return;
    int m = 0;
    while (i >= p.start[m + 1]) ++m;
    const int e = i - p.start[m];
    const uint32_t K = (uint32_t)p.K[m], n = (uint32_t)e / K, k = (uint32_t)e % K, rows = (uint32_t)p.rows[m];
    const float v = __ldg(p.src[m] + e);
    uint32_t hi, lo;
    if (fabsf(v * TcArith::SW) >= kF16Max && p.status) *reinterpret_cast<volatile uint32_t*>(p.status) = 1u;   // saturates
    wg::f16_split2(v * TcArith::SW, 0.f, hi, lo);
    uint8_t* base = p.dst[m] + wg::img16_off(n, k, K);
    *reinterpret_cast<uint16_t*>(base) = (uint16_t)hi;
    *reinterpret_cast<uint16_t*>(base + rows * K * 2u) = (uint16_t)lo;
}

size_t tc_packed_floats(const G4DDeformParams& prm) {
    const int F = prm.levels * prm.channels;
    size_t f = 2 * (size_t)128 * F;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) f += 2 * (size_t)128 * 128 + (h == 4 ? 2 * (size_t)48 * 128 : 0);
    return f + 64;
}

cudaError_t launch_tc_pack_weights(const G4DDeformParams& prm, float* blob, TcWeights* out, cudaStream_t st) {
    TcPackDesc p{};
    p.status = out->status;
    const int F = prm.levels * prm.channels;
    int m = 0, total = 0;
    uint8_t* q = reinterpret_cast<uint8_t*>(blob);
    auto add = [&](const float* src, int rows, int K) {
        p.src[m] = src; p.dst[m] = q; p.rows[m] = rows; p.K[m] = K;
        p.start[m] = total;
        total += rows * K;
        uint8_t* r = q;
        q += 2 * (size_t)rows * K * TcArith::ES;
        ++m;
        return reinterpret_cast<const float*>(r);
    };
    out->w0 = add(prm.w0, 128, F);
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        out->w1[h] = nullptr; out->w2[h] = nullptr;
        if (!(prm.head_mask & (1 << h))) continue;
        out->w1[h] = add(prm.w1[h], 128, 128);
        if (h == 4) out->w2[h] = add(prm.w2[h], 48, 128);   // the small heads' layer 2 runs in fp32 from the caller's tensors
    }
    p.start[m] = total; p.count = m;
    return launch_k(tc_pack_weights_kernel, (total + 255) / 256, 256, 0, st, kOrdinary, p);
}

// ---- fragments ----------------------------------------------------------------------------------------------------------
using wg::Frags;

// two values of row g (x0, x1 = columns c, c + 1) and the same columns of row g + 8 (y0, y1), in accumulator block j,
// -> the A fragment slots they occupy
template <int NS>
__device__ __forceinline__ void put_block(Frags<NS>& a, int j, float x0, float x1, float y0, float y1) {
    const int s = j >> 1, o = (j & 1) * 2;
    wg::f16_split2(x0, x1, a.hi[s][o], a.lo[s][o]);
    wg::f16_split2(y0, y1, a.hi[s][o + 1], a.lo[s][o + 1]);
}

// D[64 x N] = A * B^T, three products; B = (hi | lo) K-major image with `bcols` columns
template <int N, int NS>
__device__ __forceinline__ void gemm3(float (&d)[N / 2], const Frags<NS>& a, uint32_t b_hi, uint32_t b_lo, uint32_t bcols) {
    const uint64_t dh = wg::desc_kmajor(b_hi, bcols, TcArith::EPC), dl = wg::desc_kmajor(b_lo, bcols, TcArith::EPC);
    wg::fence_regs(d);
    wg::fence();
#pragma unroll
    for (int p = 0; p < 3; ++p) {
#pragma unroll
        for (int s = 0; s < NS; ++s) {
            const uint64_t bd = ((p == 1) ? dl : dh) + (uint64_t)(16 * s);      // + 256 bytes per slice
            const uint32_t acc = (p > 0 || s > 0) ? 1u : 0u;
            wg::mma_f16_rs<N, 0>(d, p == 0 ? a.lo[s] : a.hi[s], bd, acc);
        }
    }
    wg::commit();
    wg::wait_all();
    wg::fence_regs(d);
}

// bias + ReLU of a 64 x 128 accumulator -> next A operand; sign bits of rows g / g + 8 (4 words each, complete for every lane
// of the quad); running maximum of the converted values
__device__ __forceinline__ void relu_to_frags(const float (&d)[64], float inv, const float* __restrict__ bias, int t, Frags<128 / TcArith::KS>& a,
                                              uint32_t (&b0)[4], uint32_t (&b1)[4], float& mx) {
#pragma unroll
    for (int w = 0; w < 4; ++w) { b0[w] = 0u; b1[w] = 0u; }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * t;
        const float2 bb = *reinterpret_cast<const float2*>(bias + c);
        const float x0 = fmaf(d[4 * j], inv, bb.x), x1 = fmaf(d[4 * j + 1], inv, bb.y);
        const float y0 = fmaf(d[4 * j + 2], inv, bb.x), y1 = fmaf(d[4 * j + 3], inv, bb.y);
        const int sh = 8 * (j & 3) + 2 * t;
        b0[j >> 2] |= ((x0 > 0.f ? 1u : 0u) | (x1 > 0.f ? 2u : 0u)) << sh;
        b1[j >> 2] |= ((y0 > 0.f ? 1u : 0u) | (y1 > 0.f ? 2u : 0u)) << sh;
        const float r0 = fmaxf(x0, 0.f), r1 = fmaxf(x1, 0.f), r2 = fmaxf(y0, 0.f), r3 = fmaxf(y1, 0.f);
        mx = fmaxf(mx, fmaxf(fmaxf(r0, r1), fmaxf(r2, r3)));
        put_block(a, j, r0, r1, r2, r3);
    }
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        b0[w] |= __shfl_xor_sync(0xffffffffu, b0[w], 1); b0[w] |= __shfl_xor_sync(0xffffffffu, b0[w], 2);
        b1[w] |= __shfl_xor_sync(0xffffffffu, b1[w], 1); b1[w] |= __shfl_xor_sync(0xffffffffu, b1[w], 2);
    }
}

// lane t of the quad stores word t of both rows' 128 sign bits: [slot][N][4 words], word w = hidden units [32w, 32w + 32)
__device__ __forceinline__ void store_bits(uint32_t* base, int slot, int64_t n, int64_t g0, int64_t g1, int t, const uint32_t (&b0)[4],
                                           const uint32_t (&b1)[4]) {
    const uint32_t w0 = t == 0 ? b0[0] : t == 1 ? b0[1] : t == 2 ? b0[2] : b0[3];
    const uint32_t w1 = t == 0 ? b1[0] : t == 1 ? b1[1] : t == 2 ? b1[2] : b1[3];
    if (g0 < n) base[((size_t)slot * (size_t)n + (size_t)g0) * 4 + t] = w0;
    if (g1 < n) base[((size_t)slot * (size_t)n + (size_t)g1) * 4 + t] = w1;
}

__device__ __forceinline__ void mbar_arrive(void* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// MODE as deform_kernel's (g4d_geom.cu): 0 deform only, 1 fused with M = 16 SH coefficients, 2 fused with M < 16
// NWG consumer warpgroups of 64 Gaussians each (tc_warpgroups).  tw is __grid_constant__: the W1 ring indexes tw.w1[] at run
// time, and nvcc would otherwise copy a parameter struct of 128 bytes or less to local memory to do so.
template <int NWG, int MODE, int C, int L, bool SAVE>
__global__ void __launch_bounds__(NWG * 128, 1)
deform_tc_kernel(DeformDesc d, const __grid_constant__ TcWeights tw, TcSmem Ls, const CameraDev* __restrict__ camp, int64_t n, DeformIO io) {
    using A = TcArith;
    constexpr int F = C * L, NS0 = F / A::KS, NS1 = 128 / A::KS, TM = 64 * NWG, NT = 128 * NWG;
    static_assert(F % 16 == 0 && F <= 64, "feature width must be 32, 48 or 64");
    constexpr float kInvL0 = A::SA / (A::SF * A::SW), kInvH = 1.f / (A::SA * A::SW), kInvHS = 1.f / A::SW;
    extern __shared__ __align__(128) uint8_t smem[];   // (every operand image and barrier is placed at a multiple of 128 B)
    __shared__ CameraDev cam;
    const int tid = threadIdx.x, wgi = tid >> 7, t128 = tid & 127, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int r0 = ((t128 >> 5) << 4) + g, r1 = r0 + 8;          // rows of this lane inside the warpgroup's 64
    float* sBias = reinterpret_cast<float*>(smem + Ls.bias);     // b0 * SA [128] | b1[5][128] (SH head * SA) | b2s[4][4] | b2sh[48]
    float4* sW2s = reinterpret_cast<float4*>(smem + Ls.w2s);     // [4 small heads][128 hidden]: (W2[0][j], W2[1][j], W2[2][j], W2[3][j])
    float* stage = reinterpret_cast<float*>(smem + Ls.stage) + wgi * 64 * kStageCols;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Ls.bars);
    uint64_t *bar_w0 = bars, *bar_full = bars + 1, *bar_empty = bars + 3;
    for (int i = tid; i < 128; i += NT) sBias[i] = __ldg(d.b0 + i) * A::SA;
    for (int i = tid; i < 64; i += NT) sBias[128 + G4D_NUM_HEADS * 128 + i] = 0.f;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        for (int i = tid; i < 128; i += NT) sBias[128 + h * 128 + i] = __ldg(d.b1[h] + i) * (h == 4 ? A::SA : 1.f);
        if (h < 4) {
            const int ko = head_out(h);
            for (int j = tid; j < 128; j += NT)
                sW2s[h * 128 + j] = make_float4(__ldg(d.w2[h] + j), ko > 1 ? __ldg(d.w2[h] + 128 + j) : 0.f,
                                               ko > 2 ? __ldg(d.w2[h] + 256 + j) : 0.f, ko > 3 ? __ldg(d.w2[h] + 384 + j) : 0.f);
        }
    }
    __syncthreads();      // (the zero fill of the b2 block above must land before the per-head values)
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        for (int i = tid; i < head_out(h); i += NT) sBias[128 + G4D_NUM_HEADS * 128 + (h < 4 ? 4 * h : 16) + i] = __ldg(d.b2[h] + i);
    }
    if (tid == 0) {
        mbar_init(bar_w0, 1);
        mbar_init(bar_full, 1); mbar_init(bar_full + 1, 1);
        mbar_init(bar_empty, 4 * NWG); mbar_init(bar_empty + 1, 4 * NWG);
        fence_barrier_init();
    }
    pdl_wait();           // from here on: the camera, the staged features
    pdl_trigger();
    if (MODE != 0) stage_cameras(&cam, &camp, 1);
    __syncthreads();

    const bool hsh = d.head_mask & G4D_HEAD_SHS;
    const int m_heads = __popc(d.head_mask & 31);
    uint32_t hseq = 0;                         // head of position k (3 bits each): the small heads in order, the SH head last
    {
        int k = 0;
        for (int h = 0; h < G4D_NUM_HEADS; ++h)
            if (d.head_mask & (1 << h)) hseq |= (uint32_t)h << (3 * k++);
    }
    const int64_t ntiles = (n + TM - 1) / TM;
    const int64_t my_tiles = (int64_t)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const uint32_t per_tile = (uint32_t)m_heads, total_items = (uint32_t)my_tiles * per_tile;
    // W1 ring: item u = (tile, head position) in consumption order, slot u & 1; thread 0 loads one item ahead
    auto issue = [&](uint32_t u) {
        const uint32_t s = u & 1u;
        if (u >= 2) mbar_wait(bar_empty + s, ((u >> 1) - 1u) & 1u);
        const int h = (int)((hseq >> (3 * (u % per_tile))) & 7u);
        mbar_expect_tx(bar_full + s, Ls.slot_bytes);
        tma_bulk_g2s(smem + Ls.w1 + s * Ls.slot_bytes, tw.w1[h], Ls.slot_bytes, bar_full + s);
    };
    if (tid == 0) {
        const uint32_t w0b = 2u * 128u * F * A::ES, w2b = hsh ? 2u * 48u * 128u * A::ES : 0u;
        mbar_expect_tx(bar_w0, w0b + w2b);
        tma_bulk_g2s(smem + Ls.w0, tw.w0, w0b, bar_w0);
        if (hsh) tma_bulk_g2s(smem + Ls.w2, tw.w2[4], w2b, bar_w0);
        if (total_items) issue(0);
    }
    __syncwarp();
    mbar_wait(bar_w0, 0);
    const uint32_t sW0 = wg::smem_addr(smem + Ls.w0), sW1 = wg::smem_addr(smem + Ls.w1), sW2 = wg::smem_addr(smem + Ls.w2);
    const float* b2s = sBias + 128 + G4D_NUM_HEADS * 128;
    float mx = 0.f;        // running maximum of every value converted to f16 (range check), in operand units
    uint32_t u = 0;
    const bool dbg = tw.dbg && tid == 0;      // G4D_OPT_TC_DEBUG: cycles of the whole kernel / spent waiting for W1 images
    const long long t_start = dbg ? clock64() : 0;
    long long t_wait = 0;

    for (int64_t it = 0; it < my_tiles; ++it) {
        const int64_t tile = (int64_t)blockIdx.x + it * gridDim.x;
        const int64_t row0 = tile * TM + wgi * 64, g0 = row0 + r0, g1 = row0 + r1;
        // ---- layer 0: D = feat W0^T, the features ([N][F] fp32 from deform_features_kernel) loaded as A fragments
        float acc[64];
        {
            Frags<NS0> x;
            const float* f0 = tw.feat + g0 * F;
            const float* f1 = tw.feat + g1 * F;
#pragma unroll
            for (int s = 0; s < NS0; ++s) {
                float v[8];   // (row g: c, c + 1 | row g + 8: c, c + 1) for the two column pairs of the slice
#pragma unroll
                for (int hlf = 0; hlf < 2; ++hlf) {
                    const int c = 16 * s + 8 * hlf + 2 * t;
                    const float2 p0 = g0 < n ? __ldg(reinterpret_cast<const float2*>(f0 + c)) : make_float2(0.f, 0.f);
                    const float2 p1 = g1 < n ? __ldg(reinterpret_cast<const float2*>(f1 + c)) : make_float2(0.f, 0.f);
                    v[4 * hlf] = p0.x * A::SF; v[4 * hlf + 1] = p0.y * A::SF; v[4 * hlf + 2] = p1.x * A::SF; v[4 * hlf + 3] = p1.y * A::SF;
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) mx = fmaxf(mx, fabsf(v[e]));
                wg::f16_split2(v[0], v[1], x.hi[s][0], x.lo[s][0]);
                wg::f16_split2(v[2], v[3], x.hi[s][1], x.lo[s][1]);
                wg::f16_split2(v[4], v[5], x.hi[s][2], x.lo[s][2]);
                wg::f16_split2(v[6], v[7], x.hi[s][3], x.lo[s][3]);
            }
            gemm3<128, NS0>(acc, x, sW0, sW0 + 128u * F * A::ES, F);
        }
        // ---- epilogue 0: a1 = relu(D / s + b0) -> A fragments (pre-scaled by SA); sign bits for the backward
        Frags<NS1> a1;
        {
            uint32_t bw0[4], bw1[4];
            relu_to_frags(acc, kInvL0, sBias, t, a1, bw0, bw1, mx);
            if (SAVE) store_bits(tw.relu_bits, 0, n, g0, g1, t, bw0, bw1);
        }
        if (t == 0) {
#pragma unroll
            for (int j = 0; j < 11; ++j) { stage[r0 * kStageCols + j] = 0.f; stage[r1 * kStageCols + j] = 0.f; }
        }
#pragma unroll 1
        for (int k = 0; k < m_heads; ++k) {
            const int h = (int)((hseq >> (3 * k)) & 7u);
            // ---- layer 1: D = a1 W1^T, W1 out of the ring
            {
                if (tid == 0 && u + 1 < total_items) issue(u + 1);
                __syncwarp();
                const uint32_t s = u & 1u;
                const long long t0 = dbg ? clock64() : 0;
                mbar_wait(bar_full + s, (u >> 1) & 1u);
                if (dbg) t_wait += clock64() - t0;
                const uint32_t b = sW1 + s * Ls.slot_bytes;
                gemm3<128, NS1>(acc, a1, b, b + Ls.slot_bytes / 2, 128);
                if (lane == 0) mbar_arrive(bar_empty + s);      // this warp's MMAs have retired: the slot may be refilled
                ++u;
            }
            uint32_t bw0[4], bw1[4];
            if (h < 4) {
                // ---- small head: a2 = relu(D / s + b1), layer 2 (<= 4 outputs) in exact fp32; each lane sums its 32 hidden
                //      units, the quad completes the row
                const float* b1 = sBias + 128 + h * 128;
                const float4* w2 = sW2s + h * 128;
                float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int w = 0; w < 4; ++w) { bw0[w] = 0u; bw1[w] = 0u; }
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int c = 8 * j + 2 * t;
                    const float2 bb = *reinterpret_cast<const float2*>(b1 + c);
                    const float x0 = fmaf(acc[4 * j], kInvH, bb.x), x1 = fmaf(acc[4 * j + 1], kInvH, bb.y);
                    const float y0 = fmaf(acc[4 * j + 2], kInvH, bb.x), y1 = fmaf(acc[4 * j + 3], kInvH, bb.y);
                    const int sh = 8 * (j & 3) + 2 * t;
                    bw0[j >> 2] |= ((x0 > 0.f ? 1u : 0u) | (x1 > 0.f ? 2u : 0u)) << sh;
                    bw1[j >> 2] |= ((y0 > 0.f ? 1u : 0u) | (y1 > 0.f ? 2u : 0u)) << sh;
                    const float4 wa = w2[c], wb = w2[c + 1];
                    const float ax = fmaxf(x0, 0.f), ay = fmaxf(x1, 0.f), bx = fmaxf(y0, 0.f), by = fmaxf(y1, 0.f);
                    o0[0] = fmaf(ay, wb.x, fmaf(ax, wa.x, o0[0])); o0[1] = fmaf(ay, wb.y, fmaf(ax, wa.y, o0[1]));
                    o0[2] = fmaf(ay, wb.z, fmaf(ax, wa.z, o0[2])); o0[3] = fmaf(ay, wb.w, fmaf(ax, wa.w, o0[3]));
                    o1[0] = fmaf(by, wb.x, fmaf(bx, wa.x, o1[0])); o1[1] = fmaf(by, wb.y, fmaf(bx, wa.y, o1[1]));
                    o1[2] = fmaf(by, wb.z, fmaf(bx, wa.z, o1[2])); o1[3] = fmaf(by, wb.w, fmaf(bx, wa.w, o1[3]));
                }
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    o0[o] += __shfl_xor_sync(0xffffffffu, o0[o], 1); o0[o] += __shfl_xor_sync(0xffffffffu, o0[o], 2);
                    o1[o] += __shfl_xor_sync(0xffffffffu, o1[o], 1); o1[o] += __shfl_xor_sync(0xffffffffu, o1[o], 2);
                }
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    bw0[w] |= __shfl_xor_sync(0xffffffffu, bw0[w], 1); bw0[w] |= __shfl_xor_sync(0xffffffffu, bw0[w], 2);
                    bw1[w] |= __shfl_xor_sync(0xffffffffu, bw1[w], 1); bw1[w] |= __shfl_xor_sync(0xffffffffu, bw1[w], 2);
                }
                if (t == 0) {
                    const int ko = head_out(h), col = head_col(h);
#pragma unroll
                    for (int o = 0; o < 4; ++o) {
                        if (o < ko) {
                            stage[r0 * kStageCols + col + o] = o0[o] + b2s[4 * h + o];
                            stage[r1 * kStageCols + col + o] = o1[o] + b2s[4 * h + o];
                        }
                    }
                }
            } else {
                // ---- SH head (always last: a1 is dead once its layer-1 GEMM has retired): hidden layer -> A fragments,
                //      layer 2 as a GEMM with N = 48, SH deltas to the stage
                relu_to_frags(acc, kInvHS, sBias + 128 + 4 * 128, t, a1, bw0, bw1, mx);
                float acc2[24];
                gemm3<48, NS1>(acc2, a1, sW2, sW2 + 48u * 128u * A::ES, 128);
                const float* b2sh = b2s + 16;
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    const int c = 8 * j + 2 * t;
                    stage[r0 * kStageCols + 11 + c] = fmaf(acc2[4 * j], kInvH, b2sh[c]);
                    stage[r0 * kStageCols + 12 + c] = fmaf(acc2[4 * j + 1], kInvH, b2sh[c + 1]);
                    stage[r1 * kStageCols + 11 + c] = fmaf(acc2[4 * j + 2], kInvH, b2sh[c]);
                    stage[r1 * kStageCols + 12 + c] = fmaf(acc2[4 * j + 3], kInvH, b2sh[c + 1]);
                }
            }
            if (SAVE) store_bits(tw.relu_bits, 1 + h, n, g0, g1, t, bw0, bw1);
        }
        // ---- per-Gaussian tail: threads 0-63 the geometry, 64-127 the colour of Gaussian (t128 & 63) of the warpgroup
        bar_sync(1 + wgi, 128);
        {
            const int row = t128 & 63;
            const int64_t gi = row0 + row;
            const float* o = stage + row * kStageCols;
            if (gi < n) {
                const Vec3 p{io.xyz[3 * gi] + o[0], io.xyz[3 * gi + 1] + o[1], io.xyz[3 * gi + 2] + o[2]};
                if (t128 < 64) {
                    float sl[3] = {0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f}, ol = 0.f;
                    if (io.scaling) { sl[0] = io.scaling[3 * gi]; sl[1] = io.scaling[3 * gi + 1]; sl[2] = io.scaling[3 * gi + 2]; }
                    if (io.rotation) { const float4 r4 = *reinterpret_cast<const float4*>(io.rotation + 4 * gi); q[0] = r4.x; q[1] = r4.y; q[2] = r4.z; q[3] = r4.w; }
                    if (io.opacity) ol = io.opacity[gi];
                    sl[0] += o[3]; sl[1] += o[4]; sl[2] += o[5];
                    q[0] += o[6]; q[1] += o[7]; q[2] += o[8]; q[3] += o[9];
                    ol += o[10];
                    if (MODE == 0) {
                        io.out_xyz[3 * gi] = p.x; io.out_xyz[3 * gi + 1] = p.y; io.out_xyz[3 * gi + 2] = p.z;
                        if (io.out_scaling) { io.out_scaling[3 * gi] = sl[0]; io.out_scaling[3 * gi + 1] = sl[1]; io.out_scaling[3 * gi + 2] = sl[2]; }
                        if (io.out_rotation) *reinterpret_cast<float4*>(io.out_rotation + 4 * gi) = make_float4(q[0], q[1], q[2], q[3]);
                        if (io.out_opacity) io.out_opacity[gi] = ol;
                    } else {
                        fused_finish_geometry(cam, io, gi, p, sl, q, ol);
                    }
                } else {
                    float dsh[48];
#pragma unroll
                    for (int j = 0; j < 48; ++j) dsh[j] = hsh ? o[11 + j] : 0.f;
                    if (MODE == 0) {
                        if (io.out_shs && hsh) {
#pragma unroll
                            for (int j = 0; j < 48; j += 4) {
                                const float4 b = *reinterpret_cast<const float4*>(io.sh.shs + gi * 48 + j);
                                *reinterpret_cast<float4*>(io.out_shs + gi * 48 + j) = make_float4(b.x + dsh[j], b.y + dsh[j + 1], b.z + dsh[j + 2], b.w + dsh[j + 3]);
                            }
                        }
                    } else {
                        if (MODE == 1) fused_finish_colour(cam, io, gi, p, hsh, dsh);
                        else fused_finish_colour_reduced(cam, io, gi, p);
                    }
                }
            }
        }
        bar_sync(1 + wgi, 128);   // the stage is read before the next tile's deltas overwrite it
    }
    // range check of everything that went through an f16 conversion (already in operand units)
    if (mx >= kF16Max && tw.status) *reinterpret_cast<volatile uint32_t*>(tw.status) = 1u;
    if (dbg) { tw.dbg[blockIdx.x * 12] = clock64() - t_start; tw.dbg[blockIdx.x * 12 + 1] = t_wait; tw.dbg[blockIdx.x * 12 + 2] = NWG; }
}

// ---- spatial walk order of the gather: a permutation of [0, n) in Z (Morton) order of each Gaussian's cell on a
// kOrderGrid^3 grid over the normalised HexPlane coordinates.  Counting sort by cell: count (the atomic also hands each
// Gaussian its rank inside its cell, in no particular order), exclusive scan of the counts, scatter.
constexpr int kOrderBits = 6;   // 64 cells per axis: about as fine as level 0 of the planes (dynerf: 64)
static_assert(kOrderCells == 1 << (3 * kOrderBits) && kOrderCells / 1024 == 256, "one scan CTA per 1024 cells, 256 of them");

G4D_D uint32_t order_cell(const AabbNorm& nrm, const float* __restrict__ xyz, int64_t g) {
    constexpr float hi = (float)((1 << kOrderBits) - 1);
    uint32_t code = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        // clamped as make_tap clamps: points outside the aabb, on its faces or with a NaN coordinate land in a valid cell
        const float x = fminf(fmaxf((nrm(a, xyz[3 * g + a]) + 1.f) * (0.5f * (hi + 1.f)), 0.f), hi);
        const uint32_t c = (uint32_t)x;
#pragma unroll
        for (int b = 0; b < kOrderBits; ++b) code |= ((c >> b) & 1u) << (3 * b + a);
    }
    return code;
}

// exclusive prefix sum of v over the 256 threads of the block (sm: 8 words of shared memory)
G4D_D uint32_t block_exclusive_scan_256(uint32_t v, uint32_t* sm) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) sm[w] = inc;
    __syncthreads();
    uint32_t base = 0;
    for (int i = 0; i < w; ++i) base += sm[i];
    return base + inc - v;
}

__global__ void __launch_bounds__(256) order_count_kernel(const float* __restrict__ aabb, int64_t n, const float* __restrict__ xyz,
                                                         GatherOrderBuffers b) {
    const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (g >= n) return;
    const uint32_t c = order_cell(AabbNorm(aabb), xyz, g);
    b.key[g] = make_uint2(c, atomicAdd(b.cell_start + c, 1u));
}

// per block of 1024 cells: counts -> exclusive prefix inside the block, and the block's total
__global__ void __launch_bounds__(256) order_scan_kernel(GatherOrderBuffers b) {
    __shared__ uint32_t sm[8];
    uint4* p = reinterpret_cast<uint4*>(b.cell_start) + (size_t)blockIdx.x * 256 + threadIdx.x;
    const uint4 c = *p;
    const uint32_t s = c.x + c.y + c.z + c.w;
    const uint32_t e = block_exclusive_scan_256(s, sm);
    *p = make_uint4(e, e + c.x, e + c.x + c.y, e + c.x + c.y + c.z);
    if (threadIdx.x == 255) b.block_total[blockIdx.x] = e + s;
}

__global__ void __launch_bounds__(256) order_scatter_kernel(int64_t n, GatherOrderBuffers b) {
    __shared__ uint32_t sm[8], base[256];
    base[threadIdx.x] = block_exclusive_scan_256(b.block_total[threadIdx.x], sm);
    __syncthreads();
    const int64_t g = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (g >= n) return;
    const uint2 k = b.key[g];
    b.order[base[k.x >> 10] + b.cell_start[k.x] + k.y] = (uint32_t)g;
}

cudaError_t launch_gather_order(const float* aabb, int64_t n, const float* xyz, const GatherOrderBuffers& b, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(b.cell_start, 0, (size_t)kOrderCells * 4, st);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((n + 255) / 256);
    if ((e = launch_k(order_count_kernel, grid, 256, 0, st, kOrdinary, aabb, n, xyz, b)) != cudaSuccess) return e;
    if ((e = launch_k(order_scan_kernel, kOrderCells / 1024, 256, 0, st, kOrdinary, b)) != cudaSuccess) return e;
    return launch_k(order_scatter_kernel, grid, 256, 0, st, kOrdinary, n, b);
}

// ---- HexPlane gather at full occupancy: C/4 threads per Gaussian, one channel vector each -> feat [N][F] fp32 -----------
// The gather of every path (FFMA and tensor-core network, forward and backward): the forward launches it dependent on
// collapse_time_rows, the backward as an ordinary launch.  PER_ROW: Gaussian g is sampled at its own time d.times[g] (no
// collapsed rows).  Thread
// group j gathers Gaussian order[j] (j itself when order is NULL): in spatial order the 8 Gaussians of a warp, and the warps
// of an SM, tap neighbouring plane texels and share them in L1.  feat[g] depends on xyz[g] (and times[g]) alone, so any order
// gives the same bits.
template <int C4, bool PER_ROW>
__global__ void __launch_bounds__(256) deform_features_kernel(DeformDesc d, int64_t n, const float* __restrict__ xyz,
                                                              const uint32_t* __restrict__ order, float* __restrict__ feat) {
    pdl_wait();         // the collapsed time rows come from the previous kernel of the stream
    pdl_trigger();
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t j = t / C4;
    const int v = (int)(t % C4);
    if (j >= n) return;
    const int64_t g = order ? (int64_t)__ldg(order + j) : j;
    const AabbNorm nrm(d.aabb);
    float pcs[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) pcs[a] = nrm(a, xyz[3 * g + a]);
    const float tg = PER_ROW ? __ldg(d.times + g) : 0.f;
    for (int l = 0; l < d.levels; ++l) {
        Tap1D tx[PER_ROW ? 4 : 3];
#pragma unroll
        for (int a = 0; a < 3; ++a) tx[a] = make_tap(pcs[a], d.res[l][a]);
        if (PER_ROW) tx[PER_ROW ? 3 : 0] = make_tap(tg, d.res[l][3]);
        *reinterpret_cast<float4*>(feat + g * d.F + l * d.C + 4 * v) = sample_vector<PER_ROW>(d.planes[l], d.trow[l], d.res[l], tx, v, C4);
    }
}

cudaError_t launch_deform_features(const DeformDesc& d, int64_t n, const float* xyz, const uint32_t* order, float* feat, bool pdl,
                                   cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const int C4 = d.C / 4;
    const unsigned grid = (unsigned)((n * C4 + 255) / 256);
    switch (C4) {   // every channel width the C-ABI takes: C = 4 .. 32
#define G4D_GATHER_CASE(K)                                                                                                  \
        case K: return launch_k(d.times ? deform_features_kernel<K, true> : deform_features_kernel<K, false>, grid, 256, 0, st,   \
                                pdl ? kPdl : kOrdinary, d, n, xyz, order, feat);
        G4D_GATHER_CASE(1) G4D_GATHER_CASE(2) G4D_GATHER_CASE(3) G4D_GATHER_CASE(4)
        G4D_GATHER_CASE(5) G4D_GATHER_CASE(6) G4D_GATHER_CASE(7) G4D_GATHER_CASE(8)
#undef G4D_GATHER_CASE
    }
    return cudaErrorInvalidValue;
}

bool tc_deform_supported(const G4DDeformParams& prm) {
    const int C = prm.channels, L = prm.levels;
    if (prm.net_width != 128 || prm.depth > 1) return false;   // no trunk layers (deep trunks: the FFMA kernels)
    if (!((C == 16 && (L == 2 || L == 3)) || (C == 32 && L == 2))) return false;
    return tc_warpgroups(C * L, (prm.head_mask & G4D_HEAD_SHS) != 0) != 0;
}

template <int NWG, int MODE, int C, int L>
static cudaError_t launch_deform_tc_t(const DeformDesc& d, const TcWeights& tw, const CameraDev* cam, int64_t n, const DeformIO& io,
                                      int sm_count, cudaStream_t st) {
    const TcSmem Ls = tc_smem_layout(NWG, d.F, (d.head_mask & G4D_HEAD_SHS) != 0);
    const size_t bytes = Ls.total;
    const int64_t ntiles = (n + 64 * NWG - 1) / (64 * NWG);
    const int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
    return launch_k(tw.relu_bits ? deform_tc_kernel<NWG, MODE, C, L, true> : deform_tc_kernel<NWG, MODE, C, L, false>, grid, NWG * 128,
                    bytes, st, kPdl, d, tw, Ls, cam, n, io);
}

cudaError_t launch_deform_tc(const DeformDesc& d, const TcWeights& tw, int mode, const CameraDev* cam, int64_t n,
                             const DeformIO& io, int sm_count, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    if (!tw.feat) return cudaErrorInvalidValue;
    const int nwg = tc_warpgroups(d.F, (d.head_mask & G4D_HEAD_SHS) != 0);
    // the (C, L, warpgroups) that tc_warpgroups can choose: F = 32 always fits three warpgroups, F = 48 / 64 fit three
    // without the SH head and two with it
#define G4D_TC_CASE(NW, CC, LL)                                                                                              \
    if (nwg == NW && d.C == CC && d.levels == LL)                                                                            \
        return mode == 0                   ? launch_deform_tc_t<NW, 0, CC, LL>(d, tw, cam, n, io, sm_count, st)             \
               : io.sh.m == kShCoeffs ? launch_deform_tc_t<NW, 1, CC, LL>(d, tw, cam, n, io, sm_count, st)             \
                                      : launch_deform_tc_t<NW, 2, CC, LL>(d, tw, cam, n, io, sm_count, st);
    G4D_TC_CASE(3, 16, 2)
    G4D_TC_CASE(3, 16, 3)
    G4D_TC_CASE(2, 16, 3)
    G4D_TC_CASE(3, 32, 2)
    G4D_TC_CASE(2, 32, 2)
#undef G4D_TC_CASE
    return cudaErrorInvalidValue;
}

}  // namespace g4d
