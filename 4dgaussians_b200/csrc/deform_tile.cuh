// deform_tile.cuh -- deformation MLP of the FFMA path for a tile of TG Gaussians held in shared memory.
//
// Algorithm (verified spec: SURVEY.md Appendix B):
//   /root/reference/scene/hexplane.py:19-20,73-106,160-183   normalize_aabb, 6-plane bilinear product, level concat
//   /root/reference/scene/deformation.py:67-83               hidden = Linear(F->Wd)(feat)      (no activation)
//   /root/reference/scene/deformation.py:55-60               defor_depth D > 1: hidden = W_j relu(hidden) + b_j, j < D
//   /root/reference/scene/deformation.py:97-148              heads ReLU-Linear-ReLU-Linear, residual add
//
// Layout decisions (DESIGN.md §3):
//   * the HexPlane features arrive gathered, feat [N][F] (deform_features_kernel, the gather of every path); a tile of
//     them is loaded into a0;
//   * a CTA of 256 threads owns TG Gaussians; activations live in shared memory row-major [TG][K+4];
//     W0^T and one W x W image are staged in shared memory ([K][Wd]); the W x W slot takes each trunk layer's W_j^T and
//     then each head's W1^T by a TMA bulk copy that overlaps the previous GEMM's epilogue; each thread accumulates an
//     RM x (Wd/16) register tile with FFMA.
#pragma once
#include "g4d_common.cuh"
#include "hexplane.cuh"

namespace g4d {

constexpr int kDeformThreads = 256;

struct DeformDesc {
    int levels, C, F, WD, head_mask;
    int res[G4D_MAX_LEVELS][4];
    const float* planes[G4D_MAX_LEVELS][6];   // channel-last
    const float* trow[G4D_MAX_LEVELS][3];     // collapsed time rows for planes 2,4,5: [res[c0]][C]
    const float* aabb;                        // [2][3]
    const float* w0t;                         // packed [F][WD]
    const float* b0;                          // [WD]
    const float* w1t[G4D_NUM_HEADS];          // packed [WD][WD]
    const float* b1[G4D_NUM_HEADS];
    const float* w2[G4D_NUM_HEADS];           // torch layout [k][WD]
    const float* b2[G4D_NUM_HEADS];
    int ntrunk;                               // trunk layers behind W0: max(defor_depth, 1) - 1
    const float* wtt[G4D_MAX_DEPTH - 1];      // packed [WD][WD]: W_j^T of trunk layer j = 1 .. ntrunk
    const float* bt[G4D_MAX_DEPTH - 1];       // [WD]
    const float* times;                       // [N] one time per Gaussian (the per-row gather and scatter; trow unused),
                                              // or NULL: every Gaussian at the time of the collapsed rows trow
};

// Hands out consecutive regions of a shared-memory layout in the order they are taken, as offsets in floats, each region
// rounded up to 4 floats so that every one starts 16-byte aligned (float4 access).  off ends as the layout's total.
struct SmemFloats {
    int off = 0;
    int take(int n) { const int o = off; off += (n + 3) & ~3; return o; }
};

// shared-memory carve-up (offsets in floats), computed on the host by deform_smem_layout()
struct DeformSmem {
    int w0t, b0, w1t, b1, bt, w2, b2, a0, a1, a2, out, in, mbar, total_floats;
    int lda0, lda1, w2_stride;
    int w2_off[G4D_NUM_HEADS];   // row offset (in rows of w2_stride floats) of head h inside w2
};

inline DeformSmem deform_smem_layout(int TG, int F, int WD, int head_mask, int ntrunk) {
    DeformSmem s{};
    SmemFloats m;
    s.lda0 = F + 4; s.lda1 = WD + 4; s.w2_stride = WD + 4;
    s.w0t = m.take(F * WD);
    s.b0 = m.take(WD);
    s.w1t = m.take(WD * WD);
    s.b1 = m.take(G4D_NUM_HEADS * WD);
    s.bt = m.take(ntrunk * WD);
    int rows = 0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) { s.w2_off[h] = rows; if (head_mask & (1 << h)) rows += head_out(h); }
    s.w2 = m.take(rows * s.w2_stride);
    s.b2 = m.take(64);
    s.a0 = m.take(TG * s.lda0);
    s.a1 = m.take(TG * s.lda1);
    s.a2 = m.take(TG * s.lda1);
    s.out = m.take(TG * 60);
    s.in = m.take(TG * 12);
    s.mbar = m.take(4);
    s.total_floats = m.off;
    return s;
}

#if defined(__CUDACC__)

// ---- mbarrier + TMA bulk copy (1-D) helpers --------------------------------------------------------
G4D_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
G4D_D void mbar_init(void* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
G4D_D void mbar_expect_tx(void* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
G4D_D void mbar_wait(void* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
G4D_D void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, void* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
G4D_D void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---- register-tiled shared-memory GEMM --------------------------------------------------------------
// acc[r][c] (+)= sum_k A[ty*RM + r][k] * B[k][col(c)],  col(c) = (c/4)*64 + tx*4 + (c%4)
template <int RM, int CG>
G4D_D void tile_gemm(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, int K, int ty, int tx,
                     float (&acc)[RM][CG * 4]) {
    const float* arow = A + ty * RM * lda;
    const float* bcol = B + tx * 4;
#pragma unroll 1
    for (int k = 0; k < K; k += 4) {
        float4 a[RM];
#pragma unroll
        for (int r = 0; r < RM; ++r) a[r] = *reinterpret_cast<const float4*>(arow + r * lda + k);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            float4 b[CG];
#pragma unroll
            for (int c = 0; c < CG; ++c) b[c] = *reinterpret_cast<const float4*>(bcol + (k + kk) * ldb + c * 64);
#pragma unroll
            for (int r = 0; r < RM; ++r) {
                const float av = kk == 0 ? a[r].x : kk == 1 ? a[r].y : kk == 2 ? a[r].z : a[r].w;
#pragma unroll
                for (int c = 0; c < CG; ++c) {
                    acc[r][c * 4 + 0] = fmaf(av, b[c].x, acc[r][c * 4 + 0]);
                    acc[r][c * 4 + 1] = fmaf(av, b[c].y, acc[r][c * 4 + 1]);
                    acc[r][c * 4 + 2] = fmaf(av, b[c].z, acc[r][c * 4 + 2]);
                    acc[r][c * 4 + 3] = fmaf(av, b[c].w, acc[r][c * 4 + 3]);
                }
            }
        }
    }
}

// out[ty*RM + r][col] = act(acc + bias[col]);  RELU selects max(.,0)
template <int RM, int CG, bool RELU>
G4D_D void tile_store(float* __restrict__ O, int ldo, const float* __restrict__ bias, int ty, int tx,
                      const float (&acc)[RM][CG * 4]) {
#pragma unroll
    for (int c = 0; c < CG; ++c) {
        const float4 bv = *reinterpret_cast<const float4*>(bias + c * 64 + tx * 4);
#pragma unroll
        for (int r = 0; r < RM; ++r) {
            float4 v = make_float4(acc[r][c * 4 + 0] + bv.x, acc[r][c * 4 + 1] + bv.y, acc[r][c * 4 + 2] + bv.z,
                                   acc[r][c * 4 + 3] + bv.w);
            if (RELU) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            *reinterpret_cast<float4*>(O + (ty * RM + r) * ldo + c * 64 + tx * 4) = v;
        }
    }
}

// Last layer of a head: out[g][col0 + o] = b2[o] + sum_j A2[g][j] * W2[o][j]   (W2 rows padded to w2_stride)
template <int TG>
G4D_D void head_output(const float* __restrict__ A2, int lda, const float* __restrict__ W2, int w2_stride,
                       const float* __restrict__ b2, int kout, int WD, float* __restrict__ out, int col0) {
    if (kout <= 4) {
        for (int idx = threadIdx.x; idx < TG * 4; idx += kDeformThreads) {
            const int g = idx >> 2, o = idx & 3;
            if (o < kout) {
                const float* a = A2 + g * lda;
                const float* w = W2 + o * w2_stride;
                float acc0 = 0.f, acc1 = 0.f;
                for (int j = 0; j < WD; j += 8) {
                    const float4 a0 = *reinterpret_cast<const float4*>(a + j), a1 = *reinterpret_cast<const float4*>(a + j + 4);
                    const float4 w0 = *reinterpret_cast<const float4*>(w + j), w1 = *reinterpret_cast<const float4*>(w + j + 4);
                    acc0 = fmaf(a0.x, w0.x, acc0); acc0 = fmaf(a0.y, w0.y, acc0); acc0 = fmaf(a0.z, w0.z, acc0); acc0 = fmaf(a0.w, w0.w, acc0);
                    acc1 = fmaf(a1.x, w1.x, acc1); acc1 = fmaf(a1.y, w1.y, acc1); acc1 = fmaf(a1.z, w1.z, acc1); acc1 = fmaf(a1.w, w1.w, acc1);
                }
                out[g * 60 + col0 + o] = (acc0 + acc1) + b2[o];
            }
        }
    } else {   // kout == 48: thread (g, og) owns outputs og + 4*i
        for (int idx = threadIdx.x; idx < TG * 4; idx += kDeformThreads) {
            const int g = idx >> 2, og = idx & 3;
            const float* a = A2 + g * lda;
            float acc[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) acc[i] = 0.f;
            for (int j = 0; j < WD; j += 4) {
                const float4 av = *reinterpret_cast<const float4*>(a + j);
#pragma unroll
                for (int i = 0; i < 12; ++i) {
                    const float4 wv = *reinterpret_cast<const float4*>(W2 + (og + 4 * i) * w2_stride + j);
                    acc[i] = fmaf(av.x, wv.x, acc[i]); acc[i] = fmaf(av.y, wv.y, acc[i]);
                    acc[i] = fmaf(av.z, wv.z, acc[i]); acc[i] = fmaf(av.w, wv.w, acc[i]);
                }
            }
#pragma unroll
            for (int i = 0; i < 12; ++i) out[g * 60 + col0 + og + 4 * i] = acc[i] + b2[og + 4 * i];
        }
    }
}

// The W x W images one tile streams through the slot at L.w1t, in order: the trunk layers' W_j^T, then the active heads' W1^T.
G4D_D int wslot_images(const DeformDesc& d) { return d.ntrunk + __popc((unsigned)d.head_mask & ((1u << G4D_NUM_HEADS) - 1)); }
G4D_D const float* wslot_image(const DeformDesc& d, int i) {
    if (i < d.ntrunk) return d.wtt[i];
    i -= d.ntrunk;
    for (int h = 0; h < G4D_NUM_HEADS; ++h)
        if (d.head_mask & (1 << h)) { if (i == 0) return d.w1t[h]; --i; }
    return nullptr;
}
// thread 0: the bulk copy of image i of the tile's list into the slot
template <int WD>
G4D_D void wslot_issue(const DeformDesc& d, const DeformSmem& L, float* smem, int i) {
    mbar_expect_tx(smem + L.mbar, (uint32_t)(WD * WD * sizeof(float)));
    tma_bulk_g2s(smem + L.w1t, wslot_image(d, i), (uint32_t)(WD * WD * sizeof(float)), smem + L.mbar);
}

// Per-CTA one-time staging of the persistent weights (W0^T, biases, W2 of the active heads).
G4D_D void stage_persistent_weights(const DeformDesc& d, const DeformSmem& L, float* smem) {
    const int n0 = d.F * d.WD;
    for (int i = threadIdx.x * 4; i < n0; i += kDeformThreads * 4)
        *reinterpret_cast<float4*>(smem + L.w0t + i) = __ldg(reinterpret_cast<const float4*>(d.w0t + i));
    for (int i = threadIdx.x; i < d.WD; i += kDeformThreads) smem[L.b0 + i] = __ldg(d.b0 + i);
    for (int j = 0; j < d.ntrunk; ++j)
        for (int i = threadIdx.x; i < d.WD; i += kDeformThreads) smem[L.bt + j * d.WD + i] = __ldg(d.bt[j] + i);
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        for (int i = threadIdx.x; i < d.WD; i += kDeformThreads) smem[L.b1 + h * d.WD + i] = __ldg(d.b1[h] + i);
        const int ko = head_out(h);
        for (int i = threadIdx.x; i < ko * d.WD; i += kDeformThreads) {
            const int o = i / d.WD, j = i - o * d.WD;
            smem[L.w2 + (L.w2_off[h] + o) * L.w2_stride + j] = __ldg(d.w2[h] + i);
        }
        for (int i = threadIdx.x; i < ko; i += kDeformThreads) smem[L.b2 + L.w2_off[h] + i] = __ldg(d.b2[h] + i);
    }
}

// a0[g][0 .. F) = feat[base + g][0 .. F) for the tile's Gaussians g < rem, zero for the rows past n; the caller syncs.
template <int TG>
G4D_D void load_feature_tile(const float* __restrict__ feat, int F, int64_t base, int64_t rem, float* __restrict__ a0, int lda0) {
    const int F4 = F >> 2;
    for (int i = threadIdx.x; i < TG * F4; i += kDeformThreads) {
        const int g = i / F4, v = i - g * F4;
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (g < rem) val = __ldg(reinterpret_cast<const float4*>(feat + (base + g) * F + 4 * v));
        *reinterpret_cast<float4*>(a0 + g * lda0 + 4 * v) = val;
    }
}

// Runs the whole network for the TG Gaussians whose features are in smem[L.a0] (load_feature_tile).
// On return smem[L.out + g*60 + head_col(h) + o] holds the delta of every ACTIVE head (inactive: untouched).
// `phase` is the running mbarrier parity for the W x W staging slot (caller keeps it across tiles).
// PRE: thread 0 has already issued the bulk copy of image 0 of the tile's list (wslot_image): the first trunk layer's W_j^T,
// or with no trunk layer the first active head's W1^T.  Each image's GEMM issues the next one of the list -- past the last,
// image 0 again when prefetch_next_tile -- so the next copy overlaps the epilogue.
template <int TG, int WD>
G4D_D void deform_mlp_tile(const DeformDesc& d, const DeformSmem& L, float* smem, uint32_t& phase, bool prefetch_next_tile) {
    constexpr int RM = TG / 16, CG = WD / 64;
    const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
    void* bar = smem + L.mbar;
    const int nimg = wslot_images(d);
    auto prefetch_after = [&](int i) {   // thread 0, once everyone is done reading image i
        if (i + 1 < nimg) wslot_issue<WD>(d, L, smem, i + 1);
        else if (prefetch_next_tile) wslot_issue<WD>(d, L, smem, 0);
    };
    // the trunk ping-pongs between a1 and a2 and ends in a1, where the heads read relu(h_{D-1})
    float* cur = smem + ((d.ntrunk & 1) ? L.a2 : L.a1);

    {   // hidden = feat W0^T + b0 ; relu(hidden)  (every head and trunk layer starts with ReLU: deformation.py:55-65)
        float acc[RM][CG * 4];
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
        tile_gemm<RM, CG>(smem + L.a0, L.lda0, smem + L.w0t, WD, d.F, ty, tx, acc);
        tile_store<RM, CG, true>(cur, L.lda1, smem + L.b0, ty, tx, acc);
    }
    __syncthreads();
#pragma unroll 1
    for (int j = 0; j < d.ntrunk; ++j) {   // hidden = relu(hidden) W_j^T + b_j
        float* nxt = smem + (cur == smem + L.a1 ? L.a2 : L.a1);
        mbar_wait(bar, phase);   // W_j^T has landed
        phase ^= 1u;
        float acc[RM][CG * 4];
#pragma unroll
        for (int r = 0; r < RM; ++r)
#pragma unroll
            for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
        tile_gemm<RM, CG>(cur, L.lda1, smem + L.w1t, WD, WD, ty, tx, acc);
        __syncthreads();   // everyone is done reading W_j^T and cur
        if (threadIdx.x == 0) prefetch_after(j);
        tile_store<RM, CG, true>(nxt, L.lda1, smem + L.bt + j * WD, ty, tx, acc);
        __syncthreads();
        cur = nxt;
    }
    for (int h = 0, img = d.ntrunk; h < G4D_NUM_HEADS; ++h) {
        if (!(d.head_mask & (1 << h))) continue;
        mbar_wait(bar, phase);   // W1^T of head h has landed
        phase ^= 1u;
        {
            float acc[RM][CG * 4];
#pragma unroll
            for (int r = 0; r < RM; ++r)
#pragma unroll
                for (int c = 0; c < CG * 4; ++c) acc[r][c] = 0.f;
            tile_gemm<RM, CG>(smem + L.a1, L.lda1, smem + L.w1t, WD, WD, ty, tx, acc);
            __syncthreads();   // everyone is done reading W1^T (and the previous head's a2)
            if (threadIdx.x == 0) prefetch_after(img);   // overlap the next image's fetch with this head's epilogue
            ++img;
            tile_store<RM, CG, true>(smem + L.a2, L.lda1, smem + L.b1 + h * WD, ty, tx, acc);
        }
        __syncthreads();
        head_output<TG>(smem + L.a2, L.lda1, smem + L.w2 + L.w2_off[h] * L.w2_stride, L.w2_stride,
                        smem + L.b2 + L.w2_off[h], head_out(h), WD, smem + L.out, head_col(h));
        // no barrier needed here: the next head rewrites a2 only after its own GEMM + __syncthreads()
    }
    __syncthreads();
}

#endif  // __CUDACC__

}  // namespace g4d
