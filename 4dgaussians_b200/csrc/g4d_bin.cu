// g4d_bin.cu -- tile binning (SURVEY.md Appendix A.2) as TWO hand-written launches, no library sort, no host round trip:
//
//   bin_sort_kernel  (cooperative, persistent, one 1024-thread CTA per SM, grid-wide syncs between phases)
//       0. the keys are sorted as (depth bits - min) -- min / max of the visible Gaussians' depth bits are reduced by the
//          projection stage -- 24-27 significant bits instead of 32, i.e. 3 radix passes instead of 4
//       1. LSD radix sort (9-bit digits, stable) of the VISIBLE Gaussians by depth; the first pass compacts away the
//          invisible ones while it scatters.  Ties keep Gaussian-index order.                            -> perm[n_visible]
//       2. the depth-ordered list is cut into one chunk per CTA with equal numbers of tile instances (near Gaussians cover
//          many more tiles than far ones)                                                                  -> chunk_start
//       3. every chunk counts its instances per tile (shared-memory histogram)                            -> M[tile][chunk]
//       4. per tile: exclusive scan over the chunks (one warp per tile), then an exclusive scan over the tiles
//                                                                                                -> ranges[tile], R
//   bin_place_kernel (one 1024-thread CTA per chunk, tile rows processed in bands that fit shared memory)
//       every warp walks its share of the chunk IN DEPTH ORDER and drops each (Gaussian, tile) instance at
//       tile_start[tile] + M[tile][chunk] + (instances of earlier warps of the chunk) + (its own running count): a stable
//       counting placement.  Because the Gaussians arrive depth-sorted, every tile's segment comes out depth-sorted: the
//       reference's sort of R 64-bit (tile | depth) keys (6 radix passes over 12 B x R) is replaced by ONE 4-byte write per
//       instance, and the sorted list / tile ranges are bit-identical to the reference's (tests: sorted ids, ranges, keys).
//
// Both walks are PAIR-parallel: a warp flattens the (Gaussian, tile) pairs of 32 consecutive Gaussians (prefix sum of their
// tile counts, binary search by shuffle) and handles 32 pairs per step whatever the rect sizes -- a far chunk holds thousands
// of 1-4 tile Gaussians, a near one a few 1000-tile ones.  Pairs of one step that fall on the same tile are ranked with
// match.any in lane (= depth) order.
//
// The instance count R never has to visit the host: the placement clamps to the buffer capacity and the overflow is
// reported through the context (G4D_OPT_SYNC_MODE = 0); in the default exact mode the host reads R between the two
// launches only to size the buffer.
//
// Reference stage replaced: duplicateWithKeys + cub::DeviceRadixSort + identifyTileRanges of the CUDA rasterizer behind
// /root/reference/gaussian_renderer/__init__.py:120-128 (SURVEY.md App. A.2).
#include <cooperative_groups.h>
#include <cstddef>

#include "g4d_internal.h"
#include "raster_cull.cuh"

namespace cg = cooperative_groups;

namespace g4d {

namespace {

constexpr int kBinThreads = 1024;
constexpr int kDigitBits = 9;
constexpr int kRadix = 1 << kDigitBits;
constexpr uint32_t kSortSmemBytes = 32u * kRadix * 4u;   // per-warp digit counters of one scatter round

// inclusive scan of v over the 1024 threads of the block; total = block sum.  s_w: 33 words of shared scratch.
__device__ __forceinline__ uint32_t block_scan_incl(uint32_t v, uint32_t* s_w, uint32_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();   // previous users of s_w are done
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = s_w[lane];
        uint32_t ws = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, ws, o);
            if (lane >= o) ws += y;
        }
        s_w[lane] = ws - w;
        if (lane == 31) s_w[32] = ws;
    }
    __syncthreads();
    total = s_w[32];
    return x + s_w[warp];
}

// Grid-wide barrier of the cooperative bin_sort_kernel (all CTAs co-resident: a kCooperative launch).  A monotonic arrival
// counter, one release-arrive and an acquire-spin by thread 0 of every CTA, lighter than cooperative_groups' grid.sync() (nine
// of them are on the critical path of one forward).
struct GridBar {
    uint32_t* ctr; uint32_t gen, G;
    __device__ __forceinline__ void sync() {
        __syncthreads();
        if (threadIdx.x == 0) {
            ++gen;
            __threadfence();
            atomicAdd(ctr, 1u);
            const uint32_t target = gen * G;
            uint32_t v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < target);
        }
        __syncthreads();
    }
};

#define G4D_BIN_MARK(i) do { if (blockIdx.x == 0 && threadIdx.x == 0) a.ctl->phase_clk[i] = clock64(); } while (0)
#define G4D_BIN_MARK1(i) do { if (FIRST) G4D_BIN_MARK(i); } while (0)   // inside the first radix pass only

struct SortShared {
    uint32_t hist[kRadix];
    uint32_t part[4 * kRadix];   // [0,2): totals of one half of the CTAs per digit, [2,4): totals of the CTAs before mine
    uint32_t base[kRadix];       // running output position per digit for my slice
    uint32_t sw[33];
    uint32_t mm[2];
};

// One stable LSD pass over digit (key >> shift) & 511.  FIRST: input = the N raw Gaussians (key = depth bits - kmin,
// value = index), invisible ones are dropped.
template <bool FIRST, bool LAST>
__device__ __forceinline__ uint32_t radix_pass(const BinSortArgs& a, GridBar& grid, SortShared& s, uint32_t* wc, int shift,
                                               uint32_t kmin, uint32_t count, const uint32_t* __restrict__ kin,
                                               const uint32_t* __restrict__ vin, uint32_t* __restrict__ kout,
                                               uint32_t* __restrict__ vout) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t G = gridDim.x, c = blockIdx.x;
    const uint32_t per = (count + G - 1) / G;
    const uint32_t lo = min(c * per, count), hi = min(lo + per, count);
    auto load = [&](uint32_t i, uint32_t& key, uint32_t& val) -> bool {
        if (FIRST) {
            if (a.tiles_touched[i] == 0) return false;
            key = __float_as_uint(a.rec2[i].y) - kmin;   // depth > 0.2: sign bit clear, integer order = float order
            val = i;
            return true;
        }
        key = kin[i]; val = vin[i];
        return true;
    };
    // ---- (a) digit histogram of my slice
    if (tid < kRadix) s.hist[tid] = 0;
    __syncthreads();
    for (uint32_t i = lo + tid; i < hi; i += kBinThreads) {
        uint32_t key, val;
        if (load(i, key, val)) atomicAdd(&s.hist[(key >> shift) & (kRadix - 1)], 1u);
    }
    __syncthreads();
    if (tid < kRadix) a.H[c * kRadix + tid] = s.hist[tid];
    G4D_BIN_MARK1(6);
    grid.sync();
    G4D_BIN_MARK1(7);
    // ---- (b) my output base per digit = (all smaller digits of every CTA) + (same digit of the CTAs before me)
    {
        const uint32_t d = tid & (kRadix - 1), q = tid >> kDigitBits;       // 2 halves of the CTA range
        const uint32_t qs = (G + 1) / 2, c0 = q * qs, c1 = min(G, c0 + qs);
        uint32_t tot = 0, bef = 0;
        for (uint32_t cc = c0; cc < c1; ++cc) {
            const uint32_t v = __ldcg(a.H + cc * kRadix + d);
            tot += v;
            if (cc < c) bef += v;
        }
        s.part[q * kRadix + d] = tot;
        s.part[(2 + q) * kRadix + d] = bef;
    }
    __syncthreads();
    uint32_t tot = 0, bef = 0;
    if (tid < kRadix) { tot = s.part[tid] + s.part[kRadix + tid]; bef = s.part[2 * kRadix + tid] + s.part[3 * kRadix + tid]; }
    uint32_t total;
    const uint32_t incl = block_scan_incl(tot, s.sw, total);
    if (tid < kRadix) s.base[tid] = incl - tot + bef;
    __syncthreads();
    G4D_BIN_MARK1(8);
    // ---- (c) stable scatter, 1024 elements per round: rank inside the warp by match, then across the warps by a scan
    for (uint32_t b0 = lo; b0 < hi; b0 += kBinThreads) {
        for (int j = tid; j < 32 * kRadix; j += kBinThreads) wc[j] = 0;
        __syncthreads();
        const uint32_t i = b0 + tid;
        uint32_t key = 0, val = 0;
        const bool valid = i < hi && load(i, key, val);
        const uint32_t digit = (key >> shift) & (kRadix - 1);
        const uint32_t peers = __match_any_sync(0xffffffffu, valid ? digit : ((uint32_t)kRadix + (uint32_t)lane));
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) wc[warp * kRadix + digit] = __popc(peers);
        __syncthreads();
        if (tid < kRadix) {
            uint32_t run = s.base[tid];
#pragma unroll 8
            for (int w = 0; w < 32; ++w) {
                const uint32_t t = wc[w * kRadix + tid];
                wc[w * kRadix + tid] = run;
                run += t;
            }
            s.base[tid] = run;
        }
        __syncthreads();
        if (valid) {
            const uint32_t pos = wc[warp * kRadix + digit] + rank;
            if (!LAST) kout[pos] = key;
            vout[pos] = val;
        }
        __syncthreads();
    }
    G4D_BIN_MARK1(9);
    grid.sync();
    G4D_BIN_MARK1(10);
    return total;
}

// ---- unordered walk over the (Gaussian, tile) pairs of perm[ks, ke) restricted to the tile rows [y0, y1) ------------------
// f(tile index inside the band, position k of the Gaussian in perm).  No order is promised inside the range: small rects
// (< 32 tiles) are walked by ONE LANE each (a far chunk holds thousands of 1-4 tile Gaussians: 32 of them advance per
// iteration), large ones by the whole warp (32 tiles per step).
// f(tile index inside the band, position k of the Gaussian in perm, Gaussian index); f4(tiles[4] (-1 = none), k, index)
// handles up to four pairs of one Gaussian at once
template <class F, class F4>
__device__ __forceinline__ void walk_unordered(const uint32_t* __restrict__ perm, const uint2* __restrict__ rect,
                                               const float4* __restrict__ rec0, const float4* __restrict__ rec1, int tight, uint32_t ks,
                                               uint32_t ke, int y0, int y1, int grid_x, F&& f, F4&& f4) {
    const int lane = threadIdx.x & 31;
    // two-deep register prefetch (perm two groups ahead, rect one group ahead): both are L2 round trips, and a far chunk is a
    // long chain of such groups with only a few tiles of work each
    uint32_t gi_n = ks + lane < ke ? perm[ks + lane] : 0u;
    uint32_t gi_nn = ks + 32u + lane < ke ? perm[ks + 32u + lane] : 0u;
    uint2 rc_n = ks + lane < ke ? rect[gi_n] : make_uint2(0u, 0u);
    for (uint32_t k0 = ks; k0 < ke; k0 += 32u) {
        const uint32_t k = k0 + lane;
        int minx = 0, miny = 0, w = 0, h = 0;
        const uint32_t gi = gi_n;
        const uint2 rc = rc_n;
        gi_n = gi_nn;
        rc_n = k + 32u < ke ? rect[gi_n] : make_uint2(0u, 0u);
        gi_nn = k + 64u < ke ? perm[k + 64u] : 0u;
        float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
        if (k < ke) {
            minx = (int)(rc.x & 0xFFFFu);
            w = (int)(rc.y & 0xFFFFu) - minx;
            miny = max((int)(rc.x >> 16), y0);
            h = min((int)(rc.y >> 16), y1) - miny;
            if (h < 0) h = 0;
            if (tight) { r0 = rec0[gi]; r1 = rec1[gi]; }
        }
        const int nt = w * h;
        const bool big = nt >= 32;
        if (!big) {
            int x = 0, y = 0;
            for (int i = 0; i < nt; i += 4) {          // four pairs per trip: their atomics overlap (see f4 below)
                int tl[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    tl[u] = -1;
                    if (i + u < nt) {
                        if (!tight || tile_contributes(r0, r1, minx + x, miny + y)) tl[u] = (miny + y - y0) * grid_x + minx + x;
                        if (++x == w) { x = 0; ++y; }
                    }
                }
                f4(tl, k, gi);
            }
        }
        uint32_t todo = __ballot_sync(0xffffffffu, big);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const int bx = __shfl_sync(0xffffffffu, minx, src), by = __shfl_sync(0xffffffffu, miny, src);
            const int bw = __shfl_sync(0xffffffffu, w, src), bn = __shfl_sync(0xffffffffu, nt, src);
            const uint32_t bk = __shfl_sync(0xffffffffu, k, src), bg = __shfl_sync(0xffffffffu, gi, src);
            float4 q0 = r0, q1 = r1;
            if (tight) {
                q0.x = __shfl_sync(0xffffffffu, r0.x, src); q0.y = __shfl_sync(0xffffffffu, r0.y, src);
                q0.z = __shfl_sync(0xffffffffu, r0.z, src); q0.w = __shfl_sync(0xffffffffu, r0.w, src);
                q1.x = __shfl_sync(0xffffffffu, r1.x, src); q1.y = __shfl_sync(0xffffffffu, r1.y, src);
            }
            for (int t = lane; t < bn; t += 32) {
                const int ty = t / bw, tx = t - ty * bw;
                if (!tight || tile_contributes(q0, q1, bx + tx, by + ty)) f((by + ty - y0) * grid_x + bx + tx, bk, bg);
            }
        }
    }
}

// walk cost of a Gaussian in units of tile instances: its pairs plus a fixed per-Gaussian share of the group overhead
__device__ __forceinline__ uint32_t chunk_weight(uint32_t tiles_touched) { return tiles_touched + 4u; }

}  // namespace


__global__ void __launch_bounds__(kBinThreads, 1) bin_sort_kernel(BinSortArgs a) {
    GridBar grid{a.grid_bar, 0u, gridDim.x};
    extern __shared__ __align__(16) uint32_t dyn[];   // scatter: per-warp digit counters; count: tile histogram of a band
    __shared__ SortShared s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t G = gridDim.x, c = blockIdx.x;
    const uint32_t N = (uint32_t)a.n;

    pdl_trigger();      // (ordinary cooperative launch; lets the placement kernel queue up behind this grid)
    G4D_BIN_MARK(0);
    // ---- 0. range of the visible depth bits: reduced by the projection stage (RED.MIN / RED.MAX into the context's CameraDev)
    if (blockIdx.x == 0 && tid == 0) { a.ctl->R = 0u; a.ctl->overflow = 0u; }
    uint32_t kmin, kbits;
    {
        const uint32_t mn = __ldcg(a.depth_range), mx = __ldcg(a.depth_range + 1);
        kmin = mn <= mx ? mn : 0u;
        const uint32_t span = mn <= mx ? mx - mn : 0u;
        kbits = span ? 32u - (uint32_t)__clz((int)span) : 1u;
    }
    // (S is reused by phase 2, several grid-wide syncs later)

    G4D_BIN_MARK(1);
    // ---- 1. depth order of the visible Gaussians: ceil(kbits / 9) stable passes (uniform over the grid)
    const int passes = (int)((kbits + kDigitBits - 1) / kDigitBits);
    uint32_t nvis;
    if (passes == 1) {
        nvis = radix_pass<true, true>(a, grid, s, dyn, 0, kmin, N, nullptr, nullptr, nullptr, a.perm);
    } else {
        nvis = radix_pass<true, false>(a, grid, s, dyn, 0, kmin, N, nullptr, nullptr, a.kA, a.vA);
        uint32_t *ki = a.kA, *vi = a.vA, *ko = a.kB, *vo = a.vB;
        for (int p = 1; p < passes - 1; ++p) {
            radix_pass<false, false>(a, grid, s, dyn, p * kDigitBits, 0u, nvis, ki, vi, ko, vo);
            uint32_t* t0 = ki; ki = ko; ko = t0;
            t0 = vi; vi = vo; vo = t0;
        }
        radix_pass<false, true>(a, grid, s, dyn, (passes - 1) * kDigitBits, 0u, nvis, ki, vi, nullptr, a.perm);
    }

    G4D_BIN_MARK(2);
    // ---- 2. chunks of (nearly) equal walk cost (instances + a per-Gaussian constant) along the depth order
    const uint32_t per = (nvis + G - 1) / G;
    const uint32_t lo = min(c * per, nvis), hi = min(lo + per, nvis);
    {
        uint32_t sum = 0;
        for (uint32_t k = lo + tid; k < hi; k += kBinThreads) sum += chunk_weight(a.tiles_touched[a.perm[k]]);
        uint32_t total;
        block_scan_incl(sum, s.sw, total);
        if (tid == 0) a.S[c] = total;
        if (c == 0) {
            for (uint32_t j = tid; j <= G; j += kBinThreads) a.chunk_start[j] = j == 0 ? 0u : nvis;
        }
    }
    grid.sync();
    {
        uint32_t v = 0, before = 0;
        if ((uint32_t)tid < G) { v = __ldcg(a.S + tid); before = (uint32_t)tid < c ? v : 0u; }
        uint32_t est, my_excl;
        block_scan_incl(v, s.sw, est);
        block_scan_incl(before, s.sw, my_excl);
        const uint32_t T = max(1u, (est + G - 1) / G);
        uint32_t run = my_excl;
        for (uint32_t b0 = lo; b0 < hi; b0 += kBinThreads) {
            const uint32_t k = b0 + tid;
            const uint32_t tt = k < hi ? chunk_weight(a.tiles_touched[a.perm[k]]) : 0u;
            uint32_t tot;
            const uint32_t incl = block_scan_incl(tt, s.sw, tot);
            if (k < hi) {
                const uint32_t e0 = run + incl - tt, e1 = run + incl;      // exclusive / inclusive prefix of element k
                const uint32_t ja = e0 / T, jb = min(e1 / T, G - 1);       // element k + 1 opens chunks (ja, jb]
                for (uint32_t j = ja + 1; j <= jb; ++j) a.chunk_start[j] = k + 1;
            }
            run += tot;
        }
    }
    grid.sync();

    G4D_BIN_MARK(3);
    // ---- 3. instances per (tile, chunk): shared-memory histogram of my chunk, band by band
    const uint32_t cs = __ldcg(a.chunk_start + c), ce = __ldcg(a.chunk_start + c + 1);
    {
        const uint32_t len = ce - cs, wper = (len + 31) / 32;
        const uint32_t ks = cs + min((uint32_t)warp * wper, len), ke = cs + min((uint32_t)(warp + 1) * wper, len);
        for (int y0 = 0; y0 < a.grid_y; y0 += a.count_band_rows) {
            const int y1 = min(a.grid_y, y0 + a.count_band_rows);
            const int bn = (y1 - y0) * a.grid_x;
            for (int j = tid; j < bn; j += kBinThreads) dyn[j] = 0;
            __syncthreads();
            walk_unordered(a.perm, a.rect, a.rec0, a.rec1, a.tight, ks, ke, y0, y1, a.grid_x,
                           [&](int tile, uint32_t, uint32_t) { atomicAdd(&dyn[tile], 1u); },
                           [&](const int (&tl)[4], uint32_t, uint32_t) {
#pragma unroll
                               for (int u = 0; u < 4; ++u) if (tl[u] >= 0) atomicAdd(&dyn[tl[u]], 1u);
                           });
            __syncthreads();
            for (int j = tid; j < bn; j += kBinThreads) a.M[(size_t)(y0 * a.grid_x + j) * G + c] = dyn[j];
            __syncthreads();
        }
    }
    grid.sync();

    G4D_BIN_MARK(4);
    // ---- 4. per tile: exclusive scan over the chunks (one warp per tile) and the tile's total; R = sum of the totals.
    //         (the exclusive scan over the TILES -- tile_start, ranges -- is done by the placement kernel: one grid-wide sync
    //         less here, 5440 values re-scanned per CTA there)
    {
        uint32_t my_total = 0;
        for (uint32_t t = c * 32u + warp; t < (uint32_t)a.num_tiles; t += G * 32u) {
            uint32_t* row = a.M + (size_t)t * G;
            uint32_t run = 0;
            for (uint32_t j0 = 0; j0 < G; j0 += 32) {
                const uint32_t j = j0 + lane;
                const uint32_t v = j < G ? __ldcg(row + j) : 0u;
                uint32_t x = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                    if (lane >= o) x += y;
                }
                if (j < G) row[j] = run + x - v;
                run += __shfl_sync(0xffffffffu, x, 31);
            }
            if (lane == 0) { a.tile_total[t] = run; my_total += run; }
        }
        uint32_t cta_total;
        block_scan_incl(my_total, s.sw, cta_total);
        if (tid == 0) {
            if (cta_total) atomicAdd(&a.ctl->R, cta_total);
            if (c == 0) a.ctl->n_visible = nvis;
        }
    }
    G4D_BIN_MARK(5);
    if (blockIdx.x == 0 && threadIdx.x == 0) a.ctl->phase_clk[15] = (long long)kbits;
}

// ------------------------------------------------------------------------------------------------------------------
// Placement.  CTA c owns chunk c of the depth-ordered list; inside the segment of tile t the instances of chunk c occupy
// the private sub-segment [tile_start[t] + M[t][c], tile_start[t] + M[t][c+1]).  The CTA keeps one cursor per tile in
// shared memory and drops its (Gaussian, tile) pairs with shared-memory atomics in whatever order the lanes reach them --
// the sub-segments are already in depth order with respect to each other, so only the few entries INSIDE a sub-segment
// (4 on average) are left unordered.  What is stored is the Gaussian's position k in the depth order, not its index.
__global__ void __launch_bounds__(kBinThreads, 1) bin_place_kernel(BinPlaceArgs a) {
    extern __shared__ __align__(16) uint32_t cur[];     // [tiles of the band] next free slot of my sub-segment
    __shared__ uint32_t s_w[33];
    const int tid = threadIdx.x, warp = tid >> 5;
    const uint32_t c = blockIdx.x, G = gridDim.x;
    pdl_wait();
    pdl_trigger();
    const uint32_t cs = a.chunk_start[c], ce = a.chunk_start[c + 1];
    const uint32_t len = ce - cs, per = (len + 31) / 32;
    const uint32_t ks = cs + min((uint32_t)warp * per, len), ke = cs + min((uint32_t)(warp + 1) * per, len);
    for (int y0 = 0; y0 < a.grid_y; y0 += a.band_rows) {
        const int y1 = min(a.grid_y, y0 + a.band_rows);
        const uint32_t bn = (uint32_t)((y1 - y0) * a.grid_x), t0 = (uint32_t)(y0 * a.grid_x);
        // ---- exclusive scan of the tile totals: start slot of every tile of the band (+ ranges, written once)
        {
            uint32_t before = 0;
            for (uint32_t t = tid; t < t0; t += kBinThreads) before += __ldg(a.tile_total + t);
            uint32_t run;
            block_scan_incl(before, s_w, run);          // run = sum of every tile before the band
            for (uint32_t b0 = 0; b0 < bn; b0 += kBinThreads) {
                const uint32_t t = b0 + tid;
                const uint32_t v = t < bn ? __ldg(a.tile_total + t0 + t) : 0u;
                uint32_t tot;
                const uint32_t start = run + block_scan_incl(v, s_w, tot) - v;
                if (t < bn) {
                    cur[t] = start + a.M[(size_t)(t0 + t) * G + c];
                    if (c == 0) {
                        a.tile_start[t0 + t] = start;
                        // empty tiles keep (0, 0) like the reference's zero-initialised range array (identifyTileRanges, A.2)
                        a.ranges[t0 + t] = v ? make_uint2(min(start, a.capacity), min(start + v, a.capacity)) : make_uint2(0u, 0u);
                    }
                }
                run += tot;
            }
        }
        __syncthreads();
        walk_unordered(a.perm, a.rect, a.rec0, a.rec1, a.tight, ks, ke, y0, y1, a.grid_x,
                       [&](int tile, uint32_t k, uint32_t gi) {
                           const uint32_t slot = atomicAdd(&cur[tile], 1u);
                           if (slot < a.capacity) a.kbuf[slot] = make_uint2(k, gi);
                       },
                       [&](const int (&tl)[4], uint32_t k, uint32_t gi) {
                           uint32_t slot[4];
#pragma unroll
                           for (int u = 0; u < 4; ++u) slot[u] = tl[u] >= 0 ? atomicAdd(&cur[tl[u]], 1u) : 0xFFFFFFFFu;
#pragma unroll
                           for (int u = 0; u < 4; ++u) if (slot[u] < a.capacity) a.kbuf[slot[u]] = make_uint2(k, gi);
                       });
        __syncthreads();
    }
}

// Fix-up: order every (tile, chunk) sub-segment by depth rank.  One warp per (tile, 32 chunks); it reads 32 sub-segment bounds
// (the M row of a tile is contiguous: coalesced) and every lane loads the first eight (rank, Gaussian) pairs of ITS
// sub-segment at once -- one memory round trip per round, not one per entry; sub-segments of up to eight entries (the bulk:
// the average is ~4) are ranked in registers by their lane, longer ones by the whole warp with shuffles.  Ranks are unique,
// so the final position of an entry is the number of smaller ranks in its sub-segment.
// one lane orders its sub-segment [lo, lo + n) (n <= T, else it is left to the caller): ranks are unique, so the final position of
// an entry is the number of smaller ranks in the sub-segment
template <int T>
__device__ __forceinline__ void rank_tier(const BinPlaceArgs& a, uint32_t lo, uint32_t n) {
    constexpr bool kKeepId = T <= 16;      // the big tiers re-read the Gaussian index at store time (L1 hits) instead of
    const bool mine = n <= (uint32_t)T;    // holding 2 T registers
    uint32_t key[T], id[kKeepId ? T : 1];
#pragma unroll
    for (int q = 0; q < T; ++q) {
        key[q] = 0xFFFFFFFFu;
        if (mine && (uint32_t)q < n) {
            if (kKeepId) { const uint2 e = a.kbuf[lo + q]; key[q] = e.x; id[q] = e.y; }
            else key[q] = a.kbuf[lo + q].x;
        }
    }
#pragma unroll
    for (int q = 0; q < T; ++q) {
        uint32_t r = 0;
#pragma unroll
        for (int p = 0; p < T; ++p)
            if (p != q) r += key[p] < key[q] ? 1u : 0u;
        if (mine && (uint32_t)q < n) a.ids[lo + r] = kKeepId ? id[q] : a.kbuf[lo + q].y;
    }
}

// the whole warp orders ONE sub-segment [lo, lo + n), 32 < n <= 32 S: lane l holds entries l, l + 32, ...
template <int S>
__device__ __forceinline__ void coop_rank(const BinPlaceArgs& a, uint32_t lo, uint32_t n, int lane) {
    uint2 e[S];
    uint32_t r[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
        const uint32_t i = (uint32_t)lane + 32u * s;
        e[s] = i < n ? a.kbuf[lo + i] : make_uint2(0xFFFFFFFFu, 0u);
        r[s] = 0u;
    }
#pragma unroll
    for (int s2 = 0; s2 < S; ++s2) {
        if (32u * s2 >= n) break;                     // warp-uniform
#pragma unroll 8
        for (int l = 0; l < 32; ++l) {
            const uint32_t kj = __shfl_sync(0xffffffffu, e[s2].x, l);      // (padding keys are never smaller than anything)
#pragma unroll
            for (int s = 0; s < S; ++s) r[s] += kj < e[s].x ? 1u : 0u;
        }
    }
#pragma unroll
    for (int s = 0; s < S; ++s)
        if ((uint32_t)lane + 32u * s < n) a.ids[lo + r[s]] = e[s].y;
}

// any length: 256 entries at a time in registers (8 per lane), every key of the sub-segment streamed past them 32 at a time
// (coalesced re-read, next block prefetched) and broadcast by shuffle -- n^2 / 256 shuffles instead of n^2 / 32 dependent loads
__device__ __noinline__ void coop_rank_big(const BinPlaceArgs& a, uint32_t lo, uint32_t n, int lane) {
    constexpr int S = 8;
    for (uint32_t base = 0; base < n; base += 32u * S) {
        uint2 e[S];
        uint32_t r[S];
#pragma unroll
        for (int s = 0; s < S; ++s) {
            const uint32_t i = base + (uint32_t)lane + 32u * s;
            e[s] = i < n ? a.kbuf[lo + i] : make_uint2(0xFFFFFFFFu, 0u);
            r[s] = 0u;
        }
        uint32_t nxt = (uint32_t)lane < n ? a.kbuf[lo + lane].x : 0xFFFFFFFFu;
        for (uint32_t j0 = 0; j0 < n; j0 += 32u) {
            const uint32_t cur = nxt;
            const uint32_t jn = j0 + 32u + (uint32_t)lane;
            nxt = jn < n ? a.kbuf[lo + jn].x : 0xFFFFFFFFu;
#pragma unroll 8
            for (int l = 0; l < 32; ++l) {
                const uint32_t kj = __shfl_sync(0xffffffffu, cur, l);
#pragma unroll
                for (int s = 0; s < S; ++s) r[s] += kj < e[s].x ? 1u : 0u;
            }
        }
#pragma unroll
        for (int s = 0; s < S; ++s)
            if (base + (uint32_t)lane + 32u * s < n) a.ids[lo + r[s]] = e[s].y;
    }
}

__global__ void __launch_bounds__(256, 4) bin_fix_kernel(BinPlaceArgs a, int chunks) {
    const int lane = threadIdx.x & 31;
    const int rounds = (chunks + 31) / 32;
    pdl_wait();
    pdl_trigger();
    const uint32_t item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);      // (tile, round): a dense tile's rounds run
    const uint32_t t = item / (uint32_t)rounds;                                   // on different warps
    if (t >= (uint32_t)a.num_tiles) return;
    const uint32_t* mrow = a.M + (size_t)t * chunks;
    {
        // the four words that locate a lane's sub-segment are independent loads: ONE memory round trip in front of the
        // entries' own, not three (total -> start -> M row); a warp's life is a handful of such round trips
        const int c = (int)(item - t * (uint32_t)rounds) * 32 + lane;
        const uint32_t total = __ldg(a.tile_total + t);
        const uint32_t start = __ldg(a.tile_start + t);
        const uint32_t m0 = c < chunks ? __ldg(mrow + c) : 0u;
        const uint32_t m1 = c + 1 < chunks ? __ldg(mrow + c + 1) : 0u;
        if (total == 0) return;
        uint32_t lo = 0, hi = 0;
        if (c < chunks) {
            lo = start + m0;
            hi = start + (c + 1 < chunks ? m1 : total);
            lo = min(lo, a.capacity); hi = min(hi, a.capacity);
        }
        const uint32_t n = hi - lo;
        // Every lane ranks ITS sub-segment in registers, all 32 sub-segments of the warp in parallel: one memory round trip for
        // the whole round.  The register tier T is the smallest that holds the longest sub-segment of the warp (warp-uniform):
        // T loads, T^2 compares, T stores per lane -- the fixed 8 / 32 tiers of the first version spent ~1100 instructions per
        // warp (ncu: 29.5 M for the kernel, issue bound), most of them compares against padding.
        const uint32_t nmax = __reduce_max_sync(0xffffffffu, n);
        uint32_t done_limit;            // sub-segments of up to this many entries are finished by the per-lane code
        if (nmax <= 4u) { rank_tier<4>(a, lo, n); done_limit = 4u; }
        else if (nmax <= 8u) { rank_tier<8>(a, lo, n); done_limit = 8u; }
        else if (nmax <= 12u) { rank_tier<12>(a, lo, n); done_limit = 12u; }
        else if (nmax <= 16u) { rank_tier<16>(a, lo, n); done_limit = 16u; }
        else if (nmax <= 24u) { rank_tier<24>(a, lo, n); done_limit = 24u; }
        else { rank_tier<32>(a, lo, n); done_limit = 32u; }
        // sub-segments longer than 32 entries (a tile under the few dozen nearest, screen-filling Gaussians of a chunk): the whole
        // warp ranks one at a time, S entries per lane in registers, every key broadcast once by shuffle (n shuffles + n S
        // compares for n entries).  The first version re-read the list from L1 once per entry: ~16 k cycles for n = 100, ten such
        // sub-segments in one warp were the critical path of the kernel (74 .. 110 us depending on the camera).
        uint32_t todo = __ballot_sync(0xffffffffu, n > done_limit);
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const uint32_t clo = __shfl_sync(0xffffffffu, lo, src), cnn = __shfl_sync(0xffffffffu, n, src);
            if (cnn <= 64u) coop_rank<2>(a, clo, cnn, lane);
            else if (cnn <= 128u) coop_rank<4>(a, clo, cnn, lane);
            else if (cnn <= 256u) coop_rank<8>(a, clo, cnn, lane);
            else coop_rank_big(a, clo, cnn, lane);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
namespace {
constexpr size_t kCountSmemBudget = 160 * 1024;
constexpr size_t kPlaceSmemBudget = 96 * 1024;

// the aux area of the binning: sort ping-pong buffers, per-chunk histograms and counts, tile totals and starts, BinCtl
void carve_bin_aux(Carve& m, int64_t n, int num_tiles, int sm_count, BinSortArgs& a, uint32_t*& tile_start) {
    const size_t N = (size_t)(n > 0 ? n : 1), G = (size_t)sm_count;
    a.kA = m.take<uint32_t>(N); a.vA = m.take<uint32_t>(N); a.kB = m.take<uint32_t>(N); a.vB = m.take<uint32_t>(N);
    a.H = m.take<uint32_t>(G * kRadix); a.S = m.take<uint32_t>(2 * G); a.chunk_start = m.take<uint32_t>(G + 1);
    a.M = m.take<uint32_t>(G * (size_t)num_tiles);
    a.tile_total = m.take<uint32_t>((size_t)num_tiles);
    tile_start = m.take<uint32_t>((size_t)num_tiles);
    a.ctl = m.take<BinCtl>(1);
}
}  // namespace

size_t bin_aux_bytes(int64_t n, int num_tiles, int sm_count) {
    Carve m;
    BinSortArgs a{};
    uint32_t* tile_start;
    carve_bin_aux(m, n, num_tiles, sm_count, a, tile_start);
    return m.bytes();
}

cudaError_t launch_bin_sort(int64_t n, int grid_x, int grid_y, const GeomBuffers& g, void* aux, int tight, int sm_count,
                            BinLayout* out, cudaStream_t st) {
    const int num_tiles = grid_x * grid_y;
    BinSortArgs a{};
    a.n = n; a.rec2 = g.rec2; a.tiles_touched = g.tiles_touched; a.rect = g.rect; a.rec0 = g.rec0; a.rec1 = g.rec1;
    a.depth_range = g.depth_range;
    a.grid_bar = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(g.depth_range) - offsetof(CameraDev, depth_min) + offsetof(CameraDev, grid_bar));
    a.perm = g.perm;
    Carve m(aux);
    uint32_t* tile_start;
    carve_bin_aux(m, n, num_tiles, sm_count, a, tile_start);
    a.grid_x = grid_x; a.grid_y = grid_y; a.num_tiles = num_tiles; a.tight = tight;
    int rows = (int)(kCountSmemBudget / ((size_t)grid_x * 4));
    if (rows < 1) return cudaErrorInvalidValue;
    a.count_band_rows = rows < grid_y ? rows : grid_y;
    size_t smem = (size_t)a.count_band_rows * grid_x * 4;
    if (smem < kSortSmemBytes) smem = kSortSmemBytes;
    out->chunk_start = a.chunk_start; out->M = a.M; out->tile_total = a.tile_total; out->tile_start = tile_start; out->ctl = a.ctl;
    out->chunks = sm_count;
    return launch_k(bin_sort_kernel, dim3((unsigned)sm_count), dim3(kBinThreads), smem, st, kCooperative, a);
}

cudaError_t launch_bin_place(int grid_x, int grid_y, const GeomBuffers& g, const BinLayout& lay, uint32_t* ids, uint2* kbuf,
                             uint2* ranges, uint32_t capacity, int tight, cudaStream_t st) {
    const int num_tiles = grid_x * grid_y;
    BinPlaceArgs a{};
    a.perm = g.perm; a.rect = g.rect; a.rec0 = g.rec0; a.rec1 = g.rec1; a.chunk_start = lay.chunk_start; a.M = lay.M;
    a.tile_total = lay.tile_total; a.tile_start = lay.tile_start; a.ranges = ranges; a.ids = ids; a.kbuf = kbuf;
    a.capacity = capacity; a.grid_x = grid_x; a.grid_y = grid_y; a.num_tiles = num_tiles; a.tight = tight;
    a.band_rows = (int)(kPlaceSmemBudget / (4 * (size_t)grid_x));
    if (a.band_rows < 1) return cudaErrorInvalidValue;
    if (a.band_rows > grid_y) a.band_rows = grid_y;
    const size_t smem = 4 * (size_t)a.band_rows * grid_x;
    const cudaError_t e = launch_k(bin_place_kernel, dim3(lay.chunks), dim3(kBinThreads), smem, st, kPdl, a);
    if (e != cudaSuccess) return e;
    const int rounds = (lay.chunks + 31) / 32;
    return launch_k(bin_fix_kernel, dim3((num_tiles * rounds + 7) / 8), dim3(256), 0, st, kPdl, a, lay.chunks);
}

// One thread, ordinary launch (after the blend: no programmatic edge to break).  The forwards of a stream run one after the
// other, so the read-modify-write of the host-mapped words needs no atomics.
__global__ void record_overflow_kernel(const BinCtl* ctl, uint32_t capacity, volatile uint32_t* words) {
    const uint32_t R = ctl->R;
    if (R <= capacity) return;
    words[0] = words[0] + 1u;
    if (R > words[1]) words[1] = R;
}

cudaError_t launch_record_overflow(const BinCtl* ctl, uint32_t capacity, uint32_t* words, cudaStream_t st) {
    return launch_k(record_overflow_kernel, 1, 1, 0, st, kOrdinary, ctl, capacity, words);
}

}  // namespace g4d
