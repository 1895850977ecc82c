// g4d_knn.cu -- mean squared distance to the 3 nearest neighbours of every point (SURVEY.md 8f N4).
//
// Replaces simple_knn._C.distCUDA2 (submodules/simple-knn, absent from the reference tree), called once per scene at
// /root/reference/scene/gaussian_model.py:148:  dist2 = clamp_min(distCUDA2(points), 1e-7); scales = log(sqrt(dist2)).
// Published behaviour restated: for every point the EXACT three smallest squared Euclidean distances to the OTHER points
// (self excluded by index, duplicates count as distance 0), result = (d0 + d1 + d2) / 3 in fp32.
//
// Upstream walks a Morton-sorted list with 1024-point boxes.  Here: a uniform grid over the bounding box (~4 points per
// cell), points counting-sorted by cell, one thread per point visiting Chebyshev rings of cells until the third-best
// distance is no larger than the distance to the unvisited region -- exact, not approximate.
// Compiled with -fmad=false: d2 = (dx*dx + dy*dy) + dz*dz evaluates bit-identically to the numpy oracle.
#include <cfloat>

#include "g4d_internal.h"

namespace g4d {

namespace {

struct KnnGrid {
    float bmin[3], cs[3], inv_cs[3];
    int dim[3];
    int64_t n;
};

__device__ __forceinline__ uint32_t f2ord(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float ord2f(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o); }

__global__ void __launch_bounds__(256) knn_bbox_kernel(const float* __restrict__ xyz, int64_t n, uint32_t* __restrict__ mm) {
    uint32_t lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0u, 0u, 0u};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { const uint32_t o = f2ord(xyz[3 * i + a]); lo[a] = min(lo[a], o); hi[a] = max(hi[a], o); }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_min_sync(0xffffffffu, lo[a]); hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
        if ((threadIdx.x & 31) == 0) { atomicMin(&mm[a], lo[a]); atomicMax(&mm[3 + a], hi[a]); }
    }
}

// one thread: grid geometry from the bounding box (~4 points per cell, at most 128 cells per axis)
__global__ void knn_setup_kernel(const uint32_t* __restrict__ mm, int64_t n, KnnGrid* g) {
    float ext[3];
    for (int a = 0; a < 3; ++a) { g->bmin[a] = ord2f(mm[a]); ext[a] = fmaxf(ord2f(mm[3 + a]) - g->bmin[a], 0.f); }
    const float longest = fmaxf(fmaxf(ext[0], ext[1]), fmaxf(ext[2], 1e-30f));
    const float target = cbrtf(fmaxf((float)n / 4.f, 1.f));             // cells along the longest axis
    for (int a = 0; a < 3; ++a) {
        int d = (int)ceilf(target * ext[a] / longest);
        d = d < 1 ? 1 : (d > 128 ? 128 : d);
        g->dim[a] = d;
        g->cs[a] = ext[a] > 0.f ? ext[a] / (float)d : 1.f;
        g->inv_cs[a] = 1.f / g->cs[a];
    }
    g->n = n;
}

__device__ __forceinline__ int cell_coord(const KnnGrid& g, float v, int a) {
    int c = (int)floorf((v - g.bmin[a]) * g.inv_cs[a]);
    return c < 0 ? 0 : (c >= g.dim[a] ? g.dim[a] - 1 : c);
}
__device__ __forceinline__ uint32_t cell_index(const KnnGrid& g, int cx, int cy, int cz) { return ((uint32_t)cz * g.dim[1] + cy) * g.dim[0] + cx; }

__global__ void __launch_bounds__(256) knn_count_kernel(const float* __restrict__ xyz, const KnnGrid* __restrict__ gp, uint32_t* __restrict__ cnt,
                                                        uint32_t* __restrict__ cell_of) {
    const KnnGrid g = *gp;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.n) return;
    const uint32_t c = cell_index(g, cell_coord(g, xyz[3 * i], 0), cell_coord(g, xyz[3 * i + 1], 1), cell_coord(g, xyz[3 * i + 2], 2));
    cell_of[i] = c;
    atomicAdd(&cnt[c], 1u);
}

// exclusive scan of cnt[0, cells) by ONE block (init-time helper: at most 128^3 cells)
__global__ void __launch_bounds__(1024) knn_scan_kernel(const KnnGrid* __restrict__ gp, uint32_t* __restrict__ cnt, uint32_t* __restrict__ start) {
    __shared__ uint32_t s_w[33];
    const uint32_t cells = (uint32_t)gp->dim[0] * gp->dim[1] * gp->dim[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t run = 0;
    for (uint32_t b = 0; b < cells; b += 4096) {
        uint32_t v[4], sum = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) { const uint32_t i = b + threadIdx.x * 4 + k; v[k] = i < cells ? cnt[i] : 0u; sum += v[k]; }
        uint32_t x = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        __syncthreads();
        if (lane == 31) s_w[warp] = x;
        __syncthreads();
        if (warp == 0) {
            const uint32_t w = s_w[lane];
            uint32_t ws = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += y; }
            s_w[lane] = ws - w;
            if (lane == 31) s_w[32] = ws;
        }
        __syncthreads();
        uint32_t e = run + s_w[warp] + x - sum;
#pragma unroll
        for (int k = 0; k < 4; ++k) { const uint32_t i = b + threadIdx.x * 4 + k; if (i < cells) { start[i] = e; cnt[i] = 0; } e += v[k]; }
        run += s_w[32];
    }
    if (threadIdx.x == 0) start[cells] = run;
}

__global__ void __launch_bounds__(256) knn_scatter_kernel(const KnnGrid* __restrict__ gp, const uint32_t* __restrict__ cell_of,
                                                          const uint32_t* __restrict__ start, uint32_t* __restrict__ fill,
                                                          uint32_t* __restrict__ sorted) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= gp->n) return;
    const uint32_t c = cell_of[i];
    sorted[start[c] + atomicAdd(&fill[c], 1u)] = (uint32_t)i;
}

__device__ __forceinline__ void insert3(float d, float (&best)[3]) {
    if (d < best[2]) {
        if (d < best[1]) {
            best[2] = best[1];
            if (d < best[0]) { best[1] = best[0]; best[0] = d; } else best[1] = d;
        } else best[2] = d;
    }
}

__global__ void __launch_bounds__(128) knn_search_kernel(const float* __restrict__ xyz, const KnnGrid* __restrict__ gp,
                                                         const uint32_t* __restrict__ start, const uint32_t* __restrict__ sorted,
                                                         float* __restrict__ out) {
    const KnnGrid g = *gp;
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= g.n) return;
    const uint32_t me = sorted[k];                     // neighbouring threads work on neighbouring cells
    const float px = xyz[3 * (size_t)me], py = xyz[3 * (size_t)me + 1], pz = xyz[3 * (size_t)me + 2];
    const float p[3] = {px, py, pz};
    const int c[3] = {cell_coord(g, px, 0), cell_coord(g, py, 1), cell_coord(g, pz, 2)};
    float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    const int rmax = max(max(g.dim[0], g.dim[1]), g.dim[2]);
    for (int r = 0; r <= rmax; ++r) {
        const int z0 = max(c[2] - r, 0), z1 = min(c[2] + r, g.dim[2] - 1);
        const int y0 = max(c[1] - r, 0), y1 = min(c[1] + r, g.dim[1] - 1);
        const int x0 = max(c[0] - r, 0), x1 = min(c[0] + r, g.dim[0] - 1);
        for (int z = z0; z <= z1; ++z)
            for (int y = y0; y <= y1; ++y) {
                const bool shell_zy = abs(z - c[2]) == r || abs(y - c[1]) == r;
                for (int x = x0; x <= x1; ++x) {
                    if (!shell_zy && abs(x - c[0]) != r) continue;   // interior of the cube: visited by an earlier ring
                    const uint32_t ci = cell_index(g, x, y, z);
                    const uint32_t e = start[ci + 1];
                    for (uint32_t j = start[ci]; j < e; ++j) {
                        const uint32_t o = sorted[j];
                        if (o == me) continue;
                        const float dx = xyz[3 * (size_t)o] - px, dy = xyz[3 * (size_t)o + 1] - py, dz = xyz[3 * (size_t)o + 2] - pz;
                        insert3((dx * dx + dy * dy) + dz * dz, best);
                    }
                }
            }
        // every unvisited point lies outside the (2r+1)^3 cube of cells: at least `face` away along some axis
        float face = FLT_MAX;
        bool open = false;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (c[a] - r > 0) { open = true; face = fminf(face, p[a] - (g.bmin[a] + (float)(c[a] - r) * g.cs[a])); }
            if (c[a] + r < g.dim[a] - 1) { open = true; face = fminf(face, (g.bmin[a] + (float)(c[a] + r + 1) * g.cs[a]) - p[a]); }
        }
        if (!open) break;
        face = fmaxf(face * 0.9999f - 1e-30f, 0.f);       // conservative against the rounding of the cell assignment
        if (best[2] <= face * face) break;
    }
    out[me] = ((best[0] + best[1]) + best[2]) / 3.0f;
}

constexpr size_t kCells = (size_t)128 * 128 * 128 + 1;   // at most 128 cells per axis, + the end of the last one

// bounding box words, the grid, per-cell counts and starts, per-point cell and the points sorted by cell
struct KnnScratch { uint32_t* mm; KnnGrid* grid; uint32_t* cnt; uint32_t* start; uint32_t* cell_of; uint32_t* sorted; };
KnnScratch carve_knn_scratch(Carve& m, int64_t n) {
    const size_t N = (size_t)(n > 0 ? n : 1);
    KnnScratch s;
    s.mm = m.take<uint32_t>(16);
    s.grid = m.take<KnnGrid>(1);
    s.cnt = m.take<uint32_t>(kCells);
    s.start = m.take<uint32_t>(kCells);
    s.cell_of = m.take<uint32_t>(N);
    s.sorted = m.take<uint32_t>(N);
    return s;
}

}  // namespace

size_t knn_scratch_bytes(int64_t n) {
    Carve m;
    carve_knn_scratch(m, n);
    return m.bytes();
}

cudaError_t launch_knn_dist2(int64_t n, const float* xyz, float* out, void* scratch, int sm_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    Carve m(scratch);
    const KnnScratch s = carve_knn_scratch(m, n);
    cudaError_t e;
    const uint32_t init[6] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u, 0u};
    if ((e = cudaMemcpyAsync(s.mm, init, sizeof(init), cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(s.cnt, 0, kCells * 4, st)) != cudaSuccess) return e;
    int blocks = (int)((n + 255) / 256);
    knn_bbox_kernel<<<blocks < sm_count * 8 ? blocks : sm_count * 8, 256, 0, st>>>(xyz, n, s.mm);
    knn_setup_kernel<<<1, 1, 0, st>>>(s.mm, n, s.grid);
    knn_count_kernel<<<blocks, 256, 0, st>>>(xyz, s.grid, s.cnt, s.cell_of);
    knn_scan_kernel<<<1, 1024, 0, st>>>(s.grid, s.cnt, s.start);
    knn_scatter_kernel<<<blocks, 256, 0, st>>>(s.grid, s.cell_of, s.start, s.cnt, s.sorted);
    knn_search_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(xyz, s.grid, s.start, s.sorted, out);
    return cudaGetLastError();
}

}  // namespace g4d
