// g4d_tc_selftest.cu -- self test of the wgmma building blocks of tc_wgmma.cuh (test-only library libg4d_selftest.so).
//
// D[128 x N] = A[128 x K] * B[N x K]^T by two warpgroups (rows 0-63 / 64-127), one operand arrangement per mode, each with
// the hi / lo split and three products the kernels use:
//   0  3xTF32, A register fragments, B K-major                  (deform forward, G4D_OPT_TENSOR_CORES = 1)
//   1  FP16x2, A register fragments, B K-major                  (deform forward, default)
//   2  BF16x2, A register fragments, B MN-major (transposed)    (backward dgrad: d(a1) = dz W1, d(feat) = dh W0)
//   3  BF16x2, A and B from shared memory, both MN-major        (backward wgrad: dW = X^T Y over the Gaussians)
//   4  BF16x2, A and B from shared memory, both K-major
#include <cuda_runtime.h>

#include "tc_wgmma.cuh"

namespace g4d {
namespace {

template <int N>
__global__ void __launch_bounds__(256, 1) wgmma_selftest_kernel(int K, int mode, const float* __restrict__ A, const float* __restrict__ B,
                                                               float* __restrict__ D) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int tid = threadIdx.x, wgi = tid >> 7, t128 = tid & 127, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int r0 = wgi * 64 + ((t128 >> 5) << 4) + g, r1 = r0 + 8;
    const bool tf32 = mode == 0;
    const uint32_t es = tf32 ? 4u : 2u;
    uint8_t* sB = smem;                                  // (hi | lo) image of B
    uint8_t* sA = smem + 2u * N * K * es;                // (hi | lo) image of A (modes 3, 4)
    const uint32_t bpart = (uint32_t)N * K * es, apart = 128u * K * 2u;
    for (int e = tid; e < N * K; e += 256) {
        const uint32_t nn = e / K, k = e % K;
        const float v = B[e];
        if (tf32) {
            uint32_t hi, lo;
            wg::tf32_split(v, hi, lo);
            *reinterpret_cast<uint32_t*>(sB + wg::img32_off(nn, k, K)) = hi;
            *reinterpret_cast<uint32_t*>(sB + bpart + wg::img32_off(nn, k, K)) = lo;
        } else {
            uint32_t hi, lo;
            if (mode == 1) wg::f16_split2(v, 0.f, hi, lo); else wg::bf16_split2(v, 0.f, hi, lo);
            const uint32_t off = (mode == 2 || mode == 3) ? wg::img16_off(k, nn, N) : wg::img16_off(nn, k, K);
            *reinterpret_cast<uint16_t*>(sB + off) = (uint16_t)hi;
            *reinterpret_cast<uint16_t*>(sB + bpart + off) = (uint16_t)lo;
        }
    }
    if (mode >= 3) {
        for (int e = tid; e < 128 * K; e += 256) {
            const uint32_t m = e / K, k = e % K;
            uint32_t hi, lo;
            wg::bf16_split2(A[e], 0.f, hi, lo);
            const uint32_t off = mode == 3 ? wg::img16_off(k, m, 128) : wg::img16_off(m, k, K);
            *reinterpret_cast<uint16_t*>(sA + off) = (uint16_t)hi;
            *reinterpret_cast<uint16_t*>(sA + apart + off) = (uint16_t)lo;
        }
    }
    wg::fence_proxy_async();
    __syncthreads();
    const uint32_t b = wg::smem_addr(sB), a = wg::smem_addr(sA);
    float d[N / 2];
    const int ks = tf32 ? 8 : 16;
    for (int s = 0; s < K / ks; ++s) {
        wg::Frags<1> f;
        if (mode <= 2) {
            if (tf32) {
                const int c0 = 8 * s + t, c1 = c0 + 4;
                wg::tf32_split(A[r0 * K + c0], f.hi[0][0], f.lo[0][0]);
                wg::tf32_split(A[r1 * K + c0], f.hi[0][1], f.lo[0][1]);
                wg::tf32_split(A[r0 * K + c1], f.hi[0][2], f.lo[0][2]);
                wg::tf32_split(A[r1 * K + c1], f.hi[0][3], f.lo[0][3]);
            } else {
#pragma unroll
                for (int hlf = 0; hlf < 2; ++hlf) {
                    const int c = 16 * s + 8 * hlf + 2 * t;
                    if (mode == 1) {
                        wg::f16_split2(A[r0 * K + c], A[r0 * K + c + 1], f.hi[0][2 * hlf], f.lo[0][2 * hlf]);
                        wg::f16_split2(A[r1 * K + c], A[r1 * K + c + 1], f.hi[0][2 * hlf + 1], f.lo[0][2 * hlf + 1]);
                    } else {
                        wg::bf16_split2(A[r0 * K + c], A[r0 * K + c + 1], f.hi[0][2 * hlf], f.lo[0][2 * hlf]);
                        wg::bf16_split2(A[r1 * K + c], A[r1 * K + c + 1], f.hi[0][2 * hlf + 1], f.lo[0][2 * hlf + 1]);
                    }
                }
            }
        }
        wg::fence_regs(d);
        wg::fence();
        for (int p = 0; p < 3; ++p) {
            const uint32_t acc = (s > 0 || p > 0) ? 1u : 0u;
            const uint32_t bb = b + (p == 1 ? bpart : 0u);
            const uint32_t aa = a + (p == 0 ? apart : 0u);
            if (mode == 0) wg::mma_tf32_rs<N>(d, p == 0 ? f.lo[0] : f.hi[0], wg::desc_kmajor(bb, K, 4) + 16u * s, acc);
            else if (mode == 1) wg::mma_f16_rs<N, 0>(d, p == 0 ? f.lo[0] : f.hi[0], wg::desc_kmajor(bb, K, 8) + 16u * s, acc);
            else if (mode == 2) wg::mma_bf16_rs<N, 1>(d, p == 0 ? f.lo[0] : f.hi[0], wg::desc_mnmajor(bb, N) + 2u * (N / 8) * 8u * s, acc);
            else if (mode == 3)
                wg::mma_bf16_ss<N, 1, 1>(d, wg::desc_mnmajor(aa + wgi * 1024u, 128) + 2u * 16u * 8u * s,
                                         wg::desc_mnmajor(bb, N) + 2u * (N / 8) * 8u * s, acc);
            else
                wg::mma_bf16_ss<N, 0, 0>(d, wg::desc_kmajor(aa + wgi * 64u * (K / 8) * 16u, K, 8) + 16u * s,
                                         wg::desc_kmajor(bb, K, 8) + 16u * s, acc);
        }
        wg::commit();
        wg::wait_all();
        wg::fence_regs(d);
    }
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
        const int c = 8 * j + 2 * t;
        D[r0 * N + c] = d[4 * j]; D[r0 * N + c + 1] = d[4 * j + 1];
        D[r1 * N + c] = d[4 * j + 2]; D[r1 * N + c + 1] = d[4 * j + 3];
    }
}

template <int N>
cudaError_t launch_n(int K, int mode, const float* A, const float* B, float* D, cudaStream_t st) {
    const size_t bytes = 2u * N * K * 4u + 2u * 128u * K * 2u;
    cudaError_t e = cudaFuncSetAttribute(wgmma_selftest_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    wgmma_selftest_kernel<N><<<1, 256, bytes, st>>>(K, mode, A, B, D);
    return cudaGetLastError();
}

}  // namespace
}  // namespace g4d

// cfg = (N, K, mode): N in {16, 48, 128}, K a multiple of 16 up to 128, mode 0..4 (above)
extern "C" int g4d_selftest_wgmma(const int* cfg, const float* A, const float* B, float* D, void* stream) {
    const int N = cfg[0], K = cfg[1], mode = cfg[2];
    if (K <= 0 || K > 128 || K % 16 != 0 || mode < 0 || mode > 4) return -1;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaErrorInvalidValue;
    if (N == 128) e = g4d::launch_n<128>(K, mode, A, B, D, st);
    else if (N == 48) e = g4d::launch_n<48>(K, mode, A, B, D, st);
    else if (N == 16) e = g4d::launch_n<16>(K, mode, A, B, D, st);
    return e == cudaSuccess ? 0 : -1;
}
