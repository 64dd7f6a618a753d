// Micro-benchmark: random-access read throughput of H100 HBM3 as a function of the contiguous chunk size.
// Each group of (S/16) lanes reads one S-byte chunk (16 B per lane) at a pseudo-random S-aligned offset of an
// 8 GB buffer; 8 independent chunks in flight per lane group per iteration.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint64_t mix(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return x; }
template <int LPG>   // lanes per group (chunk = LPG*16 bytes)
__global__ void k(const uint4* buf, uint64_t nchunks, int iters, uint32_t* out) {
    const uint64_t tid = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const uint64_t grp = tid / LPG; const int l = tid % LPG;
    uint32_t acc = 0;
    for (int it = 0; it < iters; ++it) {
        uint4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const uint64_t c = mix(grp * 1315423911ull + it * 8 + u) % nchunks;
            v[u] = __ldg(buf + c * LPG + l);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    if (acc == 0x12345) out[0] = acc;
}
template <int LPG> void run(const uint4* buf, uint64_t bytes, uint32_t* out) {
    const uint64_t nchunks = bytes / (LPG * 16);
    const int iters = 64; dim3 grid(132 * 16), block(256);
    k<LPG><<<grid, block>>>(buf, nchunks, 2, out); cudaDeviceSynchronize();
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a); k<LPG><<<grid, block>>>(buf, nchunks, iters, out); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    const double total = (double)grid.x * block.x * iters * 8 * 16;
    printf("chunk %4d B: %.2f ms  %.1f GB/s  %.2f G chunks/s\n", LPG * 16, ms, total / ms / 1e6, total / (LPG * 16) / ms / 1e6);
}
int main() {
    const uint64_t bytes = 8ull << 30; uint4* buf; uint32_t* out;
    cudaMalloc(&buf, bytes); cudaMemset(buf, 1, bytes); cudaMalloc(&out, 4);
    run<1>(buf, bytes, out); run<2>(buf, bytes, out); run<4>(buf, bytes, out); run<8>(buf, bytes, out); run<16>(buf, bytes, out); run<32>(buf, bytes, out);
    return 0;
}
