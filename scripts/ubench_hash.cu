// Micro-benchmark: issue rate of the branch-free FNV/CBOR block hash alone (no memory traffic),
// as a function of resident warps per SM.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/ubench scripts/ubench_hash.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#include "../llm-d-kv-cache-manager_b200/csrc/fnv_cbor.cuh"
using namespace kvx;
__global__ void k(uint64_t* out, const uint32_t* tok, int iters) {
    uint32_t t[16];
    for (int i = 0; i < 16; ++i) t[i] = tok[(threadIdx.x * 16 + i) & 1023];
    uint64_t h = 0xcbf29ce484222325ull + threadIdx.x + blockIdx.x * 977;
    for (int it = 0; it < iters; ++it) {
        Fnv f; f.begin_block(h, 16);
#pragma unroll
        for (int i = 0; i < 16; ++i) f.token(t[i]);
        h = f.end_block();
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = h;
}
int main() {
    uint32_t ht[1024]; uint64_t s = 1;
    for (int i = 0; i < 1024; ++i) { s = s * 6364136223846793005ull + 1442695040888963407ull; ht[i] = (uint32_t)((s >> 33) % 128256); }
    uint32_t* dt; uint64_t* dout; cudaMalloc(&dt, sizeof ht); cudaMemcpy(dt, ht, sizeof ht, cudaMemcpyHostToDevice);
    cudaMalloc(&dout, 132 * 2048 * 8);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int iters = 2000;
    for (int wps = 4; wps <= 64; wps *= 2) {          // warps per SM
        dim3 grid(p.multiProcessorCount * (wps >= 8 ? wps / 8 : 1)), block(wps >= 8 ? 256 : wps * 32);
        k<<<grid, block>>>(dout, dt, 10); cudaDeviceSynchronize();
        cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
        cudaEventRecord(a); k<<<grid, block>>>(dout, dt, iters); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b);
        double blocks = (double)grid.x * block.x * iters;
        int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);   // max SM clock
        printf("warps/SM %2d: %.3f ms  %.3e block-hashes/s  cycles/block/warp @%.3fGHz = %.0f\n", wps, ms, blocks / (ms * 1e-3),
               khz / 1e6, ms * 1e-3 * khz * 1e3 / iters);
    }
    return 0;
}
