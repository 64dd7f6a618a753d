// ubench_peer.cu -- how fast can one H100 read random 32-byte slots out of ANOTHER H100's HBM over NVLink (the access the
// sharded index's walk makes), next to the same reads from its own HBM?  Independent reads, every lane its own address,
// a slot as two 16-byte loads (LDG.E.128, Hopper's widest) -- no dependence between a thread's loads except through the final checksum.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench_peer scripts/ubench_peer.cu ; scripts/ubench_peer
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t mix(uint64_t z) { z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull; z ^= z >> 27; z *= 0x94D049BB133111EBull; return z ^ (z >> 31); }

template <int PER>
__global__ void rd(const uint4* __restrict__ tab, uint64_t mask_slots, int iters, unsigned long long* sink) {
    uint64_t s = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ull + 1;
    uint32_t acc = 0;
    for (int it = 0; it < iters; ++it) {
        uint4 a[PER], b[PER];
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            s = mix(s + u);
            const uint4* p = tab + 2 * (s & mask_slots);
            asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(a[u].x), "=r"(a[u].y), "=r"(a[u].z), "=r"(a[u].w) : "l"(p) : "memory");
            asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(b[u].x), "=r"(b[u].y), "=r"(b[u].z), "=r"(b[u].w) : "l"(p + 1) : "memory");
        }
#pragma unroll
        for (int u = 0; u < PER; ++u) acc += a[u].x ^ b[u].w;
    }
    if (acc == 0x12345678u) *sink = acc;
}

int main() {
    int nd = 0; cudaGetDeviceCount(&nd);
    const uint64_t slots = 1ull << 25;                      // 32 Mi slots x 32 B = 1 GiB
    uint4 *local = nullptr, *peer = nullptr; unsigned long long* sink;
    cudaSetDevice(0);
    cudaMalloc(&local, slots * 32); cudaMemset(local, 1, slots * 32); cudaMalloc(&sink, 8);
    if (nd > 1) {
        cudaSetDevice(1); cudaMalloc(&peer, slots * 32); cudaMemset(peer, 2, slots * 32); cudaDeviceSynchronize();
        cudaSetDevice(0);
        if (cudaDeviceEnablePeerAccess(1, 0) != cudaSuccess) { printf("no peer access\n"); peer = nullptr; cudaGetLastError(); }
    }
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("%-8s %-10s %-8s %14s %10s\n", "memory", "threads", "per-thr", "reads/s", "GB/s");
    for (int which = 0; which < 2; ++which) {
        const uint4* tab = which ? peer : local;
        if (!tab) continue;
        int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
        for (int ctas : {sms, sms * 4, sms * 16}) {
            const int T = 256, iters = 64;
            for (int per : {1, 4}) {
                for (int rep = 0; rep < 2; ++rep) {
                    cudaEventRecord(e0);
                    if (per == 1) rd<1><<<ctas, T>>>(tab, slots - 1, iters, sink); else rd<4><<<ctas, T>>>(tab, slots - 1, iters, sink);
                    cudaEventRecord(e1); cudaEventSynchronize(e1);
                }
                float ms; cudaEventElapsedTime(&ms, e0, e1);
                const double n = (double)ctas * T * iters * per;
                printf("%-8s %-10d %-8d %14.3e %10.1f\n", which ? "peer" : "local", ctas * T, per, n / (ms / 1e3), n * 32 / (ms / 1e3) / 1e9);
            }
        }
    }
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    return 0;
}
