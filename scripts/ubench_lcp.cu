// ubench_lcp.cu -- how fast can "is this prompt's next chunk (32 blocks = 2 KB) equal to its list neighbour's, and if not, in which
// block do they part" be answered lane-parallel?  Lane i of a warp owns prompt i of the (sorted) list: it reads its own chunk and
// its predecessor's 16 bytes at a time (lane i's second load is lane i-1's first: the load unit merges them, nothing is read twice),
// no shared memory, no shuffles.  Compare with kernel G's warp-serial streaming (one chunk at a time through a shared-memory ring).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench_lcp scripts/ubench_lcp.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int UNROLL, bool NC>
__global__ void __launch_bounds__(256) lcp(const uint32_t* __restrict__ tok, const uint32_t* __restrict__ list, int n, int T, int round, uint8_t* __restrict__ fb_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = list[i], q = i > 0 ? list[i - 1] : p;
    const uint4* a = reinterpret_cast<const uint4*>(tok + (size_t)p * T + (size_t)round * 512);
    const uint4* b = reinterpret_cast<const uint4*>(tok + (size_t)q * T + (size_t)round * 512);
    int fb = 32;
    for (int j = 0; j < 128; j += UNROLL) {
        uint4 x[UNROLL], y[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            if (NC) {
                asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x[u].x), "=r"(x[u].y), "=r"(x[u].z), "=r"(x[u].w) : "l"(a + j + u));
                asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y[u].x), "=r"(y[u].y), "=r"(y[u].z), "=r"(y[u].w) : "l"(b + j + u));
            } else { x[u] = a[j + u]; y[u] = b[j + u]; }
        }
#pragma unroll
        for (int u = UNROLL - 1; u >= 0; --u)
            if (((x[u].x ^ y[u].x) | (x[u].y ^ y[u].y) | (x[u].z ^ y[u].z) | (x[u].w ^ y[u].w)) != 0u) fb = min(fb, (j + u) >> 2);
    }
    fb_out[i] = (uint8_t)fb;
}

__global__ void fill(uint32_t* tok, size_t n, int T, int docs) {
    for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n * T; k += (size_t)gridDim.x * blockDim.x) {
        const size_t p = k / T, c = k % T;
        const uint32_t d = (uint32_t)(p * 2654435761u) % docs;          // document of prompt p
        const uint32_t m = (uint32_t)((p * 40503u) >> 3) % 257u;         // blocks it shares with the document
        tok[k] = c < m * 16 ? d * 7919u + (uint32_t)c : (uint32_t)(k * 0x9E3779B1u >> 7);
    }
}

int main() {
    const int n = 1 << 18, T = 4096, docs = n / 27;
    uint32_t *tok, *list; uint8_t* fb;
    cudaMalloc(&tok, (size_t)n * T * 4); cudaMalloc(&list, n * 4); cudaMalloc(&fb, n);
    fill<<<132 * 8, 256>>>(tok, n, T, docs);
    // list: prompts sorted by document (what the prefix sort produces)
    uint32_t* h = new uint32_t[n];
    { uint32_t* key = new uint32_t[n]; for (int p = 0; p < n; ++p) { key[p] = (uint32_t)(p * 2654435761u) % docs; h[p] = p; }
      // counting sort by doc
      int* cnt = new int[docs + 1](); for (int p = 0; p < n; ++p) cnt[key[p] + 1]++; for (int d = 0; d < docs; ++d) cnt[d + 1] += cnt[d];
      for (int p = 0; p < n; ++p) h[cnt[key[p]]++] = p; }
    cudaMemcpy(list, h, n * 4, cudaMemcpyHostToDevice);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    printf("%-28s %10s %10s\n", "variant", "us/chunk-pass", "GB/s");
    auto run = [&](const char* name, auto kern, int threads) {
        float best = 1e9f;
        for (int rep = 0; rep < 6; ++rep) {
            const int round = rep % 8;
            cudaEventRecord(e0);
            kern<<<(n + threads - 1) / threads, threads>>>(tok, list, n, T, round, fb);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (rep >= 2 && ms < best) best = ms;
        }
        printf("%-28s %10.1f %10.1f\n", name, best * 1e3, (double)n * 2048 / (best / 1e3) / 1e9);
    };
    run("unroll 4, ld", lcp<4, false>, 256);
    run("unroll 8, ld", lcp<8, false>, 256);
    run("unroll 8, ld, 128 thr", lcp<8, false>, 128);
    run("unroll 16, ld", lcp<16, false>, 256);
    run("unroll 8, ld.nc", lcp<8, true>, 256);
    run("unroll 16, ld.nc", lcp<16, true>, 256);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    return 0;
}
