// ubench_green.cu -- can an SM partition (CUDA green contexts) keep a latency-chain kernel fast beside a bandwidth-bound one?
// The class pipeline's short kernels run about twice as long beside the token-streaming kernel G as alone (DESIGN.md 5): their
// dependent instruction chains share issue slots with G's 24 warps per SM.  This probe (1) checks that runtime-API launches,
// events and cross-stream waits work on streams created with cuGreenCtxStreamCreate, and that the kernels stay on their SMs;
// (2) times a serial-chain kernel (an FNV-like dependent multiply chain + dependent loads, one warp per CTA, few CTAs) alone,
// beside a DRAM-streaming kernel on ordinary streams with priorities, and beside it with the two kernels on disjoint partitions.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench_green scripts/ubench_green.cu -lcuda
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <cuda.h>
#include <cuda_runtime.h>

#define CU(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { const char* s_ = nullptr; cuGetErrorString(r_, &s_); printf("%s -> %d %s (line %d)\n", #x, (int)r_, s_ ? s_ : "?", __LINE__); return 2; } } while (0)
#define RT(x) do { cudaError_t r_ = (x); if (r_ != cudaSuccess) { printf("%s -> %s (line %d)\n", #x, cudaGetErrorString(r_), __LINE__); return 3; } } while (0)

__device__ __forceinline__ unsigned smid() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }

// bandwidth hog: streams `n` uint4 through the SMs, persistent grid
__global__ void __launch_bounds__(256) hog(const uint4* __restrict__ src, size_t n, unsigned long long* sink, unsigned* sm_mask) {
    if (threadIdx.x == 0) atomicOr(&sm_mask[smid() >> 5], 1u << (smid() & 31));
    uint32_t acc = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint4 v; asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
        acc += v.x ^ v.w;
    }
    if (acc == 0x12345u) *sink = acc;
}

// latency chain: per lane a dependent multiply chain (like the lane-serial FNV) with a dependent scattered load every 64 steps
__global__ void __launch_bounds__(256) chain(const uint32_t* __restrict__ tab, uint32_t mask, int steps, unsigned long long* out, unsigned* sm_mask) {
    if (threadIdx.x == 0) atomicOr(&sm_mask[smid() >> 5], 1u << (smid() & 31));
    uint64_t h = 0xcbf29ce484222325ull + blockIdx.x * 977 + threadIdx.x;
    for (int s = 0; s < steps; ++s) {
        h = (h ^ (s & 0xff)) * 0x100000001b3ull;
        if ((s & 63) == 63) h += tab[(uint32_t)(h >> 20) & mask];
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = h;
}

static int popc_mask(const unsigned* m) { int c = 0; for (int i = 0; i < 8; ++i) c += __builtin_popcount(m[i]); return c; }

int main() {
    RT(cudaSetDevice(0)); RT(cudaFree(0));
    CUdevice dev; CU(cuDeviceGet(&dev, 0));
    cudaDeviceProp prop; RT(cudaGetDeviceProperties(&prop, 0));
    const size_t hog_n = (size_t)3 << 26;                      // 3 GiB of uint4
    uint4* big; RT(cudaMalloc(&big, hog_n * 16)); RT(cudaMemset(big, 1, hog_n * 16));
    uint32_t* tab; const uint32_t tmask = (1u << 26) - 1; RT(cudaMalloc(&tab, ((size_t)tmask + 1) * 4)); RT(cudaMemset(tab, 0, ((size_t)tmask + 1) * 4));
    unsigned long long *sink, *out; RT(cudaMalloc(&sink, 8)); RT(cudaMalloc(&out, 8 * 256 * 1024));
    unsigned *mask_h, *mask_c; RT(cudaMalloc(&mask_h, 32)); RT(cudaMalloc(&mask_c, 32));
    int lo = 0, hi = 0; RT(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    cudaEvent_t e0, e1, eh; RT(cudaEventCreate(&e0)); RT(cudaEventCreate(&e1)); RT(cudaEventCreateWithFlags(&eh, cudaEventDisableTiming));
    const int chain_ctas = 40, chain_steps = 60000;            // ~ kernel H: a few hundred warps, tens of microseconds

    auto run = [&](const char* name, cudaStream_t s_chain, cudaStream_t s_hog, int hog_ctas_per_sm, int sms_hog, bool with_hog) -> int {
        float best = 1e9f, sum = 0; unsigned mh[8] = {}, mc[8] = {};
        for (int rep = 0; rep < 6; ++rep) {
            RT(cudaMemsetAsync(mask_h, 0, 32, s_hog)); RT(cudaMemsetAsync(mask_c, 0, 32, s_chain));
            RT(cudaDeviceSynchronize());
            if (with_hog) hog<<<sms_hog * hog_ctas_per_sm, 256, 0, s_hog>>>(big, hog_n, sink, mask_h);
            RT(cudaEventRecord(e0, s_chain));
            chain<<<chain_ctas, 256, 0, s_chain>>>(tab, tmask, chain_steps, out, mask_c);
            RT(cudaEventRecord(e1, s_chain));
            RT(cudaEventSynchronize(e1));
            float ms; RT(cudaEventElapsedTime(&ms, e0, e1));
            RT(cudaDeviceSynchronize());
            if (rep >= 1) { best = ms < best ? ms : best; sum += ms; }
            RT(cudaMemcpy(mh, mask_h, 32, cudaMemcpyDeviceToHost)); RT(cudaMemcpy(mc, mask_c, 32, cudaMemcpyDeviceToHost));
        }
        unsigned both = 0; for (int i = 0; i < 8; ++i) both += __builtin_popcount(mh[i] & mc[i]);
        printf("%-64s chain: min %7.1f us  mean %7.1f us   SMs used: chain %3d, hog %3d, shared %3d\n", name, best * 1e3, sum / 5 * 1e3, popc_mask(mc), popc_mask(mh), both);
        return 0;
    };

    cudaStream_t s1, s2, shi, slo;
    RT(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking)); RT(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
    RT(cudaStreamCreateWithPriority(&shi, cudaStreamNonBlocking, hi)); RT(cudaStreamCreateWithPriority(&slo, cudaStreamNonBlocking, lo));
    if (run("alone", s1, s2, 3, prop.multiProcessorCount, false)) return 1;
    if (run("beside the hog (3 CTAs/SM), ordinary streams", s1, s2, 3, prop.multiProcessorCount, true)) return 1;
    if (run("beside the hog (3 CTAs/SM), chain high / hog low priority", shi, slo, 3, prop.multiProcessorCount, true)) return 1;
    if (run("beside the hog (2 CTAs/SM), chain high / hog low priority", shi, slo, 2, prop.multiProcessorCount, true)) return 1;

    // ---- green contexts: `small` SMs for the chain, the rest for the hog
    for (unsigned small : {8u, 16u, 32u}) {
        CUdevResource all; CU(cuDeviceGetDevResource(dev, &all, CU_DEV_RESOURCE_TYPE_SM));
        CUdevResource grp[1], rem; unsigned int ng = 1;
        CU(cuDevSmResourceSplitByCount(grp, &ng, &all, &rem, 0, small));
        printf("split: asked %u SMs -> group %u SMs, remaining %u SMs (device %u)\n", small, grp[0].sm.smCount, rem.sm.smCount, all.sm.smCount);
        CUdevResourceDesc d_small, d_big; CU(cuDevResourceGenerateDesc(&d_small, &grp[0], 1)); CU(cuDevResourceGenerateDesc(&d_big, &rem, 1));
        CUgreenCtx g_small, g_big; CU(cuGreenCtxCreate(&g_small, d_small, dev, CU_GREEN_CTX_DEFAULT_STREAM)); CU(cuGreenCtxCreate(&g_big, d_big, dev, CU_GREEN_CTX_DEFAULT_STREAM));
        CUstream cs_small, cs_big; CU(cuGreenCtxStreamCreate(&cs_small, g_small, CU_STREAM_NON_BLOCKING, hi)); CU(cuGreenCtxStreamCreate(&cs_big, g_big, CU_STREAM_NON_BLOCKING, lo));
        // events of the primary context on a partition's stream, and a wait across the partitions
        cudaError_t er = cudaEventRecord(eh, (cudaStream_t)cs_big);
        printf("cudaEventRecord(primary-context event, partition stream): %s\n", cudaGetErrorString(er)); cudaGetLastError();
        er = cudaStreamWaitEvent((cudaStream_t)cs_small, eh, 0);
        printf("cudaStreamWaitEvent(other partition's stream, that event): %s\n", cudaGetErrorString(er)); cudaGetLastError();
        er = cudaStreamWaitEvent(s1, eh, 0);
        printf("cudaStreamWaitEvent(ordinary stream, that event): %s\n", cudaGetErrorString(er)); cudaGetLastError();
        RT(cudaDeviceSynchronize());
        char nm[128];
        snprintf(nm, sizeof nm, "partition %u | %u SMs: chain alone on the small one", grp[0].sm.smCount, rem.sm.smCount);
        if (run(nm, (cudaStream_t)cs_small, (cudaStream_t)cs_big, 3, rem.sm.smCount, false)) return 1;
        snprintf(nm, sizeof nm, "partition %u | %u SMs: chain beside the hog (3 CTAs/SM)", grp[0].sm.smCount, rem.sm.smCount);
        if (run(nm, (cudaStream_t)cs_small, (cudaStream_t)cs_big, 3, rem.sm.smCount, true)) return 1;
        // the hog's own rate on the big partition vs the whole device
        for (int which = 0; which < 2; ++which) {
            cudaStream_t hs = which ? (cudaStream_t)cs_big : s2; const int sms = which ? rem.sm.smCount : prop.multiProcessorCount;
            RT(cudaDeviceSynchronize());
            RT(cudaEventRecord(e0, hs)); hog<<<sms * 3, 256, 0, hs>>>(big, hog_n, sink, mask_h); RT(cudaEventRecord(e1, hs)); RT(cudaEventSynchronize(e1));
            float ms; RT(cudaEventElapsedTime(&ms, e0, e1));
            printf("   hog alone on %3d SMs: %.3f ms = %.0f GB/s\n", sms, ms, hog_n * 16 / (ms / 1e3) / 1e9);
        }
        RT(cudaDeviceSynchronize());
        CU(cuStreamDestroy(cs_small)); CU(cuStreamDestroy(cs_big));
        CU(cuGreenCtxDestroy(g_small)); CU(cuGreenCtxDestroy(g_big));
    }
    printf("done\n");
    return 0;
}
