// ubench_fnv.cu -- the lane-serial FNV-64a / CBOR block hash as a DEPENDENCY CHAIN: cycles per 16-token block for one warp per
// SM sub-partition (what a launch with few chains waits for: the class pipeline's kernel H runs about one warp per SM
// sub-partition) and at full occupancy (issue bound), for several ways of writing
// the byte step.  All variants must give the same hash.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench_fnv scripts/ubench_fnv.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

// token widths: CBOR uint of a 32-bit token = 1 / 2 / 3 / 5 bytes (header + 0 / 1 / 2 / 4)
#define SETUP "setp.ge.u32 p1, %2, 24;\n\tsetp.ge.u32 p2, %2, 256;\n\tsetp.ge.u32 p3, %2, 65536;\n\tmov.u32 b, %2;\n\t@p1 mov.u32 b, 0x18;\n\t@p2 mov.u32 b, 0x19;\n\t@p3 mov.u32 b, 0x1a;\n\t"

struct VA {   // round-1/2 form: hi chain = two dependent IMADs, low word committed by a predicated move
    uint32_t lo, hi;
    __device__ __forceinline__ void step(uint32_t b) { const uint32_t x = lo ^ b; const uint64_t w = (uint64_t)x * 0x1b3u; const uint32_t u = hi * 0x1b3u + (uint32_t)(w >> 32); hi = x * 256u + u; lo = (uint32_t)w; }
#define SU(BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\tmad.lo.u32 u, %1, 0x1b3, wh;\n\tmad.lo.u32 %1, x, 256, u;\n\tmov.u32 %0, wl;\n\t"
#define SP(P, BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\tmad.lo.u32 u, %1, 0x1b3, wh;\n\t@" P " mad.lo.u32 %1, x, 256, u;\n\t@" P " mov.u32 %0, wl;\n\t"
    __device__ __forceinline__ void token(uint32_t t) {
        asm("{\n\t.reg .pred p1, p2, p3;\n\t.reg .u32 x, u, b, wl, wh;\n\t.reg .u64 w;\n\t" SETUP
            SU("") SP("p3", "shr.u32 b, %2, 24;\n\t") SP("p3", "bfe.u32 b, %2, 16, 8;\n\t") SP("p2", "bfe.u32 b, %2, 8, 8;\n\t") SP("p1", "and.b32 b, %2, 0xff;\n\t")
            "}" : "+r"(lo), "+r"(hi) : "r"(t));
    }
#undef SU
#undef SP
};

struct VB {   // hi = hi * 0x1b3 + (x * 256 + carry): ONE IMAD on the hi chain
    uint32_t lo, hi;
    __device__ __forceinline__ void step(uint32_t b) { const uint32_t x = lo ^ b; const uint64_t w = (uint64_t)x * 0x1b3u; const uint32_t c = x * 256u + (uint32_t)(w >> 32); hi = hi * 0x1b3u + c; lo = (uint32_t)w; }
#define SU(BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\tmad.lo.u32 u, x, 256, wh;\n\tmad.lo.u32 %1, %1, 0x1b3, u;\n\tmov.u32 %0, wl;\n\t"
#define SP(P, BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\tmad.lo.u32 u, x, 256, wh;\n\t@" P " mad.lo.u32 %1, %1, 0x1b3, u;\n\t@" P " mov.u32 %0, wl;\n\t"
    __device__ __forceinline__ void token(uint32_t t) {
        asm("{\n\t.reg .pred p1, p2, p3;\n\t.reg .u32 x, u, b, wl, wh;\n\t.reg .u64 w;\n\t" SETUP
            SU("") SP("p3", "shr.u32 b, %2, 24;\n\t") SP("p3", "bfe.u32 b, %2, 16, 8;\n\t") SP("p2", "bfe.u32 b, %2, 8, 8;\n\t") SP("p1", "and.b32 b, %2, 0xff;\n\t")
            "}" : "+r"(lo), "+r"(hi) : "r"(t));
    }
#undef SU
#undef SP
};

struct VC {   // no select on either chain: a skipped byte is the step (h ^ 0) * 1 -- multiplier and byte are chosen per token
    uint32_t lo, hi;
    __device__ __forceinline__ void step(uint32_t b) { const uint32_t x = lo ^ b; const uint64_t w = (uint64_t)x * 0x1b3u; const uint32_t c = x * 256u + (uint32_t)(w >> 32); hi = hi * 0x1b3u + c; lo = (uint32_t)w; }
    __device__ __forceinline__ void stepm(uint32_t b, uint32_t m, uint32_t k) {      // m = 0x1b3 / 1, k = 256 / 0
        const uint32_t x = lo ^ b; const uint64_t w = (uint64_t)x * m; const uint32_t c = x * k + (uint32_t)(w >> 32); hi = hi * m + c; lo = (uint32_t)w;
    }
    __device__ __forceinline__ void token(uint32_t t) {
        const bool p1 = t >= 24u, p2 = t >= 256u, p3 = t >= 65536u;
        const uint32_t hdr = p3 ? 0x1au : p2 ? 0x19u : p1 ? 0x18u : t;
        step(hdr);
        const uint32_t m3 = p3 ? 0x1b3u : 1u, k3 = p3 ? 256u : 0u, m2 = p2 ? 0x1b3u : 1u, k2 = p2 ? 256u : 0u, m1 = p1 ? 0x1b3u : 1u, k1 = p1 ? 256u : 0u;
        stepm(p3 ? t >> 24 : 0u, m3, k3);
        stepm(p3 ? (t >> 16) & 0xffu : 0u, m3, k3);
        stepm(p2 ? (t >> 8) & 0xffu : 0u, m2, k2);
        stepm(p1 ? t & 0xffu : 0u, m1, k1);
    }
};

struct VD {   // low chain through a 32-bit IMAD (mul.lo), carry word by mul.hi beside it; predicated commits as in VB
    uint32_t lo, hi;
    __device__ __forceinline__ void step(uint32_t b) { const uint32_t x = lo ^ b; const uint32_t c = x * 256u + __umulhi(x, 0x1b3u); hi = hi * 0x1b3u + c; lo = x * 0x1b3u; }
#define SU(BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.hi.u32 wh, x, 0x1b3;\n\tmul.lo.u32 %0, x, 0x1b3;\n\tmad.lo.u32 u, x, 256, wh;\n\tmad.lo.u32 %1, %1, 0x1b3, u;\n\t"
#define SP(P, BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.hi.u32 wh, x, 0x1b3;\n\t@" P " mul.lo.u32 %0, x, 0x1b3;\n\tmad.lo.u32 u, x, 256, wh;\n\t@" P " mad.lo.u32 %1, %1, 0x1b3, u;\n\t"
    __device__ __forceinline__ void token(uint32_t t) {
        asm("{\n\t.reg .pred p1, p2, p3;\n\t.reg .u32 x, u, b, wh;\n\t" SETUP
            SU("") SP("p3", "shr.u32 b, %2, 24;\n\t") SP("p3", "bfe.u32 b, %2, 16, 8;\n\t") SP("p2", "bfe.u32 b, %2, 8, 8;\n\t") SP("p1", "and.b32 b, %2, 0xff;\n\t")
            "}" : "+r"(lo), "+r"(hi) : "r"(t));
    }
#undef SU
#undef SP
};

template <class F>
__device__ __forceinline__ uint64_t block_hash(uint64_t parent, const uint32_t (&t)[16]) {
    F f;
    const uint64_t after = ((0xCBF29CE484222325ull ^ 0x83ull) * 0x100000001B3ull ^ 0x1bull) * 0x100000001B3ull;
    f.lo = (uint32_t)after; f.hi = (uint32_t)(after >> 32);
    const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
    f.step(ph >> 24); f.step((ph >> 16) & 0xffu); f.step((ph >> 8) & 0xffu); f.step(ph & 0xffu);
    f.step(pl >> 24); f.step((pl >> 16) & 0xffu); f.step((pl >> 8) & 0xffu); f.step(pl & 0xffu);
    f.step(0x90u);
#pragma unroll
    for (int i = 0; i < 16; ++i) f.token(t[i]);
    f.step(0xf6u);
    return ((uint64_t)f.hi << 32) | f.lo;
}

template <class F>
__global__ void k(uint64_t* out, const uint32_t* tok, int iters) {
    uint32_t t[16];
    for (int i = 0; i < 16; ++i) t[i] = tok[(threadIdx.x * 16 + i) & 1023];
    uint64_t h = 0xcbf29ce484222325ull + threadIdx.x + blockIdx.x * 977;
    for (int it = 0; it < iters; ++it) h = block_hash<F>(h | (1ull << 63), t);
    out[blockIdx.x * blockDim.x + threadIdx.x] = h;
}

template <class F>
void run(const char* name, uint64_t* dout, const uint32_t* dt, int sms, uint64_t* first) {
    const int iters = 2000;
    printf("%-44s", name);
    for (int wps : {4, 8, 32, 64}) {          // warps per SM
        dim3 grid(sms * (wps >= 8 ? wps / 8 : 1)), block(wps >= 8 ? 256 : wps * 32);
        k<F><<<grid, block>>>(dout, dt, 10); cudaDeviceSynchronize();
        cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
        cudaEventRecord(a); k<F><<<grid, block>>>(dout, dt, iters); cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b);
        printf("  %2d w/SM: %5.0f cyc/blk %.2e blk/s", wps, ms * 1e-3 * 1.965e9 / iters, (double)grid.x * block.x * iters / (ms * 1e-3));
    }
    uint64_t h0; cudaMemcpy(&h0, dout + 5, 8, cudaMemcpyDeviceToHost);
    if (*first == 0) *first = h0;
    printf("  %s\n", h0 == *first ? "same hash" : "HASH DIFFERS");
}

int main() {
    uint32_t ht[1024]; uint64_t s = 1;
    for (int i = 0; i < 1024; ++i) { s = s * 6364136223846793005ull + 1442695040888963407ull; ht[i] = (uint32_t)((s >> 33) % 128256); if (i % 7 == 0) ht[i] %= 200; if (i % 11 == 0) ht[i] %= 20; }
    uint32_t* dt; uint64_t* dout; cudaMalloc(&dt, sizeof ht); cudaMemcpy(dt, ht, sizeof ht, cudaMemcpyHostToDevice);
    cudaMalloc(&dout, 132 * 2048 * 8);
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    uint64_t first = 0;
    run<VA>("A  two IMADs on the hi chain, pred. move", dout, dt, p.multiProcessorCount, &first);
    run<VB>("B  one IMAD on the hi chain, pred. move", dout, dt, p.multiProcessorCount, &first);
    run<VC>("C  multiplier / byte selected, no predicates", dout, dt, p.multiProcessorCount, &first);
    run<VD>("D  mul.lo + mul.hi, one IMAD on the hi chain", dout, dt, p.multiProcessorCount, &first);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("cuda error\n"); return 1; }
    return 0;
}
