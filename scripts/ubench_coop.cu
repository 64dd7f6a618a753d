// ubench_coop.cu -- cycles per 16-token block of the warp-cooperative FNV (kernels_coop.cuh) vs the plain serial chain,
// ONE warp, tokens already in shared memory; checks both against each other.  Build on the GPU box:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o scripts/ubench_coop scripts/ubench_coop.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include "../llm-d-kv-cache-manager_b200/csrc/kernels_coop.cuh"
using namespace kvx;

__global__ void k_coop(const uint32_t* tok, int nchunks, uint64_t init, uint64_t* out, long long* cyc) {
    extern __shared__ __align__(128) unsigned char smem[];
    CoopSmem& sm = *reinterpret_cast<CoopSmem*>(smem);
    const int lane = threadIdx.x & 31;
    const uint32_t lt = (1u << lane) - 1u;
    for (int i = threadIdx.x; i <= kCoopMaxPayload; i += 32) { unsigned long long p = 1; for (int q = 0; q < i; ++q) p *= kFnvPrime; sm.tab.pw[i] = p; sm.tab.c0[i] = kFnvOffset * p; }
    __syncwarp();
    CoopSmem::Warp& W = sm.w[0];
    uint64_t h = init;
    long long t_layout = 0, t_hash = 0;
    for (int c = 0; c < nchunks; ++c) {
        for (int x = lane; x < 512; x += 32) W.tok[0][x] = tok[c * 512 + x];
        __syncwarp();
        long long t0 = clock64();
        coop_layout_chunk(W, W.tok[0], 32, lane);
        __syncwarp();
        long long t1 = clock64();
        uint64_t key = 0, last = 0;
        // same loop as coop_hash_chunk without the probe hook
        uint32_t tb, b0, b1, b2, vm;
        coop_block_bytes(W, 0, lane, tb, b0, b1, b2, vm);
        for (int j = 0; j < 32; ++j) {
            uint32_t ntb = 0, nb0 = 0, nb1 = 0, nb2 = 0, nvm = 0;
            if (j + 1 < 32) coop_block_bytes(W, j + 1, lane, ntb, nb0, nb1, nb2, nvm);
            h = coop_hash_block(sm.tab, h, tb, b0, b1, b2, vm, lane, lt);
            if (lane == j) key = h;
            tb = ntb; b0 = nb0; b1 = nb1; b2 = nb2; vm = nvm;
        }
        last = h;
        long long t2 = clock64();
        t_layout += t1 - t0; t_hash += t2 - t1;
        out[c * 32 + lane] = key;
        (void)last;
    }
    if (lane == 0) { cyc[0] = t_layout; cyc[1] = t_hash; }
}

// the plain chain with WARP-UNIFORM control flow (one chain per warp, every lane the same): exactly the bytes a token has,
// critical path = xor + 32-bit multiply per byte
__global__ void k_uniform(const uint32_t* tok, int nblocks, uint64_t init, uint64_t* out, long long* cyc) {
    uint64_t h = init;
    long long t0 = clock64();
    for (int b = 0; b < nblocks; ++b) {
        Fnv f; f.begin_block(h, 16);
#pragma unroll
        for (int c = 0; c < 16; ++c) f.uint32(tok[b * 16 + c]);
        h = f.end_block();
        if (threadIdx.x == 0) out[b] = h;
    }
    if (threadIdx.x == 0) cyc[0] = clock64() - t0;
}

__global__ void k_serial(const uint32_t* tok, int nblocks, uint64_t init, uint64_t* out, long long* cyc) {
    uint64_t h = init;
    long long t0 = clock64();
    for (int b = 0; b < nblocks; ++b) {
        Fnv f; f.begin_block(h, 16);
        for (int c = 0; c < 16; ++c) f.token(tok[b * 16 + c]);
        h = f.end_block();
        if (threadIdx.x == 0) out[b] = h;
    }
    if (threadIdx.x == 0) cyc[0] = clock64() - t0;
}

int main() {
    const int nchunks = 8, nb = nchunks * 32;
    std::vector<uint32_t> tok(nb * 16);
    uint64_t s = 12345;
    for (auto& t : tok) { s = s * 6364136223846793005ull + 1442695040888963407ull; t = (uint32_t)((s >> 33) % 128256); }
    tok[3] = 5; tok[4] = 200; tok[5] = 65535; tok[6] = 65536; tok[7] = 0xffffffffu; tok[8] = 23; tok[9] = 24;
    uint32_t* d_tok; uint64_t *d_o1, *d_o2; long long* d_c;
    cudaMalloc(&d_tok, tok.size() * 4); cudaMalloc(&d_o1, nb * 8); cudaMalloc(&d_o2, nb * 8); cudaMalloc(&d_c, 64);
    cudaMemcpy(d_tok, tok.data(), tok.size() * 4, cudaMemcpyHostToDevice);
    cudaFuncSetAttribute(k_coop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem));
    long long c[4];
    for (int rep = 0; rep < 3; ++rep) {
        k_coop<<<1, 32, sizeof(CoopSmem)>>>(d_tok, nchunks, kFnvOffset, d_o1, d_c);
        cudaMemcpy(c, d_c, 16, cudaMemcpyDeviceToHost);
        k_serial<<<1, 32>>>(d_tok, nb, kFnvOffset, d_o2, d_c + 2);
        cudaMemcpy(c + 2, d_c + 2, 8, cudaMemcpyDeviceToHost);
        k_uniform<<<1, 32>>>(d_tok, nb, kFnvOffset, d_o2, d_c + 3);
        cudaMemcpy(c + 3, d_c + 3, 8, cudaMemcpyDeviceToHost);
        if (cudaDeviceSynchronize() != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
        printf("coop: layout %.1f cycles/block, hash %.1f cycles/block | branch-free lane chain %.1f | warp-uniform exact-byte chain %.1f cycles/block\n",
               (double)c[0] / nb, (double)c[1] / nb, (double)c[2] / nb, (double)c[3] / nb);
    }
    std::vector<uint64_t> o1(nb), o2(nb);
    cudaMemcpy(o1.data(), d_o1, nb * 8, cudaMemcpyDeviceToHost); cudaMemcpy(o2.data(), d_o2, nb * 8, cudaMemcpyDeviceToHost);
    int bad = 0;
    for (int i = 0; i < nb; ++i) bad += o1[i] != o2[i];
    printf("keys equal: %s (%d mismatches)\n", bad ? "NO" : "yes", bad);
    return bad != 0;
}
