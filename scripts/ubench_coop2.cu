// ubench_coop2.cu -- where do the cycles of one cooperative block hash go?  ONE warp, chained blocks (each block's parent is
// the previous result), variants of the same code:
//   0 full (8 bit planes + dot product + 3 REDUX)      1 bit planes only (+1 REDUX to keep the chain)
//   2 dot product + REDUX only (planes skipped)        3 full, warp sum by five 64-bit shuffle-adds instead of REDUX
//   4 full without the per-block shared-memory byte fetch (same bytes every block)
//   5 bit planes only, ballot + popcount replaced by a 5-step shuffle XOR scan (what the ballot saves)
//   6 full, TWO bit planes per ballot round: the upper plane's ballot for both outcomes of the lower plane's prefix parity
//     (B0, BE) is issued together with the lower plane's ballot, the true upper ballot is B0 ^ (BE & prefix_xor(B_lower))
// Build on the GPU box:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o scripts/ubench_coop2 scripts/ubench_coop2.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include "../llm-d-kv-cache-manager_b200/csrc/kernels_coop.cuh"
using namespace kvx;

__device__ __forceinline__ uint32_t ballot_bit2(uint32_t z, uint32_t bit) {
    uint32_t r;
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tand.b32 t, %1, %2;\n\tsetp.ne.u32 p, t, 0;\n\tvote.sync.ballot.b32 %0, p, 0xffffffff;\n\t}" : "=r"(r) : "r"(z), "r"(bit));
    return r;
}

template <int MODE>
__device__ __forceinline__ uint64_t hash_v(const CoopTables& tab, uint64_t parent, uint32_t tb, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t vmask, int lane, uint32_t lt) {
    if (lane < 4) {
        const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
        if (lane == 0) b2 = ph >> 24;
        else if (lane == 1) { b0 = (ph >> 16) & 0xffu; b1 = (ph >> 8) & 0xffu; b2 = ph & 0xffu; }
        else if (lane == 2) { b0 = pl >> 24; b1 = (pl >> 16) & 0xffu; b2 = (pl >> 8) & 0xffu; }
        else b0 = pl & 0xffu;
    }
    constexpr uint32_t L0 = (uint32_t)(kFnvOffset & 0xffu);
    const uint32_t bs = b0 ^ b1 ^ b2;
    uint32_t X0 = 0, X1 = 0, X2 = 0, Y0 = 0, Y1 = 0, Y2 = 0;
    if (MODE != 2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t bit = 1u << k;
            const uint32_t z0 = b0 ^ Y0, z01 = z0 ^ b1 ^ Y1;
            uint32_t par;
            if (MODE == 5) {
                uint32_t g = ((bs ^ Y0 ^ Y1 ^ Y2) >> k) & 1u, incl = g;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl ^= u; }
                par = (incl ^ g) << k;
            } else {
                const uint32_t B = ballot_bit2(bs ^ Y0 ^ Y1 ^ Y2, bit);
                par = (uint32_t)__popc(B & lt) << k;
            }
            const uint32_t t0 = (par ^ L0 ^ b0) & bit, t1 = (par ^ L0 ^ z0 ^ b1) & bit, t2 = (par ^ L0 ^ z01 ^ b2) & bit;
            X0 |= t0; X1 |= t1; X2 |= t2;
            Y0 += t0 * 0xb3u; Y1 += t1 * 0xb3u; Y2 += t2 * 0xb3u;
        }
    } else { X0 = b0 ^ (uint32_t)parent; X1 = b1; X2 = b2; }
    if (MODE == 1 || MODE == 5) return parent * 0x9E3779B97F4A7C15ull + __reduce_xor_sync(0xffffffffu, X0 ^ (X1 << 8) ^ (X2 << 16)) + (1ull << 40);
    const uint32_t n = tb + 12u, j0 = 3u * (uint32_t)lane;
    unsigned long long s = 0;
    if (vmask & 1u) s += (unsigned long long)(long long)((int)X0 - (int)(X0 ^ b0)) * tab.pw[n - j0];
    if (vmask & 2u) s += (unsigned long long)(long long)((int)X1 - (int)(X1 ^ b1)) * tab.pw[n - j0 - 1];
    if (vmask & 4u) s += (unsigned long long)(long long)((int)X2 - (int)(X2 ^ b2)) * tab.pw[n - j0 - 2];
    if (MODE == 3) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        return tab.c0[n] + s;
    }
    const uint32_t r0 = __reduce_add_sync(0xffffffffu, (uint32_t)s & 0x3fffffu), r1 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 22) & 0x1fffffu);
    const uint32_t r2 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 43));
    return tab.c0[n] + (unsigned long long)r0 + ((unsigned long long)r1 << 22) + ((unsigned long long)r2 << 43);
}

__device__ __forceinline__ uint32_t ballot_nz(uint32_t z) {
    uint32_t r;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\tvote.sync.ballot.b32 %0, p, 0xffffffff;\n\t}" : "=r"(r) : "r"(z));
    return r;
}
// mode 6
__device__ __forceinline__ uint64_t hash_pairs(const CoopTables& tab, uint64_t parent, uint32_t tb, uint32_t b0, uint32_t b1, uint32_t b2, uint32_t vmask, int lane, uint32_t lt) {
    if (lane < 4) {
        const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
        if (lane == 0) b2 = ph >> 24;
        else if (lane == 1) { b0 = (ph >> 16) & 0xffu; b1 = (ph >> 8) & 0xffu; b2 = ph & 0xffu; }
        else if (lane == 2) { b0 = pl >> 24; b1 = (pl >> 16) & 0xffu; b2 = (pl >> 8) & 0xffu; }
        else b0 = pl & 0xffu;
    }
    constexpr uint32_t L0 = (uint32_t)(kFnvOffset & 0xffu);
    const uint32_t bs = b0 ^ b1 ^ b2;
    uint32_t X0 = 0, X1 = 0, X2 = 0, Y0 = 0, Y1 = 0, Y2 = 0;
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
        const uint32_t bj = 1u << j, bn = 2u << j, inc = 0xb3u << j, inc2 = 0xb3u << (j + 1);
        // everything the three ballots need comes from the state at the start of the pair
        const uint32_t ys = bs ^ Y0 ^ Y1 ^ Y2;
        const uint32_t z0 = b0 ^ Y0, z1 = b1 ^ Y1;
        const uint32_t c0 = (L0 ^ b0) & bj, c1 = (L0 ^ z0 ^ b1) & bj, c2 = (L0 ^ z0 ^ z1 ^ b2) & bj;          // at bit j
        const uint32_t e0 = (Y0 ^ (Y0 + inc)) & bn, e1 = (Y1 ^ (Y1 + inc)) & bn, e2 = (Y2 ^ (Y2 + inc)) & bn; // at bit j+1
        const uint32_t g0 = (ys & bn) ^ ((c0 << 1) & e0) ^ ((c1 << 1) & e1) ^ ((c2 << 1) & e2);
        const uint32_t Bj = ballot_nz(ys & bj), B0 = ballot_nz(g0), BE = ballot_nz(e0 ^ e1 ^ e2);
        // lower plane: this lane's prefix parity, its x bits, the carry words of the upper plane
        const uint32_t parj = ((uint32_t)__popc(Bj & lt) & 1u) << j;
        const uint32_t t0 = parj ^ c0, t1 = parj ^ c1, t2 = parj ^ c2;
        X0 |= t0; X1 |= t1; X2 |= t2;
        Y0 += t0 * 0xb3u; Y1 += t1 * 0xb3u; Y2 += t2 * 0xb3u;
        // upper plane: every lane's lower parity as a word (exclusive prefix XOR of Bj), hence the true upper ballot
        uint32_t px = Bj; px ^= px << 1; px ^= px << 2; px ^= px << 4; px ^= px << 8; px ^= px << 16; px <<= 1;
        const uint32_t Bn = B0 ^ (BE & px);
        const uint32_t parn = ((uint32_t)__popc(Bn & lt) & 1u) << (j + 1);
        const uint32_t w0 = b0 ^ Y0, w1 = b1 ^ Y1;
        const uint32_t u0 = (parn ^ L0 ^ b0) & bn, u1 = (parn ^ L0 ^ w0 ^ b1) & bn, u2 = (parn ^ L0 ^ w0 ^ w1 ^ b2) & bn;
        X0 |= u0; X1 |= u1; X2 |= u2;
        Y0 += u0 * 0xb3u; Y1 += u1 * 0xb3u; Y2 += u2 * 0xb3u;
        (void)inc2;
    }
    const uint32_t n = tb + 12u, j0 = 3u * (uint32_t)lane;
    unsigned long long s = 0;
    if (vmask & 1u) s += (unsigned long long)(long long)((int)X0 - (int)(X0 ^ b0)) * tab.pw[n - j0];
    if (vmask & 2u) s += (unsigned long long)(long long)((int)X1 - (int)(X1 ^ b1)) * tab.pw[n - j0 - 1];
    if (vmask & 4u) s += (unsigned long long)(long long)((int)X2 - (int)(X2 ^ b2)) * tab.pw[n - j0 - 2];
    const uint32_t r0 = __reduce_add_sync(0xffffffffu, (uint32_t)s & 0x3fffffu), r1 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 22) & 0x1fffffu);
    const uint32_t r2 = __reduce_add_sync(0xffffffffu, (uint32_t)(s >> 43));
    return tab.c0[n] + (unsigned long long)r0 + ((unsigned long long)r1 << 22) + ((unsigned long long)r2 << 43);
}

// plain serial reference for the check
__device__ __forceinline__ uint64_t hash_ref(uint64_t parent, const uint32_t* tk) {
    Fnv f; f.begin_block(parent, 16);
    for (int c = 0; c < 16; ++c) f.uint32(tk[c]);
    return f.end_block();
}

template <int MODE>
__global__ void k(const uint32_t* tok, int nchunks, uint64_t init, uint64_t* out, long long* cyc) {
    extern __shared__ __align__(128) unsigned char smem[];
    CoopSmem& sm = *reinterpret_cast<CoopSmem*>(smem);
    const int lane = threadIdx.x & 31;
    const uint32_t lt = (1u << lane) - 1u;
    for (int i = threadIdx.x; i <= kCoopMaxPayload; i += 32) { unsigned long long p = 1; for (int q = 0; q < i; ++q) p *= kFnvPrime; sm.tab.pw[i] = p; sm.tab.c0[i] = kFnvOffset * p; }
    __syncwarp();
    CoopSmem::Warp& W = sm.w[0];
    uint64_t h = init | (1ull << 40);
    long long tt = 0;
    const bool check = cyc[1] != 0;
    int bad = 0;
    for (int c = 0; c < nchunks; ++c) {
        for (int x = lane; x < 512; x += 32) W.tok[0][x] = tok[c * 512 + x];
        __syncwarp();
        coop_layout_chunk(W, W.tok[0], 32, lane);
        __syncwarp();
        uint32_t tb, b0, b1, b2, vm;
        coop_block_bytes(W, 0, lane, tb, b0, b1, b2, vm);
        long long t1 = clock64();
        for (int j = 0; j < 32; ++j) {
            uint32_t ntb = tb, nb0 = b0, nb1 = b1, nb2 = b2, nvm = vm;
            if (MODE != 4 && j + 1 < 32) coop_block_bytes(W, j + 1, lane, ntb, nb0, nb1, nb2, nvm);
            if (MODE == 6 || MODE == 7) {
                const uint64_t hh = MODE == 6 ? hash_pairs(sm.tab, h, tb, b0, b1, b2, vm, lane, lt) : hash_v<0>(sm.tab, h, tb, b0, b1, b2, vm, lane, lt);
                if (check && hh != hash_ref(h, &W.tok[0][j * 16])) bad++;
                h = hh | (1ull << 40);
            } else
            h = hash_v<MODE>(sm.tab, h, tb, b0, b1, b2, vm, lane, lt) | (1ull << 40);
            tb = ntb; b0 = nb0; b1 = nb1; b2 = nb2; vm = nvm;
        }
        tt += clock64() - t1;
        out[c] = h;
    }
    if (lane == 0) { cyc[0] = tt; cyc[2] = bad; }
}

template <int MODE> void run(const char* what, const uint32_t* d_tok, int nchunks, uint64_t* d_o, long long* d_c) {
    cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem));
    long long c = 0;
    long long z[3] = {0, 0, 0};
    cudaMemcpy(d_c, z, 24, cudaMemcpyHostToDevice);
    for (int rep = 0; rep < 2; ++rep) { k<MODE><<<1, 32, sizeof(CoopSmem)>>>(d_tok, nchunks, kFnvOffset, d_o, d_c); cudaMemcpy(&c, d_c, 8, cudaMemcpyDeviceToHost); }
    printf("%-72s %8.1f cycles/block", what, (double)c / (nchunks * 32));
    if (MODE >= 6) {                                  // once more with every block checked against the plain chain
        z[1] = 1; cudaMemcpy(d_c, z, 24, cudaMemcpyHostToDevice);
        k<MODE><<<1, 32, sizeof(CoopSmem)>>>(d_tok, nchunks, kFnvOffset, d_o, d_c);
        cudaMemcpy(z, d_c, 24, cudaMemcpyDeviceToHost);
        printf("   [%lld of %d blocks differ from the plain chain]", z[2], nchunks * 32);
    }
    printf("\n");
}

int main() {
    const int nchunks = 8, nb = nchunks * 32;
    std::vector<uint32_t> tok(nb * 16);
    uint64_t s = 12345;
    for (auto& t : tok) { s = s * 6364136223846793005ull + 1442695040888963407ull; t = (uint32_t)((s >> 33) % 128256); }
    uint32_t* d_tok; uint64_t* d_o; long long* d_c;
    cudaMalloc(&d_tok, tok.size() * 4); cudaMalloc(&d_o, nb * 8); cudaMalloc(&d_c, 64);
    cudaMemcpy(d_tok, tok.data(), tok.size() * 4, cudaMemcpyHostToDevice);
    run<0>("0 full: 8 bit planes + dot product + 3 REDUX", d_tok, nchunks, d_o, d_c);
    run<1>("1 bit planes only (+1 REDUX)", d_tok, nchunks, d_o, d_c);
    run<2>("2 dot product + 3 REDUX only", d_tok, nchunks, d_o, d_c);
    run<3>("3 full, warp sum by 5 x 64-bit shuffle-add", d_tok, nchunks, d_o, d_c);
    run<4>("4 full, no per-block byte fetch from shared memory", d_tok, nchunks, d_o, d_c);
    run<5>("5 bit planes only, shuffle XOR scan instead of ballot + popcount", d_tok, nchunks, d_o, d_c);
    run<6>("6 full, two bit planes per ballot round", d_tok, nchunks, d_o, d_c);
    run<7>("7 full (variant 0 again, checked)", d_tok, nchunks, d_o, d_c);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("cuda error %s\n", cudaGetErrorString(cudaGetLastError())); return 1; }
    return 0;
}
