// fnv_cbor.cuh -- FNV-64a over canonical CBOR, evaluated byte-serially in registers.
//
// Replaces ChunkedTokenDatabase.hash (pkg/kvcache/kvblock/token_processor.go:94-112):
//   key = FNV64a( CBOR_canonical( [parent uint64, tokens []uint32, nil] ) )
// bytes: 0x83, uint(parent) shortest form, array header(B), B x uint(token) shortest form, 0xf6.
// No payload is ever materialised: each CBOR byte is folded into the running hash as it
// is produced.  The 64-bit state lives in two 32-bit registers so one FNV step is
//   x  = lo ^ b                      (LOP3, alu pipe)
//   t  = hi * 0x1b3 + (x << 8)       (IMAD + SHF/LEA)
//   {lo,hi} = x * 0x1b3 + (t << 32)  (IMAD.WIDE)
// because prime = 2^40 + 0x1b3:  (h^b)*prime = (h^b)*0x1b3 + ((h^b) << 40)  (mod 2^64).
#pragma once
#include <stdint.h>

namespace kvx {

constexpr uint64_t kFnvOffset = 0xCBF29CE484222325ull;
constexpr uint64_t kFnvPrime  = 0x100000001B3ull;

constexpr uint64_t kAfter83 = (kFnvOffset ^ 0x83ull) * kFnvPrime;          // FNV state after the array(3) head
constexpr uint64_t kAfter83_1b = (kAfter83 ^ 0x1bull) * kFnvPrime;         // ... and after the uint64 head byte

struct Fnv {
    uint32_t lo, hi;
    __host__ __device__ __forceinline__ void init() { lo = 0x84222325u; hi = 0xCBF29CE4u; }
    __host__ __device__ __forceinline__ void set(uint64_t h) { lo = (uint32_t)h; hi = (uint32_t)(h >> 32); }
    __host__ __device__ __forceinline__ uint64_t get() const { return ((uint64_t)hi << 32) | lo; }
    // one FNV-1a byte step; b must be < 256
    __host__ __device__ __forceinline__ void step(uint32_t b) {
        const uint32_t x = lo ^ b;                                  // LOP3
        const uint64_t w = (uint64_t)x * 0x1b3u;                    // IMAD.WIDE
        const uint32_t u = hi * 0x1b3u + (uint32_t)(w >> 32);       // IMAD
        hi = x * 256u + u;                                          // IMAD   ((x << 40) term)
        lo = (uint32_t)w;
    }
    // One CBOR-encoded token folded in with NO divergent control flow: every lane issues the same
    // 33 instructions; the up-to-four extra bytes of wider tokens are committed under predicates
    // (hi by a predicated IMAD, lo by a select).  ncu on the branchy form showed the compiler's
    // jump chain re-executing the shared byte steps once per divergent group (7 steps / token
    // instead of 5 for a warp that mixes 3- and 5-byte tokens).
#define KVX_STEP_U(BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\t" \
        "mad.lo.u32 u, %1, 0x1b3, wh;\n\tmad.lo.u32 %1, x, 256, u;\n\tmov.u32 %0, wl;\n\t"
#define KVX_STEP_P(P, BYTE) BYTE "xor.b32 x, %0, b;\n\tmul.wide.u32 w, x, 0x1b3;\n\tmov.b64 {wl, wh}, w;\n\t" \
        "mad.lo.u32 u, %1, 0x1b3, wh;\n\t@" P " mad.lo.u32 %1, x, 256, u;\n\t@" P " mov.u32 %0, wl;\n\t"
    __device__ __forceinline__ void token(uint32_t t) {
#ifdef __CUDA_ARCH__
        asm("{\n\t"
            ".reg .pred p1, p2, p3;\n\t"
            ".reg .u32 x, u, b, wl, wh;\n\t"
            ".reg .u64 w;\n\t"
            "setp.ge.u32 p1, %2, 24;\n\t"
            "setp.ge.u32 p2, %2, 256;\n\t"
            "setp.ge.u32 p3, %2, 65536;\n\t"
            "mov.u32 b, %2;\n\t"
            "@p1 mov.u32 b, 0x18;\n\t"
            "@p2 mov.u32 b, 0x19;\n\t"
            "@p3 mov.u32 b, 0x1a;\n\t"
            KVX_STEP_U("")
            KVX_STEP_P("p3", "shr.u32 b, %2, 24;\n\t")
            KVX_STEP_P("p3", "bfe.u32 b, %2, 16, 8;\n\t")
            KVX_STEP_P("p2", "bfe.u32 b, %2, 8, 8;\n\t")
            KVX_STEP_P("p1", "and.b32 b, %2, 0xff;\n\t")
            "}" : "+r"(lo), "+r"(hi) : "r"(t));
#else
        uint32(t);
#endif
    }
#undef KVX_STEP_U
#undef KVX_STEP_P
    // CBOR unsigned (major 0) of a 32-bit value, shortest form.  The four possible extra
    // bytes are guarded by monotone thresholds so a warp executes at most 5 steps per token
    // whatever mix of token widths its lanes hold.
    __host__ __device__ __forceinline__ void uint32(uint32_t v) {
        const uint32_t hdr = v < 24u ? v : (v < 256u ? 0x18u : (v < 65536u ? 0x19u : 0x1au));
        step(hdr);
        if (v >= 65536u) { step(v >> 24); step((v >> 16) & 0xffu); }
        if (v >= 256u) step((v >> 8) & 0xffu);
        if (v >= 24u) step(v & 0xffu);
    }
    // CBOR head with a major type for a 64-bit argument (parent hash, array length)
    __host__ __device__ __forceinline__ void head64(uint32_t major, uint64_t v) {
        const uint32_t m = major << 5;
        if (v < 24ull) { step(m | (uint32_t)v); return; }
        int nb;
        if (v < (1ull << 8)) { step(m | 24u); nb = 1; }
        else if (v < (1ull << 16)) { step(m | 25u); nb = 2; }
        else if (v < (1ull << 32)) { step(m | 26u); nb = 4; }
        else { step(m | 27u); nb = 8; }
        for (int i = nb - 1; i >= 0; --i) step((uint32_t)(v >> (8 * i)) & 0xffu);
    }
    // 0x83 + parent: the prefix of a block payload.  A full-width parent (the overwhelmingly
    // common case: parent >= 2^32) takes the straight-line 8-byte path.
    __host__ __device__ __forceinline__ void begin_block(uint64_t parent, uint32_t block_size) {
        if (parent >> 32) {
            const uint32_t ph = (uint32_t)(parent >> 32), pl = (uint32_t)parent;
            set(kAfter83_1b);                     // offset, 0x83, 0x1b folded at compile time
            step(ph >> 24); step((ph >> 16) & 0xffu); step((ph >> 8) & 0xffu); step(ph & 0xffu);
            step(pl >> 24); step((pl >> 16) & 0xffu); step((pl >> 8) & 0xffu); step(pl & 0xffu);
        } else {
            set(kAfter83);
            head64(0, parent);
        }
        if (block_size < 24u) step(0x80u | block_size);
        else head64(4, block_size);
    }
    __host__ __device__ __forceinline__ uint64_t end_block() { step(0xf6u); return get(); }
};

// murmur3 finaliser: spreads FNV output (and the model id) over the slot index bits.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}
__host__ __device__ __forceinline__ uint64_t home_of(uint64_t hash, uint32_t model) {
    return mix64(hash ^ ((uint64_t)model * 0x9E3779B97F4A7C15ull));
}

}  // namespace kvx
