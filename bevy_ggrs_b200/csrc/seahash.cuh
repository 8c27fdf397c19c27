// SeaHash 4.1 arithmetic for device and host (the reference's `checksum_hasher()`,
// src/snapshot/mod.rs:315-317; call sites: component_checksum.rs:44-48,77-93,
// entity_checksum.rs:35-43, particles.rs:107-120,207-222).
//
// Pure u64 wrapping mul / shift / xor — no tensor cores, no floating point.  Only the shapes the
// hot path needs are specialised:
//   hash of one 8-byte word                       (ChecksumPart of a raw XOR result)
//   hash of 12 bytes = 3 x u32 fields             (Velocity / Transform.translation `to_bits`)
//   hash of 16 bytes = (order:u64, custom:u64)    (per-entity hash, component_checksum.rs:85-86)
//   generic byte stream                           (derive(Hash) PODs on the stepwise path)
#pragma once
#ifdef __CUDACC_RTC__
#include "rtc_prelude.cuh"
#else
#include <cstdint>
#endif

#if defined(__CUDACC__)
#define BGR_HD __host__ __device__ __forceinline__ constexpr
#else
#define BGR_HD inline constexpr
#endif

namespace bgr {

constexpr uint64_t kSeaA = 0x16f11fe89b0d677cULL;
constexpr uint64_t kSeaB = 0xb480a793d8e6c86cULL;
constexpr uint64_t kSeaC = 0x6fe2e5aaf078ebc9ULL;
constexpr uint64_t kSeaD = 0x14f994a4c5259381ULL;
constexpr uint64_t kSeaP = 0x6eed0e9da4d94a4fULL;

// x * P (mod 2^64).  The device form is three instructions of the integer multiply-add pipe: the low product, then the
// two cross products chained onto its high word as the addend.  Written as a u64 multiply, ptxas emits the low
// product and the two cross products as three independent multiplies and a fourth instruction to add their high words.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint64_t sea_mul_p(uint64_t x) {
    uint64_t r;
    asm("{\n\t.reg .u32 l, h, wl, wh;\n\t"
        "mov.b64 {l, h}, %1;\n\t"
        "mul.wide.u32 %0, l, %2;\n\t"
        "mov.b64 {wl, wh}, %0;\n\t"
        "mad.lo.u32 wh, h, %2, wh;\n\t"
        "mad.lo.u32 wh, l, %3, wh;\n\t"
        "mov.b64 %0, {wl, wh};\n\t}"
        : "=l"(r) : "l"(x), "n"(uint32_t(kSeaP)), "n"(uint32_t(kSeaP >> 32)));
    return r;
}
#else
inline constexpr uint64_t sea_mul_p(uint64_t x) { return x * kSeaP; }
#endif

// x *= P; x ^= (x >> 32) >> (x >> 60); x *= P
// (x >> 32) >> (x >> 60) only involves the high word: hi >> (hi >> 28), a 32-bit value.
BGR_HD uint64_t sea_diffuse(uint64_t x) {
    x = sea_mul_p(x);
    uint32_t hi = uint32_t(x >> 32);
    x ^= uint64_t(hi >> (hi >> 28));
    return sea_mul_p(x);
}
// the same in a constant expression (the device form above is inline PTX)
BGR_HD uint64_t sea_diffuse_const(uint64_t x) {
    x *= kSeaP;
    uint32_t hi = uint32_t(x >> 32);
    x ^= uint64_t(hi >> (hi >> 28));
    return x * kSeaP;
}

// seahash of exactly 8 bytes (one LE word)
BGR_HD uint64_t sea_hash_u64(uint64_t w) {
    uint64_t t = sea_diffuse(kSeaA ^ w);
    return sea_diffuse(kSeaB ^ kSeaC ^ kSeaD ^ t ^ 8ULL);
}

// seahash of 12 bytes: w0 = first 8 bytes (LE), tail = last 4 bytes zero-extended
BGR_HD uint64_t sea_hash_12(uint64_t w0, uint32_t tail) {
    uint64_t t = sea_diffuse(kSeaA ^ w0);            // state -> (B, C, D, t)
    uint64_t a = sea_diffuse(kSeaB ^ uint64_t(tail));  // tail goes into the new first lane
    return sea_diffuse(a ^ kSeaC ^ kSeaD ^ t ^ 12ULL);
}
// the tail lane when the last field is +0.0f (a 2-D game's z): a compile-time constant
constexpr uint64_t kSeaTailZero = sea_diffuse_const(kSeaB);
// same hash with the tail lane supplied by the caller (kSeaTailZero when the caller knows tail == 0)
BGR_HD uint64_t sea_hash_12_lane(uint64_t w0, uint64_t tail_lane) {
    uint64_t t = sea_diffuse(kSeaA ^ w0);
    return sea_diffuse(tail_lane ^ kSeaC ^ kSeaD ^ t ^ 12ULL);
}

// first lane of the per-entity hash: depends only on the RollbackOrdered index, so it is
// computed once per entity per launch and reused for every frame and every column
BGR_HD uint64_t sea_order_lane(uint64_t order) { return sea_diffuse(kSeaA ^ order); }

// seahash of 16 bytes (order, custom) given t0 = sea_order_lane(order)
BGR_HD uint64_t sea_hash_entity(uint64_t t0, uint64_t custom) {
    uint64_t t1 = sea_diffuse(kSeaB ^ custom);  // state -> (C, D, t0, t1)
    return sea_diffuse(kSeaC ^ kSeaD ^ t0 ^ t1 ^ 16ULL);
}

// seahash of 16 bytes (a, b)
BGR_HD uint64_t sea_hash_2xu64(uint64_t a, uint64_t b) { return sea_hash_entity(sea_order_lane(a), b); }

// Generic stream over `n` bytes delivered by a callable byte(i) -> uint8_t (stepwise path only).
template <class ByteAt>
#if defined(__CUDACC__)
__host__ __device__ __forceinline__
#else
inline
#endif
uint64_t sea_hash_stream(uint32_t n, ByteAt byte_at) {
    uint64_t a = kSeaA, b = kSeaB, c = kSeaC, d = kSeaD;
    uint32_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w = 0;
        for (uint32_t k = 0; k < 8; ++k) w |= uint64_t(byte_at(i + k)) << (8 * k);
        uint64_t t = sea_diffuse(a ^ w);
        a = b; b = c; c = d; d = t;
    }
    if (i < n) {
        uint64_t w = 0;
        for (uint32_t k = 0; i + k < n; ++k) w |= uint64_t(byte_at(i + k)) << (8 * k);
        a = sea_diffuse(a ^ w);
    }
    return sea_diffuse(a ^ b ^ c ^ d ^ uint64_t(n));
}

}  // namespace bgr
