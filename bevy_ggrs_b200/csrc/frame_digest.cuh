// Frame digest (bgr_frame_digest, P2P desync reports): per block of BGR_DIGEST_BLOCK_ROWS = 512 rows (one tile) of a
// stored frame image, one u64 per registered column and one for existence / presence (see include/bevy_ggrs_b200.h
// "P2P desync reports").  Two peers exchange these words to find the few blocks whose images differ.
//
// One 512-thread block per tile of every image of an image table, one row per thread.  Every word plane of the tile is read from HBM once, coalesced (a
// warp reads 128 contiguous bytes per plane; lanes whose row does not hold the column issue no load), streaming
// (__ldcs).  The element hash is sea_hash_stream's, fed byte by byte.
// Each thread's per-column hash is XOR-reduced over the warp (__reduce_xor_sync on both 32-bit halves), then over the
// 16 warps through shared memory: one store per block and word, no atomics, so the words do not depend on the
// scheduling.  The block's alive-row count is stored the same way (the header's `active`).
#pragma once
#include "desync_diff.cuh"

namespace bgr {

static_assert(BGR_DIGEST_BLOCK_ROWS == kTileRows, "a digest block is one tile");

// one registered column: its word planes, its element size (the bytes hashed) and its absent bit (0: not optional)
struct DigestColumn { uint32_t first_plane, elem_bytes, absent; };

// An image table: the images one launch of k_frame_digest, k_ckpt_measure, k_ckpt_pack, k_ckpt_unpack or k_ckpt_commit
// covers, of one registration.  Their blocks are numbered in table order: image i holds blocks
// [first_block, first_block + ceil(rows / 512)).
struct ImageEntry {
    const uint8_t* img;
    unsigned long long order_base;  // bgr_config.order_base of the image's engine
    unsigned long long out_off;     // byte offset of the image's payload in k_ckpt_pack's output or k_ckpt_unpack's upload
    uint32_t rows, first_block;
};
static_assert(sizeof(ImageEntry) == 32, "ImageEntry layout");

// the entry of global block `b` (first_block ascends; n >= 1)
__device__ __forceinline__ const ImageEntry& image_of(const ImageEntry* t, uint32_t n, uint32_t b) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) / 2u;
        if (t[mid].first_block <= b) lo = mid;
        else hi = mid;
    }
    return t[lo];
}

struct DigestParams {
    const ImageEntry* images;
    uint32_t n_images, words, n_cols;
    const DigestColumn* cols;   // [n_cols]
    unsigned long long* out;    // [blocks][n_cols + 1]
    unsigned int* active;       // [blocks] alive rows of each block
};

__device__ __forceinline__ uint64_t warp_xor_u64(uint64_t v) {
    const uint32_t lo = __reduce_xor_sync(0xffffffffu, uint32_t(v));
    const uint32_t hi = __reduce_xor_sync(0xffffffffu, uint32_t(v >> 32));
    return uint64_t(lo) | (uint64_t(hi) << 32);
}

// dynamic shared memory: (kTileRows / 32) warps x (n_cols + 1) u64
__global__ void __launch_bounds__(kTileRows) k_frame_digest(const __grid_constant__ DigestParams p) {
    extern __shared__ unsigned long long s_part[];
    __shared__ uint32_t s_warp[kTileRows / 32u];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const ImageEntry& im = image_of(p.images, p.n_images, blockIdx.x);
    const uint32_t t = blockIdx.x - im.first_block;
    const uint8_t* tile = im.img + size_t(t) * tile_bytes_of(p.words);
    const uint32_t row = t * kTileRows + threadIdx.x;
    const uint32_t m = diff_mask_tile(tile, p.words, row, im.rows);
    const uint64_t order = im.order_base + row;
    for (uint32_t c = 0; c < p.n_cols; ++c) {
        const DigestColumn col = p.cols[c];
        uint64_t h = 0;
        if (m && !(m & col.absent)) {
            // byte i of the element is byte i % 4 of word plane first_plane + i / 4 (the repeated loads of a word hit L1)
            const uint8_t* base = tile + size_t(col.first_plane) * kPlaneBytes + size_t(threadIdx.x) * 4u;
            auto byte_at = [base](uint32_t i) -> uint8_t {
                return uint8_t(__ldcs(reinterpret_cast<const uint32_t*>(base + size_t(i >> 2) * kPlaneBytes)) >> (8u * (i & 3u)));
            };
            h = sea_hash_2xu64(order, sea_hash_stream(col.elem_bytes, byte_at));
        }
        h = warp_xor_u64(h);
        if (lane == 0) s_part[warp * (p.n_cols + 1u) + c] = h;
    }
    uint64_t hm = m ? sea_hash_2xu64(order, uint64_t(m & 0xFFu)) : 0ull;
    hm = warp_xor_u64(hm);
    if (lane == 0) s_part[warp * (p.n_cols + 1u) + p.n_cols] = hm;
    const uint32_t alive = block_sum_512(m ? 1u : 0u, s_warp);  // synchronises the block: s_part is complete
    for (uint32_t w = threadIdx.x; w <= p.n_cols; w += blockDim.x) {
        uint64_t x = 0;
        for (uint32_t k = 0; k < kTileRows / 32u; ++k) x ^= s_part[k * (p.n_cols + 1u) + w];
        p.out[size_t(blockIdx.x) * (p.n_cols + 1u) + w] = x;
    }
    if (threadIdx.x == 0) p.active[blockIdx.x] = alive;
}

}  // namespace bgr
