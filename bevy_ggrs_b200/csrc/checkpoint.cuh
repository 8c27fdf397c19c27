// World checkpoints (bgr_checkpoint_save / bgr_checkpoint_restore): a frame image encoded per 512-row tile and per
// vector (each word plane, then the mask plane read as 128 u32) as CONST, SPARSE or RAW, see include/bevy_ggrs_b200.h
// "world checkpoints".
//
// Save is three launches over the source slot, one 512-thread block per tile and one row per thread:
//   measure (k_ckpt_measure): reads every plane of the tile once, coalesced, canonicalises in registers (words of rows
//            that do not exist or lack the column are zero, the mask byte of a row that does not exist is zero), and
//            decides each vector's kind with block votes: __syncthreads_and against element 0 broadcast through shared
//            memory, __syncthreads_count for the non-zero elements.  Writes the kinds and the block's byte length.
//   scan     (k_ckpt_scan, one block): the lengths become the u64 offsets and the total; no ordering depends on atomics.
//   pack     (k_ckpt_pack): re-reads the tile and writes the kind bytes and the bodies at the block's offset: CONST by
//            one thread, the SPARSE bitmap from warp ballots with each non-zero element ranked by a popc prefix plus the
//            warp totals in shared memory, RAW coalesced.
// Restore is one launch (k_ckpt_unpack) per uploaded blob: warp 0 validates the kind bytes, the padding and the length
// the kinds and bitmaps imply against the block's offsets, reading a bitmap only after checking it lies inside the
// block; then the mask plane is expanded and an existing row whose mask byte has a bit outside the alive bit and the
// registered absent bits makes the block bad.  A bad block sets the error word and writes nothing.  Otherwise every
// thread expands its row of every vector into a scratch image, canonical as above.
#pragma once
#include "desync_diff.cuh"

namespace bgr {

constexpr uint32_t kCkptConst = BGR_CKPT_CONST, kCkptSparse = BGR_CKPT_SPARSE, kCkptRaw = BGR_CKPT_RAW;
constexpr uint32_t kCkptScanBlock = 1024;
constexpr uint32_t kCkptMaskWords = kTileRows / 4u;  // the mask plane as u32

// u32 words of a block's kind bytes (one per vector, zero-padded to a multiple of 4)
__host__ __device__ inline uint32_t ckpt_kind_words(uint32_t words) { return (words + 1u + 3u) / 4u; }
// elements of vector v: a word plane, or the mask plane
__host__ __device__ inline uint32_t ckpt_elems(uint32_t v, uint32_t words) { return v < words ? kTileRows : kCkptMaskWords; }
__host__ __device__ inline uint32_t ckpt_kind(bool all_equal, uint32_t n, uint32_t nnz) {
    return all_equal ? kCkptConst : nnz < n - n / 32u ? kCkptSparse : kCkptRaw;
}
__host__ __device__ inline uint32_t ckpt_body_words(uint32_t kind, uint32_t n, uint32_t nnz) {
    return kind == kCkptConst ? 1u : kind == kCkptSparse ? n / 32u + nnz : n;
}
// the largest block: every vector RAW
__host__ __device__ inline uint32_t ckpt_max_block_words(uint32_t words) {
    return ckpt_kind_words(words) + words * kTileRows + kCkptMaskWords;
}

struct CkptParams {
    const uint8_t* img;                  // save: the source slot's image; restore: the scratch image written
    uint32_t words, rows;
    const uint32_t* plane_absent;        // [words] the absent bit of the column each plane belongs to (0: not optional)
    const uint32_t* plane_pad;           // restore: [words] the bits of a plane's word past its column's element bytes
    uint32_t mask_bits;                  // restore: the bits a mask byte may hold (alive and the registered absent bits)
    uint8_t* kinds;                      // save: [tiles][words + 1]
    unsigned int* lens;                  // save: [tiles] bytes of each block
    const unsigned long long* offsets;   // [tiles + 1]
    uint32_t* payload;
    unsigned int* err;                   // restore: lowest bad block (0xFFFFFFFF: none)
};

// thread threadIdx.x's canonical word of plane `plane` (m: its canonical mask byte)
__device__ __forceinline__ uint32_t ckpt_word(const uint8_t* tile, uint32_t plane, uint32_t m, uint32_t absent) {
    return (m && !(m & absent)) ? __ldcs(reinterpret_cast<const uint32_t*>(tile + size_t(plane) * kPlaneBytes + threadIdx.x * 4u))
                                : 0u;
}

// Vector v of the tile for this thread: a canonical word, or the mask plane's u32 (s_mask holds the canonical bytes).
__device__ __forceinline__ uint32_t ckpt_value(const CkptParams& p, const uint8_t* tile, uint32_t v, uint32_t m,
                                               const uint32_t* s_mask) {
    if (v < p.words) return ckpt_word(tile, v, m, p.plane_absent[v]);
    return threadIdx.x < kCkptMaskWords ? s_mask[threadIdx.x] : 0u;
}

__global__ void __launch_bounds__(kTileRows) k_ckpt_measure(const __grid_constant__ CkptParams p) {
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_first;
    const uint32_t tile = blockIdx.x;
    const uint8_t* tb = p.img + size_t(tile) * tile_bytes_of(p.words);
    const uint32_t m = diff_mask_tile(tb, p.words, tile * kTileRows + threadIdx.x, p.rows);
    reinterpret_cast<uint8_t*>(s_mask)[threadIdx.x] = uint8_t(m);
    uint32_t len = ckpt_kind_words(p.words);  // thread 0's
    for (uint32_t v = 0; v <= p.words; ++v) {
        const uint32_t n = ckpt_elems(v, p.words);
        const bool in = threadIdx.x < n;
        __syncthreads();  // s_mask is complete; s_first of the previous vector has been read
        const uint32_t x = ckpt_value(p, tb, v, m, s_mask);
        if (threadIdx.x == 0) s_first = x;
        __syncthreads();
        const bool eq = __syncthreads_and(!in || x == s_first);
        const uint32_t nnz = __syncthreads_count(in && x != 0u);
        if (threadIdx.x == 0) {
            const uint32_t kind = ckpt_kind(eq, n, nnz);
            p.kinds[size_t(tile) * (p.words + 1u) + v] = uint8_t(kind);
            len += ckpt_body_words(kind, n, nnz);
        }
    }
    if (threadIdx.x == 0) p.lens[tile] = len * 4u;
}

// offsets[i] = sum of lens[0 .. i), offsets[n_tiles] = the total, in u64
__global__ void __launch_bounds__(kCkptScanBlock) k_ckpt_scan(const unsigned int* __restrict__ lens, uint32_t n_tiles,
                                                              unsigned long long* __restrict__ offsets) {
    __shared__ unsigned long long s_warp[kCkptScanBlock / 32u];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned long long carry = 0;
    for (uint32_t base = 0; base < n_tiles; base += kCkptScanBlock) {  // uniform trip count
        const uint32_t i = base + threadIdx.x;
        const unsigned long long v = i < n_tiles ? lens[i] : 0ull;
        unsigned long long incl = v;
        for (uint32_t o = 1; o < 32u; o <<= 1) {
            const unsigned long long u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        __syncthreads();  // s_warp of the previous chunk has been read
        if (lane == 31u) s_warp[warp] = incl;
        __syncthreads();
        unsigned long long before = 0, sum = 0;
        for (uint32_t k = 0; k < kCkptScanBlock / 32u; ++k) {
            const unsigned long long x = s_warp[k];
            before += k < warp ? x : 0ull;
            sum += x;
        }
        if (i < n_tiles) offsets[i] = carry + before + incl - v;
        carry += sum;
    }
    if (threadIdx.x == 0) offsets[n_tiles] = carry;
}

__global__ void __launch_bounds__(kTileRows) k_ckpt_pack(const __grid_constant__ CkptParams p) {
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_warp[kTileRows / 32u];
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint8_t* tb = p.img + size_t(tile) * tile_bytes_of(p.words);
    const uint32_t m = diff_mask_tile(tb, p.words, tile * kTileRows + threadIdx.x, p.rows);
    reinterpret_cast<uint8_t*>(s_mask)[threadIdx.x] = uint8_t(m);
    const uint8_t* kinds = p.kinds + size_t(tile) * (p.words + 1u);
    uint32_t* out = p.payload + p.offsets[tile] / 4u;
    const uint32_t kw = ckpt_kind_words(p.words);
    for (uint32_t i = threadIdx.x; i < kw; i += blockDim.x) {
        uint32_t k = 0;
        for (uint32_t b = 0; b < 4u; ++b)
            if (4u * i + b <= p.words) k |= uint32_t(kinds[4u * i + b]) << (8u * b);
        out[i] = k;
    }
    uint32_t pos = kw;
    for (uint32_t v = 0; v <= p.words; ++v) {
        const uint32_t n = ckpt_elems(v, p.words), kind = kinds[v];
        const bool in = threadIdx.x < n;
        __syncthreads();  // s_mask is complete; s_warp of the previous vector has been read
        const uint32_t x = ckpt_value(p, tb, v, m, s_mask);
        if (kind == kCkptConst) {
            if (threadIdx.x == 0) out[pos] = x;
            pos += 1u;
        } else if (kind == kCkptRaw) {
            if (in) out[pos + threadIdx.x] = x;
            pos += n;
        } else {  // kind is uniform over the block: the barrier below is reached by every thread
            const bool nz = in && x != 0u;
            const unsigned bal = __ballot_sync(0xffffffffu, nz);
            if (lane == 0) {
                if (warp < n / 32u) out[pos + warp] = bal;
                s_warp[warp] = __popc(bal);
            }
            __syncthreads();
            uint32_t before = 0, nnz = 0;
            for (uint32_t k = 0; k < kTileRows / 32u; ++k) {
                const uint32_t c = s_warp[k];
                before += k < warp ? c : 0u;
                nnz += c;
            }
            if (nz) out[pos + n / 32u + before + __popc(bal & ((1u << lane) - 1u))] = x;
            pos += n / 32u + nnz;
        }
    }
}

// dynamic shared memory: (words + 1) u32, the first body word of each vector
__global__ void __launch_bounds__(kTileRows) k_ckpt_unpack(const __grid_constant__ CkptParams p) {
    extern __shared__ uint32_t s_start[];
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_bad;
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u;
    const unsigned long long o0 = p.offsets[tile];
    // the host checked: offsets ascend in multiples of 4 inside the upload, and a block is at most ckpt_max_block_words
    const uint32_t len = uint32_t((p.offsets[tile + 1] - o0) / 4u);
    const uint32_t* blk = p.payload + o0 / 4u;
    const uint32_t kw = ckpt_kind_words(p.words), nv = p.words + 1u;
    auto kind_of = [blk](uint32_t v) { return (blk[v / 4u] >> (8u * (v % 4u))) & 0xFFu; };
    if (threadIdx.x < 32u) {  // warp 0: every value below is uniform over the warp
        bool bad = len < kw;
        uint32_t pos = kw;
        for (uint32_t v = 0; v < nv && !bad; ++v) {
            const uint32_t kind = kind_of(v), n = ckpt_elems(v, p.words);
            if (lane == 0) s_start[v] = pos;
            if (kind > kCkptRaw) { bad = true; break; }
            uint32_t nnz = 0;
            if (kind == kCkptSparse) {
                if (pos + n / 32u > len) { bad = true; break; }  // the bitmap would lie outside the block
                nnz = __reduce_add_sync(0xffffffffu, lane < n / 32u ? uint32_t(__popc(blk[pos + lane])) : 0u);
            }
            pos += ckpt_body_words(kind, n, nnz);
            bad = pos > len;
        }
        for (uint32_t b = nv; b < 4u * kw && !bad; ++b) bad = kind_of(b) != 0u;  // padding
        bad = bad || pos != len;
        if (lane == 0) s_bad = bad ? 1u : 0u;
    }
    __syncthreads();
    if (s_bad) {
        if (threadIdx.x == 0) atomicMin(p.err, tile);
        return;
    }
    // this thread's element of vector v (zero past the vector's n)
    auto element = [&](uint32_t v) -> uint32_t {
        const uint32_t n = ckpt_elems(v, p.words), kind = kind_of(v), start = s_start[v];
        if (threadIdx.x >= n) return 0u;
        if (kind == kCkptConst) return blk[start];
        if (kind == kCkptRaw) return blk[start + threadIdx.x];
        const uint32_t j = threadIdx.x / 32u, bm = blk[start + j];
        if (!((bm >> lane) & 1u)) return 0u;
        uint32_t rank = __popc(bm & ((1u << lane) - 1u));
        for (uint32_t k = 0; k < j; ++k) rank += __popc(blk[start + k]);
        return blk[start + n / 32u + rank];
    };
    uint8_t* tb = const_cast<uint8_t*>(p.img) + size_t(tile) * tile_bytes_of(p.words);
    const uint32_t mw = element(p.words);
    if (threadIdx.x < kCkptMaskWords) s_mask[threadIdx.x] = mw;
    __syncthreads();
    const uint32_t mb = reinterpret_cast<const uint8_t*>(s_mask)[threadIdx.x];
    const uint32_t m = (tile * kTileRows + threadIdx.x < p.rows && (mb & 1u)) ? mb : 0u;
    if (__syncthreads_or(m & ~p.mask_bits)) {  // a presence bit of a column this registration does not have
        if (threadIdx.x == 0) atomicMin(p.err, tile);
        return;
    }
    tb[size_t(p.words) * kPlaneBytes + threadIdx.x] = uint8_t(m);
    uint32_t stray = 0;   // bits past a sub-word element's end: no digest covers them, so they are refused here
    for (uint32_t v = 0; v < p.words; ++v) {
        const uint32_t x = (m && !(m & p.plane_absent[v])) ? element(v) : 0u;
        stray |= x & p.plane_pad[v];
        *reinterpret_cast<uint32_t*>(tb + size_t(v) * kPlaneBytes + threadIdx.x * 4u) = x;
    }
    if (__syncthreads_or(stray != 0u) && threadIdx.x == 0) atomicMin(p.err, tile);
}

}  // namespace bgr
