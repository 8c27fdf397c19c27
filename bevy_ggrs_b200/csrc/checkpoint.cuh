// World checkpoints (bgr_checkpoint_save / bgr_checkpoint_restore): a frame image encoded per 512-row tile and per
// vector (each word plane, then the mask plane read as 128 u32) as CONST, SPARSE or RAW, see include/bevy_ggrs_b200.h
// "world checkpoints".
//
// Save is three launches over an image table (frame_digest.cuh ImageEntry: one image for bgr_checkpoint_save, every
// keyframe of a launch for bgr_replay_keyframes), one 512-thread block per tile of every image and one row per thread:
//   measure (k_ckpt_measure): reads every plane of the tile once, coalesced, canonicalises in registers (words of rows
//            that do not exist or lack the column are zero, the mask byte of a row that does not exist is zero), and
//            decides each vector's kind with block votes: __syncthreads_and against element 0 broadcast through shared
//            memory, __syncthreads_count for the non-zero elements.  Writes the kinds and the block's byte length.
//   scan     (k_ckpt_scan, one block): the lengths of all blocks become the u64 offsets and the total; an image's own
//            offsets are differences from its first block's.  No ordering depends on atomics.
//   pack     (k_ckpt_pack): re-reads the tile and writes the kind bytes and the bodies at the block's offset in its
//            image's payload (ImageEntry::out_off): CONST by
//            one thread, the SPARSE bitmap from warp ballots with each non-zero element ranked by a popc prefix plus the
//            warp totals in shared memory, RAW coalesced.
// Restore decodes every uploaded blob in one launch (k_ckpt_unpack) over an image table whose entries are the blobs'
// scratch images (bgr_checkpoint_restore: one blob; bgr_batch_checkpoint_restore: one per listed world), one 512-thread
// block per tile of every blob: warp 0 validates the kind bytes, the padding and the length the kinds and bitmaps imply
// against the block's offsets, reading a bitmap only after checking it lies inside the block; then the mask plane is
// expanded and an existing row whose mask byte has a bit outside the alive bit and the registered absent bits makes the
// block bad.  A bad block sets its blob's error word and writes nothing.  Otherwise every thread expands its row of
// every vector into the scratch image, canonical as above.  Once k_frame_digest has verified every scratch image,
// k_ckpt_commit copies each to its engine's image 0 and restored ring slot, in one launch over the same table.
//
// Checkpoint deltas (bgr_checkpoint_save_delta / bgr_checkpoint_restore_delta) are instances of the same kernels:
//   k_ckpt_measure_delta / k_ckpt_pack_delta read each block's base tile and row count from the parallel per-image
//            array CkptParams::base, canonicalise both tiles in registers and code canon(target) XOR canon(base);
//   k_ckpt_unpack_delta expands each block onto the scratch image that already holds the decoded (canonical) base,
//            zero past the base's blocks, XORs, and refuses a result that is not canonical: a non-zero word of a row that
//            does not exist or lacks the column, a mask byte of a row that does not exist, a presence bit the
//            registration lacks, or bits past an element's bytes.
// The plain kernels are the <false> instances of the same bodies and compile to the code they had before.
#pragma once
#include "frame_digest.cuh"

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

// The base of one image of a delta's table: its image and row count
struct CkptBase {
    const uint8_t* img;
    uint32_t rows, reserved;
};
static_assert(sizeof(CkptBase) == 16, "CkptBase layout");

struct CkptParams {
    const ImageEntry* images;            // the image table (restore: the scratch images written)
    uint32_t n_images;
    uint32_t words;
    const uint32_t* plane_absent;        // [words] the absent bit of the column each plane belongs to (0: not optional)
    const uint32_t* plane_pad;           // restore: [words] the bits of a plane's word past its column's element bytes
    uint32_t mask_bits;                  // restore: the bits a mask byte may hold (alive and the registered absent bits)
    uint8_t* kinds;                      // save: [tiles][words + 1]
    unsigned int* lens;                  // save: [blocks] bytes of each block
    const unsigned long long* offsets;   // [blocks + 1] (restore: bytes into the concatenated payloads of every blob)
    uint32_t* payload;
    unsigned int* err;                   // restore: [n_images] each blob's lowest bad block (0xFFFFFFFF: none)
    const CkptBase* base;                // delta save: [n_images] each image's base
};

// A delta's base tile of this thread's block, and the thread's canonical base mask byte (both zero without a delta)
struct CkptBaseTile {
    const uint8_t* tb;
    uint32_t m;
};
template <bool DELTA>
__device__ __forceinline__ CkptBaseTile ckpt_base_tile(const CkptParams& p, const ImageEntry& im, uint32_t t) {
    if constexpr (DELTA) {
        const CkptBase b = p.base[&im - p.images];
        const uint8_t* tb = b.img + size_t(t) * tile_bytes_of(p.words);
        return CkptBaseTile{tb, diff_mask_tile(tb, p.words, t * kTileRows + threadIdx.x, b.rows)};
    } else {
        return CkptBaseTile{nullptr, 0u};
    }
}

// thread threadIdx.x's canonical word of plane `plane` (m: its canonical mask byte)
__device__ __forceinline__ uint32_t ckpt_word(const uint8_t* tile, uint32_t plane, uint32_t m, uint32_t absent) {
    return (m && !(m & absent)) ? __ldcs(reinterpret_cast<const uint32_t*>(tile + size_t(plane) * kPlaneBytes + threadIdx.x * 4u))
                                : 0u;
}

// Vector v of the tile for this thread: a canonical word, or the mask plane's u32 (s_mask holds the canonical bytes).
// A delta's is the XOR with the base tile's (s_mask then holds the XOR of both canonical mask bytes).
template <bool DELTA>
__device__ __forceinline__ uint32_t ckpt_value(const CkptParams& p, const uint8_t* tile, const CkptBaseTile& bt, uint32_t v,
                                               uint32_t m, const uint32_t* s_mask) {
    if (v < p.words) {
        uint32_t x = ckpt_word(tile, v, m, p.plane_absent[v]);
        if constexpr (DELTA) x ^= ckpt_word(bt.tb, v, bt.m, p.plane_absent[v]);
        return x;
    }
    return threadIdx.x < kCkptMaskWords ? s_mask[threadIdx.x] : 0u;
}

template <bool DELTA>
__device__ __forceinline__ void ckpt_measure(const CkptParams& p) {
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_first;
    const uint32_t tile = blockIdx.x;
    const ImageEntry& im = image_of(p.images, p.n_images, tile);
    const uint32_t t = tile - im.first_block;
    const uint8_t* tb = im.img + size_t(t) * tile_bytes_of(p.words);
    const uint32_t m = diff_mask_tile(tb, p.words, t * kTileRows + threadIdx.x, im.rows);
    const CkptBaseTile bt = ckpt_base_tile<DELTA>(p, im, t);
    reinterpret_cast<uint8_t*>(s_mask)[threadIdx.x] = uint8_t(m ^ bt.m);
    uint32_t len = ckpt_kind_words(p.words);  // thread 0's
    for (uint32_t v = 0; v <= p.words; ++v) {
        const uint32_t n = ckpt_elems(v, p.words);
        const bool in = threadIdx.x < n;
        __syncthreads();  // s_mask is complete; s_first of the previous vector has been read
        const uint32_t x = ckpt_value<DELTA>(p, tb, bt, v, m, s_mask);
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

__global__ void __launch_bounds__(kTileRows) k_ckpt_measure(const __grid_constant__ CkptParams p) { ckpt_measure<false>(p); }
__global__ void __launch_bounds__(kTileRows) k_ckpt_measure_delta(const __grid_constant__ CkptParams p) { ckpt_measure<true>(p); }

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

template <bool DELTA>
__device__ __forceinline__ void ckpt_pack(const CkptParams& p) {
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_warp[kTileRows / 32u];
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const ImageEntry& im = image_of(p.images, p.n_images, tile);
    const uint32_t t = tile - im.first_block;
    const uint8_t* tb = im.img + size_t(t) * tile_bytes_of(p.words);
    const uint32_t m = diff_mask_tile(tb, p.words, t * kTileRows + threadIdx.x, im.rows);
    const CkptBaseTile bt = ckpt_base_tile<DELTA>(p, im, t);
    reinterpret_cast<uint8_t*>(s_mask)[threadIdx.x] = uint8_t(m ^ bt.m);
    const uint8_t* kinds = p.kinds + size_t(tile) * (p.words + 1u);
    uint32_t* out = p.payload + (im.out_off + p.offsets[tile] - p.offsets[im.first_block]) / 4u;
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
        const uint32_t x = ckpt_value<DELTA>(p, tb, bt, v, m, s_mask);
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

__global__ void __launch_bounds__(kTileRows) k_ckpt_pack(const __grid_constant__ CkptParams p) { ckpt_pack<false>(p); }
__global__ void __launch_bounds__(kTileRows) k_ckpt_pack_delta(const __grid_constant__ CkptParams p) { ckpt_pack<true>(p); }

// dynamic shared memory: (words + 1) u32, the first body word of each vector
template <bool DELTA>
__device__ __forceinline__ void ckpt_unpack(const CkptParams& p) {
    extern __shared__ uint32_t s_start[];
    __shared__ uint32_t s_mask[kCkptMaskWords];
    __shared__ uint32_t s_bad;
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u;
    const ImageEntry& im = image_of(p.images, p.n_images, tile);
    const uint32_t t = tile - im.first_block;
    unsigned int* err = p.err + (&im - p.images);
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
        if (threadIdx.x == 0) atomicMin(err, t);
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
    uint8_t* tb = const_cast<uint8_t*>(im.img) + size_t(t) * tile_bytes_of(p.words);
    uint32_t mw = element(p.words);
    if constexpr (DELTA)  // the base's canonical mask bytes, read before any thread writes its row's
        if (threadIdx.x < kCkptMaskWords) mw ^= reinterpret_cast<const uint32_t*>(tb + size_t(p.words) * kPlaneBytes)[threadIdx.x];
    if (threadIdx.x < kCkptMaskWords) s_mask[threadIdx.x] = mw;
    __syncthreads();
    const uint32_t mb = reinterpret_cast<const uint8_t*>(s_mask)[threadIdx.x];
    const bool exists = t * kTileRows + threadIdx.x < im.rows && (mb & 1u);
    const uint32_t m = exists ? mb : 0u;
    // a presence bit of a column this registration does not have (a delta: also a mask byte of a row that does not exist)
    if (__syncthreads_or((m & ~p.mask_bits) | (DELTA && !exists ? mb : 0u))) {
        if (threadIdx.x == 0) atomicMin(err, t);
        return;
    }
    tb[size_t(p.words) * kPlaneBytes + threadIdx.x] = uint8_t(m);
    uint32_t stray = 0;   // bits past a sub-word element's end: no digest covers them, so they are refused here
    for (uint32_t v = 0; v < p.words; ++v) {
        uint32_t x;
        if constexpr (DELTA) {  // the base word XOR the delta's; a non-zero word of a row that lacks the column is refused
            x = element(v) ^ *reinterpret_cast<const uint32_t*>(tb + size_t(v) * kPlaneBytes + threadIdx.x * 4u);
            stray |= (m && !(m & p.plane_absent[v])) ? x & p.plane_pad[v] : x;
        } else {
            x = (m && !(m & p.plane_absent[v])) ? element(v) : 0u;
            stray |= x & p.plane_pad[v];
        }
        *reinterpret_cast<uint32_t*>(tb + size_t(v) * kPlaneBytes + threadIdx.x * 4u) = x;
    }
    if (__syncthreads_or(stray != 0u) && threadIdx.x == 0) atomicMin(err, t);
}

__global__ void __launch_bounds__(kTileRows) k_ckpt_unpack(const __grid_constant__ CkptParams p) { ckpt_unpack<false>(p); }
__global__ void __launch_bounds__(kTileRows) k_ckpt_unpack_delta(const __grid_constant__ CkptParams p) { ckpt_unpack<true>(p); }

// Block b copies tile b of the table's (verified) scratch images to both destinations of its image, dst[2i] and
// dst[2i + 1]: the engine's image 0 and its restored ring slot.  16-byte units (tile_bytes is a multiple of 16).
__global__ void __launch_bounds__(kTileRows) k_ckpt_commit(const ImageEntry* __restrict__ images, uint32_t n_images,
                                                           uint8_t* const* __restrict__ dst, uint32_t tile_bytes) {
    const ImageEntry& im = image_of(images, n_images, blockIdx.x);
    const size_t i = size_t(&im - images), off = size_t(blockIdx.x - im.first_block) * tile_bytes;
    const uint4* src = reinterpret_cast<const uint4*>(im.img + off);
    uint4* d0 = reinterpret_cast<uint4*>(dst[2u * i] + off);
    uint4* d1 = reinterpret_cast<uint4*>(dst[2u * i + 1u] + off);
    for (uint32_t k = threadIdx.x; k < tile_bytes / 16u; k += blockDim.x) {
        const uint4 v = __ldcs(src + k);
        d0[k] = v;
        d1[k] = v;
    }
}

}  // namespace bgr
