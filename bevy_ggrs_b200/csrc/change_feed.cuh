// Change feed (bgr_feed_*): report to the host only the live rows whose existence, presence or tracked field bytes
// changed since the feed's last report (see include/bevy_ggrs_b200.h "change feed").
//
// Per feed the device keeps the REPORTED state of every row, tile-planar like the images (kernels.cuh): per 512-row tile
// one plane of 512 u32 per tracked field word, then one byte per row, the row's reported mask byte: the image's mask
// byte reduced to the bits the record's state is made of (alive and the absent bits of the tracked columns), 0 for a row
// that did not exist.  Field words of a field that was not present are stored as zero.  A report is four launches:
//   pass 1 (k_feed_count, engine stream): one 512-thread block per tile, one row per thread, reads the tracked word
//          planes and the mask byte of image 0 and the reported state (coalesced: a warp reads 128 B per plane).  A row
//          differs when its reduced mask byte or any tracked word (zero where not present) differs.  Warp ballots, one
//          count per tile, no atomics.
//   scan   (k_feed_scan, one block): exclusive scan of the tile counts in tile order, the cap applied, and the ascending
//          list of tiles that hold one of the first `cap` records; writes n_records / pending.
//   pass 2 (k_feed_records): only the listed tiles; a block-level exclusive scan of the per-row flags gives each row its
//          record index, so records land in ascending row order whatever the scheduling.  Rows with an index < cap write
//          their record into the staging buffer and become the reported state.
//   copy   (k_feed_copy, copy stream, behind an event after pass 2): moves n_records records from device memory into
//          page-locked host memory, so PCIe carries n_records * record_bytes; the 16-byte info follows by cudaMemcpyAsync.
#pragma once
#include "kernels.cuh"

namespace bgr {

constexpr uint32_t kFeedMaxFields = 8;   // == BGR_MAX_FEED_FIELDS
constexpr uint32_t kFeedBlock = kTileRows;  // one thread per row of a tile
constexpr uint32_t kFeedScanBlock = 1024;

struct FeedField { uint32_t plane, words, absent, rep_plane; };  // image word plane, words, absent bit (0: not optional), reported plane

struct FeedParams {
    const uint8_t* img;          // image 0
    uint8_t* rep;                // reported state, tile-planar with `rep_words` planes
    uint32_t words, rep_words, n_fields, keep;  // keep: mask bits the state is made of
    uint32_t rows;               // RollbackOrdered::len() of image 0
    uint32_t n_tiles, cap;       // tiles compared; records that may be written
    uint32_t record_words;       // 2 + rep_words
    FeedField fields[kFeedMaxFields];
    unsigned int* tile_count;    // [n_tiles] pass 1 output
    unsigned int* tile_off;      // [n_tiles] first record index of each tile
    unsigned int* tile_list;     // [n_tiles] tiles holding a record below cap, ascending
    unsigned int* info;          // [0] n_records [1] pending [2] rows [3] record_bytes [4] listed tiles
    uint32_t* out;               // [cap][record_words] staging
};

// the reduced mask byte of `row` in image 0: 0 unless the row exists
__device__ __forceinline__ uint32_t feed_cur_mask(const FeedParams& p, const uint8_t* tile, uint32_t row) {
    const uint32_t m = row < p.rows ? uint32_t(tile[size_t(p.words) * kPlaneBytes + row % kTileRows]) : 0u;
    return (m & 1u) ? (m & p.keep) : 0u;
}
__device__ __forceinline__ bool feed_present(uint32_t m, uint32_t absent) { return (m & 1u) && !(m & absent); }

// current and reported (mask, words) of one row; calls on_word(k, w, rep_plane, cur) for every tracked word and
// returns whether the row differs
template <class OnWord>
__device__ __forceinline__ bool feed_row(const FeedParams& p, uint32_t tile, uint32_t row, uint32_t cm, uint32_t rm,
                                         OnWord&& on_word) {
    const uint8_t* it = p.img + size_t(tile) * tile_bytes_of(p.words);
    const uint8_t* rt = p.rep + size_t(tile) * tile_bytes_of(p.rep_words);
    const size_t lane_off = size_t(row % kTileRows) * 4u;
    bool diff = cm != rm;
    for (uint32_t k = 0; k < p.n_fields; ++k) {
        const FeedField f = p.fields[k];
        const bool pc = feed_present(cm, f.absent), pr = feed_present(rm, f.absent);
        for (uint32_t w = 0; w < f.words; ++w) {
            const uint32_t c = pc ? *reinterpret_cast<const uint32_t*>(it + size_t(f.plane + w) * kPlaneBytes + lane_off) : 0u;
            if (!diff) {
                const uint32_t r = pr ? *reinterpret_cast<const uint32_t*>(rt + size_t(f.rep_plane + w) * kPlaneBytes + lane_off) : 0u;
                diff = c != r;
            }
            on_word(k, w, f.rep_plane + w, c);
        }
    }
    return diff;
}

__global__ void __launch_bounds__(kFeedBlock) k_feed_count(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedBlock / 32u];
    const uint32_t tile = blockIdx.x, row = tile * kTileRows + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint8_t* it = p.img + size_t(tile) * tile_bytes_of(p.words);
    const uint32_t cm = feed_cur_mask(p, it, row);
    const uint32_t rm = p.rep[size_t(tile) * tile_bytes_of(p.rep_words) + size_t(p.rep_words) * kPlaneBytes + threadIdx.x];
    const bool diff = feed_row(p, tile, row, cm, rm, [](uint32_t, uint32_t, uint32_t, uint32_t) {});
    const uint32_t n = __popc(__ballot_sync(0xffffffffu, diff));
    if (lane == 0) s_warp[warp] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (uint32_t k = 0; k < kFeedBlock / 32u; ++k) t += s_warp[k];
        p.tile_count[tile] = t;
    }
}

// exclusive scan of one value per thread over a 1024-thread block; returns the exclusive prefix, *total the sum
__device__ __forceinline__ uint32_t feed_block_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t incl = v;
    for (uint32_t o = 1; o < 32u; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    __syncthreads();  // s_warp of the previous call has been read
    if (lane == 31u) s_warp[warp] = incl;
    __syncthreads();
    uint32_t base = 0, sum = 0;
    for (uint32_t k = 0; k < kFeedScanBlock / 32u; ++k) {
        const uint32_t x = s_warp[k];
        base += k < warp ? x : 0u;
        sum += x;
    }
    *total = sum;
    return base + incl - v;
}

__global__ void __launch_bounds__(kFeedScanBlock) k_feed_scan(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedScanBlock / 32u];
    uint32_t carry = 0, listed = 0;
    for (uint32_t base = 0; base < p.n_tiles; base += kFeedScanBlock) {  // uniform trip count
        const uint32_t t = base + threadIdx.x;
        const uint32_t v = t < p.n_tiles ? p.tile_count[t] : 0u;
        uint32_t sum, lsum;
        const uint32_t off = carry + feed_block_scan(v, s_warp, &sum);
        const uint32_t in_list = (v != 0u && off < p.cap) ? 1u : 0u;
        const uint32_t pos = listed + feed_block_scan(in_list, s_warp, &lsum);
        if (t < p.n_tiles) p.tile_off[t] = off;
        if (in_list) p.tile_list[pos] = t;
        carry += sum;
        listed += lsum;
    }
    if (threadIdx.x == 0) {
        const uint32_t n = carry < p.cap ? carry : p.cap;
        p.info[0] = n;
        p.info[1] = carry - n;
        p.info[2] = p.rows;
        p.info[3] = 4u * p.record_words;
        p.info[4] = listed;
    }
}

__global__ void __launch_bounds__(kFeedBlock) k_feed_records(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedBlock / 32u];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t n_list = p.info[4];
    for (uint32_t i = blockIdx.x; i < n_list; i += gridDim.x) {
        const uint32_t tile = p.tile_list[i], row = tile * kTileRows + threadIdx.x;
        const uint8_t* it = p.img + size_t(tile) * tile_bytes_of(p.words);
        uint8_t* rt = p.rep + size_t(tile) * tile_bytes_of(p.rep_words);
        const uint32_t cm = feed_cur_mask(p, it, row);
        const uint32_t rm = rt[size_t(p.rep_words) * kPlaneBytes + threadIdx.x];
        const bool diff = feed_row(p, tile, row, cm, rm, [](uint32_t, uint32_t, uint32_t, uint32_t) {});
        const unsigned bal = __ballot_sync(0xffffffffu, diff);
        __syncthreads();  // s_warp of the previous tile has been read
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        uint32_t pos = p.tile_off[tile] + __popc(bal & ((1u << lane) - 1u));
        for (uint32_t k = 0; k < warp; ++k) pos += s_warp[k];
        if (!diff || pos >= p.cap) continue;  // no collective follows in this iteration
        uint32_t state = cm ? 1u : 0u;
        for (uint32_t k = 0; k < p.n_fields; ++k)
            if (feed_present(cm, p.fields[k].absent)) state |= 2u << k;
        uint32_t* rec = p.out + size_t(pos) * p.record_words;
        rec[0] = row;
        rec[1] = state;
        uint32_t at = 2;
        const size_t lane_off = size_t(threadIdx.x) * 4u;
        feed_row(p, tile, row, cm, cm, [&](uint32_t, uint32_t, uint32_t rp, uint32_t c) {
            rec[at++] = c;
            *reinterpret_cast<uint32_t*>(rt + size_t(rp) * kPlaneBytes + lane_off) = c;
        });
        rt[size_t(p.rep_words) * kPlaneBytes + threadIdx.x] = uint8_t(cm);
    }
}

// staging -> page-locked host memory: n_records * record_words words
__global__ void __launch_bounds__(256) k_feed_copy(const uint32_t* __restrict__ stage, const unsigned int* __restrict__ info,
                                                   uint32_t* host_records) {
    const size_t n = size_t(info[0]) * (info[3] / 4u);
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x)
        host_records[t] = stage[t];
}

}  // namespace bgr
