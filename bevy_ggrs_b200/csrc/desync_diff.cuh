// Desync diff (BGR_CFG_DESYNC_CAPTURE): compare a frame's first-recorded image with its current ring image, row by row,
// with the keyed-map semantics of component_snapshot.rs:99-115 (see include/bevy_ggrs_b200.h "desync capture").
//
// Two passes over tile-planar images (kernels.cuh), one 512-thread block per tile, one row per thread:
//   pass 1 (k_desync_count): every word plane of both images is read once, coalesced (a warp reads 128 contiguous bytes
//           per plane and image; lanes whose row does not exist in both images issue no load).  Per-column row counts
//           and the totals are warp ballots / reductions with one global atomic per warp and counter, and only when
//           non-zero; each block writes its tile's record count.
//   host  : exclusive scan of the per-tile record counts (at most ~20k tiles at 10M rows) and the list of tiles that
//           hold one of the first `cap` records.
//   pass 2 (k_desync_records): only the listed tiles; a block-level exclusive scan of the per-row record counts gives
//           every row its output position, so records land in ascending (row, column, word) order whatever the
//           scheduling: the output is deterministic.
// Integer counts only: the result does not depend on the order the atomics land in.
//
// P2P remote diff (bgr_desync_diff_remote): `latest` is not an image but a staging buffer of tiles uploaded from a
// peer's export blob.  `visit` then lists the tiles to compare, ascending: work position i (pass 1: block i; pass 2:
// tile_list entries are positions) compares local tile visit[i] of `first` with the tile at position i of `latest`.
// Without `visit` (SyncTest capture) position i is tile i of both images, as before.
#pragma once
#include "kernels.cuh"

namespace bgr {

constexpr uint32_t kDiffBlock = kTileRows;  // one thread per row of a tile
constexpr uint32_t kDiffNone = 0xFFFFFFFFu;

// one registered column: its word planes, its absent bit (0: not optional) and the words that overlap its checksummed
// byte range [hash_off, hash_off + hash_len): word w is inside iff 4w < ck_end && 4w + 4 > ck_begin (ck_end = 0: none)
struct DiffColumn { uint32_t first_plane, words, absent, ck_begin, ck_end; };
struct DiffRecord { uint32_t row, column, word, first, latest; };  // == bgr_desync_record

struct DiffParams {
    const uint8_t* first;
    const uint8_t* latest;
    uint32_t words, n_cols, rows_first, rows_latest;
    const DiffColumn* cols;          // [n_cols]
    unsigned int* col_counts;        // [n_cols][3]: rows with a word difference, ... inside the checksum, presence differences
    unsigned long long* totals;      // [0] rows with any difference, [1] existence differences, [2] differing words
    unsigned int* tile_records;      // [tiles] records of each tile (pass 1 output)
    const unsigned int* tile_list;   // pass 2: [n_list] work position, [n_list + i] its first record's output index
    uint32_t n_list, cap;
    DiffRecord* out;                 // [cap]
    const unsigned int* visit;       // optional: [positions] local tile of each work position (remote diff)
};

// the local tile and the two tile bases of work position `pos`
struct DiffTiles { uint32_t tile; const uint8_t* first; const uint8_t* latest; };
__device__ __forceinline__ DiffTiles diff_tiles(const DiffParams& p, uint32_t pos) {
    const uint32_t tile = p.visit ? p.visit[pos] : pos;
    const size_t tb = tile_bytes_of(p.words);
    return DiffTiles{tile, p.first + size_t(tile) * tb, p.latest + size_t(p.visit ? pos : tile) * tb};
}

// the mask byte of row `row` (tile-local index row % kTileRows) from the base of its tile: 0 unless the row exists
// there (stale bytes past the image's row count are not data)
__device__ __forceinline__ uint32_t diff_mask_tile(const uint8_t* tile, uint32_t words, uint32_t row, uint32_t n_rows) {
    const uint32_t m = row < n_rows ? uint32_t(tile[size_t(words) * kPlaneBytes + row % kTileRows]) : 0u;
    return (m & 1u) ? m : 0u;
}
__device__ __forceinline__ uint32_t diff_mask(const uint8_t* img, uint32_t words, uint32_t row, uint32_t n_rows) {
    return diff_mask_tile(img + size_t(row / kTileRows) * tile_bytes_of(words), words, row, n_rows);
}

// Walks the records of one row in (column, word) order.  Every lane of a warp runs the same loop trip counts (the
// column / word loops do not depend on the row), so callers may use warp collectives inside `per_column`.
//   on_record(column, word, first, latest)             for every record of the row
//   per_column(column, word_diff, ck_diff, presence)   after each column (not called for existence-only rows' columns
//                                                      with any flag set: all false there)
template <class OnRecord, class PerColumn>
__device__ __forceinline__ void diff_row(const DiffParams& p, const DiffTiles& t, uint32_t row, OnRecord&& on_record,
                                         PerColumn&& per_column) {
    const uint32_t mf = diff_mask_tile(t.first, p.words, row, p.rows_first);
    const uint32_t ml = diff_mask_tile(t.latest, p.words, row, p.rows_latest);
    const bool both = mf && ml;
    if ((mf != 0u) != (ml != 0u)) on_record(kDiffNone, kDiffNone, mf, ml);
    for (uint32_t c = 0; c < p.n_cols; ++c) {
        const DiffColumn col = p.cols[c];
        const bool pf = both && !(mf & col.absent), pl = both && !(ml & col.absent);
        const bool presence = both && pf != pl;
        if (presence) on_record(c, kDiffNone, mf, ml);
        bool word_diff = false, ck_diff = false;
        const size_t base = size_t(row % kTileRows) * 4u;
        for (uint32_t w = 0; w < col.words; ++w) {
            if (pf && pl) {
                const size_t off = base + size_t(col.first_plane + w) * kPlaneBytes;
                const uint32_t a = __ldcs(reinterpret_cast<const uint32_t*>(t.first + off));
                const uint32_t b = __ldcs(reinterpret_cast<const uint32_t*>(t.latest + off));
                if (a != b) {
                    on_record(c, w, a, b);
                    word_diff = true;
                    ck_diff = ck_diff || (4u * w < col.ck_end && 4u * w + 4u > col.ck_begin);
                }
            }
        }
        per_column(c, word_diff, ck_diff, presence);
    }
}

__device__ __forceinline__ uint32_t block_sum_512(uint32_t v, uint32_t* s_warp) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    v = __reduce_add_sync(0xffffffffu, v);
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    uint32_t t = 0;
    for (uint32_t k = 0; k < kDiffBlock / 32u; ++k) t += s_warp[k];
    return t;
}

__global__ void __launch_bounds__(kDiffBlock) k_desync_count(const __grid_constant__ DiffParams p) {
    __shared__ uint32_t s_warp[kDiffBlock / 32u];
    const unsigned full = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31u;
    const DiffTiles t = diff_tiles(p, blockIdx.x);
    const uint32_t row = t.tile * kTileRows + threadIdx.x;
    uint32_t n_rec = 0, n_words = 0;
    bool existence = false;
    diff_row(p, t, row,
             [&](uint32_t c, uint32_t w, uint32_t, uint32_t) {
                 ++n_rec;
                 if (w != kDiffNone) ++n_words;
                 if (c == kDiffNone) existence = true;
             },
             [&](uint32_t c, bool word_diff, bool ck_diff, bool presence) {
                 const uint32_t a = __popc(__ballot_sync(full, word_diff));
                 const uint32_t b = __popc(__ballot_sync(full, ck_diff));
                 const uint32_t d = __popc(__ballot_sync(full, presence));
                 if (lane == 0) {
                     if (a) atomicAdd(&p.col_counts[3 * c + 0], a);
                     if (b) atomicAdd(&p.col_counts[3 * c + 1], b);
                     if (d) atomicAdd(&p.col_counts[3 * c + 2], d);
                 }
             });
    const uint32_t rows_any = __popc(__ballot_sync(full, n_rec != 0));
    const uint32_t rows_ex = __popc(__ballot_sync(full, existence));
    const uint32_t words_w = __reduce_add_sync(full, n_words);
    if (lane == 0) {
        if (rows_any) atomicAdd(&p.totals[0], (unsigned long long)rows_any);
        if (rows_ex) atomicAdd(&p.totals[1], (unsigned long long)rows_ex);
        if (words_w) atomicAdd(&p.totals[2], (unsigned long long)words_w);
    }
    const uint32_t tile_total = block_sum_512(n_rec, s_warp);
    if (threadIdx.x == 0) p.tile_records[blockIdx.x] = tile_total;
}

__global__ void __launch_bounds__(kDiffBlock) k_desync_records(const __grid_constant__ DiffParams p) {
    __shared__ uint32_t s_warp[kDiffBlock / 32u];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const DiffTiles t = diff_tiles(p, p.tile_list[blockIdx.x]);
    const uint32_t base = p.tile_list[p.n_list + blockIdx.x];
    const uint32_t row = t.tile * kTileRows + threadIdx.x;
    auto no_column = [](uint32_t, bool, bool, bool) {};
    uint32_t n_rec = 0;
    diff_row(p, t, row, [&](uint32_t, uint32_t, uint32_t, uint32_t) { ++n_rec; }, no_column);
    // exclusive scan of n_rec over the block (row order)
    uint32_t incl = n_rec;
    for (uint32_t o = 1; o < 32u; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31u) s_warp[warp] = incl;
    __syncthreads();
    uint32_t warp_base = 0;
    for (uint32_t k = 0; k < warp; ++k) warp_base += s_warp[k];
    uint32_t pos = base + warp_base + incl - n_rec;
    if (n_rec == 0 || pos >= p.cap) return;  // no collective follows
    diff_row(p, t, row,
             [&](uint32_t c, uint32_t w, uint32_t a, uint32_t b) {
                 if (pos < p.cap) p.out[pos] = DiffRecord{row, c, w, a, b};
                 ++pos;
             },
             no_column);
}

}  // namespace bgr
