// Change feed (bgr_feed_*): report to the host only the live rows whose existence, presence or tracked field bytes
// changed since the feed's last report (see include/bevy_ggrs_b200.h "change feed").
//
// Per feed the device keeps the REPORTED state of every row, tile-planar like the images (kernels.cuh): per 512-row tile
// one plane of 512 u32 per tracked field word, then one byte per row, the row's reported mask byte: the image's mask
// byte reduced to the bits the record's state is made of (alive and the absent bits of the tracked columns), 0 for a row
// that did not exist.  Field words of a field that was not present are stored as zero.
//
// The passes are driven by a table of listed worlds (FeedWorld, one per world, ascending first global tile), the way
// ImageEntry drives the checkpoint kernels: bgr_batch_feed_begin lists many members of a world batch.  bgr_feed_begin
// runs its own instances of the passes (kTable = false, below) on the same per-row body, its one world in the kernel
// parameters.  The registration is the same for every listed
// world, so the field list and the record size are launch-wide.  A report is four launches:
//   pass 1 (k_feed_count, engine stream): one 512-thread block per tile of every listed world (its world found by binary
//          search over the table), one row per thread, reads the tracked word planes and the mask byte of image 0 and
//          the reported state (coalesced: a warp reads 128 B per plane).  A row differs when its reduced mask byte or any
//          tracked word (zero where not present) differs.  Warp ballots, one count per global tile, no atomics.
//   scan   (k_feed_scan, one block): walks the global tile sequence three times: the exclusive prefix of the counts; per
//          world its differing rows, n_records / pending under its own cap and its first record in the packed output
//          (an exclusive scan of the capped totals in list order); per tile its global record offset and the ascending
//          list of tiles that hold a reported record.  bgr_feed_begin runs k_feed_scan_one, the same
//          results for one world in one walk.
//   pass 2 (k_feed_records): only the listed tiles; a block-level exclusive scan of the per-row flags gives each row its
//          record index, so records land in ascending row order whatever the scheduling.  Rows below their world's cap
//          write their record at its packed position in the staging buffer and become the reported state.
//   copy   (k_feed_copy, copy stream, behind an event after pass 2): moves the records of every listed world from device
//          memory into page-locked host memory, so PCIe carries n_records * record_bytes; the 16-byte infos follow by
//          cudaMemcpyAsync.
// k_trace_gather (below) writes the same records for a row range whether or not they changed: the samples of a replay
// trace (bgr_replay_trace) taken without a generated kernel.
#pragma once
#include "kernels.cuh"

namespace bgr {

constexpr uint32_t kFeedMaxFields = 8;   // == BGR_MAX_FEED_FIELDS
constexpr uint32_t kFeedBlock = kTileRows;  // one thread per row of a tile
constexpr uint32_t kFeedScanBlock = 1024;

struct FeedField { uint32_t plane, words, absent, rep_plane; };  // image word plane, words, absent bit (0: not optional), reported plane

// one listed world of a report
struct FeedWorld {
    const uint8_t* img;          // image 0
    uint8_t* rep;                // the feed's reported state, tile-planar with `rep_words` planes
    uint32_t rows;               // RollbackOrdered::len() of image 0
    uint32_t n_tiles;            // tiles compared: those of max(rows, the feed's bound)
    uint32_t tile0;              // its first global tile (pass 1 block)
    uint32_t cap;                // records it may report
};

struct FeedParams {
    const FeedWorld* worlds;     // [n_worlds], ascending tile0; nullptr: the one world is `one` (bgr_feed_begin)
    FeedWorld one;
    uint32_t n_worlds, n_tiles;  // listed worlds; tiles of all of them
    uint32_t words, rep_words, n_fields, keep;  // keep: mask bits the state is made of
    uint32_t record_words;       // 2 + rep_words
    FeedField fields[kFeedMaxFields];
    unsigned int* tile_count;    // [n_tiles] pass 1 output
    unsigned int* tile_off;      // [n_tiles] global index of each tile's first record
    unsigned int* tile_list;     // [n_tiles] tiles holding a reported record, ascending
    unsigned int* world_scan;    // [n_worlds][2] the count prefix at the world's first tile, its first record
    unsigned int* info;          // [n_worlds][4] bgr_feed_info: n_records, pending, rows, record_bytes
    unsigned int* head;          // [0] records of every listed world [1] listed tiles
    uint32_t* out;               // the records, packed in list order
};

// The passes are instantiated twice.  kTable: the listed worlds are in p.worlds (bgr_batch_feed_begin).  Otherwise the
// one world is p.one (bgr_feed_begin), read from the parameter space with no lookup, as the single report's fields were
// before the passes took a table: its instances compile to the one-world code, and only the per-row body is shared.

// entry k of the listed worlds
template <bool kTable>
__device__ __forceinline__ FeedWorld feed_entry(const FeedParams& p, uint32_t k) { return kTable ? p.worlds[k] : p.one; }

// the listed world global tile `t` belongs to: the last entry whose tile0 <= t (a world without tiles shares the next
// one's tile0 and comes before it)
template <bool kTable>
__device__ __forceinline__ uint32_t feed_world_of(const FeedParams& p, uint32_t t) {
    if (!kTable) return 0;
    uint32_t lo = 0, hi = p.n_worlds;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (p.worlds[mid].tile0 <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// the reduced mask byte of `row` (of a world of `rows` rows) in image 0: 0 unless the row exists
__device__ __forceinline__ uint32_t feed_cur_mask(const FeedParams& p, const uint8_t* tile, uint32_t rows, uint32_t row) {
    const uint32_t m = row < rows ? uint32_t(tile[size_t(p.words) * kPlaneBytes + row % kTileRows]) : 0u;
    return (m & 1u) ? (m & p.keep) : 0u;
}
__device__ __forceinline__ bool feed_present(uint32_t m, uint32_t absent) { return (m & 1u) && !(m & absent); }

// current and reported (mask, words) of this thread's row of image tile `it` and reported tile `rt`; calls
// on_word(k, w, rep_plane, cur) for every tracked word and returns whether the row differs
template <class OnWord>
__device__ __forceinline__ bool feed_row(const FeedParams& p, const uint8_t* it, const uint8_t* rt, uint32_t cm, uint32_t rm,
                                         OnWord&& on_word) {
    const size_t lane_off = size_t(threadIdx.x) * 4u;
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

template <bool kTable>
__global__ void __launch_bounds__(kFeedBlock) k_feed_count(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedBlock / 32u];
    const uint32_t g = blockIdx.x;
    const FeedWorld w = feed_entry<kTable>(p, feed_world_of<kTable>(p, g));
    const uint32_t tile = g - w.tile0, row = tile * kTileRows + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint8_t* it = w.img + size_t(tile) * tile_bytes_of(p.words);
    const uint8_t* rt = w.rep + size_t(tile) * tile_bytes_of(p.rep_words);
    const uint32_t cm = feed_cur_mask(p, it, w.rows, row);
    const uint32_t rm = rt[size_t(p.rep_words) * kPlaneBytes + threadIdx.x];
    const bool diff = feed_row(p, it, rt, cm, rm, [](uint32_t, uint32_t, uint32_t, uint32_t) {});
    const uint32_t n = __popc(__ballot_sync(0xffffffffu, diff));
    if (lane == 0) s_warp[warp] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (uint32_t k = 0; k < kFeedBlock / 32u; ++k) t += s_warp[k];
        p.tile_count[g] = t;
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

// Every loop has a uniform trip count (feed_block_scan is a block collective).  The prefixes are u32 and wrap: only
// differences within one world are used, and no world has 2^32 rows.
__global__ void __launch_bounds__(kFeedScanBlock) k_feed_scan(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedScanBlock / 32u];
    uint32_t carry = 0;  // 1. tile_off = the exclusive prefix of the counts over the global tile sequence
    for (uint32_t base = 0; base < p.n_tiles; base += kFeedScanBlock) {
        const uint32_t t = base + threadIdx.x;
        uint32_t sum;
        const uint32_t off = carry + feed_block_scan(t < p.n_tiles ? p.tile_count[t] : 0u, s_warp, &sum);
        if (t < p.n_tiles) p.tile_off[t] = off;
        carry += sum;
    }
    __syncthreads();  // tile_off of every tile is written
    uint32_t records = 0;  // 2. per world: differing rows, records under its cap, its first record
    for (uint32_t base = 0; base < p.n_worlds; base += kFeedScanBlock) {
        const uint32_t i = base + threadIdx.x;
        uint32_t g0 = 0, differ = 0, n = 0, rows = 0;
        if (i < p.n_worlds) {
            const FeedWorld w = feed_entry<true>(p, i);
            const uint32_t end = w.tile0 + w.n_tiles;
            g0 = w.tile0 < p.n_tiles ? p.tile_off[w.tile0] : carry;
            differ = (end < p.n_tiles ? p.tile_off[end] : carry) - g0;
            n = differ < w.cap ? differ : w.cap;
            rows = w.rows;
        }
        uint32_t sum;
        const uint32_t first = records + feed_block_scan(n, s_warp, &sum);
        if (i < p.n_worlds) {
            p.world_scan[2u * i] = g0;
            p.world_scan[2u * i + 1u] = first;
            p.info[4u * i] = n;
            p.info[4u * i + 1u] = differ - n;
            p.info[4u * i + 2u] = rows;
            p.info[4u * i + 3u] = 4u * p.record_words;
        }
        records += sum;
    }
    __syncthreads();  // world_scan is written
    uint32_t listed = 0;  // 3. per tile: its global record offset, and the list of tiles that hold a reported record
    for (uint32_t base = 0; base < p.n_tiles; base += kFeedScanBlock) {
        const uint32_t t = base + threadIdx.x;
        uint32_t in_list = 0, off = 0;
        if (t < p.n_tiles) {
            const uint32_t i = feed_world_of<true>(p, t);
            const uint32_t in_world = p.tile_off[t] - p.world_scan[2u * i];
            off = p.world_scan[2u * i + 1u] + in_world;
            in_list = (p.tile_count[t] != 0u && in_world < feed_entry<true>(p, i).cap) ? 1u : 0u;
        }
        uint32_t lsum;
        const uint32_t pos = listed + feed_block_scan(in_list, s_warp, &lsum);
        if (t < p.n_tiles) p.tile_off[t] = off;  // only this thread reads tile_off[t] in this pass
        if (in_list) p.tile_list[pos] = t;
        listed += lsum;
    }
    if (threadIdx.x == 0) {
        p.head[0] = records;
        p.head[1] = listed;
    }
}

// bgr_feed_begin's scan: one world, so one walk does all k_feed_scan's three do (on a 1M-row report with 1 % of the
// rows changed, the three walks cost about 5 us of wall time per report)
__global__ void __launch_bounds__(kFeedScanBlock) k_feed_scan_one(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedScanBlock / 32u];
    uint32_t carry = 0, listed = 0;
    for (uint32_t base = 0; base < p.n_tiles; base += kFeedScanBlock) {  // uniform trip count
        const uint32_t t = base + threadIdx.x;
        const uint32_t v = t < p.n_tiles ? p.tile_count[t] : 0u;
        uint32_t sum, lsum;
        const uint32_t off = carry + feed_block_scan(v, s_warp, &sum);
        const uint32_t in_list = (v != 0u && off < p.one.cap) ? 1u : 0u;
        const uint32_t pos = listed + feed_block_scan(in_list, s_warp, &lsum);
        if (t < p.n_tiles) p.tile_off[t] = off;
        if (in_list) p.tile_list[pos] = t;
        carry += sum;
        listed += lsum;
    }
    if (threadIdx.x == 0) {
        const uint32_t n = carry < p.one.cap ? carry : p.one.cap;
        p.info[0] = n;
        p.info[1] = carry - n;
        p.info[2] = p.one.rows;
        p.info[3] = 4u * p.record_words;
        p.head[0] = n;
        p.head[1] = listed;
    }
}

// at most 32 registers: four blocks per SM stay resident, so the grid of four blocks per SM is one wave (at 40, the
// compiler's choice for the table, a 1M-row report's pass 2 took a second wave)
template <bool kTable>
__global__ void __launch_bounds__(kFeedBlock, 4) k_feed_records(const __grid_constant__ FeedParams p) {
    __shared__ uint32_t s_warp[kFeedBlock / 32u];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t n_list = p.head[1];
    for (uint32_t i = blockIdx.x; i < n_list; i += gridDim.x) {
        const uint32_t g = p.tile_list[i], k = feed_world_of<kTable>(p, g);
        const FeedWorld w = feed_entry<kTable>(p, k);
        const uint32_t tile = g - w.tile0, row = tile * kTileRows + threadIdx.x;
        const uint8_t* it = w.img + size_t(tile) * tile_bytes_of(p.words);
        uint8_t* rt = w.rep + size_t(tile) * tile_bytes_of(p.rep_words);
        const uint32_t cm = feed_cur_mask(p, it, w.rows, row);
        const uint32_t rm = rt[size_t(p.rep_words) * kPlaneBytes + threadIdx.x];
        const bool diff = feed_row(p, it, rt, cm, rm, [](uint32_t, uint32_t, uint32_t, uint32_t) {});
        const unsigned bal = __ballot_sync(0xffffffffu, diff);
        __syncthreads();  // s_warp of the previous tile has been read
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        uint32_t pos = p.tile_off[g] + __popc(bal & ((1u << lane) - 1u));
        for (uint32_t q = 0; q < warp; ++q) pos += s_warp[q];
        // the one world's first record is 0 (k_feed_scan_one writes no world_scan); no collective follows a continue
        if (!diff || pos - (kTable ? p.world_scan[2u * k + 1u] : 0u) >= w.cap) continue;
        uint32_t state = cm ? 1u : 0u;
        for (uint32_t q = 0; q < p.n_fields; ++q)
            if (feed_present(cm, p.fields[q].absent)) state |= 2u << q;
        uint32_t* rec = p.out + size_t(pos) * p.record_words;
        rec[0] = row;
        rec[1] = state;
        uint32_t at = 2;
        const size_t lane_off = size_t(threadIdx.x) * 4u;
        feed_row(p, it, rt, cm, cm, [&](uint32_t, uint32_t, uint32_t rp, uint32_t c) {
            rec[at++] = c;
            *reinterpret_cast<uint32_t*>(rt + size_t(rp) * kPlaneBytes + lane_off) = c;
        });
        rt[size_t(p.rep_words) * kPlaneBytes + threadIdx.x] = uint8_t(cm);
    }
}

// One listed world of a trace gather: the records of rows [first_row, first_row + n_rows) of image `img` (of `rows`
// rows) go to out; rec0 is its first record in the launch (a prefix of n_rows in table order)
struct TraceGather {
    const uint8_t* img;
    uint32_t* out;
    uint32_t rows, first_row, n_rows, rec0;
};

// The trace records of every listed world's rows (bgr_replay_trace without a generated kernel, at each sample frame):
// the change feed's record of each row (u32 row, u32 state, the field words, zero where not present), whether or not it
// changed, and state 0 with zero words for rows that do not exist.  One thread per record.
__global__ void __launch_bounds__(256) k_trace_gather(const __grid_constant__ FeedParams p, const TraceGather* __restrict__ tab,
                                                      uint32_t n_worlds, uint32_t n_records) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_records) return;
    uint32_t lo = 0, hi = n_worlds;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (tab[mid].rec0 <= t) lo = mid; else hi = mid;
    }
    const TraceGather g = tab[lo];
    const uint32_t i = t - g.rec0, row = g.first_row + i;
    const uint8_t* tile = g.img + size_t(row / kTileRows) * tile_bytes_of(p.words);  // read only where the row exists
    const uint32_t cm = feed_cur_mask(p, tile, g.rows, row);
    uint32_t* rec = g.out + size_t(i) * p.record_words;
    uint32_t state = cm ? 1u : 0u;
    for (uint32_t q = 0; q < p.n_fields; ++q)
        if (feed_present(cm, p.fields[q].absent)) state |= 2u << q;
    rec[0] = row;
    rec[1] = state;
    uint32_t at = 2;
    const size_t lane_off = size_t(row % kTileRows) * 4u;
    for (uint32_t q = 0; q < p.n_fields; ++q) {
        const FeedField f = p.fields[q];
        const bool pc = feed_present(cm, f.absent);
        for (uint32_t w = 0; w < f.words; ++w)
            rec[at++] = pc ? *reinterpret_cast<const uint32_t*>(tile + size_t(f.plane + w) * kPlaneBytes + lane_off) : 0u;
    }
}

// staging -> page-locked host memory: head[0] records of record_words words
__global__ void __launch_bounds__(256) k_feed_copy(const uint32_t* __restrict__ stage, const unsigned int* __restrict__ head,
                                                   uint32_t record_words, uint32_t* host_records) {
    const size_t n = size_t(head[0]) * record_words;
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x)
        host_records[t] = stage[t];
}

}  // namespace bgr
