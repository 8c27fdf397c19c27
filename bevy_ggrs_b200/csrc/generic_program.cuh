// The one-launch path for ANY registered schema and the compiled GgrsSchedule systems: a whole Vec<GgrsRequest>
// (Load / Advance / Save ...) interpreted by one kernel, like k_particles_program, but without knowing the columns at
// compile time.  One 512-row tile per block iteration lives in SHARED MEMORY for the whole program:
//
//     cp.async.bulk  slot/live image --> shared tile              (LOAD, or the program's first read)
//     ADVANCE : every registered system updates its rows of the shared tile in place (a thread owns its rows for the
//               whole program, so no barrier separates systems; despawn commands are applied after the last system,
//               then spawn_particles' newborn rows are written: a row is not updated in the frame it is born)
//     SAVE    : cp.async.bulk shared tile --> the frame's slot, while all threads hash the checksummed byte ranges
//               of their rows out of the same tile (component_checksum.rs:67-108) and count live rows
//     end     : cp.async.bulk shared tile --> live image
//
// so a SyncTest tick of a box_game / score-and-health style world is ONE launch instead of one launch per request
// and per system (round 1's "stepwise" path, which stays as the fallback for schemas wider than a shared-memory tile).
// Per-entity component presence (BGR_STRATEGY_OPTIONAL) is the row's mask byte: it travels with the tile, and every
// system / checksum applies the reference's query filter per row (kernels.cuh row_matches).
//
// Reference semantics: handle_requests (schedule_systems.rs:170-289) over ComponentSnapshotPlugin::save / load
// (component_snapshot.rs:66-123), the checksum plugins, and the systems listed in include/bevy_ggrs_b200.h.
#pragma once
#ifdef __CUDACC_RTC__  // NVRTC (the engine's run-time specialisation, generic_program_jit.cuh): no host headers
#include "rtc_prelude.cuh"
#else
#include <cuda_runtime.h>
#include <cmath>
#include <cstdint>
#include <cstring>
#endif

#include "kernels.cuh"
#include "seahash.cuh"
#include "tma_copy.cuh"

namespace bgr {

constexpr int kMaxGenericSys = 8;
// threads per block: 128 = 4 rows of the tile per thread, four independent hash chains interleaved per thread (DESIGN.md
// has the measurements against 1, 2 and 8 rows).  This kernel is the INTERPRETER: it reads the
// schema from its parameter block.  bgr_build also compiles the registration's own kernel with NVRTC when it can
// (generic_program_jit.cuh, jit.hpp), and this one is then only the fallback.
constexpr int kGenericBlock = 128;

struct GenericParams {
    uint8_t* arena;
    unsigned long long order_base;
    unsigned long long* accum;  // device [kMaxSaves][kAccStride]
    unsigned long long* out;    // host-mapped result block (same layout / protocol as k_particles_program)
    unsigned int* ticket;       // [0] block-completion ticket, [1] dynamic tile counter
    unsigned long long seq;
    unsigned long long* trace;
    const float2* spawn_vals;      // (vx, vy) of every row an OPF_SPAWN ADVANCE spawns (host-mapped; the op's call_count indexes it)
    unsigned long long spawn_ttl;  // Ttl of a spawned row (spawn_particles' param)
    uint32_t words, tile_bytes, n_ops, n_saves, n_tiles, live_rows, flags, n_hash, n_sys;
    // overlap of consecutive launches (generated kernel only; the protocol of k_particles_program's PF_TILE_SIGNAL / PF_TILE_WAIT
    // per WORK ITEM): item_done[i] = sequence number of the last signalling launch whose stores of item i are visible
    unsigned int* item_done;
    uint32_t done_seq, wait_seq, wait_items;
    HashSpec hash[kMaxHashCols];
    SysSpec sys[kMaxGenericSys];
    Op ops[kMaxOps];
};
static_assert(sizeof(GenericParams) <= 4000, "kernel parameter block must fit 4 KB");

// One request vector of one engine on the generated kernel, without its ops and registration: the per-world record of
// a batched launch (k_generic_jit_batch, generic_program_jit.cuh), copied to the device with the worlds' ops behind the
// records.  run_generic builds the same record for its own GenericParams.
struct JitWorld {
    uint8_t* arena;
    unsigned long long order_base;
    unsigned long long* accum;
    unsigned int* ticket;
    unsigned long long* out;
    unsigned long long seq;
    const float2* spawn_vals;
    unsigned long long spawn_ttl;
    uint32_t n_ops, n_saves, n_tiles, live_rows, flags;
    uint32_t item0;    // batched launch: the world's first block (sum of the item counts of the worlds before it)
    uint32_t ops_off;  // batched launch: index of the world's first op in the launch's op array
    uint32_t pad;
};
static_assert(sizeof(JitWorld) == 96, "JitWorld layout");

// ---- replays (bgr_replay): the ADVANCE op of frame j of an input log, derived from the frame index ----
// What compile_requests builds for AdvanceFrame j of the stream, field by field, from values fixed before the log starts.
// The host evaluates everything that needs the C library (powf) once; the rest is integer arithmetic.
struct ReplayClock {
    int32_t f0;               // RollbackFrameCount before frame 0
    uint32_t fps;
    uint32_t n_players;       // PlayerInputs<T>.len() of every frame
    uint32_t dt0, fr0;        // the first step's (dt_bits, fr_bits): Time<GgrsTime> may have been set by a restore
    uint32_t dt[2], fr[2];    // every later step lasts floor(1e9 / fps) ns ([0]) or one more ([1])
    uint32_t call0;           // BGR_SYS_U32_STORE_CALL_COUNT counter before frame 0
    uint32_t n_counter;       // counter systems: the counter grows by this per frame
    uint32_t spawn;           // 1: the registration has spawn_particles (an INPUT_SPAWN frame sets OPF_SPAWN)
    uint32_t rate;            // its rows per spawn frame
    uint32_t rows0;           // RollbackOrdered::len() before frame 0
};
static_assert(sizeof(ReplayClock) == 56, "ReplayClock layout (the engine and the NVRTC module must agree)");

#ifndef __CUDACC_RTC__
// The clock of a log that starts at RollbackFrameCount f0 with Time<GgrsTime> at `elapsed_ns` (the caller has checked
// that the first step does not move it backwards): each step's (dt_bits, fr_bits) as compile_requests evaluates them,
// Duration::as_secs_f32 and the C library's powf (move_cube_system's friction, box_game.rs:188-193).  Host only.
inline ReplayClock replay_clock(int32_t f0, uint32_t fps, uint64_t elapsed_ns, uint32_t n_players, uint32_t call0,
                                uint32_t n_counter, bool spawn, uint32_t rate, uint32_t rows0) {
    auto step = [](uint64_t ns, uint32_t* dt, uint32_t* fr) {
        const float secs = float(ns / 1000000000ULL) + float(uint32_t(ns % 1000000000ULL)) / 1000000000.0f;
        const float f = powf(0.0018f, secs);
        std::memcpy(dt, &secs, 4);
        std::memcpy(fr, &f, 4);
    };
    ReplayClock c;
    std::memset(&c, 0, sizeof c);
    c.f0 = f0; c.fps = fps; c.n_players = n_players; c.call0 = call0; c.n_counter = n_counter;
    c.spawn = spawn ? 1u : 0u; c.rate = spawn ? rate : 0u; c.rows0 = rows0;
    step(uint64_t(int64_t(f0) + 1) * 1000000000ULL / fps - elapsed_ns, &c.dt0, &c.fr0);
    const uint64_t base = 1000000000ULL / fps;
    step(base, &c.dt[0], &c.fr[0]);
    step(base + 1, &c.dt[1], &c.fr[1]);
    return c;
}
#endif

// Checksum frames of a log that starts at f0, with interval k: the first frame index j in [a, b) with (f0 + j) % k == 0
// (~0: none), and how many there are
__host__ __device__ inline unsigned long long replay_first_point(int32_t f0, uint32_t k, uint32_t a, uint32_t b) {
    if (!k) return ~0ULL;
    const unsigned long long rem = (unsigned long long)(int64_t(f0) + a) % k;
    const unsigned long long j = (unsigned long long)a + (rem ? k - rem : 0u);
    return j < b ? j : ~0ULL;
}
__host__ __device__ inline uint32_t replay_points_in(int32_t f0, uint32_t k, uint32_t a, uint32_t b) {
    const unsigned long long f = replay_first_point(f0, k, a, b);
    return f == ~0ULL ? 0u : uint32_t((b - 1u - f) / k + 1u);
}

// `in`: the frame's n_players input bytes; `prefix`: the spawn frames before frame j
__host__ __device__ inline Op replay_op(const ReplayClock& c, uint32_t j, const uint8_t* in, uint32_t prefix) {
    Op op;
    op.kind = OP_ADVANCE;
    op.image_off256 = 0; op.save_index = 0;
    if (j == 0) {
        op.dt_bits = c.dt0; op.fr_bits = c.fr0;
    } else {  // GgrsTimePlugin::update: advance_to(frame * 1e9 / fps), from frame f0 + j to f0 + j + 1
        const unsigned long long f = (unsigned long long)(c.f0 + int32_t(j)), ns = 1000000000ULL;
        const bool longer = (f + 1ULL) * ns / c.fps - f * ns / c.fps != ns / c.fps;
        op.dt_bits = longer ? c.dt[1] : c.dt[0];  // selects, not an index: the clock stays in registers
        op.fr_bits = longer ? c.fr[1] : c.fr[0];
    }
    op.n_rows = c.rows0 + c.rate * prefix;
    op.call_count = c.call0 + c.n_counter * j;
    op.flags = (c.n_players & 0xFu) << 8;
    uint32_t pressed = 0;
    for (uint32_t k = 0; k < 8u; ++k) {
        const uint8_t v = k < c.n_players ? in[k] : uint8_t(0);
        op.inputs[k] = v;
        pressed |= v & 0x10u;  // BGR_INPUT_SPAWN
    }
    if (c.spawn && pressed) {  // spawn_particles' rows: first row, count, offset into the log's spawn values
        op.flags |= OPF_SPAWN;
        op.image_off256 = op.n_rows;
        op.save_index = c.rate;
        op.call_count = c.rate * prefix;
    }
    return op;
}

// One world's frames [j0, j1) of a replay on the generated kernel (k_generic_jit_replay, generic_program_jit.cuh).
// Rows come from and go back to the live image.  The block's checksum points go to acc[point][kAccStride], point 0
// being the first checksum frame at or after j0.
struct ReplayWorld {
    uint8_t* arena;
    unsigned long long order_base;
    unsigned long long* acc;
    const uint8_t* inputs;         // the whole log, frame-major (n_players bytes per frame)
    const uint32_t* prefix;        // [n_frames + 1] spawn frames before each frame; nullptr without spawn_particles (all 0)
    const float2* spawn_vals;      // (vx, vy) of every row the log spawns, in frame order
    unsigned long long spawn_ttl;
    unsigned long long next_point; // first checksum frame >= j0 (>= j1: none)
    ReplayClock c;
    uint32_t interval;             // checksum_interval (0: none)
    uint32_t j0, j1;
    uint32_t n_tiles, live_rows;   // tiles of the rows at j1; rows of the live image at j0
    uint32_t item0;                // first block of the world
};
static_assert(sizeof(ReplayWorld) == 144, "ReplayWorld layout (the engine and the NVRTC module must agree)");

// The keyframes of one world's frames [j0, j1) (bgr_replay_keyframes), parallel to the ReplayWorld array and read only by
// k_generic_jit_replay_kf: at frame first + q * interval < j1 the block stores its registers, before advancing that
// frame, into keyframe image q at staging + q * stride.
struct ReplayKeyframes {
    uint8_t* staging;
    unsigned long long stride;     // bytes per keyframe image (>= the world's tiles in this launch)
    unsigned long long first;      // first keyframe frame >= j0 (>= j1: none)
    uint32_t interval, reserved;
};
static_assert(sizeof(ReplayKeyframes) == 32, "ReplayKeyframes layout (the engine and the NVRTC module must agree)");

// The trace samples of one world's frames [j0, j1) (bgr_replay_trace), parallel to the ReplayWorld array and read only by
// k_generic_jit_replay_trace: at frame first + q * interval < j1, before advancing that frame, the block writes the
// record of each of its rows in [first_row, first_row + n_rows) to staging + q * stride + (row - first_row) * record bytes.
struct ReplayTrace {
    uint8_t* staging;
    unsigned long long stride;     // bytes per sample: n_rows records
    unsigned long long first;      // first sample frame >= j0 (>= j1: none)
    uint32_t interval;
    uint32_t first_row, n_rows;
    uint32_t reserved;
};
static_assert(sizeof(ReplayTrace) == 40, "ReplayTrace layout (the engine and the NVRTC module must agree)");

// Where a trace record's field words come from, built on the host from the change feed's field list and passed to
// k_generic_jit_replay_trace by value: record word 2 + slot[s] for s in [word_first[j], word_first[j + 1]) is word plane j
// (zero unless the row exists and word_absent[j], its column's absent bit, is clear).  A plane listed by several fields
// has several slots.  The generated kernel takes rows of at most 24 words, so a record holds at most 8 * 24 field words.
constexpr uint32_t kTraceMaxWords = 24;
constexpr uint32_t kTraceMaxSlots = 8u * kTraceMaxWords;
struct TraceMap {
    uint32_t n_fields, record_words;       // record_words: 2 + the field words
    uint8_t field_absent[8];               // field k's absent bit: state bit 1 + k
    uint8_t word_absent[kTraceMaxWords];
    uint8_t word_first[kTraceMaxWords + 1];
    uint8_t slot[kTraceMaxSlots];
    uint8_t pad[3];
};
static_assert(sizeof(TraceMap) == 260, "TraceMap layout (the engine and the NVRTC module must agree)");

// seahash of bytes [off, off+len) of one row's element whose words are `col[w * kTileRows]` (a column of the shared tile)
// (__noinline__: inlined per checksummed column and per row the interpreter grew to 11k instructions — 176 KB of code,
// more than the SM's instruction cache — and ran 2.7x slower per frame than the specialised bundle kernel)
__device__ __noinline__ uint64_t hash_row_range(const uint32_t* col, uint32_t off, uint32_t len) {
    if (((off | len) & 3u) == 0u) {  // word-aligned range (every POD of u32 / f32 / u64 fields): no byte shuffling
        const uint32_t* w = col + size_t(off >> 2) * kTileRows;
        // the common element sizes without a loop (warp-uniform switch: every row of a column has the same range)
        switch (len) {
        case 4: return sea_diffuse(sea_diffuse(kSeaA ^ uint64_t(w[0])) ^ kSeaB ^ kSeaC ^ kSeaD ^ 4ULL);
        case 8: return sea_hash_u64(uint64_t(w[0]) | (uint64_t(w[kTileRows]) << 32));
        case 12: return sea_hash_12(uint64_t(w[0]) | (uint64_t(w[kTileRows]) << 32), w[2 * kTileRows]);
        case 16: return sea_hash_2xu64(uint64_t(w[0]) | (uint64_t(w[kTileRows]) << 32), uint64_t(w[2 * kTileRows]) | (uint64_t(w[3 * kTileRows]) << 32));
        default: break;
        }
        uint64_t a = kSeaA, b = kSeaB, c = kSeaC, d = kSeaD;
        uint32_t i = 0;
        for (; i + 8 <= len; i += 8) {
            const uint64_t x = uint64_t(w[0]) | (uint64_t(w[kTileRows]) << 32);
            w += 2 * kTileRows;
            const uint64_t t = sea_diffuse(a ^ x);
            a = b; b = c; c = d; d = t;
        }
        if (i < len) a = sea_diffuse(a ^ uint64_t(w[0]));
        return sea_diffuse(a ^ b ^ c ^ d ^ uint64_t(len));
    }
    auto byte_at = [&](uint32_t q) -> uint8_t {
        const uint32_t bb = off + q;
        return uint8_t(col[size_t(bb >> 2) * kTileRows] >> (8 * (bb & 3u)));
    };
    return sea_hash_stream(len, byte_at);
}

// One checksummed column whose element is NW whole words (4 * NW bytes, word-aligned) for the thread's R rows:
// `col` points at the first word of the thread's first row, rows are `B` words apart, words of an element kTileRows apart.
// Branch-free per row (a row without the component contributes 0), so the rows' hash chains interleave.
template <int NW, int R, int B>
__device__ __forceinline__ void hash_words_column(const uint32_t* col, const uint32_t (&m)[R], uint32_t absent, uint32_t finite,
                                                  const uint64_t (&t0)[R], uint64_t& hx, uint32_t& bad) {
#pragma unroll
    for (int k = 0; k < R; ++k) {
        uint32_t w[NW];
#pragma unroll
        for (int j = 0; j < NW; ++j) w[j] = col[k * B + j * kTileRows];
        const bool has = row_matches(m[k], absent);  // Query<(&RollbackId, &T)>: exists and has the component
        uint32_t nonfinite = 0;
#pragma unroll
        for (int j = 0; j < NW; ++j) nonfinite |= f32_bits_nonfinite(w[j]);
        bad |= (has && finite) ? nonfinite : 0u;
        uint64_t h;
        if (NW == 1) h = sea_diffuse(sea_diffuse(kSeaA ^ uint64_t(w[0])) ^ kSeaB ^ kSeaC ^ kSeaD ^ 4ULL);
        else if (NW == 2) h = sea_hash_u64(uint64_t(w[0]) | (uint64_t(w[1 % NW]) << 32));
        else if (NW == 3) h = sea_hash_12(uint64_t(w[0]) | (uint64_t(w[1 % NW]) << 32), w[2 % NW]);
        else h = sea_hash_2xu64(uint64_t(w[0]) | (uint64_t(w[1 % NW]) << 32), uint64_t(w[2 % NW]) | (uint64_t(w[3 % NW]) << 32));
        const uint64_t e = sea_hash_entity(t0[k], h);
        hx ^= has ? e : 0ULL;
    }
}

#ifndef __CUDACC_RTC__  // the run-time specialisation only needs the structs and helpers: its cubin holds its own entry points alone
__global__ void __launch_bounds__(kGenericBlock) k_generic_program(const __grid_constant__ GenericParams p) {
    constexpr int kRows = kTileRows / kGenericBlock;  // rows of a tile per thread
    extern __shared__ __align__(128) uint8_t s_buf[];  // one tile
    __shared__ unsigned int s_acc[kMaxSaves * kAccStride * 2];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ uint32_t s_next;
    __shared__ unsigned int s_last;

    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    if (p.trace && tid == 0) atomicMin(&p.trace[0], globaltimer_ns());
    for (uint32_t i = tid; i < p.n_saves * kAccStride * 2; i += kGenericBlock) s_acc[i] = 0u;
    if (tid == 0) { mbar_init(&s_bar, 1); fence_mbar_init(); }
    __syncthreads();

    // ONE tile buffer.  (A ping-pong pair — ADVANCE reading one buffer and writing the other so that a SAVE's bulk store
    // could keep reading — was measured: no faster, the store has long finished reading when the next ADVANCE starts,
    // and it costs a copy of every word per frame and half the resident blocks.)
    uint8_t* const s_tile = s_buf;
    uint8_t* const s_alive = s_tile + size_t(p.words) * kPlaneBytes;
    uint32_t* const tile_w = reinterpret_cast<uint32_t*>(s_tile);  // word (plane, row) = tile_w[plane * kTileRows + row]
    uint32_t phase = 0;
    bool store_pending = false;  // a bulk store may still be reading the shared tile (block-uniform)

    // the shared tile is about to be modified: pending bulk stores must have read it
    auto before_write = [&]() {
        if (store_pending) {
            if (tid == 0) tma_wait_read<0>();
            __syncthreads();
            store_pending = false;
        }
    };
    // bring tile `t` of image `img` into shared memory; rows the image never contained come back dead
    auto load_tile = [&](const uint8_t* img, uint32_t t, uint32_t n_rows_src) {
        __syncthreads();  // every thread is done with the previous content
        if (tid == 0) {
            tma_wait_read<0>();
            mbar_arrive_expect_tx(&s_bar, p.tile_bytes);
            tma_load_1d(s_tile, img + size_t(t) * p.tile_bytes, p.tile_bytes, &s_bar);
        }
        mbar_wait(&s_bar, phase);
        phase ^= 1u;
        store_pending = false;
        if (size_t(t + 1) * kTileRows > n_rows_src) {
#pragma unroll
            for (int k = 0; k < kRows; ++k) {
                const uint32_t r = tid + k * kGenericBlock;
                if (t * kTileRows + r >= n_rows_src) s_alive[r] = 0;
            }
        }
    };
    auto store_tile = [&](uint8_t* img, uint32_t t) {
        fence_proxy_async();  // generic-proxy writes of this thread are visible to the bulk (async-proxy) store
        __syncthreads();
        if (tid == 0) {
            tma_store_1d(img + size_t(t) * p.tile_bytes, s_tile, p.tile_bytes);
            tma_commit();
        }
        store_pending = true;
    };

    const uint8_t* first_img = p.arena + ((p.flags & PF_READ_LIVE) ? size_t(0) : (size_t(p.ops[0].image_off256) << 8));
    const uint32_t first_rows = (p.flags & PF_READ_LIVE) ? p.live_rows : p.ops[0].n_rows;

    for (uint32_t tile = blockIdx.x; tile < p.n_tiles;) {
        __syncthreads();  // every thread has read the previous s_next
        if (tid == 0) s_next = gridDim.x + atomicAdd(&p.ticket[1], 1u);  // the block's next tile (read after the barrier in load_tile)
        load_tile(first_img, tile, first_rows);
        const uint32_t next_tile = s_next;
        // first lane of the per-entity hash: only depends on the RollbackOrdered index — once per tile, not per SAVE
        const unsigned long long row0 = p.order_base + size_t(tile) * kTileRows + tid;
        uint64_t t0[kRows];
#pragma unroll
        for (int k = 0; k < kRows; ++k) t0[k] = sea_order_lane(row0 + uint32_t(k * kGenericBlock));

        for (uint32_t i = (p.flags & PF_READ_LIVE) ? 0u : 1u; i < p.n_ops; ++i) {
            const Op& op = p.ops[i];
            if (op.kind == OP_ADVANCE) {
                before_write();
                // systems outside, the thread's rows inside (run_system): a system's spec is decoded once for all of them
                uint32_t m[kRows];
                bool kill[kRows];
#pragma unroll
                for (int k = 0; k < kRows; ++k) { m[k] = s_alive[tid + k * kGenericBlock]; kill[k] = false; }
                auto word = [&](int k, uint32_t plane) -> uint32_t& { return tile_w[plane * uint32_t(kTileRows) + tid + k * kGenericBlock]; };
#pragma unroll 1
                for (uint32_t s = 0; s < p.n_sys; ++s) {
                    const SysSpec sy = p.sys[s];
                    run_system<kRows>(sy, word, m, kill, op, row0, kGenericBlock);
                }
#pragma unroll
                for (int k = 0; k < kRows; ++k)
                    if (kill[k]) s_alive[tid + k * kGenericBlock] = 0;
                if (op.flags & OPF_SPAWN) {  // spawn_particles' Commands: rows [first, first + count) are born after the despawns
                    uint32_t s = 0;
                    while (p.sys[s].id != BGR_SYS_PARTICLES_SPAWN) ++s;  // OPF_SPAWN: the registration has the system (compile_requests)
                    const SysSpec sy = p.sys[s];
#pragma unroll
                    for (int k = 0; k < kRows; ++k) {
                        const uint32_t born = tile * kTileRows + tid + k * kGenericBlock - op.image_off256;  // index among the spawned rows
                        if (born < op.save_index) {
                            spawn_row(sy, word, k, p.words, p.spawn_vals[op.call_count + born], p.spawn_ttl);
                            s_alive[tid + k * kGenericBlock] = 1;
                        }
                    }
                }
            } else if (op.kind == OP_SAVE) {
                // the bulk store streams the tile to the frame's slot while the threads hash their rows out of it
                if (!(op.flags & OPF_NO_STORE)) store_tile(p.arena + (size_t(op.image_off256) << 8), tile);
                uint32_t m[kRows];
                uint32_t n_alive = 0, bad = 0;
#pragma unroll
                for (int k = 0; k < kRows; ++k) {
                    m[k] = s_alive[tid + k * kGenericBlock];
                    n_alive += m[k] & 1u;
                }
                const unsigned full = 0xffffffffu;
                unsigned int* a = &s_acc[op.save_index * kAccStride * 2];
#pragma unroll 1
                for (uint32_t c = 0; c < p.n_hash; ++c) {  // one checksummed column at a time
                    const HashSpec hs = p.hash[c];
                    const uint32_t* col = tile_w + (hs.first_plane + (hs.off >> 2)) * uint32_t(kTileRows) + tid;
                    uint64_t hx = 0;
                    // the common element shapes (whole u32 / f32 / u64 fields, 4..16 bytes) inline and branch-free per
                    // row; anything else through the one out-of-line copy of the general hash.  The switch is uniform.
                    const uint32_t shape = ((hs.off | hs.len) & 3u) == 0u ? hs.len >> 2 : 0u;
                    switch (shape) {
                    case 1: hash_words_column<1, kRows, kGenericBlock>(col, m, hs.absent, hs.finite, t0, hx, bad); break;
                    case 2: hash_words_column<2, kRows, kGenericBlock>(col, m, hs.absent, hs.finite, t0, hx, bad); break;
                    case 3: hash_words_column<3, kRows, kGenericBlock>(col, m, hs.absent, hs.finite, t0, hx, bad); break;
                    case 4: hash_words_column<4, kRows, kGenericBlock>(col, m, hs.absent, hs.finite, t0, hx, bad); break;
                    default: {
                        const uint32_t* base = tile_w + hs.first_plane * uint32_t(kTileRows) + tid;
#pragma unroll
                        for (int k = 0; k < kRows; ++k) {
                            if (!row_matches(m[k], hs.absent)) continue;  // Query<(&RollbackId, &T)>: exists and has the component
                            if (hs.finite)
                                for (uint32_t q = 0; q + 4 <= hs.len; q += 4) bad |= f32_bits_nonfinite(base[k * kGenericBlock + ((hs.off + q) >> 2) * uint32_t(kTileRows)]);
                            hx ^= sea_hash_entity(t0[k], hash_row_range(base + k * kGenericBlock, hs.off, hs.len));
                        }
                    }
                    }
                    const uint32_t lo = __reduce_xor_sync(full, uint32_t(hx)), hi = __reduce_xor_sync(full, uint32_t(hx >> 32));
                    if (lane == 0) { atomicXor(&a[2 * hs.slot], lo); atomicXor(&a[2 * hs.slot + 1], hi); }
                }
                const uint32_t cnt = __reduce_add_sync(full, n_alive);
                const uint32_t anybad = __reduce_or_sync(full, bad);
                if (lane == 0) { atomicAdd(&a[12], cnt); if (anybad) atomicOr(&a[14], 1u); }
            } else {  // OP_LOAD
                load_tile(p.arena + (size_t(op.image_off256) << 8), tile, op.n_rows);
            }
        }
        if (p.flags & PF_WRITE_LIVE_ACTIVE) store_tile(p.arena, tile);
        tile = next_tile;
    }
    if (tid == 0) tma_wait_all();  // every bulk store has landed before the results are published

    // ---- block partials -> global accumulators -> (last block) host-visible results: k_particles_program's protocol ----
    __syncthreads();
    for (uint32_t i = tid; i < p.n_saves * kAccStride; i += kGenericBlock) {
        unsigned long long v = (unsigned long long)s_acc[2 * i] | ((unsigned long long)s_acc[2 * i + 1] << 32);
        const uint32_t c = i % kAccStride;
        if (v) {
            if (c == 6) atomicAdd(&p.accum[i], v);
            else if (c == 7) atomicOr(&p.accum[i], v);
            else atomicXor(&p.accum[i], v);
        }
    }
    __threadfence();
    __syncthreads();
    if (p.trace && tid == 0) atomicMax(&p.trace[1], globaltimer_ns());
    if (tid == 0) s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1u);
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (uint32_t i = tid; i < p.n_saves * kAccStride; i += kGenericBlock)
            publish_pair(p.out, i, atomicExch(&p.accum[i], 0ULL), p.seq);
        if (tid == 0) publish_pair(p.out, kSeqIndex, p.seq, p.seq);
        __syncthreads();
        if (tid == 0) {
            p.ticket[0] = 0u;
            p.ticket[1] = 0u;
            if (p.trace) p.trace[2] = globaltimer_ns();
        }
    }
}
#endif  // !__CUDACC_RTC__

}  // namespace bgr
