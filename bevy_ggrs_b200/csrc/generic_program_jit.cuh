// k_generic_program SPECIALISED AT RUN TIME for one registration (compiled by NVRTC inside bgr_build: engine.cu `jit_specialise`, jit.hpp).
//
// The interpreter (generic_program.cuh) reads the schema — which planes a system touches, which byte ranges are hashed —
// from its parameter block, so a tile has to live in shared memory (registers cannot be indexed at run time; the
// register-resident attempts with select chains / jump tables are recorded in DESIGN.md).  With the schema as
// COMPILE-TIME constants every plane index is a literal, and the same program becomes what k_particles_program is for
// the particles bundle:
//
//     LOAD / first read : coalesced ld.global of the row's words, plane by plane, from the slot / live image
//     ADVANCE           : the registered systems update the register copy (indices are constants: plain register ops),
//                         then the despawns, then spawn_particles' newborn rows (kernels.cuh spawn_row)
//     SAVE              : coalesced st.global of the words to the frame's slot + the per-entity seahash of every
//                         checksummed column, folded warp-REDUX -> shared atomics like the interpreter
//     end               : st.global to the live image
//
// no shared-memory tile, no bulk copy, no block barrier inside a tile's program, no spec decoding.  The engine generates
// a prelude of #defines (BGR_JIT_*) from the registration and compiles prelude + this file; parameter block, result
// protocol, tile claiming and op semantics are the interpreter's, and every parity test of the generic path runs on
// both (BGR_TUNE_JIT=0 / 2).
//
// Reference semantics: handle_requests (schedule_systems.rs:170-289) over ComponentSnapshotPlugin::save / load
// (component_snapshot.rs:66-123) and the checksum plugins (component_checksum.rs:67-108).
#pragma once
#include "generic_program.cuh"

namespace bgr {

constexpr int kJitWords = BGR_JIT_WORDS;  // word planes per row
constexpr int kJitRows = BGR_JIT_ROWS;    // rows of a work item per thread
// rows per WORK ITEM: a tile (512) for worlds of many tiles per SM; 256 / 128 for small worlds — 100k entities are 196 tiles on
// 132 SMs, so with whole tiles half of the SMs carry two tiles and set the kernel's duration (they are bound by the integer
// multiply pipe of the seahash, scripts/frame_cost_fit.py) while the others idle half of it; quarter tiles spread the rows evenly
constexpr int kJitItemRows = BGR_JIT_ITEM_ROWS;
constexpr int kJitSubs = int(kTileRows) / kJitItemRows;  // work items per tile
constexpr int kJitNSys = BGR_JIT_NSYS;
constexpr int kJitNHash = BGR_JIT_NHASH;
constexpr SysSpec kJitSys[kJitNSys + 1] = {BGR_JIT_SYS_LIST};      // {id, plane0, plane1, need, param}, ... + one dummy
constexpr HashSpec kJitHash[kJitNHash + 1] = {BGR_JIT_HASH_LIST};  // {first_plane, off, len, finite, slot, absent}, ... + one dummy

// index of spawn_particles in kJitSys, or -1: a registration without it compiles no spawn code at all
__host__ __device__ constexpr int jit_spawn_index() {
    for (int s = 0; s < kJitNSys; ++s)
        if (kJitSys[s].id == BGR_SYS_PARTICLES_SPAWN) return s;
    return -1;
}
constexpr int kJitSpawn = jit_spawn_index();

// seahash of the NWORDS whole words at planes [F, F + NWORDS) of a row: the stream form of seahash.cuh with the lane
// rotation done by renaming (word pair q goes to lane q % 4, the odd tail word to the next lane)
template <int F, int NWORDS>
__device__ __forceinline__ uint64_t jit_hash_words(const uint32_t (&w)[kJitWords]) {
    uint64_t s[4] = {kSeaA, kSeaB, kSeaC, kSeaD};
#pragma unroll
    for (int q = 0; q < NWORDS / 2; ++q)
        s[q & 3] = sea_diffuse(s[q & 3] ^ (uint64_t(w[F + 2 * q]) | (uint64_t(w[F + 2 * q + 1]) << 32)));
    if (NWORDS & 1) s[(NWORDS / 2) & 3] = sea_diffuse(s[(NWORDS / 2) & 3] ^ uint64_t(w[F + NWORDS - 1]));
    return sea_diffuse(s[0] ^ s[1] ^ s[2] ^ s[3] ^ uint64_t(NWORDS * 4));
}

struct JitRows {
    uint32_t w[kJitRows][kJitWords];  // the rows' words
    uint32_t m[kJitRows];             // mask bytes: bit 0 alive, bits 1.. absent bits of the optional columns
    uint64_t t0[kJitRows];            // first lane of the per-entity hash (RollbackOrdered index): once per tile
    bool kill[kJitRows];
};

// the S-th registered system on the register copy (run_system with a constexpr spec: plain register ops)
template <int S>
__device__ __forceinline__ void jit_run_systems(JitRows& r, const Op& op, unsigned long long row0, int B) {
    if constexpr (S < kJitNSys) {
        constexpr SysSpec sy = kJitSys[S];
        run_system<kJitRows>(sy, [&](int k, uint32_t plane) -> uint32_t& { return r.w[k][plane]; }, r.m, r.kill, op, row0, uint32_t(B));
        jit_run_systems<S + 1>(r, op, row0, B);
    }
}

// the C-th checksummed column: per-entity hash of the thread's rows, folded into the save's shared accumulators
template <int C>
__device__ __forceinline__ void jit_hash_columns(const JitRows& r, unsigned int* a, uint32_t lane, uint32_t& bad) {
    if constexpr (C < kJitNHash) {
        constexpr HashSpec hs = kJitHash[C];
        constexpr int F = int(hs.first_plane + (hs.off >> 2)), NWORDS = int(hs.len >> 2);
        uint64_t hx = 0;
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) {
            const bool has = row_matches(r.m[k], hs.absent);  // Query<(&RollbackId, &T)>: exists and has the component
            if constexpr (hs.finite != 0) {
                uint32_t nonfinite = 0;
#pragma unroll
                for (int j = 0; j < NWORDS; ++j) nonfinite |= f32_bits_nonfinite(r.w[k][F + j]);
                bad |= has ? nonfinite : 0u;
            }
            const uint64_t e = sea_hash_entity(r.t0[k], jit_hash_words<F, NWORDS>(r.w[k]));
            hx ^= has ? e : 0ULL;
        }
        const unsigned full = 0xffffffffu;
        const uint32_t lo = __reduce_xor_sync(full, uint32_t(hx)), hi = __reduce_xor_sync(full, uint32_t(hx >> 32));
        if (lane == 0) { atomicXor(&a[2 * hs.slot], lo); atomicXor(&a[2 * hs.slot + 1], hi); }
        jit_hash_columns<C + 1>(r, a, lane, bad);
    }
}

// A work item's rows: which tile and which rows of it the thread owns.  load / store move the register copy from / to an
// image; advance and checksum are the one definition of what an ADVANCE and a SAVE do on the generated kernel, which
// k_generic_jit, k_generic_jit_batch and the replay entry points all run.
struct JitItem {
    static constexpr int B = kJitItemRows / kJitRows;  // threads per work item
    static constexpr uint32_t kTileBytes = kTileRows * (4u * kJitWords + 1u);
    static constexpr uint32_t kAliveOff = uint32_t(kJitWords) * kPlaneBytes;  // the mask bytes follow the word planes inside a tile
    uint32_t tile, sub_row0;  // first row of the thread inside the tile
    size_t tile_off;
    unsigned long long row0;

    __device__ __forceinline__ JitItem(unsigned long long order_base, uint32_t item, uint32_t tid) {
        tile = item / uint32_t(kJitSubs);
        sub_row0 = (item % uint32_t(kJitSubs)) * uint32_t(kJitItemRows) + tid;
        tile_off = size_t(tile) * kTileBytes;
        row0 = order_base + size_t(tile) * kTileRows + sub_row0;
    }
    __device__ __forceinline__ void load(JitRows& r, const uint8_t* img, uint32_t n_rows_src) const {
        const uint8_t* t = img + tile_off;
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) {
            const uint32_t row = sub_row0 + k * B;
#pragma unroll
            for (int j = 0; j < kJitWords; ++j) r.w[k][j] = __ldcg(reinterpret_cast<const uint32_t*>(t + size_t(j) * kPlaneBytes + size_t(row) * 4u));
            const uint32_t mm = __ldcg(t + kAliveOff + row);  // .cg: L2 only — overlapping grids share an SM's L1 without a kernel boundary in between
            r.m[k] = (tile * kTileRows + row < n_rows_src) ? mm : 0u;  // rows the image never contained come back dead
        }
    }
    __device__ __forceinline__ void store(const JitRows& r, uint8_t* img) const {
        uint8_t* t = img + tile_off;
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) {
            const uint32_t row = sub_row0 + k * B;
#pragma unroll
            for (int j = 0; j < kJitWords; ++j) *reinterpret_cast<uint32_t*>(t + size_t(j) * kPlaneBytes + size_t(row) * 4u) = r.w[k][j];
            t[kAliveOff + row] = uint8_t(r.m[k]);
        }
    }
    __device__ __forceinline__ void order_lanes(JitRows& r) const {
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) r.t0[k] = sea_order_lane(row0 + uint32_t(k * B));
    }
    // `spawn_vals` / `spawn_ttl`: what an OPF_SPAWN ADVANCE writes into its newborn rows (GenericParams)
    template <int SPAWN = kJitSpawn>  // a template, so that a registration without spawn_particles discards the spawn code
    __device__ __forceinline__ void advance(JitRows& r, const Op& op, const float2* spawn_vals, unsigned long long spawn_ttl) const {
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) r.kill[k] = false;
        jit_run_systems<0>(r, op, row0, B);
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) r.m[k] = r.kill[k] ? 0u : r.m[k];  // despawn commands: after the last system
        if constexpr (SPAWN >= 0) {
            if (op.flags & OPF_SPAWN) {  // spawn_particles' Commands: rows [first, first + count) are born after the despawns
                constexpr SysSpec sy = kJitSys[SPAWN];
#pragma unroll
                for (int k = 0; k < kJitRows; ++k) {
                    const uint32_t born = tile * kTileRows + sub_row0 + k * B - op.image_off256;  // index among the spawned rows
                    if (born < op.save_index) {
                        spawn_row(sy, [&](int kk, uint32_t plane) -> uint32_t& { return r.w[kk][plane]; }, k, kJitWords,
                                  spawn_vals[op.call_count + born], spawn_ttl);
                        r.m[k] = 1u;
                    }
                }
            }
        }
    }
    // a SAVE's checksum of the register copy into the shared accumulators `a` of its save (kAccStride pairs of u32)
    __device__ __forceinline__ static void checksum(const JitRows& r, unsigned int* a, uint32_t lane) {
        uint32_t n_alive = 0, bad = 0;
#pragma unroll
        for (int k = 0; k < kJitRows; ++k) n_alive += r.m[k] & 1u;
        jit_hash_columns<0>(r, a, lane, bad);
        const unsigned full = 0xffffffffu;
        const uint32_t cnt = __reduce_add_sync(full, n_alive);
        const uint32_t anybad = __reduce_or_sync(full, bad);
        if (lane == 0) { atomicAdd(&a[12], cnt); if (anybad) atomicOr(&a[14], 1u); }
    }
};

// One work item of a request vector: the rows' first read from `first_img`, the vector's ops (LOAD, ADVANCE, SAVE with its
// hash into the save's shared accumulators `s_acc`) and the live store.  k_generic_jit and k_generic_jit_batch both run
// it.  `op_at(i)` is op i of the vector.
template <class OpAt>
__device__ __forceinline__ void jit_run_item(uint8_t* arena, unsigned long long order_base, uint32_t flags, uint32_t n_ops, OpAt op_at,
                                             const uint8_t* first_img, uint32_t first_rows, uint32_t item, unsigned int* s_acc,
                                             uint32_t tid, uint32_t lane, const float2* spawn_vals, unsigned long long spawn_ttl) {
    const JitItem it(order_base, item, tid);
    JitRows r;
    it.load(r, first_img, first_rows);
    it.order_lanes(r);
    for (uint32_t i = (flags & PF_READ_LIVE) ? 0u : 1u; i < n_ops; ++i) {
        const Op& op = op_at(i);
        if (op.kind == OP_ADVANCE) {
            it.advance(r, op, spawn_vals, spawn_ttl);
        } else if (op.kind == OP_SAVE) {
            if (!(op.flags & OPF_NO_STORE)) it.store(r, arena + (size_t(op.image_off256) << 8));
            JitItem::checksum(r, &s_acc[op.save_index * kAccStride * 2], lane);
        } else {  // OP_LOAD
            it.load(r, arena + (size_t(op.image_off256) << 8), op.n_rows);
        }
    }
    if (flags & PF_WRITE_LIVE_ACTIVE) it.store(r, arena);
}

// Shared accumulators of `n_saves` saves folded into global ones: XOR for the column words, add for the active rows,
// OR for the flags
__device__ __forceinline__ void jit_fold_acc(unsigned long long* accum, const unsigned int* s_acc, uint32_t n_saves, uint32_t tid) {
    constexpr int B = kJitItemRows / kJitRows;
    for (uint32_t i = tid; i < n_saves * kAccStride; i += B) {
        unsigned long long v = (unsigned long long)s_acc[2 * i] | ((unsigned long long)s_acc[2 * i + 1] << 32);
        const uint32_t c = i % kAccStride;
        if (v) {
            if (c == 6) atomicAdd(&accum[i], v);
            else if (c == 7) atomicOr(&accum[i], v);
            else atomicXor(&accum[i], v);
        }
    }
}

// The end of a block: its shared accumulators folded into the vector's `accum`; the block that completes the vector's
// `n_blocks`-th ticket then publishes the results as self-validating pairs plus the completion pair (k_particles_program's
// protocol) and re-arms the ticket for the vector's next launch.
__device__ __forceinline__ void jit_fold_publish(unsigned long long* accum, unsigned int* ticket, unsigned long long* out,
                                                 unsigned long long seq, uint32_t n_saves, uint32_t n_blocks, const unsigned int* s_acc,
                                                 unsigned int& s_last, unsigned long long* trace, uint32_t tid) {
    constexpr int B = kJitItemRows / kJitRows;
    __syncthreads();
    jit_fold_acc(accum, s_acc, n_saves, tid);
    __threadfence();
    __syncthreads();
    if (trace && tid == 0) atomicMax(&trace[1], globaltimer_ns());
    if (tid == 0) s_last = (atomicAdd(ticket, 1u) == n_blocks - 1u);
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (uint32_t i = tid; i < n_saves * kAccStride; i += B)
            publish_pair(out, i, atomicExch(&accum[i], 0ULL), seq);
        if (tid == 0) publish_pair(out, kSeqIndex, seq, seq);
        __syncthreads();
        if (tid == 0) {
            ticket[0] = 0u;
            ticket[1] = 0u;
            if (trace) trace[2] = globaltimer_ns();
        }
    }
}

extern "C" __global__ void __launch_bounds__(BGR_JIT_ITEM_ROWS / BGR_JIT_ROWS, BGR_JIT_MINB) k_generic_jit(const __grid_constant__ GenericParams p) {
    constexpr int B = kJitItemRows / kJitRows;  // threads per work item
    __shared__ unsigned int s_acc[kMaxSaves * kAccStride * 2];
    __shared__ uint32_t s_next;
    __shared__ unsigned int s_last;

    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    // Overlap of consecutive request vectors (bgr_submit_requests with others un-collected): work item i of tick k+1 only
    // depends on work item i of tick k.  A signalling launch lets the next one be scheduled as its own blocks retire
    // (griddepcontrol.launch_dependents); a waiting launch was started with programmatic stream serialisation, skips the
    // grid-level wait and instead waits per item for item_done[i] >= wait_seq.  Both grids are at most one wave of resident
    // blocks and every block of the earlier grid has started before the first block of the later one does, so the spin
    // cannot starve what it waits for.  (k_particles_program's protocol, DESIGN.md "Overlapping consecutive ticks".)
    const bool signal_items = (p.flags & PF_TILE_SIGNAL) != 0u, wait_items = (p.flags & PF_TILE_WAIT) != 0u;
    if (signal_items || wait_items) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (p.trace && tid == 0) atomicMin(&p.trace[0], globaltimer_ns());
    for (uint32_t i = tid; i < p.n_saves * kAccStride * 2; i += B) s_acc[i] = 0u;
    if (!wait_items) asm volatile("griddepcontrol.wait;" ::: "memory");  // a no-op unless launched as a programmatic dependent
    __syncthreads();

    const uint8_t* first_img = p.arena + ((p.flags & PF_READ_LIVE) ? size_t(0) : (size_t(p.ops[0].image_off256) << 8));
    const uint32_t first_rows = (p.flags & PF_READ_LIVE) ? p.live_rows : p.ops[0].n_rows;

    const uint32_t n_items = p.n_tiles * uint32_t(kJitSubs);
    for (uint32_t item = blockIdx.x; item < n_items;) {
        __syncthreads();  // every thread has read the previous s_next
        if (tid == 0) {
            s_next = gridDim.x + atomicAdd(&p.ticket[1], 1u);
            if (wait_items && item < p.wait_items)
                while (int32_t(ld_acquire_gpu(&p.item_done[item]) - p.wait_seq) < 0) {}  // the previous tick's stores of this item are visible
        }
        __syncthreads();
        const uint32_t next_item = s_next;
        jit_run_item(p.arena, p.order_base, p.flags, p.n_ops, [&](uint32_t i) -> const Op& { return p.ops[i]; }, first_img, first_rows,
                     item, s_acc, tid, lane, p.spawn_vals, p.spawn_ttl);
        if (signal_items) {  // every thread's stores of this item are visible at gpu scope, then one release store announces it
            __threadfence();
            __syncthreads();
            if (tid == 0) st_release_gpu(&p.item_done[item], p.done_seq);
        }
        item = next_item;
    }
    jit_fold_publish(p.accum, p.ticket, p.out, p.seq, p.n_saves, gridDim.x, s_acc, s_last, p.trace, tid);
}

// The request vectors of many engines with this registration in ONE launch (bgr_batch_handle_requests).  Block b runs
// one work item of one world: the world whose first block (JitWorld::item0, a prefix of the worlds' item counts) is the
// last one <= b.  Each world keeps k_generic_jit's completion protocol on its own accumulators, ticket and result block,
// with its item count in place of gridDim.x.  No dynamic claiming, no overlap of consecutive launches (PF_TILE_SIGNAL /
// PF_TILE_WAIT) and no trace rows.
extern "C" __global__ void __launch_bounds__(BGR_JIT_ITEM_ROWS / BGR_JIT_ROWS, BGR_JIT_MINB)
    k_generic_jit_batch(const JitWorld* __restrict__ worlds, uint32_t n_worlds, const Op* __restrict__ ops) {
    constexpr int B = kJitItemRows / kJitRows;
    __shared__ unsigned int s_acc[kMaxSaves * kAccStride * 2];
    __shared__ unsigned int s_last;
    const uint32_t tid = threadIdx.x, lane = tid & 31u;

    uint32_t lo = 0, hi = n_worlds;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) / 2u;
        if (worlds[mid].item0 <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    const JitWorld w = worlds[lo];
    for (uint32_t i = tid; i < w.n_saves * kAccStride * 2; i += B) s_acc[i] = 0u;
    __syncthreads();

    const Op* wops = ops + w.ops_off;
    const uint8_t* first_img = w.arena + ((w.flags & PF_READ_LIVE) ? size_t(0) : (size_t(wops[0].image_off256) << 8));
    const uint32_t first_rows = (w.flags & PF_READ_LIVE) ? w.live_rows : wops[0].n_rows;
    jit_run_item(w.arena, w.order_base, w.flags, w.n_ops, [&](uint32_t i) -> const Op& { return wops[i]; }, first_img, first_rows,
                 blockIdx.x - w.item0, s_acc, tid, lane, w.spawn_vals, w.spawn_ttl);
    jit_fold_publish(w.accum, w.ticket, w.out, w.seq, w.n_saves, w.n_tiles * uint32_t(kJitSubs), s_acc, s_last, nullptr, tid);
}

// A recorded input log through many worlds in ONE launch (bgr_replay, bgr_batch_replay).  Block b runs one work item of
// one world (the binary search of k_generic_jit_batch) through every frame [j0, j1) of the world's log: its rows are
// read from the live image once, stay in registers, and are written back once.  Each frame's ADVANCE op is derived
// on the device (replay_op) from the frame index, the input bytes and the spawn prefix, which the block stages into
// shared memory kReplayChunk frames at a time.  A checksum frame hashes the registers into a window of kReplayWindow
// shared accumulators; a full window (and the last one) is folded into the world's acc[point][kAccStride] with one
// global atomic per non-zero word.  No barrier runs on frames that are neither checksum points nor chunk starts.
// k_generic_jit_replay_kf also stores the registers at each keyframe frame into the world's keyframe staging (one plain
// store per row and word, no barrier, no extra read); k_generic_jit_replay_trace writes the change-feed record of each
// traced row at each trace sample frame, from the registers too.  The three entry points are this one body, STORES
// selecting the stores.
constexpr uint32_t kReplayChunk = 256;  // frames of the log per staging step
constexpr uint32_t kReplayWindow = 32;  // checksum points per shared window
enum ReplayStores : int { kReplayPlain = 0, kReplayKeyframes = 1, kReplayTraces = 2 };

// The trace records of the thread's rows in [first_row, first_row + n_rows) into one sample's staging `img`: u32 row,
// u32 state (bit 0 the row exists, bit 1 + k field k is present), then the field words, zero where not present.  The
// words come from the register copy; the plane of each is a literal (the loop over kJitWords is unrolled) and the run-time
// map only says which record words it goes to, so the rows stay in registers.
__device__ __forceinline__ void jit_trace_store(const JitRows& r, const JitItem& it, uint8_t* img, uint32_t first_row,
                                                uint32_t n_rows, const TraceMap& map) {
#pragma unroll
    for (int k = 0; k < kJitRows; ++k) {
        const uint32_t row = it.tile * kTileRows + it.sub_row0 + uint32_t(k * JitItem::B);
        const uint32_t i = row - first_row;
        if (i >= n_rows) continue;
        uint32_t* rec = reinterpret_cast<uint32_t*>(img) + size_t(i) * map.record_words;
        const uint32_t m = r.m[k];
        uint32_t state = m & 1u;
        for (uint32_t f = 0; f < map.n_fields; ++f) state |= row_matches(m, map.field_absent[f]) ? 2u << f : 0u;
        rec[0] = row;
        rec[1] = state;
#pragma unroll
        for (int j = 0; j < kJitWords; ++j) {
            const uint32_t v = row_matches(m, map.word_absent[j]) ? r.w[k][j] : 0u;
            for (uint32_t s = map.word_first[j]; s < map.word_first[j + 1]; ++s) rec[2u + map.slot[s]] = v;
        }
    }
}

template <int STORES>
__device__ __forceinline__ void jit_replay(const ReplayWorld* __restrict__ worlds, uint32_t n_worlds,
                                           const ReplayKeyframes* __restrict__ kfs, const ReplayTrace* __restrict__ trs,
                                           const TraceMap* map) {
    constexpr int B = kJitItemRows / kJitRows;
    __shared__ unsigned int s_acc[kReplayWindow * kAccStride * 2];
    __shared__ uint8_t s_in[kReplayChunk * 8];
    __shared__ uint32_t s_pre[kReplayChunk];
    __shared__ Op s_op[B];
    const uint32_t tid = threadIdx.x, lane = tid & 31u;

    uint32_t lo = 0, hi = n_worlds;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) / 2u;
        if (worlds[mid].item0 <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    const ReplayWorld& w = worlds[lo];
    const ReplayClock c = w.c;
    const uint32_t j1 = w.j1, np = c.n_players, interval = w.interval;
    for (uint32_t i = tid; i < kReplayWindow * kAccStride * 2; i += B) s_acc[i] = 0u;

    const JitItem it(w.order_base, blockIdx.x - w.item0, tid);
    JitRows r;
    it.load(r, w.arena, w.live_rows);
    it.order_lanes(r);

    unsigned long long next_point = w.next_point;
    uint32_t point = 0, win0 = 0;  // checksum points seen, first point of the shared window
    unsigned long long next_kf = ~0ULL;
    uint8_t* kf_img = nullptr;
    if constexpr (STORES == kReplayKeyframes) { next_kf = kfs[lo].first; kf_img = kfs[lo].staging; }
    unsigned long long next_tr = ~0ULL;
    uint8_t* tr_img = nullptr;
    bool tr_rows = false;  // the work item holds a traced row: uniform over the block
    if constexpr (STORES == kReplayTraces) {
        next_tr = trs[lo].first;
        tr_img = trs[lo].staging;
        const uint32_t item = blockIdx.x - w.item0;
        const uint32_t r0 = (item / uint32_t(kJitSubs)) * kTileRows + (item % uint32_t(kJitSubs)) * uint32_t(kJitItemRows);
        tr_rows = r0 < trs[lo].first_row + trs[lo].n_rows && trs[lo].first_row < r0 + uint32_t(kJitItemRows);
    }
    auto flush = [&](uint32_t n) {
        __syncthreads();
        jit_fold_acc(w.acc + size_t(win0) * kAccStride, s_acc, n, tid);
        __syncthreads();
        for (uint32_t i = tid; i < n * kAccStride * 2; i += B) s_acc[i] = 0u;
        __syncthreads();
    };
    for (uint32_t j = w.j0, chunk0 = w.j0; j < j1; ++j) {
        if (j == chunk0 || j - chunk0 == kReplayChunk) {  // the log's next kReplayChunk frames into shared memory
            chunk0 = j;
            const uint32_t n = min(kReplayChunk, j1 - j);
            __syncthreads();  // every thread is done with the previous chunk (and the accumulators are zeroed)
            for (uint32_t i = tid; i < n * np; i += B) s_in[i] = w.inputs[size_t(j) * np + i];
            for (uint32_t i = tid; i < n; i += B) s_pre[i] = w.prefix ? w.prefix[j + i] : 0u;
            __syncthreads();
        }
        const uint32_t q = j - chunk0;
        if (j == next_point) {  // SaveGameState{f0 + j} with no store: the checksum of the registers
            if (point - win0 == kReplayWindow) { flush(kReplayWindow); win0 = point; }
            JitItem::checksum(r, &s_acc[(point - win0) * kAccStride * 2], lane);
            point += 1;
            next_point += interval;
        }
        if constexpr (STORES == kReplayKeyframes) {
            if (j == next_kf) {  // keyframe f0 + j: the registers as they stand before the frame is advanced
                it.store(r, kf_img);
                kf_img += kfs[lo].stride;
                next_kf += kfs[lo].interval;
            }
        }
        if constexpr (STORES == kReplayTraces) {
            if (j == next_tr) {  // trace sample f0 + j: the traced rows as they stand before the frame is advanced
                if (tr_rows) jit_trace_store(r, it, tr_img, trs[lo].first_row, trs[lo].n_rows, *map);
                tr_img += trs[lo].stride;
                next_tr += trs[lo].interval;
            }
        }
        Op& op = s_op[tid];  // the thread's own copy: box_move indexes its inputs by row, which would put a local one on the stack
        op = replay_op(c, j, &s_in[q * np], s_pre[q]);
        it.advance(r, op, w.spawn_vals, w.spawn_ttl);
    }
    if (point > win0) flush(point - win0);
    it.store(r, w.arena);
}

extern "C" __global__ void __launch_bounds__(BGR_JIT_ITEM_ROWS / BGR_JIT_ROWS, BGR_JIT_MINB)
    k_generic_jit_replay(const ReplayWorld* __restrict__ worlds, uint32_t n_worlds) {
    jit_replay<kReplayPlain>(worlds, n_worlds, nullptr, nullptr, nullptr);
}

// bgr_replay_keyframes, bgr_batch_replay_keyframes: kfs[i] belongs to worlds[i]
extern "C" __global__ void __launch_bounds__(BGR_JIT_ITEM_ROWS / BGR_JIT_ROWS, BGR_JIT_MINB)
    k_generic_jit_replay_kf(const ReplayWorld* __restrict__ worlds, uint32_t n_worlds, const ReplayKeyframes* __restrict__ kfs) {
    jit_replay<kReplayKeyframes>(worlds, n_worlds, kfs, nullptr, nullptr);
}

// bgr_replay_trace, bgr_batch_replay_trace: trs[i] belongs to worlds[i]; one field map for the launch (a batched call
// has one field list)
extern "C" __global__ void __launch_bounds__(BGR_JIT_ITEM_ROWS / BGR_JIT_ROWS, BGR_JIT_MINB)
    k_generic_jit_replay_trace(const ReplayWorld* __restrict__ worlds, uint32_t n_worlds, const ReplayTrace* __restrict__ trs,
                               const __grid_constant__ TraceMap map) {
    jit_replay<kReplayTraces>(worlds, n_worlds, nullptr, trs, &map);
}

}  // namespace bgr
