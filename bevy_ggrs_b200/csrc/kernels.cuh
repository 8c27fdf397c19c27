// CUDA kernels of the rollback engine (sm_90a).  HBM-bound integer / f32 streaming work:
// no tensor cores (there is no dense contraction on this path); what matters is coalescing,
// vector accesses, TMA bulk copies for bytes nobody computes on, instruction count per byte
// and ONE launch per request vector.
//
// Data layout (DESIGN.md "Data layout in HBM") — TILE-PLANAR images:
//   an image is a sequence of tiles of kTileRows = 512 rows; inside a tile every registered
//   column is split into 4-byte word planes, followed by the 1-byte-per-row alive plane:
//       tile = [plane 0: 512 words | plane 1 | ... | plane W-1 | alive: 512 bytes]      (512*(4W+1) bytes)
//       image = tile 0 | tile 1 | ...
//   * every warp access is a contiguous 128..512 B run (coalesced) whatever the element size,
//   * all planes of a tile sit within 64 KB, so a thread reaches them with ONE base pointer plus
//     compile-time immediates (the first profile of the plane-major layout spent ~4 address
//     instructions per store),
//   * a whole tile — or any run of adjacent planes — is ONE contiguous chunk for cp.async.bulk (TMA),
//   * an image is flat: save/load of any schema is a flat copy of n_tiles * tile_bytes.
// Image 0 is the live world, image s+1 is snapshot slot s of the ring.  A row is one rollback
// entity; its RollbackOrdered index is order_base + row (rollback.rs:66-83).
//
// Reference semantics implemented here (paths relative to the upstream repo):
//   save  : component_snapshot.rs:66-84   (copy every registered column into the frame's snapshot)
//   load  : component_snapshot.rs:95-123  (overwrite live columns from the snapshot; entity.rs:55-99 -> alive plane)
//   cksum : component_checksum.rs:67-108, entity_checksum.rs:29-52 (XOR of per-entity seahashes; count of live rows)
//   systems: examples/stress_tests/particles.rs:272-289 (update_particles, despawn_particles)
#pragma once
#ifdef __CUDACC_RTC__  // NVRTC (the engine's run-time specialisation, generic_program_jit.cuh): no host headers
#include "rtc_prelude.cuh"
#else
#include <cuda_runtime.h>
#include <cstdint>
#endif

#include "seahash.cuh"

namespace bgr {

#ifndef BGR_TILE_ROWS
#define BGR_TILE_ROWS 512
#endif
constexpr uint32_t kTileRows = BGR_TILE_ROWS;
constexpr uint32_t kPlaneBytes = kTileRows * 4;  // one word plane inside a tile
constexpr int kMaxOps = 80;       // == BGR_MAX_REQUESTS
constexpr int kMaxSaves = 40;
constexpr int kMaxPassive = 64;   // word planes that no compiled system touches (per-thread fallback)
constexpr int kMaxRuns = 8;       // runs of adjacent passive planes (TMA path)
constexpr int kAccStride = 8;     // u64 per save: [0..5] column xors, [6] active rows, [7] flags
// Result block (host-mapped, one per buffer): kResultPairs PAIRS of u64.  Result word i is published as
// (v, v ^ result_tag(seq, i)); pair kSeqIndex is the completion pair (v = seq).  The host accepts a word when the two
// halves XOR to the tag of the sequence number it is waiting for: every word validates itself, so the GPU needs no
// system-scope fence and no separate flag store behind the data (that round trip was 3.2 us of every synchronous call,
// tools/launch_latency.cu), a torn or stale pair simply fails the test and is polled again.
constexpr int kSeqIndex = kMaxSaves * kAccStride;   // index of the completion pair
constexpr int kResultPairs = kSeqIndex + 1;
constexpr int kResultStride = 2 * kResultPairs + 6;  // u64 words per result block
__host__ __device__ inline unsigned long long result_tag(unsigned long long seq, uint32_t i) {
    return ((seq * 0x9E3779B97F4A7C15ULL) ^ ((unsigned long long)(i + 1) * 0xD6E8FEB86659FD93ULL)) | 1ULL;  // never 0: zeroed memory is invalid
}

__host__ __device__ inline uint32_t tile_bytes_of(uint32_t words) { return kTileRows * (4u * words + 1u); }
__host__ __device__ inline size_t word_offset(uint32_t words, uint32_t row, uint32_t plane) {
    return size_t(row / kTileRows) * tile_bytes_of(words) + size_t(plane) * kPlaneBytes + size_t(row % kTileRows) * 4u;
}
// The byte per row behind the word planes: bit 0 = the entity exists (Rollback marker alive); bit 1+k = optional
// column k is ABSENT from this entity (component_snapshot.rs:106-115: a column registered with
// BGR_STRATEGY_OPTIONAL can be removed from / inserted into single entities).  Spawning writes 1: alive, everything
// present.  A row takes part in a query over columns whose absent bits are `need` iff (m & (1 | need)) == 1.
__host__ __device__ inline bool row_matches(uint32_t m, uint32_t need) { return (m & (1u | need)) == 1u; }
__host__ __device__ inline size_t alive_offset(uint32_t words, uint32_t row) {
    return size_t(row / kTileRows) * tile_bytes_of(words) + size_t(words) * kPlaneBytes + size_t(row % kTileRows);
}

enum OpKind : uint32_t { OP_SAVE = 0, OP_LOAD = 1, OP_ADVANCE = 2 };
enum OpFlags : uint32_t {
    OPF_NO_STORE = 1u,  // SAVE with ring depth 0: checksum only
    OPF_SPAWN = 2u,     // ADVANCE: spawn_particles fired; rows [spawn_first, spawn_first+spawn_count) are born at the end of the frame
    // SAVE: the slot already holds the current content of the passive planes (content versions, engine.cu HostState).
    // Only this bundle kernel honours it; every other kernel stores whole images, which keeps the versions true.  A
    // kernel that stores partial images must keep versions of its own.
    OPF_SKIP_PASSIVE = 4u,
    // bits 8..11 of an ADVANCE op's flags: number of players (PlayerInputs<T>.len())
};

struct Op {
    uint32_t kind;
    uint32_t image_off256;  // LOAD/SAVE: byte offset of the image read / written, in 256-byte units.  ADVANCE+SPAWN: first spawned row
    uint32_t dt_bits;       // ADVANCE: Time<GgrsTime>::delta_secs as f32 bits (time.rs:63-76)
    uint32_t fr_bits;       // ADVANCE: 0.0018f.powf(dt) as f32 bits (box_game.rs:188-193), from the host's C library powf
    uint32_t n_rows;       // rows that exist while this op runs (RollbackOrdered::len())
    uint32_t save_index;    // SAVE: which accumulator row.  ADVANCE+SPAWN: number of spawned rows
    uint32_t flags;
    uint32_t call_count;    // ADVANCE: value of the un-rolled-back host counter (test system).  ADVANCE+SPAWN: offset into spawn_vals
    uint8_t inputs[8];      // ADVANCE: PlayerInputs<T>.0[handle].0 for every handle (u8, BGR_MAX_PLAYERS)
};
static_assert(sizeof(Op) == 40, "Op layout");

enum ProgFlags : uint32_t {
    PF_READ_LIVE = 1u,           // program does not start with LOAD: initial state comes from image 0
    PF_WRITE_LIVE_ACTIVE = 2u,   // program contains LOAD or ADVANCE: final active planes go to image 0
    PF_WRITE_LIVE_PASSIVE = 4u,  // program contains LOAD: final passive planes go to image 0
    PF_PASSIVE_TMA = 8u,         // at most one LOAD and it is ops[0]: passive planes move by TMA bulk copies
    PF_CK_T = 16u, PF_CK_V = 32u, PF_FIN_T = 64u, PF_FIN_V = 128u,  // which bundle columns are checksummed / assert finite
    PF_DYNAMIC_TILES = 256u,     // tiles handed out by an atomic counter instead of a static stride
    PF_PREFETCH_NEXT = 512u,     // warp 0 pulls the next tile's active planes into L2 while this tile computes
    PF_TILE_SIGNAL = 1024u,      // announce each block's FIRST tile in tile_done[] as soon as its stores are visible, and the
                                 // whole launch in *grid_done: what the next launch's first wave needs to start early
    PF_PASSIVE_EARLY = 8192u,    // single-wave grid: issue the passive planes' bulk stores at the top of a tile
    PF_TILE_WAIT = 2048u,        // the previous launch on the stream was a PF_TILE_SIGNAL launch: start without waiting for
                                 // its grid (no griddepcontrol.wait) and wait per tile for tile_done[tile] or grid_done >=
                                 // wait_seq instead.  Tile i of tick k+1 only depends on tile i of tick k, so this grid's
                                 // first wave runs in the previous grid's tail instead of after it.
};

struct PassiveRun { uint32_t off, bytes; };  // inside a tile; adjacent passive planes form one run

struct ProgramParams {
    uint8_t* arena;
    unsigned long long order_base;
    unsigned long long* accum;  // device [kMaxSaves][kAccStride]
    unsigned long long* out;    // host-mapped [kMaxSaves][kAccStride]
    unsigned int* ticket;       // [0] block-completion ticket, [1] dynamic tile counter
    const float2* spawn_vals;   // (vx, vy) of every particle spawned by this program (host-mapped), particles.rs:265
    unsigned long long seq;     // sequence number of this launch: tags every published result pair (result_tag)
    unsigned long long* trace;  // nullptr, or this launch's row of the launch trace: [0] min block start, [1] max block end, [2] results published (globaltimer ns)
    uint32_t words, tile_bytes, n_ops, n_saves;
    uint32_t n_tiles;              // this launch covers tiles [0, n_tiles)
    unsigned int* tile_done;       // [tiles] sequence number of the last PF_TILE_SIGNAL launch that finished the tile
    unsigned int* tile_cnt;        // [tiles] warps of the current launch that finished the tile
    unsigned int* grid_done;       // sequence number of the last PF_TILE_SIGNAL launch that completed entirely
    uint32_t done_seq, wait_seq, wait_tiles;  // PF_TILE_WAIT: tiles < wait_tiles wait for tile_done >= wait_seq
    uint32_t live_rows, flags;
    uint32_t t_off, v_off, l_off, alive_off;  // byte offsets inside a tile of Transform / Velocity / Ttl word 0 / alive plane
    uint32_t ck_t_slot, ck_v_slot;            // accumulator column of each checksummed type
    uint32_t n_runs, passive_bytes;           // TMA path
    uint32_t n_passive;                       // per-thread fallback path
    uint32_t spawn_ttl_lo, spawn_ttl_hi;      // Ttl of a spawned particle (fps * 5, particles.rs:260)
    // MODE 2 (per-entity presence, BGR_STRATEGY_OPTIONAL): absent bits (of the row's mask byte) that take a row out of
    // update_particles' query (Transform | Velocity), despawn_particles' (Ttl) and the two checksum queries
    uint32_t need_tv, need_l, need_t, need_v;
    // A grid that starts on an idle GPU has every block in the same phase of the same op (all load, then all hash, then
    // all store): HBM idles while the ALUs work and vice versa until latency noise has dephased them.  Delaying the
    // second / third resident block of every SM by a fraction of one frame's time starts them out of phase.
    uint32_t stagger_ns, stagger_div;
    PassiveRun runs[kMaxRuns];
    uint16_t passive[kMaxPassive];
    uint32_t passive_template[kMaxPassive];   // value of each passive word in a freshly spawned row (Transform::default())
    Op ops[kMaxOps];
};
static_assert(sizeof(ProgramParams) <= 4000, "kernel parameter block must fit 4 KB");

// ---------------------------------------------------------------------------------------------
// vector access helpers: VEC consecutive rows of one word plane = one 4*VEC byte access
// ---------------------------------------------------------------------------------------------
template <int VEC> __device__ __forceinline__ void vec_load(const uint8_t* p, uint32_t (&r)[VEC]);
template <> __device__ __forceinline__ void vec_load<2>(const uint8_t* p, uint32_t (&r)[2]) { uint2 v = __ldcs(reinterpret_cast<const uint2*>(p)); r[0] = v.x; r[1] = v.y; }

template <int VEC> __device__ __forceinline__ void vec_store(uint8_t* p, const uint32_t (&r)[VEC]);
template <> __device__ __forceinline__ void vec_store<2>(uint8_t* p, const uint32_t (&r)[2]) { __stcs(reinterpret_cast<uint2*>(p), make_uint2(r[0], r[1])); }

// alive plane: VEC bytes packed little-endian into one register
template <int VEC> __device__ __forceinline__ uint32_t alive_load(const uint8_t* p);
template <> __device__ __forceinline__ uint32_t alive_load<2>(const uint8_t* p) { return __ldcs(reinterpret_cast<const unsigned short*>(p)); }
template <int VEC> __device__ __forceinline__ void alive_store(uint8_t* p, uint32_t a);
template <> __device__ __forceinline__ void alive_store<2>(uint8_t* p, uint32_t a) { __stcs(reinterpret_cast<unsigned short*>(p), (unsigned short)a); }

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void publish_pair(unsigned long long* out, uint32_t i, unsigned long long v, unsigned long long seq) {
    reinterpret_cast<ulonglong2*>(out)[i] = make_ulonglong2(v, v ^ result_tag(seq, i));  // one 16-byte store
}
__device__ __forceinline__ uint32_t f32_bits_nonfinite(uint32_t b) { return ((b & 0x7f800000u) == 0x7f800000u) ? 1u : 0u; }

// mask with byte j = 0x01 for every row (row0 + j) < n_rows
template <int VEC> __device__ __forceinline__ uint32_t rows_mask(uint32_t row0, uint32_t n_rows) {
    uint32_t m = 0;
#pragma unroll
    for (int j = 0; j < VEC; ++j) m |= (row0 + j < n_rows) ? (1u << (8 * j)) : 0u;
    return m;
}
// ... byte j = 0xFF: keeps the absent bits of the row's mask byte (per-entity presence)
template <int VEC> __device__ __forceinline__ uint32_t rows_mask_full(uint32_t row0, uint32_t n_rows) {
    uint32_t m = 0;
#pragma unroll
    for (int j = 0; j < VEC; ++j) m |= (row0 + j < n_rows) ? (0xFFu << (8 * j)) : 0u;
    return m;
}

// ---- TMA / mbarrier primitives (cp.async.bulk, SASS UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ uint32_t ld_acquire_gpu(const unsigned int* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned int* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// release / acquire fence at gpu scope (MEMBAR.ALL.GPU): __threadfence() is the sequentially-consistent one
// (MEMBAR.SC.GPU + ERRBAR + L1 invalidate), several times more expensive and not needed for a flag hand-off
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// update_particles (particles.rs:272-280) for one entity: every mul and add individually rounded
// (Rust/glam scalar Vec3, no FMA contraction); gravity = Vec3::NEG_Y * 200.0 = (0*200, -1*200, 0*200)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void particle_step(uint32_t& tx, uint32_t& ty, uint32_t& tz,
                                              uint32_t& vx, uint32_t& vy, uint32_t& vz, float dt) {
    const float gx = __fmul_rn(0.0f, 200.0f), gy = __fmul_rn(-1.0f, 200.0f), gz = __fmul_rn(0.0f, 200.0f);
    float fvx = __uint_as_float(vx), fvy = __uint_as_float(vy), fvz = __uint_as_float(vz);
    fvx = __fadd_rn(fvx, __fmul_rn(gx, dt));   // **velocity += gravity * time_step
    fvy = __fadd_rn(fvy, __fmul_rn(gy, dt));
    fvz = __fadd_rn(fvz, __fmul_rn(gz, dt));
    float ftx = __fadd_rn(__uint_as_float(tx), __fmul_rn(fvx, dt));  // translation += **velocity * time_step
    float fty = __fadd_rn(__uint_as_float(ty), __fmul_rn(fvy, dt));
    float ftz = __fadd_rn(__uint_as_float(tz), __fmul_rn(fvz, dt));
    vx = __float_as_uint(fvx); vy = __float_as_uint(fvy); vz = __float_as_uint(fvz);
    tx = __float_as_uint(ftx); ty = __float_as_uint(fty); tz = __float_as_uint(ftz);
}

// =============================================================================================
// THE fused kernel: interprets the whole request vector (Load / Advance / Save ...) for the
// particles bundle.  One launch per handle_requests; one tile (512 rows) per block iteration.
//   * active words (translation, velocity, ttl, alive) live in registers for the whole program:
//       LOAD    : read them from the snapshot image once
//       ADVANCE : update_particles + despawn_particles in registers (0 bytes)
//       SAVE    : stream them into the frame's slot and fold the per-entity seahashes of the
//                 checksummed columns: warp REDUX.XOR -> shared atomics -> one global atomic per
//                 block per (save, column) -> last block publishes to host-mapped memory
//       end     : write the live image once
//   * passive planes (rotation, scale, any registered column no compiled system writes) never
//     touch a register: one cp.async.bulk brings the tile's passive runs into shared memory and
//     one cp.async.bulk per SAVE (and one for the live image) streams them out again.
// Frames of one entity are sequentially dependent, so the frame loop is per thread; entities are
// independent, so the grid dimension is the entity dimension.
// Dead rows are advanced and hashed like live ones and masked at the fold: their bytes are not
// observable (a row only comes back to life through LOAD, which restores data and flag together).
// =============================================================================================
// MODE 0: checksum flags tested at run time; MODE 1: both columns checksummed with the finite assertion (the stress
// test's registration) — the flag tests fold away; MODE 2: MODE 0 + per-entity component presence: the row's mask
// byte carries absent bits (BGR_STRATEGY_OPTIONAL), every system and checksum applies the reference's query filter
// (`Query<(&RollbackId, &T)>`, component_checksum.rs:73-77; `Query<(&mut Transform, &mut Velocity)>`, particles.rs:273)
// per row, and Save / Load move the mask with the image (= the four-way match of component_snapshot.rs:99-115).
// Two rows per thread, 256 threads per tile, three resident blocks (768 threads) per SM: DESIGN.md "What a synchronous
// call costs" has the measurements against 1 and 4 rows per thread and the other launch-bounds tiers.
template <int MODE>
__global__ void __launch_bounds__(256, 3) k_particles_program(const __grid_constant__ ProgramParams p) {
    constexpr int VEC = 2, BLOCK = 256;  // rows per thread, threads per block (__launch_bounds__)
    static_assert(VEC * BLOCK == int(kTileRows), "a block iteration covers one tile");
    constexpr bool STATIC_CK = MODE == 1;
    constexpr bool OPT = MODE == 2;
    // STATIC_CK: both columns checksummed with the finite assertion (the stress test's registration) —
    // the flag tests fold away; otherwise they are warp-uniform runtime tests.
    const bool CKT = STATIC_CK ? true : (p.flags & PF_CK_T) != 0;
    const bool CKV = STATIC_CK ? true : (p.flags & PF_CK_V) != 0;
    const bool FINT = STATIC_CK ? true : (p.flags & PF_FIN_T) != 0;
    const bool FINV = STATIC_CK ? true : (p.flags & PF_FIN_V) != 0;
    extern __shared__ __align__(128) uint8_t s_passive[];  // 2 x passive_bytes (double buffer)
    __shared__ unsigned int s_acc[kMaxSaves * kAccStride * 2];  // 32-bit halves: native shared atomics, no CAS loop
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ unsigned int s_last;

    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    if (p.trace && tid == 0) atomicMin(&p.trace[0], globaltimer_ns());  // bgr_trace_enable: when did this launch's first block start
    // Programmatic dependent launch: let the NEXT request vector's kernel be launched and its blocks scheduled
    // into SM slots as this grid drains (hides launch latency and block ramp-up between back-to-back ticks) ...
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    for (uint32_t i = tid; i < p.n_saves * kAccStride * 2; i += BLOCK) s_acc[i] = 0u;
    const bool use_tma = (p.flags & PF_PASSIVE_TMA) && p.n_runs > 0;
    // the passive planes of a tile as bulk-copy chunks: whole runs of adjacent planes; f(offset inside the tile, bytes)
    auto for_each_passive_chunk = [&](auto&& f) {
        for (uint32_t r = 0; r < p.n_runs; ++r) f(p.runs[r].off, p.runs[r].bytes);
    };
    if (tid == 0 && use_tma) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    // ... while this grid touches no global memory before the previous grid has completed and flushed
    const bool tile_wait = (p.flags & PF_TILE_WAIT) != 0, tile_signal = (p.flags & PF_TILE_SIGNAL) != 0;
    if (!tile_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    if (p.stagger_ns) {
        const unsigned long long until = globaltimer_ns() + (unsigned long long)(blockIdx.x / p.stagger_div) * p.stagger_ns;
        while (globaltimer_ns() < until) __nanosleep(64);
    }

    // Dynamic tile hand-off WITHOUT a block barrier: at the top of a tile thread 0 claims the block's NEXT tile
    // from a global counter (late binding: one tile ahead, so the tail stays balanced) and publishes it a little
    // later — once the atomic has returned, hidden behind the tile's loads — through a 4-slot ring guarded by
    // full/empty mbarriers.  A fast warp never waits for a slow one (a per-tile __syncthreads cost 13 % of all
    // warp time in the round-1 profile).
    constexpr uint32_t kRing = 4;
    __shared__ uint32_t s_tile[kRing];
    __shared__ __align__(8) uint64_t s_full[kRing], s_empty[kRing];
    const bool dynamic = (p.flags & PF_DYNAMIC_TILES) != 0;
    if (dynamic) {
        if (tid == 0) {
            for (uint32_t k = 0; k < kRing; ++k) { mbar_init(&s_full[k], 1); mbar_init(&s_empty[k], BLOCK / 32); }
            fence_mbar_init();
        }
        __syncthreads();
    }
    // ring entry of the tile that iteration j (>= 1) runs: slot (j-1) % kRing, in its ((j-1) / kRing)-th use;
    // iteration 0 runs tile blockIdx.x and never enters the ring
    uint32_t claimed = 0;        // thread 0: tile claimed for iteration it + 1
    uint32_t it = 0;
    // PF_TILE_SIGNAL: a fence per announced tile stalls the warp until its stores are acknowledged (8 % when every tile
    // was announced), so only the first tile of each block is — the tiles the next grid's first wave starts with
    auto signal_tile = [&](uint32_t t) {
        if (use_tma && tid == 0) tma_wait_all();  // that tile's bulk stores have landed (not just released their buffer)
        fence_acq_rel_gpu();                      // every thread's stores are visible gpu-wide before its warp arrives
        __syncwarp();
        if (lane == 0) {
            if (atomicAdd(&p.tile_cnt[t], 1u) == kTileRows / (32 * VEC) - 1) {  // last warp to announce this tile
                p.tile_cnt[t] = 0u;
                fence_acq_rel_gpu();
                st_release_gpu(&p.tile_done[t], p.done_seq);
            }
        }
    };
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; ++it) {
        if (dynamic && tid == 0) claimed = gridDim.x + atomicAdd(&p.ticket[1], 1u);  // published after the loads below
        const uint32_t i0 = tid * VEC;  // first row of this thread inside the tile
        if (tile_wait && tile < p.wait_tiles) {
            // the previous tick's kernel may still be running: this tile's images are complete once it has signalled
            if (lane == 0)
                while (int32_t(ld_acquire_gpu(&p.tile_done[tile]) - p.wait_seq) < 0 &&
                       int32_t(ld_acquire_gpu(p.grid_done) - p.wait_seq) < 0) __nanosleep(100);
            __syncwarp();
            if (tid == 0) fence_proxy_async_global();  // ... also for the bulk (async-proxy) loads below
        }
        const size_t tile_off = size_t(tile) * p.tile_bytes;
        const uint32_t row0 = tile * kTileRows + i0;
        const size_t woff = tile_off + size_t(i0) * 4u;  // + plane offset (+ image offset) = address of this thread's words
        const size_t aoff = tile_off + p.alive_off + i0;

        // ---- passive planes, TMA path: issue the load of this tile's passive runs now ----
        const uint32_t buf = it & 1u;
        if (use_tma && tid == 0) {
            tma_wait_read<1>();  // the stores issued two tiles ago have finished reading this buffer
            const uint8_t* src = p.arena + ((p.flags & PF_READ_LIVE) ? size_t(0) : (size_t(p.ops[0].image_off256) << 8)) + tile_off;
            uint8_t* dst = s_passive + size_t(buf) * p.passive_bytes;
            mbar_arrive_expect_tx(&s_bar[buf], p.passive_bytes);
            uint32_t o = 0;
            for_each_passive_chunk([&](uint32_t off, uint32_t bytes) {
                tma_load_1d(dst + o, src + off, bytes, &s_bar[buf]);
                o += bytes;
            });
        }

        // ------------------------------ active words ------------------------------
        uint32_t tr[3][VEC], vl[3][VEC], tl[2][VEC];
        uint32_t alive = 0;

        auto load_active = [&](const uint8_t* img, uint32_t n_rows) {
            const uint8_t* pt = img + p.t_off + woff;
            const uint8_t* pv = img + p.v_off + woff;
            const uint8_t* pl = img + p.l_off + woff;
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_load<VEC>(pt + k * kPlaneBytes, tr[k]);
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_load<VEC>(pv + k * kPlaneBytes, vl[k]);
#pragma unroll
            for (int k = 0; k < 2; ++k) vec_load<VEC>(pl + k * kPlaneBytes, tl[k]);
            alive = alive_load<VEC>(img + aoff) & (OPT ? rows_mask_full<VEC>(row0, n_rows) : rows_mask<VEC>(row0, n_rows));
        };
        auto store_active = [&](uint8_t* img) {
            uint8_t* pt = img + p.t_off + woff;
            uint8_t* pv = img + p.v_off + woff;
            uint8_t* pl = img + p.l_off + woff;
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_store<VEC>(pt + k * kPlaneBytes, tr[k]);
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_store<VEC>(pv + k * kPlaneBytes, vl[k]);
#pragma unroll
            for (int k = 0; k < 2; ++k) vec_store<VEC>(pl + k * kPlaneBytes, tl[k]);
            alive_store<VEC>(img + aoff, alive);
        };

        if (p.flags & PF_READ_LIVE) load_active(p.arena, p.live_rows);
        else load_active(p.arena + (size_t(p.ops[0].image_off256) << 8), p.ops[0].n_rows);  // ops[0] is a LOAD

        // lane of the per-entity hash that only depends on the RollbackOrdered index
        uint64_t t0[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) t0[j] = sea_order_lane(p.order_base + row0 + j);

        if (dynamic && tid == 0) {  // publish the tile of iteration it + 1 (ring entry `it`)
            const uint32_t slot = it % kRing, use = it / kRing;
            if (use > 0) mbar_wait(&s_empty[slot], (use - 1) & 1u);  // every warp has read the previous occupant
            s_tile[slot] = claimed;
            mbar_arrive(&s_full[slot]);
        }
        if (dynamic && (p.flags & PF_PREFETCH_NEXT) && tid < 32) {
            // the next tile's first touch is a dependent DRAM read at the top of the tile (20 % of all stall samples in
            // the round-1 profile): pull its active planes (8 word planes + alive = 132 lines) into L2 now
            const uint32_t nxt = __shfl_sync(0xffffffffu, claimed, 0);
            if (nxt < p.n_tiles) {
                const uint8_t* img = p.arena + ((p.flags & PF_READ_LIVE) ? size_t(0) : (size_t(p.ops[0].image_off256) << 8)) + size_t(nxt) * p.tile_bytes;
                constexpr uint32_t kLines = kPlaneBytes / 128u, kAliveLines = (kTileRows + 127u) / 128u;  // per plane / alive plane of a tile
                for (uint32_t l = lane; l < 8u * kLines + kAliveLines; l += 32u) {
                    const uint32_t plane = l / kLines, line = l % kLines;
                    const size_t off = plane < 3 ? p.t_off + size_t(plane) * kPlaneBytes
                                     : plane < 6 ? p.v_off + size_t(plane - 3) * kPlaneBytes
                                     : plane < 8 ? p.l_off + size_t(plane - 6) * kPlaneBytes
                                                 : size_t(p.alive_off);
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(img + off + size_t(line) * 128u));
                }
            }
        }

        // ---- passive planes, TMA path: one bulk store per SAVE (+ live) out of the staged copy.  They depend on no frame.
        // Single-wave grids (small worlds, PF_PASSIVE_EARLY) issue them NOW, while the frames below are computed: issued
        // after the last frame their completion sits on the tile's — and with one tile per block the grid's — tail
        // (100k entities: 17.2 -> 15.7 us per tick).  Multi-wave grids keep them behind the frames: up front the 140 KB
        // burst queues ahead of the tile's own loads and the HBM-bound steady state gets slower (1M: +2.5 us per tick). ----
        auto issue_passive_stores = [&]() {
            mbar_wait(&s_bar[buf], (it >> 1) & 1u);
            const uint8_t* src = s_passive + size_t(buf) * p.passive_bytes;
            for (uint32_t i = 0; i < p.n_ops; ++i) {
                if (p.ops[i].kind != OP_SAVE || (p.ops[i].flags & (OPF_NO_STORE | OPF_SKIP_PASSIVE))) continue;
                uint8_t* img = p.arena + (size_t(p.ops[i].image_off256) << 8) + tile_off;
                uint32_t o = 0;
                for_each_passive_chunk([&](uint32_t off, uint32_t bytes) { tma_store_1d(img + off, src + o, bytes); o += bytes; });
            }
            if (p.flags & PF_WRITE_LIVE_PASSIVE) {
                uint8_t* img = p.arena + tile_off;
                uint32_t o = 0;
                for_each_passive_chunk([&](uint32_t off, uint32_t bytes) { tma_store_1d(img + off, src + o, bytes); o += bytes; });
            }
            tma_commit();
        };
        const bool passive_early = (p.flags & PF_PASSIVE_EARLY) != 0;
        if (use_tma && tid == 0 && passive_early) issue_passive_stores();

        uint32_t pend[6] = {0, 0, 0, 0, 0, 0};
        uint32_t pend_row = 0;
        bool pend_valid = false;
        auto flush_pending = [&]() {
            if (pend_valid && lane == 0) {
                unsigned int* a = &s_acc[pend_row * 2];
                if (CKT) { atomicXor(&a[2 * p.ck_t_slot], pend[0]); atomicXor(&a[2 * p.ck_t_slot + 1], pend[1]); }
                if (CKV) { atomicXor(&a[2 * p.ck_v_slot], pend[2]); atomicXor(&a[2 * p.ck_v_slot + 1], pend[3]); }
                atomicAdd(&a[12], pend[4]);
                if (pend[5]) atomicOr(&a[14], 1u);
            }
            pend_valid = false;
        };

        for (uint32_t i = (p.flags & PF_READ_LIVE) ? 0u : 1u; i < p.n_ops; ++i) {
            const uint32_t kind = p.ops[i].kind;
            if (kind == OP_ADVANCE) {
                const float dt = __uint_as_float(p.ops[i].dt_bits);
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                    if (OPT) {
                        // the queries only match entities that have the components (and exist)
                        const uint32_t m = (alive >> (8 * j)) & 0xFFu;
                        uint32_t a0 = tr[0][j], a1 = tr[1][j], a2 = tr[2][j], b0 = vl[0][j], b1 = vl[1][j], b2 = vl[2][j];
                        particle_step(a0, a1, a2, b0, b1, b2, dt);
                        if (row_matches(m, p.need_tv)) { tr[0][j] = a0; tr[1][j] = a1; tr[2][j] = a2; vl[0][j] = b0; vl[1][j] = b1; vl[2][j] = b2; }
                        if (row_matches(m, p.need_l)) {
                            uint32_t lo = tl[0][j], hi = tl[1][j];
                            hi -= (lo == 0u) ? 1u : 0u;
                            lo -= 1u;
                            tl[0][j] = lo; tl[1][j] = hi;
                            alive &= ((lo | hi) == 0u) ? ~(0xFFu << (8 * j)) : 0xFFFFFFFFu;
                        }
                        continue;
                    }
                    particle_step(tr[0][j], tr[1][j], tr[2][j], vl[0][j], vl[1][j], vl[2][j], dt);
                    // despawn_particles (particles.rs:282-289): ttl -= 1 (wrapping usize); despawn at 0
                    uint32_t lo = tl[0][j], hi = tl[1][j];
                    hi -= (lo == 0u) ? 1u : 0u;
                    lo -= 1u;
                    tl[0][j] = lo; tl[1][j] = hi;
                    alive &= ((lo | hi) == 0u) ? ~(0xFFu << (8 * j)) : 0xFFFFFFFFu;
                }
                if (p.ops[i].flags & OPF_SPAWN) {
                    // spawn_particles (particles.rs:258-270): Commands are applied after the schedule, so the
                    // newborn rows appear now, un-updated: Transform::default(), Velocity(vx, vy, 0), Ttl(ttl)
                    const uint32_t first = p.ops[i].image_off256, count = p.ops[i].save_index, off = p.ops[i].call_count;
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        const uint32_t k = row0 + j - first;
                        if (k < count) {
                            const float2 v = p.spawn_vals[off + k];
                            tr[0][j] = 0u; tr[1][j] = 0u; tr[2][j] = 0u;
                            vl[0][j] = __float_as_uint(v.x); vl[1][j] = __float_as_uint(v.y); vl[2][j] = 0u;
                            tl[0][j] = p.spawn_ttl_lo; tl[1][j] = p.spawn_ttl_hi;
                            alive = (alive & ~(0xFFu << (8 * j))) | (1u << (8 * j));  // exists, every component present
                        }
                    }
                }
            } else if (kind == OP_SAVE) {
                uint8_t* img = p.arena + (size_t(p.ops[i].image_off256) << 8);
                if (!(p.ops[i].flags & OPF_NO_STORE)) store_active(img);
                // ---- checksum partials (component_checksum.rs:81-90) ----
                uint64_t hx_t = 0, hx_v = 0;
                uint32_t bad = 0;
                // z == +0.0f for every row of the warp (a 2-D world): the tail lane of the 12-byte hash is a
                // compile-time constant, one diffusion less per entity and column.  Warp-uniform test.
                uint32_t tz_any = 0, vz_any = 0;
#pragma unroll
                for (int j = 0; j < VEC; ++j) { tz_any |= tr[2][j]; vz_any |= vl[2][j]; }
#ifndef BGR_ZERO_TAIL
#define BGR_ZERO_TAIL 1
#endif
                const bool tz_zero = BGR_ZERO_TAIL && CKT && __all_sync(0xffffffffu, tz_any == 0u);
                const bool vz_zero = BGR_ZERO_TAIL && CKV && __all_sync(0xffffffffu, vz_any == 0u);
#pragma unroll
                for (int j = 0; j < VEC; ++j) {
                    const uint32_t m = (alive >> (8 * j)) & 0xFFu;
                    const uint64_t live = (m & 1u) ? ~0ULL : 0ULL;
                    const uint64_t live_t = OPT ? (row_matches(m, p.need_t) ? ~0ULL : 0ULL) : live;
                    const uint64_t live_v = OPT ? (row_matches(m, p.need_v) ? ~0ULL : 0ULL) : live;
                    if (CKT) {
                        if (FINT) bad |= (f32_bits_nonfinite(tr[0][j]) | f32_bits_nonfinite(tr[1][j]) | f32_bits_nonfinite(tr[2][j])) & uint32_t(live_t);
                        const uint64_t lane_t = tz_zero ? kSeaTailZero : sea_diffuse(kSeaB ^ uint64_t(tr[2][j]));
                        uint64_t c = sea_hash_12_lane(uint64_t(tr[0][j]) | (uint64_t(tr[1][j]) << 32), lane_t);
                        hx_t ^= sea_hash_entity(t0[j], c) & live_t;
                    }
                    if (CKV) {
                        if (FINV) bad |= (f32_bits_nonfinite(vl[0][j]) | f32_bits_nonfinite(vl[1][j]) | f32_bits_nonfinite(vl[2][j])) & uint32_t(live_v);
                        const uint64_t lane_v = vz_zero ? kSeaTailZero : sea_diffuse(kSeaB ^ uint64_t(vl[2][j]));
                        uint64_t c = sea_hash_12_lane(uint64_t(vl[0][j]) | (uint64_t(vl[1][j]) << 32), lane_v);
                        hx_v ^= sea_hash_entity(t0[j], c) & live_v;
                    }
                }
                const uint32_t n_alive = __popc(alive & 0x01010101u);
                // warp-level fold (REDUX) now, shared-memory atomics at the NEXT save (or after the op
                // loop): the REDUX latency is covered by the following ADVANCE instead of stalling lane 0
                flush_pending();
                const unsigned full = 0xffffffffu;
                if (CKT) { pend[0] = __reduce_xor_sync(full, uint32_t(hx_t)); pend[1] = __reduce_xor_sync(full, uint32_t(hx_t >> 32)); }
                if (CKV) { pend[2] = __reduce_xor_sync(full, uint32_t(hx_v)); pend[3] = __reduce_xor_sync(full, uint32_t(hx_v >> 32)); }
                pend[4] = __reduce_add_sync(full, n_alive);
                pend[5] = (FINT || FINV) ? __reduce_or_sync(full, bad) : 0u;
                pend_row = p.ops[i].save_index * kAccStride;
                pend_valid = true;
            } else {  // OP_LOAD
                load_active(p.arena + (size_t(p.ops[i].image_off256) << 8), p.ops[i].n_rows);
            }
        }
        flush_pending();
        if (p.flags & PF_WRITE_LIVE_ACTIVE) store_active(p.arena);

        // ------------------------------ passive planes ------------------------------
        if (use_tma) {
            if (tid == 0 && !passive_early) issue_passive_stores();
        } else {
            // generic fallback (several LOADs in one program): the same program per passive plane,
            // a value is only ever loaded and stored, never computed on
            for (uint32_t pp = 0; pp < p.n_passive; pp += 4) {
                uint32_t v[4][VEC];
                const uint32_t nk = min(4u, p.n_passive - pp);
                if (p.flags & PF_READ_LIVE) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (k < nk) vec_load<VEC>(p.arena + size_t(p.passive[pp + k]) * kPlaneBytes + woff, v[k]);
                }
                for (uint32_t i = 0; i < p.n_ops; ++i) {
                    const uint32_t kind = p.ops[i].kind;
                    uint8_t* img = p.arena + (size_t(p.ops[i].image_off256) << 8);
                    if (kind == OP_LOAD) {
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            if (k < nk) vec_load<VEC>(img + size_t(p.passive[pp + k]) * kPlaneBytes + woff, v[k]);
                    } else if (kind == OP_SAVE && !(p.ops[i].flags & (OPF_NO_STORE | OPF_SKIP_PASSIVE))) {
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            if (k < nk) vec_store<VEC>(img + size_t(p.passive[pp + k]) * kPlaneBytes + woff, v[k]);
                    } else if (kind == OP_ADVANCE && (p.ops[i].flags & OPF_SPAWN)) {
                        const uint32_t first = p.ops[i].image_off256, count = p.ops[i].save_index;
#pragma unroll
                        for (int j = 0; j < VEC; ++j)
                            if (row0 + j - first < count) {
#pragma unroll
                                for (int k = 0; k < 4; ++k)
                                    if (k < nk) v[k][j] = p.passive_template[pp + k];
                            }
                    }
                }
                if (p.flags & PF_WRITE_LIVE_PASSIVE) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (k < nk) vec_store<VEC>(p.arena + size_t(p.passive[pp + k]) * kPlaneBytes + woff, v[k]);
                }
            }
        }
        if (tile_signal && it == 0) signal_tile(tile);
        if (dynamic) {
            const uint32_t slot = it % kRing, use = it / kRing;  // entry of iteration it + 1
            mbar_wait(&s_full[slot], use & 1u);
            tile = s_tile[slot];
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_empty[slot]);
        } else {
            tile += gridDim.x;
        }
    }
    if (use_tma && tid == 0) tma_wait_all();  // every bulk store has landed before the results are published

    // ---- block partials -> global accumulators -> (last block) host-visible results ----
    __syncthreads();
    for (uint32_t i = tid; i < p.n_saves * kAccStride; i += BLOCK) {
        unsigned long long v = (unsigned long long)s_acc[2 * i] | ((unsigned long long)s_acc[2 * i + 1] << 32);
        uint32_t c = i % kAccStride;
        if (v) {
            if (c == 6) atomicAdd(&p.accum[i], v);
            else if (c == 7) atomicOr(&p.accum[i], v);
            else atomicXor(&p.accum[i], v);
        }
    }
    __threadfence();
    __syncthreads();
    if (p.trace && tid == 0) atomicMax(&p.trace[1], globaltimer_ns());  // ... and when did its last block finish its tiles
    if (tid == 0) s_last = (atomicAdd(p.ticket, 1u) == gridDim.x - 1u);
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (uint32_t i = tid; i < p.n_saves * kAccStride; i += BLOCK)
            publish_pair(p.out, i, atomicExch(&p.accum[i], 0ULL), p.seq);  // publish (self-validating pair) and re-arm for the next launch
        if (tid == 0) publish_pair(p.out, kSeqIndex, p.seq, p.seq);       // completion pair: also there when nothing was saved
        __syncthreads();
        if (tid == 0) {
            if (tile_signal) st_release_gpu(p.grid_done, p.done_seq);  // every block's stores precede its ticket (fence above)
            p.ticket[0] = 0u;
            p.ticket[1] = 0u;
            if (p.trace) p.trace[2] = globaltimer_ns();
        }
    }
}

// =============================================================================================
// Stepwise (generic) path: one kernel per request, any registered schema / system list.
// =============================================================================================
#ifndef __CUDACC_RTC__  // the run-time specialisation (generic_program_jit.cuh) only needs the structs and helpers

// flat copy of tiles [0, n_tiles) of an image (fallback when the TMA kernel cannot be used);
// mask bytes of rows >= n_rows_src are forced to 0 (a Load that shrinks the world); the others are copied whole, with
// the absent bits of the optional columns.
__global__ void __launch_bounds__(256) k_copy_image(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                    uint32_t words, uint32_t n_tiles, uint32_t n_rows_src) {
    const uint32_t tb = tile_bytes_of(words);
    const size_t n_vec = size_t(n_tiles) * tb / 16u;
    for (size_t v = size_t(blockIdx.x) * blockDim.x + threadIdx.x; v < n_vec; v += size_t(gridDim.x) * blockDim.x) {
        uint4 x = __ldcs(reinterpret_cast<const uint4*>(src) + v);
        const size_t byte = v * 16u;
        const uint32_t tile = uint32_t(byte / tb), in_tile = uint32_t(byte % tb);
        if (in_tile >= words * kPlaneBytes) {  // alive plane: mask rows the source never contained
            const uint32_t r0 = tile * kTileRows + (in_tile - words * kPlaneBytes);
            uint32_t* w = reinterpret_cast<uint32_t*>(&x);
#pragma unroll
            for (int k = 0; k < 4; ++k) w[k] &= rows_mask_full<4>(r0 + 4 * k, n_rows_src);
        }
        __stcs(reinterpret_cast<uint4*>(dst) + v, x);
    }
}

// per-column XOR of per-entity hashes over live rows (component_checksum.rs:67-108), generic
// byte range [off, off+len) of an element stored as word planes starting at first_plane.
// acc[col_slot] ^= ..., acc[6] += live rows (only when count_alive), acc[7] |= nonfinite.
__global__ void __launch_bounds__(256) k_checksum_column(const uint8_t* __restrict__ img, uint32_t words,
                                                         uint32_t first_plane, uint32_t off, uint32_t len,
                                                         uint32_t finite_flag, uint32_t n_rows,
                                                         unsigned long long order_base, unsigned long long* acc,
                                                         uint32_t col_slot, uint32_t count_alive, uint32_t hash_column,
                                                         uint32_t absent) {
    const uint32_t lane = threadIdx.x & 31u;
    uint64_t hx = 0;
    uint32_t cnt = 0, bad = 0;
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r - lane < n_rows; r += gridDim.x * blockDim.x) {
        const uint32_t m = r < n_rows ? img[alive_offset(words, r)] : 0u;
        if (m & 1u) {
            ++cnt;
            if (hash_column && !(m & absent)) {
                const uint8_t* base = img + word_offset(words, r, first_plane);
                auto byte_at = [&](uint32_t i) -> uint8_t {
                    uint32_t b = off + i;
                    uint32_t w = *reinterpret_cast<const uint32_t*>(base + size_t(b >> 2) * kPlaneBytes);
                    return uint8_t(w >> (8 * (b & 3u)));
                };
                if (finite_flag)
                    for (uint32_t i = 0; i + 4 <= len; i += 4)
                        bad |= f32_bits_nonfinite(*reinterpret_cast<const uint32_t*>(base + size_t((off + i) >> 2) * kPlaneBytes));
                uint64_t custom = sea_hash_stream(len, byte_at);
                hx ^= sea_hash_2xu64(order_base + r, custom);
            }
        }
    }
    const unsigned full = 0xffffffffu;
    uint32_t lo = __reduce_xor_sync(full, uint32_t(hx)), hi = __reduce_xor_sync(full, uint32_t(hx >> 32));
    uint32_t c = __reduce_add_sync(full, cnt);
    uint32_t b = __reduce_or_sync(full, bad);
    if (lane == 0) {
        if (hash_column) atomicXor(&acc[col_slot], (unsigned long long)lo | ((unsigned long long)hi << 32));
        if (count_alive) atomicAdd(&acc[6], (unsigned long long)c);
        if (b) atomicOr(&acc[7], 1ULL);
    }
}

// copy the accumulators of n_saves saves to the host-mapped result block and re-arm them
__global__ void k_publish(unsigned long long* accum, unsigned long long* out, uint32_t n, unsigned long long seq) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) publish_pair(out, i, atomicExch(&accum[i], 0ULL), seq);
    if (threadIdx.x == 0) publish_pair(out, kSeqIndex, seq, seq);
}

// ---- ECS column (array of T, `stride` bytes apart) <-> tile-planar image -----------------------
// one thread per (row, word); tail words of an element whose size is not a multiple of 4 are zero-padded
__global__ void __launch_bounds__(256) k_scatter_column(uint8_t* img, uint32_t words, uint32_t first_plane,
                                                        uint32_t col_words, uint32_t elem_bytes, uint32_t first_row,
                                                        uint32_t count, const uint8_t* __restrict__ stage, uint32_t stride) {
    const size_t n = size_t(count) * col_words;
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x) {
        const uint32_t i = uint32_t(t / col_words), w = uint32_t(t % col_words);
        const uint8_t* s = stage + size_t(i) * stride + 4u * w;
        uint32_t v = 0;
        const uint32_t nb = min(4u, elem_bytes - 4u * w);
        for (uint32_t b = 0; b < nb; ++b) v |= uint32_t(s[b]) << (8 * b);
        *reinterpret_cast<uint32_t*>(img + word_offset(words, first_row + i, first_plane + w)) = v;
    }
}
__global__ void __launch_bounds__(256) k_gather_column(const uint8_t* __restrict__ img, uint32_t words, uint32_t first_plane,
                                                       uint32_t col_words, uint32_t elem_bytes, uint32_t first_row,
                                                       uint32_t count, uint8_t* stage, uint32_t stride) {
    const size_t n = size_t(count) * col_words;
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x) {
        const uint32_t i = uint32_t(t / col_words), w = uint32_t(t % col_words);
        uint32_t v = *reinterpret_cast<const uint32_t*>(img + word_offset(words, first_row + i, first_plane + w));
        uint8_t* d = stage + size_t(i) * stride + 4u * w;
        const uint32_t nb = min(4u, elem_bytes - 4u * w);
        for (uint32_t b = 0; b < nb; ++b) d[b] = uint8_t(v >> (8 * b));
    }
}
// words [first_word, first_word + n_words) of a column for rows [first_row, first_row+count), packed densely: consecutive
// threads write consecutive words of the output (coalesced stores; the plane reads are n_words interleaved streams)
__global__ void __launch_bounds__(256) k_gather_fields(const uint8_t* __restrict__ img, uint32_t words, uint32_t first_word,
                                                       uint32_t n_words, uint32_t first_row, uint32_t count,
                                                       uint32_t* __restrict__ out) {
    const size_t n = size_t(count) * n_words;
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x) {
        const uint32_t i = uint32_t(t / n_words), w = uint32_t(t % n_words);
        out[t] = *reinterpret_cast<const uint32_t*>(img + word_offset(words, first_row + i, first_word + w));
    }
}
// alive bytes of rows [first, first+count): gather to a dense array / set to a value
// out[i] = 1 iff the row exists and none of the `need` absent bits is set (need = 0: the alive flag itself)
__global__ void __launch_bounds__(256) k_gather_alive(const uint8_t* __restrict__ img, uint32_t words, uint32_t first_row,
                                                      uint32_t count, uint32_t n_rows, uint8_t* out, uint32_t need) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x)
        out[i] = (first_row + i < n_rows && row_matches(img[alive_offset(words, first_row + i)], need)) ? uint8_t(1) : uint8_t(0);
}
// Commands::entity(e).remove::<T>() / .insert(T): set / clear one absent bit of a live row
__global__ void k_set_absent(uint8_t* img, uint32_t words, uint32_t row, uint32_t bit, uint32_t absent) {
    uint8_t* m = img + alive_offset(words, row);
    if (*m & 1u) *m = absent ? uint8_t(*m | bit) : uint8_t(*m & ~bit);
}
// `commands.spawn((..., Rollback))`: zeroed components, alive = 1
__global__ void __launch_bounds__(256) k_spawn_rows(uint8_t* img, uint32_t words, uint32_t first_row, uint32_t count) {
    const size_t n = size_t(count) * (words + 1);
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x) {
        const uint32_t i = uint32_t(t / (words + 1)), w = uint32_t(t % (words + 1));
        if (w < words) *reinterpret_cast<uint32_t*>(img + word_offset(words, first_row + i, w)) = 0u;
        else img[alive_offset(words, first_row + i)] = 1;
    }
}
__global__ void k_set_alive(uint8_t* img, uint32_t words, uint32_t row, uint8_t value) { img[alive_offset(words, row)] = value; }

// ---- GgrsSchedule systems on the live image (stepwise path) ----
__global__ void __launch_bounds__(256) k_sys_particles_update(uint8_t* img, uint32_t words, uint32_t t_plane,
                                                              uint32_t v_plane, uint32_t n_rows, uint32_t dt_bits, uint32_t need) {
    const float dt = __uint_as_float(dt_bits);
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        if (!row_matches(img[alive_offset(words, r)], need)) continue;
        uint32_t* t = reinterpret_cast<uint32_t*>(img + word_offset(words, r, t_plane));
        uint32_t* v = reinterpret_cast<uint32_t*>(img + word_offset(words, r, v_plane));
        uint32_t tx = t[0], ty = t[kTileRows], tz = t[2 * kTileRows], vx = v[0], vy = v[kTileRows], vz = v[2 * kTileRows];
        particle_step(tx, ty, tz, vx, vy, vz, dt);
        t[0] = tx; t[kTileRows] = ty; t[2 * kTileRows] = tz; v[0] = vx; v[kTileRows] = vy; v[2 * kTileRows] = vz;
    }
}

// `kill` receives the despawns; they are applied after every system of the schedule has run
// (Commands are deferred to the end of GgrsSchedule).
__global__ void __launch_bounds__(256) k_sys_particles_despawn(uint8_t* img, uint32_t words, uint32_t l_plane,
                                                               uint32_t n_rows, uint8_t* kill, uint32_t need) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        if (!row_matches(img[alive_offset(words, r)], need)) continue;
        uint32_t* l = reinterpret_cast<uint32_t*>(img + word_offset(words, r, l_plane));
        uint64_t ttl = (uint64_t(l[kTileRows]) << 32) | l[0];
        ttl -= 1;
        l[0] = uint32_t(ttl); l[kTileRows] = uint32_t(ttl >> 32);
        if (ttl == 0) kill[r] = 1;
    }
}

// x.0 += k   (tests/component_rollback.rs:25-29)
__global__ void __launch_bounds__(256) k_sys_u32_add(uint8_t* img, uint32_t words, uint32_t plane, uint32_t n_rows, uint32_t k, uint32_t need) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x)
        if (row_matches(img[alive_offset(words, r)], need)) *reinterpret_cast<uint32_t*>(img + word_offset(words, r, plane)) += k;
}

// h = h.saturating_sub(k); despawn at 0   (tests/synctest.rs:38-45)
__global__ void __launch_bounds__(256) k_sys_u32_satsub_despawn(uint8_t* img, uint32_t words, uint32_t plane,
                                                                uint32_t n_rows, uint32_t k, uint8_t* kill, uint32_t need) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        if (!row_matches(img[alive_offset(words, r)], need)) continue;
        uint32_t* x = reinterpret_cast<uint32_t*>(img + word_offset(words, r, plane));
        uint32_t v = *x;
        v = v > k ? v - k : 0u;
        *x = v;
        if (v == 0) kill[r] = 1;
    }
}

// commands.entity(e).despawn() for every entity that has the bound component (tests/hierarchy.rs:36-45; launched only
// on frames whose input matches)
__global__ void __launch_bounds__(256) k_sys_despawn_having(const uint8_t* img, uint32_t words, uint32_t n_rows, uint8_t* kill, uint32_t need) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x)
        if (row_matches(img[alive_offset(words, r)], need)) kill[r] = 1;
}

// c.0 = count  (the deliberately non-deterministic system of tests/synctest.rs:92-97)
__global__ void __launch_bounds__(256) k_sys_u32_store(uint8_t* img, uint32_t words, uint32_t plane, uint32_t n_rows, uint32_t value, uint32_t need) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x)
        if (row_matches(img[alive_offset(words, r)], need)) *reinterpret_cast<uint32_t*>(img + word_offset(words, r, plane)) = value;
}

// spawn_particles (particles.rs:258-270) on the live image: rows [first, first+count) become
// Transform::default(), Velocity(vx, vy, 0), Ttl(ttl), alive; every other registered word is zero.
__global__ void __launch_bounds__(256) k_sys_particles_spawn(uint8_t* img, uint32_t words, uint32_t t_plane, uint32_t v_plane,
                                                             uint32_t l_plane, uint32_t first, uint32_t count,
                                                             const float2* __restrict__ vals, uint32_t ttl_lo, uint32_t ttl_hi) {
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < count; k += gridDim.x * blockDim.x) {
        const uint32_t r = first + k;
        for (uint32_t w = 0; w < words; ++w) *reinterpret_cast<uint32_t*>(img + word_offset(words, r, w)) = 0u;
        uint32_t* t = reinterpret_cast<uint32_t*>(img + word_offset(words, r, t_plane));
        t[6 * kTileRows] = 0x3f800000u;                                                          // rotation.w = 1
        t[7 * kTileRows] = 0x3f800000u; t[8 * kTileRows] = 0x3f800000u; t[9 * kTileRows] = 0x3f800000u;  // scale = 1
        uint32_t* v = reinterpret_cast<uint32_t*>(img + word_offset(words, r, v_plane));
        const float2 xy = vals[k];
        v[0] = __float_as_uint(xy.x); v[kTileRows] = __float_as_uint(xy.y);
        uint32_t* l = reinterpret_cast<uint32_t*>(img + word_offset(words, r, l_plane));
        l[0] = ttl_lo; l[kTileRows] = ttl_hi;
        img[alive_offset(words, r)] = 1;
    }
}

#endif  // !__CUDACC_RTC__

// move_cube_system (box_game.rs:154-206), BASELINE config C1.  player handle == RollbackOrdered index.
// `fr` is `FRICTION.powf(dt)` (FRICTION = 0.0018), evaluated once per Advance by the host with the C library's powf,
// the function the reference calls (Op::fr_bits).  A device powf is only good to about one ulp and rounds some frame
// rates' factor the other way, so every result here is bit-exact with the CPU only because the factor comes from the host.
__device__ __forceinline__ void box_move_step(float& tx, float& ty, float& tz, float& vx, float& vy, float& vz, float dt, float fr,
                                              uint32_t input) {
    const float ACCELERATION = 18.0f, MAX_SPEED = 3.0f, PLANE_SIZE = 5.0f, CUBE_SIZE = 0.2f;
    const bool up = input & 1u, down = input & 2u, left = input & 4u, right = input & 8u;
    const float a = __fmul_rn(ACCELERATION, dt);
    if (up && !down) vz = __fsub_rn(vz, a);
    if (!up && down) vz = __fadd_rn(vz, a);
    if (left && !right) vx = __fsub_rn(vx, a);
    if (!left && right) vx = __fadd_rn(vx, a);
    if (!up && !down) vz = __fmul_rn(vz, fr);
    if (!left && !right) vx = __fmul_rn(vx, fr);
    vy = __fmul_rn(vy, fr);
    // glam Vec3::clamp_length_max(MAX_SPEED)
    const float len_sq = __fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), __fmul_rn(vz, vz));
    if (len_sq > __fmul_rn(MAX_SPEED, MAX_SPEED)) {
        const float l = __fsqrt_rn(len_sq);
        vx = __fmul_rn(MAX_SPEED, __fdiv_rn(vx, l)); vy = __fmul_rn(MAX_SPEED, __fdiv_rn(vy, l)); vz = __fmul_rn(MAX_SPEED, __fdiv_rn(vz, l));
    }
    tx = __fadd_rn(tx, __fmul_rn(vx, dt)); ty = __fadd_rn(ty, __fmul_rn(vy, dt)); tz = __fadd_rn(tz, __fmul_rn(vz, dt));
    const float hw = __fmul_rn(__fsub_rn(PLANE_SIZE, CUBE_SIZE), 0.5f);
    tx = tx < -hw ? -hw : (tx > hw ? hw : tx);
    tz = tz < -hw ? -hw : (tz > hw ? hw : tz);
}
#ifndef __CUDACC_RTC__
__global__ void k_sys_box_move(uint8_t* img, uint32_t words, uint32_t t_plane, uint32_t v_plane, uint32_t n_rows,
                               uint32_t dt_bits, uint32_t fr_bits, unsigned long long inputs_packed, uint32_t n_players,
                               unsigned long long order_base, uint32_t need) {
    const float dt = __uint_as_float(dt_bits), fr = __uint_as_float(fr_bits);
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        if (!row_matches(img[alive_offset(words, r)], need)) continue;
        float* t = reinterpret_cast<float*>(img + word_offset(words, r, t_plane));
        float* v = reinterpret_cast<float*>(img + word_offset(words, r, v_plane));
        float tx = t[0], ty = t[kTileRows], tz = t[2 * kTileRows];
        float vx = v[0], vy = v[kTileRows], vz = v[2 * kTileRows];
        const unsigned long long handle = order_base + r;
        const uint32_t input = handle < n_players && handle < 8 ? uint32_t(inputs_packed >> (8 * uint32_t(handle))) & 0xffu : 0u;
        box_move_step(tx, ty, tz, vx, vy, vz, dt, fr, input);
        t[0] = tx; t[kTileRows] = ty; t[2 * kTileRows] = tz;
        v[0] = vx; v[kTileRows] = vy; v[2 * kTileRows] = vz;
    }
}

// apply deferred despawn commands: alive &= !kill ; kill = 0
__global__ void __launch_bounds__(256) k_apply_despawns(uint8_t* img, uint32_t words, uint32_t n_rows, uint8_t* kill) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x)
        if (kill[r]) { img[alive_offset(words, r)] = 0; kill[r] = 0; }
}

#endif  // !__CUDACC_RTC__

}  // namespace bgr
