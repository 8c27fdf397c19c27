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

#ifndef __CUDACC_RTC__
#include "../../include/bevy_ggrs_b200.h"
#endif  // NVRTC: the engine's generated prelude defines the BGR_SYS_* ids (host function declarations cannot be parsed there)
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
    // SAVE: the slot already holds the active planes and alive byte of the registers on every row below the row count
    // (content ids, engine.cu HostState): no active store, no stamp.  The checksum is still computed from the
    // registers.  Only this bundle kernel honours it, like OPF_SKIP_PASSIVE; it says nothing about passive planes.
    OPF_HELD = 16u,
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
    uint32_t call_count;    // ADVANCE: value of the un-rolled-back host counter (test system).  ADVANCE+SPAWN: offset into spawn_vals.
                            // LOAD/SAVE in the bundle kernel: index of the image (its row of the content-stamp table)
    uint8_t inputs[8];     // ADVANCE: PlayerInputs<T>.0[handle].0 for every handle (u8, BGR_MAX_PLAYERS)
};
static_assert(sizeof(Op) == 40, "Op layout");

// One registered GgrsSchedule system as the kernels run it (run_system), fixed at bgr_build
struct SysSpec {
    uint32_t id;      // bgr_system
    uint32_t plane0;  // first word plane the system touches (column's first plane + byte_offset / 4)
    uint32_t plane1;  // second bound column's first plane (Velocity for the Transform/Velocity systems)
    uint32_t need;    // absent bits of the bound columns: the query matches a row iff row_matches(mask, need)
    uint32_t param;   // k (U32_ADD / U32_SATSUB_DESPAWN), the system's index among the call-count systems, or
                      // player handle | value << 8 (DESPAWN_ON_INPUT)
};

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

// Content stamps of the bundle kernel's active planes (translation x/y/z, velocity x/y/z, ttl lo/hi, alive: plane q in
// that order), one u32 per (image, 64-row warp segment, plane); the invariant is in engine.cu HostState.
constexpr uint32_t kActivePlanes = 9;
constexpr uint32_t kAlivePlaneBit = 1u << 8;
constexpr uint32_t kSegRows = 64;
constexpr uint32_t kSegsPerTile = kTileRows / kSegRows;
// The stamped instances keep the active words and alive bytes of the last stamp point in shared memory, one snapshot per
// thread laid out [word group][thread]: four uint4 groups (two planes of its two rows each) and one alive word.
constexpr uint32_t kSnapBytes = (4u * 16u + 4u) * (kTileRows / 2u);
// Checksum partials of the bundle kernel, at the front of its dynamic shared memory.  Lane fold (the default): per Save
// kLaneWords words per lane, laid out [save][word][lane]: the XOR of the lane's Translation hashes (lo, hi), of its
// Velocity hashes (lo, hi), and its live rows with bit 31 set once it saw a non-finite value.  Warp fold (launches where
// those slots would cost a resident block): per Save the kAccStride columns as 32-bit halves, fed by warp reductions.
constexpr uint32_t kLaneWords = 5;
__host__ __device__ constexpr uint32_t fold_bytes(bool warp_fold, uint32_t n_saves) {
    return n_saves * (warp_fold ? uint32_t(kAccStride) * 2u * 4u : kLaneWords * 32u * 4u);
}

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
    uint32_t* stamps;               // [images][segments][kActivePlanes] content stamps (0 = unknown)
    uint32_t stamp_image;           // words of one image's row of `stamps`
    uint32_t stamp_base;            // this launch's fresh stamps: stamp_base + op index, stamp_base + n_ops for the live write
    unsigned long long* held_check;  // nullptr, or (BGR_TUNE_HELD_SAVES=2) where held Saves count the words the target lacks
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
template <bool B> struct BoolConst { static constexpr bool value = B; };  // a compile-time flag passed to a generic lambda
// f32_bits_nonfinite of any of three words, on the FP32 pipe: x * 0 is NaN exactly when x is an infinity or a NaN (and
// +-0 otherwise), and a NaN addend carries through the fused multiply-adds.  Three FP32 instructions and one compare
// instead of three masks and three compares on the integer pipes the checksum keeps busy.
__device__ __forceinline__ uint32_t f32x3_bits_nonfinite(uint32_t a, uint32_t b, uint32_t c) {
    const float z = __fmaf_rn(__uint_as_float(a), 0.0f, __fmaf_rn(__uint_as_float(b), 0.0f, __fmul_rn(__uint_as_float(c), 0.0f)));
    return z != z ? 1u : 0u;
}

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

// PlayerInputs<T>.0[handle].0; 0 for a handle the frame has no input for.  (A u32 player handle is compared in 32 bits,
// a u64 RollbackOrdered index in 64.)
template <class Handle>
__host__ __device__ __forceinline__ uint32_t player_input(const Op& op, Handle handle) {
    const uint32_t n_players = (op.flags >> 8) & 0xFu;
    return handle < n_players && handle < 8 ? op.inputs[handle] : 0u;
}

// =============================================================================================
// THE per-row definition of every compiled GgrsSchedule system (include/bevy_ggrs_b200.h): one registered system
// applied to the R rows a thread owns.  The interpreter (k_generic_program) runs it on its shared-memory tile, the
// generated kernel (k_generic_jit) on its register copy with a constexpr spec (the switch folds away), the stepwise
// path (k_sys_rows) on the live image with R = 1.
//   word(k, plane) : reference to row k's word in `plane`
//   m[k]           : row k's mask byte as it was before the frame (every system of a frame sees the same presence)
//   kill[k]        : set when the system despawns row k; the caller applies it after the schedule's last system
//                    (Commands are deferred to the end of GgrsSchedule)
//   row0, row_step : row k's RollbackOrdered index is row0 + k * row_step
// The switch sits outside the row loop (a system's spec is decoded once for all rows) and a word is written only on
// rows the query matches.
// =============================================================================================
template <int R, class Word>
__device__ __forceinline__ void run_system(const SysSpec& sy, Word&& word, const uint32_t (&m)[R], bool (&kill)[R], const Op& op,
                                           unsigned long long row0, uint32_t row_step) {
    const float dt = __uint_as_float(op.dt_bits);
    switch (sy.id) {
    case BGR_SYS_U32_ADD:  // x.0 += k   (tests/component_rollback.rs:25-29)
#pragma unroll
        for (int k = 0; k < R; ++k)
            if (row_matches(m[k], sy.need)) word(k, sy.plane0) += sy.param;
        break;
    case BGR_SYS_U32_SATSUB_DESPAWN:  // h = h.saturating_sub(k); despawn at 0   (tests/synctest.rs:38-45)
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const bool on = row_matches(m[k], sy.need);
            uint32_t v = word(k, sy.plane0);
            v = v > sy.param ? v - sy.param : 0u;
            if (on) word(k, sy.plane0) = v;
            kill[k] = kill[k] || (on && v == 0u);
        }
        break;
    case BGR_SYS_U32_STORE_CALL_COUNT:  // c.0 = count  (the deliberately non-deterministic system of tests/synctest.rs:92-97)
#pragma unroll
        for (int k = 0; k < R; ++k)
            if (row_matches(m[k], sy.need)) word(k, sy.plane0) = op.call_count + sy.param;
        break;
    case BGR_SYS_DESPAWN_ON_INPUT: {  // commands.entity(e).despawn() for every entity that has the bound component (tests/hierarchy.rs:36-45)
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const bool on = row_matches(m[k], sy.need);
            const uint32_t input = player_input(op, sy.param & 0xFFu);
            kill[k] = kill[k] || (on && input == (sy.param >> 8));
        }
        break;
    }
    case BGR_SYS_PARTICLES_UPDATE:  // update_particles (particles.rs:272-280)
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const bool on = row_matches(m[k], sy.need);
            uint32_t tx = word(k, sy.plane0), ty = word(k, sy.plane0 + 1), tz = word(k, sy.plane0 + 2);
            uint32_t vx = word(k, sy.plane1), vy = word(k, sy.plane1 + 1), vz = word(k, sy.plane1 + 2);
            particle_step(tx, ty, tz, vx, vy, vz, dt);
            if (on) {
                word(k, sy.plane0) = tx; word(k, sy.plane0 + 1) = ty; word(k, sy.plane0 + 2) = tz;
                word(k, sy.plane1) = vx; word(k, sy.plane1 + 1) = vy; word(k, sy.plane1 + 2) = vz;
            }
        }
        break;
    case BGR_SYS_PARTICLES_DESPAWN:  // despawn_particles (particles.rs:282-289): ttl -= 1 (wrapping usize); despawn at 0
#pragma unroll
        for (int k = 0; k < R; ++k) {
            const bool on = row_matches(m[k], sy.need);
            uint64_t ttl = (uint64_t(word(k, sy.plane0 + 1)) << 32) | word(k, sy.plane0);
            ttl -= 1;
            if (on) { word(k, sy.plane0) = uint32_t(ttl); word(k, sy.plane0 + 1) = uint32_t(ttl >> 32); }
            kill[k] = kill[k] || (on && ttl == 0);
        }
        break;
    case BGR_SYS_BOX_MOVE:  // move_cube_system (box_game.rs:154-206)
#pragma unroll
        for (int k = 0; k < R; ++k)
            if (row_matches(m[k], sy.need)) {  // two to four entities: a branch costs nothing and keeps the step off the other rows
                float tx = __uint_as_float(word(k, sy.plane0)), ty = __uint_as_float(word(k, sy.plane0 + 1)), tz = __uint_as_float(word(k, sy.plane0 + 2));
                float vx = __uint_as_float(word(k, sy.plane1)), vy = __uint_as_float(word(k, sy.plane1 + 1)), vz = __uint_as_float(word(k, sy.plane1 + 2));
                const uint32_t input = player_input(op, row0 + uint32_t(k) * row_step);
                box_move_step(tx, ty, tz, vx, vy, vz, dt, __uint_as_float(op.fr_bits), input);
                word(k, sy.plane0) = __float_as_uint(tx); word(k, sy.plane0 + 1) = __float_as_uint(ty); word(k, sy.plane0 + 2) = __float_as_uint(tz);
                word(k, sy.plane1) = __float_as_uint(vx); word(k, sy.plane1 + 1) = __float_as_uint(vy); word(k, sy.plane1 + 2) = __float_as_uint(vz);
            }
        break;
    default: break;
    }
}

// THE definition of a row born to spawn_particles (particles.rs:258-270): row k's words become every registered word
// zero, then Transform::default() (rotation.w and scale 1), Velocity(vx, vy, 0) and Ttl(ttl).  `sy` is the spawn
// system's spec: plane0 = Transform, plane1 = Velocity, param = Ttl (build_specs).  The caller sets the row's mask byte
// to 1: alive, every optional column present.  The stepwise path (k_sys_particles_spawn), the interpreter and the
// generated kernel write newborn rows through it; the bundle kernel keeps its own register layout.
template <class Word>
__device__ __forceinline__ void spawn_row(const SysSpec& sy, Word&& word, int k, uint32_t words, float2 v, unsigned long long ttl) {
#pragma unroll
    for (uint32_t j = 0; j < words; ++j) word(k, j) = 0u;
    word(k, sy.plane0 + 6) = 0x3f800000u;  // rotation.w = 1
    word(k, sy.plane0 + 7) = 0x3f800000u; word(k, sy.plane0 + 8) = 0x3f800000u; word(k, sy.plane0 + 9) = 0x3f800000u;  // scale = 1
    word(k, sy.plane1) = __float_as_uint(v.x); word(k, sy.plane1 + 1) = __float_as_uint(v.y);
    word(k, sy.param) = uint32_t(ttl); word(k, sy.param + 1) = uint32_t(ttl >> 32);
}

// =============================================================================================
// THE fused kernel: interprets the whole request vector (Load / Advance / Save ...) for the
// particles bundle.  One launch per handle_requests; one tile (512 rows) per block iteration.
//   * active words (translation, velocity, ttl, alive) live in registers for the whole program:
//       LOAD    : read them from the snapshot image once
//       ADVANCE : update_particles + despawn_particles in registers (0 bytes)
//       SAVE    : stream them into the frame's slot and fold the per-entity seahashes of the
//                 checksummed columns: every lane XORs its partials into its own shared-memory slot ->
//                 after the tiles one warp reduction and one global atomic per block per (save, column)
//                 -> last block publishes to host-mapped memory.  A warp stores
//                 only the planes of its 64-row segment whose content stamp the slot does not hold
//                 already (ProgramParams::stamps): in a 2-D world z, velocity.x, ttl.hi and alive
//                 keep their bits from frame to frame and are stored once per slot
//       end     : write the live image once (same stamp rule)
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
// STAMPS: stable-plane elision (content stamps, below).  It pays on bandwidth-bound grids of several waves; a single-wave
// grid is latency-bound, and there the instance without it runs (engine.cu run_fused), which stores every active plane.
// VERIFY: BGR_TUNE_HELD_SAVES=2, every held Save compares its target with the registers (check_held).  The instances
// that run by default do not carry that code.
// WARP_FOLD: a Save's partials are reduced over the warp (REDUX) and lane 0 adds them to the block's columns, instead of
// every lane adding its own to its lane slot (fold_bytes).  The lane slots take 640 bytes of shared memory per Save;
// launch_particles runs this instance only where they would cost a resident block (a wide passive double buffer and
// many Saves in one vector).
template <int MODE, bool STAMPS, bool VERIFY, bool WARP_FOLD = false>
__global__ void __launch_bounds__(256, 3) k_particles_program(const __grid_constant__ ProgramParams p) {  // budget: prologue
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
    // the checksum partials (fold_bytes); STAMPS: the stamp-point snapshot (kSnapBytes); then 2 x passive_bytes (double buffer)
    extern __shared__ __align__(128) uint8_t s_dyn[];
    unsigned int* const s_fold = reinterpret_cast<unsigned int*>(s_dyn);  // 32-bit words: native shared atomics, no CAS loop
    uint4* const s_snap = reinterpret_cast<uint4*>(s_dyn + fold_bytes(WARP_FOLD, p.n_saves));
    uint8_t* const s_passive = reinterpret_cast<uint8_t*>(s_snap) + (STAMPS ? kSnapBytes : 0u);
    __shared__ __align__(8) uint64_t s_bar[2];
    __shared__ unsigned int s_last;
    __shared__ unsigned int s_stored;  // bgr_trace_enable: 64-byte units of active planes this block stored

    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    if (p.trace && tid == 0) atomicMin(&p.trace[0], globaltimer_ns());  // bgr_trace_enable: when did this launch's first block start
    if (tid == 0) s_stored = 0u;
    // Programmatic dependent launch: let the NEXT request vector's kernel be launched and its blocks scheduled
    // into SM slots as this grid drains (hides launch latency and block ramp-up between back-to-back ticks) ...
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    for (uint32_t i = tid; i < fold_bytes(WARP_FOLD, p.n_saves) / 4u; i += BLOCK) s_fold[i] = 0u;
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
    // The stamps of a tile's segments are read and written only by the warps that run that tile, so the next launch's
    // stamp reads need exactly what its data reads need: the stamp stores are ordinary stores of those warps, behind the
    // same fence as the tile's data (and behind the grid's __threadfence for tiles that only grid_done announces).
    auto signal_tile = [&](uint32_t t) {
        if (use_tma && tid == 0) tma_wait_all();  // that tile's bulk stores have landed (not just released their buffer)
        fence_acq_rel_gpu();                      // every thread's stores (data and stamps) are visible gpu-wide before its warp arrives
        __syncwarp();
        if (lane == 0) {
            if (atomicAdd(&p.tile_cnt[t], 1u) == kTileRows / (32 * VEC) - 1) {  // last warp to announce this tile
                p.tile_cnt[t] = 0u;
                fence_acq_rel_gpu();
                st_release_gpu(&p.tile_done[t], p.done_seq);
            }
        }
    };
    for (uint32_t tile = blockIdx.x; tile < p.n_tiles; ++it) {  // budget: tile_loop
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

        // ------------------------------ active words ------------------------------  budget: load
        uint32_t tr[3][VEC], vl[3][VEC], tl[2][VEC];
        uint32_t alive = 0;
        // Stable-plane elision.  Lane q < kActivePlanes holds `st`, the stamp of the content plane q of this warp's
        // segment had at the last stamp point (a Load or read of the live image, a stored Save, the live write; 0 =
        // unknown).  Each thread keeps its words and alive bytes of that point in s_snap.  A stored Save compares the
        // registers with the snapshot once, gives every plane that differs (or is unknown) a fresh stamp and stores only
        // the planes whose stamp the target image does not already hold.  `dirty` is only the spawn bit: a spawning
        // Advance marks every plane.
        uint32_t st = 0, dirty = 0;
        uint32_t* const seg_stamps = p.stamps + (size_t(tile) * kSegsPerTile + (tid >> 5)) * kActivePlanes + min(lane, kActivePlanes - 1u);
        const bool stamp_lane = lane < kActivePlanes;
        auto put_snapshot = [&](uint32_t a) {
            s_snap[0 * BLOCK + tid] = make_uint4(tr[0][0], tr[0][1], tr[1][0], tr[1][1]);
            s_snap[1 * BLOCK + tid] = make_uint4(tr[2][0], tr[2][1], vl[0][0], vl[0][1]);
            s_snap[2 * BLOCK + tid] = make_uint4(vl[1][0], vl[1][1], vl[2][0], vl[2][1]);
            s_snap[3 * BLOCK + tid] = make_uint4(tl[0][0], tl[0][1], tl[1][0], tl[1][1]);
            reinterpret_cast<uint32_t*>(s_snap + 4 * BLOCK)[tid] = a;
        };

        auto load_active = [&](const uint8_t* img, uint32_t n_rows, uint32_t img_idx) {
            const uint8_t* pt = img + p.t_off + woff;
            const uint8_t* pv = img + p.v_off + woff;
            const uint8_t* pl = img + p.l_off + woff;
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_load<VEC>(pt + k * kPlaneBytes, tr[k]);
#pragma unroll
            for (int k = 0; k < 3; ++k) vec_load<VEC>(pv + k * kPlaneBytes, vl[k]);
#pragma unroll
            for (int k = 0; k < 2; ++k) vec_load<VEC>(pl + k * kPlaneBytes, tl[k]);
            const uint32_t raw = alive_load<VEC>(img + aoff);
            alive = raw & (OPT ? rows_mask_full<VEC>(row0, n_rows) : rows_mask<VEC>(row0, n_rows));
            if (STAMPS) {
                // the image's bytes: where the row count cleared alive bytes the image holds, the alive plane differs
                put_snapshot(raw);
                dirty = 0;
                st = stamp_lane ? __ldcg(seg_stamps + size_t(img_idx) * p.stamp_image) : 0u;
            }
        };
        // first half of a stamped store into image img_idx: stamps the planes whose bits differ from the snapshot with
        // `fresh`, takes the registers as the new snapshot and issues the read of the image's stamps, which store_active
        // consumes later (the checksum of a Save hides part of its latency)
        auto claim_stamps = [&](uint32_t img_idx, uint32_t fresh) -> uint32_t {
            if (!STAMPS) return 0u;
            // bits, not values: -0.0 -> +0.0 and a changed NaN payload are changes
            const uint4 s0 = s_snap[0 * BLOCK + tid], s1 = s_snap[1 * BLOCK + tid];
            const uint4 s2 = s_snap[2 * BLOCK + tid], s3 = s_snap[3 * BLOCK + tid];
            const uint32_t sa = reinterpret_cast<const uint32_t*>(s_snap + 4 * BLOCK)[tid];
            uint32_t d = dirty;
            auto note = [&](uint32_t q, uint32_t a0, uint32_t a1, uint32_t b0, uint32_t b1) {
                d |= ((a0 ^ b0) | (a1 ^ b1)) != 0u ? 1u << q : 0u;
            };
            note(0, tr[0][0], tr[0][1], s0.x, s0.y); note(1, tr[1][0], tr[1][1], s0.z, s0.w);
            note(2, tr[2][0], tr[2][1], s1.x, s1.y); note(3, vl[0][0], vl[0][1], s1.z, s1.w);
            note(4, vl[1][0], vl[1][1], s2.x, s2.y); note(5, vl[2][0], vl[2][1], s2.z, s2.w);
            note(6, tl[0][0], tl[0][1], s3.x, s3.y); note(7, tl[1][0], tl[1][1], s3.z, s3.w);
            if (alive != sa) d |= kAlivePlaneBit;
            d = __reduce_or_sync(0xffffffffu, d);
            dirty = 0;
            if (d) put_snapshot(alive);  // else the registers equal it already
            if (stamp_lane && (((d >> lane) & 1u) || st == 0u)) st = fresh;
            return stamp_lane ? __ldcg(seg_stamps + size_t(img_idx) * p.stamp_image) : st;
        };
        // stores the planes whose stamp in image img_idx (`held`, from claim_stamps) differs and records the new stamps;
        // without STAMPS every plane
        auto store_active = [&](uint8_t* img, uint32_t img_idx, uint32_t held) {
            uint32_t planes = (1u << kActivePlanes) - 1u;
            if (STAMPS) {
                const bool put = held != st;
                planes = __ballot_sync(0xffffffffu, put);
                if (put) __stcg(seg_stamps + size_t(img_idx) * p.stamp_image, st);
            }
            // a word plane-segment is 4 units of 64 B, the alive plane-segment 1
            if (p.trace && lane == 0) atomicAdd(&s_stored, 4u * __popc(planes & 0xFFu) + (planes >> 8));
            uint8_t* pt = img + p.t_off + woff;
            uint8_t* pv = img + p.v_off + woff;
            uint8_t* pl = img + p.l_off + woff;
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (planes & (1u << k)) vec_store<VEC>(pt + k * kPlaneBytes, tr[k]);
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (planes & (8u << k)) vec_store<VEC>(pv + k * kPlaneBytes, vl[k]);
#pragma unroll
            for (int k = 0; k < 2; ++k)
                if (planes & (64u << k)) vec_store<VEC>(pl + k * kPlaneBytes, tl[k]);
            if (planes & kAlivePlaneBit) alive_store<VEC>(img + aoff, alive);
        };
        // BGR_TUNE_HELD_SAVES=2: count the active words and alive bytes, on rows below the row count, in which a held
        // Save's target differs from the registers
        auto check_held = [&](const uint8_t* img, uint32_t n_rows) {
            uint32_t r[8][VEC];
            const uint8_t* pt = img + p.t_off + woff;
            const uint8_t* pv = img + p.v_off + woff;
            const uint8_t* pl = img + p.l_off + woff;
#pragma unroll
            for (int k = 0; k < 3; ++k) { vec_load<VEC>(pt + k * kPlaneBytes, r[k]); vec_load<VEC>(pv + k * kPlaneBytes, r[3 + k]); }
#pragma unroll
            for (int k = 0; k < 2; ++k) vec_load<VEC>(pl + k * kPlaneBytes, r[6 + k]);
            const uint32_t a = alive_load<VEC>(img + aoff);
            uint32_t bad = 0;
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
                if (row0 + j >= n_rows) continue;
                bad += (r[0][j] != tr[0][j]) + (r[1][j] != tr[1][j]) + (r[2][j] != tr[2][j]) + (r[3][j] != vl[0][j]) +
                       (r[4][j] != vl[1][j]) + (r[5][j] != vl[2][j]) + (r[6][j] != tl[0][j]) + (r[7][j] != tl[1][j]) +
                       (((a ^ alive) >> (8 * j)) & 0xFFu ? 1u : 0u);
            }
            bad = __reduce_add_sync(0xffffffffu, bad);
            if (lane == 0 && bad) atomicAdd(p.held_check, (unsigned long long)bad);
        };

        if (p.flags & PF_READ_LIVE) load_active(p.arena, p.live_rows, 0u);
        else load_active(p.arena + (size_t(p.ops[0].image_off256) << 8), p.ops[0].n_rows, p.ops[0].call_count);  // ops[0] is a LOAD

        // lane of the per-entity hash that only depends on the RollbackOrdered index
        uint64_t t0[VEC];
#pragma unroll
        for (int j = 0; j < VEC; ++j) t0[j] = sea_order_lane(p.order_base + row0 + j);

        // budget: tile_loop
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

        // WARP_FOLD only: the warp's partials of the last Save, added to the block's columns at the next one
        uint32_t pend[5] = {0, 0, 0, 0, 0};
        uint32_t pend_row = 0;
        bool pend_valid = false;
        auto flush_pending = [&]() {
            if (WARP_FOLD && pend_valid && lane == 0) {
                unsigned int* a = &s_fold[pend_row * 2];
                if (CKT) { atomicXor(&a[2 * p.ck_t_slot], pend[0]); atomicXor(&a[2 * p.ck_t_slot + 1], pend[1]); }
                if (CKV) { atomicXor(&a[2 * p.ck_v_slot], pend[2]); atomicXor(&a[2 * p.ck_v_slot + 1], pend[3]); }
                atomicAdd(&a[12], pend[4] & 0xFFFFu);
                if (pend[4] >> 16) atomicOr(&a[14], 1u);
            }
            pend_valid = false;
        };

        for (uint32_t i = (p.flags & PF_READ_LIVE) ? 0u : 1u; i < p.n_ops; ++i) {
            const uint32_t kind = p.ops[i].kind;
            if (kind == OP_ADVANCE) {  // budget: advance
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
                            dirty = (1u << kActivePlanes) - 1u;
                        }
                    }
                }
            } else if (kind == OP_SAVE) {  // budget: save_store
                uint8_t* img = p.arena + (size_t(p.ops[i].image_off256) << 8);
                // a held Save stores nothing and claims no stamp: the snapshot and `st` stay at the last stamp point,
                // and the target's stamps still name its bytes
                const bool store = !(p.ops[i].flags & (OPF_NO_STORE | OPF_HELD));
                const uint32_t held = store ? claim_stamps(p.ops[i].call_count, p.stamp_base + i) : 0u;  // budget: save_track
                if (store && !STAMPS) store_active(img, p.ops[i].call_count, held);  // nothing to wait for: issue the stores first  budget: save_store
                if (VERIFY && (p.ops[i].flags & OPF_HELD)) check_held(img, p.ops[i].n_rows);
                // ---- checksum partials (component_checksum.rs:81-90) ----  budget: save_hash
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
                // One warp-uniform branch around the whole block: when every checksummed column's z is +0.0f, the block has
                // no branch inside and ptxas interleaves the four independent hash chains of the thread.  (A branch per row
                // and column around a tail diffusion splits them into separate blocks, and the 1M tick gets slower.)
                auto hash_rows = [&](auto zero_tails) {
                    constexpr bool Z = decltype(zero_tails)::value;
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        const uint32_t m = (alive >> (8 * j)) & 0xFFu;
                        const uint64_t live = (m & 1u) ? ~0ULL : 0ULL;
                        const uint64_t live_t = OPT ? (row_matches(m, p.need_t) ? ~0ULL : 0ULL) : live;
                        const uint64_t live_v = OPT ? (row_matches(m, p.need_v) ? ~0ULL : 0ULL) : live;
                        if (CKT) {
                            if (FINT) bad |= f32x3_bits_nonfinite(tr[0][j], tr[1][j], tr[2][j]) & uint32_t(live_t);
                            const uint64_t lane_t = (Z || tz_zero) ? kSeaTailZero : sea_diffuse(kSeaB ^ uint64_t(tr[2][j]));
                            uint64_t c = sea_hash_12_lane(uint64_t(tr[0][j]) | (uint64_t(tr[1][j]) << 32), lane_t);
                            hx_t ^= sea_hash_entity(t0[j], c) & live_t;
                        }
                        if (CKV) {
                            if (FINV) bad |= f32x3_bits_nonfinite(vl[0][j], vl[1][j], vl[2][j]) & uint32_t(live_v);
                            const uint64_t lane_v = (Z || vz_zero) ? kSeaTailZero : sea_diffuse(kSeaB ^ uint64_t(vl[2][j]));
                            uint64_t c = sea_hash_12_lane(uint64_t(vl[0][j]) | (uint64_t(vl[1][j]) << 32), lane_v);
                            hx_v ^= sea_hash_entity(t0[j], c) & live_v;
                        }
                    }
                };
                if ((tz_zero || !CKT) && (vz_zero || !CKV)) hash_rows(BoolConst<true>{});
                else hash_rows(BoolConst<false>{});
                const uint32_t n_alive = __popc(alive & 0x01010101u);  // budget: save_fold
                if (!WARP_FOLD) {
                    // XOR and + are associative: the lane's slot takes its partials now, the warp and block reductions
                    // run once, after the tiles.  32 consecutive words per instruction, no bank conflict; the results
                    // are unused, so nothing waits on them.  A lane's count stays below 2^31: 2 rows x 8 warps x at
                    // most 2^23 tiles.
                    unsigned int* a = &s_fold[p.ops[i].save_index * (kLaneWords * 32u) + lane];
                    if (CKT) { atomicXor(&a[0], uint32_t(hx_t)); atomicXor(&a[32], uint32_t(hx_t >> 32)); }
                    if (CKV) { atomicXor(&a[64], uint32_t(hx_v)); atomicXor(&a[96], uint32_t(hx_v >> 32)); }
                    atomicAdd(&a[128], n_alive);
                    if (bad) atomicOr(&a[128], 0x80000000u);
                } else {
                    // warp-level fold (REDUX) now, shared-memory atomics at the NEXT save (or after the op
                    // loop): the REDUX latency is covered by the following ADVANCE instead of stalling lane 0
                    flush_pending();
                    const unsigned full = 0xffffffffu;
                    if (CKT) { pend[0] = __reduce_xor_sync(full, uint32_t(hx_t)); pend[1] = __reduce_xor_sync(full, uint32_t(hx_t >> 32)); }
                    if (CKV) { pend[2] = __reduce_xor_sync(full, uint32_t(hx_v)); pend[3] = __reduce_xor_sync(full, uint32_t(hx_v >> 32)); }
                    // one REDUX for two counts: live rows (at most 32 * VEC) in the low half, lanes that saw a non-finite
                    // value in the high half
                    pend[4] = __reduce_add_sync(full, n_alive | (bad << 16));
                    pend_row = p.ops[i].save_index * kAccStride;
                    pend_valid = true;
                }
                if (store && STAMPS) store_active(img, p.ops[i].call_count, held);  // budget: save_store
            } else {  // OP_LOAD  budget: load
                load_active(p.arena + (size_t(p.ops[i].image_off256) << 8), p.ops[i].n_rows, p.ops[i].call_count);
            }
        }
        flush_pending();  // budget: save_fold
        if (p.flags & PF_WRITE_LIVE_ACTIVE) store_active(p.arena, 0u, claim_stamps(0u, p.stamp_base + p.n_ops));  // budget: save_store

        // ------------------------------ passive planes ------------------------------  budget: tile_loop
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
    if (use_tma && tid == 0) tma_wait_all();  // every bulk store has landed before the results are published  budget: epilogue

    // ---- block partials -> global accumulators -> (last block) host-visible results ----
    __syncthreads();
    if (WARP_FOLD) {
        for (uint32_t i = tid; i < p.n_saves * kAccStride; i += BLOCK) {
            unsigned long long v = (unsigned long long)s_fold[2 * i] | ((unsigned long long)s_fold[2 * i + 1] << 32);
            uint32_t c = i % kAccStride;
            if (v) {
                if (c == 6) atomicAdd(&p.accum[i], v);
                else if (c == 7) atomicOr(&p.accum[i], v);
                else atomicXor(&p.accum[i], v);
            }
        }
    } else {
        // one warp per Save: reduce the 32 lane slots of each word, then the same global atomics as above
        const unsigned full = 0xffffffffu;
        for (uint32_t s = tid >> 5; s < p.n_saves; s += BLOCK / 32) {
            const unsigned int* a = &s_fold[s * (kLaneWords * 32u) + lane];
            const unsigned long long t = __reduce_xor_sync(full, a[0]) | ((unsigned long long)__reduce_xor_sync(full, a[32]) << 32);
            const unsigned long long v = __reduce_xor_sync(full, a[64]) | ((unsigned long long)__reduce_xor_sync(full, a[96]) << 32);
            const uint32_t n = __reduce_add_sync(full, a[128] & 0x7FFFFFFFu);  // at most the world's rows
            const bool bad = __any_sync(full, a[128] >> 31);
            if (lane == 0) {
                unsigned long long* acc = &p.accum[s * kAccStride];
                if (t) atomicXor(&acc[p.ck_t_slot], t);
                if (v) atomicXor(&acc[p.ck_v_slot], v);
                if (n) atomicAdd(&acc[6], (unsigned long long)n);
                if (bad) atomicOr(&acc[7], 1ULL);
            }
        }
    }
    if (p.trace && tid == 0 && s_stored) atomicAdd(&p.trace[3], (unsigned long long)s_stored);
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
// The last entry of a table of `n` whose `key` is <= g: the entry global index g belongs to, for tables in ascending key
// order where an entry owns [its key, the next entry's key).  An entry that owns nothing shares the next one's key and
// comes before it, so it is never found.
template <class Entry, class Key>
__device__ __forceinline__ uint32_t table_entry_of(const Entry* tab, uint32_t n, Key Entry::*key, uint64_t g) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1u) {
        const uint32_t mid = (lo + hi) >> 1;
        if (uint64_t(tab[mid].*key) <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// one spawning world of a batched edit call (bgr_batch_apply_edits): rows [first_row, first_row + count) of its image
// 0, global spawned rows [row0, row0 + count)
struct SpawnWorld {
    uint8_t* img;
    uint32_t row0, first_row, count, pad;
};
static_assert(sizeof(SpawnWorld) == 24, "SpawnWorld layout (the engine and the kernels must agree)");

// `commands.spawn((..., Rollback))`: zeroed components, alive = 1.  kTable: `count` rows over every world of `worlds`
// (bgr_batch_apply_edits; img and first_row unused), each row's world found by binary search.  Otherwise rows
// [first_row, first_row + count) of `img`.
template <bool kTable>
__global__ void __launch_bounds__(256) k_spawn_rows(uint8_t* img, uint32_t words, uint32_t first_row, uint32_t count,
                                                    const SpawnWorld* worlds, uint32_t n_worlds) {
    const size_t n = size_t(count) * (words + 1);
    for (size_t t = size_t(blockIdx.x) * blockDim.x + threadIdx.x; t < n; t += size_t(gridDim.x) * blockDim.x) {
        const uint32_t i = uint32_t(t / (words + 1)), w = uint32_t(t % (words + 1));
        uint8_t* im = img;
        uint32_t row = first_row + i;
        if (kTable) {
            const SpawnWorld s = worlds[table_entry_of(worlds, n_worlds, &SpawnWorld::row0, i)];
            im = s.img;
            row = s.first_row + (i - s.row0);
        }
        if (w < words) *reinterpret_cast<uint32_t*>(im + word_offset(words, row, w)) = 0u;
        else im[alive_offset(words, row)] = 1;
    }
}
__global__ void k_set_alive(uint8_t* img, uint32_t words, uint32_t row, uint8_t value) { img[alive_offset(words, row)] = value; }

// A batch of host edits (bgr_apply_edits) folded by the host into one patch of image 0, read from page-locked memory:
//   words:  (row, plane, value) stores, one per word, sorted by address so that neighbouring threads store neighbouring
//           words of a plane;
//   masks:  (row, and | or << 8 | despawn << 16) per row, the batch's presence records composed in order.  Like
//           k_set_absent they only change a row that is alive here (a queued vector may have despawned it); a despawn
//           clears the byte whatever it held;
//   stamps: indices into image 0's content-stamp row whose stamps become unknown.
// The three lists touch disjoint bytes, so one flat index space covers them in any order.
// bgr_batch_apply_edits patches many worlds in one launch: their words and masks are the concatenation of each world's
// own lists (in list order), and `worlds` (kTable, below) gives each world its share.  Batch members never run the
// bundle kernel, so a batched patch has no stamps.
struct EditWorld {
    uint8_t* img;            // image 0
    uint32_t t0;             // its first global index: its words, then its masks, up to the next entry's t0
    uint32_t n_words;
    uint32_t word0, mask0;   // its first word in `words`, its first mask in `masks`
};
static_assert(sizeof(EditWorld) == 24, "EditWorld layout (the engine and the kernels must agree)");
struct EditPatch {
    const uint4* words;
    const uint2* masks;
    const uint32_t* stamps;
    uint32_t n_words, n_masks, n_stamps;
    const EditWorld* worlds;  // kTable: [n_worlds], ascending t0
    uint32_t n_worlds;
};
__device__ __forceinline__ void edit_word(uint8_t* img, uint32_t words, const uint4 w) {
    *reinterpret_cast<uint32_t*>(img + word_offset(words, w.x, w.y)) = w.z;
}
__device__ __forceinline__ void edit_mask(uint8_t* img, uint32_t words, const uint2 m) {
    uint8_t* a = img + alive_offset(words, m.x);
    if (m.y >> 16) *a = 0;
    else if (*a & 1u) *a = uint8_t((*a & m.y) | (m.y >> 8));
}
// kTable: the patch of every world of p.worlds (img and stamps unused), each index's world found by binary search.
// Otherwise the one world `img` with its stamps, as bgr_apply_edits has always run it.
template <bool kTable>
__global__ void __launch_bounds__(256) k_apply_edits(uint8_t* img, uint32_t words, uint32_t* stamps, const EditPatch p) {
    const uint32_t n = p.n_words + p.n_masks + p.n_stamps;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        if (kTable) {
            const EditWorld w = p.worlds[table_entry_of(p.worlds, p.n_worlds, &EditWorld::t0, t)];
            const uint32_t k = t - w.t0;
            if (k < w.n_words) edit_word(w.img, words, p.words[w.word0 + k]);
            else edit_mask(w.img, words, p.masks[w.mask0 + (k - w.n_words)]);
        } else if (t < p.n_words) {
            edit_word(img, words, p.words[t]);
        } else if (t < p.n_words + p.n_masks) {
            edit_mask(img, words, p.masks[t - p.n_words]);
        } else {
            stamps[p.stamps[t - p.n_words - p.n_masks]] = 0u;
        }
    }
}

// ---- GgrsSchedule systems on the live image (stepwise path) ----
// One registered system (run_system) over rows [0, n_rows), one row per thread.  `kill` receives the despawns;
// k_apply_despawns applies them after every system of the schedule has run (Commands are deferred to the end of GgrsSchedule).
// Eight resident blocks per SM (at most 32 registers): the grid (engine grid_for, 8 blocks per SM) is then one wave, as it
// was with one small kernel per system.  Left to itself the union of all systems takes 37 registers, six blocks per SM,
// and a 1M-entity stepwise tick was 8 % slower (H100 80GB HBM3, 400 W power limit).
__global__ void __launch_bounds__(256, 8) k_sys_rows(uint8_t* img, uint32_t words, uint32_t n_rows, const SysSpec sy,
                                                  const __grid_constant__ Op op,
                                                  unsigned long long order_base, uint8_t* kill) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x) {
        const uint32_t m[1] = {img[alive_offset(words, r)]};
        if (!row_matches(m[0], sy.need)) continue;  // no system touches a row its query does not match: read none of its words
        bool despawn[1] = {false};
        run_system<1>(sy, [&](int, uint32_t plane) -> uint32_t& { return *reinterpret_cast<uint32_t*>(img + word_offset(words, r, plane)); },
                      m, despawn, op, order_base + r, 0u);
        if (despawn[0]) kill[r] = 1;
    }
}

// spawn_particles (particles.rs:258-270) on the live image: rows [first, first+count) become spawn_row's newborn rows
// (`sy` the spawn system's spec), alive.
__global__ void __launch_bounds__(256) k_sys_particles_spawn(uint8_t* img, uint32_t words, const SysSpec sy, uint32_t first, uint32_t count,
                                                             const float2* __restrict__ vals, unsigned long long ttl) {
    for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < count; k += gridDim.x * blockDim.x) {
        const uint32_t r = first + k;
        spawn_row(sy, [&](int, uint32_t plane) -> uint32_t& { return *reinterpret_cast<uint32_t*>(img + word_offset(words, r, plane)); },
                  0, words, vals[k], ttl);
        img[alive_offset(words, r)] = 1;
    }
}

// apply deferred despawn commands: alive &= !kill ; kill = 0
__global__ void __launch_bounds__(256) k_apply_despawns(uint8_t* img, uint32_t words, uint32_t n_rows, uint8_t* kill) {
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += gridDim.x * blockDim.x)
        if (kill[r]) { img[alive_offset(words, r)] = 0; kill[r] = 0; }
}

#endif  // !__CUDACC_RTC__

}  // namespace bgr
