// bevy_ggrs_b200 engine: host logic of the rollback hot path + the C ABI of include/bevy_ggrs_b200.h.
//
// Host side restates, request by request, what handle_requests does to the frame resources
// (reference src/schedule_systems.rs:189-270) and to the snapshot ring (src/snapshot/mod.rs:144-270),
// compiles the whole request vector into a small op program, and launches ONE fused kernel
// (kernels.cuh: k_particles_program) — or, for schemas/systems without a compiled bundle, one
// generic kernel per request ("stepwise" path).  No CPU compute path exists: without a GPU every
// entry point that touches state returns BGR_ERR_CUDA.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>  // header-only; a no-op unless a profiler is attached

#include <algorithm>
#include <array>
#include <cassert>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "content_ids.hpp"
#include "kernels.cuh"
#include "particle_rng.hpp"
#include "ring.hpp"
#include "seahash.cuh"
#include "shard_group.hpp"
#include "tma_copy.cuh"
#include "generic_program.cuh"
#include "desync_diff.cuh"
#include "change_feed.cuh"
#include "frame_digest.cuh"
#include "checkpoint.cuh"
#include "checkpoint_check.hpp"
#include "batch_call.hpp"
#include "edit_batch.hpp"
#include "feed_check.hpp"
#include "replay_keyframes.hpp"
#include "replay_trace.hpp"
#include "jit.hpp"
#include "vmm_range.hpp"
#include "device_memory.hpp"

using namespace bgr;

namespace {

thread_local std::string g_err;
int fail(int status, const std::string& text) { g_err = text; return status; }

#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess)                                                                      \
            return fail(BGR_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
    } while (0)

struct Column {
    std::string name;
    uint32_t elem_bytes = 0, words = 0, first_plane = 0, strategy = 0;
    uint32_t hash_kind = BGR_HASH_NONE, hash_off = 0, hash_len = 0, hash_flags = 0;
    int ck_slot = -1;  // index among checksummed columns (registration order)
    uint32_t absent = 0;  // optional column: its absent bit in the per-row mask byte (kernels.cuh row_matches)
};

struct SystemReg {
    uint32_t id = 0;
    std::vector<uint32_t> cols, params;
};

constexpr uint32_t kReqAdvanceNoBump = 100;  // bgr_advance_world: caller already bumped RollbackFrameCount

constexpr uint32_t kMaxSpawnVals = 1u << 16;  // particles spawned by one request vector

// checksum points one replay launch accumulates (64 MB of accumulators); BGR_TUNE_REPLAY_POINTS lowers it (tests of logs
// that take several launches)
constexpr uint32_t kReplayLaunchPoints = 1u << 20;

// bytes of keyframe images one replay launch stages (bgr_replay_keyframes); a launch always holds at least one keyframe
// of each unfinished world.  256 MB is a choice, not a measurement: a few 1M-row stress frames, or every keyframe of a
// thousand box_game worlds over a minute.  BGR_TUNE_KEYFRAME_BYTES lowers it (tests of replays that take many launches).
constexpr uint64_t kKeyframeLaunchBytes = 256ull << 20;
// bytes of trace records one replay launch stages (bgr_replay_trace), split over the unfinished worlds; a launch always
// holds at least one sample of each.  256 MB is a choice, not a measurement, made like the keyframe budget: every
// sample of a 3 600-frame match tracing 64 rows of 32-byte records at T = 1 is 7.4 MB, so a thousand such worlds take a
// few launches.  BGR_TUNE_TRACE_BYTES lowers it (tests of replays that take many launches).
constexpr uint64_t kTraceLaunchBytes = 256ull << 20;

constexpr uint32_t kMaxDeferredOps = 4;  // trailing ADVANCEs a deferred live image replays (SyncTest / P2P ticks: 1)

// Deferred live image (BGR_TUNE_DEFER_LIVE).  A fused program that ends in `Save(f), Advance...` need not write image 0:
// a Save stores the program's state verbatim and the kernels are bit-deterministic, so image 0 is exactly the base
// slot's image with the trailing ADVANCEs replayed, on every tile the program would have written.  The next program
// starts from the base slot instead (or with its own Load), and entry points that touch image 0 materialise it first.
struct DeferredLive {
    bool active = false;
    bool passive = false;          // the eager program would also have written the passive planes (bundle)
    uint32_t base_off256 = 0;      // the image the program's last stored Save wrote
    uint32_t base_rows = 0;        // RollbackOrdered::len() at that Save
    uint32_t max_rows = 0;         // image 0 is pending on tiles [0, max(1, tiles_for(max_rows)))
    uint32_t n_ops = 0;
    Op ops[kMaxDeferredOps];       // the ADVANCEs after the Save, verbatim
};

// Every host-side resource handle_requests / the schedules mutate.  A request vector is compiled
// against a copy and committed only if the whole vector is valid.
struct HostState {  // trivially copyable: copying it per call must not allocate
    SlotRing ring;
    std::array<uint32_t, SlotRing::kMaxSlots> slot_rows{};        // RollbackOrdered::len() captured by each snapshot (mod.rs:339)
    std::array<uint64_t, SlotRing::kMaxSlots> slot_elapsed_ns{};  // Time<GgrsTime> captured by each snapshot (time.rs:100)
    int32_t frame_count = 0;                // RollbackFrameCount (mod.rs:66-67)
    int32_t confirmed = 0;                  // ConfirmedFrameCount (mod.rs:76-77), init_resource -> 0
    bool has_maxpred = false;               // MaxPredictionWindow inserted? (lib.rs:116-117)
    uint32_t maxpred = 0;
    uint64_t elapsed_ns = 0;                // Time<GgrsTime>::elapsed
    uint32_t n_rows = 0;                    // RollbackOrdered::len()
    uint32_t call_count = 0;                // un-rolled-back counter of BGR_SYS_U32_STORE_CALL_COUNT
    ParticleRng rng;                        // ParticleRng resource (particles.rs:128)
    std::array<ParticleRng, SlotRing::kMaxSlots> slot_rng{};  // its per-snapshot clones
    // Content versions of the passive planes (those no registered system writes).  Every engine relies on:
    //   slot_passive_ver[s] == live_passive_ver  =>  slot s holds the live image's passive bytes on every row below
    //   the row count, dead rows included
    // so a Save into such a slot stores no passive plane (OPF_SKIP_PASSIVE) and a Load from it rewrites none.  A version
    // also fixes the row count: rows grow only through spawns (in a program, bgr_spawn, the startup system), which bump
    // it, and a Load takes the slot's row count with its version, so a matching slot covers every row a later program
    // touches.  Who writes image 0 or a slot, and why the invariant holds:
    //   - compile_requests: a Save takes the live version; a Load makes the slot's version live; a spawn bumps
    //     (newborn rows carry Transform::default()).
    //   - deferred live image: the version is settled when the deferring program compiles.  The materialisation
    //     launch, the prepended LOAD(base) and the early write restore exactly the bytes that version names
    //     (DeferredLive::passive keeps the live passive write the eager program would have made).
    //   - host writes of image 0 bump: transfer_column to the device (bgr_write_component, bgr_insert_component),
    //     bgr_spawn, bgr_run_startup_system, bgr_remove_component.  bgr_despawn writes only the alive byte, an active
    //     plane.  bgr_reset_session, bgr_set_depth and bgr_confirm move no bytes; slots keep bytes and versions.
    //   - bgr_apply_edits (host edits) writes image 0 and bumps only when the batch changes passive bytes or row count:
    //     a WRITE with a word on a passive plane, and every SPAWN, INSERT and REMOVE (what their single calls do).  A
    //     DESPAWN writes the mask byte and a WRITE confined to active planes writes only active words: every slot's
    //     passive bytes still equal the live image's, so a matching version stays true.
    //   - slots are written only by Saves; desync capture and retention hand a slot index out again with its
    //     bytes, and the version is per slot index.
    //   - the stepwise path, the interpreter and k_generic_jit ignore OPF_SKIP_PASSIVE and store whole images, which
    //     keeps the invariant.  A sharded engine keeps its own versions.
    //   - overlapping launches (PF_TILE_WAIT): elision only drops passive reads and stores, and a tick after a bump
    //     stages the passive planes exactly as every tick did before, so no launch reads what an earlier one writes.
    //   - growth (BGR_CFG_GROWABLE, grow_to): maps new memory behind every image's bytes and zeroes it.  Every row it
    //     writes is at or past every image's row count, so no version changes.
    //
    // Content stamps of the active planes (bgr_engine::stamps, engines that run the bundle kernel), the device-side
    // counterpart for the planes the systems write, decided per warp segment because it depends on the values:
    //   stamp[img][seg][q] == S != 0  =>  the bytes of active plane q of 64-row segment seg in image img are exactly
    //   the content that stamp S names.  0 = unknown.
    // Stamps are issued by the host, a fresh range per bundle launch (stamp_base + op index), and never reused: when
    // the 32-bit range runs out the whole table is cleared on the stream and the range starts again.  Who writes:
    //   - the bundle kernel keeps the invariant itself: a Load takes the source's stamps, a plane whose bits a frame
    //     changed (or whose stamp is unknown) gets a fresh stamp at the next Save, a store writes the stamp with the bytes.
    //     Its instance without stamps (single-wave grids, run_fused) stores whole active planes and writes no stamp: it
    //     marks the table stale, and the next stamped launch clears the whole table first.
    //   - every other writer of an image clears that image's stamps (clear_stamps): transfer_column to the device
    //     (bgr_write_component, bgr_insert_component), bgr_spawn, bgr_run_startup_system, bgr_remove_component,
    //     bgr_insert_component's presence bit, and bgr_despawn (the alive byte is an active plane).
    //   - bgr_apply_edits clears only image 0's stamps of the (segment, plane) pairs its patch writes, in the same launch,
    //     behind every queued vector: an active word's plane, the mask byte's plane (q = 8) for presence and despawn
    //     records, every plane of the segments a spawn's rows fall in.  Every other stamp names bytes it did not touch.
    //   - the deferred live image is materialised by the bundle kernel itself; while it is pending, image 0 keeps the
    //     bytes and the stamps of its last write.
    //   - the stepwise path (k_image_tma, k_copy_image), the interpreter and k_generic_jit only run on engines that do
    //     not use the bundle (use_bundle is fixed at bgr_build); those have no stamp table.
    //   - desync capture, retention, digests, export, bgr_reset_session and bgr_set_depth write no image bytes.  A
    //     sharded engine keeps its own table.
    //   - growth maps the table's new segments behind every image's row and zeroes them (unknown); the stamps of the
    //     segments that existed keep their positions and values, as the image bytes they name do.
    //
    // Content ids (content_ids.hpp, engines that run the bundle kernel), which name whole images across launches:
    //   cids.live / cids.slot[s].cid == X != 0  =>  the active planes and alive byte of image 0 / slot s, on every row
    //   below its row count, are exactly the bytes derivation X produces, and the row count is X's
    // A Save whose target slot already holds the registers' id (and row count) is held (OPF_HELD): the bundle kernel
    // stores nothing of it and still checksums the registers.  In the steady state of a SyncTest the re-simulation
    // from f-d repeats the last tick's Advances on the same content and gets back the same slots (SlotRing frees LIFO),
    // so every re-save is held and only the new frame is stored.  Who writes an image, and why the invariant holds:
    //   - derive_content_ids, on the final op list (after consume_deferred rewrote it, before the launch): a LOAD takes
    //     the slot's record, an ADVANCE takes the id of a slot derived from the same content by an ADVANCE with the same
    //     key (advance_key: every Op field the result depends on) or a fresh id, an ADVANCE that spawns a fresh id, a
    //     SAVE gives the target the registers' record, the program's end gives it to image 0.  The derivation is exact:
    //     equal ids mean equal derivations, never equal hashes.
    //   - the deferred live image: cids.live names the image the deferring program would have written, and its record
    //     (base slot's id, the last ADVANCE's key) is searched like a slot's (ContentIds::advance).  The prepended
    //     [LOAD(base), pending ADVANCEs] derives that same id from the base slot; the materialisation holds no Save.
    //   - every host write of an image goes through clear_stamps, which also gives the image a fresh id:
    //     transfer_column to the device (bgr_write_component, bgr_insert_component), bgr_spawn, the startup system,
    //     bgr_remove_component, bgr_insert_component's presence bit, bgr_despawn, and bgr_checkpoint_restore (image 0
    //     and the restored slot).  bgr_apply_edits writes image 0 in its own launch and gives it a fresh id itself.
    //   - growth, desync capture, retention, bgr_reset_session and bgr_set_depth move no bytes below a row count; ids
    //     stay with their slot indices as the bytes do.
    //   - every clear of the stamp table (range rollover, stamps_stale) forgets every id (cids.epoch), and the launch
    //     that clears it stores its held Saves after all: a vector at a clear stores everything, as it did before.
    //   - only the bundle kernel honours OPF_HELD; an engine that runs any other kernel derives no ids.  A sharded
    //     engine keeps its own ids.
    uint64_t live_passive_ver = 1, ver_counter = 1;
    std::array<uint64_t, SlotRing::kMaxSlots> slot_passive_ver{};  // 0 = never written
    ContentIds<SlotRing::kMaxSlots> cids;
};
static_assert(std::is_trivially_copyable<HostState>::value, "handle_requests copies HostState on every call");

// The patch k_apply_edits applies (kernels.cuh EditPatch), folded on the host from a validated batch.  The engine keeps
// one across calls: a batch of thousands of rows allocated (and page-faulted) a megabyte of fresh memory otherwise.
struct EditFold {
    struct Word { uint64_t key; uint32_t row, plane, value; };  // key: the word's offset in image 0 / 4
    std::vector<Word> words, sorted;
    std::vector<uint2> masks;                // (row, and | or << 8 | despawn << 16)
    std::vector<uint32_t> stamps;
    std::unordered_map<uint32_t, uint32_t> mask_of;  // row -> index into masks
    bool bump = false;                       // the live passive version moves (HostState)
    // per word plane, fixed at bgr_build and filled by the first batch: its content-stamp plane (kernels.cuh:
    // translation, velocity, ttl; the mask byte is q = 8; -1 passive; empty without a stamp table) and whether it is
    // a passive plane
    std::vector<int8_t> stamp_q;
    std::vector<uint8_t> passive;
    void clear() { words.clear(); masks.clear(); stamps.clear(); mask_of.clear(); bump = false; }
};

struct Pending {
    uint32_t buf = 0;
    unsigned long long seq = 0;
    unsigned long long gseq = 0;    // shard group sequence number (0: not in a group)
    bool finished = false;          // the GPU work is known to be complete (drain() synchronised the stream)
    uint32_t n_saves = 0;
    int32_t frames[kMaxSaves];
    uint32_t totals[kMaxSaves];
};

float duration_as_secs_f32(uint64_t ns) {  // core::time::Duration::as_secs_f32
    uint64_t secs = ns / 1000000000ULL;
    uint32_t nanos = uint32_t(ns % 1000000000ULL);
    return float(secs) + float(nanos) / 1000000000.0f;
}
uint32_t f32_bits(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }

uint64_t host_ns() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return uint64_t(ts.tv_sec) * 1000000000ULL + uint64_t(ts.tv_nsec);
}

// The reference's tracing spans as NVTX ranges (no-ops unless a profiler is attached): `HandleRequests` around the
// whole call (schedule_systems.rs:171) and `SaveWorld` / `LoadWorld` / `AdvanceWorld` per request (:224-253) — around
// the host half of each request (ring push / rollback, frame resources, GgrsTime) while the vector is compiled, and
// around each request's kernel launches on the stepwise path.  On the fused paths the device half of all requests is
// ONE launch, which sits inside the HandleRequests range.
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
inline const char* span_name(uint32_t request_kind) {
    return request_kind == BGR_REQ_SAVE ? "SaveWorld" : request_kind == BGR_REQ_LOAD ? "LoadWorld" : "AdvanceWorld";
}

int env_int(const char* name, int dflt) {
    const char* v = std::getenv(name);
    return v && *v ? std::atoi(v) : dflt;
}

}  // namespace

struct bgr_engine {
    bgr_config cfg{};
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int num_sms = 0;

    std::vector<Column> cols;
    std::vector<SystemReg> systems;
    // the registration as every kernel reads it, fixed at bgr_build (build_specs): one SysSpec per system in schedule
    // order (and whether it can despawn), one HashSpec per checksummed column
    std::vector<SysSpec> sys_specs;
    std::vector<bool> sys_despawns;
    std::vector<HashSpec> hash_specs;
    uint32_t n_ck = 0;
    bool built = false;

    uint32_t epad = 0, words = 0, tile_bytes = 0, n_tiles_cap = 0;
    size_t image_bytes = 0;
    StridedRange arena;  // image 0 = live, image s+1 = slot s (tile-planar, kernels.cuh)
    StridedRange kill;
    DeviceBuffer<uint8_t> stage;  // device staging for ECS column <-> image transposition
    // asynchronous mirror downloads: packed on the main stream, copied D2H on copy_stream
    struct Download { DeviceBuffer<uint8_t> buf; Event packed, done; bool busy = false; };
    Download dl[BGR_MAX_DOWNLOADS];
    cudaStream_t copy_stream = nullptr;
    uint32_t next_dl = 0;
    // change feeds (bgr_feed_*, change_feed.cuh): reported state in HBM, both passes on the main stream, the records
    // cross PCIe on copy_stream
    struct Feed {
        bool used = false, busy = false;
        FeedParams p{};              // fields, keep, rep_words, record_words, p.one.rep and views of the buffers below
        uint32_t bound = 0;          // no row at or past it has a reported state other than (0, zeros)
        uint32_t ticket = 0;         // of the report in flight (single or batched)
        StridedRange rep, count;     // p.one.rep, and p.tile_count / tile_off / tile_list one stride each
        DeviceBuffer<unsigned int> info;  // [8]: p.info [4], p.head [2], p.world_scan [2]
        DeviceBuffer<uint32_t> out;  // the records of a report
        MappedHostBuffer<unsigned int> h_info;  // [4]: the info, copied behind the records
        Event packed, done;
    };
    Feed feeds[BGR_MAX_FEEDS];
    uint32_t feed_seq = 0;
    // host edits (bgr_apply_edits): page-locked patches the kernel reads in place, reused once their launch finished
    struct EditStage { MappedHostBuffer<uint8_t> h; Event done; bool busy = false; };
    static constexpr int kEditBufs = 4;
    EditStage edit_stage[kEditBufs];
    uint32_t next_edit = 0;
    EditFold edit_fold;

    HostState st;

    static constexpr int kBufs = 8;  // result / spawn buffers = max un-collected submits (== PendingRing capacity)
    // accumulator / ticket sets: one per in-flight request vector, so that overlapping launches (tile dependencies)
    // never share one; set 0 serves every launch that overlaps nothing
    unsigned long long* d_accum_set[kBufs] = {};
    unsigned int* d_ticket_set[kBufs] = {};
    DeviceBuffer<unsigned long long> accum;
    DeviceBuffer<unsigned int> ticket;
    MappedHostBuffer<float2> spawn[kBufs];  // (vx, vy) of spawned particles
    int spawn_sys = -1;             // index of BGR_SYS_PARTICLES_SPAWN in `systems`, or -1
    // result blocks: views of the engine's own (out_block) or, in a shard group, of the group's segment
    MappedHostBuffer<unsigned long long> out_block[kBufs];
    unsigned long long* h_out[kBufs] = {};
    unsigned long long* d_out[kBufs] = {};
    Event ev[kBufs];
    // un-collected request vectors, oldest first: a fixed ring (a std::deque allocated a chunk per push — the hot path
    // allocates nothing)
    struct PendingRing {
        Pending slot[8];
        uint32_t head = 0, count = 0;
        bool empty() const { return count == 0; }
        size_t size() const { return count; }
        void push_back(const Pending& p) { slot[(head + count) % 8u] = p; ++count; }
        Pending& front() { return slot[head]; }
        void pop_front() { head = (head + 1u) % 8u; --count; }
        template <class F> void for_each(F f) { for (uint32_t i = 0; i < count; ++i) f(slot[(head + i) % 8u]); }
    } pending;
    uint32_t next_buf = 0;
    std::vector<bgr_partial> last_partials;

    // shard group (multi-GPU): result blocks live in a shared host segment every rank's GPU and CPU map
    ShardGroup* group = nullptr;
    unsigned long long gseq = 0;
    bool ticked = false;            // a request vector has been executed (the initial population is over)
    DeferredLive deferred;          // committed by submit() together with `st`
    bool live_touched = false;      // an entry point read or wrote image 0 since the last submit: the next one stays eager
    int tune_defer_live = 1;        // 0: every fused program writes image 0 itself
    DeviceBuffer<unsigned long long> internal_out;  // result block of internal launches (materialisation)
    // device-side launch trace (bgr_trace_enable): per launch [first block start, last block end] in globaltimer ns
    DeviceBuffer<unsigned long long> trace;
    uint32_t trace_cap = 0;
    unsigned long long trace_first_seq = 0;

    uint64_t launches = 0;
    uint64_t prof[8] = {};          // host-side time of the hot loop: [0] calls, [1] compile ns, [2] launch ns, [3] wait ns, [4] fold ns
    bool last_fused = false;
    uint32_t last_kernel = BGR_KERNEL_NONE;  // bgr_last_kernel: what the last request vector ran
    unsigned long long seq = 0;   // sequence number of the last submit (completion flag value)
    int tune_poll = 1;            // collect() spins on the host-mapped flag before falling back to the event
    int tune_tiledep = 1;         // consecutive fused launches overlap: per-tile dependencies instead of grid-level (PF_TILE_WAIT)
    StridedRange tile_done;       // [tiles + 1] see ProgramParams::tile_done
    StridedRange tile_cnt;
    bool tiledep_chain = false;   // the last operation enqueued on the main stream was a PF_TILE_SIGNAL launch
    uint32_t tiledep_seq = 0, tiledep_tiles = 0;
    int tune_grid = 0;            // experiment / tests: cap the one-launch kernels' grid (0 = SMs x resident blocks)
    int tune_prefetch = 1;        // L2 prefetch of the next tile's active planes
    int tune_dynamic = 1;         // dynamic tile scheduling in the fused kernel (measured +5% over a static stride)

    // compiled bundle: particles (update_particles + despawn_particles)
    bool bundle_particles = false;
    uint32_t bt = 0, bv = 0, bl = 0;
    std::vector<uint16_t> passive;
    std::vector<PassiveRun> runs;
    uint32_t passive_bytes = 0;
    StridedRange stamps;            // content stamps of the active planes (HostState): [images][segments][kActivePlanes]
    uint32_t stamp_next = 1;        // first stamp of the next bundle launch
    bool stamps_stale = false;      // a bundle launch without stamps wrote images since the table was last cleared
    uint64_t stamp_epoch = 0;       // clears of the whole stamp table (HostState::cids forgets every id at one)
    // held Saves (HostState content ids).  BGR_TUNE_HELD_SAVES: 0 store every Save, 1 hold (default), 2 hold and
    // compare each held Save's target with the registers (mismatching words counted in held_check)
    int tune_held_saves = 1;
    uint32_t last_held = 0;         // held Saves of the last request vector
    uint64_t held_total = 0;        // ... of every request vector
    DeviceBuffer<unsigned long long> held_check;
    bool bundle_static_ck = false;  // both columns checksummed with the finite assertion: fully specialised kernel
    // generic one-launch program (generic_program.cuh): any schema whose tile fits shared memory + the compiled systems
    bool generic_ok = false;
    int generic_bps = 0;            // resident blocks per SM of k_generic_program (occupancy query, cached)
    int tune_jit = 1;               // 0 never, 1 worlds of >= 16k entities, 2 always: NVRTC-specialised generic program (jit.hpp)
    int tune_jit_rows = 4;          // rows of a tile per thread in the specialised kernel (1, 2, 4)
    JitKernel jit;                  // fn == nullptr: the interpreter kernel runs.  Work item = a whole tile
    JitKernel jit_small;            // the same kernel with quarter-tile work items: worlds of few tiles per SM (optional)
    int tune_jit_tiledep = 0;       // 1: consecutive launches of the generated kernel overlap through per-item dependencies (queued submits)
    StridedRange item_done;         // [4 * tiles + 4] GenericParams::item_done (quarter-tile work items at most)
    // replays (bgr_replay): the generated kernel of an engine that has none (compiled by its first replay; whole tiles and
    // 128-row items), and the device copies of a call's logs, spawn tables, records and checksum accumulators
    JitKernel replay_jit, replay_jit_small;
    uint32_t tune_replay_points = 0;  // checksum points per replay launch (kReplayLaunchPoints unless BGR_TUNE_REPLAY_POINTS)
    DeviceBuffer<uint8_t> replay_stage;
    uint64_t tune_keyframe_bytes = 0;  // keyframe images one replay launch stages (kKeyframeLaunchBytes unless BGR_TUNE_KEYFRAME_BYTES)
    uint64_t tune_trace_bytes = 0;     // trace records one replay launch stages (kTraceLaunchBytes unless BGR_TUNE_TRACE_BYTES)
    DeviceBuffer<unsigned long long> replay_acc;
    const void* jit_chain_kernel = nullptr;  // the signalling launch `tiledep_chain` refers to (its work-item partition must match)
    int tune_jit_item = 0;          // 0 auto (quarter tiles below 3 tiles per SM), 512 / 256 / 128 force the rows per work item
    int tune_passive_early = -1;    // -1: early passive stores for single-wave grids (auto); 0 never; 1 always
    int tune_stagger_ns = 800;      // start-of-grid phase stagger between the resident blocks of an SM (synchronous launches; measured -1.3 %)
    int tune_generic = 1;
    int tune_bundle = 1;            // 0: never use the specialised particles kernel (A/B tests of the generic program)
    bool bundle_opt = false;        // a registered column is BGR_STRATEGY_OPTIONAL: the presence-aware kernel variant (MODE 2)
    int tune_bps = 0, tune_passive_tma = 1;
    int tune_tma = 1;          // stepwise Save/Load through the TMA-staged bulk-copy kernel
    uint32_t tma_stage_tiles = 0;  // one-tile stages of the TMA copy kernel (0: schema too wide for two stages of shared memory)
    DeviceBuffer<unsigned int> tma_ticket;
    // [WARP_FOLD][passive TMA][MODE][STAMPS][VERIFY][Saves in the vector]: blocks per SM of k_particles_program
    int occ_cache[2][2][3][2][2][kMaxSaves + 1] = {};
    int snap_fits = -1;              // -1 unknown; 0: the stamp-point snapshot would cost the passive-TMA launches a block per SM
    // desync diff scratch (BGR_CFG_DESYNC_CAPTURE), allocated by the first bgr_desync_diff
    DeviceBuffer<DiffColumn> diff_cols;
    DeviceBuffer<unsigned int> diff_counts;      // [n_cols][3] then the per-tile record counts
    DeviceBuffer<unsigned long long> diff_totals;
    DeviceBuffer<unsigned int> diff_list;        // [2 * tiles]
    DeviceBuffer<DiffRecord> diff_records;
    // P2P desync reports: retention of confirmed frames (bgr_retain_confirmed) and the digest / remote diff scratch,
    // allocated by their first use
    uint32_t retain_interval = 0, retain_count = 0;
    DeviceBuffer<DigestColumn> digest_cols;
    DeviceBuffer<ImageEntry> digest_table;          // bgr_frame_digest's one-image table
    DeviceBuffer<unsigned long long> digest_words;  // [tiles][n_cols + 1]
    DeviceBuffer<unsigned int> digest_active;       // [tiles]
    DeviceBuffer<uint8_t> remote;                   // tiles uploaded from a peer's export blob
    DeviceBuffer<unsigned int> remote_visit;        // [n_tiles_cap] the local tiles a remote diff visits

    // BGR_CFG_GROWABLE: cfg.max_entities, epad and n_tiles_cap are the current capacity, image_bytes (and stamp_image())
    // the fixed stride of an image, sized for the ceiling.  Every buffer whose size follows the capacity and that a
    // queued launch may use is a strided range (vmm_range.hpp, capacity_buffers) that grow_to maps further; none of their
    // pointers ever changes.
    uint32_t ceiling = 0;  // most rows the engine can hold (== the capacity without the flag)

    uint8_t* image(uint32_t idx) const { return arena.ptr() + size_t(idx) * image_bytes; }
    bool capture() const { return cfg.flags & BGR_CFG_DESYNC_CAPTURE; }
    bool growable() const { return cfg.flags & BGR_CFG_GROWABLE; }
    uint32_t stamp_words() const { return n_tiles_cap * kSegsPerTile * kActivePlanes; }  // stamps of one image's rows
    uint32_t stamp_image() const { return uint32_t(stamps.stride / sizeof(uint32_t)); }  // words between two images' stamps
    // frame slots behind the live image
    uint32_t n_slots() const { return (capture() ? 2u * cfg.max_depth : cfg.max_depth) + retain_count; }
    uint32_t image_off256(uint32_t idx) const { return uint32_t((size_t(idx) * image_bytes) >> 8); }
    uint32_t tiles_for(uint32_t rows) const { return (rows + kTileRows - 1) / kTileRows; }
    uint32_t grid_for(uint32_t n, uint32_t per_block) const {
        uint32_t need = (n + per_block - 1) / per_block;
        uint32_t cap = uint32_t(num_sms) * 8u;
        return std::max(1u, std::min(need, cap));
    }
};

namespace {

// A write outside the bundle kernel: image `idx`'s content stamps become unknown and its content id fresh (HostState).
// Stream-ordered behind every launch that could still write them.
int clear_stamps(bgr_engine* e, uint32_t idx) {
    ContentIds<SlotRing::kMaxSlots>& c = e->st.cids;
    if (idx == 0) c.live = c.fresh(e->st.n_rows);
    else c.slot[idx - 1] = c.fresh(e->st.slot_rows[idx - 1]);
    if (e->stamps.empty()) return BGR_OK;
    CUDA_TRY(cudaMemsetAsync(e->stamps.ptr<uint32_t>() + size_t(idx) * e->stamp_image(), 0, size_t(e->stamp_words()) * sizeof(uint32_t), e->stream));
    e->tiledep_chain = false;
    return BGR_OK;
}

// The whole stamp table: the stamps of every image's rows (one memset while the images' stamps are contiguous).
int clear_stamp_table(bgr_engine* e) {
    CUDA_TRY(e->stamps.zero(0, size_t(e->stamp_words()) * sizeof(uint32_t), e->stream));
    e->tiledep_chain = false;
    e->stamp_epoch += 1;
    return BGR_OK;
}

// ---------------------------------------------------------------------------------------------
// compile: requests -> ops, mutating `s` exactly like handle_requests mutates the World
// ---------------------------------------------------------------------------------------------
struct Program {
    Op ops[kMaxOps];
    uint32_t n_ops = 0, n_saves = 0;
    int32_t save_frames[kMaxSaves];
    uint32_t save_totals[kMaxSaves];
    uint32_t max_rows = 0, live_rows = 0;
    uint64_t rows_needed = 0;        // BGR_CFG_GROWABLE: the capacity the spawns need, when more than the engine has
    bool has_load = false, has_advance = false, first_is_load = false, has_spawn = false;
    bool passive_to_slots = false;   // at least one SAVE must (re)write the passive planes
    bool passive_to_live = false;    // a LOAD changed the content of the live passive planes
    bool defer_live = false;         // launch without the live-write flags (DeferredLive)
    bool from_deferred = false;      // ops[0] is the LOAD of a deferred live image's base slot, followed by its ADVANCEs
    bool internal = false;           // not a request vector: own result block, no trace row, no overlap with other launches
    std::vector<float2> spawn_vals;
    bool writes_live_passive() const { return (has_load && passive_to_live) || has_spawn; }
};

int compile_requests(bgr_engine* e, HostState& s, const bgr_session_info* sess, const bgr_request* reqs, uint32_t n,
                     Program& pg) {
    if (n > kMaxOps) return fail(BGR_ERR_CAPACITY, "too many requests in one handle_requests call");
    pg.live_rows = s.n_rows;
    pg.max_rows = s.n_rows;
    uint32_t n_counter_systems = 0;
    for (auto& sy : e->systems) n_counter_systems += (sy.id == BGR_SYS_U32_STORE_CALL_COUNT);
    for (uint32_t i = 0; i < n; ++i) {
        const bgr_request& rq = reqs[i];
        NvtxRange span(span_name(rq.kind));
        // schedule_systems.rs:190-220 — resources recomputed from the session before every request
        const int32_t current_frame = s.frame_count;
        if (sess) {
            switch (sess->kind) {
            case BGR_SESSION_P2P:
                s.has_maxpred = true; s.maxpred = sess->max_prediction;
                s.confirmed = sess->confirmed_frame;
                break;
            case BGR_SESSION_SYNCTEST: {
                s.has_maxpred = true; s.maxpred = sess->max_prediction;
                int32_t cf = current_frame - int32_t(sess->check_distance);
                if (cf >= 0) s.confirmed = cf;
                break;
            }
            case BGR_SESSION_SPECTATOR:
                s.has_maxpred = true; s.maxpred = 0;
                s.confirmed = current_frame;
                break;
            default: break;
            }
        }
        Op& op = pg.ops[pg.n_ops];
        std::memset(&op, 0, sizeof op);
        switch (rq.kind) {
        case BGR_REQ_SAVE: {  // :223-237 -> SaveWorld: sync_depth, discard_old_snapshots, save (component_snapshot.rs:135-144)
            if (pg.n_saves >= kMaxSaves) return fail(BGR_ERR_CAPACITY, "too many SaveGameState requests in one call");
            if (s.has_maxpred) s.ring.set_depth(s.maxpred);
            s.ring.confirm(s.confirmed);
            uint32_t slot = s.ring.push(s.frame_count);
            if (slot == SlotRing::kNoSlot)
                return fail(BGR_ERR_CAPACITY, "snapshot ring needs more frame slots than bgr_config.max_depth");
            op.kind = OP_SAVE;
            if (slot == SlotRing::kNoSlot - 1) { op.flags |= OPF_NO_STORE; op.image_off256 = 0; }
            else {
                op.image_off256 = e->image_off256(slot + 1);
                s.slot_rows[slot] = s.n_rows;
                s.slot_elapsed_ns[slot] = s.elapsed_ns;
                s.slot_rng[slot] = s.rng;
                if (s.slot_passive_ver[slot] == s.live_passive_ver)
                    op.flags |= OPF_SKIP_PASSIVE;
                else
                    pg.passive_to_slots = true;
                s.slot_passive_ver[slot] = s.live_passive_ver;
            }
            op.n_rows = s.n_rows;
            op.save_index = pg.n_saves;
            pg.save_frames[pg.n_saves] = rq.frame;
            pg.save_totals[pg.n_saves] = s.n_rows;
            ++pg.n_saves;
            break;
        }
        case BGR_REQ_LOAD: {  // :238-250 -> LoadWorld
            s.frame_count = rq.frame;
            std::string err;
            if (!s.ring.rollback(rq.frame, &err)) return fail(BGR_ERR_NO_SNAPSHOT, err);
            uint32_t slot = 0;
            if (!s.ring.get(&slot, &err)) return fail(BGR_ERR_NO_SNAPSHOT, err);
            s.n_rows = s.slot_rows[slot];
            s.elapsed_ns = s.slot_elapsed_ns[slot];
            s.rng = s.slot_rng[slot];
            if (s.slot_passive_ver[slot] != s.live_passive_ver)
                pg.passive_to_live = true;
            s.live_passive_ver = s.slot_passive_ver[slot];
            op.kind = OP_LOAD;
            op.image_off256 = e->image_off256(slot + 1);
            op.n_rows = s.n_rows;
            if (pg.n_ops == 0) pg.first_is_load = true;
            pg.has_load = true;
            break;
        }
        case BGR_REQ_ADVANCE:
        case kReqAdvanceNoBump: {  // :251-269 -> AdvanceWorld
            if (rq.kind == BGR_REQ_ADVANCE) s.frame_count += 1;
            if (rq.n_players > BGR_MAX_PLAYERS) return fail(BGR_ERR_INVALID_ARGUMENT, "n_players > BGR_MAX_PLAYERS");
            // GgrsTimePlugin::update (time.rs:63-76): advance_to(frame * 1e9 / fps)
            uint64_t runtime = uint64_t(int64_t(s.frame_count)) * 1000000000ULL / uint64_t(e->cfg.fps);
            if (runtime < s.elapsed_ns)
                return fail(BGR_ERR_STATE, "tried to move Time<GgrsTime> backwards (RollbackFrameCount went back without LoadWorld)");
            uint64_t delta = runtime - s.elapsed_ns;
            s.elapsed_ns = runtime;
            op.kind = OP_ADVANCE;
            op.dt_bits = f32_bits(duration_as_secs_f32(delta));
            // move_cube_system's friction (box_game.rs:188-193) with the C library's powf, as the reference evaluates it
            op.fr_bits = f32_bits(powf(0.0018f, duration_as_secs_f32(delta)));
            op.n_rows = s.n_rows;
            op.call_count = s.call_count;
            s.call_count += n_counter_systems;
            for (uint32_t k = 0; k < BGR_MAX_PLAYERS && k < rq.n_players; ++k) op.inputs[k] = rq.inputs[k];
            op.flags |= (rq.n_players & 0xFu) << 8;  // PlayerInputs<T>.len() for systems that index it (box_game.rs:171)
            pg.has_advance = true;
            if (e->spawn_sys >= 0) {  // spawn_particles.run_if(spawn_pressed) (particles.rs:236, 254-256)
                bool pressed = false;
                for (uint32_t k = 0; k < rq.n_players; ++k) pressed = pressed || (rq.inputs[k] & BGR_INPUT_SPAWN);
                if (pressed) {
                    const SystemReg& sy = e->systems[size_t(e->spawn_sys)];
                    const uint32_t rate = sy.params[0];
                    if (uint64_t(s.n_rows) + rate > e->cfg.max_entities) {
                        if (!e->growable()) return fail(BGR_ERR_CAPACITY, "spawn_particles exceeds max_entities");
                        pg.rows_needed = std::max(pg.rows_needed, uint64_t(s.n_rows) + rate);  // submit grows first
                    }
                    if (pg.spawn_vals.size() + rate > kMaxSpawnVals)
                        return fail(BGR_ERR_CAPACITY, "too many particles spawned by one request vector");
                    op.flags |= OPF_SPAWN;
                    op.image_off256 = s.n_rows;                      // first spawned row
                    op.save_index = rate;                            // count
                    op.call_count = uint32_t(pg.spawn_vals.size());  // offset into spawn_vals
                    for (uint32_t k = 0; k < rate; ++k) {            // particles.rs:262-268
                        float2 v;
                        v.x = s.rng.random_range(-200.0f, 200.0f);
                        v.y = s.rng.random_range(-200.0f, 200.0f);
                        pg.spawn_vals.push_back(v);
                    }
                    s.n_rows += rate;  // Rollback on_add -> RollbackOrdered.push, applied at the end of the frame
                    s.live_passive_ver = ++s.ver_counter;  // newborn rows carry Transform::default() rotation / scale
                    pg.has_spawn = true;
                    pg.max_rows = std::max(pg.max_rows, s.n_rows);
                }
            }
            break;
        }
        default: return fail(BGR_ERR_INVALID_ARGUMENT, "unknown request kind");
        }
        pg.max_rows = std::max(pg.max_rows, op.n_rows);
        ++pg.n_ops;
    }
    return BGR_OK;
}

// The fields of an ADVANCE op its result depends on (content_ids.hpp).  A spawning ADVANCE also depends on the
// spawned values: it never derives a known id.
AdvanceKey advance_key(const Op& op) {
    AdvanceKey k;
    k.dt_bits = op.dt_bits; k.fr_bits = op.fr_bits; k.n_rows = op.n_rows; k.call_count = op.call_count;
    k.n_players = (op.flags >> 8) & 0xFu;
    std::memcpy(k.inputs, op.inputs, sizeof k.inputs);
    return k;
}

// Content ids through the final op list of a bundle program (HostState), and OPF_HELD on every Save whose target slot
// already holds the registers' content and row count (ContentIds::save).  A held Save must also skip the passive
// planes: it then stores nothing at all.
void derive_content_ids(bgr_engine* e, HostState& s, Program& pg) {
    ContentIds<SlotRing::kMaxSlots>& c = s.cids;
    c.sync_epoch(e->stamp_epoch);  // a clear of the stamp table since the last program forgets every id
    auto slot_of = [&](const Op& op) { return uint32_t((size_t(op.image_off256) << 8) / e->image_bytes) - 1u; };
    ContentRecord reg = c.live;  // the registers' content
    for (uint32_t i = 0; i < pg.n_ops; ++i) {
        Op& op = pg.ops[i];
        if (op.kind == OP_LOAD) {
            reg = c.slot[slot_of(op)];
        } else if (op.kind == OP_ADVANCE) {
            reg = (op.flags & OPF_SPAWN) ? c.fresh(op.n_rows + op.save_index) : c.advance(reg, advance_key(op));
        } else if (!(op.flags & OPF_NO_STORE)) {
            const bool may_hold = e->tune_held_saves && (op.flags & OPF_SKIP_PASSIVE);
            if (c.save(slot_of(op), reg, op.n_rows, may_hold)) op.flags |= OPF_HELD;
        }
    }
    c.live = reg;
}

// ---------------------------------------------------------------------------------------------
// launch: fused bundle kernel
// ---------------------------------------------------------------------------------------------
// Every instance opts into the most dynamic shared memory any launch of it can ask for (a 96 KB passive double buffer,
// the snapshot and 40 Saves' lane slots), so that no engine lowers the limit another engine's launches rely on.
constexpr size_t kBundleSmemMax = 96u * 1024u + kSnapBytes + fold_bytes(false, kMaxSaves);

// blocks per SM of one k_particles_program instance at `smem` bytes of dynamic shared memory
template <int MODE, bool STAMPS, bool VERIFY, bool WARP_FOLD>
int bundle_blocks_per_sm(size_t smem, int& nb) {
    auto kern = k_particles_program<MODE, STAMPS, VERIFY, WARP_FOLD>;
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kBundleSmemMax)));
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, int(kTileRows) / 2, smem));
    return BGR_OK;
}

// A mode runs with and without the passive double buffer (spawns and multi-Load vectors move passive planes per
// thread), and the checksum partials grow with the vector's Saves: the occupancy is per (fold, buffer, mode, Saves).
// passive_bytes is fixed at bgr_build, so one entry per setting is exact.  The stamped instances also hold the
// stamp-point snapshot.
template <int MODE, bool STAMPS, bool VERIFY, bool WARP_FOLD>
int bundle_occupancy(bgr_engine* e, size_t base, uint32_t n_saves, int ti, int& nb) {
    int& occ = e->occ_cache[WARP_FOLD ? 1 : 0][ti][MODE][STAMPS ? 1 : 0][VERIFY ? 1 : 0][n_saves];
    if (occ == 0) {
        int n = 0;
        if (int rc = bundle_blocks_per_sm<MODE, STAMPS, VERIFY, WARP_FOLD>(base + fold_bytes(WARP_FOLD, n_saves), n); rc != BGR_OK) return rc;
        occ = std::max(1, n);
    }
    nb = occ;
    return BGR_OK;
}

template <int MODE, bool STAMPS, bool VERIFY, bool WARP_FOLD>
int launch_bundle(bgr_engine* e, const ProgramParams& pp, size_t smem, int occ) {
    auto kern = k_particles_program<MODE, STAMPS, VERIFY, WARP_FOLD>;
    constexpr int kBlock = int(kTileRows) / 2;  // two rows per thread
    const int ti = (pp.flags & PF_PASSIVE_TMA) ? 1 : 0;
    int bps = occ;
    if (e->tune_bps > 0) bps = std::min(e->tune_bps, bps);
    uint32_t grid = std::max(1u, std::min(pp.n_tiles, uint32_t(e->num_sms * bps)));
    if (e->tune_grid > 0) grid = std::min(grid, uint32_t(e->tune_grid));
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(grid); lc.blockDim = dim3(kBlock); lc.dynamicSmemBytes = smem; lc.stream = e->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = attr; lc.numAttrs = (pp.flags & PF_TILE_WAIT) ? 1 : 0;
    CUDA_TRY(cudaLaunchKernelEx(&lc, kern, pp));
    CUDA_TRY(cudaGetLastError());
    e->launches += 1;
    // bit 12: the passive-TMA configuration (double buffer, its own opt-in and occupancy); whether this launch moved any
    // passive plane at all is BGR_KERNEL_PASSIVE_PLANES: a steady-state tick whose slots already hold them moves none
    const bool passive = pp.n_runs > 0 || pp.n_passive > 0;
    // VEC 2, launch-bounds tier 1 (768 threads per SM), whole-tile work items
    e->last_kernel = BGR_KERNEL_BUNDLE | (2u << 4) | (uint32_t(MODE) << 8) | (1u << 10) | (ti ? 1u << 12 : 0u) |
                     (passive ? BGR_KERNEL_PASSIVE_PLANES : 0u) | (uint32_t(kTileRows) << 16) | (STAMPS ? BGR_KERNEL_STABLE_PLANES : 0u) |
                     (WARP_FOLD ? BGR_KERNEL_WARP_FOLD : 0u);
    return BGR_OK;
}

// The lane slots of the checksum fold take 640 bytes of shared memory per Save.  Where they would cost a resident block
// against the warp fold's 64 bytes per Save (a passive double buffer near a block boundary and many Saves in the
// vector), the launch runs the warp-fold instance.  The held-Save check (VERIFY) always runs the lane fold.
template <int MODE, bool STAMPS, bool VERIFY>
int launch_particles(bgr_engine* e, const ProgramParams& pp) {
    const int ti = (pp.flags & PF_PASSIVE_TMA) ? 1 : 0;
    const size_t base = (ti ? size_t(2) * pp.passive_bytes : 0) + (STAMPS ? kSnapBytes : 0);
    int lane = 0;
    if (int rc = bundle_occupancy<MODE, STAMPS, VERIFY, false>(e, base, pp.n_saves, ti, lane); rc != BGR_OK) return rc;
    if constexpr (!VERIFY) {
        int warp = 0;
        if (int rc = bundle_occupancy<MODE, STAMPS, false, true>(e, base, pp.n_saves, ti, warp); rc != BGR_OK) return rc;
        if (lane < warp) return launch_bundle<MODE, STAMPS, false, true>(e, pp, base + fold_bytes(true, pp.n_saves), warp);
    }
    return launch_bundle<MODE, STAMPS, VERIFY, false>(e, pp, base + fold_bytes(false, pp.n_saves), lane);
}

// The stamped instances add the stamp-point snapshot (kSnapBytes) to the passive double buffer.  With more than about
// 13 passive planes that costs the passive-TMA launches a resident block per SM; such a registration runs the instance
// without stamps instead.  Launches without the double buffer (17 KB of shared memory) always keep three blocks.
// The test holds the checksum partials at their least: the warp fold of 40 Saves.
template <int MODE>
int snapshot_fits_mode(bgr_engine* e, bool& fits) {
    fits = true;
    if (e->runs.empty() || 2u * e->passive_bytes > 96u * 1024u) return BGR_OK;  // never the passive-TMA configuration
    const size_t buf = size_t(2) * e->passive_bytes + fold_bytes(true, kMaxSaves), with = buf + kSnapBytes;
    int nb_without = 0, nb_with = 0;
    if (int rc = bundle_blocks_per_sm<MODE, true, false, true>(buf, nb_without); rc != BGR_OK) return rc;
    if (int rc = bundle_blocks_per_sm<MODE, true, false, true>(with, nb_with); rc != BGR_OK) return rc;
    fits = nb_with >= nb_without;
    return BGR_OK;
}

int snapshot_fits(bgr_engine* e, bool& fits) {
    if (e->snap_fits < 0) {
        const int rc = e->bundle_opt ? snapshot_fits_mode<2>(e, fits) : e->bundle_static_ck ? snapshot_fits_mode<1>(e, fits)
                                                                                             : snapshot_fits_mode<0>(e, fits);
        if (rc != BGR_OK) return rc;
        e->snap_fits = fits ? 1 : 0;
    }
    fits = e->snap_fits == 1;
    return BGR_OK;
}

template <bool STAMPS, bool VERIFY>
int launch_fused_variant(bgr_engine* e, const ProgramParams& pp) {
    if (e->bundle_opt) return launch_particles<2, STAMPS, VERIFY>(e, pp);         // per-entity presence
    if (e->bundle_static_ck) return launch_particles<1, STAMPS, VERIFY>(e, pp);   // both columns checksummed with the finite assertion
    return launch_particles<0, STAMPS, VERIFY>(e, pp);
}

int run_fused(bgr_engine* e, const Program& pg, uint32_t buf) {
    ProgramParams pp;
    std::memset(&pp, 0, sizeof pp);
    pp.seq = e->seq;
    pp.arena = e->arena.ptr();
    pp.order_base = e->cfg.order_base;
    pp.words = e->words; pp.tile_bytes = e->tile_bytes;
    pp.n_tiles = std::max(1u, e->tiles_for(pg.max_rows));  // at least one tile so a result block is published
    pp.n_ops = pg.n_ops; pp.n_saves = pg.n_saves;
    pp.live_rows = pg.live_rows;
    pp.flags = 0;
    if (!pg.first_is_load) pp.flags |= PF_READ_LIVE;
    if ((pg.has_load || pg.has_advance) && !pg.defer_live) pp.flags |= PF_WRITE_LIVE_ACTIVE;
    if (pg.writes_live_passive() && !pg.defer_live) pp.flags |= PF_WRITE_LIVE_PASSIVE;
    const bool passive_needed = pg.passive_to_slots || (pp.flags & PF_WRITE_LIVE_PASSIVE) || pg.has_spawn;
    uint32_t n_loads = 0;
    for (uint32_t i = 0; i < pg.n_ops; ++i) n_loads += (pg.ops[i].kind == OP_LOAD);
    const bool simple = n_loads == 0 || (n_loads == 1 && pg.first_is_load);
    if (e->tune_dynamic) pp.flags |= PF_DYNAMIC_TILES;
    if (e->tune_prefetch) pp.flags |= PF_PREFETCH_NEXT;
    pp.spawn_vals = e->spawn[buf].dev();
    if (e->spawn_sys >= 0) {
        const uint64_t ttl = e->systems[size_t(e->spawn_sys)].params[1];
        pp.spawn_ttl_lo = uint32_t(ttl); pp.spawn_ttl_hi = uint32_t(ttl >> 32);
    }
    if (!pg.has_spawn && simple && e->tune_passive_tma && !e->runs.empty() && 2u * e->passive_bytes <= 96u * 1024u) pp.flags |= PF_PASSIVE_TMA;
    // one wave of blocks (every block runs one or two tiles): the tile's tail is the grid's tail
    if (e->tune_passive_early == 1 || (e->tune_passive_early < 0 && pp.n_tiles <= 3u * uint32_t(e->num_sms))) pp.flags |= PF_PASSIVE_EARLY;
    // Stable-plane elision pays where the grid is bandwidth-bound (several waves).  A single-wave grid is latency-bound:
    // there the change tracking and the stamp round trip of every stored Save only lengthen the critical path
    // (100k entities: -9 % e2e), so it runs the instance without stamps.
    bool snap_fits = true;
    if (int rc = snapshot_fits(e, snap_fits); rc != BGR_OK) return rc;
    const bool stamps = !(pp.flags & PF_PASSIVE_EARLY) && snap_fits;
    const Column& ct = e->cols[e->bt]; const Column& cv = e->cols[e->bv];
    if (ct.hash_kind != BGR_HASH_NONE) { pp.flags |= PF_CK_T; if (ct.hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32) pp.flags |= PF_FIN_T; pp.ck_t_slot = uint32_t(ct.ck_slot); }
    if (cv.hash_kind != BGR_HASH_NONE) { pp.flags |= PF_CK_V; if (cv.hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32) pp.flags |= PF_FIN_V; pp.ck_v_slot = uint32_t(cv.ck_slot); }
    pp.t_off = ct.first_plane * kPlaneBytes; pp.v_off = cv.first_plane * kPlaneBytes;
    pp.l_off = e->cols[e->bl].first_plane * kPlaneBytes; pp.alive_off = e->words * kPlaneBytes;
    pp.need_t = ct.absent; pp.need_v = cv.absent; pp.need_tv = ct.absent | cv.absent; pp.need_l = e->cols[e->bl].absent;
    pp.n_runs = passive_needed ? uint32_t(e->runs.size()) : 0u;
    pp.passive_bytes = e->passive_bytes;
    for (size_t i = 0; i < e->runs.size(); ++i) pp.runs[i] = e->runs[i];
    pp.n_passive = passive_needed ? uint32_t(e->passive.size()) : 0u;
    for (size_t i = 0; i < e->passive.size(); ++i) {
        pp.passive[i] = e->passive[i];
        // Transform::default(): rotation = (0,0,0,1), scale = (1,1,1); every other passive word of a newborn row is 0
        const uint32_t tw = uint32_t(e->passive[i]) - ct.first_plane;
        pp.passive_template[i] = (uint32_t(e->passive[i]) >= ct.first_plane && tw >= 6 && tw <= 9) ? 0x3f800000u : 0u;
    }
    std::memcpy(pp.ops, pg.ops, sizeof(Op) * pg.n_ops);
    for (uint32_t i = 0; i < pg.n_ops; ++i)  // the stamp-table row of each image a LOAD / SAVE touches
        if (pp.ops[i].kind != OP_ADVANCE) pp.ops[i].call_count = uint32_t((size_t(pp.ops[i].image_off256) << 8) / e->image_bytes);
    // a fresh stamp range: one stamp per op and one for the live write.  The table is cleared when the range runs out,
    // and before the first stamped launch after launches without stamps (they rewrote images behind the stamps' back;
    // a world changes sides only when its row count crosses the one-wave size)
    if (stamps && (e->stamps_stale || e->stamp_next > 0xFFFFFFFFu - uint32_t(kMaxOps + 1))) {
        int rc = clear_stamp_table(e);
        if (rc != BGR_OK) return rc;
        e->stamp_next = 1;
        e->stamps_stale = false;
        // the clear forgets every content id (HostState): this launch stores its held Saves after all
        for (uint32_t i = 0; i < pg.n_ops; ++i) pp.ops[i].flags &= ~uint32_t(OPF_HELD);
    }
    uint32_t held = 0;
    for (uint32_t i = 0; i < pg.n_ops; ++i) held += (pp.ops[i].flags & OPF_HELD) ? 1u : 0u;
    if (held && e->tune_held_saves == 2) pp.held_check = e->held_check.get();
    if (!stamps) e->stamps_stale = true;
    pp.stamps = e->stamps.ptr<uint32_t>();
    pp.stamp_image = e->stamp_image();
    pp.stamp_base = e->stamp_next;
    if (stamps) e->stamp_next += pg.n_ops + 1;

    // only worth it when request vectors are queued behind each other (bgr_submit_requests with others un-collected):
    // a synchronous caller collects before the next submit, so there is nothing to overlap with
    // ... and only on a stream the engine owns: on a caller's stream foreign work may sit between two submits and
    // become the programmatic-launch primary, which the per-tile flags know nothing about
    const bool tiledep = e->tune_tiledep && !e->tile_done.empty() && e->own_stream && !pg.internal &&
                         (e->tune_tiledep > 1 || !e->pending.empty());
    if (e->tiledep_chain && pp.n_tiles != e->tiledep_tiles) {
        // The tile range changed (rows crossed a tile boundary): a tile outside the previous launch's range may still be
        // in use by an OLDER overlapping launch that nothing would make this one wait for.  Rare: drain the stream.
        CUDA_TRY(cudaStreamSynchronize(e->stream));
        e->tiledep_chain = false;
    }
    if (tiledep) {
        pp.flags |= PF_TILE_SIGNAL;
        pp.tile_done = e->tile_done.ptr<unsigned int>(); pp.tile_cnt = e->tile_cnt.ptr<unsigned int>();
        pp.grid_done = pp.tile_done + e->tiles_for(e->cfg.max_entities);  // the extra word behind the per-tile flags
        pp.done_seq = uint32_t(e->seq);
        if (e->tiledep_chain) { pp.flags |= PF_TILE_WAIT; pp.wait_seq = e->tiledep_seq; pp.wait_tiles = e->tiledep_tiles; }
    }
    // start stagger: only launches that start on an idle GPU with at least two resident blocks per SM (overlapping
    // launches arrive dephased already)
    if (e->tune_stagger_ns > 0 && !(pp.flags & PF_TILE_WAIT) && pp.n_tiles >= 2u * uint32_t(e->num_sms)) {
        pp.stagger_ns = uint32_t(e->tune_stagger_ns); pp.stagger_div = uint32_t(e->num_sms);
    }
    // overlapping launches (tile dependencies) must not share accumulators / tickets: rotate over kBufs sets — at most
    // kBufs request vectors are un-collected, so a set is re-armed (before its launch's completion word is written) long
    // before the launch kBufs later touches it
    const uint32_t set = tiledep ? uint32_t(e->seq % bgr_engine::kBufs) : 0u;
    pp.accum = e->d_accum_set[set];
    pp.ticket = e->d_ticket_set[set];
    pp.out = pg.internal ? e->internal_out.get() : e->d_out[buf];
    if (e->trace.get() && !pg.internal && e->seq - e->trace_first_seq < e->trace_cap) pp.trace = e->trace.get() + (e->seq - e->trace_first_seq) * 4;
    int rc = pp.held_check ? (stamps ? launch_fused_variant<true, true>(e, pp) : launch_fused_variant<false, true>(e, pp))
                           : (stamps ? launch_fused_variant<true, false>(e, pp) : launch_fused_variant<false, false>(e, pp));
    if (rc != BGR_OK) return rc;
    if (!pg.internal) {
        e->last_held = held;
        e->held_total += held;
        if (held) e->last_kernel |= BGR_KERNEL_HELD_SAVES;
    }
    e->tiledep_chain = tiledep;
    e->tiledep_seq = uint32_t(e->seq); e->tiledep_tiles = pp.n_tiles;
    return BGR_OK;
}

// ---------------------------------------------------------------------------------------------
// launch: TMA-staged image copy (+ fused checksum for a Save)
// ---------------------------------------------------------------------------------------------
int launch_tma(bgr_engine* e, const uint8_t* src, uint8_t* dst, uint32_t n_rows_src, uint32_t n_rows_copy, bool save,
               unsigned long long* acc, bool store) {
    TmaCopyParams tp;
    std::memset(&tp, 0, sizeof tp);
    tp.src = src; tp.dst = dst;
    tp.order_base = e->cfg.order_base;
    tp.accum = save ? acc : nullptr;
    tp.words = e->words; tp.tile_bytes = e->tile_bytes; tp.stages = e->tma_stage_tiles;
    tp.ticket = e->tma_ticket.get();
    tp.n_tiles = e->tiles_for(n_rows_copy);
    tp.n_rows_src = n_rows_src;
    tp.count_alive = save ? 1u : 0u;
    tp.store = store ? 1u : 0u;
    if (save) {
        tp.n_hash = uint32_t(e->hash_specs.size());
        std::copy(e->hash_specs.begin(), e->hash_specs.end(), tp.hash);
    }
    uint32_t grid = std::max(1u, std::min(tp.n_tiles, uint32_t(e->num_sms)));
    size_t smem = size_t(tp.stages) * e->tile_bytes;
    k_image_tma<<<grid, kTmaBlock, smem, e->stream>>>(tp);
    CUDA_TRY(cudaGetLastError());
    e->launches += 1;
    return BGR_OK;
}

// ---------------------------------------------------------------------------------------------
// launch: stepwise path (generic schemas / systems)
// ---------------------------------------------------------------------------------------------
int run_stepwise(bgr_engine* e, const Program& pg, uint32_t buf) {
    e->tiledep_chain = false;
    uint32_t live_rows = pg.live_rows;
    uint8_t* live = e->image(0);
    for (uint32_t i = 0; i < pg.n_ops; ++i) {
        const Op& op = pg.ops[i];
        NvtxRange span(span_name(op.kind == OP_SAVE ? uint32_t(BGR_REQ_SAVE) : op.kind == OP_LOAD ? uint32_t(BGR_REQ_LOAD) : uint32_t(BGR_REQ_ADVANCE)));
        switch (op.kind) {
        case OP_SAVE: {
            unsigned long long* acc = e->accum.get() + size_t(op.save_index) * kAccStride;
            if (e->tune_tma && e->tma_stage_tiles) {
                int rc = launch_tma(e, live, e->arena.ptr() + (size_t(op.image_off256) << 8), op.n_rows, op.n_rows, true, acc, !(op.flags & OPF_NO_STORE));
                if (rc != BGR_OK) return rc;
                break;
            }
            bool counted = false;
            for (const HashSpec& h : e->hash_specs) {
                k_checksum_column<<<e->grid_for(std::max(1u, op.n_rows), 256), 256, 0, e->stream>>>(
                    live, e->words, h.first_plane, h.off, h.len, h.finite, op.n_rows, e->cfg.order_base, acc,
                    h.slot, counted ? 0u : 1u, 1u, h.absent);
                counted = true;
                e->launches += 1;
            }
            if (!counted) {
                k_checksum_column<<<e->grid_for(std::max(1u, op.n_rows), 256), 256, 0, e->stream>>>(
                    live, e->words, 0, 0, 0, 0, op.n_rows, e->cfg.order_base, acc, 0, 1u, 0u, 0u);
                e->launches += 1;
            }
            if (!(op.flags & OPF_NO_STORE) && op.n_rows > 0) {
                uint32_t nt = e->tiles_for(op.n_rows);
                k_copy_image<<<e->grid_for(uint32_t(size_t(nt) * e->tile_bytes / 16u), 256), 256, 0, e->stream>>>(
                    live, e->arena.ptr() + (size_t(op.image_off256) << 8), e->words, nt, op.n_rows);
                e->launches += 1;
            }
            break;
        }
        case OP_LOAD: {
            uint32_t n_copy = std::max(op.n_rows, live_rows);
            if (n_copy > 0 && e->tune_tma && e->tma_stage_tiles) {
                int rc = launch_tma(e, e->arena.ptr() + (size_t(op.image_off256) << 8), live, op.n_rows, n_copy, false, nullptr, true);
                if (rc != BGR_OK) return rc;
            } else if (n_copy > 0) {
                uint32_t nt = e->tiles_for(n_copy);
                k_copy_image<<<e->grid_for(uint32_t(size_t(nt) * e->tile_bytes / 16u), 256), 256, 0, e->stream>>>(
                    e->arena.ptr() + (size_t(op.image_off256) << 8), live, e->words, nt, op.n_rows);
                e->launches += 1;
            }
            live_rows = op.n_rows;
            break;
        }
        case OP_ADVANCE: {
            bool any_despawn = false;
            uint32_t n = op.n_rows;
            uint32_t grid = e->grid_for(std::max(1u, n), 256);
            for (size_t s = 0; s < e->sys_specs.size() && n > 0; ++s) {
                const SysSpec& sy = e->sys_specs[s];
                if (sy.id == BGR_SYS_PARTICLES_SPAWN) continue;  // Commands: applied after the schedule (below)
                // despawn_on_input's run condition is host-known: no launch on frames whose input does not match
                if (sy.id == BGR_SYS_DESPAWN_ON_INPUT && player_input(op, sy.param & 0xFFu) != (sy.param >> 8)) continue;
                k_sys_rows<<<grid, 256, 0, e->stream>>>(live, e->words, n, sy, op, e->cfg.order_base, e->kill.ptr());
                e->launches += 1;
                any_despawn = any_despawn || e->sys_despawns[s];
            }
            if (any_despawn) {
                k_apply_despawns<<<grid, 256, 0, e->stream>>>(live, e->words, n, e->kill.ptr());
                e->launches += 1;
            }
            break;
        }
        default: break;
        }
        if (op.kind == OP_ADVANCE && (op.flags & OPF_SPAWN)) {
            k_sys_particles_spawn<<<e->grid_for(op.save_index, 256), 256, 0, e->stream>>>(
                live, e->words, e->sys_specs[size_t(e->spawn_sys)], op.image_off256, op.save_index, e->spawn[buf].dev() + op.call_count,
                e->systems[size_t(e->spawn_sys)].params[1]);
            e->launches += 1;
            live_rows = std::max(live_rows, op.image_off256 + op.save_index);
        }
    }
    k_publish<<<1, 128, 0, e->stream>>>(e->accum.get(), e->d_out[buf], std::max(1u, pg.n_saves) * kAccStride, e->seq);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    e->last_kernel = (e->tune_tma && e->tma_stage_tiles) ? BGR_KERNEL_STEPWISE_TMA : BGR_KERNEL_STEPWISE_FLAT;
    return BGR_OK;
}


// The registration as the kernels read it (bgr_engine::sys_specs / sys_despawns / hash_specs); called by bgr_build.  The
// interpreter's parameter block, the generated kernel's prelude, the TMA Save and the stepwise path all use these tables.
void build_specs(bgr_engine* e) {
    e->hash_specs.clear();
    e->sys_specs.clear();
    e->sys_despawns.clear();
    for (const Column& c : e->cols)
        if (c.hash_kind != BGR_HASH_NONE) {
            HashSpec h{};
            h.first_plane = c.first_plane; h.off = c.hash_off; h.len = c.hash_len;
            h.finite = c.hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32; h.slot = uint32_t(c.ck_slot);
            h.absent = c.absent;
            e->hash_specs.push_back(h);
        }
    uint32_t counter_index = 0;
    for (const SystemReg& sy : e->systems) {
        SysSpec sp{};
        sp.id = sy.id;
        for (uint32_t c : sy.cols) sp.need |= e->cols[c].absent;  // the query matches entities that have every bound column
        sp.plane0 = e->cols[sy.cols[0]].first_plane;
        bool despawns = false;
        switch (sy.id) {
        case BGR_SYS_U32_ADD: sp.plane0 += sy.params[0] / 4; sp.param = sy.params[1]; break;
        case BGR_SYS_U32_SATSUB_DESPAWN: sp.plane0 += sy.params[0] / 4; sp.param = sy.params[1]; despawns = true; break;
        case BGR_SYS_U32_STORE_CALL_COUNT: sp.plane0 += sy.params[0] / 4; sp.param = counter_index++; break;
        case BGR_SYS_DESPAWN_ON_INPUT: sp.param = sy.params[0] | (sy.params[1] << 8); despawns = true; break;
        case BGR_SYS_PARTICLES_DESPAWN: despawns = true; break;
        case BGR_SYS_PARTICLES_UPDATE:
        case BGR_SYS_BOX_MOVE: sp.plane1 = e->cols[sy.cols[1]].first_plane; break;
        // Transform, Velocity and Ttl: what spawn_row writes.  The spec is part of the registration (a batch compares it);
        // rate, ttl and seed are not, and reach the kernels through the ops and parameter blocks.
        case BGR_SYS_PARTICLES_SPAWN: sp.plane1 = e->cols[sy.cols[1]].first_plane; sp.param = e->cols[sy.cols[2]].first_plane; break;
        default: break;
        }
        e->sys_specs.push_back(sp);
        e->sys_despawns.push_back(despawns);
    }
}

// the system ids the generated kernel's sources switch on: NVRTC cannot parse the public header, the prelude defines them
#define BGR_SYS_ID(name) {#name, name}
constexpr std::pair<const char*, uint32_t> kSystemIds[] = {
    BGR_SYS_ID(BGR_SYS_PARTICLES_UPDATE), BGR_SYS_ID(BGR_SYS_PARTICLES_DESPAWN), BGR_SYS_ID(BGR_SYS_BOX_MOVE),
    BGR_SYS_ID(BGR_SYS_U32_ADD), BGR_SYS_ID(BGR_SYS_U32_SATSUB_DESPAWN), BGR_SYS_ID(BGR_SYS_U32_STORE_CALL_COUNT),
    BGR_SYS_ID(BGR_SYS_PARTICLES_SPAWN), BGR_SYS_ID(BGR_SYS_DESPAWN_ON_INPUT),
};
#undef BGR_SYS_ID

// Why the generated kernel cannot take this registration, or nullptr when it can
const char* jit_unsupported(const bgr_engine* e) {
    if (e->words < 1 || e->words > 24) return "the row has to fit the register file (1..24 words)";
    for (const HashSpec& h : e->hash_specs)  // whole-word byte ranges only (every POD of u32 / f32 / u64 fields)
        if (((h.off | h.len) & 3u) != 0u || h.len < 4 || h.len > 64) return "a checksummed byte range is not 1..16 whole words";
    return nullptr;
}

// The generated kernel of this registration with `item_rows`-row work items and `rows` rows per thread: its prelude is
// compiled by NVRTC, or fetched from jit.hpp's per-prelude cache.  False (and the reason in *why) when it cannot be.
bool jit_compile(const bgr_engine* e, int item_rows, int rows, JitKernel* out, std::string* why) {
    const int threads = item_rows / rows;
    std::string pre;
    auto def = [&](const char* name, unsigned long long v) { pre += "#define " + std::string(name) + " " + std::to_string(v) + "\n"; };
    for (const auto& id : kSystemIds) def(id.first, id.second);
    def("BGR_TILE_ROWS", kTileRows);
    def("BGR_JIT_WORDS", e->words); def("BGR_JIT_ROWS", rows); def("BGR_JIT_ITEM_ROWS", item_rows);
    // resident blocks the register allocation has to allow: ~512 threads per SM for narrow rows, ~256 for wide ones
    def("BGR_JIT_MINB", std::max(1, (e->words <= 8 ? 512 : 256) / threads));
    def("BGR_JIT_NSYS", e->sys_specs.size()); def("BGR_JIT_NHASH", e->hash_specs.size());
    auto u = [](uint32_t v) { return std::to_string(v) + "u"; };
    pre += "#define BGR_JIT_SYS_LIST ";
    for (const SysSpec& y : e->sys_specs)
        pre += "{" + u(y.id) + "," + u(y.plane0) + "," + u(y.plane1) + "," + u(y.need) + "," + u(y.param) + "}, ";
    pre += "{0u,0u,0u,0u,0u}\n#define BGR_JIT_HASH_LIST ";
    for (const HashSpec& h : e->hash_specs)
        pre += "{" + u(h.first_plane) + "," + u(h.off) + "," + u(h.len) + "," + u(h.finite) + "," + u(h.slot) + "," + u(h.absent) + "}, ";
    pre += "{0u,0u,0u,0u,0u,0u}\n";
    const bool ok = jit_generic_program(pre, threads, reinterpret_cast<const void*>(&bgr_abi_version), out, why);
    out->item_rows = item_rows;
    return ok;
}

// rows per thread of the whole-tile instance (BGR_TUNE_JIT_ROWS), and the work item BGR_TUNE_JIT_ITEM forces (0: none)
int jit_rows(const bgr_engine* e) { return e->tune_jit_rows == 1 || e->tune_jit_rows == 2 ? e->tune_jit_rows : 4; }
int jit_forced_item(const bgr_engine* e) {
    return e->tune_jit_item == 512 || e->tune_jit_item == 256 || e->tune_jit_item == 128 ? e->tune_jit_item : 0;
}

// NVRTC specialisation of the generic program for this registration (jit.hpp, generic_program_jit.cuh); called by bgr_build
void jit_specialise(bgr_engine* e) {
    e->jit = JitKernel{};
    e->jit_small = JitKernel{};
    if (!e->generic_ok || !e->tune_generic || e->tune_jit == 0 || (e->cfg.flags & BGR_CFG_FORCE_STEPWISE)) return;
    if (e->bundle_particles && e->tune_bundle) return;  // the bundle has its own kernel
    if (e->tune_jit == 1 && e->cfg.max_entities < 16384) return;  // small worlds: a tick is launch latency, not worth a compile
    if (jit_unsupported(e)) return;
    auto compile = [&](int item_rows, int rows, JitKernel* out) {
        std::string why;
        if (!jit_compile(e, item_rows, rows, out, &why) && std::getenv("BGR_JIT_VERBOSE"))
            std::fprintf(stderr, "[bevy_ggrs_b200] generic program not specialised, the interpreter kernel runs: %s\n", why.c_str());
    };
    const int forced = jit_forced_item(e);
    compile(forced ? forced : int(kTileRows), std::min(jit_rows(e), (forced ? forced : int(kTileRows)) / 32), &e->jit);  // a block is at least one warp
    // worlds of few tiles per SM: quarter-tile items, two rows per thread
    if (!forced && e->jit.fn) compile(128, 2, &e->jit_small);
}

// ---------------------------------------------------------------------------------------------
// launch: generic one-launch program (any schema, compiled systems; generic_program.cuh)
// ---------------------------------------------------------------------------------------------
// The launch record of one request vector on the generic program (ops and registration aside): what run_generic puts
// into its parameter block and a world batch into its per-world record.  Sets no batch fields.
JitWorld launch_record(const bgr_engine* e, const Program& pg, uint32_t buf) {
    JitWorld w;
    std::memset(&w, 0, sizeof w);
    w.arena = e->arena.ptr();
    w.order_base = e->cfg.order_base;
    w.accum = e->d_accum_set[0];
    w.ticket = e->d_ticket_set[0];
    w.out = pg.internal ? e->internal_out.get() : e->d_out[buf];
    w.seq = e->seq;
    w.n_ops = pg.n_ops; w.n_saves = pg.n_saves;
    w.n_tiles = std::max(1u, e->tiles_for(pg.max_rows));
    w.live_rows = pg.live_rows;
    w.spawn_vals = e->spawn[buf].dev();  // compile_requests' draws, copied in by submit / the batch
    if (e->spawn_sys >= 0) w.spawn_ttl = e->systems[size_t(e->spawn_sys)].params[1];
    if (!pg.first_is_load) w.flags |= PF_READ_LIVE;
    if ((pg.has_load || pg.has_advance) && !pg.defer_live) w.flags |= PF_WRITE_LIVE_ACTIVE;
    return w;
}

int run_generic(bgr_engine* e, const Program& pg, uint32_t buf) {
    const bool prev_chain = e->tiledep_chain;  // the last operation on the stream was a signalling launch of the generated kernel
    e->tiledep_chain = false;
    const JitWorld w = launch_record(e, pg, buf);
    GenericParams gp;
    std::memset(&gp, 0, sizeof gp);
    gp.arena = w.arena;
    gp.order_base = w.order_base;
    gp.accum = w.accum;
    gp.ticket = w.ticket;
    gp.out = w.out;
    gp.seq = w.seq;
    gp.spawn_vals = w.spawn_vals;
    gp.spawn_ttl = w.spawn_ttl;
    if (e->trace.get() && !pg.internal && e->seq - e->trace_first_seq < e->trace_cap) gp.trace = e->trace.get() + (e->seq - e->trace_first_seq) * 4;
    gp.words = e->words; gp.tile_bytes = e->tile_bytes;
    gp.n_ops = w.n_ops; gp.n_saves = w.n_saves;
    gp.n_tiles = w.n_tiles;
    gp.live_rows = w.live_rows;
    gp.flags = w.flags;
    gp.n_hash = uint32_t(e->hash_specs.size());
    gp.n_sys = uint32_t(e->sys_specs.size());  // <= kMaxGenericSys: generic_ok
    std::copy(e->hash_specs.begin(), e->hash_specs.end(), gp.hash);
    std::copy(e->sys_specs.begin(), e->sys_specs.end(), gp.sys);
    std::memcpy(gp.ops, pg.ops, sizeof(Op) * pg.n_ops);
    if (e->jit.fn) {  // the registration's own register-resident kernel
        // few tiles per SM: with whole tiles some SMs carry twice the rows of others and set the kernel's duration
        const JitKernel& k = (e->jit_small.fn && gp.n_tiles < 3u * uint32_t(e->num_sms)) ? e->jit_small : e->jit;
        const uint32_t n_items = gp.n_tiles * (kTileRows / uint32_t(k.item_rows));
        uint32_t grid = std::max(1u, std::min(n_items, uint32_t(e->num_sms * k.bps)));
        if (e->tune_grid > 0) grid = std::min(grid, uint32_t(e->tune_grid));
        // Overlap of consecutive launches: only when request vectors are queued behind each other (a synchronous caller
        // collects before its next submit), only on a stream the engine owns, and only between launches of the SAME kernel
        // over the SAME items (the per-item flags mean nothing across partitions: drain instead — rare, rows crossed a tile).
        const bool tiledep = e->tune_jit_tiledep && !e->item_done.empty() && e->own_stream && !pg.internal &&
                             (e->tune_jit_tiledep > 1 || !e->pending.empty());
        bool wait = false;
        if (prev_chain) {
            if (tiledep && e->jit_chain_kernel == k.fn && e->tiledep_tiles == n_items) wait = true;
            else CUDA_TRY(cudaStreamSynchronize(e->stream));  // an earlier overlapping launch may still be running
        }
        if (tiledep) {
            gp.flags |= PF_TILE_SIGNAL;
            gp.item_done = e->item_done.ptr<unsigned int>();
            gp.done_seq = uint32_t(e->seq);
            if (wait) { gp.flags |= PF_TILE_WAIT; gp.wait_seq = e->tiledep_seq; gp.wait_items = n_items; }
            // overlapping launches must not share accumulators / tickets: one set per in-flight request vector (run_fused)
            const uint32_t set = uint32_t(e->seq % bgr_engine::kBufs);
            gp.accum = e->d_accum_set[set];
            gp.ticket = e->d_ticket_set[set];
        }
        void* args[] = {&gp};
        cudaLaunchConfig_t cfg;
        std::memset(&cfg, 0, sizeof cfg);
        cfg.gridDim = dim3(grid); cfg.blockDim = dim3(k.threads); cfg.dynamicSmemBytes = 0; cfg.stream = e->stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = wait ? 1u : 0u;
        CUDA_TRY(cudaLaunchKernelExC(&cfg, k.fn, args));
        CUDA_TRY(cudaGetLastError());
        e->launches += 1;
        e->last_kernel = BGR_KERNEL_GENERIC_NVRTC | (uint32_t(k.item_rows) << 16);
        e->tiledep_chain = tiledep;
        e->tiledep_seq = uint32_t(e->seq); e->tiledep_tiles = n_items; e->jit_chain_kernel = k.fn;
        return BGR_OK;
    }
    const size_t smem = size_t((e->tile_bytes + 127u) & ~127u);
    const void* fn = (const void*)k_generic_program;
    if (e->generic_bps == 0) {
        if (smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        int nb = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fn, kGenericBlock, smem));
        e->generic_bps = std::max(1, nb);
    }
    uint32_t grid = std::max(1u, std::min(gp.n_tiles, uint32_t(e->num_sms * e->generic_bps)));
    if (e->tune_grid > 0) grid = std::min(grid, uint32_t(e->tune_grid));  // tests: several tiles per block on small worlds
    void* args[] = {&gp};
    CUDA_TRY(cudaLaunchKernel(fn, dim3(grid), dim3(kGenericBlock), args, smem, e->stream));
    CUDA_TRY(cudaGetLastError());
    e->launches += 1;
    e->last_kernel = BGR_KERNEL_GENERIC_INTERPRETER;
    return BGR_OK;
}


bool use_bundle(const bgr_engine* e) {
    return e->bundle_particles && e->tune_bundle && !(e->cfg.flags & BGR_CFG_FORCE_STEPWISE);
}
bool use_generic(const bgr_engine* e) {
    return !use_bundle(e) && e->generic_ok && e->tune_generic && !(e->cfg.flags & BGR_CFG_FORCE_STEPWISE);
}
uint32_t program_tiles(const bgr_engine* e, uint32_t rows) { return std::max(1u, e->tiles_for(rows)); }

// Writes the deferred live image: the internal program [LOAD(base), pending ADVANCEs] with the live-write flags over
// the deferred tile range.  It publishes into the engine's own result block (queued submits keep theirs), takes no
// trace row and leaves bgr_last_kernel alone; it is counted by bgr_launch_count.
int materialize_live(bgr_engine* e) {
    if (!e->deferred.active) return BGR_OK;
    const DeferredLive d = e->deferred;
    e->deferred.active = false;
    Program pg;
    Op& ld = pg.ops[0];
    std::memset(&ld, 0, sizeof ld);
    ld.kind = OP_LOAD; ld.image_off256 = d.base_off256; ld.n_rows = d.base_rows;
    std::memcpy(pg.ops + 1, d.ops, sizeof(Op) * d.n_ops);
    pg.n_ops = 1 + d.n_ops;
    pg.max_rows = d.max_rows; pg.live_rows = d.base_rows;
    pg.has_load = pg.first_is_load = true;
    pg.has_advance = d.n_ops > 0;
    pg.passive_to_live = d.passive;
    pg.internal = true;
    const uint32_t kernel = e->last_kernel;
    const int rc = use_bundle(e) ? run_fused(e, pg, 0) : run_generic(e, pg, 0);
    e->last_kernel = kernel;
    return rc;
}

// Every entry point that reads or writes image 0 outside a program calls this (after drain(), where it drains).  The
// next request vector then writes image 0 eagerly: a caller that reads the live world every tick pays at most one
// materialisation instead of one per tick.
int touch_live(bgr_engine* e) {
    e->live_touched = true;
    return materialize_live(e);
}

// The previous fused program deferred its live write.  A program that starts with its own Load reads nothing of image
// 0 and rewrites it (the record is dropped); one that would read image 0 starts from the base slot instead:
// [LOAD(base), pending ADVANCEs, its own ops].  Otherwise image 0 is written first: a Save of this program would
// overwrite the base slot (shallow rings), the rewritten vector would not fit, or this program covers fewer tiles than
// the deferred range (rows shrank through a Load), whose tiles it would otherwise leave stale.
int consume_deferred(bgr_engine* e, Program& pg) {
    const DeferredLive& d = e->deferred;
    if (!d.active) return BGR_OK;
    if (program_tiles(e, pg.max_rows) >= program_tiles(e, d.max_rows)) {
        if (pg.first_is_load) {
            if (d.passive) pg.passive_to_live = true;  // the live passive planes were not written either
            return BGR_OK;
        }
        bool base_saved = false;
        for (uint32_t i = 0; i < pg.n_ops; ++i)
            base_saved = base_saved || (pg.ops[i].kind == OP_SAVE && !(pg.ops[i].flags & OPF_NO_STORE) &&
                                        pg.ops[i].image_off256 == d.base_off256);
        if (!base_saved && pg.n_ops + 1 + d.n_ops <= uint32_t(kMaxOps)) {
            std::memmove(pg.ops + 1 + d.n_ops, pg.ops, sizeof(Op) * pg.n_ops);
            Op& ld = pg.ops[0];
            std::memset(&ld, 0, sizeof ld);
            ld.kind = OP_LOAD; ld.image_off256 = d.base_off256; ld.n_rows = d.base_rows;
            std::memcpy(pg.ops + 1, d.ops, sizeof(Op) * d.n_ops);
            pg.n_ops += 1 + d.n_ops;
            pg.has_load = pg.first_is_load = true;
            pg.has_advance = pg.has_advance || d.n_ops > 0;
            // the prepended LOAD rewrites the live passive planes exactly when the deferring program would have
            pg.passive_to_live = pg.passive_to_live || d.passive;
            pg.max_rows = std::max(pg.max_rows, d.base_rows);
            pg.from_deferred = true;
            return BGR_OK;
        }
    }
    return materialize_live(e);
}

// A fused program defers its live write when its last stored Save is followed only by ADVANCEs that spawn nothing
// (at most kMaxDeferredOps of them).  Returns the record submit() commits.
DeferredLive plan_deferral(Program& pg) {
    DeferredLive d;
    if (!(pg.has_load || pg.has_advance)) return d;  // the program writes no live image
    uint32_t i = pg.n_ops;
    while (i > 0 && pg.ops[i - 1].kind == OP_ADVANCE && !(pg.ops[i - 1].flags & OPF_SPAWN)) --i;
    const uint32_t n_tail = pg.n_ops - i;
    if (i == 0 || n_tail > kMaxDeferredOps) return d;
    const Op& sv = pg.ops[i - 1];
    if (sv.kind != OP_SAVE || (sv.flags & OPF_NO_STORE)) return d;
    d.active = true;
    d.passive = pg.writes_live_passive();
    d.base_off256 = sv.image_off256;
    d.base_rows = sv.n_rows;
    d.max_rows = pg.max_rows;
    d.n_ops = n_tail;
    std::memcpy(d.ops, pg.ops + i, sizeof(Op) * n_tail);
    pg.defer_live = true;
    return d;
}

// A buffer whose size follows the row capacity: `n` strides of bytes(tiles) each for a capacity of `tiles` tiles.
struct CapacityBuffer {
    StridedRange* range;
    uint32_t n;
    size_t per_tile, fixed, align;
    bool wanted;  // bgr_build creates it
    size_t bytes(uint64_t tiles) const { return round_up(tiles * per_tile + fixed, align); }
};

// The reported state of a feed (one stride) and its per-tile counters tile_count / tile_off / tile_list (three).
std::array<CapacityBuffer, 2> feed_buffers(bgr_engine::Feed& fd) {
    return {{{&fd.rep, 1, tile_bytes_of(fd.p.rep_words), 0, 1, true}, {&fd.count, 3, sizeof(unsigned int), 0, 1, true}}};
}

// Every capacity-sized buffer: the engine's own first (the arena leads), then those of its feeds.
std::vector<CapacityBuffer> capacity_buffers(bgr_engine* e) {
    const uint32_t images = e->n_slots() + 1u;
    const size_t u32 = sizeof(unsigned int);
    std::vector<CapacityBuffer> v = {
        {&e->arena, images, e->tile_bytes, 0, 256, true},  // ops address images in 256-byte units
        {&e->kill, 1, kTileRows, 0, 1, true},
        {&e->tile_done, 1, u32, u32, 1, e->tune_tiledep != 0},  // one word per tile and the grid's word behind them
        {&e->tile_cnt, 1, u32, u32, 1, e->tune_tiledep != 0},
        {&e->stamps, images, kSegsPerTile * kActivePlanes * sizeof(uint32_t), 0, 1, use_bundle(e)},  // one stride per image
        // quarter-tile work items at most; a growable engine may compile the generated kernel later (grow_to)
        {&e->item_done, 1, 4 * u32, 4 * u32, 1, e->tune_jit_tiledep && (e->growable() ? e->generic_ok : e->jit.fn != nullptr)},
    };
    for (auto& fd : e->feeds)
        if (fd.used)
            for (const CapacityBuffer& b : feed_buffers(fd)) v.push_back(b);
    return v;
}

// The one place that knows how capacity buffers are allocated: a growable engine reserves address space for the
// ceiling and maps nothing yet (map_tiles maps); any other engine allocates the capacity with cudaMalloc.
bool create_range(bgr_engine* e, const CapacityBuffer& b, std::string* err) {
    if (e->growable()) return b.range->reserve(e->cfg.device, b.n, b.bytes(e->ceiling / kTileRows), err);
    return b.range->allocate(b.n, b.bytes(e->n_tiles_cap), err);
}

// Maps every capacity buffer for `tiles` tiles and zeroes the new bytes on the stream, behind every queued launch.
// Either every range grows or none does.  host_ns spent mapping: [0] the arena, [1] the rest.
int map_tiles(bgr_engine* e, uint64_t tiles, uint64_t* map_ns = nullptr) {
    struct Step { StridedRange* r; size_t bytes; size_t old; };
    std::vector<Step> steps;
    for (const CapacityBuffer& b : capacity_buffers(e))
        if (!b.range->empty()) steps.push_back({b.range, b.bytes(tiles), b.range->mapped});
    std::string err;
    uint64_t t = host_ns();
    for (size_t i = 0; i < steps.size(); ++i) {
        if (!steps[i].r->map_to(steps[i].bytes, &err)) {
            for (size_t k = 0; k < i; ++k) steps[k].r->shrink(steps[k].old);
            return fail(BGR_ERR_CAPACITY, "growing to " + std::to_string(tiles * kTileRows) + " rows: " + err);
        }
        if (map_ns && i == 0) { const uint64_t u = host_ns(); map_ns[0] += u - t; t = u; }
    }
    if (map_ns) map_ns[1] += host_ns() - t;
    for (const Step& s : steps) CUDA_TRY(s.r->zero_new(e->stream));
    e->tiledep_chain = false;  // the next launch waits for the whole stream, the zeroing included
    return BGR_OK;
}

// BGR_CFG_GROWABLE: capacity >= rows afterwards.  No byte moves, so compiled ops, queued launches, the deferred live
// image, the slots with their passive versions and content stamps, and every feed's reported state stay valid.
int grow_to(bgr_engine* e, uint64_t rows) {
    if (rows <= e->cfg.max_entities) return BGR_OK;
    if (rows > e->ceiling)
        return fail(BGR_ERR_CAPACITY, std::to_string(rows) + " rows exceed the engine's ceiling of " + std::to_string(e->ceiling) +
                                          " rows (BGR_CFG_GROWABLE)");
    const uint64_t t0 = host_ns();
    // max(rows needed, 2 x capacity) in whole tiles, plus the tiles the arena's mapping granularity pays for anyway
    uint64_t tiles = (std::max<uint64_t>(rows, 2ull * e->cfg.max_entities) + kTileRows - 1) / kTileRows;
    tiles = round_up(tiles * e->tile_bytes, e->arena.gran) / e->tile_bytes;
    tiles = std::min<uint64_t>(tiles, e->ceiling / kTileRows);
    uint64_t map_ns[2] = {0, 0};
    int rc = map_tiles(e, tiles, map_ns);
    if (rc != BGR_OK) return rc;
    const bool verbose = std::getenv("BGR_GROW_VERBOSE") != nullptr;
    const uint64_t t1 = host_ns();
    if (verbose) CUDA_TRY(cudaStreamSynchronize(e->stream));  // the zeroing, timed (it is otherwise asynchronous)
    const uint64_t t2 = host_ns();
    const uint32_t old_cap = e->cfg.max_entities;
    e->cfg.max_entities = uint32_t(tiles * kTileRows);
    e->epad = e->cfg.max_entities;
    e->n_tiles_cap = uint32_t(tiles);
    // the registration's own kernel, compiled where bgr_build would have compiled it at this capacity
    if (!e->jit.fn && e->tune_jit == 1 && old_cap < 16384 && e->cfg.max_entities >= 16384) jit_specialise(e);
    const uint64_t t3 = host_ns();
    if (verbose)
        std::fprintf(stderr, "[bevy_ggrs_b200] grew %u -> %u rows: map arena %llu ns, map side tables %llu ns, zero %llu ns, "
                             "jit %llu ns, total %llu ns\n", old_cap, e->cfg.max_entities, (unsigned long long)map_ns[0],
                     (unsigned long long)map_ns[1], (unsigned long long)(t2 - t1), (unsigned long long)(t3 - t2),
                     (unsigned long long)(t3 - t0));
    return BGR_OK;
}

// A request vector compiled against a copy of its engine's HostState: what submit() executes and commits
struct Prepared {
    HostState s;
    Program pg;
    DeferredLive next;        // the vector's own deferred live image (plan)
    uint64_t t_begin = 0, t_compiled = 0;
};

// submit(), first half: validates the vector and compiles it against a copy of the HostState.  Executes and changes
// nothing, so a batch prepares every world before any of them runs.
int prepare(bgr_engine* e, const bgr_session_info* sess, const bgr_request* reqs, uint32_t n, Prepared& p) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (!e->built) return fail(BGR_ERR_STATE, "bgr_build has not been called");
    if (e->pending.size() >= size_t(bgr_engine::kBufs)) return fail(BGR_ERR_STATE, "too many un-collected submits");
    if (n && !reqs) return fail(BGR_ERR_INVALID_ARGUMENT, "null requests");
    p.t_begin = host_ns();
    p.s = e->st;
    p.pg.~Program();
    new (&p.pg) Program;
    p.next = DeferredLive{};
    return compile_requests(e, p.s, sess, reqs, n, p.pg);
}

// ... the vector takes its sequence number, consumes the previous vector's deferred live image (which may launch its
// materialisation) and plans its own
int plan(bgr_engine* e, Prepared& p) {
    e->seq += 1;
    e->ticked = true;
    const bool bundle = use_bundle(e), fused = bundle || use_generic(e);  // one launch for the whole request vector
    const int rc = fused ? consume_deferred(e, p.pg) : materialize_live(e);
    if (rc != BGR_OK) return rc;
    if (bundle) derive_content_ids(e, p.s, p.pg);
    if (fused && e->tune_defer_live && !e->live_touched) p.next = plan_deferral(p.pg);
    return BGR_OK;
}

// submit(), second half, behind the launch into result buffer `buf`: the last_kernel bits, the vector's pending
// results, the state commit
int commit(bgr_engine* e, const Prepared& p, uint32_t buf) {
    const Program& pg = p.pg;
    if (pg.defer_live) e->last_kernel |= BGR_KERNEL_DEFERRED_LIVE;
    if (pg.from_deferred) e->last_kernel |= BGR_KERNEL_FROM_DEFERRED;
    // an event between two launches would serialise them; with host polling it is only a fallback, taken lazily
    if (!(e->tune_tiledep && e->tune_poll)) CUDA_TRY(cudaEventRecord(e->ev[buf].get(), e->stream));
    e->last_fused = use_bundle(e) || use_generic(e);
    e->st = p.s;
    e->deferred = p.next;
    e->live_touched = false;
    Pending pd;
    pd.buf = buf; pd.n_saves = pg.n_saves; pd.seq = e->seq; pd.gseq = e->group ? e->gseq : 0;
    std::memcpy(pd.frames, pg.save_frames, sizeof(int32_t) * pg.n_saves);
    std::memcpy(pd.totals, pg.save_totals, sizeof(uint32_t) * pg.n_saves);
    e->pending.push_back(pd);
    e->next_buf = (buf + 1) % bgr_engine::kBufs;
    e->prof[0] += 1; e->prof[1] += p.t_compiled - p.t_begin; e->prof[2] += host_ns() - p.t_compiled;
    return BGR_OK;
}

// submit() after prepare(): grows, launches the vector and commits it
int execute(bgr_engine* e, Prepared& p) {
    int rc = BGR_OK;
    const Program& pg = p.pg;
    // the program does not depend on the capacity: growing behind the compile leaves it (and its ParticleRng draws) valid
    if (pg.rows_needed) rc = grow_to(e, pg.rows_needed);
    if (rc != BGR_OK) return rc;
    p.t_compiled = host_ns();
    uint32_t buf = e->next_buf;
    if (e->group) {
        // the buffer of this request vector was last used kBufs vectors ago: every peer must have folded that one
        std::string err;
        if (!e->group->wait_reusable(e->gseq + 1, &err)) return fail(BGR_ERR_STATE, err);
        e->gseq += 1;
        buf = ShardGroup::buf_of(e->gseq);
        e->group->publish_meta(e->gseq, pg.n_saves, e->n_ck, pg.save_frames, pg.save_totals);
    }
    if (!pg.spawn_vals.empty()) std::memcpy(e->spawn[buf].get(), pg.spawn_vals.data(), pg.spawn_vals.size() * sizeof(float2));
    rc = plan(e, p);
    if (rc != BGR_OK) return rc;
    rc = use_bundle(e) ? run_fused(e, pg, buf) : use_generic(e) ? run_generic(e, pg, buf) : run_stepwise(e, pg, buf);
    if (rc != BGR_OK) return rc;
    return commit(e, p, buf);
}

int submit(bgr_engine* e, const bgr_session_info* sess, const bgr_request* reqs, uint32_t n) {
    NvtxRange span("HandleRequests");
    Prepared p;
    const int rc = prepare(e, sess, reqs, n, p);
    if (rc != BGR_OK) return rc;  // nothing executed, nothing committed
    return execute(e, p);
}

void fold(const bgr_partial& p, bgr_checksum* out) {
    // EntityChecksumPlugin::update (entity_checksum.rs:35-43)
    uint64_t x = sea_hash_2xu64(p.active, p.total);
    // ComponentChecksumPlugin: `result.hash(&mut hasher)` (component_checksum.rs:93-95), then
    // ChecksumPlugin::update XORs every part (checksum.rs:88-99)
    for (uint32_t c = 0; c < p.n_columns && c < BGR_MAX_CHECKSUM_COLUMNS; ++c) x ^= sea_hash_u64(p.xor_[c]);
    out->frame = p.frame;
    out->has_checksum = 1;
    out->lo = x;
    out->hi = 0;
}

// `bad_frame`: where the first Save whose finite assertion failed goes (left alone when none did)
int collect(bgr_engine* e, bgr_checksum* out, uint32_t cap, uint32_t* n_out, int32_t* bad_frame = nullptr) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (e->pending.empty()) return fail(BGR_ERR_STATE, "nothing to collect");
    Pending pd = e->pending.front();
    e->pending.pop_front();
    const uint64_t t_wait0 = host_ns();
    // Completion: the last block of the kernel publishes every result word as a self-validating pair
    // (v, v ^ result_tag(seq, i)) plus a completion pair; a word is accepted when its halves XOR to this launch's tag.
    const volatile unsigned long long* blk = e->h_out[pd.buf];
    const uint32_t n_words = pd.n_saves * kAccStride;
    unsigned long long r[kMaxSaves * kAccStride];
    uint32_t valid = 0;
    bool seq_ok = false;
    auto ready = [&]() {
        if (!seq_ok) {
            const unsigned long long a = blk[2 * kSeqIndex], b = blk[2 * kSeqIndex + 1];
            if ((a ^ b) != result_tag(pd.seq, kSeqIndex)) return false;
            seq_ok = true;
        }
        while (valid < n_words) {
            const unsigned long long a = blk[2 * valid], b = blk[2 * valid + 1];
            if ((a ^ b) != result_tag(pd.seq, valid)) return false;
            r[valid++] = a;
        }
        return true;
    };
    bool done = false;
    if (e->tune_poll && !pd.finished) {
        for (int spin = 0; spin < 200000; ++spin) {
            if (ready()) { done = true; break; }
            __builtin_ia32_pause();
        }
    }
    if (!done) {  // the event / the stream is ordered after the launch
        if (!pd.finished) {
            if (e->tune_tiledep && e->tune_poll) CUDA_TRY(cudaStreamSynchronize(e->stream));
            else CUDA_TRY(cudaEventSynchronize(e->ev[pd.buf].get()));
        }
        if (!ready()) return fail(BGR_ERR_CUDA, "request vector completed without publishing valid results");
    }
    const uint64_t t_wait1 = host_ns();
    e->prof[3] += t_wait1 - t_wait0;
    e->last_partials.clear();
    bool nonfinite = false;
    // shard group: wait for every rank's block of this request vector and combine (XOR / sum / OR) across ranks
    bgr_partial combined[kMaxSaves];
    if (pd.gseq) {
        uint32_t n = 0;
        uint64_t flags = 0;
        std::string err;
        if (!e->group || !e->group->combine(pd.gseq, combined, kMaxSaves, &n, &flags, &err))
            return fail(BGR_ERR_STATE, e->group ? err : "request vector was submitted inside a shard group that has been left");
        if (flags & 1ULL) nonfinite = true;
    }
    for (uint32_t k = 0; k < pd.n_saves; ++k) {
        bgr_partial p;
        std::memset(&p, 0, sizeof p);
        p.frame = pd.frames[k];
        p.n_columns = e->n_ck;
        p.active = r[k * kAccStride + 6];
        p.total = pd.totals[k];
        for (uint32_t c = 0; c < e->n_ck; ++c) p.xor_[c] = r[k * kAccStride + c];
        if ((r[k * kAccStride + 7] & 1ULL) && !nonfinite && bad_frame) *bad_frame = pd.frames[k];
        if (r[k * kAccStride + 7] & 1ULL) nonfinite = true;
        e->last_partials.push_back(p);
    }
    if (n_out) *n_out = pd.n_saves;
    for (uint32_t k = 0; k < pd.n_saves && k < cap && out; ++k) {
        if (pd.gseq) {
            fold(combined[k], &out[k]);  // the frame checksum of the WHOLE world, identical on every rank
        } else if (e->cfg.flags & BGR_CFG_SHARDED) {
            out[k].frame = pd.frames[k]; out[k].has_checksum = 0; out[k].lo = 0; out[k].hi = 0;
        } else {
            fold(e->last_partials[k], &out[k]);
        }
    }
    e->prof[4] += host_ns() - t_wait1;
    if (nonfinite) return fail(BGR_ERR_NON_FINITE, "Hashing is not stable for NaN f32 values.");
    return BGR_OK;
}

// Entry points that touch the live world (read / write / spawn / peek ...) first wait for every submitted request
// vector.  The results of un-collected submits STAY queued: a later bgr_collect still returns their checksums (and
// the non-finite status), in order — nothing is dropped on the floor.
int drain(bgr_engine* e) {
    e->tiledep_chain = false;  // callers enqueue ordinary (fully ordered) work next
    if (e->pending.empty()) return BGR_OK;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->pending.for_each([](Pending& pd) { pd.finished = true; });
    return BGR_OK;
}

// ECS column (array of T, `stride` bytes apart) <-> tile-planar image: one H2D/D2H copy of the AoS
// bytes + one transposition kernel (k_scatter_column / k_gather_column).
int transfer_column(bgr_engine* e, uint32_t image_idx, uint32_t column, uint32_t first, uint32_t count, void* host,
                    uint32_t stride, bool to_device) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (column >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown column");
    const Column& c = e->cols[column];
    if (stride < c.elem_bytes) return fail(BGR_ERR_INVALID_ARGUMENT, "stride < elem_bytes");
    if (uint64_t(first) + count > e->cfg.max_entities) return fail(BGR_ERR_CAPACITY, "row range exceeds max_entities");
    if (count == 0) return BGR_OK;
    int rc = drain(e);
    if (rc == BGR_OK && image_idx == 0) rc = touch_live(e);
    if (rc != BGR_OK) return rc;
    const size_t bytes = size_t(count) * stride;
    CUDA_TRY(e->stage.ensure(std::max<size_t>(bytes, 1u << 20)));
    uint8_t* img = e->image(image_idx);
    uint32_t grid = e->grid_for(uint32_t(std::min<size_t>(size_t(count) * c.words, 0x7fffffffu)), 256);
    if (to_device) {
        e->st.live_passive_ver = ++e->st.ver_counter;  // host wrote a column: live content is new
        CUDA_TRY(cudaMemcpyAsync(e->stage.get(), host, bytes, cudaMemcpyHostToDevice, e->stream));
        k_scatter_column<<<grid, 256, 0, e->stream>>>(img, e->words, c.first_plane, c.words, c.elem_bytes, first, count, e->stage.get(), stride);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        rc = clear_stamps(e, image_idx);
        if (rc != BGR_OK) return rc;
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    } else {
        if (stride != c.elem_bytes) CUDA_TRY(cudaMemcpyAsync(e->stage.get(), host, bytes, cudaMemcpyHostToDevice, e->stream));  // keep the caller's padding bytes
        k_gather_column<<<grid, 256, 0, e->stream>>>(img, e->words, c.first_plane, c.words, c.elem_bytes, first, count, e->stage.get(), stride);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(host, e->stage.get(), bytes, cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    return BGR_OK;
}

int read_alive_image(bgr_engine* e, uint32_t image_idx, uint32_t first, uint32_t count, uint32_t n_rows, uint8_t* dst,
                     uint32_t need = 0) {
    if (count == 0) return BGR_OK;
    int rc = drain(e);
    if (rc == BGR_OK && image_idx == 0) rc = touch_live(e);
    if (rc != BGR_OK) return rc;
    if (uint64_t(first) + count > e->cfg.max_entities) return fail(BGR_ERR_CAPACITY, "row range exceeds max_entities");
    CUDA_TRY(e->stage.ensure(std::max<size_t>(count, 1u << 20)));
    k_gather_alive<<<e->grid_for(count, 256), 256, 0, e->stream>>>(e->image(image_idx), e->words, first, count, n_rows, e->stage.get(), need);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(dst, e->stage.get(), count, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return BGR_OK;
}

int download_begin(bgr_engine* e, uint32_t column, uint32_t off, uint32_t len, uint32_t first, uint32_t count, void* host,
                   uint32_t* ticket_out) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (!host || !ticket_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (column >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown column");
    const Column& c = e->cols[column];
    if ((off & 3u) || (len & 3u) || len == 0 || uint64_t(off) + len > uint64_t(c.words) * 4u)
        return fail(BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element");
    if (uint64_t(first) + count > e->st.n_rows) return fail(BGR_ERR_CAPACITY, "row range exceeds the spawned rows");
    uint32_t slot = BGR_MAX_DOWNLOADS;
    for (uint32_t k = 0; k < BGR_MAX_DOWNLOADS; ++k) {
        const uint32_t i = (e->next_dl + k) % BGR_MAX_DOWNLOADS;
        if (!e->dl[i].busy) { slot = i; break; }
    }
    if (slot == BGR_MAX_DOWNLOADS) return fail(BGR_ERR_STATE, "too many downloads in flight (BGR_MAX_DOWNLOADS)");
    int rc = touch_live(e);  // stream-ordered behind the queued submits, like the gather below
    if (rc != BGR_OK) return rc;
    bgr_engine::Download& d = e->dl[slot];
    const size_t bytes = size_t(count) * len;
    if (!e->copy_stream) CUDA_TRY(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
    CUDA_TRY(d.packed.ensure());
    CUDA_TRY(d.done.ensure());
    CUDA_TRY(d.buf.ensure(bytes));  // the slot is idle: its last copy was waited for
    if (count) {
        const uint32_t n_words = len / 4u;
        const uint32_t grid = e->grid_for(uint32_t(std::min<size_t>(size_t(count) * n_words, 0x7fffffffu)), 256);
        k_gather_fields<<<grid, 256, 0, e->stream>>>(e->image(0), e->words, c.first_plane + off / 4u, n_words, first, count,
                                                      reinterpret_cast<uint32_t*>(d.buf.get()));
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        e->tiledep_chain = false;
        CUDA_TRY(cudaEventRecord(d.packed.get(), e->stream));
        CUDA_TRY(cudaStreamWaitEvent(e->copy_stream, d.packed.get(), 0));
        CUDA_TRY(cudaMemcpyAsync(host, d.buf.get(), bytes, cudaMemcpyDeviceToHost, e->copy_stream));
    }
    CUDA_TRY(cudaEventRecord(d.done.get(), e->copy_stream));
    d.busy = true;
    e->next_dl = (slot + 1) % BGR_MAX_DOWNLOADS;
    *ticket_out = slot;
    return BGR_OK;
}

int download_wait(bgr_engine* e, uint32_t ticket) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (ticket >= BGR_MAX_DOWNLOADS || !e->dl[ticket].busy) return fail(BGR_ERR_STATE, "no such download in flight");
    CUDA_TRY(cudaEventSynchronize(e->dl[ticket].done.get()));
    e->dl[ticket].busy = false;
    return BGR_OK;
}

// ---- change feed (change_feed.cuh) ----
// feed_fields (feed_check.hpp) over the engine's registered columns
int engine_feed_fields(const bgr_engine* e, const bgr_feed_field* fields, uint32_t n_fields, FeedParams& p, std::string* err) {
    auto col_at = [e](uint32_t c) { return FeedColumn{e->cols[c].first_plane, e->cols[c].words, e->cols[c].absent}; };
    return feed_fields(uint32_t(e->cols.size()), col_at, e->words, fields, n_fields, p, err);
}

int feed_create(bgr_engine* e, const bgr_feed_field* fields, uint32_t n_fields, uint32_t* feed_out) {
    if (!e || !feed_out || (n_fields && !fields)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (!e->built) return fail(BGR_ERR_STATE, "bgr_feed_create before bgr_build");
    if (n_fields > BGR_MAX_FEED_FIELDS) return fail(BGR_ERR_CAPACITY, "too many fields (BGR_MAX_FEED_FIELDS)");
    uint32_t id = BGR_MAX_FEEDS;
    for (uint32_t i = 0; i < BGR_MAX_FEEDS && id == BGR_MAX_FEEDS; ++i)
        if (!e->feeds[i].used) id = i;
    if (id == BGR_MAX_FEEDS) return fail(BGR_ERR_CAPACITY, "too many feeds (BGR_MAX_FEEDS)");
    FeedParams p{};
    std::string err;
    const int rc = engine_feed_fields(e, fields, n_fields, p, &err);
    if (rc != BGR_OK) return fail(rc, err);
    bgr_engine::Feed& fd = e->feeds[id];
    fd.p = p;
    bool ok = true;
    for (const CapacityBuffer& b : feed_buffers(fd))
        ok = ok && create_range(e, b, &err) && b.range->map_to(b.bytes(e->n_tiles_cap), &err);
    cudaError_t ce = ok ? cudaSuccess : cudaErrorMemoryAllocation;
    // the reported state starts as (0, zeros) on every row; ordered before any pass on the engine stream
    if (ce == cudaSuccess) ce = fd.rep.zero_new(e->stream);
    if (ce == cudaSuccess) ce = fd.count.zero_new(e->stream);
    if (ce == cudaSuccess) ce = fd.info.ensure(8);
    if (ce == cudaSuccess) ce = fd.h_info.ensure(4);
    if (ce == cudaSuccess) ce = fd.packed.ensure();
    if (ce == cudaSuccess) ce = fd.done.ensure();
    if (ce == cudaSuccess && !e->copy_stream) ce = cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking);
    if (ce != cudaSuccess) {
        cudaStreamSynchronize(e->stream);  // a memset may be queued on the ranges released here
        fd = bgr_engine::Feed{};
        return fail(BGR_ERR_CUDA, "bgr_feed_create: " + (ok ? std::string(cudaGetErrorString(ce)) : err));
    }
    const size_t count_stride = fd.count.stride / sizeof(unsigned int);  // words between tile_count, tile_off and tile_list
    fd.p.one.rep = fd.rep.ptr();
    fd.p.n_worlds = 1;
    fd.p.tile_count = fd.count.ptr<unsigned int>();
    fd.p.info = fd.info.get();
    fd.p.head = fd.p.info + 4;
    fd.p.world_scan = fd.p.head + 2;
    fd.p.tile_off = fd.p.tile_count + count_stride;
    fd.p.tile_list = fd.p.tile_off + count_stride;
    fd.used = true;
    e->tiledep_chain = false;
    *feed_out = id;
    return BGR_OK;
}

int feed_reset(bgr_engine* e, uint32_t feed) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (feed >= BGR_MAX_FEEDS || !e->feeds[feed].used) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown feed");
    bgr_engine::Feed& fd = e->feeds[feed];
    // stream-ordered behind a report in flight, whose pass 2 is the last writer of the reported state
    CUDA_TRY(cudaMemsetAsync(fd.rep.ptr(), 0, size_t(e->tiles_for(fd.bound)) * tile_bytes_of(fd.p.rep_words), e->stream));
    e->tiledep_chain = false;
    fd.bound = 0;
    return BGR_OK;
}

// The device address of page-locked memory from bgr_host_alloc (mapped into the device address space: unified
// addressing), or nullptr
uint32_t* mapped_host(void* host) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, host) != cudaSuccess || a.type != cudaMemoryTypeHost || !a.devicePointer) {
        cudaGetLastError();
        return nullptr;
    }
    return static_cast<uint32_t*>(a.devicePointer);
}

// The passes of the report `p` describes (table, scratch and staging set) on e's stream, counted on e; then on `copy`,
// behind `packed`, the records into page-locked `host_dev` (nullptr: none) and the infos of every listed world into
// `h_info`, with `done` behind them.  bgr_feed_begin and bgr_batch_feed_begin.
int feed_report(bgr_engine* e, const FeedParams& p, uint32_t* host_dev, cudaStream_t copy, cudaEvent_t packed, cudaEvent_t done,
                unsigned int* h_info) {
    if (p.n_tiles) {
        if (p.worlds) k_feed_count<true><<<p.n_tiles, kFeedBlock, 0, e->stream>>>(p);
        else k_feed_count<false><<<p.n_tiles, kFeedBlock, 0, e->stream>>>(p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    if (p.worlds) k_feed_scan<<<1, kFeedScanBlock, 0, e->stream>>>(p);
    else k_feed_scan_one<<<1, kFeedScanBlock, 0, e->stream>>>(p);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    const uint32_t grid2 = std::max(1u, std::min(p.n_tiles, uint32_t(e->num_sms) * 4u));
    if (p.worlds) k_feed_records<true><<<grid2, kFeedBlock, 0, e->stream>>>(p);
    else k_feed_records<false><<<grid2, kFeedBlock, 0, e->stream>>>(p);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    e->tiledep_chain = false;
    CUDA_TRY(cudaEventRecord(packed, e->stream));
    CUDA_TRY(cudaStreamWaitEvent(copy, packed, 0));
    if (host_dev) {
        k_feed_copy<<<std::max(1, e->num_sms), 256, 0, copy>>>(p.out, p.head, p.record_words, host_dev);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaMemcpyAsync(h_info, p.info, sizeof(bgr_feed_info) * p.n_worlds, cudaMemcpyDeviceToHost, copy));
    CUDA_TRY(cudaEventRecord(done, copy));
    return BGR_OK;
}

// A report of `fd` has started: its rows up to `rows` may now hold a reported state, and it is busy under a fresh ticket
void feed_started(bgr_engine* e, uint32_t feed, uint32_t rows) {
    bgr_engine::Feed& fd = e->feeds[feed];
    fd.bound = std::max(fd.bound, rows);
    fd.busy = true;
    e->feed_seq = (e->feed_seq + 1u) & 0x0FFFFFFFu;
    fd.ticket = feed + BGR_MAX_FEEDS * e->feed_seq;
}

// bgr_feed_begin: the one-world case of the table-driven passes, its entry in the kernel parameters
int feed_begin(bgr_engine* e, uint32_t feed, void* host, uint32_t cap, uint32_t* ticket_out) {
    if (!e || !ticket_out || (cap && !host)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (!e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (feed >= BGR_MAX_FEEDS || !e->feeds[feed].used) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown feed");
    bgr_engine::Feed& fd = e->feeds[feed];
    if (fd.busy) return fail(BGR_ERR_STATE, "a report of this feed is in flight");
    uint32_t* host_dev = cap ? mapped_host(host) : nullptr;
    if (cap && !host_dev) return fail(BGR_ERR_INVALID_ARGUMENT, "host_dst must come from bgr_host_alloc");
    // no report has more records than the rows it compares
    const uint32_t cap_eff = std::min<uint64_t>(cap, uint64_t(e->n_tiles_cap) * kTileRows);
    CUDA_TRY(fd.out.ensure(size_t(cap_eff) * fd.p.record_words));  // no report of this feed is in flight
    fd.p.out = fd.out.get();
    int rc = touch_live(e);  // stream-ordered behind the queued submits, like the passes below
    if (rc != BGR_OK) return rc;
    FeedParams p = fd.p;
    p.one.img = e->image(0);
    p.one.rows = e->st.n_rows;
    p.one.n_tiles = p.n_tiles = e->tiles_for(std::max(p.one.rows, fd.bound));
    p.one.cap = cap_eff;
    rc = feed_report(e, p, host_dev, e->copy_stream, fd.packed.get(), fd.done.get(), fd.h_info.get());
    if (rc != BGR_OK) return rc;
    feed_started(e, feed, p.one.rows);
    *ticket_out = fd.ticket;
    return BGR_OK;
}

int feed_wait(bgr_engine* e, uint32_t ticket, bgr_feed_info* info) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    bgr_engine::Feed& fd = e->feeds[ticket % BGR_MAX_FEEDS];
    if (!fd.used || !fd.busy || fd.ticket != ticket) return fail(BGR_ERR_STATE, "no such feed report in flight");
    CUDA_TRY(cudaEventSynchronize(fd.done.get()));
    fd.busy = false;
    if (info) {
        const volatile unsigned int* h = fd.h_info.get();
        info->n_records = h[0]; info->pending = h[1]; info->rows = h[2]; info->record_bytes = h[3];
    }
    return BGR_OK;
}

// ---- host edits (bgr_apply_edits) ----
int edit_fail(uint32_t i, int status, const std::string& text) { return fail(status, "edit " + std::to_string(i) + ": " + text); }

// Checks the whole batch against the row count each record sees; returns the row count after it.
int validate_edits(bgr_engine* e, const bgr_edit* edits, uint32_t n, size_t values_bytes, uint64_t* rows_out) {
    uint64_t rows = e->st.n_rows;
    for (uint32_t i = 0; i < n; ++i) {
        const bgr_edit& d = edits[i];
        const bool has_col = d.kind == BGR_EDIT_WRITE || d.kind == BGR_EDIT_INSERT || d.kind == BGR_EDIT_REMOVE;
        if (d.kind > BGR_EDIT_SPAWN) return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "unknown edit kind");
        if (has_col && d.column >= e->cols.size()) return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "unknown column");
        const Column* c = has_col ? &e->cols[d.column] : nullptr;
        if ((d.kind == BGR_EDIT_INSERT || d.kind == BGR_EDIT_REMOVE) && !c->absent)
            return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "column was not registered with BGR_STRATEGY_OPTIONAL");
        switch (d.kind) {
        case BGR_EDIT_WRITE: {
            const uint64_t end = uint64_t(d.byte_offset) + d.byte_len;
            if ((d.byte_offset & 3u) || d.byte_len == 0 || end > c->elem_bytes || ((d.byte_len & 3u) && end != c->elem_bytes))
                return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element, "
                                                              "its length a multiple of 4 or ending at the element's end");
            if (uint64_t(d.row) + d.count > rows) return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "row range exceeds the spawned rows");
            if (uint64_t(d.value_offset) + uint64_t(d.count) * d.byte_len > values_bytes)
                return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "values range exceeds values_bytes");
            break;
        }
        case BGR_EDIT_INSERT:
            if (uint64_t(d.value_offset) + c->elem_bytes > values_bytes)
                return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "values range exceeds values_bytes");
            [[fallthrough]];
        case BGR_EDIT_REMOVE:
        case BGR_EDIT_DESPAWN:
            if (d.row >= rows) return edit_fail(i, BGR_ERR_INVALID_ARGUMENT, "row out of range");
            break;
        case BGR_EDIT_SPAWN:
            rows += d.count;
            break;
        }
    }
    const uint64_t spawned = rows - e->st.n_rows;
    if (spawned) {
        if (rows > e->cfg.max_entities && !e->growable()) return fail(BGR_ERR_CAPACITY, "spawn exceeds max_entities");
        if (rows > 0xFFFFFFFFull) return fail(BGR_ERR_CAPACITY, "spawn exceeds the row index range");
        if (e->ticked && ((e->cfg.flags & BGR_CFG_SHARDED) || e->cfg.order_base != 0))
            return fail(BGR_ERR_UNSUPPORTED, "spawning after the initial population is not supported on a sharded engine "
                                             "(the new rows' RollbackOrdered indices would collide with the next shard's range)");
    }
    *rows_out = rows;
    return BGR_OK;
}

int fold_edits(bgr_engine* e, const bgr_edit* edits, uint32_t n, const uint8_t* values, EditFold& f) {
    if (f.passive.size() != e->words) {
        if (!e->stamps.empty()) {
            f.stamp_q.assign(e->words, -1);
            for (uint32_t k = 0; k < 3; ++k) {
                f.stamp_q[e->cols[e->bt].first_plane + k] = int8_t(k);
                f.stamp_q[e->cols[e->bv].first_plane + k] = int8_t(3 + k);
            }
            for (uint32_t k = 0; k < 2; ++k) f.stamp_q[e->cols[e->bl].first_plane + k] = int8_t(6 + k);
        }
        f.passive.assign(e->words, 0);
        for (uint16_t p : e->passive) f.passive[p] = 1;
    }
    const std::vector<int8_t>& stamp_q = f.stamp_q;
    const std::vector<uint8_t>& passive = f.passive;
    auto stamp = [&](uint32_t row, uint32_t q) { f.stamps.push_back((row / kSegRows) * kActivePlanes + q); };
    auto word = [&](uint32_t row, uint32_t plane, uint32_t value) {
        f.words.push_back({word_offset(e->words, row, plane) / 4u, row, plane, value});
        if (passive[plane]) f.bump = true;
    };
    size_t n_words = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const bgr_edit& d = edits[i];
        if (d.kind == BGR_EDIT_WRITE) n_words += size_t(d.count) * ((d.byte_offset + d.byte_len + 3u) / 4u - d.byte_offset / 4u);
        if (d.kind == BGR_EDIT_INSERT) n_words += e->cols[d.column].words;
    }
    f.words.reserve(n_words);
    // little-endian word `w` of an element whose bytes [lo, hi) come from `src` (src[0] is byte lo); other bytes 0
    auto pack = [](const uint8_t* src, uint32_t lo, uint32_t hi, uint32_t w) {
        uint32_t v = 0;
        if (4u * w + 4u <= hi) { std::memcpy(&v, src + (4u * w - lo), 4); return v; }  // a whole word (lo is aligned)
        for (uint32_t b = std::max(4u * w, lo); b < std::min(4u * w + 4u, hi); ++b) v |= uint32_t(src[b - lo]) << (8 * (b - 4u * w));
        return v;
    };
    auto mask = [&](uint32_t row) -> uint2& {
        auto it = f.mask_of.emplace(row, uint32_t(f.masks.size()));
        if (it.second) {
            f.masks.push_back(make_uint2(row, 0xFFu));
            if (!stamp_q.empty()) stamp(row, 8u);
        }
        return f.masks[it.first->second];
    };
    uint32_t rows = e->st.n_rows;
    for (uint32_t i = 0; i < n; ++i) {
        const bgr_edit& d = edits[i];
        switch (d.kind) {
        case BGR_EDIT_WRITE: {
            const Column& c = e->cols[d.column];
            const uint32_t w0 = d.byte_offset / 4u, w1 = (d.byte_offset + d.byte_len + 3u) / 4u;
            for (uint32_t k = 0; k < d.count; ++k) {
                const uint8_t* src = values + d.value_offset + size_t(k) * d.byte_len;
                for (uint32_t w = w0; w < w1; ++w)
                    word(d.row + k, c.first_plane + w, pack(src, d.byte_offset, d.byte_offset + d.byte_len, w));
            }
            break;
        }
        case BGR_EDIT_INSERT: {
            const Column& c = e->cols[d.column];
            for (uint32_t w = 0; w < c.words; ++w) word(d.row, c.first_plane + w, pack(values + d.value_offset, 0, c.elem_bytes, w));
            uint2& m = mask(d.row);
            if (!(m.y >> 16)) m.y = (m.y & ~c.absent) & ~(c.absent << 8);
            f.bump = true;
            break;
        }
        case BGR_EDIT_REMOVE: {
            uint2& m = mask(d.row);
            if (!(m.y >> 16)) m.y |= e->cols[d.column].absent << 8;
            f.bump = true;
            break;
        }
        case BGR_EDIT_DESPAWN:
            mask(d.row).y = 1u << 16;
            break;
        case BGR_EDIT_SPAWN:
            if (d.count) {
                for (uint64_t s = rows / kSegRows; s <= (uint64_t(rows) + d.count - 1) / kSegRows && !stamp_q.empty(); ++s)
                    for (uint32_t q = 0; q < kActivePlanes; ++q) f.stamps.push_back(uint32_t(s) * kActivePlanes + q);
                rows += d.count;
            }
            f.bump = true;
            break;
        }
    }
    // in address order (a stable LSD radix sort: words of one address stay in record order), one store per word, the
    // last record's
    uint64_t max_key = 0;
    for (const EditFold::Word& w : f.words) max_key = std::max(max_key, w.key);
    std::vector<EditFold::Word>& tmp = f.sorted;
    tmp.resize(f.words.size());
    constexpr uint32_t kDigit = 12, kBins = 1u << kDigit;
    uint32_t bins[kBins + 1];
    for (uint32_t shift = 0; shift < 64 && (max_key >> shift); shift += kDigit) {
        std::fill(bins, bins + kBins + 1, 0u);
        for (const EditFold::Word& w : f.words) ++bins[((w.key >> shift) & (kBins - 1)) + 1];
        for (uint32_t b = 1; b <= kBins; ++b) bins[b] += bins[b - 1];
        for (const EditFold::Word& w : f.words) tmp[bins[(w.key >> shift) & (kBins - 1)]++] = w;
        f.words.swap(tmp);
    }
    size_t out = 0;
    for (size_t k = 0; k < f.words.size(); ++k)
        if (k + 1 == f.words.size() || f.words[k + 1].key != f.words[k].key) f.words[out++] = f.words[k];
    f.words.resize(out);
    // the stamps the stores clear: sorted words of one (segment, plane) are adjacent.  A duplicate left elsewhere (a
    // spawn's segments) zeroes the same stamp twice.
    for (const EditFold::Word& w : f.words) {
        if (stamp_q.empty() || stamp_q[w.plane] < 0) continue;
        const uint32_t s = (w.row / kSegRows) * kActivePlanes + uint32_t(stamp_q[w.plane]);
        if (f.stamps.empty() || f.stamps.back() != s) f.stamps.push_back(s);
    }
    if (f.words.size() + f.masks.size() + f.stamps.size() > 0x7FFFFFFFull) return fail(BGR_ERR_CAPACITY, "edit batch too large");
    return BGR_OK;
}

// The staging buffer of a patch: the next one of a ring, once the batch that last used it has finished.  It grows to the
// largest patch and stays (16 B per stored word): freeing the smaller buffer synchronises the device.  Even an empty
// patch gets a buffer, so that the kernel always has a mapped address to read from.
int take_edit_stage(bgr_engine::EditStage& sg, size_t bytes) {
    CUDA_TRY(sg.done.ensure());
    if (sg.busy) CUDA_TRY(cudaEventSynchronize(sg.done.get()));
    sg.busy = false;
    CUDA_TRY(sg.h.ensure(std::max<size_t>(bytes, 64u << 10)));
    return BGR_OK;
}

int apply_edits(bgr_engine* e, const bgr_edit* edits, uint32_t n, const void* values, size_t values_bytes) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (!e->built) return fail(BGR_ERR_STATE, "engine not built");
    if ((n && !edits) || (values_bytes && !values)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (n == 0) return BGR_OK;
    uint64_t rows = 0;
    int rc = validate_edits(e, edits, n, values_bytes, &rows);
    if (rc != BGR_OK) return rc;
    EditFold& f = e->edit_fold;
    f.clear();
    rc = fold_edits(e, edits, n, static_cast<const uint8_t*>(values), f);
    if (rc != BGR_OK) return rc;
    bgr_engine::EditStage& sg = e->edit_stage[e->next_edit];
    const size_t bytes_w = f.words.size() * sizeof(uint4), bytes_m = f.masks.size() * sizeof(uint2);
    const size_t bytes = bytes_w + bytes_m + f.stamps.size() * sizeof(uint32_t);
    rc = take_edit_stage(sg, bytes);
    if (rc != BGR_OK) return rc;
    // nothing fails past the capacity: growing is the last step that can refuse
    if (rows > e->st.n_rows) rc = grow_to(e, rows);
    if (rc == BGR_OK) rc = touch_live(e);  // stream-ordered behind the queued submits, like the launches below
    if (rc != BGR_OK) return rc;
    uint4* hw = reinterpret_cast<uint4*>(sg.h.get());
    for (size_t k = 0; k < f.words.size(); ++k) hw[k] = make_uint4(f.words[k].row, f.words[k].plane, f.words[k].value, 0u);
    if (bytes_m) std::memcpy(sg.h.get() + bytes_w, f.masks.data(), bytes_m);
    if (!f.stamps.empty()) std::memcpy(sg.h.get() + bytes_w + bytes_m, f.stamps.data(), f.stamps.size() * sizeof(uint32_t));
    const uint8_t* dev = sg.h.dev();
    if (rows > e->st.n_rows) {
        const uint32_t count = uint32_t(rows - e->st.n_rows);
        k_spawn_rows<false><<<e->grid_for(count, 64), 256, 0, e->stream>>>(e->image(0), e->words, e->st.n_rows, count, nullptr, 0);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    EditPatch p{};
    p.words = reinterpret_cast<const uint4*>(dev);
    p.masks = reinterpret_cast<const uint2*>(dev + bytes_w);
    p.stamps = reinterpret_cast<const uint32_t*>(dev + bytes_w + bytes_m);
    p.n_words = uint32_t(f.words.size()); p.n_masks = uint32_t(f.masks.size()); p.n_stamps = uint32_t(f.stamps.size());
    const uint32_t total = p.n_words + p.n_masks + p.n_stamps;
    k_apply_edits<false><<<e->grid_for(total, 256), 256, 0, e->stream>>>(e->image(0), e->words, e->stamps.ptr<uint32_t>(), p);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(sg.done.get(), e->stream));
    sg.busy = true;
    e->next_edit = (e->next_edit + 1) % bgr_engine::kEditBufs;
    e->tiledep_chain = false;
    e->st.n_rows = uint32_t(rows);
    if (f.bump) e->st.live_passive_ver = ++e->st.ver_counter;
    e->st.cids.live = e->st.cids.fresh(e->st.n_rows);
    return BGR_OK;
}

void detect_bundles(bgr_engine* e) {
    e->bundle_particles = false;
    e->passive.clear();
    e->bundle_opt = false;
    for (const Column& c : e->cols)
        if (c.absent) e->bundle_opt = true;  // per-entity presence: the MODE 2 variant of the fused kernel
    const SystemReg* up = nullptr; const SystemReg* de = nullptr; const SystemReg* sp = nullptr;
    for (auto& s : e->systems) {
        if (s.id == BGR_SYS_PARTICLES_UPDATE && !up) up = &s;
        else if (s.id == BGR_SYS_PARTICLES_DESPAWN && !de) de = &s;
        else if (s.id == BGR_SYS_PARTICLES_SPAWN && !sp) sp = &s;
        else return;  // any other system: generic path
    }
    if (!up || !de) return;
    uint32_t t = up->cols[0], v = up->cols[1], l = de->cols[0];
    if (sp && (sp->cols[0] != t || sp->cols[1] != v || sp->cols[2] != l)) return;
    if (t == v || t == l || v == l) return;
    auto ck_ok = [&](const Column& c) {
        return c.hash_kind == BGR_HASH_NONE || (c.hash_kind == BGR_HASH_BYTES && c.hash_off == 0 && c.hash_len == 12);
    };
    if (!ck_ok(e->cols[t]) || !ck_ok(e->cols[v])) return;
    for (size_t i = 0; i < e->cols.size(); ++i)
        if (i != t && i != v && e->cols[i].hash_kind != BGR_HASH_NONE) return;  // other checksums: generic path
    // active planes: translation (3 words of Transform), velocity (3), ttl (2)
    std::vector<uint8_t> active(e->words, 0);
    for (uint32_t k = 0; k < 3; ++k) { active[e->cols[t].first_plane + k] = 1; active[e->cols[v].first_plane + k] = 1; }
    for (uint32_t k = 0; k < 2; ++k) active[e->cols[l].first_plane + k] = 1;
    for (uint32_t p = 0; p < e->words; ++p)
        if (!active[p]) e->passive.push_back(uint16_t(p));
    if (e->passive.size() > size_t(kMaxPassive)) { e->passive.clear(); return; }
    // runs of adjacent passive planes: one cp.async.bulk each
    e->runs.clear(); e->passive_bytes = 0;
    for (size_t i = 0; i < e->passive.size();) {
        size_t j = i;
        while (j + 1 < e->passive.size() && e->passive[j + 1] == e->passive[j] + 1) ++j;
        PassiveRun r{uint32_t(e->passive[i]) * kPlaneBytes, uint32_t(j - i + 1) * kPlaneBytes};
        e->runs.push_back(r);
        e->passive_bytes += r.bytes;
        i = j + 1;
    }
    if (e->runs.size() > size_t(kMaxRuns)) { e->runs.clear(); e->passive_bytes = 0; }
    const bool fin_t = e->cols[t].hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32, fin_v = e->cols[v].hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32;
    const bool ck_t = e->cols[t].hash_kind != BGR_HASH_NONE, ck_v = e->cols[v].hash_kind != BGR_HASH_NONE;
    e->bundle_static_ck = ck_t && ck_v && fin_t && fin_v;
    e->bt = t; e->bv = v; e->bl = l;
    e->bundle_particles = true;
}

// Points the result views h_out / d_out at the engine's own blocks (outside a shard group).
void use_own_blocks(bgr_engine* e) {
    for (int b = 0; b < bgr_engine::kBufs; ++b) { e->h_out[b] = e->out_block[b].get(); e->d_out[b] = e->out_block[b].dev(); }
}

// Unregisters the group's segment and points the result views back at the engine's own blocks (the caller has
// synchronised the stream).
void leave_group(bgr_engine* e) {
    cudaHostUnregister(e->group->blocks_base());
    use_own_blocks(e);
    delete e->group;
    e->group = nullptr;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

BGR_API uint32_t bgr_abi_version(void) { return BGR_ABI_VERSION; }
BGR_API const char* bgr_last_error(void) { return g_err.c_str(); }

BGR_API int bgr_engine_create(const bgr_config* cfg, bgr_engine** out) {
    if (!cfg || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (cfg->abi_version != BGR_ABI_VERSION) return fail(BGR_ERR_INVALID_ARGUMENT, "ABI version mismatch");
    if (cfg->max_entities == 0 || cfg->fps == 0) return fail(BGR_ERR_INVALID_ARGUMENT, "max_entities and fps must be > 0");
    if (cfg->max_depth == 0 || cfg->max_depth > 64) return fail(BGR_ERR_INVALID_ARGUMENT, "max_depth must be in 1..64");
    if (cfg->flags & BGR_CFG_DESYNC_CAPTURE) {
        if (cfg->flags & BGR_CFG_SHARDED) return fail(BGR_ERR_UNSUPPORTED, "BGR_CFG_DESYNC_CAPTURE is not supported on a sharded engine");
        if (cfg->max_depth > SlotRing::kMaxSlots / 2)
            return fail(BGR_ERR_INVALID_ARGUMENT, "BGR_CFG_DESYNC_CAPTURE needs max_depth <= 32 (2 * max_depth frame slots)");
    }
    // a shard's rows are a fixed range of RollbackOrdered indices, and sharded engines do not spawn
    if ((cfg->flags & BGR_CFG_GROWABLE) && ((cfg->flags & BGR_CFG_SHARDED) || cfg->order_base != 0))
        return fail(BGR_ERR_UNSUPPORTED, "BGR_CFG_GROWABLE is not supported on a sharded engine (BGR_CFG_SHARDED / order_base != 0)");
    int n_dev = 0;
    cudaError_t ce = cudaGetDeviceCount(&n_dev);
    if (ce != cudaSuccess || n_dev == 0)
        return fail(BGR_ERR_CUDA, std::string("no CUDA device available (bevy_ggrs_b200 has no CPU fallback): ") + cudaGetErrorString(ce));
    if (cfg->device < 0 || cfg->device >= n_dev) return fail(BGR_ERR_INVALID_ARGUMENT, "bad device ordinal");
    CUDA_TRY(cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(BGR_ERR_CUDA, "device is not sm_90 (Hopper); this library only carries sm_90a code");
    bgr_engine* e = new bgr_engine();
    e->cfg = *cfg;
    e->num_sms = prop.multiProcessorCount;
    if (cfg->stream) { e->stream = static_cast<cudaStream_t>(cfg->stream); e->own_stream = false; }
    else {
        cudaError_t se = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
        if (se != cudaSuccess) { delete e; return fail(BGR_ERR_CUDA, cudaGetErrorString(se)); }
        e->own_stream = true;
    }
    e->tune_bps = env_int("BGR_TUNE_BPS", 0);
    e->tune_tma = env_int("BGR_TUNE_TMA", 1);
    e->tune_passive_tma = env_int("BGR_TUNE_PASSIVE_TMA", 1);
    e->tune_poll = env_int("BGR_TUNE_POLL", 1);
    e->tune_dynamic = env_int("BGR_TUNE_DYNAMIC", 1);
    e->tune_prefetch = env_int("BGR_TUNE_PREFETCH", 1);
    e->tune_grid = env_int("BGR_TUNE_GRID", 0);
    e->tune_tiledep = env_int("BGR_TUNE_TILEDEP", 1);
    e->tune_generic = env_int("BGR_TUNE_GENERIC", 1);
    e->tune_jit = env_int("BGR_TUNE_JIT", 1);
    e->tune_jit_rows = env_int("BGR_TUNE_JIT_ROWS", 4);
    e->tune_jit_item = env_int("BGR_TUNE_JIT_ITEM", 0);
    e->tune_replay_points = uint32_t(std::max(1, env_int("BGR_TUNE_REPLAY_POINTS", int(kReplayLaunchPoints))));
    e->tune_keyframe_bytes = uint64_t(std::max(1, env_int("BGR_TUNE_KEYFRAME_BYTES", int(kKeyframeLaunchBytes))));
    e->tune_trace_bytes = uint64_t(std::max(1, env_int("BGR_TUNE_TRACE_BYTES", int(kTraceLaunchBytes))));
    e->tune_jit_tiledep = env_int("BGR_TUNE_JIT_TILEDEP", 0);
    e->tune_passive_early = env_int("BGR_TUNE_PASSIVE_EARLY", -1);
    e->tune_stagger_ns = env_int("BGR_TUNE_STAGGER_NS", 800);
    e->tune_bundle = env_int("BGR_TUNE_BUNDLE", 1);
    e->tune_defer_live = env_int("BGR_TUNE_DEFER_LIVE", 1);
    e->tune_held_saves = env_int("BGR_TUNE_HELD_SAVES", 1);
    // tests: the first content stamp issued, so that the range rollover in run_fused is reached within a few launches
    if (const char* v = std::getenv("BGR_TEST_STAMP_FIRST"); v && *v)
        e->stamp_next = uint32_t(std::max(1ul, std::min(std::strtoul(v, nullptr, 0), 0xFFFFFFFFul)));
    e->st.confirmed = 0;
    *out = e;
    return BGR_OK;
}

BGR_API void bgr_engine_destroy(bgr_engine* e) {
    if (!e) return;
    cudaSetDevice(e->cfg.device);
    // nothing is released while a stream that could still use it runs
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->copy_stream) { cudaStreamSynchronize(e->copy_stream); cudaStreamDestroy(e->copy_stream); }
    if (e->group) leave_group(e);
    cudaStream_t own = e->own_stream ? e->stream : nullptr;
    delete e;
    if (own) cudaStreamDestroy(own);
}

BGR_API int bgr_rollback_component(bgr_engine* e, const char* type_name, uint32_t elem_bytes, uint32_t strategy,
                                   uint32_t* column_out) {
    if (!e || !column_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (e->built) return fail(BGR_ERR_STATE, "components must be registered before bgr_build");
    if (elem_bytes == 0 || elem_bytes > 1024) return fail(BGR_ERR_INVALID_ARGUMENT, "elem_bytes must be in 1..1024");
    const bool optional = strategy & BGR_STRATEGY_OPTIONAL;
    strategy &= ~BGR_STRATEGY_OPTIONAL;
    if (strategy != BGR_STRATEGY_COPY && strategy != BGR_STRATEGY_CLONE)
        return fail(BGR_ERR_UNSUPPORTED, "only Copy/Clone strategies of POD types are supported (ReflectStrategy is out of scope)");
    Column c;
    if (optional) {
        uint32_t n_opt = 0;
        for (const Column& o : e->cols) n_opt += o.absent ? 1u : 0u;
        if (n_opt >= BGR_MAX_OPTIONAL_COLUMNS) return fail(BGR_ERR_CAPACITY, "more than BGR_MAX_OPTIONAL_COLUMNS optional columns");
        c.absent = 2u << n_opt;
    }
    c.name = type_name ? type_name : "";
    c.elem_bytes = elem_bytes;
    c.words = (elem_bytes + 3) / 4;
    c.strategy = strategy;
    e->cols.push_back(c);
    *column_out = uint32_t(e->cols.size() - 1);
    return BGR_OK;
}

BGR_API int bgr_checksum_component(bgr_engine* e, uint32_t column, uint32_t hash_kind, uint32_t byte_offset,
                                   uint32_t byte_len, uint32_t flags) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (e->built) return fail(BGR_ERR_STATE, "checksums must be registered before bgr_build");
    if (column >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown column");
    Column& c = e->cols[column];
    if (hash_kind != BGR_HASH_BYTES) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown hash kind");
    if (uint64_t(byte_offset) + byte_len > c.elem_bytes) return fail(BGR_ERR_INVALID_ARGUMENT, "hash range exceeds element");
    if ((flags & BGR_HASH_FLAG_ASSERT_FINITE_F32) && ((byte_offset | byte_len) & 3u))
        return fail(BGR_ERR_INVALID_ARGUMENT, "finite-f32 assertion needs a 4-byte aligned range");
    c.hash_kind = hash_kind; c.hash_off = byte_offset; c.hash_len = byte_len; c.hash_flags = flags;
    return BGR_OK;
}

BGR_API int bgr_add_system(bgr_engine* e, uint32_t system, const uint32_t* columns, uint32_t n_columns,
                           const uint32_t* params, uint32_t n_params) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (e->built) return fail(BGR_ERR_STATE, "systems must be added before bgr_build");
    SystemReg s;
    s.id = system;
    for (uint32_t i = 0; i < n_columns; ++i) {
        if (columns[i] >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "system binds an unknown column");
        s.cols.push_back(columns[i]);
    }
    for (uint32_t i = 0; i < n_params; ++i) s.params.push_back(params[i]);
    auto need = [&](size_t nc, size_t np) { return s.cols.size() == nc && s.params.size() >= np; };
    auto eb = [&](size_t i) { return e->cols[s.cols[i]].elem_bytes; };
    switch (system) {
    case BGR_SYS_PARTICLES_UPDATE:
        if (!need(2, 0) || eb(0) != 40 || eb(1) != 12)
            return fail(BGR_ERR_INVALID_ARGUMENT, "update_particles binds {Transform(40B), Velocity(12B)}");
        break;
    case BGR_SYS_PARTICLES_DESPAWN:
        if (!need(1, 0) || eb(0) != 8) return fail(BGR_ERR_INVALID_ARGUMENT, "despawn_particles binds {Ttl(8B)}");
        break;
    case BGR_SYS_U32_ADD:
    case BGR_SYS_U32_SATSUB_DESPAWN:
        if (!need(1, 2) || (s.params[0] & 3u) || s.params[0] + 4 > eb(0))
            return fail(BGR_ERR_INVALID_ARGUMENT, "u32 system binds {C} with params {aligned byte_offset, k}");
        break;
    case BGR_SYS_U32_STORE_CALL_COUNT:
        if (!need(1, 1) || (s.params[0] & 3u) || s.params[0] + 4 > eb(0))
            return fail(BGR_ERR_INVALID_ARGUMENT, "store_call_count binds {C} with params {aligned byte_offset}");
        break;
    case BGR_SYS_PARTICLES_SPAWN:
        if (!need(3, 4) || eb(0) != 40 || eb(1) != 12 || eb(2) != 8)
            return fail(BGR_ERR_INVALID_ARGUMENT, "spawn_particles binds {Transform(40B), Velocity(12B), Ttl(8B)} with params {rate, ttl, seed_lo, seed_hi}");
        if (e->spawn_sys >= 0) return fail(BGR_ERR_INVALID_ARGUMENT, "spawn_particles registered twice");
        // A shard appends rows locally: the RollbackOrdered index order_base + row of a newborn would collide with the
        // next shard's range, and every shard would draw the same ParticleRng stream.  Dynamic spawning needs one GPU.
        if ((e->cfg.flags & BGR_CFG_SHARDED) || e->cfg.order_base != 0)
            return fail(BGR_ERR_UNSUPPORTED, "spawn_particles is not supported on a sharded engine (BGR_CFG_SHARDED / order_base != 0)");
        if (s.params[0] == 0 || s.params[0] > 4096) return fail(BGR_ERR_INVALID_ARGUMENT, "spawn rate must be in 1..4096");
        e->spawn_sys = int(e->systems.size());
        e->st.rng.seed_from_u64(uint64_t(s.params[2]) | (uint64_t(s.params[3]) << 32));  // insert_resource(ParticleRng(seed_from_u64(seed)))
        break;
    case BGR_SYS_BOX_MOVE:
        if (!need(2, 0) || eb(0) != 40 || eb(1) != 12)
            return fail(BGR_ERR_INVALID_ARGUMENT, "move_cube_system binds {Transform(40B), Velocity(12B)}");
        break;
    case BGR_SYS_DESPAWN_ON_INPUT:
        if (!need(1, 2) || s.params[0] >= BGR_MAX_PLAYERS || s.params[1] > 0xFF)
            return fail(BGR_ERR_INVALID_ARGUMENT, "despawn_on_input binds {C} with params {player_handle < 8, value <= 255}");
        break;
    default: return fail(BGR_ERR_INVALID_ARGUMENT, "unknown system id");
    }
    e->systems.push_back(std::move(s));
    return BGR_OK;
}

BGR_API int bgr_build(bgr_engine* e) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (e->built) return fail(BGR_ERR_STATE, "bgr_build called twice");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    uint32_t plane = 0;
    e->n_ck = 0;
    for (Column& c : e->cols) {
        c.first_plane = plane;
        plane += c.words;
        if (c.hash_kind != BGR_HASH_NONE) {
            if (e->n_ck >= BGR_MAX_CHECKSUM_COLUMNS) return fail(BGR_ERR_CAPACITY, "too many checksummed columns");
            c.ck_slot = int(e->n_ck++);
        }
    }
    e->words = plane;
    e->epad = (e->cfg.max_entities + kTileRows - 1) / kTileRows * kTileRows;
    e->n_tiles_cap = e->epad / kTileRows;
    e->tile_bytes = tile_bytes_of(e->words);
    e->image_bytes = (size_t(e->n_tiles_cap) * e->tile_bytes + 255u) & ~size_t(255);  // ops address images in 256-byte units
    if (e->n_slots() > SlotRing::kMaxSlots)
        return fail(BGR_ERR_INVALID_ARGUMENT, "bgr_retain_confirmed: " + std::to_string(e->n_slots() - e->retain_count) +
                                                  " ring slots + " + std::to_string(e->retain_count) + " retained frames = " +
                                                  std::to_string(e->n_slots()) + " frame slots, more than " +
                                                  std::to_string(SlotRing::kMaxSlots));
    if ((e->image_bytes * (size_t(e->n_slots()) + 1u)) >> 8 > 0xffffffffull)
        return fail(BGR_ERR_CAPACITY, "arena larger than 1 TB");
    e->ceiling = e->cfg.max_entities;
    if (e->growable()) {
        // The ceiling: ops address images in 256-byte units with 32 bits, so all images together stay within 1 TB, and a
        // row index is 32 bits.  Every image gets a stride of whole mapping granules sized for the ceiling.
        std::string err;
        const size_t gran = StridedRange::granularity(e->cfg.device, &err);
        if (!gran) return fail(BGR_ERR_CUDA, err);
        const uint64_t per_image = ((uint64_t(1) << 40) / (e->n_slots() + 1u)) / gran * gran;
        const uint64_t ceil_tiles = std::min<uint64_t>(per_image / e->tile_bytes, 0xFFFFFFFFull / kTileRows);
        if (ceil_tiles < e->n_tiles_cap)
            return fail(BGR_ERR_CAPACITY, "max_entities exceeds the ceiling of a growable engine with this schema and slot count (" +
                                              std::to_string(ceil_tiles * kTileRows) + " rows)");
        e->ceiling = uint32_t(ceil_tiles * kTileRows);
    }
    const size_t acc_bytes = sizeof(unsigned long long) * kMaxSaves * kAccStride;
    CUDA_TRY(e->accum.ensure(kMaxSaves * kAccStride * bgr_engine::kBufs));
    CUDA_TRY(cudaMemsetAsync(e->accum.get(), 0, acc_bytes * bgr_engine::kBufs, e->stream));
    CUDA_TRY(e->ticket.ensure(4 * bgr_engine::kBufs));
    CUDA_TRY(cudaMemsetAsync(e->ticket.get(), 0, 4 * sizeof(unsigned int) * bgr_engine::kBufs, e->stream));
    for (int s = 0; s < bgr_engine::kBufs; ++s) {
        e->d_accum_set[s] = e->accum.get() + size_t(s) * kMaxSaves * kAccStride;
        e->d_ticket_set[s] = e->ticket.get() + 4 * s;
    }
    CUDA_TRY(e->internal_out.ensure(kResultStride));
    for (int i = 0; i < bgr_engine::kBufs; ++i) {
        CUDA_TRY(e->out_block[i].ensure(kResultStride));
        std::memset(e->out_block[i].get(), 0, sizeof(unsigned long long) * kResultStride);
        CUDA_TRY(e->ev[i].ensure());
    }
    use_own_blocks(e);
    e->st.ring.reset(e->n_slots(), e->capture());
    e->st.ring.set_retention(e->retain_interval, e->retain_count);
    e->st.slot_rows.fill(0);
    e->st.slot_elapsed_ns.fill(0);
    e->st.slot_passive_ver.fill(0);
    if (e->spawn_sys >= 0)
        for (int i = 0; i < bgr_engine::kBufs; ++i) CUDA_TRY(e->spawn[i].ensure(kMaxSpawnVals));
    build_specs(e);
    detect_bundles(e);
    // generic one-launch program: every row system runs on its tile (run_system) and spawned rows are written after the
    // frame's despawns (spawn_row); the parameter block holds kMaxGenericSys systems; the tile fits twice per SM
    e->generic_ok = e->sys_specs.size() <= size_t(kMaxGenericSys) && e->tile_bytes <= 100u * 1024u;
    jit_specialise(e);
    {   // TMA copy kernel: up to six one-tile stages in ~200 KB of shared memory, at least two
        uint32_t st = uint32_t(std::min<size_t>((200u * 1024u) / e->tile_bytes, size_t(kTmaMaxStages)));
        if (env_int("BGR_TUNE_TMA_STAGES", 0) > 0) st = std::min(st, uint32_t(env_int("BGR_TUNE_TMA_STAGES", 0)));
        e->tma_stage_tiles = st >= 2 ? st : 0;
        if (e->tma_stage_tiles) {
            size_t smem = size_t(e->tma_stage_tiles) * e->tile_bytes;
            CUDA_TRY(cudaFuncSetAttribute(k_image_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
            CUDA_TRY(e->tma_ticket.ensure(4));
            CUDA_TRY(cudaMemsetAsync(e->tma_ticket.get(), 0, 4 * sizeof(unsigned int), e->stream));
        }
    }
    if (e->tune_held_saves == 2 && use_bundle(e)) {
        CUDA_TRY(e->held_check.ensure(1));
        CUDA_TRY(cudaMemsetAsync(e->held_check.get(), 0, sizeof(unsigned long long), e->stream));
    }
    std::string err;
    for (const CapacityBuffer& b : capacity_buffers(e))
        if (b.wanted && !create_range(e, b, &err)) return fail(BGR_ERR_CUDA, err);
    e->image_bytes = e->arena.stride;
    const int rc = map_tiles(e, e->n_tiles_cap);  // maps the capacity and zeroes every capacity buffer
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->built = true;
    return BGR_OK;
}

BGR_API int bgr_run_startup_system(bgr_engine* e, uint32_t system) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (system != BGR_SYS_PARTICLES_SPAWN || e->spawn_sys < 0)
        return fail(BGR_ERR_INVALID_ARGUMENT, "only a registered spawn_particles system can run at Startup");
    int rc = drain(e);
    if (rc == BGR_OK) rc = touch_live(e);
    if (rc != BGR_OK) return rc;
    const SystemReg& sy = e->systems[size_t(e->spawn_sys)];
    const uint32_t rate = sy.params[0];
    if (uint64_t(e->st.n_rows) + rate > e->cfg.max_entities) {
        if (!e->growable()) return fail(BGR_ERR_CAPACITY, "spawn_particles exceeds max_entities");
        rc = grow_to(e, uint64_t(e->st.n_rows) + rate);
        if (rc != BGR_OK) return rc;
    }
    for (uint32_t k = 0; k < rate; ++k) {
        e->spawn[0].get()[k].x = e->st.rng.random_range(-200.0f, 200.0f);
        e->spawn[0].get()[k].y = e->st.rng.random_range(-200.0f, 200.0f);
    }
    const uint64_t ttl = sy.params[1];
    k_sys_particles_spawn<<<e->grid_for(rate, 256), 256, 0, e->stream>>>(e->image(0), e->words, e->sys_specs[size_t(e->spawn_sys)],
                                                                         e->st.n_rows, rate, e->spawn[0].dev(), ttl);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    e->st.n_rows += rate;  // before clear_stamps: the fresh content id carries the new row count
    rc = clear_stamps(e, 0);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->st.live_passive_ver = ++e->st.ver_counter;
    return BGR_OK;
}

BGR_API int bgr_spawn(bgr_engine* e, uint32_t count, uint32_t* first_row_out) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    int rc = drain(e);
    if (rc == BGR_OK) rc = touch_live(e);
    if (rc != BGR_OK) return rc;
    if (uint64_t(e->st.n_rows) + count > e->cfg.max_entities && !e->growable()) return fail(BGR_ERR_CAPACITY, "spawn exceeds max_entities");
    if (count && e->ticked && ((e->cfg.flags & BGR_CFG_SHARDED) || e->cfg.order_base != 0))
        return fail(BGR_ERR_UNSUPPORTED, "bgr_spawn after the initial population is not supported on a sharded engine "
                                         "(the new rows' RollbackOrdered indices would collide with the next shard's range)");
    rc = grow_to(e, uint64_t(e->st.n_rows) + count);
    if (rc != BGR_OK) return rc;
    uint32_t first = e->st.n_rows;
    if (count) {
        k_spawn_rows<false><<<e->grid_for(count, 64), 256, 0, e->stream>>>(e->image(0), e->words, first, count, nullptr, 0);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        e->st.n_rows += count;  // before clear_stamps: the fresh content id carries the new row count
        rc = clear_stamps(e, 0);
        if (rc != BGR_OK) return rc;
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    e->st.live_passive_ver = ++e->st.ver_counter;
    if (first_row_out) *first_row_out = first;
    return BGR_OK;
}

BGR_API int bgr_reserve(bgr_engine* e, uint32_t rows) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (rows <= e->cfg.max_entities) return BGR_OK;
    if (!e->growable()) return fail(BGR_ERR_UNSUPPORTED, "bgr_reserve past the capacity needs an engine created with BGR_CFG_GROWABLE");
    return grow_to(e, rows);
}

BGR_API int bgr_capacity(bgr_engine* e, uint32_t* capacity_out, uint32_t* ceiling_out) {
    if (!e || !capacity_out || !ceiling_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (!e->built) return fail(BGR_ERR_STATE, "engine not built");
    *capacity_out = e->cfg.max_entities;
    *ceiling_out = e->ceiling;
    return BGR_OK;
}

BGR_API int bgr_despawn(bgr_engine* e, uint32_t row) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    int rc = drain(e);
    if (rc == BGR_OK) rc = touch_live(e);
    if (rc != BGR_OK) return rc;
    if (row >= e->st.n_rows) return fail(BGR_ERR_INVALID_ARGUMENT, "row out of range");
    k_set_alive<<<1, 1, 0, e->stream>>>(e->image(0), e->words, row, 0);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    rc = clear_stamps(e, 0);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return BGR_OK;
}

BGR_API int bgr_row_count(bgr_engine* e, uint32_t* rows_out) {
    if (!e || !rows_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *rows_out = e->st.n_rows;
    return BGR_OK;
}

BGR_API int bgr_active_count(bgr_engine* e, uint64_t* active_out) {
    if (!e || !e->built || !active_out) return fail(BGR_ERR_STATE, "engine not built");
    std::vector<uint8_t> a(e->st.n_rows);
    int rc = read_alive_image(e, 0, 0, e->st.n_rows, e->st.n_rows, a.data());
    if (rc != BGR_OK) return rc;
    uint64_t n = 0;
    for (uint8_t v : a) n += v ? 1 : 0;
    *active_out = n;
    return BGR_OK;
}

BGR_API int bgr_write_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count, const void* host_src,
                                uint32_t stride) {
    if (!host_src && count) return fail(BGR_ERR_INVALID_ARGUMENT, "null host buffer");
    return transfer_column(e, 0, column, first_row, count, const_cast<void*>(host_src), stride, true);
}

BGR_API int bgr_read_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count, void* host_dst,
                               uint32_t stride) {
    if (!host_dst && count) return fail(BGR_ERR_INVALID_ARGUMENT, "null host buffer");
    return transfer_column(e, 0, column, first_row, count, host_dst, stride, false);
}

static int presence_args(bgr_engine* e, uint32_t column, uint32_t row) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (column >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown column");
    if (!e->cols[column].absent) return fail(BGR_ERR_INVALID_ARGUMENT, "column was not registered with BGR_STRATEGY_OPTIONAL");
    if (row >= e->st.n_rows) return fail(BGR_ERR_INVALID_ARGUMENT, "row out of range");
    const int rc = drain(e);
    return rc == BGR_OK ? touch_live(e) : rc;
}
BGR_API int bgr_remove_component(bgr_engine* e, uint32_t column, uint32_t row) {
    int rc = presence_args(e, column, row);
    if (rc != BGR_OK) return rc;
    k_set_absent<<<1, 1, 0, e->stream>>>(e->image(0), e->words, row, e->cols[column].absent, 1u);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    rc = clear_stamps(e, 0);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    e->st.live_passive_ver = ++e->st.ver_counter;
    return BGR_OK;
}
BGR_API int bgr_insert_component(bgr_engine* e, uint32_t column, uint32_t row, const void* value) {
    if (!value) return fail(BGR_ERR_INVALID_ARGUMENT, "null value");
    int rc = presence_args(e, column, row);
    if (rc != BGR_OK) return rc;
    rc = transfer_column(e, 0, column, row, 1, const_cast<void*>(value), e->cols[column].elem_bytes, true);
    if (rc != BGR_OK) return rc;
    k_set_absent<<<1, 1, 0, e->stream>>>(e->image(0), e->words, row, e->cols[column].absent, 0u);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    rc = clear_stamps(e, 0);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return BGR_OK;
}
BGR_API int bgr_has_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count, uint8_t* host_dst) {
    if (!e || !e->built || !host_dst) return fail(BGR_ERR_STATE, "engine not built");
    if (column >= e->cols.size()) return fail(BGR_ERR_INVALID_ARGUMENT, "unknown column");
    return read_alive_image(e, 0, first_row, count, e->st.n_rows, host_dst, e->cols[column].absent);
}

BGR_API int bgr_apply_edits(bgr_engine* e, const bgr_edit* edits, uint32_t n, const void* values, size_t values_bytes) {
    return apply_edits(e, edits, n, values, values_bytes);
}

BGR_API int bgr_host_alloc(size_t bytes, void** out) {
    if (!out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    CUDA_TRY(cudaHostAlloc(out, std::max<size_t>(bytes, 1), cudaHostAllocPortable));
    return BGR_OK;
}
BGR_API int bgr_host_free(void* p) {
    if (p) CUDA_TRY(cudaFreeHost(p));
    return BGR_OK;
}
BGR_API int bgr_download_begin(bgr_engine* e, uint32_t column, uint32_t byte_offset, uint32_t byte_len, uint32_t first_row,
                               uint32_t count, void* host_dst, uint32_t* ticket_out) {
    return download_begin(e, column, byte_offset, byte_len, first_row, count, host_dst, ticket_out);
}
BGR_API int bgr_download_wait(bgr_engine* e, uint32_t ticket) { return download_wait(e, ticket); }
BGR_API int bgr_feed_create(bgr_engine* e, const bgr_feed_field* fields, uint32_t n_fields, uint32_t* feed_out) {
    return feed_create(e, fields, n_fields, feed_out);
}
BGR_API int bgr_feed_reset(bgr_engine* e, uint32_t feed) {
    return feed_reset(e, feed);
}
BGR_API int bgr_feed_begin(bgr_engine* e, uint32_t feed, void* host_dst, uint32_t records_cap, uint32_t* ticket_out) {
    return feed_begin(e, feed, host_dst, records_cap, ticket_out);
}
BGR_API int bgr_feed_wait(bgr_engine* e, uint32_t ticket, bgr_feed_info* info) {
    return feed_wait(e, ticket, info);
}

BGR_API int bgr_read_alive(bgr_engine* e, uint32_t first_row, uint32_t count, uint8_t* host_dst) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    return read_alive_image(e, 0, first_row, count, e->st.n_rows, host_dst);
}

BGR_API int bgr_rollback_frame_count(bgr_engine* e, int32_t* out) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = e->st.frame_count; return BGR_OK;
}
BGR_API int bgr_set_rollback_frame_count(bgr_engine* e, int32_t frame) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    e->st.frame_count = frame; return BGR_OK;
}
BGR_API int bgr_confirmed_frame_count(bgr_engine* e, int32_t* out) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = e->st.confirmed; return BGR_OK;
}
BGR_API int bgr_max_prediction_window(bgr_engine* e, uint32_t* out) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = e->st.has_maxpred ? e->st.maxpred : 0; return BGR_OK;
}

// Ring operations outside a program can hand the slot of a deferred live image's base to a later Save: the live image
// is written first.
BGR_API int bgr_set_depth(bgr_engine* e, uint32_t depth) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    const int rc = materialize_live(e);
    if (rc != BGR_OK) return rc;
    e->st.has_maxpred = true; e->st.maxpred = depth;  // MaxPredictionWindow: sync_depth applies it before every save
    e->st.ring.set_depth(depth);
    return BGR_OK;
}
BGR_API int bgr_confirm(bgr_engine* e, int32_t confirmed_frame) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    const int rc = materialize_live(e);
    if (rc != BGR_OK) return rc;
    e->st.confirmed = confirmed_frame;
    e->st.ring.confirm(confirmed_frame);
    return BGR_OK;
}
BGR_API int bgr_snapshot_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    std::vector<int32_t> f;
    e->st.ring.frames(&f);
    for (uint32_t i = 0; i < f.size() && i < cap && frames_out; ++i) frames_out[i] = f[i];
    if (n_out) *n_out = uint32_t(f.size());
    return BGR_OK;
}

BGR_API int bgr_peek(bgr_engine* e, int32_t frame, uint32_t column, uint32_t first_row, uint32_t count, void* host_dst,
                     uint32_t stride, uint8_t* alive_dst, int32_t* found) {
    if (!e || !e->built || !found) return fail(BGR_ERR_STATE, "engine not built");
    uint32_t slot = 0;
    if (!e->st.ring.peek(frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    int rc = transfer_column(e, slot + 1, column, first_row, count, host_dst, stride, false);
    if (rc != BGR_OK) return rc;
    // alive_dst[i] = the snapshot of `frame` holds this column for row first_row+i (the row existed and had the component)
    if (alive_dst) return read_alive_image(e, slot + 1, first_row, count, e->st.slot_rows[slot], alive_dst, e->cols[column].absent);
    return BGR_OK;
}

// ---- desync capture (BGR_CFG_DESYNC_CAPTURE; ring.hpp keeps the witnesses, desync_diff.cuh compares) ----
static int capture_args(bgr_engine* e) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (!e->capture()) return fail(BGR_ERR_STATE, "the engine was not created with BGR_CFG_DESYNC_CAPTURE");
    return drain(e);
}

BGR_API int bgr_desync_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out) {
    int rc = capture_args(e);
    if (rc != BGR_OK) return rc;
    std::vector<int32_t> f;
    e->st.ring.desync_frames(&f);
    for (uint32_t i = 0; i < f.size() && i < cap && frames_out; ++i) frames_out[i] = f[i];
    if (n_out) *n_out = uint32_t(f.size());
    return BGR_OK;
}

BGR_API int bgr_peek_first(bgr_engine* e, int32_t frame, uint32_t column, uint32_t first_row, uint32_t count,
                           void* host_dst, uint32_t stride, uint8_t* alive_dst, int32_t* found) {
    if (!found) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = capture_args(e);
    if (rc != BGR_OK) return rc;
    uint32_t slot = 0;
    if (!e->st.ring.first(frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    rc = transfer_column(e, slot + 1, column, first_row, count, host_dst, stride, false);
    if (rc != BGR_OK) return rc;
    if (alive_dst) return read_alive_image(e, slot + 1, first_row, count, e->st.slot_rows[slot], alive_dst, e->cols[column].absent);
    return BGR_OK;
}

// the column table and counters of k_desync_*, allocated by the first diff; records grow with records_cap
static int ensure_diff_scratch(bgr_engine* e, uint32_t records_cap) {
    const uint32_t n_cols = uint32_t(e->cols.size());
    if (!e->diff_cols.get()) {
        std::vector<DiffColumn> dc(n_cols);
        for (uint32_t c = 0; c < n_cols; ++c) {
            const Column& k = e->cols[c];
            const bool ck = k.hash_kind != BGR_HASH_NONE && k.hash_len > 0;
            dc[c] = DiffColumn{k.first_plane, k.words, k.absent, ck ? k.hash_off : 0u, ck ? k.hash_off + k.hash_len : 0u};
        }
        CUDA_TRY(e->diff_cols.ensure(std::max(1u, n_cols)));
        // on the engine's (non-blocking) stream: ordered before the pass-1 launch that reads the table
        CUDA_TRY(cudaMemcpyAsync(e->diff_cols.get(), dc.data(), sizeof(DiffColumn) * n_cols, cudaMemcpyHostToDevice, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));  // `dc` is a pageable host vector that goes out of scope below
        CUDA_TRY(e->diff_totals.ensure(3));
    }
    CUDA_TRY(e->diff_counts.ensure(3u * n_cols + e->n_tiles_cap));
    CUDA_TRY(e->diff_list.ensure(2u * e->n_tiles_cap));
    CUDA_TRY(e->diff_records.ensure(records_cap));
    return BGR_OK;
}

// Both passes of the diff over `n_pos` work positions (tiles, or the entries of p.visit); fills the summary's counts.
static int run_diff(bgr_engine* e, DiffParams p, uint32_t n_pos, int32_t frame, bgr_desync_summary* summary,
                    bgr_desync_column* cols, uint32_t cols_cap, bgr_desync_record* records, uint32_t records_cap,
                    uint32_t* n_records) {
    const uint32_t n_cols = uint32_t(e->cols.size());
    int rc = ensure_diff_scratch(e, records_cap);
    if (rc != BGR_OK) return rc;
    p.words = e->words;
    p.n_cols = n_cols;
    p.cols = e->diff_cols.get();
    p.col_counts = e->diff_counts.get();
    p.totals = e->diff_totals.get();
    p.tile_records = e->diff_counts.get() + 3u * n_cols;
    p.cap = records_cap;
    p.out = e->diff_records.get();
    std::vector<unsigned int> counts(3u * n_cols + n_pos, 0u);
    unsigned long long totals[3] = {0, 0, 0};
    if (n_pos) {
        CUDA_TRY(cudaMemsetAsync(e->diff_counts.get(), 0, sizeof(unsigned int) * 3u * n_cols, e->stream));
        CUDA_TRY(cudaMemsetAsync(e->diff_totals.get(), 0, sizeof(unsigned long long) * 3u, e->stream));
        k_desync_count<<<n_pos, kDiffBlock, 0, e->stream>>>(p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(counts.data(), e->diff_counts.get(), sizeof(unsigned int) * counts.size(), cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaMemcpyAsync(totals, e->diff_totals.get(), sizeof totals, cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    // exclusive scan of the per-position record counts: the positions that hold one of the first records_cap records
    std::vector<unsigned int> list;
    uint64_t offset = 0;
    for (uint32_t t = 0; t < n_pos && offset < records_cap; ++t) {
        const uint32_t n = counts[3u * n_cols + t];
        if (n) { list.push_back(t); list.push_back(uint32_t(offset)); }
        offset += n;
    }
    const uint32_t n_list = uint32_t(list.size() / 2);
    const uint32_t n_out = uint32_t(std::min<uint64_t>(offset, records_cap));
    if (n_list) {
        std::vector<unsigned int> packed(2u * n_list);  // [positions..., bases...]
        for (uint32_t i = 0; i < n_list; ++i) { packed[i] = list[2 * i]; packed[n_list + i] = list[2 * i + 1]; }
        CUDA_TRY(cudaMemcpyAsync(e->diff_list.get(), packed.data(), sizeof(unsigned int) * packed.size(), cudaMemcpyHostToDevice, e->stream));
        p.tile_list = e->diff_list.get();
        p.n_list = n_list;
        k_desync_records<<<n_list, kDiffBlock, 0, e->stream>>>(p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(records, e->diff_records.get(), sizeof(DiffRecord) * n_out, cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    if (n_records) *n_records = n_out;
    std::memset(summary, 0, sizeof *summary);
    summary->frame = frame;
    summary->rows_first = p.rows_first;
    summary->rows_latest = p.rows_latest;
    summary->rows_differing = uint32_t(totals[0]);
    summary->existence_differing = uint32_t(totals[1]);
    summary->words_differing = totals[2];
    for (uint32_t c = 0; c < cols_cap; ++c) {
        cols[c] = bgr_desync_column{0, 0, 0, 0};
        if (c < n_cols) cols[c] = bgr_desync_column{counts[3 * c], counts[3 * c + 1], counts[3 * c + 2], 0};
    }
    return BGR_OK;
}

BGR_API int bgr_desync_diff(bgr_engine* e, int32_t frame, bgr_desync_summary* summary, bgr_desync_column* cols,
                            uint32_t cols_cap, bgr_desync_record* records, uint32_t records_cap, uint32_t* n_records,
                            int32_t* found) {
    static_assert(sizeof(DiffRecord) == sizeof(bgr_desync_record), "DiffRecord mirrors bgr_desync_record");
    if (!summary || !found || (!cols && cols_cap) || (!records && records_cap))
        return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = capture_args(e);
    if (rc != BGR_OK) return rc;
    if (n_records) *n_records = 0;
    uint32_t sf = 0, sl = 0;
    if (!e->st.ring.first(frame, &sf) || !e->st.ring.peek(frame, &sl)) { *found = 0; return BGR_OK; }
    *found = 1;
    DiffParams p{};
    p.first = e->image(sf + 1);
    p.latest = e->image(sl + 1);
    p.rows_first = e->st.slot_rows[sf];
    p.rows_latest = e->st.slot_rows[sl];
    rc = run_diff(e, p, e->tiles_for(std::max(p.rows_first, p.rows_latest)), frame, summary, cols, cols_cap, records,
                  records_cap, n_records);
    if (rc != BGR_OK) return rc;
    summary->host_state_differs = (std::memcmp(&e->st.slot_rng[sf], &e->st.slot_rng[sl], sizeof(ParticleRng)) != 0 ? 1u : 0u) |
                                  (e->st.slot_elapsed_ns[sf] != e->st.slot_elapsed_ns[sl] ? 2u : 0u);
    summary->elapsed_ns_first = e->st.slot_elapsed_ns[sf];
    summary->elapsed_ns_latest = e->st.slot_elapsed_ns[sl];
    return BGR_OK;
}

// ---- P2P desync reports (ring.hpp retains confirmed frames, frame_digest.cuh digests, desync_diff.cuh compares) ----
BGR_API int bgr_retain_confirmed(bgr_engine* e, uint32_t interval, uint32_t count) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (e->built) return fail(BGR_ERR_STATE, "bgr_retain_confirmed must be called before bgr_build");
    if (e->cfg.flags & BGR_CFG_SHARDED) return fail(BGR_ERR_UNSUPPORTED, "bgr_retain_confirmed is not supported on a sharded engine");
    if (interval == 0 || count == 0) return fail(BGR_ERR_INVALID_ARGUMENT, "bgr_retain_confirmed needs interval >= 1 and count >= 1");
    e->retain_interval = interval;
    e->retain_count = count;
    return BGR_OK;
}

BGR_API int bgr_retained_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    std::vector<int32_t> f;
    e->st.ring.retained_frames(&f);
    for (uint32_t i = 0; i < f.size() && i < cap && frames_out; ++i) frames_out[i] = f[i];
    if (n_out) *n_out = uint32_t(f.size());
    return BGR_OK;
}

static int p2p_args(bgr_engine* e) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (e->cfg.flags & BGR_CFG_SHARDED) return fail(BGR_ERR_UNSUPPORTED, "P2P desync reports are not supported on a sharded engine");
    return drain(e);
}

// the slot of `frame`: a queued snapshot first, then a retained one
static bool p2p_slot(const bgr_engine* e, int32_t frame, uint32_t* slot) {
    return e->st.ring.peek(frame, slot) || e->st.ring.retained(frame, slot);
}


// what makes two engines' images comparable (registered systems deliberately excluded); order_base too, because every
// digest word hashes the RollbackOrdered index order_base + row
static uint64_t digest_layout(const bgr_engine* e) {
    std::vector<uint32_t> v{BGR_DIGEST_BLOCK_ROWS, e->words, uint32_t(e->cols.size()), uint32_t(e->cfg.order_base),
                            uint32_t(e->cfg.order_base >> 32)};
    for (const Column& c : e->cols) {
        const bool ck = c.hash_kind != BGR_HASH_NONE;
        v.insert(v.end(), {c.elem_bytes, c.first_plane, c.words, c.absent ? 1u : 0u, ck ? 1u : 0u, ck ? c.hash_off : 0u,
                           ck ? c.hash_len : 0u});
    }
    return bgr_seahash(v.data(), v.size() * sizeof(uint32_t));
}

// k_frame_digest over the `blocks` blocks of the device image table `d_table` (images of e's registration): the block
// words ([blocks][n_columns + 1]) to `words` and the alive rows of each block to `active`.  Enqueued; the caller
// synchronises before reading them.
static int digest_launch(bgr_engine* e, const ImageEntry* d_table, uint32_t n_images, uint32_t blocks,
                         std::vector<uint64_t>* words, std::vector<unsigned int>* active) {
    const uint32_t n_cols = uint32_t(e->cols.size()), per = n_cols + 1u;
    // dynamic shared memory: 16 warps x (n_cols + 1) words, next to the kernel's static s_warp[16] (48 KB in all)
    const size_t smem = sizeof(unsigned long long) * (kTileRows / 32u) * per;
    if (smem + sizeof(uint32_t) * (kTileRows / 32u) > 48u * 1024u)
        return fail(BGR_ERR_UNSUPPORTED, "bgr_frame_digest supports at most 382 registered columns");
    if (!e->digest_cols.get()) {
        std::vector<DigestColumn> dc(n_cols);
        for (uint32_t c = 0; c < n_cols; ++c) dc[c] = DigestColumn{e->cols[c].first_plane, e->cols[c].elem_bytes, e->cols[c].absent};
        CUDA_TRY(e->digest_cols.ensure(std::max(1u, n_cols)));
        CUDA_TRY(cudaMemcpyAsync(e->digest_cols.get(), dc.data(), sizeof(DigestColumn) * n_cols, cudaMemcpyHostToDevice, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));  // `dc` goes out of scope below
    }
    CUDA_TRY(e->digest_words.ensure(size_t(per) * std::max(e->n_tiles_cap, blocks)));
    CUDA_TRY(e->digest_active.ensure(std::max(e->n_tiles_cap, blocks)));
    words->assign(size_t(blocks) * per, 0);
    active->assign(blocks, 0u);
    if (!blocks) return BGR_OK;
    DigestParams p{};
    p.images = d_table;
    p.n_images = n_images;
    p.words = e->words;
    p.n_cols = n_cols;
    p.cols = e->digest_cols.get();
    p.out = e->digest_words.get();
    p.active = e->digest_active.get();
    k_frame_digest<<<blocks, kTileRows, smem, e->stream>>>(p);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(words->data(), e->digest_words.get(), sizeof(uint64_t) * words->size(), cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaMemcpyAsync(active->data(), e->digest_active.get(), sizeof(unsigned int) * blocks, cudaMemcpyDeviceToHost, e->stream));
    return BGR_OK;
}

// k_frame_digest over the first ceil(rows / 512) tiles of `img`: the block words ([n_blocks][n_columns + 1]), their root
// and the alive rows
static int digest_image(bgr_engine* e, const uint8_t* img, uint32_t rows, std::vector<uint64_t>* words, uint64_t* root,
                        uint64_t* active_rows) {
    const uint32_t n_blocks = e->tiles_for(rows);
    const ImageEntry t{img, e->cfg.order_base, 0ull, rows, 0u};
    CUDA_TRY(e->digest_table.ensure(1));
    CUDA_TRY(cudaMemcpyAsync(e->digest_table.get(), &t, sizeof t, cudaMemcpyHostToDevice, e->stream));
    std::vector<unsigned int> active;
    int rc = digest_launch(e, e->digest_table.get(), 1, n_blocks, words, &active);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));  // also keeps `t` alive until its upload is done
    *active_rows = 0;
    for (unsigned int a : active) *active_rows += a;
    *root = bgr_seahash(words->data(), words->size() * sizeof(uint64_t));
    return BGR_OK;
}

BGR_API int bgr_frame_digest(bgr_engine* e, int32_t frame, bgr_frame_digest_header* header, uint64_t* words, uint32_t words_cap,
                             int32_t* found) {
    if (!header || !found || (!words && words_cap)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = p2p_args(e);
    if (rc != BGR_OK) return rc;
    uint32_t slot = 0;
    if (!p2p_slot(e, frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    const uint32_t rows = e->st.slot_rows[slot];
    std::vector<uint64_t> w;
    uint64_t root = 0, active = 0;
    rc = digest_image(e, e->image(slot + 1), rows, &w, &root, &active);
    if (rc != BGR_OK) return rc;
    std::memset(header, 0, sizeof *header);
    header->layout = digest_layout(e);
    header->frame = frame;
    header->rows = rows;
    header->n_blocks = e->tiles_for(rows);
    header->n_columns = uint32_t(e->cols.size());
    header->active = active;
    header->elapsed_ns = e->st.slot_elapsed_ns[slot];
    static_assert(sizeof(ParticleRng) == sizeof(header->rng), "ParticleRng is four u64 words");
    std::memcpy(header->rng, &e->st.slot_rng[slot], sizeof header->rng);
    header->root = root;
    if (words) std::memcpy(words, w.data(), sizeof(uint64_t) * std::min<size_t>(words_cap, w.size()));
    return BGR_OK;
}

BGR_API int bgr_digest_mismatch(const bgr_frame_digest_header* lh, const uint64_t* lw, const bgr_frame_digest_header* rh,
                                const uint64_t* rw, uint32_t* blocks_out, uint32_t cap, uint32_t* n_out,
                                uint32_t* host_state_differs) {
    if (!lh || !rh || !n_out || (!blocks_out && cap) || (!lw && lh->n_blocks) || (!rw && rh->n_blocks))
        return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (lh->layout != rh->layout)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the digests come from engines with different registrations (layout differs)");
    if (lh->frame != rh->frame)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the digests are of different frames (" + std::to_string(lh->frame) + " and " +
                                                  std::to_string(rh->frame) + ")");
    if (lh->n_columns != rh->n_columns)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the digests have different column counts (" + std::to_string(lh->n_columns) +
                                                  " and " + std::to_string(rh->n_columns) + ")");
    const size_t per = size_t(lh->n_columns) + 1u;
    const uint32_t common = std::min(lh->n_blocks, rh->n_blocks), most = std::max(lh->n_blocks, rh->n_blocks);
    uint32_t n = 0;
    for (uint32_t b = 0; b < most; ++b) {
        const bool differs = b >= common || std::memcmp(lw + b * per, rw + b * per, per * sizeof(uint64_t)) != 0;
        if (!differs) continue;
        if (n < cap) blocks_out[n] = b;
        ++n;
    }
    *n_out = n;
    if (host_state_differs)
        *host_state_differs = (std::memcmp(lh->rng, rh->rng, sizeof lh->rng) != 0 ? 1u : 0u) |
                              (lh->elapsed_ns != rh->elapsed_ns ? 2u : 0u);
    return BGR_OK;
}

static constexpr size_t kBlobBlockHeader = 8;  // u32 block index + u32 zero ahead of each tile

BGR_API int bgr_frame_export(bgr_engine* e, int32_t frame, const uint32_t* blocks, uint32_t n_blocks, void* dst,
                             size_t dst_cap, size_t* bytes, int32_t* found) {
    if (!bytes || !found || (!blocks && n_blocks)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = p2p_args(e);
    if (rc != BGR_OK) return rc;
    uint32_t slot = 0;
    if (!p2p_slot(e, frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    const uint32_t rows = e->st.slot_rows[slot], total = e->tiles_for(rows);
    for (uint32_t i = 0; i < n_blocks; ++i) {
        if (blocks[i] >= total)
            return fail(BGR_ERR_INVALID_ARGUMENT, "block " + std::to_string(blocks[i]) + " is past the frame's " +
                                                      std::to_string(total) + " blocks");
        if (i && blocks[i] <= blocks[i - 1]) return fail(BGR_ERR_INVALID_ARGUMENT, "the block list must be ascending without duplicates");
    }
    const size_t tb = e->tile_bytes;
    const size_t need = sizeof(bgr_frame_blob_header) + size_t(n_blocks) * (kBlobBlockHeader + tb);
    *bytes = need;
    if (!dst) return BGR_OK;
    if (dst_cap < need) return fail(BGR_ERR_CAPACITY, "the export needs " + std::to_string(need) + " bytes");
    uint8_t* out = static_cast<uint8_t*>(dst);
    bgr_frame_blob_header h{};
    h.magic = BGR_FRAME_BLOB_MAGIC;
    h.version = BGR_FRAME_BLOB_VERSION;
    h.layout = digest_layout(e);
    h.frame = frame;
    h.rows = rows;
    h.words = e->words;
    h.n_blocks = total;
    h.n_exported = n_blocks;
    h.elapsed_ns = e->st.slot_elapsed_ns[slot];
    std::memcpy(h.rng, &e->st.slot_rng[slot], sizeof h.rng);
    std::memcpy(out, &h, sizeof h);
    for (uint32_t i = 0; i < n_blocks; ++i) {
        uint8_t* rec = out + sizeof h + size_t(i) * (kBlobBlockHeader + tb);
        const uint32_t idx[2] = {blocks[i], 0u};
        std::memcpy(rec, idx, sizeof idx);
        CUDA_TRY(cudaMemcpyAsync(rec + kBlobBlockHeader, e->image(slot + 1) + size_t(blocks[i]) * tb, tb, cudaMemcpyDeviceToHost, e->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    // rows >= rows of the last block hold whatever an older frame left there: zero their words and mask bytes
    if (n_blocks && blocks[n_blocks - 1] == total - 1 && rows % kTileRows) {
        uint8_t* tile = out + sizeof h + size_t(n_blocks - 1) * (kBlobBlockHeader + tb) + kBlobBlockHeader;
        const uint32_t r0 = rows % kTileRows;
        for (uint32_t w = 0; w < e->words; ++w) std::memset(tile + size_t(w) * kPlaneBytes + r0 * 4u, 0, (kTileRows - r0) * 4u);
        std::memset(tile + size_t(e->words) * kPlaneBytes + r0, 0, kTileRows - r0);
    }
    return BGR_OK;
}

BGR_API int bgr_desync_diff_remote(bgr_engine* e, int32_t frame, const void* blob, size_t bytes,
                                   bgr_desync_summary* summary, bgr_desync_column* cols, uint32_t cols_cap,
                                   bgr_desync_record* records, uint32_t records_cap, uint32_t* n_records, int32_t* found) {
    if (!summary || !found || !blob || (!cols && cols_cap) || (!records && records_cap))
        return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = p2p_args(e);
    if (rc != BGR_OK) return rc;
    if (n_records) *n_records = 0;
    // the blob comes from another machine: check every field before using it
    const uint8_t* in = static_cast<const uint8_t*>(blob);
    bgr_frame_blob_header h;
    if (bytes < sizeof h) return fail(BGR_ERR_INVALID_ARGUMENT, "blob truncated: shorter than its header");
    std::memcpy(&h, in, sizeof h);
    if (h.magic != BGR_FRAME_BLOB_MAGIC) return fail(BGR_ERR_INVALID_ARGUMENT, "not a frame export blob (bad magic)");
    if (h.version != BGR_FRAME_BLOB_VERSION)
        return fail(BGR_ERR_INVALID_ARGUMENT, "unsupported blob format version " + std::to_string(h.version));
    if (h.layout != digest_layout(e) || h.words != e->words)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the blob comes from an engine with a different registration (layout differs)");
    if (h.frame != frame)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the blob holds frame " + std::to_string(h.frame) + ", not " + std::to_string(frame));
    if (h.reserved != 0) return fail(BGR_ERR_INVALID_ARGUMENT, "blob header: reserved field is not zero");
    if (h.n_blocks != e->tiles_for(h.rows) || h.n_blocks > e->n_tiles_cap || h.n_exported > h.n_blocks)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the blob's row and block counts are inconsistent or exceed this engine's capacity");
    const size_t tb = e->tile_bytes, rec = kBlobBlockHeader + tb;
    if (bytes != sizeof h + size_t(h.n_exported) * rec)
        return fail(BGR_ERR_INVALID_ARGUMENT, "blob length " + std::to_string(bytes) + " does not match its " +
                                                  std::to_string(h.n_exported) + " blocks (truncated or overlong)");
    std::vector<unsigned int> visit(h.n_exported);
    for (uint32_t i = 0; i < h.n_exported; ++i) {
        uint32_t idx[2];
        std::memcpy(idx, in + sizeof h + size_t(i) * rec, sizeof idx);
        if (idx[1] != 0) return fail(BGR_ERR_INVALID_ARGUMENT, "blob block " + std::to_string(i) + ": reserved word is not zero");
        if (idx[0] >= h.n_blocks)
            return fail(BGR_ERR_INVALID_ARGUMENT, "blob block index " + std::to_string(idx[0]) + " >= its " +
                                                      std::to_string(h.n_blocks) + " blocks");
        if (i && idx[0] <= visit[i - 1]) return fail(BGR_ERR_INVALID_ARGUMENT, "blob block list is unsorted or has duplicates");
        visit[i] = idx[0];
    }
    uint32_t slot = 0;
    if (!p2p_slot(e, frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    // The local blocks at or past the peer's block count exist only here: every row of them is >= h.rows, so the peer
    // has none of them and the blob cannot carry them.  They are visited after the exported blocks (positions
    // n_exported.. of the list, whose staging address is never read: diff_mask_tile answers 0 for a row >= rows_latest
    // before loading, and words are only loaded for rows that exist on both sides).  Ascending, at most n_tiles_cap.
    for (uint32_t b = h.n_blocks; b < e->tiles_for(e->st.slot_rows[slot]); ++b) visit.push_back(b);
    const uint32_t n_visit = uint32_t(visit.size());
    CUDA_TRY(e->remote_visit.ensure(e->n_tiles_cap));
    CUDA_TRY(e->remote.ensure(tb * h.n_exported));  // staging for the peer's tiles
    for (uint32_t i = 0; i < h.n_exported; ++i)
        CUDA_TRY(cudaMemcpyAsync(e->remote.get() + size_t(i) * tb, in + sizeof h + size_t(i) * rec + kBlobBlockHeader, tb,
                                 cudaMemcpyHostToDevice, e->stream));
    if (n_visit)
        CUDA_TRY(cudaMemcpyAsync(e->remote_visit.get(), visit.data(), sizeof(unsigned int) * n_visit, cudaMemcpyHostToDevice, e->stream));
    DiffParams p{};
    p.first = e->image(slot + 1);
    p.latest = e->remote.get();  // null while nothing was ever exported to this engine: then no position reads it
    p.visit = e->remote_visit.get();
    p.rows_first = e->st.slot_rows[slot];
    p.rows_latest = h.rows;
    rc = run_diff(e, p, n_visit, frame, summary, cols, cols_cap, records, records_cap, n_records);
    if (rc != BGR_OK) return rc;
    summary->host_state_differs = (std::memcmp(&e->st.slot_rng[slot], h.rng, sizeof h.rng) != 0 ? 1u : 0u) |
                                  (e->st.slot_elapsed_ns[slot] != h.elapsed_ns ? 2u : 0u);
    summary->elapsed_ns_first = e->st.slot_elapsed_ns[slot];
    summary->elapsed_ns_latest = h.elapsed_ns;
    return BGR_OK;
}

// ---- world checkpoints (checkpoint.cuh encodes and decodes, k_frame_digest verifies a decoded world) ----
static int checkpoint_args(bgr_engine* e) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (e->cfg.flags & BGR_CFG_SHARDED) return fail(BGR_ERR_UNSUPPORTED, "world checkpoints are not supported on a sharded engine");
    return BGR_OK;
}

// the absent bit of the column each word plane belongs to (0: not optional)
static std::vector<uint32_t> plane_absent(const bgr_engine* e) {
    std::vector<uint32_t> a(std::max(1u, e->words), 0u);
    for (const Column& c : e->cols)
        for (uint32_t w = 0; w < c.words; ++w) a[c.first_plane + w] = c.absent;
    return a;
}

// the bits of each plane's word that lie past its column's element bytes (the last word of a sub-word element)
static std::vector<uint32_t> plane_pad(const bgr_engine* e) {
    std::vector<uint32_t> a(std::max(1u, e->words), 0u);
    for (const Column& c : e->cols)
        if (c.elem_bytes % 4u) a[c.first_plane + c.words - 1u] = ~0u << (8u * (c.elem_bytes % 4u));
    return a;
}

// ---- the image-table encoder: the checkpoints of many images of one registration in four launches ----
// k_frame_digest, k_ckpt_measure and k_ckpt_scan run once over every block of every image (one scan: an image's offsets
// are differences from its first block's), then, with the blob sizes known on the host, k_ckpt_pack writes every payload
// where its blob lies in host memory relative to the others (runs of blobs that follow each other there, 8-byte aligned,
// are contiguous on the device too), and all of them come back with one copy.  Headers and offsets are written on the
// host.

// One image to encode.  The caller sets img, order_base and the header (checkpoint_header); encode_measure adds
// active, digest_root, payload_bytes and the offsets; encode_pack writes the blob to dst.  A checkpoint delta also sets
// base and base_rows (the image it is coded against; h.n_blocks then covers both frames' rows) and `delta`, the header
// encode_pack writes in place of h, which the caller completes from h after encode_measure.
struct EncodeImage {
    const uint8_t* img = nullptr;
    unsigned long long order_base = 0;
    bgr_checkpoint_header h{};
    std::vector<uint64_t> offsets;
    uint8_t* dst = nullptr;
    const uint8_t* base = nullptr;
    uint32_t base_rows = 0;
    const bgr_checkpoint_delta_header* delta = nullptr;
};

static size_t blob_prefix(const EncodeImage& x) {
    return x.delta ? checkpoint_delta_prefix(x.h.n_blocks) : checkpoint_prefix(x.h.n_blocks);
}
static size_t blob_bytes(const EncodeImage& x) { return blob_prefix(x) + x.h.payload_bytes; }
static size_t align8(size_t v) { return (v + 7u) & ~size_t(7); }
static size_t align16(size_t v) { return (v + 15u) & ~size_t(15); }

// The header of a checkpoint of e's frame `frame` with `rows` rows (active, digest_root and payload_bytes: encode_measure)
static bgr_checkpoint_header checkpoint_header(const bgr_engine* e, int32_t frame, uint32_t rows, uint64_t elapsed_ns,
                                               const ParticleRng& rng) {
    bgr_checkpoint_header h{};
    h.magic = BGR_CHECKPOINT_MAGIC;
    h.version = BGR_CHECKPOINT_VERSION;
    h.layout = digest_layout(e);
    h.frame = frame;
    h.rows = rows;
    h.words = e->words;
    h.n_blocks = e->tiles_for(rows);
    h.n_columns = uint32_t(e->cols.size());
    h.fps = e->cfg.fps;
    h.elapsed_ns = elapsed_ns;
    static_assert(sizeof(ParticleRng) == sizeof(h.rng), "ParticleRng is four u64 words");
    std::memcpy(h.rng, &rng, sizeof h.rng);
    return h;
}

// The images of one encoding and the device memory it uses (allocated by the first call that needs it, freed with the
// encoder).  `e` gives the stream, the word planes and the columns, which every image's engine shares.  `delta`: every
// image is a checkpoint delta (k_ckpt_measure_delta / k_ckpt_pack_delta over the parallel array of bases).
struct ImageEncoder {
    bgr_engine* e = nullptr;
    bool delta = false;
    std::vector<EncodeImage> im;
    std::vector<ImageEntry> table;
    uint32_t blocks = 0;
    DeviceBuffer<ImageEntry> d_table;
    std::vector<CkptBase> bases;  // delta: [images] each image's base
    DeviceBuffer<CkptBase> d_base;
    DeviceBuffer<uint32_t> d_absent, d_out;
    DeviceBuffer<uint8_t> d_kinds;
    DeviceBuffer<unsigned int> d_lens;
    DeviceBuffer<unsigned long long> d_offsets;
    std::vector<unsigned long long> offsets;  // [blocks + 1] over every image
    std::vector<uint64_t> digest;
    std::vector<unsigned int> active;
    CkptParams p{};
};

// digest, measure and scan: every image's digest root, active rows, offsets and payload size.  Synchronous.
static int encode_measure(ImageEncoder& x) {
    bgr_engine* e = x.e;
    const uint32_t n = uint32_t(x.im.size()), per = uint32_t(e->cols.size()) + 1u;
    x.table.resize(n);
    x.blocks = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const EncodeImage& m = x.im[i];
        x.table[i] = ImageEntry{m.img, m.order_base, 0ull, m.h.rows, x.blocks};
        x.blocks += m.h.n_blocks;
    }
    x.offsets.assign(size_t(x.blocks) + 1u, 0ull);
    if (x.blocks) {
        const std::vector<uint32_t> absent = plane_absent(e);
        CUDA_TRY(x.d_table.ensure(n));
        CUDA_TRY(x.d_absent.ensure(absent.size()));
        CUDA_TRY(x.d_kinds.ensure(size_t(x.blocks) * (e->words + 1u)));
        CUDA_TRY(x.d_lens.ensure(x.blocks));
        CUDA_TRY(x.d_offsets.ensure(size_t(x.blocks) + 1u));
        CUDA_TRY(cudaMemcpyAsync(x.d_table.get(), x.table.data(), sizeof(ImageEntry) * n, cudaMemcpyHostToDevice, e->stream));
        CUDA_TRY(cudaMemcpyAsync(x.d_absent.get(), absent.data(), sizeof(uint32_t) * absent.size(), cudaMemcpyHostToDevice, e->stream));
        int rc = digest_launch(e, x.d_table.get(), n, x.blocks, &x.digest, &x.active);
        if (rc != BGR_OK) return rc;
        x.p = CkptParams{};
        x.p.images = x.d_table.get();
        x.p.n_images = n;
        x.p.words = e->words;
        x.p.plane_absent = x.d_absent.get();
        x.p.kinds = x.d_kinds.get();
        x.p.lens = x.d_lens.get();
        x.p.offsets = x.d_offsets.get();
        if (x.delta) {
            x.bases.resize(n);
            for (uint32_t i = 0; i < n; ++i) x.bases[i] = CkptBase{x.im[i].base, x.im[i].base_rows, 0u};
            CUDA_TRY(x.d_base.ensure(n));
            CUDA_TRY(cudaMemcpyAsync(x.d_base.get(), x.bases.data(), sizeof(CkptBase) * n, cudaMemcpyHostToDevice, e->stream));
            x.p.base = x.d_base.get();
            k_ckpt_measure_delta<<<x.blocks, kTileRows, 0, e->stream>>>(x.p);
        } else {
            k_ckpt_measure<<<x.blocks, kTileRows, 0, e->stream>>>(x.p);
        }
        k_ckpt_scan<<<1, kCkptScanBlock, 0, e->stream>>>(x.d_lens.get(), x.blocks, x.d_offsets.get());
        e->launches += 2;
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaMemcpyAsync(x.offsets.data(), x.d_offsets.get(), sizeof(uint64_t) * x.offsets.size(), cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));  // also keeps `absent` and the table alive until their uploads are done
    } else {
        x.digest.clear();
        x.active.clear();
    }
    for (EncodeImage& m : x.im) {
        const ImageEntry& t = x.table[&m - x.im.data()];
        const size_t nb = m.h.n_blocks;
        m.h.active = 0;
        for (size_t b = 0; b < nb; ++b) m.h.active += x.active[t.first_block + b];
        // over the image's own blocks (a delta's blocks past its rows digest to zero words and are not part of its root)
        const size_t own = e->tiles_for(m.h.rows);
        m.h.digest_root = bgr_seahash(own ? &x.digest[size_t(t.first_block) * per] : nullptr, own * per * sizeof(uint64_t));
        m.offsets.resize(nb + 1u);
        for (size_t b = 0; b <= nb; ++b) m.offsets[b] = x.offsets[t.first_block + b] - x.offsets[t.first_block];
        m.h.payload_bytes = m.offsets[nb];
    }
    return BGR_OK;
}

// pack: every image's blob to its dst (after encode_measure).  Synchronous.
static int encode_pack(ImageEncoder& x) {
    bgr_engine* e = x.e;
    const size_t n = x.im.size();
    // runs of blobs that follow each other in host memory: [first image, end), the device bytes before the run
    struct Run { size_t first, end, base; };
    std::vector<Run> runs;
    size_t out_bytes = 0;
    auto payload_at = [&](size_t i) { return x.im[i].dst + blob_prefix(x.im[i]); };
    for (size_t i = 0; i < n; ++i) {
        if (i == 0 || x.im[i].dst != x.im[i - 1].dst + align8(blob_bytes(x.im[i - 1]))) {
            if (!runs.empty()) out_bytes += size_t(x.im[i - 1].dst + blob_bytes(x.im[i - 1]) - payload_at(runs.back().first));
            runs.push_back(Run{i, i, out_bytes});
        }
        runs.back().end = i + 1;
        x.table[i].out_off = runs.back().base + size_t(payload_at(i) - payload_at(runs.back().first));
    }
    if (n) out_bytes += size_t(x.im[n - 1].dst + blob_bytes(x.im[n - 1]) - payload_at(runs.back().first));
    if (x.blocks) {
        CUDA_TRY(x.d_out.ensure(std::max<size_t>(1, out_bytes / 4u)));
        CUDA_TRY(cudaMemcpyAsync(x.d_table.get(), x.table.data(), sizeof(ImageEntry) * n, cudaMemcpyHostToDevice, e->stream));
        x.p.payload = x.d_out.get();
        if (x.delta) k_ckpt_pack_delta<<<x.blocks, kTileRows, 0, e->stream>>>(x.p);
        else k_ckpt_pack<<<x.blocks, kTileRows, 0, e->stream>>>(x.p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        // one copy: straight into the caller's memory for one run, else into host staging that is then scattered to the
        // runs (one small copy per world of a batch cost more device time than the launch's replay kernel)
        const uint8_t* d_out = reinterpret_cast<const uint8_t*>(x.d_out.get());
        auto run_len = [&](const Run& r) { return size_t(x.im[r.end - 1].dst + blob_bytes(x.im[r.end - 1]) - payload_at(r.first)); };
        if (runs.size() == 1) {
            if (out_bytes) CUDA_TRY(cudaMemcpyAsync(payload_at(0), d_out, out_bytes, cudaMemcpyDeviceToHost, e->stream));
            CUDA_TRY(cudaStreamSynchronize(e->stream));
        } else {
            std::vector<uint8_t> stage(out_bytes);
            CUDA_TRY(cudaMemcpyAsync(stage.data(), d_out, out_bytes, cudaMemcpyDeviceToHost, e->stream));
            CUDA_TRY(cudaStreamSynchronize(e->stream));
            for (const Run& r : runs) std::memcpy(payload_at(r.first), stage.data() + r.base, run_len(r));
        }
    }
    for (size_t i = 0; i < n; ++i) {  // the headers, the offsets and the zero padding between blobs of a run
        EncodeImage& m = x.im[i];
        const size_t head = m.delta ? sizeof *m.delta : sizeof m.h;
        std::memcpy(m.dst, m.delta ? static_cast<const void*>(m.delta) : static_cast<const void*>(&m.h), head);
        std::memcpy(m.dst + head, m.offsets.data(), sizeof(uint64_t) * m.offsets.size());
        if (i + 1 < n && x.im[i + 1].dst == m.dst + align8(blob_bytes(m)))
            std::memset(m.dst + blob_bytes(m), 0, align8(blob_bytes(m)) - blob_bytes(m));
    }
    return BGR_OK;
}

BGR_API int bgr_checkpoint_save(bgr_engine* e, int32_t frame, void* dst, size_t dst_cap, size_t* bytes, int32_t* found) {
    if (!bytes || !found) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = checkpoint_args(e);
    if (rc == BGR_OK) rc = drain(e);
    if (rc != BGR_OK) return rc;
    uint32_t slot = 0;
    if (!p2p_slot(e, frame, &slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    const uint32_t rows = e->st.slot_rows[slot], n_blocks = e->tiles_for(rows);
    if (!dst) {
        *bytes = checkpoint_prefix(n_blocks) + size_t(n_blocks) * ckpt_max_block_words(e->words) * 4u;
        return BGR_OK;
    }
    ImageEncoder x;
    x.e = e;
    x.im.resize(1);
    EncodeImage& m = x.im[0];
    m.img = e->image(slot + 1);
    m.order_base = e->cfg.order_base;
    m.h = checkpoint_header(e, frame, rows, e->st.slot_elapsed_ns[slot], e->st.slot_rng[slot]);
    rc = encode_measure(x);
    if (rc != BGR_OK) return rc;
    const size_t need = blob_bytes(m);
    *bytes = need;
    if (dst_cap < need) return fail(BGR_ERR_CAPACITY, "the checkpoint needs " + std::to_string(need) + " bytes");
    m.dst = static_cast<uint8_t*>(dst);
    return encode_pack(x);
}

// A delta of `frame` against `base_frame`: the encoder's delta instances over the target's slot image, each block coded
// against the base slot image's (the blocks past one frame's rows against zeros), and the base's root from its own
// frame digest.
BGR_API int bgr_checkpoint_save_delta(bgr_engine* e, int32_t frame, int32_t base_frame, void* dst, size_t dst_cap,
                                      size_t* bytes, int32_t* found) {
    if (!bytes || !found) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    int rc = checkpoint_args(e);
    if (rc == BGR_OK) rc = drain(e);
    if (rc != BGR_OK) return rc;
    uint32_t slot = 0, base_slot = 0;
    if (!p2p_slot(e, frame, &slot) || !p2p_slot(e, base_frame, &base_slot)) { *found = 0; return BGR_OK; }
    *found = 1;
    const uint32_t rows = e->st.slot_rows[slot], base_rows = e->st.slot_rows[base_slot];
    const uint32_t n_blocks = e->tiles_for(std::max(rows, base_rows));
    if (!dst) {
        *bytes = checkpoint_delta_prefix(n_blocks) + size_t(n_blocks) * ckpt_max_block_words(e->words) * 4u;
        return BGR_OK;
    }
    std::vector<uint64_t> base_words;
    uint64_t base_root = 0, base_active = 0;
    rc = digest_image(e, e->image(base_slot + 1), base_rows, &base_words, &base_root, &base_active);
    if (rc != BGR_OK) return rc;
    bgr_checkpoint_delta_header dh{};
    ImageEncoder x;
    x.e = e;
    x.delta = true;
    x.im.resize(1);
    EncodeImage& m = x.im[0];
    m.img = e->image(slot + 1);
    m.order_base = e->cfg.order_base;
    m.h = checkpoint_header(e, frame, rows, e->st.slot_elapsed_ns[slot], e->st.slot_rng[slot]);
    m.h.n_blocks = n_blocks;
    m.base = e->image(base_slot + 1);
    m.base_rows = base_rows;
    m.delta = &dh;
    rc = encode_measure(x);
    if (rc != BGR_OK) return rc;
    dh.magic = BGR_CHECKPOINT_DELTA_MAGIC;
    dh.version = BGR_CHECKPOINT_DELTA_VERSION;
    dh.layout = m.h.layout;
    dh.frame = frame;
    dh.rows = rows;
    dh.base_frame = base_frame;
    dh.base_rows = base_rows;
    dh.words = m.h.words;
    dh.n_blocks = n_blocks;
    dh.n_columns = m.h.n_columns;
    dh.fps = m.h.fps;
    dh.active = m.h.active;
    dh.elapsed_ns = m.h.elapsed_ns;
    std::memcpy(dh.rng, m.h.rng, sizeof dh.rng);
    dh.digest_root = m.h.digest_root;
    dh.base_root = base_root;
    dh.payload_bytes = m.h.payload_bytes;
    const size_t need = blob_bytes(m);
    *bytes = need;
    if (dst_cap < need) return fail(BGR_ERR_CAPACITY, "the checkpoint delta needs " + std::to_string(need) + " bytes");
    m.dst = static_cast<uint8_t*>(dst);
    return encode_pack(x);
}

// ---- restore: the blobs checked on the host, decoded and verified in one pass, then committed in one launch ----
// bgr_checkpoint_restore is the one-blob case of bgr_batch_checkpoint_restore: restore_check, restore_decode and
// restore_commit serve both.

// One blob to restore into engine e, checked on the host by restore_check
struct RestoreBlob {
    bgr_engine* e = nullptr;
    const uint8_t* payload = nullptr;  // h.payload_bytes bytes inside the caller's blob
    bgr_checkpoint_header h{};
    std::vector<uint64_t> offsets;     // [n_blocks + 1]
    uint32_t slot = 0;                 // restore_commit: the ring slot that holds the restored frame
};

// The device memory of one restore (every blob's scratch image, the payloads, the tables), freed with it
struct RestorePass {
    std::vector<ImageEntry> table;  // one entry per blob, img = its scratch image
    uint32_t blocks = 0;
    DeviceBuffer<uint8_t> scratch, meta, payload;
    size_t dst_off = 0;             // k_ckpt_commit's destinations ([blobs][2] pointers) in `meta`, written by the commit
};

static CkptTarget ckpt_target(const bgr_engine* e) {
    return CkptTarget{digest_layout(e), e->words, uint32_t(e->cols.size()), e->cfg.fps, e->ceiling, e->growable()};
}

// The engine's state checks and the blob's host checks (checkpoint_check.hpp); nothing runs
static int restore_check(bgr_engine* e, const void* blob, size_t bytes, RestoreBlob* r) {
    int rc = checkpoint_args(e);
    if (rc != BGR_OK) return rc;
    if (!blob) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    if (!e->pending.empty()) return fail(BGR_ERR_STATE, "collect every submitted request vector first");
    if (e->st.ring.depth() == 0 || e->n_slots() == 0)
        return fail(BGR_ERR_STATE, "the snapshot ring has depth 0: it cannot hold the restored frame");
    std::string err;
    rc = checkpoint_check(ckpt_target(e), blob, bytes, &r->h, &r->offsets, &err);
    if (rc != BGR_OK) return fail(rc, err);
    r->e = e;
    r->payload = static_cast<const uint8_t*>(blob) + checkpoint_prefix(r->h.n_blocks);
    return BGR_OK;
}

// Decodes every blob of `r` (host-checked, into engines of one registration on one stream) into its own scratch image
// and verifies each with the frame digest, with a fixed number of launches and copies whatever the number of blobs: one
// upload of the payloads (gathered in `stage`, page-locked, when there are several; one blob is uploaded from the
// caller's memory), one of the tables and offsets, k_ckpt_unpack and k_frame_digest over every block of every blob, one
// synchronisation.  Nothing is committed.  A refusal sets *bad to the lowest index of `r` that failed.
static int restore_decode(std::vector<RestoreBlob>& r, RestorePass& x, MappedHostBuffer<uint8_t>* stage, size_t* bad) {
    bgr_engine* e = r[0].e;
    const size_t n = r.size();
    const uint32_t per = uint32_t(e->cols.size()) + 1u;
    size_t payload_bytes = 0;
    x.table.resize(n);
    x.blocks = 0;
    for (size_t i = 0; i < n; ++i) {  // scratch images and payloads follow each other in list order
        x.table[i] = ImageEntry{nullptr, r[i].e->cfg.order_base, payload_bytes, r[i].h.rows, x.blocks};
        x.blocks += r[i].h.n_blocks;
        payload_bytes += r[i].h.payload_bytes;
    }
    std::vector<uint64_t> digest;
    std::vector<unsigned int> active, err(n, 0xFFFFFFFFu);
    if (x.blocks) {
        const size_t smem = sizeof(uint32_t) * (e->words + 1u);
        if (smem + sizeof(uint32_t) * (kCkptMaskWords + 1u) > 48u * 1024u)
            return fail(BGR_ERR_UNSUPPORTED, "bgr_checkpoint_restore supports at most 12000 word planes");
        const std::vector<uint32_t> absent = plane_absent(e), pad = plane_pad(e);
        // the tables in one upload: image table, the offsets rebased onto the concatenated payloads, error words, planes
        const size_t o_off = align16(sizeof(ImageEntry) * n), o_err = align16(o_off + sizeof(uint64_t) * (x.blocks + 1u));
        const size_t o_absent = align16(o_err + sizeof(unsigned int) * n), o_pad = align16(o_absent + sizeof(uint32_t) * absent.size());
        x.dst_off = align16(o_pad + sizeof(uint32_t) * pad.size());
        const size_t meta_bytes = x.dst_off + sizeof(uint8_t*) * 2u * n;  // every allocation happens before the commit
        CUDA_TRY(x.scratch.ensure(size_t(x.blocks) * e->tile_bytes));
        CUDA_TRY(x.meta.ensure(meta_bytes));
        CUDA_TRY(x.payload.ensure(std::max<size_t>(4, payload_bytes)));
        for (size_t i = 0; i < n; ++i) x.table[i].img = x.scratch.get() + size_t(x.table[i].first_block) * e->tile_bytes;
        std::vector<uint8_t> meta(meta_bytes);
        std::memcpy(meta.data(), x.table.data(), sizeof(ImageEntry) * n);
        uint64_t* off = reinterpret_cast<uint64_t*>(meta.data() + o_off);
        for (size_t i = 0; i < n; ++i)
            for (uint32_t k = 0; k < r[i].h.n_blocks; ++k) off[x.table[i].first_block + k] = x.table[i].out_off + r[i].offsets[k];
        off[x.blocks] = payload_bytes;
        std::memcpy(meta.data() + o_err, err.data(), sizeof(unsigned int) * n);
        std::memcpy(meta.data() + o_absent, absent.data(), sizeof(uint32_t) * absent.size());
        std::memcpy(meta.data() + o_pad, pad.data(), sizeof(uint32_t) * pad.size());
        const uint8_t* src = r[0].payload;
        if (n > 1) {
            CUDA_TRY(stage->ensure(payload_bytes));
            for (size_t i = 0; i < n; ++i) std::memcpy(stage->get() + x.table[i].out_off, r[i].payload, r[i].h.payload_bytes);
            src = stage->get();
        }
        CUDA_TRY(cudaMemcpyAsync(x.payload.get(), src, payload_bytes, cudaMemcpyHostToDevice, e->stream));
        CUDA_TRY(cudaMemcpyAsync(x.meta.get(), meta.data(), meta_bytes, cudaMemcpyHostToDevice, e->stream));
        uint8_t* d = x.meta.get();
        CkptParams p{};
        p.images = reinterpret_cast<const ImageEntry*>(d);
        p.n_images = uint32_t(n);
        p.words = e->words;
        p.plane_absent = reinterpret_cast<const uint32_t*>(d + o_absent);
        p.plane_pad = reinterpret_cast<const uint32_t*>(d + o_pad);
        p.mask_bits = 1u;
        for (const Column& c : e->cols) p.mask_bits |= c.absent;
        p.offsets = reinterpret_cast<const unsigned long long*>(d + o_off);
        p.payload = reinterpret_cast<uint32_t*>(x.payload.get());
        p.err = reinterpret_cast<unsigned int*>(d + o_err);
        k_ckpt_unpack<<<x.blocks, kTileRows, smem, e->stream>>>(p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        int rc = digest_launch(e, p.images, uint32_t(n), x.blocks, &digest, &active);
        if (rc != BGR_OK) return rc;
        CUDA_TRY(cudaMemcpyAsync(err.data(), p.err, sizeof(unsigned int) * n, cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));  // `meta` goes out of scope, the staging is reused by the next call
    }
    for (size_t i = 0; i < n; ++i) {
        *bad = i;
        if (err[i] != 0xFFFFFFFFu)
            return fail(BGR_ERR_INVALID_ARGUMENT, "checkpoint block " + std::to_string(err[i]) +
                                                      ": a bad kind byte or padding, its kinds and bitmaps imply another length than its "
                                                      "offsets, a row's mask byte has a bit this registration does not use, or a word has "
                                                      "bits past its column's element bytes");
        const size_t nb = r[i].h.n_blocks, b0 = x.table[i].first_block;
        uint64_t rows_alive = 0;
        for (size_t k = 0; k < nb; ++k) rows_alive += active[b0 + k];
        const uint64_t root = bgr_seahash(nb ? &digest[b0 * per] : nullptr, nb * per * sizeof(uint64_t));
        if (root != r[i].h.digest_root || rows_alive != r[i].h.active)
            return fail(BGR_ERR_INVALID_ARGUMENT, "the decoded world's digest or active row count differs from the checkpoint header (corrupt payload)");
    }
    return BGR_OK;
}

// Commits every verified blob of `r` (after restore_decode): growable engines grow to the blob's rows (a failure sets
// *bad to that blob's index, before any world changed), each ring restarts at the blob's frame, one k_ckpt_commit launch
// copies every scratch image to its engine's image 0 and restored slot, then each engine's host state becomes the
// blob's.  Allocates nothing once a world has changed.  Synchronous: the scratch images are freed after it.
static int restore_commit(std::vector<RestoreBlob>& r, RestorePass& x, size_t* bad) {
    bgr_engine* e0 = r[0].e;
    for (size_t i = 0; i < r.size(); ++i)
        if (r[i].e->growable()) {
            *bad = i;
            int rc = grow_to(r[i].e, r[i].h.rows);
            if (rc != BGR_OK) return rc;
        }
    *bad = r.size();
    // image 0 and one slot hold the world, which the ring queues alone
    std::vector<uint8_t*> dst(2u * r.size());
    for (size_t i = 0; i < r.size(); ++i) {
        bgr_engine* e = r[i].e;
        e->deferred = DeferredLive{};  // image 0 is overwritten: nothing to materialise
        r[i].slot = e->st.ring.restart(r[i].h.frame);
        dst[2u * i] = e->image(0);
        dst[2u * i + 1u] = e->image(r[i].slot + 1);
    }
    if (x.blocks) {
        uint8_t** d_dst = reinterpret_cast<uint8_t**>(x.meta.get() + x.dst_off);
        CUDA_TRY(cudaMemcpyAsync(d_dst, dst.data(), sizeof(uint8_t*) * dst.size(), cudaMemcpyHostToDevice, e0->stream));
        k_ckpt_commit<<<x.blocks, kTileRows, 0, e0->stream>>>(reinterpret_cast<const ImageEntry*>(x.meta.get()), uint32_t(r.size()),
                                                              d_dst, uint32_t(e0->tile_bytes));
        e0->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    for (RestoreBlob& b : r) {
        bgr_engine* e = b.e;
        const bgr_checkpoint_header& h = b.h;
        const uint32_t slot = b.slot;
        int rc = clear_stamps(e, 0);
        if (rc == BGR_OK) rc = clear_stamps(e, slot + 1);
        if (rc != BGR_OK) return rc;
        e->tiledep_chain = false;
        HostState& s = e->st;
        ParticleRng rng;
        std::memcpy(&rng, h.rng, sizeof rng);
        s.frame_count = h.frame;
        s.elapsed_ns = h.elapsed_ns;
        s.n_rows = h.rows;
        s.rng = rng;
        s.slot_rows[slot] = h.rows;
        s.slot_elapsed_ns[slot] = h.elapsed_ns;
        s.slot_rng[slot] = rng;
        s.cids.live = s.cids.slot[slot] = s.cids.fresh(h.rows);
        s.live_passive_ver = ++s.ver_counter;  // image 0 holds new content; the restored slot holds the same
        s.slot_passive_ver[slot] = s.live_passive_ver;
    }
    CUDA_TRY(cudaStreamSynchronize(e0->stream));  // before the scratch images and `dst` are freed
    return BGR_OK;
}

BGR_API int bgr_checkpoint_restore(bgr_engine* e, const void* blob, size_t bytes) {
    std::vector<RestoreBlob> r(1);
    int rc = restore_check(e, blob, bytes, &r[0]);
    if (rc != BGR_OK) return rc;
    RestorePass x;
    size_t bad = 0;
    rc = restore_decode(r, x, nullptr, &bad);
    if (rc != BGR_OK) return rc;
    return restore_commit(r, x, &bad);
}

// ---- restore of a delta: the base decoded and verified as bgr_checkpoint_restore does, the delta applied onto its
// scratch image (k_ckpt_unpack_delta) and the target verified, then committed as a checkpoint of the target ----

// Applies the host-checked delta `dh` (offsets `off`, payload at `payload`) onto x's scratch image, which restore_decode
// filled with the verified base, and verifies the target's digest root and active rows.  On success x describes the
// target for restore_commit: its table (in a new `meta`) holds the scratch image with the target's rows.
static int restore_delta_decode(bgr_engine* e, const bgr_checkpoint_delta_header& dh, const std::vector<uint64_t>& off,
                                const uint8_t* payload, uint32_t base_blocks, RestorePass& x) {
    const uint32_t per = uint32_t(e->cols.size()) + 1u, own = e->tiles_for(dh.rows);
    unsigned int err = 0xFFFFFFFFu;
    std::vector<uint64_t> digest;
    std::vector<unsigned int> active;
    x.table.assign(1, ImageEntry{x.scratch.get(), e->cfg.order_base, 0ull, dh.rows, 0u});
    if (dh.n_blocks) {
        const size_t smem = sizeof(uint32_t) * (e->words + 1u);
        if (smem + sizeof(uint32_t) * (kCkptMaskWords + 1u) > 48u * 1024u)
            return fail(BGR_ERR_UNSUPPORTED, "bgr_checkpoint_restore supports at most 12000 word planes");
        const std::vector<uint32_t> absent = plane_absent(e), pad = plane_pad(e);
        // one upload, laid out as restore_decode's: image table, offsets, error word, planes, then the commit's pointers
        const size_t o_off = align16(sizeof(ImageEntry)), o_err = align16(o_off + sizeof(uint64_t) * off.size());
        const size_t o_absent = align16(o_err + sizeof(unsigned int)), o_pad = align16(o_absent + sizeof(uint32_t) * absent.size());
        const size_t dst_off = align16(o_pad + sizeof(uint32_t) * pad.size()), meta_bytes = dst_off + sizeof(uint8_t*) * 2u;
        DeviceBuffer<uint8_t> meta, d_payload;
        CUDA_TRY(meta.ensure(meta_bytes));
        CUDA_TRY(d_payload.ensure(std::max<uint64_t>(4, dh.payload_bytes)));
        std::vector<uint8_t> h(meta_bytes);
        std::memcpy(h.data(), x.table.data(), sizeof(ImageEntry));
        std::memcpy(h.data() + o_off, off.data(), sizeof(uint64_t) * off.size());
        std::memcpy(h.data() + o_err, &err, sizeof err);
        std::memcpy(h.data() + o_absent, absent.data(), sizeof(uint32_t) * absent.size());
        std::memcpy(h.data() + o_pad, pad.data(), sizeof(uint32_t) * pad.size());
        // the blocks past the base's XOR against zeros
        if (dh.n_blocks > base_blocks)
            CUDA_TRY(cudaMemsetAsync(x.scratch.get() + size_t(base_blocks) * e->tile_bytes, 0,
                                     size_t(dh.n_blocks - base_blocks) * e->tile_bytes, e->stream));
        CUDA_TRY(cudaMemcpyAsync(d_payload.get(), payload, dh.payload_bytes, cudaMemcpyHostToDevice, e->stream));
        CUDA_TRY(cudaMemcpyAsync(meta.get(), h.data(), meta_bytes, cudaMemcpyHostToDevice, e->stream));
        uint8_t* d = meta.get();
        CkptParams p{};
        p.images = reinterpret_cast<const ImageEntry*>(d);
        p.n_images = 1;
        p.words = e->words;
        p.plane_absent = reinterpret_cast<const uint32_t*>(d + o_absent);
        p.plane_pad = reinterpret_cast<const uint32_t*>(d + o_pad);
        p.mask_bits = 1u;
        for (const Column& c : e->cols) p.mask_bits |= c.absent;
        p.offsets = reinterpret_cast<const unsigned long long*>(d + o_off);
        p.payload = reinterpret_cast<uint32_t*>(d_payload.get());
        p.err = reinterpret_cast<unsigned int*>(d + o_err);
        k_ckpt_unpack_delta<<<dh.n_blocks, kTileRows, smem, e->stream>>>(p);
        e->launches += 1;
        CUDA_TRY(cudaGetLastError());
        int rc = digest_launch(e, p.images, 1u, own, &digest, &active);
        if (rc != BGR_OK) return rc;
        CUDA_TRY(cudaMemcpyAsync(&err, p.err, sizeof err, cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));  // `h` and the payload are freed below
        x.meta = std::move(meta);
        x.dst_off = dst_off;
    }
    x.blocks = own;
    if (err != 0xFFFFFFFFu)
        return fail(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta block " + std::to_string(err) +
                                                  ": a bad kind byte or padding, its kinds and bitmaps imply another length than its "
                                                  "offsets, or the target is not canonical (a non-zero word or mask byte of a row that "
                                                  "does not exist or lacks the column, a mask bit this registration does not use, or "
                                                  "bits past a column's element bytes)");
    uint64_t rows_alive = 0;
    for (uint32_t k = 0; k < own; ++k) rows_alive += active[k];
    const uint64_t root = bgr_seahash(own ? digest.data() : nullptr, size_t(own) * per * sizeof(uint64_t));
    if (root != dh.digest_root || rows_alive != dh.active)
        return fail(BGR_ERR_INVALID_ARGUMENT, "the decoded target's digest or active row count differs from the checkpoint delta "
                                              "header (corrupt payload)");
    return BGR_OK;
}

BGR_API int bgr_checkpoint_restore_delta(bgr_engine* e, const void* base, size_t base_bytes, const void* delta,
                                         size_t delta_bytes) {
    std::vector<RestoreBlob> r(1);
    int rc = restore_check(e, base, base_bytes, &r[0]);
    if (rc != BGR_OK) return rc;
    if (!delta) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    bgr_checkpoint_delta_header dh;
    std::vector<uint64_t> off;
    std::string err;
    rc = checkpoint_delta_check(ckpt_target(e), r[0].h, delta, delta_bytes, &dh, &off, &err);
    if (rc != BGR_OK) return fail(rc, err);
    RestorePass x;
    CUDA_TRY(x.scratch.ensure(std::max<size_t>(1, size_t(dh.n_blocks) * e->tile_bytes)));  // both frames' blocks
    size_t bad = 0;
    rc = restore_decode(r, x, nullptr, &bad);
    if (rc != BGR_OK) return rc;
    rc = restore_delta_decode(e, dh, off, static_cast<const uint8_t*>(delta) + checkpoint_delta_prefix(dh.n_blocks),
                              r[0].h.n_blocks, x);
    if (rc != BGR_OK) return rc;
    // commit the target as bgr_checkpoint_restore commits a checkpoint of it
    bgr_checkpoint_header& h = r[0].h;
    h.frame = dh.frame;
    h.rows = dh.rows;
    h.n_blocks = e->tiles_for(dh.rows);
    h.active = dh.active;
    h.elapsed_ns = dh.elapsed_ns;
    std::memcpy(h.rng, dh.rng, sizeof h.rng);
    h.digest_root = dh.digest_root;
    return restore_commit(r, x, &bad);
}

BGR_API int bgr_submit_requests(bgr_engine* e, const bgr_session_info* session, const bgr_request* requests,
                                uint32_t n_requests) {
    return submit(e, session, requests, n_requests);
}

BGR_API int bgr_collect(bgr_engine* e, bgr_checksum* checksums_out, uint32_t checksums_cap, uint32_t* n_checksums_out) {
    return collect(e, checksums_out, checksums_cap, n_checksums_out);
}

BGR_API int bgr_handle_requests(bgr_engine* e, const bgr_session_info* session, const bgr_request* requests,
                                uint32_t n_requests, bgr_checksum* checksums_out, uint32_t checksums_cap,
                                uint32_t* n_checksums_out) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    // the checksums returned must be THIS vector's: earlier bgr_submit_requests have to be collected first
    if (!e->pending.empty())
        return fail(BGR_ERR_STATE, "bgr_handle_requests with un-collected bgr_submit_requests pending: call bgr_collect first");
    e->tiledep_chain = false;
    int rc = submit(e, session, requests, n_requests);
    if (rc != BGR_OK) return rc;
    return collect(e, checksums_out, checksums_cap, n_checksums_out);
}

// ---- world batches: the request vectors of many engines with one registration in one launch ----
struct bgr_batch {
    std::vector<bgr_engine*> engines;
    cudaStream_t stream = nullptr;       // every member's
    JitKernel k;                         // k.batch_fn == nullptr: a call runs its worlds one after another
    std::vector<Prepared> prep;          // per member, reused by every call
    std::vector<uint32_t> buf;           // per member: its result buffer in this call
    WorldList list;                      // the members the current call has listed
    MappedHostBuffer<uint8_t> h_stage;   // a call's JitWorld records, then the listed worlds' ops
    DeviceBuffer<uint8_t> d_stage;
    MappedHostBuffer<uint8_t> h_ckpt;    // bgr_batch_checkpoint_restore: the payloads, gathered for one upload
    // bgr_batch_feed_begin: the scratch of one report in flight, grown to the largest call and never shrunk
    struct FeedScratch {
        MappedHostBuffer<FeedWorld> h_table;  // the table, uploaded with one copy
        DeviceBuffer<FeedWorld> table;
        DeviceBuffer<unsigned int> counts;    // tile_count, tile_off, tile_list [tiles each], world_scan [2n], info [4n], head [2]
        DeviceBuffer<uint32_t> out;           // the records, packed
        MappedHostBuffer<unsigned int> h_info;  // [4n]
        Event packed, done;
        cudaStream_t copy = nullptr;          // the records and infos cross PCIe here
        bool busy = false;
        uint32_t ticket = 0, seq = 0;
        std::vector<bgr_batch_feed> listed;   // the entries of the report in flight
    } feed;
    // bgr_batch_apply_edits: a ring of page-locked patches read in place (bgr_apply_edits' ring, on the batch's memory),
    // and the device copy of a call's EditWorld / SpawnWorld tables, grown to the largest call
    bgr_engine::EditStage edit_stage[bgr_engine::kEditBufs];
    uint32_t next_edit = 0;
    DeviceBuffer<uint8_t> edit_tables;
};

static bool same_specs(const bgr_engine* a, const bgr_engine* b) {
    return a->words == b->words && a->sys_specs.size() == b->sys_specs.size() && a->hash_specs.size() == b->hash_specs.size() &&
           std::equal(a->sys_specs.begin(), a->sys_specs.end(), b->sys_specs.begin(),
                      [](const SysSpec& x, const SysSpec& y) { return std::memcmp(&x, &y, sizeof x) == 0; }) &&
           std::equal(a->hash_specs.begin(), a->hash_specs.end(), b->hash_specs.begin(),
                      [](const HashSpec& x, const HashSpec& y) { return std::memcmp(&x, &y, sizeof x) == 0; });
}

// The batch's instance of the generated kernel: 128-row work items of two rows per thread unless BGR_TUNE_JIT_ITEM
// forces a size, whatever the members' sizes.  False (and the reason in *why) when the calls run sequentially.
static bool batch_specialise(bgr_batch* b, std::string* why) {
    const bgr_engine* e = b->engines[0];
    if (e->tune_jit == 0) { *why = "BGR_TUNE_JIT=0"; return false; }
    if (const char* w = jit_unsupported(e)) { *why = w; return false; }
    const int forced = jit_forced_item(e);
    const int item_rows = forced ? forced : 128, rows = forced ? std::min(jit_rows(e), forced / 32) : 2;
    if (!jit_compile(e, item_rows, rows, &b->k, why)) { b->k = JitKernel{}; return false; }
    if (!b->k.batch_fn) { *why = "the compiled module has no k_generic_jit_batch"; b->k = JitKernel{}; return false; }
    return true;
}

BGR_API int bgr_batch_create(bgr_engine* const* engines, uint32_t n, bgr_batch** out) {
    if (!engines || n == 0 || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "a batch needs at least one engine and an out pointer");
    *out = nullptr;
    for (uint32_t i = 0; i < n; ++i) {
        const bgr_engine* e = engines[i];
        const std::string who = "engine " + std::to_string(i) + ": ";
        if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, who + "null engine");
        if (!e->built) return fail(BGR_ERR_INVALID_ARGUMENT, who + "bgr_build has not been called");
        for (uint32_t j = 0; j < i; ++j)
            if (engines[j] == e) return fail(BGR_ERR_INVALID_ARGUMENT, who + "the same engine as engine " + std::to_string(j));
        if (e->cfg.device != engines[0]->cfg.device) return fail(BGR_ERR_INVALID_ARGUMENT, who + "on another device than engine 0");
        if (!same_specs(e, engines[0]))
            return fail(BGR_ERR_INVALID_ARGUMENT, who + "its registration (columns, systems, checksums) differs from engine 0's");
        if (!e->cfg.stream || e->cfg.stream != engines[0]->cfg.stream)
            return fail(BGR_ERR_INVALID_ARGUMENT, who + "every engine of a batch must be created with the same non-null bgr_config.stream");
        if ((e->cfg.flags & BGR_CFG_SHARDED) || e->group)
            return fail(BGR_ERR_UNSUPPORTED, who + "sharded engines (BGR_CFG_SHARDED, shard groups) cannot be batched");
        if (!use_generic(e))
            return fail(BGR_ERR_UNSUPPORTED, who + "only engines that run the generic one-launch program can be batched (not the particles "
                                                   "bundle or BGR_CFG_FORCE_STEPWISE)");
    }
    CUDA_TRY(cudaSetDevice(engines[0]->cfg.device));
    bgr_batch* b = new bgr_batch();
    b->engines.assign(engines, engines + n);
    b->stream = engines[0]->stream;
    b->prep.resize(n);
    b->buf.assign(n, 0);
    b->list = WorldList(n);
    std::string why;
    if (batch_specialise(b, &why)) {
        const size_t bytes = size_t(n) * (sizeof(JitWorld) + sizeof(Op) * kMaxOps);
        cudaError_t ce = b->h_stage.ensure(bytes);
        if (ce == cudaSuccess) ce = b->d_stage.ensure(bytes);
        if (ce != cudaSuccess) { delete b; return fail(BGR_ERR_CUDA, std::string("batch staging: ") + cudaGetErrorString(ce)); }
    } else if (std::getenv("BGR_JIT_VERBOSE")) {
        std::fprintf(stderr, "[bevy_ggrs_b200] world batch not specialised, its worlds run one after another: %s\n", why.c_str());
    }
    *out = b;
    return BGR_OK;
}

BGR_API void bgr_batch_destroy(bgr_batch* b) {
    if (!b) return;
    cudaStreamSynchronize(b->stream);
    if (b->feed.copy) {
        cudaStreamSynchronize(b->feed.copy);
        cudaStreamDestroy(b->feed.copy);
    }
    if (b->feed.busy)  // a batched report never waited: its feeds take reports again (no single ticket can free them)
        for (const bgr_batch_feed& r : b->feed.listed) b->engines[r.world]->feeds[r.feed].busy = false;
    delete b;
}

BGR_API int bgr_batch_specialised(bgr_batch* b, uint32_t* specialised_out) {
    if (!b || !specialised_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *specialised_out = b->k.batch_fn ? 1u : 0u;
    return BGR_OK;
}

extern "C++" {  // overloads and a template inside the C API's extern "C" block
namespace {

// entry i's world: worlds[i], or the world of a bgr_batch_feed / bgr_batch_edits entry
uint32_t world_of(uint32_t w) { return w; }
uint32_t world_of(const bgr_batch_feed& r) { return r.world; }
uint32_t world_of(const bgr_batch_edits& x) { return x.world; }

// One bgr_batch_* call over the worlds it lists, in the conventions of include/bevy_ggrs_b200.h's world batches: it
// begins the call on the batch's WorldList and sets status_out, n_sums and `counts` to 0 for every entry.  Each call keeps
// its own order of checks, with check() and fail_at() for a refusal.  A call that runs every world reports each one with
// record(), its checksums written at out() / room(), and returns outcome().
template <class Entry>
struct BatchCall {
    bgr_batch* b;
    const Entry* entries;
    int32_t* status_out;
    bgr_checksum* sums;  // every world's checksums, packed in list order as far as cap reaches
    uint32_t cap;
    uint32_t* n_sums;    // per entry: its checksum count
    uint32_t off = 0;    // the checksums of the entries recorded so far, up to cap
    int first = BGR_OK;  // the first non-OK status recorded, and its message
    std::string first_err;

    BatchCall(bgr_batch* b, const Entry* entries, uint32_t n, int32_t* status_out, bgr_checksum* sums = nullptr, uint32_t cap = 0,
              uint32_t* n_sums = nullptr, std::initializer_list<uint32_t*> counts = {})
        : b(b), entries(entries), status_out(status_out), sums(sums), cap(cap), n_sums(n_sums) {
        b->list.begin();
        std::fill_n(status_out, n, int32_t(BGR_OK));
        if (n_sums) std::fill_n(n_sums, n, 0u);
        for (uint32_t* c : counts)
            if (c) std::fill_n(c, n, 0u);
    }
    // entry i's world listed in this call (in range, not listed before), or entry i marked with the refusal
    int check(uint32_t i) {
        std::string why;
        const int rc = b->list.admit(world_of(entries[i]), &why);
        return rc == BGR_OK ? rc : fail_at(i, fail(rc, why));
    }
    // marks entry i with `status` and puts "world <index>: " in front of g_err
    int fail_at(uint32_t i, int status) {
        status_out[i] = status;
        g_err = "world " + std::to_string(world_of(entries[i])) + ": " + g_err;
        return status;
    }
    bgr_checksum* out() const { return sums && off < cap ? sums + off : nullptr; }
    uint32_t room() const { return sums && off < cap ? cap - off : 0u; }
    // entry i ran: its status (g_err its message when not OK) and the n checksums it wrote at out()
    void record(uint32_t i, int rc, uint32_t n) {
        n_sums[i] = n;
        off += std::min(n, cap - std::min(off, cap));
        if (rc != BGR_OK) {
            fail_at(i, rc);
            if (first == BGR_OK) { first = rc; first_err = g_err; }
        }
    }
    // the call's status: the first non-OK one recorded, with that world's message
    int outcome() {
        if (first != BGR_OK) g_err = first_err;
        return first;
    }
};

}  // namespace
}  // extern "C++"

BGR_API int bgr_batch_handle_requests(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const bgr_session_info* sessions,
                                      const bgr_request* requests, const uint32_t* n_requests, bgr_checksum* checksums_out,
                                      uint32_t checksums_cap, uint32_t* n_checksums_out, int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (n_worlds && (!worlds || !n_requests || !n_checksums_out || !status_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("HandleRequests");
    BatchCall call(b, worlds, n_worlds, status_out, checksums_out, checksums_cap, n_checksums_out);
    auto session = [&](uint32_t i) { return sessions ? &sessions[i] : nullptr; };
    // every world is validated and compiled before any executes
    std::vector<size_t> req_off(n_worlds + 1, 0);
    for (uint32_t i = 0; i < n_worlds; ++i) {
        int rc = call.check(i);
        if (rc != BGR_OK) return rc;
        const uint32_t w = worlds[i];
        if (n_requests[i] > BGR_MAX_REQUESTS)
            return call.fail_at(i, fail(BGR_ERR_CAPACITY, "too many requests in one handle_requests call"));
        bgr_engine* e = b->engines[w];
        if (!e->pending.empty())
            return call.fail_at(i, fail(BGR_ERR_STATE, "un-collected bgr_submit_requests pending: call bgr_collect first"));
        req_off[i + 1] = req_off[i] + n_requests[i];
        rc = prepare(e, session(i), requests ? requests + req_off[i] : nullptr, n_requests[i], b->prep[w]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    if (!b->k.batch_fn) {  // the worlds' own submit path, in list order
        for (uint32_t i = 0; i < n_worlds; ++i) {
            uint32_t n = 0;
            const int rc = bgr_handle_requests(b->engines[worlds[i]], session(i), requests ? requests + req_off[i] : nullptr, n_requests[i],
                                               call.out(), call.room(), &n);
            call.record(i, rc, n);
        }
        return call.outcome();
    }
    if (n_worlds == 0) return BGR_OK;
    // spawning worlds: growable members take the capacity their spawns need (a program does not depend on the capacity,
    // submit), and each world's ParticleRng draws go to its result buffer's spawn values.  A vector past a member's
    // ceiling is refused before any member grows.
    for (uint32_t i = 0; i < n_worlds; ++i) {
        const bgr_engine* e = b->engines[worlds[i]];
        const uint64_t rows = b->prep[worlds[i]].pg.rows_needed;
        if (rows > e->ceiling)
            return call.fail_at(i, fail(BGR_ERR_CAPACITY, std::to_string(rows) + " rows exceed the engine's ceiling of " +
                                                              std::to_string(e->ceiling) + " rows (BGR_CFG_GROWABLE)"));
    }
    for (uint32_t i = 0; i < n_worlds; ++i) {
        const uint32_t w = worlds[i];
        bgr_engine* e = b->engines[w];
        const Program& pg = b->prep[w].pg;
        if (pg.rows_needed) {
            const int rc = grow_to(e, pg.rows_needed);
            if (rc != BGR_OK) return call.fail_at(i, rc);
        }
        b->buf[w] = e->next_buf;
        if (!pg.spawn_vals.empty()) std::memcpy(e->spawn[b->buf[w]].get(), pg.spawn_vals.data(), pg.spawn_vals.size() * sizeof(float2));
    }
    // one record per world and the worlds' ops in page-locked staging, one copy, one launch
    uint8_t* h = b->h_stage.get();
    JitWorld* recs = reinterpret_cast<JitWorld*>(h);
    Op* ops = reinterpret_cast<Op*>(h + sizeof(JitWorld) * n_worlds);
    const uint32_t subs = kTileRows / uint32_t(b->k.item_rows);
    uint32_t items = 0, n_ops = 0;
    for (uint32_t i = 0; i < n_worlds; ++i) {
        const uint32_t w = worlds[i];
        bgr_engine* e = b->engines[w];
        Prepared& p = b->prep[w];
        p.t_compiled = host_ns();
        e->tiledep_chain = false;
        const int rc = plan(e, p);  // a deferred live image this vector cannot start from is written here, before the launch
        if (rc != BGR_OK) return call.fail_at(i, rc);
        JitWorld r = launch_record(e, p.pg, b->buf[w]);
        r.item0 = items;
        r.ops_off = n_ops;
        recs[i] = r;
        std::memcpy(ops + n_ops, p.pg.ops, sizeof(Op) * p.pg.n_ops);
        items += r.n_tiles * subs;
        n_ops += p.pg.n_ops;
    }
    uint8_t* d = b->d_stage.get();
    const JitWorld* d_recs = reinterpret_cast<const JitWorld*>(d);
    const Op* d_ops = reinterpret_cast<const Op*>(d + sizeof(JitWorld) * n_worlds);
    CUDA_TRY(cudaMemcpyAsync(d, h, sizeof(JitWorld) * n_worlds + sizeof(Op) * n_ops, cudaMemcpyHostToDevice, b->stream));
    void* args[] = {&d_recs, &n_worlds, &d_ops};
    CUDA_TRY(cudaLaunchKernel(b->k.batch_fn, dim3(items), dim3(b->k.threads), args, 0, b->stream));
    CUDA_TRY(cudaGetLastError());
    for (uint32_t i = 0; i < n_worlds; ++i) {
        const uint32_t w = worlds[i];
        bgr_engine* e = b->engines[w];
        e->launches += 1;
        e->last_kernel = BGR_KERNEL_GENERIC_NVRTC | (uint32_t(b->k.item_rows) << 16) | BGR_KERNEL_BATCHED;
        const int rc = commit(e, b->prep[w], b->buf[w]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    for (uint32_t i = 0; i < n_worlds; ++i) {
        uint32_t n = 0;
        const int rc = collect(b->engines[worlds[i]], call.out(), call.room(), &n);
        call.record(i, rc, n);
    }
    return call.outcome();
}

// ---- replays: a recorded input log run through a world, checksummed at an interval, without snapshots ----
namespace {


// One world's replay, validated and planned against its engine's HostState: nothing has executed yet
struct ReplayJob {
    bgr_engine* e = nullptr;
    const struct bgr_replay* r = nullptr;
    ReplayClock c{};
    std::vector<uint32_t> prefix;    // [n + 1]: spawn frames before each frame; empty without spawn_particles
    std::vector<float2> spawn_vals;  // the log's ParticleRng draws, in frame order (what compile_requests draws)
    ParticleRng rng;                 // ParticleRng after the log
    uint64_t rows_end = 0, elapsed_end = 0;
    uint32_t n_points = 0;
    std::vector<bgr_checksum> sums;
    bool bad = false;                // a checksum frame failed its finite assertion; the first is bad_frame
    int32_t bad_frame = 0;
    // keyframes (bgr_replay_keyframes): frames f0 + j, j in [0, n), with (f0 + j) % kf->interval == 0
    const struct bgr_keyframes* kf = nullptr;
    std::vector<KeyframePlan> kfp;   // every keyframe of the log (replay_keyframes.hpp)
    uint32_t n_kf = 0, kf_done = 0;  // keyframes in the log, and written
    size_t kf_bound = 0;             // bytes the blobs may take: every vector RAW, alignment included
    size_t kf_pos = 0, kf_end = 0;   // the next blob's offset in kf->dst, and the end of the last one
    // trace (bgr_replay_trace): samples at frames f0 + j, j in [0, n), with (f0 + j) % tr->interval == 0
    const struct bgr_trace* tr = nullptr;
    FeedParams tp{};                        // its field list mapped onto the image (feed_fields)
    std::vector<bgr_trace_sample> samples;  // every sample of the log (replay_trace.hpp)
    size_t tr_stride = 0;                   // bytes per sample: n_rows records
    uint32_t tr_done = 0;                   // samples written
};

uint64_t ggrs_runtime_ns(const bgr_engine* e, int64_t frame) { return uint64_t(frame) * 1000000000ULL / uint64_t(e->cfg.fps); }
// checksum frames f0 + j with j in [a, b): the first one (~0: none) and how many
uint64_t first_point(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_first_point(job.c.f0, job.r->checksum_interval, a, b); }
uint32_t points_in(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_points_in(job.c.f0, job.r->checksum_interval, a, b); }
// spawn frames before frame j, and RollbackOrdered::len() there
uint32_t prefix_at(const ReplayJob& job, uint32_t j) { return job.prefix.empty() ? 0u : job.prefix[j]; }
uint32_t rows_at(const ReplayJob& job, uint32_t j) { return job.c.rows0 + job.c.rate * prefix_at(job, j); }
// keyframe frames f0 + j with j in [a, b): the first one (~0: none) and how many
uint64_t first_kf(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_first_point(job.c.f0, job.kf ? job.kf->interval : 0u, a, b); }
uint32_t kfs_in(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_points_in(job.c.f0, job.kf ? job.kf->interval : 0u, a, b); }
// trace sample frames f0 + j with j in [a, b): the first one (~0: none) and how many
uint64_t first_tr(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_first_point(job.c.f0, job.tr ? job.tr->interval : 0u, a, b); }
uint32_t trs_in(const ReplayJob& job, uint32_t a, uint32_t b) { return replay_points_in(job.c.f0, job.tr ? job.tr->interval : 0u, a, b); }

// Validates a replay (with keyframes when kf is not null, with a trace when tr is not null) and computes everything the
// replay changes on the host, without executing or changing anything
int replay_plan(bgr_engine* e, const struct bgr_replay* r, ReplayJob& job, const struct bgr_keyframes* kf = nullptr,
                const struct bgr_trace* tr = nullptr) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (!e->built) return fail(BGR_ERR_STATE, "bgr_build has not been called");
    if (!r) return fail(BGR_ERR_INVALID_ARGUMENT, "null replay");
    if (kf && kf->interval == 0) return fail(BGR_ERR_INVALID_ARGUMENT, "bgr_keyframes.interval must be >= 1");
    if (kf && kf->reserved) return fail(BGR_ERR_INVALID_ARGUMENT, "bgr_keyframes.reserved must be 0");
    FeedParams tp{};
    if (tr) {
        std::string err;
        int rc = trace_check(*tr, e->growable() ? e->ceiling : e->cfg.max_entities, &err);
        if (rc == BGR_OK) rc = engine_feed_fields(e, tr->fields, tr->n_fields, tp, &err);
        if (rc != BGR_OK) return fail(rc, err);
    }
    if ((e->cfg.flags & BGR_CFG_SHARDED) || e->group) return fail(BGR_ERR_UNSUPPORTED, "replays do not run on sharded engines");
    if (!e->pending.empty()) return fail(BGR_ERR_STATE, "bgr_replay with un-collected bgr_submit_requests pending: call bgr_collect first");
    if (r->reserved) return fail(BGR_ERR_INVALID_ARGUMENT, "bgr_replay.reserved must be 0");
    if (r->n_players > BGR_MAX_PLAYERS) return fail(BGR_ERR_INVALID_ARGUMENT, "n_players > BGR_MAX_PLAYERS");
    if (r->n_frames > BGR_MAX_REPLAY_FRAMES) return fail(BGR_ERR_INVALID_ARGUMENT, "n_frames > BGR_MAX_REPLAY_FRAMES");
    if (r->n_frames && r->n_players && !r->inputs) return fail(BGR_ERR_INVALID_ARGUMENT, "null input log");
    const HostState& s = e->st;
    if (s.frame_count < 0) return fail(BGR_ERR_STATE, "a replay starts at RollbackFrameCount >= 0");
    if (int64_t(s.frame_count) + r->n_frames > int64_t(INT32_MAX)) return fail(BGR_ERR_INVALID_ARGUMENT, "RollbackFrameCount + n_frames overflows i32");
    const uint32_t n = r->n_frames;
    // GgrsTimePlugin::update of the first step (compile_requests)
    if (n && ggrs_runtime_ns(e, int64_t(s.frame_count) + 1) < s.elapsed_ns)
        return fail(BGR_ERR_STATE, "tried to move Time<GgrsTime> backwards (RollbackFrameCount went back without LoadWorld)");
    job = ReplayJob{};
    job.e = e; job.r = r; job.kf = kf; job.tr = tr;
    uint32_t n_counter = 0;
    for (const SystemReg& sy : e->systems) n_counter += (sy.id == BGR_SYS_U32_STORE_CALL_COUNT);
    const bool spawn = e->spawn_sys >= 0;
    job.c = replay_clock(s.frame_count, e->cfg.fps, n ? s.elapsed_ns : 0u, r->n_players, s.call_count, n_counter, spawn,
                         spawn ? e->systems[size_t(e->spawn_sys)].params[0] : 0u, s.n_rows);
    const ReplayClock& c = job.c;
    job.rng = s.rng;
    job.rows_end = s.n_rows;
    if (spawn) {  // spawn_particles.run_if(spawn_pressed)
        job.prefix.assign(size_t(n) + 1, 0u);
        uint32_t spawns = 0;
        for (uint32_t j = 0; j < n; ++j) {
            job.prefix[j] = spawns;
            bool pressed = false;
            for (uint32_t k = 0; k < r->n_players; ++k) pressed = pressed || (r->inputs[size_t(j) * r->n_players + k] & BGR_INPUT_SPAWN);
            spawns += pressed ? 1u : 0u;
        }
        job.prefix[n] = spawns;
        if (spawns && c.rate > kMaxSpawnVals) return fail(BGR_ERR_CAPACITY, "too many particles spawned by one request vector");
        job.rows_end = uint64_t(s.n_rows) + uint64_t(c.rate) * spawns;
        if (job.rows_end > e->cfg.max_entities) {
            if (!e->growable()) return fail(BGR_ERR_CAPACITY, "spawn_particles exceeds max_entities");
            if (job.rows_end > e->ceiling)
                return fail(BGR_ERR_CAPACITY, std::to_string(job.rows_end) + " rows exceed the engine's ceiling of " +
                                                  std::to_string(e->ceiling) + " rows (BGR_CFG_GROWABLE)");
        }
        job.spawn_vals.reserve(size_t(c.rate) * spawns);
        for (uint32_t i = 0; i < spawns; ++i)
            for (uint32_t k = 0; k < c.rate; ++k) {  // particles.rs:262-268, in frame order
                float2 v;
                v.x = job.rng.random_range(-200.0f, 200.0f);
                v.y = job.rng.random_range(-200.0f, 200.0f);
                job.spawn_vals.push_back(v);
            }
    }
    if (kf) {
        job.kfp = plan_replay_keyframes(c, n, kf->interval, s.elapsed_ns, job.prefix, s.rng, e->words);
        job.n_kf = uint32_t(job.kfp.size());
        for (const KeyframePlan& p : job.kfp) job.kf_bound += p.max_bytes;
    }
    if (tr) {
        job.tp = tp;
        job.samples = plan_trace_samples(c, n, tr->interval, job.prefix);
        job.tr_stride = size_t(tr->n_rows) * trace_record_bytes(tp);
    }
    job.elapsed_end = n ? ggrs_runtime_ns(e, int64_t(c.f0) + n) : s.elapsed_ns;
    job.n_points = points_in(job, 0, n);
    return BGR_OK;
}

// The output checks of a planned replay with keyframes, made before anything runs (a null dst holds nothing)
int keyframe_caps(const ReplayJob& job) {
    const struct bgr_keyframes* kf = job.kf;
    const size_t cap = kf->dst ? kf->dst_cap : 0u;
    if (cap < job.kf_bound)
        return fail(BGR_ERR_CAPACITY, "the keyframes may need " + std::to_string(job.kf_bound) + " bytes, dst_cap is " + std::to_string(cap));
    if (kf->index_cap < job.n_kf)
        return fail(BGR_ERR_CAPACITY, "the replay writes " + std::to_string(job.n_kf) + " keyframes, index_cap is " + std::to_string(kf->index_cap));
    if (job.n_kf && !kf->index) return fail(BGR_ERR_INVALID_ARGUMENT, "null keyframe index");
    return BGR_OK;
}

// The output checks of a planned replay with a trace, made before anything runs (a null dst holds nothing)
int trace_caps(const ReplayJob& job) {
    const struct bgr_trace* t = job.tr;
    const size_t need = job.samples.size() * job.tr_stride, cap = t->dst ? t->dst_cap : 0u;
    if (cap < need) return fail(BGR_ERR_CAPACITY, "the trace writes " + std::to_string(need) + " bytes, dst_cap is " + std::to_string(cap));
    if (t->samples_cap < job.samples.size())
        return fail(BGR_ERR_CAPACITY, "the replay takes " + std::to_string(job.samples.size()) + " trace samples, samples_cap is " +
                                          std::to_string(t->samples_cap));
    if (!job.samples.empty() && !t->samples) return fail(BGR_ERR_INVALID_ARGUMENT, "null sample index");
    return BGR_OK;
}

// Samples [q0, q0 + m) of a launch whose kernel covered the rows below `cover`: the traced rows at or past it exist at none
// of them, so their records (row, state 0, zero words) are written here
void trace_fill_rows(const ReplayJob& job, uint32_t q0, uint32_t m, uint32_t cover) {
    const struct bgr_trace* t = job.tr;
    const uint32_t end = t->first_row + t->n_rows, rb = trace_record_bytes(job.tp);
    for (uint32_t q = q0; q < q0 + m; ++q)
        for (uint32_t row = std::max(t->first_row, cover); row < end; ++row) {
            uint8_t* rec = static_cast<uint8_t*>(t->dst) + trace_record_offset(q, row - t->first_row, t->n_rows, rb);
            std::memset(rec, 0, rb);
            std::memcpy(rec, &row, sizeof row);
        }
}

// The records of the job's next sample from image 0 as it stands, straight to dst (the chunked replay, at a sample frame)
int trace_gather(ReplayJob& job, DeviceBuffer<uint8_t>& stage) {
    bgr_engine* e = job.e;
    const struct bgr_trace* t = job.tr;
    int rc = materialize_live(e);
    if (rc != BGR_OK) return rc;
    const size_t tab = align16(sizeof(TraceGather));
    CUDA_TRY(stage.ensure(tab + job.tr_stride));
    const TraceGather g{e->image(0), reinterpret_cast<uint32_t*>(stage.get() + tab), e->st.n_rows, t->first_row, t->n_rows, 0u};
    CUDA_TRY(cudaMemcpyAsync(stage.get(), &g, sizeof g, cudaMemcpyHostToDevice, e->stream));
    k_trace_gather<<<(t->n_rows + 255u) / 256u, 256, 0, e->stream>>>(job.tp, reinterpret_cast<const TraceGather*>(stage.get()), 1u, t->n_rows);
    e->launches += 1;
    CUDA_TRY(cudaGetLastError());
    e->tiledep_chain = false;
    uint8_t* dst = static_cast<uint8_t*>(t->dst) + size_t(job.tr_done) * job.tr_stride;
    CUDA_TRY(cudaMemcpyAsync(dst, stage.get() + tab, job.tr_stride, cudaMemcpyDeviceToHost, e->stream));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    job.tr_done += 1;
    return BGR_OK;
}

// Encodes the keyframe images of `x` (image i is the next keyframe of owner[i]; a job's images in frame order, one after
// another) into their jobs' buffers and indices
int keyframes_write(ImageEncoder& x, const std::vector<ReplayJob*>& owner) {
    int rc = encode_measure(x);
    if (rc != BGR_OK) return rc;
    for (size_t i = 0; i < x.im.size(); ++i) {
        ReplayJob& job = *owner[i];
        const size_t bytes = blob_bytes(x.im[i]);
        x.im[i].dst = static_cast<uint8_t*>(job.kf->dst) + job.kf_pos;
        bgr_keyframe& k = job.kf->index[job.kf_done++];
        k.frame = x.im[i].h.frame;
        k.reserved = 0;
        k.offset = job.kf_pos;
        k.bytes = bytes;
        job.kf_end = job.kf_pos + bytes;
        job.kf_pos = align8(job.kf_end);
    }
    return encode_pack(x);
}

// The image to encode for keyframe q of `job`, held at `img`
EncodeImage keyframe_image(const ReplayJob& job, uint32_t q, const uint8_t* img) {
    const KeyframePlan& p = job.kfp[q];
    EncodeImage m;
    m.img = img;
    m.order_base = job.e->cfg.order_base;
    m.h = checkpoint_header(job.e, job.c.f0 + int32_t(p.j), p.rows, p.elapsed_ns, p.rng);
    return m;
}

// The replay in chunks through the engine's own kernel: each chunk is one request vector of at most kMaxOps ops,
// kMaxSaves Saves and kMaxSpawnVals spawned rows, compiled by compile_requests, whose checksum points are Saves that
// store nothing (OPF_NO_STORE) and push nothing onto the ring
int replay_chunked(ReplayJob& job) {
    bgr_engine* e = job.e;
    const struct bgr_replay* r = job.r;
    const uint32_t n = r->n_frames, k = r->checksum_interval;
    std::vector<bgr_request> reqs(kMaxOps);
    Prepared p;
    Program adv;
    ImageEncoder x;
    x.e = e;
    const std::vector<ReplayJob*> owner{&job};
    DeviceBuffer<uint8_t> tr_stage;  // one sample's records: freed with the call
    for (uint32_t j = 0; j < n;) {
        if (first_kf(job, j, j + 1) == j) {  // a keyframe: image 0 as it stands before frame j, a chunk boundary
            int rc = materialize_live(e);
            if (rc != BGR_OK) return rc;
            x.im.assign(1, keyframe_image(job, job.kf_done, e->image(0)));
            rc = keyframes_write(x, owner);
            if (rc != BGR_OK) return rc;
        }
        if (first_tr(job, j, j + 1) == j) {  // a trace sample: likewise
            const int rc = trace_gather(job, tr_stage);
            if (rc != BGR_OK) return rc;
        }
        uint32_t b = j, ops = 0, saves = 0, spawned = 0;
        while (b < n && (b == j || (first_kf(job, b, b + 1) != b && first_tr(job, b, b + 1) != b))) {
            const uint32_t pt = (k && (int64_t(job.c.f0) + b) % k == 0) ? 1u : 0u;
            const uint32_t sp = prefix_at(job, b + 1) != prefix_at(job, b) ? job.c.rate : 0u;
            if (ops + pt + 1 > uint32_t(kMaxOps) || saves + pt > uint32_t(kMaxSaves) || spawned + sp > kMaxSpawnVals) break;
            ops += pt + 1; saves += pt; spawned += sp;
            ++b;
        }
        for (uint32_t i = 0; i < b - j; ++i) {
            bgr_request& rq = reqs[i];
            std::memset(&rq, 0, sizeof rq);
            rq.kind = BGR_REQ_ADVANCE;
            rq.n_players = r->n_players;
            for (uint32_t h = 0; h < r->n_players; ++h) rq.inputs[h] = r->inputs[size_t(j + i) * r->n_players + h];
        }
        p.t_begin = host_ns();
        p.s = e->st;
        p.next = DeferredLive{};
        adv.~Program();
        new (&adv) Program;
        int rc = compile_requests(e, p.s, nullptr, reqs.data(), b - j, adv);
        if (rc != BGR_OK) return rc;
        p.pg.~Program();
        new (&p.pg) Program;
        Program& pg = p.pg;
        pg.live_rows = adv.live_rows; pg.max_rows = adv.max_rows; pg.rows_needed = adv.rows_needed;
        pg.has_advance = adv.has_advance; pg.has_spawn = adv.has_spawn;
        pg.spawn_vals = std::move(adv.spawn_vals);
        for (uint32_t i = 0; i < b - j; ++i) {
            const int64_t frame = int64_t(job.c.f0) + j + i;
            if (k && frame % k == 0) {  // SaveGameState{frame}: the checksum only
                Op& sv = pg.ops[pg.n_ops++];
                std::memset(&sv, 0, sizeof sv);
                sv.kind = OP_SAVE; sv.flags = OPF_NO_STORE;
                sv.n_rows = adv.ops[i].n_rows;
                sv.save_index = pg.n_saves;
                pg.save_frames[pg.n_saves] = int32_t(frame);
                pg.save_totals[pg.n_saves] = sv.n_rows;
                ++pg.n_saves;
            }
            pg.ops[pg.n_ops++] = adv.ops[i];
        }
        rc = execute(e, p);
        if (rc != BGR_OK) return rc;
        bgr_checksum sums[kMaxSaves];
        uint32_t got = 0;
        int32_t bad_frame = 0;
        rc = collect(e, sums, kMaxSaves, &got, &bad_frame);
        if (rc == BGR_ERR_NON_FINITE) {
            if (!job.bad) { job.bad = true; job.bad_frame = bad_frame; }
        } else if (rc != BGR_OK) {
            return rc;
        }
        job.sums.insert(job.sums.end(), sums, sums + got);
        j = b;
    }
    return BGR_OK;
}

// The generated kernel's replay entry point for an engine whose rows end up in `tiles` tiles: its own kernel when bgr_build
// compiled one (the instance run_generic picks), else one compiled now.  nullptr: the replay runs in chunks.
const JitKernel* replay_kernel(bgr_engine* e, uint32_t tiles) {
    // the registrations jit_specialise takes: an engine that ticks on the stepwise path (more than kMaxGenericSys
    // systems, a tile over the generic program's limit) replays through it too
    if (!e->generic_ok || e->tune_jit == 0 || !e->tune_generic || (e->cfg.flags & BGR_CFG_FORCE_STEPWISE) || jit_unsupported(e))
        return nullptr;
    const bool few = tiles < 3u * uint32_t(e->num_sms);  // few tiles per SM: 128-row work items (run_generic)
    if (e->jit.fn) {
        const JitKernel& k = (e->jit_small.fn && few) ? e->jit_small : e->jit;
        return k.replay_fn ? &k : nullptr;
    }
    const int forced = jit_forced_item(e);
    JitKernel& k = (few && !forced) ? e->replay_jit_small : e->replay_jit;
    if (!k.fn) {
        const int item = forced ? forced : few ? 128 : int(kTileRows);
        const int rows = forced ? std::min(jit_rows(e), forced / 32) : few ? 2 : jit_rows(e);
        std::string why;
        if (!jit_compile(e, item, rows, &k, &why)) {
            k = JitKernel{};
            if (std::getenv("BGR_JIT_VERBOSE"))
                std::fprintf(stderr, "[bevy_ggrs_b200] replay kernel not compiled, the replay runs in chunks: %s\n", why.c_str());
            return nullptr;
        }
    }
    return k.replay_fn ? &k : nullptr;
}

// The replays of `jobs` (every one with frames to run) on the replay entry point of `k`: the logs, spawn tables and spawn
// values go to the device once, then each launch runs every unfinished world through its next frames, as many as keep
// the launch's checksum points within kReplayLaunchPoints (one launch for everything but very long logs at short
// intervals), and its checksum points come back with one copy.  Replays with keyframes (every job has them, or none)
// run k_generic_jit_replay_kf, whose launches also end where the keyframe images staged would pass the keyframe budget
// (at least one keyframe of each unfinished world per launch); the image-table encoder then turns all of a launch's
// keyframe images into blobs.  Replays with traces (every job has one, with one field list, or none) run
// k_generic_jit_replay_trace, whose launches likewise end where the records staged would pass the trace budget; a
// launch's records come back with one copy, straight into dst for one world, else through host memory.  Synchronous.
int replay_launch(const JitKernel& k, const std::vector<ReplayJob*>& jobs, uint32_t kernel_bits) {
    bgr_engine* e0 = jobs[0]->e;
    cudaStream_t stream = e0->stream;
    const bool kf = jobs[0]->kf != nullptr, tr = jobs[0]->tr != nullptr;
    const size_t world_bytes = align16(sizeof(ReplayWorld) * jobs.size());
    const size_t rec_bytes = world_bytes + (kf ? align16(sizeof(ReplayKeyframes) * jobs.size()) : 0u) +
                             (tr ? align16(sizeof(ReplayTrace) * jobs.size()) : 0u);
    std::vector<size_t> in_off(jobs.size()), pre_off(jobs.size()), val_off(jobs.size());
    size_t bytes = rec_bytes;
    for (size_t i = 0; i < jobs.size(); ++i) {
        const ReplayJob& j = *jobs[i];
        in_off[i] = bytes; bytes = align16(bytes + size_t(j.r->n_frames) * j.r->n_players);
        pre_off[i] = bytes; bytes = align16(bytes + j.prefix.size() * sizeof(uint32_t));
        val_off[i] = bytes; bytes = align16(bytes + j.spawn_vals.size() * sizeof(float2));
    }
    CUDA_TRY(e0->replay_stage.ensure(bytes));
    uint8_t* d = e0->replay_stage.get();
    // one copy: a copy per world from pageable memory cost more host time than a world's whole replay kernel (the
    // staging is not zeroed: alignment padding is never read)
    std::unique_ptr<uint8_t[]> h(new uint8_t[bytes - rec_bytes]);
    for (size_t i = 0; i < jobs.size(); ++i) {
        const ReplayJob& j = *jobs[i];
        if (j.r->n_players) std::memcpy(&h[in_off[i] - rec_bytes], j.r->inputs, size_t(j.r->n_frames) * j.r->n_players);
        if (!j.prefix.empty()) std::memcpy(&h[pre_off[i] - rec_bytes], j.prefix.data(), j.prefix.size() * sizeof(uint32_t));
        if (!j.spawn_vals.empty()) std::memcpy(&h[val_off[i] - rec_bytes], j.spawn_vals.data(), j.spawn_vals.size() * sizeof(float2));
    }
    CUDA_TRY(cudaMemcpyAsync(d + rec_bytes, h.get(), bytes - rec_bytes, cudaMemcpyHostToDevice, stream));
    for (ReplayJob* j : jobs) {  // image 0 is read: a pending deferred live image is written first
        int rc = materialize_live(j->e);
        if (rc != BGR_OK) return rc;
        j->e->tiledep_chain = false;
    }
    const uint32_t subs = kTileRows / uint32_t(k.item_rows);
    std::vector<uint32_t> cur(jobs.size(), 0u), seg_end(jobs.size()), seg_points(jobs.size());
    std::vector<ReplayWorld> recs;
    std::vector<ReplayKeyframes> kf_recs;
    std::vector<ReplayTrace> tr_recs;
    std::vector<size_t> rec_job, acc_off;
    std::vector<unsigned long long> acc;
    std::vector<uint8_t> h_recs(rec_bytes);
    ImageEncoder x;
    x.e = e0;
    std::vector<ReplayJob*> owner;
    DeviceBuffer<uint8_t> kf_stage;  // the keyframe images of a launch: up to the keyframe budget, freed with the call
    DeviceBuffer<uint8_t> tr_stage;  // the trace records of a launch: up to the trace budget, freed with the call
    std::vector<uint8_t> h_tr;       // ... on the host, when they belong to several worlds
    const TraceMap tr_map = tr ? trace_map(jobs[0]->tp) : TraceMap{};
    for (;;) {
        recs.clear(); kf_recs.clear(); tr_recs.clear(); rec_job.clear(); acc_off.clear();
        uint32_t active = 0;
        for (size_t i = 0; i < jobs.size(); ++i) active += cur[i] < jobs[i]->r->n_frames ? 1u : 0u;
        if (!active) break;
        const uint32_t budget = std::max(1u, e0->tune_replay_points / active);
        const uint64_t kf_budget = std::max<uint64_t>(1, e0->tune_keyframe_bytes / active);
        const uint64_t tr_budget = std::max<uint64_t>(1, e0->tune_trace_bytes / active);
        uint32_t items = 0;
        size_t points = 0, staged = 0;
        for (size_t i = 0; i < jobs.size(); ++i) {
            const ReplayJob& job = *jobs[i];
            bgr_engine* e = job.e;
            const uint32_t n = job.r->n_frames, a = cur[i], kk = job.r->checksum_interval;
            if (a >= n) continue;
            uint32_t b = n;
            const uint64_t f = first_point(job, a, n);
            if (f != ~0ULL && f + uint64_t(budget) * kk < n) b = uint32_t(f + uint64_t(budget) * kk);  // `budget` points
            // keyframe images hold every tile the world has by its end, so that the stride does not depend on b
            const uint64_t stride = uint64_t(std::max(1u, e->tiles_for(uint32_t(job.rows_end)))) * e->tile_bytes;
            if (kf) {
                const uint64_t fk = first_kf(job, a, n), m = std::max<uint64_t>(1, kf_budget / stride), kint = job.kf->interval;
                if (fk != ~0ULL && fk + m * kint < b) b = uint32_t(fk + m * kint);  // m keyframes
            }
            if (tr) b = trace_launch_end(job.c.f0, job.tr->interval, a, b, tr_budget, job.tr_stride);
            seg_end[i] = b;
            seg_points[i] = points_in(job, a, b);
            ReplayWorld w;
            std::memset(&w, 0, sizeof w);
            w.arena = e->arena.ptr();
            w.order_base = e->cfg.order_base;
            w.inputs = d + in_off[i];
            w.prefix = job.prefix.empty() ? nullptr : reinterpret_cast<const uint32_t*>(d + pre_off[i]);
            w.spawn_vals = reinterpret_cast<const float2*>(d + val_off[i]);
            if (e->spawn_sys >= 0) w.spawn_ttl = e->systems[size_t(e->spawn_sys)].params[1];
            w.next_point = first_point(job, a, b);
            w.c = job.c;
            w.interval = kk;
            w.j0 = a; w.j1 = b;
            w.live_rows = rows_at(job, a);
            w.n_tiles = std::max(1u, e->tiles_for(rows_at(job, b)));
            w.item0 = items;
            items += w.n_tiles * subs;
            acc_off.push_back(points);  // w.acc, once the buffer is sized (below)
            points += seg_points[i];
            recs.push_back(w);
            rec_job.push_back(i);
            if (kf) {
                ReplayKeyframes r;
                std::memset(&r, 0, sizeof r);
                r.staging = reinterpret_cast<uint8_t*>(staged);  // an offset until the staging is sized (below)
                r.stride = stride;
                r.first = first_kf(job, a, b);
                r.interval = job.kf->interval;
                staged += size_t(kfs_in(job, a, b)) * stride;
                kf_recs.push_back(r);
            }
            if (tr) {
                ReplayTrace r;
                std::memset(&r, 0, sizeof r);
                r.staging = reinterpret_cast<uint8_t*>(staged);  // an offset until the staging is sized (below)
                r.stride = job.tr_stride;
                r.first = first_tr(job, a, b);
                r.interval = job.tr->interval;
                r.first_row = job.tr->first_row;
                r.n_rows = job.tr->n_rows;
                staged += size_t(trs_in(job, a, b)) * job.tr_stride;
                tr_recs.push_back(r);
            }
        }
        if (kf) {
            CUDA_TRY(kf_stage.ensure(std::max<size_t>(1, staged)));
            for (ReplayKeyframes& r : kf_recs) r.staging = kf_stage.get() + reinterpret_cast<size_t>(r.staging);
        }
        if (tr) {
            CUDA_TRY(tr_stage.ensure(std::max<size_t>(1, staged)));
            for (ReplayTrace& r : tr_recs) r.staging = tr_stage.get() + reinterpret_cast<size_t>(r.staging);
        }
        CUDA_TRY(e0->replay_acc.ensure(std::max<size_t>(1, points) * kAccStride));
        for (size_t ri = 0; ri < recs.size(); ++ri) recs[ri].acc = e0->replay_acc.get() + acc_off[ri] * kAccStride;
        if (points) CUDA_TRY(cudaMemsetAsync(e0->replay_acc.get(), 0, points * kAccStride * sizeof(unsigned long long), stream));
        std::memcpy(h_recs.data(), recs.data(), sizeof(ReplayWorld) * recs.size());
        if (kf) std::memcpy(h_recs.data() + world_bytes, kf_recs.data(), sizeof(ReplayKeyframes) * kf_recs.size());
        if (tr) std::memcpy(h_recs.data() + world_bytes, tr_recs.data(), sizeof(ReplayTrace) * tr_recs.size());
        CUDA_TRY(cudaMemcpyAsync(d, h_recs.data(), rec_bytes, cudaMemcpyHostToDevice, stream));
        const ReplayWorld* d_recs = reinterpret_cast<const ReplayWorld*>(d);
        const ReplayKeyframes* d_kfs = reinterpret_cast<const ReplayKeyframes*>(d + world_bytes);
        const ReplayTrace* d_trs = reinterpret_cast<const ReplayTrace*>(d + world_bytes);
        uint32_t n_recs = uint32_t(recs.size());
        void* args[] = {&d_recs, &n_recs, &d_kfs};
        void* tr_args[] = {&d_recs, &n_recs, &d_trs, const_cast<TraceMap*>(&tr_map)};
        CUDA_TRY(cudaLaunchKernel(tr ? k.replay_trace_fn : kf ? k.replay_kf_fn : k.replay_fn, dim3(items), dim3(k.threads),
                                  tr ? tr_args : args, 0, stream));
        CUDA_TRY(cudaGetLastError());
        acc.resize(points * kAccStride);
        if (points) CUDA_TRY(cudaMemcpyAsync(acc.data(), e0->replay_acc.get(), points * kAccStride * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        const bool tr_direct = recs.size() == 1;  // one world's samples are contiguous in its dst
        if (tr && staged) {
            const ReplayJob& j0 = *jobs[rec_job[0]];
            uint8_t* to = tr_direct ? static_cast<uint8_t*>(j0.tr->dst) + size_t(j0.tr_done) * j0.tr_stride : nullptr;
            if (!tr_direct) {
                h_tr.resize(staged);
                to = h_tr.data();
            }
            CUDA_TRY(cudaMemcpyAsync(to, tr_stage.get(), staged, cudaMemcpyDeviceToHost, stream));
        }
        CUDA_TRY(cudaStreamSynchronize(stream));
        if (tr) {  // each world's samples to its dst, and the records of the rows the launch's tiles did not reach
            for (size_t ri = 0; ri < recs.size(); ++ri) {
                ReplayJob& job = *jobs[rec_job[ri]];
                const uint32_t m = trs_in(job, cur[rec_job[ri]], seg_end[rec_job[ri]]);
                if (!tr_direct && m)
                    std::memcpy(static_cast<uint8_t*>(job.tr->dst) + size_t(job.tr_done) * job.tr_stride,
                                h_tr.data() + size_t(tr_recs[ri].staging - tr_stage.get()), size_t(m) * job.tr_stride);
                trace_fill_rows(job, job.tr_done, m, uint32_t(std::min<uint64_t>(uint64_t(recs[ri].n_tiles) * kTileRows, UINT32_MAX)));
                job.tr_done += m;
            }
        }
        if (kf) {  // the launch's keyframe images, world by world in frame order, to blobs
            x.im.clear();
            owner.clear();
            for (size_t ri = 0; ri < recs.size(); ++ri) {
                ReplayJob& job = *jobs[rec_job[ri]];
                const ReplayKeyframes& r = kf_recs[ri];
                const uint32_t a = cur[rec_job[ri]], b = seg_end[rec_job[ri]], m = kfs_in(job, a, b);
                for (uint32_t q = 0; q < m; ++q) {
                    x.im.push_back(keyframe_image(job, job.kf_done + q, r.staging + q * r.stride));
                    owner.push_back(&job);
                }
            }
            int rc = keyframes_write(x, owner);
            if (rc != BGR_OK) return rc;
        }
        // each checksum point through the fold bgr_handle_requests uses
        size_t off = 0;
        for (size_t ri = 0; ri < recs.size(); ++ri) {
            const size_t i = rec_job[ri];
            ReplayJob& job = *jobs[i];
            job.e->launches += 1;
            const uint64_t f = first_point(job, cur[i], seg_end[i]);
            for (uint32_t q = 0; q < seg_points[i]; ++q, ++off) {
                const unsigned long long* a = &acc[off * kAccStride];
                const uint32_t j = uint32_t(f + uint64_t(q) * job.r->checksum_interval);
                bgr_partial part;
                std::memset(&part, 0, sizeof part);
                part.frame = int32_t(int64_t(job.c.f0) + j);
                part.n_columns = job.e->n_ck;
                part.active = a[6];
                part.total = rows_at(job, j);
                for (uint32_t col = 0; col < job.e->n_ck; ++col) part.xor_[col] = a[col];
                if ((a[7] & 1ULL) && !job.bad) { job.bad = true; job.bad_frame = part.frame; }
                bgr_checksum cs;
                fold(part, &cs);
                job.sums.push_back(cs);
            }
            cur[i] = seg_end[i];
        }
    }
    for (ReplayJob* j : jobs) j->e->last_kernel = BGR_KERNEL_GENERIC_NVRTC | (uint32_t(k.item_rows) << 16) | kernel_bits;
    return BGR_OK;
}

// After the replay ran on the generated kernel: the engine's host state moves to the end of the log.  Image 0 was written
// outside the bundle kernel's bookkeeping, like a host write: a fresh passive version, a fresh content id, unknown stamps.
int replay_commit(ReplayJob& job) {
    bgr_engine* e = job.e;
    HostState& s = e->st;
    const uint32_t n = job.r->n_frames;
    s.frame_count = job.c.f0 + int32_t(n);
    s.elapsed_ns = job.elapsed_end;
    s.call_count = job.c.call0 + job.c.n_counter * n;
    s.n_rows = uint32_t(job.rows_end);
    s.rng = job.rng;
    s.live_passive_ver = ++s.ver_counter;
    e->ticked = true;
    return clear_stamps(e, 0);
}

// Grows every growable engine its replay needs (each was checked against its ceiling when planned)
int replay_grow(const std::vector<ReplayJob*>& jobs) {
    for (ReplayJob* j : jobs)
        if (j->rows_end > j->e->cfg.max_entities) {
            const int rc = grow_to(j->e, j->rows_end);
            if (rc != BGR_OK) return rc;
        }
    return BGR_OK;
}

// A planned replay of one engine: on the generated kernel when there is one, else in chunks
int replay_run(ReplayJob& job) {
    std::vector<ReplayJob*> one{&job};
    int rc = replay_grow(one);
    if (rc != BGR_OK || job.r->n_frames == 0) return rc;
    const JitKernel* k = replay_kernel(job.e, std::max(1u, job.e->tiles_for(uint32_t(job.rows_end))));
    if (!k || (job.kf && !k->replay_kf_fn) || (job.tr && !k->replay_trace_fn)) return replay_chunked(job);
    rc = replay_launch(*k, one, BGR_KERNEL_REPLAY);
    if (rc != BGR_OK) return rc;
    return replay_commit(job);
}

// The checksums of a finished replay to caller memory and its status
int replay_results(const ReplayJob& job, bgr_checksum* out, uint32_t cap, uint32_t* n_out) {
    if (n_out) *n_out = uint32_t(job.sums.size());
    if (out) std::copy(job.sums.begin(), job.sums.begin() + std::min<size_t>(cap, job.sums.size()), out);
    if (job.bad)
        return fail(BGR_ERR_NON_FINITE, "Hashing is not stable for NaN f32 values (first at the checksum of frame " +
                                            std::to_string(job.bad_frame) + ")");
    return BGR_OK;
}

}  // namespace

BGR_API int bgr_replay(bgr_engine* e, const struct bgr_replay* r, bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out) {
    if (n_out) *n_out = 0;
    NvtxRange span("Replay");
    ReplayJob job;
    int rc = replay_plan(e, r, job);
    if (rc != BGR_OK) return rc;  // nothing executed, nothing changed
    rc = replay_run(job);
    if (rc != BGR_OK) return rc;
    return replay_results(job, checksums_out, cap, n_out);
}

BGR_API int bgr_replay_keyframes(bgr_engine* e, const struct bgr_replay* r, const struct bgr_keyframes* kf,
                                 bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out, uint32_t* n_keyframes_out,
                                 size_t* bytes_out) {
    if (n_out) *n_out = 0;
    if (!kf || !n_keyframes_out || !bytes_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *n_keyframes_out = 0;
    *bytes_out = 0;
    NvtxRange span("Replay");
    ReplayJob job;
    int rc = replay_plan(e, r, job, kf);
    if (rc != BGR_OK) return rc;  // nothing executed, nothing changed
    if (!kf->dst) {               // the query
        *n_keyframes_out = job.n_kf;
        *bytes_out = job.kf_bound;
        return BGR_OK;
    }
    rc = keyframe_caps(job);
    if (rc != BGR_OK) return rc;
    rc = replay_run(job);
    *n_keyframes_out = job.kf_done;
    *bytes_out = job.kf_end;
    if (rc != BGR_OK) return rc;
    return replay_results(job, checksums_out, cap, n_out);
}

BGR_API int bgr_replay_trace(bgr_engine* e, const struct bgr_replay* r, const struct bgr_trace* t,
                             bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out, uint32_t* n_samples_out, size_t* bytes_out) {
    if (n_out) *n_out = 0;
    if (!t || !n_samples_out || !bytes_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *n_samples_out = 0;
    *bytes_out = 0;
    NvtxRange span("Replay");
    ReplayJob job;
    int rc = replay_plan(e, r, job, nullptr, t);
    if (rc != BGR_OK) return rc;  // nothing executed, nothing changed
    *n_samples_out = uint32_t(job.samples.size());
    *bytes_out = job.samples.size() * job.tr_stride;
    if (!t->dst) return BGR_OK;  // the query
    rc = trace_caps(job);
    if (rc != BGR_OK) {
        *n_samples_out = 0;
        *bytes_out = 0;
        return rc;
    }
    std::copy(job.samples.begin(), job.samples.end(), t->samples);
    rc = replay_run(job);
    if (rc != BGR_OK) return rc;
    return replay_results(job, checksums_out, cap, n_out);
}

namespace {

// bgr_batch_replay, with kfs (one per world) bgr_batch_replay_keyframes, with trs (one per world) bgr_batch_replay_trace
int batch_replay(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                 const struct bgr_keyframes* kfs, const struct bgr_trace* trs, bgr_checksum* checksums_out, uint32_t cap,
                 uint32_t* n_checksums_out, uint32_t* n_keyframes_out, uint32_t* n_samples_out, int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (n_worlds && (!worlds || !replays || !n_checksums_out || !status_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("Replay");
    BatchCall call(b, worlds, n_worlds, status_out, checksums_out, cap, n_checksums_out, {n_keyframes_out, n_samples_out});
    // every world is validated and planned before any executes
    std::vector<ReplayJob> jobs(n_worlds);
    for (uint32_t i = 0; i < n_worlds; ++i) {
        int rc = call.check(i);
        if (rc != BGR_OK) return rc;
        rc = replay_plan(b->engines[worlds[i]], &replays[i], jobs[i], kfs ? &kfs[i] : nullptr, trs ? &trs[i] : nullptr);
        if (rc == BGR_OK && kfs) rc = keyframe_caps(jobs[i]);
        if (rc == BGR_OK && trs && i && !feed_same_fields(jobs[i].tp, jobs[0].tp))
            rc = fail(BGR_ERR_INVALID_ARGUMENT, "its trace's fields differ from those of entry 0's trace (a call has one record layout)");
        if (rc == BGR_OK && trs) rc = trace_caps(jobs[i]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    if (trs)  // every world is planned: the sample frames and row counts are known
        for (uint32_t i = 0; i < n_worlds; ++i) std::copy(jobs[i].samples.begin(), jobs[i].samples.end(), trs[i].samples);
    auto results = [&](uint32_t i, int rc) {
        uint32_t n = 0;
        if (rc == BGR_OK) rc = replay_results(jobs[i], call.out(), call.room(), &n);
        if (n_keyframes_out) n_keyframes_out[i] = jobs[i].kf_done;
        if (n_samples_out) n_samples_out[i] = jobs[i].tr_done;
        call.record(i, rc, n);
    };
    if (!b->k.replay_fn || (kfs && !b->k.replay_kf_fn) || (trs && !b->k.replay_trace_fn)) {  // each world's own replay, in list order
        for (uint32_t i = 0; i < n_worlds; ++i) results(i, replay_run(jobs[i]));
        return call.outcome();
    }
    std::vector<ReplayJob*> run;
    for (ReplayJob& j : jobs)
        if (j.r->n_frames) run.push_back(&j);
    int rc = replay_grow(run);
    if (rc == BGR_OK && !run.empty()) rc = replay_launch(b->k, run, BGR_KERNEL_REPLAY | BGR_KERNEL_BATCHED);
    for (ReplayJob* j : run)
        if (rc == BGR_OK) rc = replay_commit(*j);
    if (rc != BGR_OK) return rc;
    for (uint32_t i = 0; i < n_worlds; ++i) results(i, BGR_OK);
    return call.outcome();
}

}  // namespace

BGR_API int bgr_batch_replay(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                             bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_checksums_out, int32_t* status_out) {
    return batch_replay(b, worlds, n_worlds, replays, nullptr, nullptr, checksums_out, cap, n_checksums_out, nullptr, nullptr, status_out);
}

BGR_API int bgr_batch_replay_keyframes(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                                       const struct bgr_keyframes* kfs, bgr_checksum* checksums_out, uint32_t cap,
                                       uint32_t* n_checksums_out, uint32_t* n_keyframes_out, int32_t* status_out) {
    if (n_worlds && (!kfs || !n_keyframes_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    return batch_replay(b, worlds, n_worlds, replays, kfs, nullptr, checksums_out, cap, n_checksums_out, n_keyframes_out, nullptr,
                        status_out);
}

BGR_API int bgr_batch_replay_trace(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                                   const struct bgr_trace* traces, bgr_checksum* checksums_out, uint32_t cap,
                                   uint32_t* n_checksums_out, uint32_t* n_samples_out, int32_t* status_out) {
    if (n_worlds && (!traces || !n_samples_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    return batch_replay(b, worlds, n_worlds, replays, nullptr, traces, checksums_out, cap, n_checksums_out, nullptr, n_samples_out,
                        status_out);
}

// ---- batched checkpoints: the checkpoints of many worlds saved or restored in one pass ----
BGR_API int bgr_batch_checkpoint_save(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const int32_t* frames,
                                      void* dst, size_t dst_cap, bgr_keyframe* index, size_t* bytes_out, int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (!bytes_out || (n_worlds && (!worlds || !frames || !index || !status_out))) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("CheckpointSave");
    *bytes_out = 0;
    BatchCall call(b, worlds, n_worlds, status_out);
    for (uint32_t i = 0; i < n_worlds; ++i) {
        const int rc = call.check(i);
        if (rc != BGR_OK) return rc;
    }
    for (uint32_t i = 0; i < n_worlds; ++i) {  // every member's submitted vectors, their results left queued
        const int rc = drain(b->engines[worlds[i]]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    // one image-table encoder over the held frames of every listed world; its launches count on worlds[0]'s engine
    ImageEncoder x;
    x.e = n_worlds ? b->engines[worlds[0]] : nullptr;
    std::vector<uint32_t> of;  // the list index of each encoded image
    std::vector<bgr_keyframe> idx(n_worlds);  // copied to `index` when the call succeeds
    size_t pos = 0;
    for (uint32_t i = 0; i < n_worlds; ++i) {
        bgr_engine* e = b->engines[worlds[i]];
        bgr_keyframe& k = idx[i];
        k = bgr_keyframe{frames[i], 0u, pos, 0u};
        uint32_t slot = 0;
        if (!p2p_slot(e, frames[i], &slot)) continue;  // held neither queued nor retained: bytes 0
        const uint32_t rows = e->st.slot_rows[slot], n_blocks = e->tiles_for(rows);
        if (!dst) {
            k.bytes = checkpoint_prefix(n_blocks) + size_t(n_blocks) * ckpt_max_block_words(e->words) * 4u;
            pos = align8(pos + k.bytes);
            continue;
        }
        EncodeImage m;
        m.img = e->image(slot + 1);
        m.order_base = e->cfg.order_base;
        m.h = checkpoint_header(e, frames[i], rows, e->st.slot_elapsed_ns[slot], e->st.slot_rng[slot]);
        x.im.push_back(std::move(m));
        of.push_back(i);
    }
    *bytes_out = pos;
    if (dst) {
        int rc = x.e ? encode_measure(x) : BGR_OK;
        if (rc != BGR_OK) return rc;
        pos = 0;  // the exact layout: blobs in list order, each at a multiple of 8
        for (uint32_t i = 0, j = 0; i < n_worlds; ++i) {
            idx[i].offset = pos;
            if (j < of.size() && of[j] == i) {
                idx[i].bytes = blob_bytes(x.im[j]);
                x.im[j++].dst = static_cast<uint8_t*>(dst) + pos;
                pos = align8(pos + idx[i].bytes);
            }
        }
        *bytes_out = pos;
        if (dst_cap < pos)
            return fail(BGR_ERR_CAPACITY, "the checkpoints need " + std::to_string(pos) + " bytes, dst_cap is " + std::to_string(dst_cap));
        if (!x.im.empty()) rc = encode_pack(x);
        if (rc != BGR_OK) return rc;
        if (!x.im.empty()) {  // encode_pack zeroes the padding between blobs; the last one's is zeroed here
            const EncodeImage& last = x.im.back();
            std::memset(last.dst + blob_bytes(last), 0, align8(blob_bytes(last)) - blob_bytes(last));
        }
    }
    std::copy(idx.begin(), idx.end(), index);
    return BGR_OK;
}

BGR_API int bgr_batch_checkpoint_restore(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const void* const* blobs,
                                         const size_t* bytes, int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (n_worlds && (!worlds || !blobs || !bytes || !status_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("CheckpointRestore");
    BatchCall call(b, worlds, n_worlds, status_out);
    std::vector<RestoreBlob> r(n_worlds);
    for (uint32_t i = 0; i < n_worlds; ++i) {  // the host checks, in list order
        int rc = call.check(i);
        if (rc != BGR_OK) return rc;
        rc = restore_check(b->engines[worlds[i]], blobs[i], bytes[i], &r[i]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    if (n_worlds == 0) return BGR_OK;
    RestorePass x;
    size_t bad = n_worlds;
    int rc = restore_decode(r, x, &b->h_ckpt, &bad);
    if (rc == BGR_OK) rc = restore_commit(r, x, &bad);
    if (rc != BGR_OK) return bad < n_worlds ? call.fail_at(uint32_t(bad), rc) : rc;
    return BGR_OK;
}

// ---- batched change feed: the feeds of many batch members reported in one pass (change_feed.cuh, feed_check.hpp) ----
BGR_API int bgr_batch_feed_begin(bgr_batch* b, const bgr_batch_feed* reports, uint32_t n, void* host_dst, uint32_t* ticket_out,
                                 int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (!ticket_out || (n && (!reports || !status_out))) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("FeedReport");
    BatchCall call(b, reports, n, status_out);
    bgr_batch::FeedScratch& x = b->feed;
    if (x.busy) return fail(BGR_ERR_STATE, "a batched feed report of this batch is in flight: call bgr_batch_feed_wait first");
    uint32_t bad = 0;
    std::string why;
    const int rc = feed_batch_check(b->list, reports, n, [b](uint32_t w, uint32_t f) {
        const bgr_engine* e = b->engines[w];
        return f < BGR_MAX_FEEDS && e->feeds[f].used ? FeedView{&e->feeds[f].p, e->feeds[f].busy} : FeedView{nullptr, false};
    }, &bad, &why);
    if (rc != BGR_OK) return call.fail_at(bad, fail(rc, why));
    bool any_cap = false;
    for (uint32_t i = 0; i < n; ++i) any_cap = any_cap || reports[i].records_cap;
    uint32_t* host_dev = any_cap ? (host_dst ? mapped_host(host_dst) : nullptr) : nullptr;
    if (any_cap && !host_dev) return fail(BGR_ERR_INVALID_ARGUMENT, "host_dst must come from bgr_host_alloc");
    // every allocation before any feed changes: the table, the scratch, the staging, the infos
    CUDA_TRY(x.h_table.ensure(std::max(1u, n)));
    FeedWorld* tab = x.h_table.get();
    for (uint32_t i = 0; i < n; ++i) {
        bgr_engine* e = b->engines[reports[i].world];
        const bgr_engine::Feed& fd = e->feeds[reports[i].feed];
        tab[i] = FeedWorld{e->image(0), fd.rep.ptr(), e->st.n_rows, e->tiles_for(std::max(e->st.n_rows, fd.bound)), 0u, 0u};
    }
    uint64_t stage_records = 0;
    const uint32_t tiles = feed_layout(tab, reports, n, &stage_records);
    const FeedParams reg = n ? b->engines[reports[0].world]->feeds[reports[0].feed].p : FeedParams{};
    CUDA_TRY(x.table.ensure(std::max(1u, n)));
    CUDA_TRY(x.counts.ensure(3ull * tiles + 6ull * n + 2u));
    CUDA_TRY(x.out.ensure(std::max<uint64_t>(1u, stage_records * reg.record_words)));
    CUDA_TRY(x.h_info.ensure(4ull * std::max(1u, n)));
    CUDA_TRY(x.packed.ensure());
    CUDA_TRY(x.done.ensure());
    if (!x.copy) CUDA_TRY(cudaStreamCreateWithFlags(&x.copy, cudaStreamNonBlocking));
    for (uint32_t i = 0; i < n; ++i) {  // stream-ordered behind every queued submit, like the passes below
        const int r = touch_live(b->engines[reports[i].world]);
        if (r != BGR_OK) return call.fail_at(i, r);
    }
    if (n) {
        CUDA_TRY(cudaMemcpyAsync(x.table.get(), tab, sizeof(FeedWorld) * n, cudaMemcpyHostToDevice, b->stream));
        FeedParams p = reg;
        p.worlds = x.table.get();
        p.n_worlds = n;
        p.n_tiles = tiles;
        p.tile_count = x.counts.get();
        p.tile_off = p.tile_count + tiles;
        p.tile_list = p.tile_off + tiles;
        p.world_scan = p.tile_list + tiles;
        p.info = p.world_scan + 2u * n;
        p.head = p.info + 4u * n;
        p.out = x.out.get();
        const int r = feed_report(b->engines[reports[0].world], p, host_dev, x.copy, x.packed.get(), x.done.get(), x.h_info.get());
        if (r != BGR_OK) return r;
        for (bgr_engine* e : b->engines) e->tiledep_chain = false;  // the passes ran on the shared stream
        for (uint32_t i = 0; i < n; ++i) feed_started(b->engines[reports[i].world], reports[i].feed, tab[i].rows);
    }
    x.listed.assign(reports, reports + n);
    x.busy = true;
    x.seq = (x.seq + 1u) & 0x7FFFFFFFu;
    x.ticket = x.seq + 1u;
    *ticket_out = x.ticket;
    return BGR_OK;
}

BGR_API int bgr_batch_feed_wait(bgr_batch* b, uint32_t ticket, bgr_feed_info* infos) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    bgr_batch::FeedScratch& x = b->feed;
    if (!x.busy || ticket != x.ticket) return fail(BGR_ERR_STATE, "no such batched feed report in flight");
    if (!x.listed.empty()) CUDA_TRY(cudaEventSynchronize(x.done.get()));
    x.busy = false;
    for (const bgr_batch_feed& r : x.listed) b->engines[r.world]->feeds[r.feed].busy = false;
    if (infos) std::memcpy(infos, x.h_info.get(), sizeof(bgr_feed_info) * x.listed.size());
    return BGR_OK;
}

// ---- batched host edits: the bgr_apply_edits batches of many batch members in one call (edit_batch.hpp) ----
BGR_API int bgr_batch_apply_edits(bgr_batch* b, const bgr_batch_edits* entries, uint32_t n, int32_t* status_out) {
    if (!b) return fail(BGR_ERR_INVALID_ARGUMENT, "null batch");
    if (n && (!entries || !status_out)) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    NvtxRange span("ApplyEdits");
    BatchCall call(b, entries, n, status_out);
    // the host checks of every entry, then every fold, before anything runs
    std::vector<uint64_t> rows(n);
    uint32_t bad = 0;
    std::string why;
    int rc = edit_batch_check(b->list, entries, n,
        [b](uint32_t w, const bgr_batch_edits& x, uint64_t* r, std::string* err) {
            const int s = validate_edits(b->engines[w], x.edits, x.n_edits, x.values_bytes, r);
            if (s != BGR_OK) *err = g_err;
            return s;
        },
        [b](uint32_t w) { return uint64_t(b->engines[w]->st.n_rows); }, [b](uint32_t w) { return uint64_t(b->engines[w]->ceiling); },
        rows.data(), &bad, &why);
    if (rc != BGR_OK) return call.fail_at(bad, fail(rc, why));
    std::vector<EditCounts> counts(n);
    for (uint32_t i = 0; i < n; ++i) {
        bgr_engine* e = b->engines[entries[i].world];
        EditFold& f = e->edit_fold;  // each member folds into its own scratch
        f.clear();
        if (entries[i].n_edits) {
            rc = fold_edits(e, entries[i].edits, entries[i].n_edits, static_cast<const uint8_t*>(entries[i].values), f);
            if (rc != BGR_OK) return call.fail_at(i, rc);
            assert(f.stamps.empty() && "batch members never run the bundle kernel, so they have no content stamps");
        }
        counts[i] = EditCounts{f.words.size(), f.masks.size(), e->st.n_rows, uint32_t(rows[i] - e->st.n_rows)};
    }
    EditLayout L;
    rc = edit_layout(counts.data(), n, &L, &bad, &why);
    if (rc != BGR_OK) return call.fail_at(bad, fail(rc, why));
    if (n == 0) return BGR_OK;
    // every buffer, then growth, then the listed worlds' deferred live images, stream-ordered behind the queued submits
    bgr_engine::EditStage& sg = b->edit_stage[b->next_edit];
    rc = take_edit_stage(sg, L.bytes);
    if (rc != BGR_OK) return rc;
    const size_t table_bytes = L.bytes - L.off_patch;
    if (table_bytes) CUDA_TRY(b->edit_tables.ensure(table_bytes));
    for (uint32_t i = 0; i < n; ++i) {
        bgr_engine* e = b->engines[entries[i].world];
        if (rows[i] > e->st.n_rows) rc = grow_to(e, rows[i]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    for (uint32_t i = 0; i < n; ++i) {
        if (entries[i].n_edits) rc = touch_live(b->engines[entries[i].world]);
        if (rc != BGR_OK) return call.fail_at(i, rc);
    }
    // the staging: every world's words and masks at its offsets, then the two tables
    uint8_t* h = sg.h.get();
    uint4* hw = reinterpret_cast<uint4*>(h);
    for (size_t k = 0; k < L.patch.size(); ++k) {
        EditWorld& w = L.patch[k];
        const EditFold& f = b->engines[entries[L.patch_entry[k]].world]->edit_fold;
        w.img = b->engines[entries[L.patch_entry[k]].world]->image(0);
        for (size_t j = 0; j < f.words.size(); ++j) hw[w.word0 + j] = make_uint4(f.words[j].row, f.words[j].plane, f.words[j].value, 0u);
        if (!f.masks.empty()) std::memcpy(h + L.off_masks + size_t(w.mask0) * sizeof(uint2), f.masks.data(), f.masks.size() * sizeof(uint2));
    }
    for (size_t k = 0; k < L.spawn.size(); ++k) L.spawn[k].img = b->engines[entries[L.spawn_entry[k]].world]->image(0);
    if (!L.patch.empty()) std::memcpy(h + L.off_patch, L.patch.data(), L.patch.size() * sizeof(EditWorld));
    if (!L.spawn.empty()) std::memcpy(h + L.off_spawn, L.spawn.data(), L.spawn.size() * sizeof(SpawnWorld));
    // one table upload and at most two launches, counted on the first listed world
    bgr_engine* e0 = b->engines[entries[0].world];
    uint8_t* d_tab = b->edit_tables.get();
    if (table_bytes) CUDA_TRY(cudaMemcpyAsync(d_tab, h + L.off_patch, table_bytes, cudaMemcpyHostToDevice, b->stream));
    const uint32_t words = e0->words;  // one registration: one row stride
    if (L.n_spawned) {
        const SpawnWorld* d_spawn = reinterpret_cast<const SpawnWorld*>(d_tab + (L.off_spawn - L.off_patch));
        k_spawn_rows<true><<<e0->grid_for(L.n_spawned, 64), 256, 0, b->stream>>>(nullptr, words, 0u, L.n_spawned, d_spawn,
                                                                                  uint32_t(L.spawn.size()));
        e0->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    if (L.n_words + L.n_masks) {
        const uint8_t* dev = sg.h.dev();
        EditPatch p{};
        p.words = reinterpret_cast<const uint4*>(dev);
        p.masks = reinterpret_cast<const uint2*>(dev + L.off_masks);
        p.n_words = L.n_words; p.n_masks = L.n_masks;
        p.worlds = reinterpret_cast<const EditWorld*>(d_tab);
        p.n_worlds = uint32_t(L.patch.size());
        k_apply_edits<true><<<e0->grid_for(L.n_words + L.n_masks, 256), 256, 0, b->stream>>>(nullptr, words, nullptr, p);
        e0->launches += 1;
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaEventRecord(sg.done.get(), b->stream));
    sg.busy = true;
    b->next_edit = (b->next_edit + 1) % bgr_engine::kEditBufs;
    for (bgr_engine* e : b->engines) e->tiledep_chain = false;  // the launches ran on the shared stream
    for (uint32_t i = 0; i < n; ++i) {  // commit, as apply_edits does
        if (!entries[i].n_edits) continue;
        bgr_engine* e = b->engines[entries[i].world];
        e->st.n_rows = uint32_t(rows[i]);
        if (e->edit_fold.bump) e->st.live_passive_ver = ++e->st.ver_counter;
        e->st.cids.live = e->st.cids.fresh(e->st.n_rows);
    }
    return BGR_OK;
}

BGR_API int bgr_save_world(bgr_engine* e, bgr_checksum* checksum_out) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    bgr_request rq;
    std::memset(&rq, 0, sizeof rq);
    rq.kind = BGR_REQ_SAVE; rq.frame = e->st.frame_count;
    uint32_t n = 0;
    return bgr_handle_requests(e, nullptr, &rq, 1, checksum_out, checksum_out ? 1 : 0, &n);
}

BGR_API int bgr_load_world(bgr_engine* e) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    bgr_request rq;
    std::memset(&rq, 0, sizeof rq);
    rq.kind = BGR_REQ_LOAD; rq.frame = e->st.frame_count;
    uint32_t n = 0;
    return bgr_handle_requests(e, nullptr, &rq, 1, nullptr, 0, &n);
}

BGR_API int bgr_advance_world(bgr_engine* e, const uint8_t* inputs, const uint8_t* status, uint32_t n_players) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (n_players > BGR_MAX_PLAYERS) return fail(BGR_ERR_INVALID_ARGUMENT, "n_players > BGR_MAX_PLAYERS");
    bgr_request rq;
    std::memset(&rq, 0, sizeof rq);
    rq.kind = kReqAdvanceNoBump; rq.n_players = n_players;
    for (uint32_t i = 0; i < n_players; ++i) { rq.inputs[i] = inputs ? inputs[i] : 0; rq.status[i] = status ? status[i] : 0; }
    uint32_t n = 0;
    return bgr_handle_requests(e, nullptr, &rq, 1, nullptr, 0, &n);
}

BGR_API int bgr_last_partials(bgr_engine* e, bgr_partial* out, uint32_t cap, uint32_t* n_out) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    for (uint32_t i = 0; i < e->last_partials.size() && i < cap && out; ++i) out[i] = e->last_partials[i];
    if (n_out) *n_out = uint32_t(e->last_partials.size());
    return BGR_OK;
}

BGR_API int bgr_fold_partials(const bgr_partial* combined, bgr_checksum* out) {
    if (!combined || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    fold(*combined, out);
    return BGR_OK;
}

BGR_API int bgr_collect_partials(bgr_engine* e, bgr_partial* partials_out, uint32_t cap, uint32_t* n_out) {
    uint32_t n = 0;
    int rc = collect(e, nullptr, 0, &n);
    if (rc != BGR_OK) return rc;
    for (uint32_t i = 0; i < n && i < cap && partials_out; ++i) partials_out[i] = e->last_partials[i];
    if (n_out) *n_out = n;
    return BGR_OK;
}

BGR_API int bgr_fold_partials_n(const bgr_partial* combined, uint32_t n, bgr_checksum* out) {
    if ((!combined || !out) && n) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    for (uint32_t i = 0; i < n; ++i) fold(combined[i], &out[i]);
    return BGR_OK;
}

BGR_API uint64_t bgr_seahash(const void* bytes, uint64_t len) {
    const uint8_t* p = static_cast<const uint8_t*>(bytes);
    uint64_t a = kSeaA, b = kSeaB, c = kSeaC, d = kSeaD;
    uint64_t i = 0;
    for (; i + 8 <= len; i += 8) {
        uint64_t w;
        std::memcpy(&w, p + i, 8);  // little-endian host
        uint64_t t = sea_diffuse(a ^ w);
        a = b; b = c; c = d; d = t;
    }
    if (i < len) {
        uint64_t w = 0;
        std::memcpy(&w, p + i, size_t(len - i));
        a = sea_diffuse(a ^ w);
    }
    return sea_diffuse(a ^ b ^ c ^ d ^ len);
}

// the engine's ParticleRng arithmetic on its own (host only): known-answer tests of SplitMix64 / xoshiro256++ / the
// f32 range sampling run against exactly the code that spawn_particles uses
BGR_API int bgr_particle_rng_stream(uint64_t seed, const uint64_t* state4_or_null, uint32_t n, uint64_t* next_u64_out,
                                    float* range_out, float low, float high) {
    ParticleRng a, b;
    if (state4_or_null) { for (int i = 0; i < 4; ++i) a.s[i] = b.s[i] = state4_or_null[i]; }
    else { a.seed_from_u64(seed); b.seed_from_u64(seed); }
    for (uint32_t i = 0; i < n; ++i) {
        if (next_u64_out) next_u64_out[i] = a.next_u64();
        if (range_out) range_out[i] = b.random_range(low, high);
    }
    return BGR_OK;
}
BGR_API int bgr_splitmix64_stream(uint64_t seed, uint32_t n, uint64_t* out) {
    if (!out && n) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    SplitMix64 sm{seed};
    for (uint32_t i = 0; i < n; ++i) out[i] = sm.next_u64();
    return BGR_OK;
}

BGR_API uint32_t bgr_ggrs_time_delta_bits(uint32_t fps, int32_t frame) {
    if (fps == 0) return 0;
    uint64_t f = uint64_t(int64_t(frame));
    uint64_t now = f * 1000000000ULL / fps, prev = (f - 1) * 1000000000ULL / fps;
    return f32_bits(duration_as_secs_f32(now - prev));
}

BGR_API int bgr_launch_count(bgr_engine* e, uint64_t* out) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = e->launches; return BGR_OK;
}
BGR_API int bgr_slot_bytes(bgr_engine* e, uint64_t* out) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *out = uint64_t(e->st.n_rows) * (uint64_t(e->words) * 4u + 1u); return BGR_OK;
}
BGR_API int bgr_generic_specialised(bgr_engine* e, uint32_t* specialised_out) {
    if (!e || !specialised_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *specialised_out = e->jit.fn ? 1u : 0u;
    return BGR_OK;
}
BGR_API int bgr_last_path(bgr_engine* e, uint32_t* fused_out) {
    if (!e || !fused_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *fused_out = e->last_fused ? 1u : 0u; return BGR_OK;
}
BGR_API int bgr_last_kernel(bgr_engine* e, uint32_t* kernel_out) {
    if (!e || !kernel_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *kernel_out = e->last_kernel; return BGR_OK;
}
BGR_API int bgr_held_saves(bgr_engine* e, uint64_t* out, uint32_t cap) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    uint64_t v[3] = {e->last_held, e->held_total, 0};
    if (e->held_check.get()) {
        CUDA_TRY(cudaMemcpyAsync(&v[2], e->held_check.get(), sizeof v[2], cudaMemcpyDeviceToHost, e->stream));
        CUDA_TRY(cudaStreamSynchronize(e->stream));
    }
    for (uint32_t i = 0; i < cap && i < 3; ++i) out[i] = v[i];
    return BGR_OK;
}
BGR_API int bgr_synchronize(bgr_engine* e) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    return BGR_OK;
}


// ---- shard group (multi-GPU cross-shard exchange inside the engine; shard_group.hpp) ----
BGR_API int bgr_shard_group_join(bgr_engine* e, const char* name, uint32_t rank, uint32_t world_size, uint32_t timeout_ms) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    if (!name || !*name) return fail(BGR_ERR_INVALID_ARGUMENT, "null group name");
    if (!(e->cfg.flags & BGR_CFG_SHARDED)) return fail(BGR_ERR_STATE, "only a BGR_CFG_SHARDED engine can join a shard group");
    if (e->group) return fail(BGR_ERR_STATE, "engine is already in a shard group");
    if (!e->pending.empty()) return fail(BGR_ERR_STATE, "collect every submitted request vector before joining a shard group");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    auto* g = new ShardGroup();
    if (timeout_ms) g->timeout_ms = timeout_ms;
    std::string err;
    const uint32_t block_words = uint32_t(kResultStride);
    static_assert(bgr_engine::kBufs == int(kGroupBufs) && kMaxSaves == int(kGroupMaxSaves) && kAccStride == int(kGroupAccStride),
                  "shard_group.hpp mirrors the engine's result block layout");
    if (!g->join(name, rank, world_size, block_words, e->seq, &err)) { delete g; return fail(BGR_ERR_STATE, err); }
    // the block area becomes page-locked and visible to this GPU: the fused kernel's last block stores its result rows there
    cudaError_t ce = cudaHostRegister(g->blocks_base(), g->blocks_bytes(), cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (ce != cudaSuccess) { delete g; return fail(BGR_ERR_CUDA, std::string("cudaHostRegister(shard group segment): ") + cudaGetErrorString(ce)); }
    for (int b = 0; b < bgr_engine::kBufs; ++b) {
        e->h_out[b] = reinterpret_cast<unsigned long long*>(g->block(rank, uint32_t(b)));
        void* dp = nullptr;
        ce = cudaHostGetDevicePointer(&dp, e->h_out[b], 0);
        if (ce != cudaSuccess) {
            use_own_blocks(e);
            cudaHostUnregister(g->blocks_base());
            delete g;
            return fail(BGR_ERR_CUDA, std::string("cudaHostGetDevicePointer: ") + cudaGetErrorString(ce));
        }
        e->d_out[b] = static_cast<unsigned long long*>(dp);
    }
    e->group = g;
    e->gseq = 0;
    e->next_buf = 0;
    return BGR_OK;
}

BGR_API int bgr_shard_group_leave(bgr_engine* e) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (!e->group) return BGR_OK;
    if (!e->pending.empty()) return fail(BGR_ERR_STATE, "collect every submitted request vector before leaving the shard group");
    cudaSetDevice(e->cfg.device);
    cudaStreamSynchronize(e->stream);
    leave_group(e);
    return BGR_OK;
}

// the group's host logic on its own (no GPU): CPU tests drive join / publish / collect with a stand-in for the kernel's publish
struct bgr_group { ShardGroup g; uint32_t n_columns = 0; };
BGR_API bgr_group* bgr_group_join(const char* name, uint32_t rank, uint32_t world_size, uint32_t n_columns, uint32_t timeout_ms) {
    if (!name) { fail(BGR_ERR_INVALID_ARGUMENT, "null group name"); return nullptr; }
    auto* h = new bgr_group();
    h->n_columns = n_columns;
    if (timeout_ms) h->g.timeout_ms = timeout_ms;
    std::string err;
    if (!h->g.join(name, rank, world_size, uint32_t(kResultStride), 0, &err)) { fail(BGR_ERR_STATE, err); delete h; return nullptr; }
    return h;
}
BGR_API void bgr_group_leave(bgr_group* h) { delete h; }
BGR_API int bgr_group_publish(bgr_group* h, uint64_t gseq, const bgr_partial* partials, uint32_t n) {
    if (!h || (!partials && n) || gseq == 0 || n > uint32_t(kMaxSaves)) return fail(BGR_ERR_INVALID_ARGUMENT, "bad argument");
    std::string err;
    if (!h->g.wait_reusable(gseq, &err)) return fail(BGR_ERR_STATE, err);
    int32_t frames[kMaxSaves]; uint32_t totals[kMaxSaves];
    for (uint32_t k = 0; k < n; ++k) { frames[k] = partials[k].frame; totals[k] = uint32_t(partials[k].total); }
    h->g.publish_meta(gseq, n, h->n_columns, frames, totals);
    h->g.publish_block_from_host(gseq, partials, n);
    return BGR_OK;
}
BGR_API int bgr_group_collect(bgr_group* h, uint64_t gseq, bgr_checksum* out, uint32_t cap, uint32_t* n_out) {
    if (!h || gseq == 0) return fail(BGR_ERR_INVALID_ARGUMENT, "bad argument");
    bgr_partial combined[kMaxSaves];
    uint32_t n = 0;
    uint64_t flags = 0;
    std::string err;
    if (!h->g.combine(gseq, combined, kMaxSaves, &n, &flags, &err)) return fail(BGR_ERR_STATE, err);
    for (uint32_t k = 0; k < n && k < cap && out; ++k) fold(combined[k], &out[k]);
    if (n_out) *n_out = n;
    return BGR_OK;
}

// No session (schedule_systems.rs:70-79): "reset time data and snapshots" — the frame resources go back to their
// session-less values; the caller (run_ggrs_schedules' mirror) also clears LocalPlayers and its accumulator.
BGR_API int bgr_reset_session(bgr_engine* e) {
    if (!e) return fail(BGR_ERR_INVALID_ARGUMENT, "null engine");
    if (!e->pending.empty()) return fail(BGR_ERR_STATE, "collect every submitted request vector first");
    const int rc = materialize_live(e);
    if (rc != BGR_OK) return rc;
    e->st.frame_count = 0;        // RollbackFrameCount(0)
    e->st.confirmed = -1;         // ConfirmedFrameCount(-1)
    e->st.has_maxpred = true;     // MaxPredictionWindow(8)
    e->st.maxpred = 8;
    e->st.ring.release_witnesses();  // a new session compares nothing against the old one's first images
    e->st.ring.release_retained();   // ... and reports no desync of the old one's frames
    return BGR_OK;
}

BGR_API int bgr_host_profile(bgr_engine* e, uint64_t* out, uint32_t cap) {
    if (!e || !out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    for (uint32_t i = 0; i < cap && i < 8; ++i) out[i] = e->prof[i];
    return BGR_OK;
}

BGR_API int bgr_stream(bgr_engine* e, void** stream_out) {
    if (!e || !stream_out) return fail(BGR_ERR_INVALID_ARGUMENT, "null argument");
    *stream_out = e->stream;
    return BGR_OK;
}

// Device-side launch trace: every fused launch records when its first block started and when its last block
// finished (ns of the GPU's globaltimer) — the evidence for overlapping consecutive ticks (DESIGN.md) when no
// system profiler is available.  Two atomics per block; off unless enabled.
BGR_API int bgr_trace_enable(bgr_engine* e, uint32_t capacity) {
    if (!e || !e->built) return fail(BGR_ERR_STATE, "engine not built");
    int rc = drain(e);
    if (rc != BGR_OK) return rc;
    e->trace = {};  // a new trace starts empty, at exactly its capacity
    e->trace_cap = 0;
    if (capacity == 0) return BGR_OK;
    std::vector<unsigned long long> init(size_t(capacity) * 4, 0ULL);
    for (uint32_t i = 0; i < capacity; ++i) init[4 * i] = ~0ULL;
    CUDA_TRY(e->trace.ensure(init.size()));
    CUDA_TRY(cudaMemcpy(e->trace.get(), init.data(), init.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
    e->trace_cap = capacity;
    e->trace_first_seq = e->seq + 1;
    return BGR_OK;
}
BGR_API int bgr_trace_read(bgr_engine* e, uint64_t* start_end_ns_out, uint32_t cap, uint32_t* n_out) {
    if (!e || !e->trace.get()) return fail(BGR_ERR_STATE, "trace not enabled");
    int rc = drain(e);
    if (rc != BGR_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(e->stream));
    const uint64_t done = e->seq + 1 > e->trace_first_seq ? e->seq + 1 - e->trace_first_seq : 0;
    const uint32_t n = uint32_t(std::min<uint64_t>(std::min<uint64_t>(done, e->trace_cap), cap));
    if (n && start_end_ns_out) CUDA_TRY(cudaMemcpy(start_end_ns_out, e->trace.get(), size_t(n) * 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    if (n_out) *n_out = n;
    return BGR_OK;
}

// ---- host-side ring bookkeeping on its own (pure host logic; used by the "not gpu" KAT tests) ----
struct bgr_ring { SlotRing r; };
BGR_API bgr_ring* bgr_ring_create(uint32_t n_slots) { auto* r = new bgr_ring(); r->r.reset(n_slots); return r; }
BGR_API void bgr_ring_destroy(bgr_ring* r) { delete r; }
BGR_API uint32_t bgr_ring_depth(bgr_ring* r) { return r->r.depth(); }
BGR_API int bgr_ring_set_depth(bgr_ring* r, uint32_t depth) { r->r.set_depth(depth); return BGR_OK; }
BGR_API int bgr_ring_push(bgr_ring* r, int32_t frame, uint32_t* slot_out) {
    uint32_t s = r->r.push(frame);
    if (s == SlotRing::kNoSlot) return fail(BGR_ERR_CAPACITY, "ring out of slots");
    if (slot_out) *slot_out = s;
    return BGR_OK;
}
BGR_API int bgr_ring_confirm(bgr_ring* r, int32_t frame) { r->r.confirm(frame); return BGR_OK; }
BGR_API int bgr_ring_rollback(bgr_ring* r, int32_t frame, uint32_t* slot_out) {
    std::string err;
    if (!r->r.rollback(frame, &err)) return fail(BGR_ERR_NO_SNAPSHOT, err);
    uint32_t s = 0;
    r->r.get(&s, nullptr);
    if (slot_out) *slot_out = s;
    return BGR_OK;
}
BGR_API int bgr_ring_get(bgr_ring* r, uint32_t* slot_out) {
    std::string err;
    uint32_t s = 0;
    if (!r->r.get(&s, &err)) return fail(BGR_ERR_NO_SNAPSHOT, err);
    if (slot_out) *slot_out = s;
    return BGR_OK;
}
BGR_API int bgr_ring_peek(bgr_ring* r, int32_t frame, uint32_t* slot_out, int32_t* found) {
    uint32_t s = 0;
    bool ok = r->r.peek(frame, &s);
    if (found) *found = ok ? 1 : 0;
    if (ok && slot_out) *slot_out = s;
    return BGR_OK;
}
BGR_API bgr_ring* bgr_ring_create_capture(uint32_t n_slots) { auto* r = new bgr_ring(); r->r.reset(n_slots, true); return r; }
BGR_API int bgr_ring_first(bgr_ring* r, int32_t frame, uint32_t* slot_out, int32_t* found) {
    uint32_t s = 0;
    bool ok = r->r.first(frame, &s);
    if (found) *found = ok ? 1 : 0;
    if (ok && slot_out) *slot_out = s;
    return BGR_OK;
}
BGR_API int bgr_ring_slots_in_use(bgr_ring* r, uint32_t* n_out) {
    if (n_out) *n_out = r->r.slots_in_use();
    return BGR_OK;
}
BGR_API int bgr_ring_set_retention(bgr_ring* r, uint32_t interval, uint32_t count) {
    if (count && interval == 0) return fail(BGR_ERR_INVALID_ARGUMENT, "retention needs interval >= 1");
    r->r.set_retention(interval, count);
    return BGR_OK;
}
BGR_API int bgr_ring_retained(bgr_ring* r, int32_t* frames_out, uint32_t cap, uint32_t* n_out) {
    std::vector<int32_t> f;
    r->r.retained_frames(&f);
    for (uint32_t i = 0; i < f.size() && i < cap && frames_out; ++i) frames_out[i] = f[i];
    if (n_out) *n_out = uint32_t(f.size());
    return BGR_OK;
}

}  // extern "C"
