/*
 * bevy_ggrs_b200 — C ABI of the H100-native rollback snapshot / checksum / re-simulation engine.
 *
 * This is the drop-in boundary for ONE hot path of gschup/bevy_ggrs (reference paths are
 * relative to the upstream repo, v0.20.0):
 *
 *   - per-tick save/load of the registered component columns       src/snapshot/component_snapshot.rs:66-123
 *   - the newest-first ring of frame snapshots                      src/snapshot/mod.rs:94-271
 *   - the per-frame desync checksum                                 src/snapshot/{checksum,component_checksum,entity_checksum}.rs
 *   - the request loop that replays N frames after a rollback       src/schedule_systems.rs:170-289 (handle_requests)
 *   - the registered stress-test systems of GgrsSchedule            examples/stress_tests/particles.rs:272-289
 *
 * Everything lives in HBM: registered columns are stored word-planar (one plane of 4-byte
 * words per field word, see DESIGN.md "Data layout"), snapshots are a ring of frame slots
 * with the same layout, and a whole Vec<GgrsRequest> ( Load + N x (Advance, Save) + ... )
 * is executed by ONE kernel launch.  GGRS never receives state bytes
 * (`cell.save(frame, None, checksum)`, schedule_systems.rs:235-236), so the only things that
 * cross this boundary per tick are the request list (in) and one u128 checksum per Save (out).
 *
 * Conventions
 *   - plain C, fixed-width ints, no torch / CUDA types in signatures (a cudaStream_t is
 *     passed as void*).
 *   - every call returns a bgr_status; on failure bgr_last_error() holds the text of the
 *     panic the reference would have raised (e.g. "Could not rollback to 99: no snapshot at
 *     that moment could be found.", mod.rs:209-212).  A Rust shim turns non-zero into panic!.
 *   - one caller thread at a time per engine (the reference calls from an exclusive system,
 *     schedule_systems.rs:19,170).
 *   - u128 checksums cross as two u64 (lo, hi); hi is always 0 in the reference because every
 *     part is `u64 as u128` (component_checksum.rs:95, entity_checksum.rs:43).
 *   - the library FAILS LOUDLY (BGR_ERR_CUDA) when no sm_90 device is usable; there is no
 *     CPU fallback anywhere behind this header.
 */
#ifndef BEVY_GGRS_B200_H
#define BEVY_GGRS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BGR_API __attribute__((visibility("default")))

#define BGR_ABI_VERSION 1u
#define BGR_MAX_PLAYERS 8u      /* every handle 0..7 reaches the systems (PlayerInputs<T>.0[handle], box_game.rs:171) */
#define BGR_MAX_REQUESTS 80u  /* max requests per bgr_handle_requests call (2*32+2 for a 32-frame SyncTest) */

typedef enum bgr_status {
    BGR_OK = 0,
    BGR_ERR_INVALID_ARGUMENT = 1,
    BGR_ERR_STATE = 2,            /* call order violated (e.g. register after build) */
    BGR_ERR_CUDA = 3,             /* no usable GPU / CUDA runtime failure — never falls back to CPU */
    BGR_ERR_NO_SNAPSHOT = 4,      /* GgrsSnapshots::rollback / get panic, mod.rs:207-230 */
    BGR_ERR_MISSING_RESOURCE = 5, /* `expect(...)` on RollbackFrameCount / LocalInputs, schedule_systems.rs:90-92,245-246 */
    BGR_ERR_NON_FINITE = 6,       /* assert!(is_finite) in the stress hashers, particles.rs:111-114,212-215 */
    BGR_ERR_CAPACITY = 7,         /* more rows / slots / requests than configured */
    BGR_ERR_UNSUPPORTED = 8
} bgr_status;

/* Strategy<T> (src/snapshot/strategy.rs:22-83).  Copy and Clone of a POD are both a bitwise
 * copy; ReflectStrategy is out of scope (boxed dynamic reflection, SURVEY.md §2 row 5). */
typedef enum bgr_strategy { BGR_STRATEGY_COPY = 0, BGR_STRATEGY_CLONE = 1 } bgr_strategy;
/* OR into `strategy`: single entities may lose / regain this component inside the rollback window
 * (`Option<&mut S::Target>` in ComponentSnapshotPlugin::load, src/snapshot/component_snapshot.rs:99-115).  Save stores
 * the component only for the entities that have it, Load updates / removes / inserts / leaves alone accordingly, the
 * checksum and the GgrsSchedule systems only see entities that have it.  At most BGR_MAX_OPTIONAL_COLUMNS columns. */
#define BGR_STRATEGY_OPTIONAL 0x100u
#define BGR_MAX_OPTIONAL_COLUMNS 7

/* How `checksum_component::<T>(hasher)` hashes one element (rollback_app.rs:227-232,
 * component_checksum.rs:44-48).  BGR_HASH_BYTES = seahash over elem[offset .. offset+len):
 * this is what `#[derive(Hash)]` produces for a POD of ints (fields appended little-endian)
 * and what the particles hashers do with `x.to_bits()` (particles.rs:107-120, 207-222). */
typedef enum bgr_hash_kind { BGR_HASH_NONE = 0, BGR_HASH_BYTES = 1 } bgr_hash_kind;
#define BGR_HASH_FLAG_ASSERT_FINITE_F32 1u /* every 4-byte word in the range must be a finite f32 */

/* Systems that can be added to GgrsSchedule (`add_systems(GgrsSchedule, ...)`, lib.rs:73-74).
 * User closures cannot cross a C ABI; the systems the hot path needs are compiled in. */
typedef enum bgr_system {
    /* update_particles, particles.rs:272-280.  cols = {Transform(40B), Velocity(12B)} */
    BGR_SYS_PARTICLES_UPDATE = 1,
    /* despawn_particles, particles.rs:282-289.  cols = {Ttl(8B)} */
    BGR_SYS_PARTICLES_DESPAWN = 2,
    /* move_cube_system, box_game.rs:154-206.  cols = {Transform(40B), Velocity(12B)}; player handle = row */
    BGR_SYS_BOX_MOVE = 3,
    /* `x.0 += k` on a u32 field (tests/component_rollback.rs:25-29 increment_score).
     * cols = {C}; params = {byte_offset, k} */
    BGR_SYS_U32_ADD = 4,
    /* `h = h.saturating_sub(k); if h == 0 { despawn }` (tests/synctest.rs:38-45 decrease_health).
     * cols = {C}; params = {byte_offset, k} */
    BGR_SYS_U32_SATSUB_DESPAWN = 5,
    /* writes a host-side call counter that is NOT rolled back into a u32 field — the
     * deliberately non-deterministic system of tests/synctest.rs:83-125.
     * cols = {C}; params = {byte_offset} */
    BGR_SYS_U32_STORE_CALL_COUNT = 6,
    /* spawn_particles.run_if(spawn_pressed), particles.rs:243-270: when any player's input has INPUT_SPAWN
     * (1 << 4) set, appends `rate` rows: Transform::default(), Velocity(random_range(-200..200) x2, 0), Ttl(ttl),
     * Rollback.  Draws from the ParticleRng resource (Xoshiro256PlusPlus::seed_from_u64(seed)), which the engine
     * keeps host-side and rolls back with every snapshot (rollback_resource_with_clone::<ParticleRng>, :200).
     * Commands are deferred: the new rows exist from the end of the frame on and are not updated in it.  Every other
     * registered word of a new row is zero and every optional column is present.  A spawning world ticks in one launch
     * (the particles bundle, or the generic one-launch program for any other registration) and can be batched.
     * cols = {Transform(40B), Velocity(12B), Ttl(8B)}; params = {rate, ttl, seed_lo, seed_hi} */
    BGR_SYS_PARTICLES_SPAWN = 7,
    /* `if inputs[player].0 == value { commands.entity(e).despawn() }` for every entity that has component C — the
     * shape of tests/hierarchy.rs:36-45 delete_child_system (there the child is reached through the parent's `Children`;
     * here C is the child's own `ChildOf`, an optional 8-byte column holding the parent's RollbackOrdered index: row
     * indices are stable across rollback, so the hierarchy needs neither ChildOfSnapshotPlugin's remapping
     * (childof_snapshot.rs) nor MapEntities (component_map.rs)).  cols = {C}; params = {player_handle, value} */
    BGR_SYS_DESPAWN_ON_INPUT = 8
} bgr_system;
#define BGR_INPUT_SPAWN 0x10u /* INPUT_SPAWN, particles.rs:75 */

/* GgrsRequest<T> (ggrs; consumed at schedule_systems.rs:222-269). Input type is u8
 * (particles.rs:73 `GgrsConfig<u8>`, box_game.rs:27-29 `BoxInput(u8)`). */
typedef enum bgr_request_kind { BGR_REQ_SAVE = 0, BGR_REQ_LOAD = 1, BGR_REQ_ADVANCE = 2 } bgr_request_kind;
typedef enum bgr_input_status { BGR_INPUT_CONFIRMED = 0, BGR_INPUT_PREDICTED = 1, BGR_INPUT_DISCONNECTED = 2 } bgr_input_status;

typedef struct bgr_request {
    uint32_t kind;                    /* bgr_request_kind */
    int32_t frame;                    /* SaveGameState{frame} / LoadGameState{frame}; ignored for Advance */
    uint32_t n_players;               /* AdvanceFrame{inputs}.len() */
    uint8_t inputs[BGR_MAX_PLAYERS];  /* PlayerInputs<T>.0[i].0 */
    uint8_t status[BGR_MAX_PLAYERS];  /* PlayerInputs<T>.0[i].1 (bgr_input_status) */
} bgr_request;

/* What handle_requests reads from the Session each request (schedule_systems.rs:195-220). */
typedef enum bgr_session_kind {
    BGR_SESSION_NONE = 0, BGR_SESSION_SYNCTEST = 1, BGR_SESSION_P2P = 2, BGR_SESSION_SPECTATOR = 3
} bgr_session_kind;

typedef struct bgr_session_info {
    uint32_t kind;            /* bgr_session_kind */
    uint32_t max_prediction;  /* s.max_prediction() (forced to 0 for spectators, :200) */
    uint32_t check_distance;  /* SyncTest: s.check_distance() (:207) */
    int32_t confirmed_frame;  /* P2P: s.confirmed_frame() (:205) */
} bgr_session_info;

/* `Checksum(u128)` (checksum.rs:49) handed to `cell.save(frame, None, checksum)`. */
typedef struct bgr_checksum {
    int32_t frame;
    uint32_t has_checksum;  /* always 1 (ChecksumPlugin is part of GgrsPlugin, lib.rs:257) */
    uint64_t lo, hi;
} bgr_checksum;

/* Raw per-Save partials of ONE shard, before the cross-shard fold (multi-GPU, SURVEY §8e):
 * xor[c] is the XOR over live rows of the per-entity hash of checksummed column c
 * (component_checksum.rs:81-90, before the final `result.hash()` at :93); active = live rows. */
#define BGR_MAX_CHECKSUM_COLUMNS 6u
typedef struct bgr_partial {
    int32_t frame;
    uint32_t n_columns;
    uint64_t active;      /* active_entities.iter().len() of this shard, entity_checksum.rs:38 */
    uint64_t total;       /* rollback_ordered.len() of this shard, entity_checksum.rs:41 */
    uint64_t xor_[BGR_MAX_CHECKSUM_COLUMNS];
} bgr_partial;

typedef struct bgr_config {
    uint32_t abi_version;   /* BGR_ABI_VERSION */
    int32_t device;         /* CUDA ordinal */
    uint32_t max_entities;  /* row capacity of this shard; with BGR_CFG_GROWABLE the initial capacity (bgr_capacity) */
    uint32_t max_depth;     /* frame slots allocated in HBM; >= the largest MaxPredictionWindow used (+1 for SyncTest d == p-1 is not needed) */
    uint32_t fps;           /* RollbackFrameRate, time.rs:19-26 (default 60) */
    uint32_t flags;         /* BGR_CFG_* */
    uint64_t order_base;    /* RollbackOrdered index of local row 0 (entity-range sharding); 0 on one GPU */
    void* stream;           /* cudaStream_t to run on; NULL = engine creates its own */
} bgr_config;
#define BGR_CFG_FORCE_STEPWISE 1u  /* never use the fused one-launch program kernel (debug / A-B tests) */
#define BGR_CFG_SHARDED 2u         /* handle_requests returns partials only; caller folds across shards */
/* Accepted and ignored; kept so that code naming it still compiles.  Every engine now skips word planes whose content
 * is provably identical to what the target image already holds: it tracks a content version for the planes no
 * registered system writes (e.g. Transform.rotation/scale in the stress test), and a Save into a slot that already
 * holds the current version stores none of them, nor does a Load from it.  Snapshots stay complete images (peek, load,
 * desync capture and digests read the same bytes) and every observable result is what the reference's clone of every
 * registered component on every save (component_snapshot.rs:71-75) gives; only redundant HBM traffic is elided. */
#define BGR_CFG_SKIP_UNCHANGED_PLANES 4u
/* OPT-IN, off by default: keep the first-recorded image of every frame so a SyncTest mismatch can be inspected
 * (bgr_desync_*, below).  bgr_build allocates 2*max_depth frame slots instead of max_depth; the ring hands a frame's
 * first slot out again only once the frame is confirmed, evicted from the old end, or bgr_reset_session runs, or when
 * a Save finds no free slot: then the first images recorded earliest are released until one is free, so capture never
 * makes a Save fail.  A SyncTest never runs short (it needs at most 2*(check_distance+1) <= 2*max_depth slots); deep
 * P2P rollbacks can.  Loads, checksums, bgr_peek, bgr_snapshot_frames and the kernels launched are unchanged.  Needs
 * max_depth <= 32; not with BGR_CFG_SHARDED. */
#define BGR_CFG_DESYNC_CAPTURE 8u
/* OPT-IN: max_entities is the initial capacity; row-creating calls grow it.  RollbackOrdered only ever appends
 * (rollback.rs:66-83), so a spawning world grows for the whole session.  A request vector whose spawns do not fit,
 * bgr_spawn, bgr_run_startup_system and bgr_reserve grow the capacity to max(rows needed, 2 x capacity), rounded up to
 * whole 512-row tiles and to the memory mapping granularity and clamped to the ceiling.  bgr_build reserves virtual
 * address space for the ceiling and maps memory for the capacity; growing maps more under every image and zeroes it, so
 * no image moves, nothing in flight has to finish, and checksums, snapshots, feeds and desync reports are those of an
 * engine created with the grown capacity.  Column writes never grow the capacity.  A call that needs more rows than
 * the ceiling fails with BGR_ERR_CAPACITY and executes nothing.  Not with BGR_CFG_SHARDED or order_base != 0
 * (BGR_ERR_UNSUPPORTED at bgr_engine_create). */
#define BGR_CFG_GROWABLE 16u

typedef struct bgr_engine bgr_engine;

/* ---- lifetime ------------------------------------------------------------------------ */
BGR_API uint32_t bgr_abi_version(void);
BGR_API const char* bgr_last_error(void);  /* thread-local text of the last failure */
BGR_API int bgr_engine_create(const bgr_config* cfg, bgr_engine** out);
BGR_API void bgr_engine_destroy(bgr_engine* e);

/* ---- registration  (RollbackApp, src/snapshot/rollback_app.rs:31-248) ------------------ */
/* rollback_component_with_copy::<T>() / rollback_component_with_clone::<T>() (:157-183) */
BGR_API int bgr_rollback_component(bgr_engine* e, const char* type_name, uint32_t elem_bytes,
                                   uint32_t strategy, uint32_t* column_out);
/* checksum_component::<T>(hasher) / checksum_component_with_hash::<T>() (:199-232) */
BGR_API int bgr_checksum_component(bgr_engine* e, uint32_t column, uint32_t hash_kind,
                                   uint32_t byte_offset, uint32_t byte_len, uint32_t flags);
/* add_systems(GgrsSchedule, system) — systems run in insertion order each AdvanceFrame */
BGR_API int bgr_add_system(bgr_engine* e, uint32_t system, const uint32_t* columns, uint32_t n_columns,
                           const uint32_t* params, uint32_t n_params);
/* end of App::build: allocates live columns + max_depth frame slots in HBM */
BGR_API int bgr_build(bgr_engine* e);
/* add_systems(Startup, system): run a registered GgrsSchedule system once, outside the rollback loop
 * (particles.rs:232 `add_systems(Startup, spawn_particles)` — the initial burst).  Only BGR_SYS_PARTICLES_SPAWN. */
BGR_API int bgr_run_startup_system(bgr_engine* e, uint32_t system);
/* Capacity >= rows on return (BGR_CFG_GROWABLE; after bgr_build).  At or below the capacity: no-op.  Above it on an
 * engine without the flag: BGR_ERR_UNSUPPORTED; above the ceiling: BGR_ERR_CAPACITY, nothing changes. */
BGR_API int bgr_reserve(bgr_engine* e, uint32_t rows);
/* Rows the engine holds without growing, and the most it can ever hold (== capacity without BGR_CFG_GROWABLE). */
BGR_API int bgr_capacity(bgr_engine* e, uint32_t* capacity_out, uint32_t* ceiling_out);

/* ---- entity population (Rollback marker, src/snapshot/rollback.rs:23-94) ---------------- */
/* `commands.spawn((..., Rollback))` x count: appends rows, RollbackOrdered index = order_base + row */
BGR_API int bgr_spawn(bgr_engine* e, uint32_t count, uint32_t* first_row_out);
BGR_API int bgr_despawn(bgr_engine* e, uint32_t row);
BGR_API int bgr_row_count(bgr_engine* e, uint32_t* rows_out);   /* RollbackOrdered::len() */
BGR_API int bgr_active_count(bgr_engine* e, uint64_t* active_out);
/* ECS column <-> HBM planes.  host buffers are arrays of T with `stride` bytes between
 * elements (stride >= elem_bytes; stride = size_of::<T>() on the Rust side). */
BGR_API int bgr_write_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count,
                                const void* host_src, uint32_t stride);
BGR_API int bgr_read_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count,
                               void* host_dst, uint32_t stride);
BGR_API int bgr_read_alive(bgr_engine* e, uint32_t first_row, uint32_t count, uint8_t* host_dst);

/* ---- per-entity component presence (columns registered with BGR_STRATEGY_OPTIONAL) ----------
 * bgr_remove_component = `commands.entity(e).remove::<T>()`, bgr_insert_component = `.insert(value)` applied to the live
 * world between request vectors (value: elem_bytes bytes); bgr_has_component writes 1 per row that is alive and has it. */
BGR_API int bgr_remove_component(bgr_engine* e, uint32_t column, uint32_t row);
BGR_API int bgr_insert_component(bgr_engine* e, uint32_t column, uint32_t row, const void* value);
BGR_API int bgr_has_component(bgr_engine* e, uint32_t column, uint32_t first_row, uint32_t count, uint8_t* host_dst);

/* ---- host edits: a batch of live-world changes in one queued launch -----------------------------------------------
 * What a game does to rollback entities outside GgrsSchedule (an Update system setting Transform.translation,
 * commands.entity(e).despawn() / insert / remove, spawning with Rollback), applied to the live world as one batch.  A
 * batch is observably identical to issuing its records in order through the single calls:
 *   BGR_EDIT_WRITE   bytes [byte_offset, byte_offset+byte_len) of `column` on rows [row, row+count), a read-modify-write of
 *                    each element through bgr_write_component.  Row k's bytes are values[value_offset + k*byte_len ...].
 *                    byte_offset is a multiple of 4; byte_len > 0 is a multiple of 4 or ends at the element's end (the
 *                    element's tail word is zero-padded, as bgr_write_component pads it).
 *   BGR_EDIT_INSERT  bgr_insert_component(column, row, values + value_offset): the whole element, written whatever the
 *                    row's state, then present if the row is alive.
 *   BGR_EDIT_REMOVE  bgr_remove_component(column, row).
 *   BGR_EDIT_DESPAWN bgr_despawn(row): later presence records of the row change nothing.
 *   BGR_EDIT_SPAWN   bgr_spawn(count): appends `count` rows; later records of the batch may address them.
 * Fields a kind does not name are ignored.  Later records win where records overlap.  Every row must be below the row
 * count at that point of the batch (bgr_row_count, which counts the rows of queued request vectors, plus the batch's
 * earlier spawns).  The whole batch is validated before anything runs: a bad kind, column, optional-ness, field range
 * or value range (against values_bytes) is BGR_ERR_INVALID_ARGUMENT; spawns past max_entities are BGR_ERR_CAPACITY (or
 * grow a BGR_CFG_GROWABLE engine, past its ceiling BGR_ERR_CAPACITY); spawning after the first request vector on a
 * BGR_CFG_SHARDED engine or with order_base != 0 is BGR_ERR_UNSUPPORTED.  A refused batch changes nothing.
 * The call is ordered behind every submitted request vector on the engine stream and does not wait for them: it copies
 * the batch into the engine's own page-locked staging (the caller's buffers are free on return) and waits only when
 * every staging buffer still belongs to an unfinished earlier batch.  Each of the 4 staging buffers grows to the
 * largest patch it has held (16 bytes per stored word, plus 8 per row with presence records) and keeps that
 * page-locked memory until bgr_engine_destroy; the call that grows one waits for the device, because releasing
 * page-locked memory does.  Send a whole column with bgr_write_component instead.  Un-collected submits keep their
 * results.  Unlike
 * the single calls it keeps the skip records precise: only the content stamps of the (64-row segment, active plane)
 * pairs it changes become unknown, and the passive-plane version moves only for spawns, presence changes and writes
 * that touch a passive plane.  n == 0 does nothing. */
typedef enum bgr_edit_kind {
    BGR_EDIT_WRITE = 0,
    BGR_EDIT_INSERT = 1,
    BGR_EDIT_REMOVE = 2,
    BGR_EDIT_DESPAWN = 3,
    BGR_EDIT_SPAWN = 4
} bgr_edit_kind;
typedef struct bgr_edit {
    uint32_t kind;          /* bgr_edit_kind */
    uint32_t column;        /* WRITE, INSERT, REMOVE */
    uint32_t row;           /* WRITE (first row), INSERT, REMOVE, DESPAWN */
    uint32_t count;         /* WRITE: rows; SPAWN: rows appended */
    uint32_t byte_offset;   /* WRITE */
    uint32_t byte_len;      /* WRITE */
    uint32_t value_offset;  /* WRITE, INSERT: into `values` */
    uint32_t reserved;
} bgr_edit;
BGR_API int bgr_apply_edits(bgr_engine* e, const bgr_edit* edits, uint32_t n, const void* values, size_t values_bytes);

/* ---- asynchronous mirror download: what the ECS side reads back every tick -----------------
 * In the reference the world lives in host memory and everything after GgrsSchedule (rendering via Transform,
 * examples/stress_tests/particles.rs:191-196; game logic outside the rollback schedule) reads it there.  With the
 * world in HBM the shim mirrors only the fields those readers need: bytes [byte_offset, byte_offset+byte_len) of
 * every element of `column` for rows [first_row, first_row+count), packed densely (byte_len bytes per row) into
 * `host_dst`.  byte_offset and byte_len must be multiples of 4.
 *
 * bgr_download_begin is ordered after every request vector submitted so far (it sees the live world those leave
 * behind), returns without waiting for the GPU, and does not delay later submits: the fields are packed into a device
 * staging buffer on the engine's stream and cross PCIe on a separate copy stream.  `host_dst` should come from
 * bgr_host_alloc (page-locked); it must not be read before bgr_download_wait(ticket) returns.  At most
 * BGR_MAX_DOWNLOADS may be in flight. */
#define BGR_MAX_DOWNLOADS 4
BGR_API int bgr_host_alloc(size_t bytes, void** out);
BGR_API int bgr_host_free(void* p);
BGR_API int bgr_download_begin(bgr_engine* e, uint32_t column, uint32_t byte_offset, uint32_t byte_len,
                               uint32_t first_row, uint32_t count, void* host_dst, uint32_t* ticket_out);
BGR_API int bgr_download_wait(bgr_engine* e, uint32_t ticket);

/* ---- change feed: only the live rows that changed since the host was last told --------------------------------------
 * A feed tracks up to BGR_MAX_FEED_FIELDS fields (bytes [byte_offset, byte_offset+byte_len) of `column`, both multiples
 * of 4, inside the element) and keeps in HBM, per row, the state and field bytes it last reported; initially, and after
 * bgr_feed_reset, every row is (state 0, zero bytes).  A report lists, in ascending row order, exactly the rows whose
 * current (state, bytes) differs bit for bit from the reported one, and makes those the reported state.  A record is
 * record_bytes = 8 + sum of byte_len bytes:
 *   u32 row;
 *   u32 state: bit 0 = the row exists (row < RollbackOrdered::len() and alive); bit 1+k = it exists and field k's column
 *              is present (its absent bit is clear);
 *   the bytes of every field in order, zero where the field is not present.
 * Rows at or past the row count do not exist, whatever stale bytes image 0 holds there: rows a rollback un-spawned are
 * reported with state 0.  When more than records_cap rows differ, the lowest records_cap are reported, `pending` counts
 * the others and the next report picks them up: the records of capped reports concatenate to those of one uncapped
 * report when nothing ran in between.
 * bgr_feed_begin is ordered after every request vector submitted so far, materialises a deferred live image like
 * bgr_download_begin, returns without waiting for the GPU and does not delay later submits: both passes run on the
 * engine stream and only n_records * record_bytes cross PCIe, on a separate copy stream.  `host_dst` (records_cap *
 * record_bytes bytes) must come from bgr_host_alloc and must not be read before bgr_feed_wait(ticket) returns.  One
 * report per feed may be in flight (BGR_ERR_STATE otherwise).  Feeds are created after bgr_build (BGR_ERR_STATE before);
 * a bad field is BGR_ERR_INVALID_ARGUMENT, too many feeds or fields BGR_ERR_CAPACITY; an unknown or already-waited
 * ticket is BGR_ERR_STATE. */
#define BGR_MAX_FEEDS 8u
#define BGR_MAX_FEED_FIELDS 8u
typedef struct bgr_feed_field { uint32_t column, byte_offset, byte_len; } bgr_feed_field;
typedef struct bgr_feed_info {
    uint32_t n_records;     /* records written, <= records_cap */
    uint32_t pending;       /* rows that differed but were not reported because of the cap */
    uint32_t rows;          /* RollbackOrdered::len() of the live world that was compared */
    uint32_t record_bytes;  /* 8 + sum of byte_len */
} bgr_feed_info;
BGR_API int bgr_feed_create(bgr_engine* e, const bgr_feed_field* fields, uint32_t n_fields, uint32_t* feed_out);
BGR_API int bgr_feed_reset(bgr_engine* e, uint32_t feed);  /* forget what was reported: the next report lists every existing row */
BGR_API int bgr_feed_begin(bgr_engine* e, uint32_t feed, void* host_dst, uint32_t records_cap, uint32_t* ticket_out);
BGR_API int bgr_feed_wait(bgr_engine* e, uint32_t ticket, bgr_feed_info* info);

/* ---- frame resources (src/snapshot/mod.rs:66-77, lib.rs:116-117) ------------------------ */
BGR_API int bgr_rollback_frame_count(bgr_engine* e, int32_t* out);
BGR_API int bgr_set_rollback_frame_count(bgr_engine* e, int32_t frame);
BGR_API int bgr_confirmed_frame_count(bgr_engine* e, int32_t* out);
BGR_API int bgr_max_prediction_window(bgr_engine* e, uint32_t* out);
/* the session-less branch of run_ggrs_schedules (schedule_systems.rs:70-79): RollbackFrameCount(0),
 * ConfirmedFrameCount(-1), MaxPredictionWindow(8) */
BGR_API int bgr_reset_session(bgr_engine* e);

/* ---- snapshot ring (GgrsSnapshots, src/snapshot/mod.rs:94-271) -------------------------- */
BGR_API int bgr_set_depth(bgr_engine* e, uint32_t depth);                 /* :120-135 */
BGR_API int bgr_confirm(bgr_engine* e, int32_t confirmed_frame);          /* :182-199 */
BGR_API int bgr_snapshot_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out); /* newest first */
/* peek(frame) (:233-240): *found = 0 if no snapshot for `frame`; otherwise copies the rows. */
BGR_API int bgr_peek(bgr_engine* e, int32_t frame, uint32_t column, uint32_t first_row, uint32_t count,
                     void* host_dst, uint32_t stride, uint8_t* alive_dst, int32_t* found);

/* ---- desync capture (engines created with BGR_CFG_DESYNC_CAPTURE; BGR_ERR_STATE otherwise) ----------------------
 * The reference can only say WHICH frames mismatched (SyncTestMismatch, lib.rs:131-137); docs/debugging-desyncs.md
 * ("Known Limitations") notes the diverging snapshot cannot be inspected.  Here the first-recorded image of a frame
 * ("first", what ggrs compared against) and its current ring image ("latest", the re-simulation) are compared in HBM
 * with the keyed-map semantics of component_snapshot.rs:99-115:
 *   - row r exists in an image iff r < that image's RollbackOrdered::len() and the entity was alive;
 *   - existence difference: the row exists in exactly one image (record: column = word = 0xFFFFFFFF);
 *   - presence difference: exists in both, an optional column's absent bit differs (record: word = 0xFFFFFFFF);
 *   - word difference: exists in both, column present in both, a 4-byte word of the element differs.
 * Existence / presence records carry the two per-row mask bytes (bit 0 alive, bit 1+k optional column k absent;
 * 0 for a row that does not exist) in first / latest; word records carry the two words.  Records come in ascending
 * (row, column, word) order; only the first records_cap are returned.  Like every entry point that reads the world,
 * these wait for submitted vectors and leave their results queued for bgr_collect. */
#define BGR_DESYNC_NO_INDEX 0xFFFFFFFFu
typedef struct bgr_desync_column {
    uint32_t rows;              /* rows with a word difference in this column */
    uint32_t rows_in_checksum;  /* ... of which a differing word overlaps the column's checksummed byte range */
    uint32_t presence;          /* rows with a presence difference in this column */
    uint32_t reserved;
} bgr_desync_column;
typedef struct bgr_desync_record { uint32_t row, column, word, first, latest; } bgr_desync_record;
typedef struct bgr_desync_summary {
    int32_t frame;
    uint32_t rows_first, rows_latest;                 /* RollbackOrdered::len() captured by each image */
    uint32_t rows_differing, existence_differing;     /* rows with any difference; rows that exist in one image only */
    uint32_t host_state_differs;                      /* bit 0 ParticleRng, bit 1 Time<GgrsTime> */
    uint64_t words_differing;                         /* differing words over all rows and columns */
    uint64_t elapsed_ns_first, elapsed_ns_latest;     /* Time<GgrsTime>::elapsed captured by each image */
} bgr_desync_summary;
/* frames that have a first-recorded image AND a later save into a different slot, newest first */
BGR_API int bgr_desync_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out);
/* *found = 0 when `frame` lacks a retained first image or a current ring entry.  cols[c] for c < cols_cap;
 * *n_records = records written (<= records_cap). */
BGR_API int bgr_desync_diff(bgr_engine* e, int32_t frame, bgr_desync_summary* summary, bgr_desync_column* cols,
                            uint32_t cols_cap, bgr_desync_record* records, uint32_t records_cap, uint32_t* n_records,
                            int32_t* found);
/* bgr_peek, but of the first-recorded image of `frame` */
BGR_API int bgr_peek_first(bgr_engine* e, int32_t frame, uint32_t column, uint32_t first_row, uint32_t count,
                           void* host_dst, uint32_t stride, uint8_t* alive_dst, int32_t* found);

/* ---- P2P desync reports (any built engine without BGR_CFG_SHARDED) ---------------------------------------------
 * Serves GGRS's `GgrsEvent::DesyncDetected { frame, local_checksum, remote_checksum, addr }`, raised by a P2P session
 * with `DesyncDetection::On { interval }` when the checksums two peers computed for the confirmed frame
 * 0, interval, 2*interval, ... differ (docs/debugging-desyncs.md:61-71).  The reference cannot inspect that frame: its
 * snapshot was pruned when the frame was confirmed, and the other image lives on another machine ("Known
 * Limitations", :73-76).  Here:
 *   1. bgr_retain_confirmed keeps the last `count` frames f >= 0, f % interval == 0 after they leave the ring from the
 *      old end (confirmed or evicted for depth), in `count` extra frame slots.  Loads, checksums, bgr_peek and
 *      bgr_snapshot_frames are unchanged; bgr_launch_count can only be lower (a depth-1 ring no longer writes a
 *      deferred live image early because the next Save reuses its base slot).  bgr_reset_session releases them.
 *   2. bgr_frame_digest hashes a queued or retained frame per block of BGR_DIGEST_BLOCK_ROWS rows into n_columns + 1
 *      u64 words (~62 KB at 1M rows of the stress schema).  The peers exchange digests over the game's own channel
 *      (GGRS carries no application messages; the engine does no networking) and bgr_digest_mismatch lists the blocks
 *      that differ.
 *   3. The peer exports those of the blocks it has, the ones below its digest's n_blocks (bgr_frame_export, the tiles
 *      as stored, BGR_DIGEST_BLOCK_ROWS * (4*words + 1) B each; possibly none), and the local side diffs them against
 *      its own image (bgr_desync_diff_remote, which also compares the local blocks the peer's frame does not have): the
 *      records and summary of bgr_desync_diff, with "first" = the local image and "latest" = the remote one.
 * Digest of block b, for C registered columns (word c < C per column, word C for existence and presence); rows r of
 * the block with r < rows whose alive bit is set "exist":
 *   word c = XOR over existing rows holding column c (absent bit clear) of
 *            seahash_2xu64(order_base + r, seahash(element bytes [0, elem_bytes)))   (component_checksum.rs:81-90)
 *   word C = XOR over existing rows of seahash_2xu64(order_base + r, mask byte)
 * For a column whose checksummed range is the whole element, the XOR of its word over all blocks is the frame's
 * per-column checksum partial (bgr_partial.xor_).  The digest is a wire format between peers: the block size is fixed
 * here, not by the engine's tile size. */
#define BGR_DIGEST_BLOCK_ROWS 512u
typedef struct bgr_frame_digest_header {
    uint64_t layout;       /* seahash fingerprint of what makes two images comparable: word planes per row and, per
                              column, elem_bytes, first plane, words, optional or not and the checksummed byte range,
                              and bgr_config.order_base (registered systems are not part of it) */
    int32_t frame;
    uint32_t rows;         /* RollbackOrdered::len() captured with the frame */
    uint32_t n_blocks;     /* ceil(rows / BGR_DIGEST_BLOCK_ROWS) */
    uint32_t n_columns;
    uint64_t active;       /* alive rows */
    uint64_t elapsed_ns;   /* Time<GgrsTime>::elapsed captured with the frame */
    uint64_t rng[4];       /* ParticleRng state captured with the frame (zero without BGR_SYS_PARTICLES_SPAWN) */
    uint64_t root;         /* seahash over the n_blocks * (n_columns + 1) words, in order */
} bgr_frame_digest_header;
/* Export blob: this header, then per exported block a u32 block index, a u32 zero and the block's tile bytes as
 * stored (BGR_DIGEST_BLOCK_ROWS * (4 * words + 1) B: the word planes, then the mask bytes).  The bytes of rows >= rows
 * are zeroed, so stale memory never leaves the machine.  `reserved` and the u32 after each block index are zero; a
 * blob with anything else there is refused, so later versions can give them a meaning. */
#define BGR_FRAME_BLOB_MAGIC 0x50424752u /* "RGBP" */
#define BGR_FRAME_BLOB_VERSION 1u
typedef struct bgr_frame_blob_header {
    uint32_t magic;        /* BGR_FRAME_BLOB_MAGIC */
    uint32_t version;      /* BGR_FRAME_BLOB_VERSION */
    uint64_t layout;       /* bgr_frame_digest_header.layout */
    int32_t frame;
    uint32_t rows;
    uint32_t words;        /* word planes per row */
    uint32_t n_blocks;     /* blocks of the whole frame */
    uint32_t n_exported;   /* blocks that follow, ascending */
    uint32_t reserved;     /* 0 */
    uint64_t elapsed_ns;
    uint64_t rng[4];
} bgr_frame_blob_header;
/* Before bgr_build: retain `count` >= 1 confirmed frames that are multiples of `interval` >= 1.  bgr_build then
 * allocates max_depth (2 * max_depth with BGR_CFG_DESYNC_CAPTURE) + count frame slots, at most 64.
 * BGR_ERR_STATE after bgr_build, BGR_ERR_UNSUPPORTED on a BGR_CFG_SHARDED engine. */
BGR_API int bgr_retain_confirmed(bgr_engine* e, uint32_t interval, uint32_t count);
/* retained frames, the most recently retained first */
BGR_API int bgr_retained_frames(bgr_engine* e, int32_t* frames_out, uint32_t cap, uint32_t* n_out);
/* Digest of `frame`, looked up among the queued snapshots first, then the retained ones (*found = 0: neither).
 * Writes the header and the first min(words_cap, n_blocks * (n_columns + 1)) words; a buffer of
 * ceil(max_entities / BGR_DIGEST_BLOCK_ROWS) * (n_columns + 1) words always suffices.  Waits for submitted vectors and
 * leaves their results queued, like bgr_desync_diff. */
BGR_API int bgr_frame_digest(bgr_engine* e, int32_t frame, bgr_frame_digest_header* header, uint64_t* words, uint32_t words_cap,
                             int32_t* found);
/* Host only, the one place the digest format is interpreted.  Refuses (BGR_ERR_INVALID_ARGUMENT) digests of different
 * layouts, frames or column counts.  Lists, ascending, the blocks whose words differ and the blocks only one side has
 * (the first `cap`; *n_out = how many there are).  *host_state_differs: bit 0 rng, bit 1 elapsed_ns (the bits of
 * bgr_desync_summary.host_state_differs), state the block words cannot show. */
BGR_API int bgr_digest_mismatch(const bgr_frame_digest_header* local_header, const uint64_t* local_words,
                                const bgr_frame_digest_header* remote_header, const uint64_t* remote_words, uint32_t* blocks_out,
                                uint32_t cap, uint32_t* n_out, uint32_t* host_state_differs);
/* Writes the blob of blocks[0..n_blocks) (ascending, each < the frame's block count) of `frame` (queued or retained;
 * *found = 0: neither) to dst.  *bytes = the blob's size; dst == NULL only reports the size.  BGR_ERR_CAPACITY if
 * dst_cap is smaller. */
BGR_API int bgr_frame_export(bgr_engine* e, int32_t frame, const uint32_t* blocks, uint32_t n_blocks, void* dst,
                             size_t dst_cap, size_t* bytes, int32_t* found);
/* Diffs the blob's blocks against the same blocks of the local image of `frame` (queued or retained; *found = 0:
 * neither) with the k_desync_* kernels of bgr_desync_diff: first = local, latest = remote; rows_latest, elapsed_ns_latest
 * and host_state_differs come from the blob header.  The local blocks at or past the blob's n_blocks are compared too:
 * the peer has none of their rows, so every existing row there is an existence difference, and the blob need not (and
 * cannot: bgr_frame_export refuses them) carry them.  Rows of other blocks the blob does not carry are not compared.  The
 * blob is input from another machine: a bad magic, version or layout, another frame, a truncated or overlong blob, a
 * block index >= its n_blocks, or an unsorted or duplicate block list is refused with BGR_ERR_INVALID_ARGUMENT. */
BGR_API int bgr_desync_diff_remote(bgr_engine* e, int32_t frame, const void* blob, size_t bytes,
                                   bgr_desync_summary* summary, bgr_desync_column* cols, uint32_t cols_cap,
                                   bgr_desync_record* records, uint32_t records_cap, uint32_t* n_records, int32_t* found);

/* ---- world checkpoints (any built engine without BGR_CFG_SHARDED) -----------------------------------------------
 * A checkpoint is everything a match consists of at one saved frame: the image of every registered column, the row
 * count, each optional column's presence, RollbackFrameCount, Time<GgrsTime> and ParticleRng.  Restoring it into an
 * engine of the same registration layout (bgr_frame_digest_header.layout) and fps continues the match bit for bit, on
 * any kernel and capacity.  The registered SYSTEMS are not part of the layout (as for digests): a world restored into
 * an engine with other systems simulates with those systems.
 * Blob: this header, then u64 offsets[n_blocks + 1], then payload_bytes of payload.  Offsets count bytes into the
 * payload, start at 0, end at payload_bytes, never decrease and are multiples of 4; block b (rows [512b, 512b + 512))
 * occupies payload bytes [offsets[b], offsets[b+1]) and holds words + 1 vectors: vectors 0 .. words-1 are the block's
 * word planes (512 u32 each), vector `words` its mask bytes read as 128 little-endian u32.  A block starts with one kind
 * byte per vector, zero-padded to a multiple of 4, followed by the vectors' bodies in order; for n elements:
 *   BGR_CKPT_CONST  (0)  one u32: every element equals it;
 *   BGR_CKPT_SPARSE (1)  n/32 u32 bitmap (bit i of word j set iff element 32j+i is non-zero), then the non-zero elements
 *                        in ascending order;
 *   BGR_CKPT_RAW    (2)  n u32.
 * The encoded tile is canonical: a word of row r in a plane of column c is zero unless r < rows, the row's alive bit is
 * set and c's absent bit is clear; a mask byte is zero unless the row exists.  The kind is CONST if all elements are
 * equal, else SPARSE if nnz < n - n/32, else RAW.  So the blob is a pure function of the frame's content: two engines
 * whose digests agree produce byte-identical checkpoints. */
#define BGR_CHECKPOINT_MAGIC 0x43524742u /* "BGRC" */
#define BGR_CHECKPOINT_VERSION 1u
#define BGR_CKPT_CONST 0u
#define BGR_CKPT_SPARSE 1u
#define BGR_CKPT_RAW 2u
typedef struct bgr_checkpoint_header {  /* 104 bytes, no padding */
    uint32_t magic;          /* BGR_CHECKPOINT_MAGIC */
    uint32_t version;        /* BGR_CHECKPOINT_VERSION */
    uint64_t layout;         /* bgr_frame_digest_header.layout: same registration layout and order_base */
    int32_t frame;
    uint32_t rows;           /* RollbackOrdered::len() of the frame */
    uint32_t words;          /* word planes per row */
    uint32_t n_blocks;       /* ceil(rows / 512) */
    uint32_t n_columns;
    uint32_t fps;            /* bgr_config.fps: elapsed_ns is only continuable at the same rate */
    uint64_t active;         /* existing rows */
    uint64_t elapsed_ns;     /* Time<GgrsTime> of the frame */
    uint64_t rng[4];         /* ParticleRng of the frame */
    uint64_t digest_root;    /* bgr_frame_digest_header.root of the frame */
    uint64_t payload_bytes;
} bgr_checkpoint_header;
/* Encodes `frame` (queued or retained; *found = 0: neither) on the GPU.  dst == NULL: *bytes = an upper bound (every
 * vector RAW), nothing runs.  Otherwise the blob goes to dst (page-locked memory from bgr_host_alloc copies at the full
 * PCIe rate); BGR_ERR_CAPACITY with *bytes = the exact size if dst_cap is smaller.  Waits for submitted vectors and
 * leaves their results queued, like bgr_frame_export.  Device memory for the encoding is allocated and freed inside
 * the call. */
BGR_API int bgr_checkpoint_save(bgr_engine* e, int32_t frame, void* dst, size_t dst_cap, size_t* bytes, int32_t* found);
/* Replaces the engine's world with the blob's.  The blob is untrusted input and is checked in full before anything
 * changes: bad magic or version, another layout, fps or word count, n_blocks != ceil(rows / 512), a truncated or
 * overlong blob, bad offsets, a kind byte > 2 or non-zero padding, a block whose kinds and bitmaps imply another length
 * than its offsets give, a present word with bits set past its column's element bytes (no digest covers them), and a
 * decoded world whose digest root or active count differs from the header's are BGR_ERR_INVALID_ARGUMENT; rows past a
 * fixed engine's capacity or a growable engine's ceiling BGR_ERR_CAPACITY; un-collected submits BGR_ERR_STATE (as
 * bgr_reset_session); a sharded engine BGR_ERR_UNSUPPORTED.  A refused call changes nothing observable.  On success:
 *   - image 0 holds the decoded world (canonical: see above); RollbackFrameCount = frame, and Time<GgrsTime>,
 *     ParticleRng and the row count are the header's;
 *   - the ring keeps its depth and retention setting, and its queue holds exactly one snapshot, of `frame`, holding the
 *     same bytes, so a first Load(frame) works; with BGR_CFG_DESYNC_CAPTURE that slot is also the frame's first image;
 *   - first images (witnesses) and retained frames are released; a pending deferred live image is dropped;
 *   - a growable engine grows to `rows` (after the blob has been verified);
 *   - ConfirmedFrameCount, MaxPredictionWindow, the call counter of BGR_SYS_U32_STORE_CALL_COUNT and every change
 *     feed's reported state are left alone: the next feed report lists exactly the rows that differ from what it last
 *     reported.
 * Device memory for the decoding (a scratch image of the blob's rows) is allocated and freed inside the call. */
BGR_API int bgr_checkpoint_restore(bgr_engine* e, const void* blob, size_t bytes);

/* ---- checkpoint deltas: a frame encoded against an earlier (or later) frame's checkpoint ----------------------------
 * Blob: this header, then u64 offsets[n_blocks + 1], then payload_bytes of payload, with the offsets and the block
 * coding of a checkpoint.  Vector v of block b is canon(target) XOR canon(base) of that block (the mask plane too), with
 * canon the checkpoint's canonical form; the blocks past one frame's rows XOR against zeros.  An unchanged block codes
 * as every vector CONST zero.  Kinds follow the checkpoint's rule, so the delta is a pure function of the two frames'
 * contents: two engines whose digests agree on both frames write byte-identical deltas.  A delta applies to exactly
 * one base checkpoint (base_frame, base_rows, base_root). */
#define BGR_CHECKPOINT_DELTA_MAGIC 0x44524742u /* "BGRD" */
#define BGR_CHECKPOINT_DELTA_VERSION 1u
typedef struct bgr_checkpoint_delta_header {  /* 120 bytes, no padding */
    uint32_t magic;          /* BGR_CHECKPOINT_DELTA_MAGIC */
    uint32_t version;        /* BGR_CHECKPOINT_DELTA_VERSION */
    uint64_t layout;         /* bgr_frame_digest_header.layout */
    int32_t frame;           /* the target frame */
    uint32_t rows;           /* the target's row count */
    int32_t base_frame;
    uint32_t base_rows;
    uint32_t words;
    uint32_t n_blocks;       /* ceil(max(rows, base_rows) / 512) */
    uint32_t n_columns;
    uint32_t fps;
    uint64_t active;         /* the target's, as in bgr_checkpoint_header */
    uint64_t elapsed_ns;
    uint64_t rng[4];
    uint64_t digest_root;    /* the target's root */
    uint64_t base_root;      /* the base's root: the checkpoint this delta applies to */
    uint64_t payload_bytes;
} bgr_checkpoint_delta_header;
/* Encodes `frame` against `base_frame` (both queued or retained; *found = 0 if either is not, and nothing runs).
 * base_frame may be earlier than, later than or equal to frame.  dst == NULL: *bytes = an upper bound (every vector
 * RAW), nothing runs.  Otherwise BGR_ERR_CAPACITY with *bytes = the exact size if dst_cap is smaller.  Waits for
 * submitted vectors and leaves their results queued, like bgr_checkpoint_save. */
BGR_API int bgr_checkpoint_save_delta(bgr_engine* e, int32_t frame, int32_t base_frame, void* dst, size_t dst_cap,
                                      size_t* bytes, int32_t* found);
/* Replaces the engine's world with the delta's target frame, given the full checkpoint `base` it was written against.
 * Both blobs are untrusted and checked in full before anything changes: the base exactly as bgr_checkpoint_restore
 * checks it (its decoded world must reproduce its root); the delta's magic and version, its layout, fps and words
 * against the engine's and the base's, base_frame, base_rows and base_root against the base header's, n_blocks, its
 * length, offsets, kinds and padding.  The target must be canonical (a non-zero word in a row that does not exist or
 * lacks the column, a presence bit the registration lacks, or bits past an element's bytes are refused) and reproduce
 * digest_root and active.  Failures return BGR_ERR_INVALID_ARGUMENT, or what bgr_checkpoint_restore returns for
 * capacity (either frame's rows), un-collected submits or a sharded engine.  A refused call changes nothing observable.
 * On success the engine is exactly as bgr_checkpoint_restore of the target's full checkpoint leaves it. */
BGR_API int bgr_checkpoint_restore_delta(bgr_engine* e, const void* base, size_t base_bytes, const void* delta,
                                         size_t delta_bytes);

/* ---- the three schedules, one at a time (SnapshotPlugin-only users: benches/bench.rs:18-27,
 *      mod.rs:510-535 save_world / advance_frame / load_world helpers) -------------------- */
BGR_API int bgr_save_world(bgr_engine* e, bgr_checksum* checksum_out);         /* world.run_schedule(SaveWorld) */
BGR_API int bgr_load_world(bgr_engine* e);                                     /* world.run_schedule(LoadWorld) at RollbackFrameCount */
BGR_API int bgr_advance_world(bgr_engine* e, const uint8_t* inputs, const uint8_t* status,
                              uint32_t n_players);                             /* world.run_schedule(AdvanceWorld); caller bumps the frame count */

/* ---- THE HOT LOOP: handle_requests (src/schedule_systems.rs:170-289) ------------------- */
/* Executes the whole request vector in one kernel launch: the particles bundle's kernel when the registered systems
 * match it, otherwise the generic one-launch program (spawning worlds included).  Only BGR_CFG_FORCE_STEPWISE and
 * registrations the generic program does not take (more than 8 systems, a 512-row tile over 100 KB) run one launch
 * per request and per system.  Writes one bgr_checksum per SaveGameState, in request order, host-visible on return. */
BGR_API int bgr_handle_requests(bgr_engine* e, const bgr_session_info* session,
                                const bgr_request* requests, uint32_t n_requests,
                                bgr_checksum* checksums_out, uint32_t checksums_cap, uint32_t* n_checksums_out);
/* Asynchronous pair: submit enqueues on the engine stream and returns; collect waits and
 * returns the checksums of the oldest un-collected submit.  At most 8 submits may be un-collected.
 * Entry points that read or edit the world (bgr_read_component, bgr_spawn, bgr_peek ...) wait for the submitted
 * vectors but leave their results queued for bgr_collect; bgr_handle_requests (and the one-schedule helpers above)
 * return BGR_ERR_STATE while submits are un-collected. */
BGR_API int bgr_submit_requests(bgr_engine* e, const bgr_session_info* session,
                                const bgr_request* requests, uint32_t n_requests);
BGR_API int bgr_collect(bgr_engine* e, bgr_checksum* checksums_out, uint32_t checksums_cap,
                        uint32_t* n_checksums_out);
/* Sharded engines (BGR_CFG_SHARDED): raw partials of the last collected call, and the fold
 * that turns cross-shard combined partials into the frame checksum
 * (component_checksum.rs:93-95, entity_checksum.rs:35-43, checksum.rs:88-99). */
BGR_API int bgr_last_partials(bgr_engine* e, bgr_partial* out, uint32_t cap, uint32_t* n_out);
BGR_API int bgr_fold_partials(const bgr_partial* combined, bgr_checksum* out);
/* bgr_collect that writes the raw partials of the collected call straight into caller memory (sharded hot loop:
 * no per-tick allocation), and the fold over an array of already combined partials. */
BGR_API int bgr_collect_partials(bgr_engine* e, bgr_partial* partials_out, uint32_t cap, uint32_t* n_out);
BGR_API int bgr_fold_partials_n(const bgr_partial* combined, uint32_t n, bgr_checksum* out);

/* ---- world batches: the request vectors of many engines in ONE kernel launch ---------------------------------------
 * A batch is a fixed set of built engines ("worlds") with an identical registration (the same columns, presence flags,
 * checksums and systems in the same order), created on one device with the same non-null bgr_config.stream, that run
 * the generic one-launch program (not the particles bundle or BGR_CFG_FORCE_STEPWISE) and are not sharded.
 * Capacity, max_depth, fps, row count, session kind, frame, BGR_CFG_DESYNC_CAPTURE, BGR_CFG_GROWABLE and order_base
 * may differ, and so may a BGR_SYS_PARTICLES_SPAWN system's rate, ttl and seed (its columns may not).  A spawn past a
 * member's max_entities (or, BGR_CFG_GROWABLE, its ceiling) refuses the whole call; a growable member grows first.
 * bgr_batch_create checks all of this and names the first engine that fails.  Destroy a batch before any of its
 * engines; between calls every per-engine entry point stays usable on the members.
 * Every bgr_batch_* call below takes a list of entries, entry i naming one world by its index in the batch, and keeps
 * these conventions (each call's comment adds what its entries are checked for, in which order):
 *   - Every index is in range and listed at most once per call (BGR_ERR_INVALID_ARGUMENT: "no such world in a batch of
 *     N", "listed twice in one call").  Worlds not listed are untouched.
 *   - Every entry is checked, in list order, before anything runs in any world.  The first entry that fails is marked
 *     in status_out (every other status_out[i] is BGR_OK), the call returns its status, bgr_last_error() reads
 *     "world <index>: " and the single-world call's message, and no world changes.  A refusal of the call as a whole
 *     (a null argument) marks no entry.
 *   - A growable member grows after the checks.  A growth that fails is reported like a refusal of that world
 *     (BGR_ERR_CUDA or BGR_ERR_CAPACITY) and nothing else runs; members that grew before it keep their larger capacity.
 *   - A call that runs every world (bgr_batch_handle_requests, the batched replays) sets status_out[i] to what world
 *     i's own call would have returned and returns the first non-OK one, with that world's message.  World i's
 *     checksums follow the earlier worlds' in checksums_out, as far as the cap reaches; n_checksums_out[i] is its
 *     count, and every per-world count is 0 for a world that did not run. */
typedef struct bgr_batch bgr_batch;
BGR_API int bgr_batch_create(bgr_engine* const* engines, uint32_t n, bgr_batch** out);
BGR_API void bgr_batch_destroy(bgr_batch* b);
/* 1: calls run as ONE launch of the registration's generated kernel (k_generic_jit_batch).  0 without NVRTC, with
 * BGR_TUNE_JIT=0, or for a registration the generated kernel does not take (more than 24 words per row, checksummed
 * byte ranges that are not whole words): calls then run each world's own bgr_handle_requests in list order, with the
 * same results (BGR_JIT_VERBOSE=1 prints why). */
BGR_API int bgr_batch_specialised(bgr_batch* b, uint32_t* specialised_out);
/* Synchronous: what bgr_handle_requests on worlds[0], worlds[1], ... in that order would do, in one launch.  World
 * worlds[i] runs the n_requests[i] requests that follow the previous worlds' in `requests` under sessions[i] (sessions
 * NULL: no session).  Each world is checked for its index, n_requests[i] <= BGR_MAX_REQUESTS and no un-collected
 * bgr_submit_requests, and its vector compiled; then every world's spawns are checked against its ceiling.  Then every
 * world executes, and status_out[i] is what its own call would have returned (BGR_ERR_NON_FINITE ...).  Each listed
 * world's bgr_launch_count grows by one and its bgr_last_kernel carries BGR_KERNEL_BATCHED. */
BGR_API int bgr_batch_handle_requests(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const bgr_session_info* sessions,
                                      const bgr_request* requests, const uint32_t* n_requests, bgr_checksum* checksums_out,
                                      uint32_t checksums_cap, uint32_t* n_checksums_out, int32_t* status_out);

/* ---- replays: a recorded input log run through a world in one launch ---------------------------------------------
 * For an engine at RollbackFrameCount f0 >= 0, bgr_replay(n frames, inputs, checksum_interval k) does what this
 * request stream would do through bgr_handle_requests (no session):
 *     for j in 0 .. n-1:  if k > 0 and (f0 + j) % k == 0: SaveGameState{f0 + j};   AdvanceFrame{inputs[j*n_players ..]}
 * with three differences: no snapshot is pushed (the ring, its depth, confirmed frame, retained frames and desync
 * witnesses are left alone, so a Load of a frame from before the replay still works); frame f0 + n is not checksummed
 * (replay(a) then replay(b) equals replay(a ++ b)); and there is no BGR_MAX_REQUESTS limit.  The live world, the row
 * count, RollbackFrameCount (= f0 + n), Time<GgrsTime>, ParticleRng, the BGR_SYS_U32_STORE_CALL_COUNT counter and the
 * checksums (one per checksum frame, in frame order) equal the stream's.  A non-finite finite-asserted value at a
 * checksum frame is BGR_ERR_NON_FINITE after the whole replay has run; bgr_last_error() names the first such frame.
 * Refusals change nothing: n_players > BGR_MAX_PLAYERS, n_frames > BGR_MAX_REPLAY_FRAMES, reserved != 0, a null log
 * with n_frames > 0, or f0 + n past INT32_MAX: BGR_ERR_INVALID_ARGUMENT; un-collected submits, f0 < 0 or a first step
 * that would move Time<GgrsTime> backwards: BGR_ERR_STATE; BGR_CFG_SHARDED: BGR_ERR_UNSUPPORTED; spawns past a fixed
 * engine's max_entities or a growable engine's ceiling: BGR_ERR_CAPACITY (a growable engine otherwise grows first).
 * Synchronous.  *n_out = the number of checksum frames; the first `cap` of them go to checksums_out.
 * Runs on the registration's generated kernel (k_generic_jit_replay, bgr_last_kernel carries BGR_KERNEL_REPLAY; an
 * engine without one compiles it at its first replay) unless BGR_TUNE_JIT=0, BGR_CFG_FORCE_STEPWISE or a registration
 * the generated kernel does not take: then in chunks of at most BGR_MAX_REQUESTS ops through the engine's own kernel,
 * with the same results.  Replay serves spectator catch-up, replay seeking and match verification; it does not
 * replace bgr_handle_requests for a live session. */
#define BGR_MAX_REPLAY_FRAMES (1u << 24)
/* a struct tag without a typedef: the call below has the same name, so the type is spelled `struct bgr_replay` */
struct bgr_replay {
    uint32_t n_frames;           /* AdvanceFrame requests */
    uint32_t n_players;          /* PlayerInputs<T>.len() of every frame, <= BGR_MAX_PLAYERS */
    uint32_t checksum_interval;  /* 0: no checksums; k: frames f0+j with (f0+j) % k == 0, before advancing them */
    uint32_t reserved;           /* 0 */
    const uint8_t* inputs;       /* n_frames * n_players bytes, frame-major */
};
BGR_API int bgr_replay(bgr_engine* e, const struct bgr_replay* r, bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out);
/* bgr_replay of replays[i] on worlds[i].  Each world is checked for its index and everything bgr_replay refuses, and
 * planned, before any executes.  A specialised batch (bgr_batch_specialised) runs every world in one launch of its
 * generated kernel; otherwise each world's bgr_replay runs in list order. */
BGR_API int bgr_batch_replay(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                             bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_checksums_out, int32_t* status_out);

/* ---- replay keyframes: a world checkpoint every K frames while a replay runs ---------------------------------------
 * bgr_replay_keyframes is bgr_replay that also writes a keyframe at each frame f0 + j, j in [0, n), with
 * (f0 + j) % interval == 0, taken before that frame is advanced (where a checksum point is taken), so keyframes(a) then
 * keyframes(b) equals keyframes(a ++ b).  Keyframe f is byte for byte the blob bgr_checkpoint_save(f) writes on an
 * engine that ran the equivalent request stream with a SaveGameState{f} at that frame: the same header (frame, rows,
 * active, elapsed_ns = Time<GgrsTime> of f, rng = ParticleRng of f, digest_root, layout, fps) and canonical payload.
 * Everything else (checksums, live world, row count, RollbackFrameCount, Time, ParticleRng, the call counter, the ring,
 * retained frames, witnesses, change feeds) ends exactly as after bgr_replay of the same log.  Seeking a recorded match:
 * bgr_checkpoint_restore of the nearest keyframe at or before the target, then bgr_replay of fewer than `interval` frames.
 *   - Output: the blobs go to dst in frame order, each at a multiple of 8 bytes; index[i] describes blob i.
 *   - dst == NULL: nothing runs; *n_keyframes_out = the keyframe count and *bytes_out = an upper bound on the bytes
 *     (every vector RAW, at the row count each keyframe will have, alignment included).
 *   - Otherwise dst_cap below that bound or index_cap below the count is BGR_ERR_CAPACITY before anything runs; on
 *     return *n_keyframes_out = the keyframes written and *bytes_out = the end of the last blob.
 *   - Refusals change nothing: everything bgr_replay refuses, interval == 0 or reserved != 0 (BGR_ERR_INVALID_ARGUMENT)
 *     and the capacity checks above.  BGR_CFG_SHARDED: BGR_ERR_UNSUPPORTED.
 *   - A non-finite finite-asserted value at a checksum frame is BGR_ERR_NON_FINITE after the whole log ran; the keyframes
 *     are written anyway, as bgr_checkpoint_save would write them.
 * On the generated kernel (k_generic_jit_replay_kf, bgr_last_kernel carries BGR_KERNEL_REPLAY) each launch stores the
 * registers of its keyframe frames into device staging, whose size ends a launch early (BGR_TUNE_KEYFRAME_BYTES, 256 MB
 * by default, always at least one keyframe per world), and encodes all of them in four launches and one copy to the host.
 * The staging and the encoder's device memory are allocated and freed inside the call.
 * Without a generated kernel the replay runs in chunks that end at each keyframe, which is encoded from the live image:
 * the same bytes, slower. */
typedef struct bgr_keyframe {  /* 24 bytes */
    int32_t frame;
    uint32_t reserved;         /* 0 */
    uint64_t offset;           /* of the blob in dst; a multiple of 8 */
    uint64_t bytes;            /* the blob's exact size */
} bgr_keyframe;
struct bgr_keyframes {         /* 40 bytes */
    uint32_t interval;         /* K >= 1 */
    uint32_t index_cap;
    uint64_t reserved;         /* 0 */
    void* dst;                 /* NULL: query only */
    size_t dst_cap;
    bgr_keyframe* index;       /* [index_cap] */
};
BGR_API int bgr_replay_keyframes(bgr_engine* e, const struct bgr_replay* r, const struct bgr_keyframes* kf,
                                 bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out, uint32_t* n_keyframes_out,
                                 size_t* bytes_out);
/* bgr_batch_replay with keyframes: kfs[i] holds world i's interval and buffers, in bgr_replay_keyframes' conventions
 * (a null dst is refused with BGR_ERR_CAPACITY unless the world writes no keyframe; query a member's sizes with
 * bgr_replay_keyframes on its engine).  Each world's capacities are checked after its plan; n_keyframes_out[i] is world
 * i's keyframe count. */
BGR_API int bgr_batch_replay_keyframes(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                                       const struct bgr_keyframes* kfs, bgr_checksum* checksums_out, uint32_t cap,
                                       uint32_t* n_checksums_out, uint32_t* n_keyframes_out, int32_t* status_out);

/* ---- replay traces: chosen fields of a row range every T frames while a replay runs -------------------------------
 * bgr_replay_trace is bgr_replay that also takes a sample at each frame f0 + j, j in [0, n), with (f0 + j) % interval == 0,
 * before that frame is advanced (where a checksum point or a keyframe is taken), so trace(a) then trace(b) equals
 * trace(a ++ b).  Everything else (checksums, live world, row count, RollbackFrameCount, Time, ParticleRng, the call
 * counter, the ring, retained frames, witnesses, change feeds) ends exactly as after bgr_replay of the same log.  Replay
 * viewers and match analytics read the entities they draw or mine at every frame without a host round trip per frame.
 *   - Records: sample s, traced row i (row first_row + i) is one record at dst + (s * n_rows + i) * record_bytes, the change
 *     feed's record of that row (bgr_feed_create's fields) in the live world at the sample frame: u32 row, u32 state (bit 0
 *     the row exists, bit 1 + k it exists and field k's column is present), then the fields' bytes, zero where a field is
 *     not present.  record_bytes = 8 + the sum of byte_len.  Rows that do not exist at the sample (at or past the row
 *     count, or despawned) are written too, as state 0 with zero bytes, so the layout is dense and fixed.  samples[s] =
 *     the sample's frame and RollbackOrdered::len() there.
 *   - dst == NULL: nothing runs; *n_samples_out and *bytes_out = the exact sample count and bytes.  Otherwise a dst_cap or
 *     samples_cap below them is BGR_ERR_CAPACITY before anything runs.
 *   - Refusals change nothing: everything bgr_replay refuses; interval == 0, n_rows == 0 or reserved != 0
 *     (BGR_ERR_INVALID_ARGUMENT); a field list bgr_feed_create would refuse, with its status; first_row + n_rows past the
 *     engine's max_entities, or past its ceiling for BGR_CFG_GROWABLE (BGR_ERR_INVALID_ARGUMENT).
 *   - A non-finite finite-asserted value at a checksum frame is BGR_ERR_NON_FINITE after the whole log ran, with every
 *     sample written.
 * On the generated kernel (k_generic_jit_replay_trace, bgr_last_kernel carries BGR_KERNEL_REPLAY) each thread writes its
 * traced rows' records from its registers at each sample frame into device staging, whose size ends a launch early
 * (BGR_TUNE_TRACE_BYTES, 256 MB by default, split over the unfinished worlds, always at least one sample per world); each
 * launch's records come back with one copy.  The staging is allocated and freed inside the call.  Without a generated
 * kernel the replay runs in chunks that end at each sample frame, whose records k_trace_gather writes from the live image:
 * the same bytes, slower. */
typedef struct bgr_trace_sample {  /* 8 bytes */
    int32_t frame;
    uint32_t rows;                 /* RollbackOrdered::len() at frame */
} bgr_trace_sample;
struct bgr_trace {                 /* 56 bytes */
    uint32_t interval;             /* T >= 1 */
    uint32_t first_row, n_rows;    /* the traced rows [first_row, first_row + n_rows), n_rows >= 1 */
    uint32_t n_fields;             /* 0 .. BGR_MAX_FEED_FIELDS */
    const bgr_feed_field* fields;  /* the change feed's field type and rules */
    void* dst;                     /* NULL: query only */
    size_t dst_cap;
    bgr_trace_sample* samples;     /* [samples_cap] */
    uint32_t samples_cap;
    uint32_t reserved;             /* 0 */
};
BGR_API int bgr_replay_trace(bgr_engine* e, const struct bgr_replay* r, const struct bgr_trace* t,
                             bgr_checksum* checksums_out, uint32_t cap, uint32_t* n_out,
                             uint32_t* n_samples_out, size_t* bytes_out);
/* bgr_batch_replay with traces: traces[i] holds world i's interval, row range and buffers, in bgr_replay_trace's
 * conventions (a null dst is refused with BGR_ERR_CAPACITY unless the world takes no sample; query a member's sizes with
 * bgr_replay_trace on its engine).  Row ranges and intervals may differ between worlds; the field list must equal entry
 * 0's (BGR_ERR_INVALID_ARGUMENT otherwise), so a launch has one record layout.  Each world's field list and then its
 * capacities are checked after its plan; n_samples_out[i] is world i's sample count. */
BGR_API int bgr_batch_replay_trace(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const struct bgr_replay* replays,
                                   const struct bgr_trace* traces, bgr_checksum* checksums_out, uint32_t cap,
                                   uint32_t* n_checksums_out, uint32_t* n_samples_out, int32_t* status_out);

/* ---- batched checkpoints: the world checkpoints of many batch members saved or restored in one pass ----------------
 * Neither depends on bgr_batch_specialised: the checkpoint kernels are part of the library, so a batch that ticks its
 * worlds one after another (BGR_TUNE_JIT=0, no NVRTC) saves and restores in one pass too.  The kernels of one call are
 * counted on worlds[0]'s bgr_launch_count, and their number does not depend on n_worlds: a save is four launches
 * (k_frame_digest, k_ckpt_measure, k_ckpt_scan, k_ckpt_pack) and a restore three (k_ckpt_unpack, k_frame_digest,
 * k_ckpt_commit); fewer when no listed world has a row.  Device memory for the encoding or decoding is allocated and
 * freed inside the call.
 *
 * bgr_batch_checkpoint_save: blob i is byte for byte what bgr_checkpoint_save(worlds[i], frames[i]) writes (the frame
 * queued or retained).  The blobs go to dst in list order, each at a multiple of 8 bytes (the padding is zero);
 * index[i] = {frames[i], 0, offset in dst, bytes}, and bytes == 0 means the world holds that frame neither queued nor
 * retained (the single call's *found = 0), which is not an error.  dst == NULL: nothing runs; index[i].bytes = world i's
 * upper bound (every vector RAW), index[i].offset its place under those bounds, and *bytes_out = the total, a multiple
 * of 8.  Otherwise *bytes_out = the exact total, the end of the last blob rounded up to 8; a dst_cap below it is
 * BGR_ERR_CAPACITY, and then nothing is written to dst or index.  Once every index has passed, waits for each member's
 * submitted vectors and leaves their results queued.  The payloads of every world come back to dst with one copy
 * (page-locked dst from bgr_host_alloc copies at the full PCIe rate). */
BGR_API int bgr_batch_checkpoint_save(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds, const int32_t* frames,
                                      void* dst, size_t dst_cap, bgr_keyframe* index, size_t* bytes_out,
                                      int32_t* status_out);
/* bgr_batch_checkpoint_restore: each listed world ends exactly as bgr_checkpoint_restore(worlds[i], blobs[i], bytes[i])
 * would leave it (see there: image 0, one queued ring slot, frame, Time<GgrsTime>, ParticleRng, row count, witnesses and
 * retained frames released, a deferred live image dropped, change feeds left alone, a growable member grown to the
 * blob's rows).  All or nothing: if any blob fails any of bgr_checkpoint_restore's checks, no world changes.  The host
 * checks (header, offsets, capacity, un-collected submits: BGR_ERR_STATE) run first, in list order, and the first
 * failure is reported; the device checks (kinds, padding, implied lengths, mask bits, stray bits, digest root and active
 * count) run only if every blob passed the host checks, and the lowest listed index that failed is reported.  One blob
 * may be listed for several worlds, and a blob may come from another member when its layout (order_base included) and
 * fps match the target's.  One pass, whatever n_worlds: the payloads are gathered into page-locked staging that the
 * batch keeps (sized by its largest restore) and uploaded with one copy, the tables and offsets with another, then
 * k_ckpt_unpack and k_frame_digest run over every block of every blob, three copies bring back the error words, the
 * digest words and the active counts, and one k_ckpt_commit launch copies every world to its image 0 and restored slot.
 * Every allocation happens before any world changes: out of device memory is BGR_ERR_CUDA with no world changed.  A
 * growable member whose growth fails is named and nothing is restored. */
BGR_API int bgr_batch_checkpoint_restore(bgr_batch* b, const uint32_t* worlds, uint32_t n_worlds,
                                         const void* const* blobs, const size_t* bytes, int32_t* status_out);

/* ---- batched change feed: the change feeds of many batch members reported in one pass ------------------------------
 * Entry i reports feed reports[i].feed of member reports[i].world with at most records_cap records.  Its records and
 * infos[i] are byte for byte what bgr_feed_begin / bgr_feed_wait on that engine would give at that point, and the report
 * advances the same reported state: batched and single reports of one feed alternate freely, and bgr_feed_reset still
 * applies.  The records are packed in list order into host_dst: entry i's start at the sum of the earlier entries'
 * n_records.  host_dst must come from bgr_host_alloc and hold sum(records_cap) records (NULL when every cap is 0); it
 * must not be read before bgr_batch_feed_wait(ticket) returns.
 * A second bgr_batch_feed_begin before the wait is BGR_ERR_STATE for the whole call: one batched report per batch is in
 * flight.  Then each entry is checked for its index, a known feed (BGR_ERR_INVALID_ARGUMENT), no report of that feed in
 * flight, single or batched (BGR_ERR_STATE), and the same field list as entry 0's feed (BGR_ERR_INVALID_ARGUMENT: a call
 * has one record size).  A refused call changes nothing: no feed becomes busy and no reported state moves.  A host_dst
 * not from bgr_host_alloc is BGR_ERR_INVALID_ARGUMENT for the whole call.
 * The call is ordered behind every vector submitted on the shared stream, un-collected submits of a member included,
 * materialises a deferred live image only on the listed worlds that have one, and returns without waiting for the GPU.
 * It does not depend on bgr_batch_specialised.  Whatever n_entries, it is one table upload, four launches counted on
 * reports[0].world's bgr_launch_count (k_feed_count, k_feed_scan, k_feed_records, and k_feed_copy on a copy stream of
 * the batch; no k_feed_count when no listed world has a tile, no k_feed_copy when every cap is 0) and one copy of the
 * infos; the scratch the batch keeps grows to the largest call and is allocated before any feed changes.
 * bgr_batch_feed_wait waits for the report and writes infos[0 .. n_entries); an unknown or already-waited ticket is
 * BGR_ERR_STATE. */
typedef struct bgr_batch_feed { uint32_t world, feed, records_cap; } bgr_batch_feed;
BGR_API int bgr_batch_feed_begin(bgr_batch* b, const bgr_batch_feed* reports, uint32_t n_entries, void* host_dst,
                                 uint32_t* ticket_out, int32_t* status_out);
BGR_API int bgr_batch_feed_wait(bgr_batch* b, uint32_t ticket, bgr_feed_info* infos);

/* ---- batched host edits: the bgr_apply_edits batches of many batch members in one call -----------------------------
 * Entry i leaves member entries[i].world exactly as bgr_apply_edits(that engine, edits, n_edits, values, values_bytes)
 * would: the live image and row count, presence bytes, the passive version (moved only by spawns, inserts, removes and
 * passive-plane writes), a fresh live content id, and a deferred live image materialised first.  Worlds not listed are
 * untouched; an entry with n_edits == 0 changes nothing in its world (it materialises nothing either), but is still
 * checked for its index.
 * Each entry is checked for its index, no null pointer, every record by bgr_apply_edits' own checks (bgr_last_error()
 * "world 2: edit 3: row out of range"), spawns past a fixed member's max_entities or a growable member's ceiling
 * (BGR_ERR_CAPACITY), spawning after the first request vector with order_base != 0 (BGR_ERR_UNSUPPORTED).  A refused
 * call changes nothing anywhere: no member grows, nothing launches.
 * The call is ordered on the shared stream behind every queued vector, un-collected bgr_submit_requests of a member
 * included (they keep their results), and returns without waiting for the GPU.  The caller's buffers are free on
 * return: the patch goes into one of 4 page-locked staging buffers the batch owns, each grown to the largest call it
 * has held, and the call waits only when all 4 belong to unfinished calls (bgr_apply_edits' rule, on the batch's
 * memory).  Whatever n_entries, a call is at most one table upload and two launches, counted on entries[0].world's
 * bgr_launch_count: k_spawn_rows over every spawning world when one spawns, and k_apply_edits over every patch when
 * one is non-empty.  A listed world with a deferred live image and n_edits > 0 also gets its own materialisation,
 * counted on that world.  It does not depend on bgr_batch_specialised: the edit kernels are part of the library. */
typedef struct bgr_batch_edits {     /* 32 bytes */
    uint32_t world;                  /* index in the batch */
    uint32_t n_edits;
    const bgr_edit* edits;           /* bgr_apply_edits' records, unchanged */
    const void* values;
    size_t values_bytes;
} bgr_batch_edits;
BGR_API int bgr_batch_apply_edits(bgr_batch* b, const bgr_batch_edits* entries, uint32_t n_entries, int32_t* status_out);

/* ---- shard group: the cross-shard step inside the engine (multi-GPU, one process per GPU, one node) -----------------
 * Entity-range shards never exchange state (SURVEY.md §8e: systems read no other entity, box_game.rs:162-169; the
 * checksum is an XOR over entities, component_checksum.rs:88-89).  The only exchange is 64 bytes of partials per
 * SaveGameState.  After every rank's BGR_CFG_SHARDED engine has joined the same group, bgr_handle_requests /
 * bgr_collect on ANY rank return the frame checksum of the WHOLE world (has_checksum = 1) — what
 * `cell.save(frame, None, checksum)` needs (schedule_systems.rs:231-236) — with no call outside this library:
 * the result blocks live in one shared host segment that every rank's GPU stores into and every rank's CPU polls.
 * Every rank must be handed the same request vectors in the same order (they all replay the same GGRS session).
 * `name` must be unique per group instance (e.g. "<launcher pid>_<port>"); timeout_ms = 0 selects 60 s. */
BGR_API int bgr_shard_group_join(bgr_engine* e, const char* name, uint32_t rank, uint32_t world_size, uint32_t timeout_ms);
BGR_API int bgr_shard_group_leave(bgr_engine* e);
/* the group's host logic without an engine (no GPU call): CPU tests publish partials computed elsewhere */
typedef struct bgr_group bgr_group;
BGR_API bgr_group* bgr_group_join(const char* name, uint32_t rank, uint32_t world_size, uint32_t n_columns, uint32_t timeout_ms);
BGR_API void bgr_group_leave(bgr_group* g);
BGR_API int bgr_group_publish(bgr_group* g, uint64_t group_seq, const bgr_partial* partials, uint32_t n);  /* group_seq = 1, 2, ... */
BGR_API int bgr_group_collect(bgr_group* g, uint64_t group_seq, bgr_checksum* out, uint32_t cap, uint32_t* n_out);

/* ---- checksum_hasher() (src/snapshot/mod.rs:315-317) for host-side parts -------------------------------
 * Resources stay on the host (a few bytes, not data-parallel).  A shim that registers
 * `checksum_resource_with_hash::<R>()` (resource_checksum.rs:63-82) computes `part = bgr_seahash(bytes of R)`
 * per Save and XORs it into the engine's checksum (ChecksumPlugin::update, checksum.rs:88-99). */
BGR_API uint64_t bgr_seahash(const void* bytes, uint64_t len);

/* ---- ParticleRng arithmetic on its own (host only; examples/stress_tests/particles.rs:125-128, 258-270) -------
 * The Xoshiro256PlusPlus stream spawn_particles draws from: `state4_or_null` = Xoshiro256PlusPlus::from_seed state
 * words, or NULL for seed_from_u64(seed).  next_u64_out[i] = the i-th next_u64(); range_out[i] = the i-th
 * random_range(low..high) of an identical, separate generator.  bgr_splitmix64_stream = rand_xoshiro's SplitMix64.
 * Exposed so that published known-answer vectors run against the product's own code. */
BGR_API int bgr_particle_rng_stream(uint64_t seed, const uint64_t* state4_or_null, uint32_t n, uint64_t* next_u64_out,
                                    float* range_out, float low, float high);
BGR_API int bgr_splitmix64_stream(uint64_t seed, uint32_t n, uint64_t* out);

/* ---- GgrsTime (src/time.rs:63-76): delta_secs of the step that ends at `frame` ---------- */
BGR_API uint32_t bgr_ggrs_time_delta_bits(uint32_t fps, int32_t frame);

/* ---- introspection for benches / tests --------------------------------------------------- */
BGR_API int bgr_launch_count(bgr_engine* e, uint64_t* kernels_launched_out);
BGR_API int bgr_slot_bytes(bgr_engine* e, uint64_t* bytes_out);  /* algorithmic bytes of one frame slot at the current row count */
BGR_API int bgr_last_path(bgr_engine* e, uint32_t* fused_out);   /* 1 if the last handle_requests used the fused program kernel */
/* 1 if bgr_build compiled this registration's own kernel (NVRTC specialisation of the generic one-launch program,
 * csrc/generic_program_jit.cuh): every non-bundle request vector then runs on it; 0 = the interpreter kernel (same results).
 * Env BGR_TUNE_JIT: 0 never, 1 (default) engines created for >= 16384 entities, 2 always. */
BGR_API int bgr_generic_specialised(bgr_engine* e, uint32_t* specialised_out);
/* Which kernel the last request vector executed (0 before the first one).  Tuning knobs fall back quietly: this says
 * what actually ran.  The bundle currently always reports VEC 2, tier 1 and 512-row work items.
 *   bits 0-3   kind: BGR_KERNEL_*
 *   bits 4-7   bundle: rows per thread (VEC)
 *   bits 8-9   bundle: MODE 0 (checksum flags tested at run time), 1 (Transform and Velocity both checksummed with
 *              BGR_HASH_FLAG_ASSERT_FINITE_F32: specialised), 2 (per-entity presence of optional columns)
 *   bits 10-11 bundle: launch-bounds tier, 0 unconstrained, 1 768 threads per SM, 2 1024 threads per SM
 *   bit 12     bundle: launched in the passive-TMA configuration (shared-memory double buffer): passive planes the
 *              launch moves go by TMA bulk copies; clear: they go per thread (spawns, several Loads, BGR_TUNE_PASSIVE_TMA=0)
 *   bit 13     BGR_KERNEL_DEFERRED_LIVE: the vector ended in Save, Advance... and did not write the live image; it is
 *              rebuilt from that Save's slot when something needs it (env BGR_TUNE_DEFER_LIVE, default 1)
 *   bit 14     BGR_KERNEL_FROM_DEFERRED: the vector would have read a deferred live image and started from the base
 *              slot instead (a Load of that slot and its pending Advances ran first, inside the same launch)
 *   bit 15     BGR_KERNEL_PASSIVE_PLANES, bundle: the launch read or wrote passive planes.  Clear on a tick whose Saves
 *              go into slots that already hold the live passive content and whose Load does not change it
 *              (BGR_CFG_SKIP_UNCHANGED_PLANES above)
 *   bits 16-25 bundle and generic NVRTC: rows per work item (512 = a whole tile)
 *   bit 26     BGR_KERNEL_STABLE_PLANES, bundle: stable-plane elision.  Each warp stored only the active planes of its
 *              64-row segment whose content the target image did not already hold (device-side content stamps).  Set on
 *              grids of several waves; a single-wave (latency-bound) grid stores every active plane
 *   bit 27     BGR_KERNEL_HELD_SAVES, bundle: at least one Save was held: its target slot already held the content and
 *              row count it would have stored (host-side content ids), so it stored nothing and only checksummed
 *              (bgr_held_saves; env BGR_TUNE_HELD_SAVES, default 1)
 *   bit 28     BGR_KERNEL_BATCHED, generic NVRTC: the vector ran inside a world batch's launch (bgr_batch_handle_requests)
 *   bit 29     BGR_KERNEL_REPLAY, generic NVRTC: the last bgr_replay / bgr_batch_replay ran on the generated kernel's replay
 *              entry point (k_generic_jit_replay); clear when it ran in chunks through the engine's own kernel
 *   bit 30     BGR_KERNEL_WARP_FOLD, bundle: each Save's checksum partials were reduced over the warp as it ran, not
 *              added to per-lane shared-memory slots and reduced once per block: the slots (640 bytes per Save) would
 *              have cost the launch a resident block per SM (a wide passive double buffer and many Saves) */
#define BGR_KERNEL_DEFERRED_LIVE (1u << 13)
#define BGR_KERNEL_FROM_DEFERRED (1u << 14)
#define BGR_KERNEL_PASSIVE_PLANES (1u << 15)
#define BGR_KERNEL_STABLE_PLANES (1u << 26)
#define BGR_KERNEL_HELD_SAVES (1u << 27)
#define BGR_KERNEL_BATCHED (1u << 28)
#define BGR_KERNEL_REPLAY (1u << 29)
#define BGR_KERNEL_WARP_FOLD (1u << 30)
#define BGR_KERNEL_NONE 0u
#define BGR_KERNEL_STEPWISE_TMA 1u       /* one kernel per request; Save / Load through the TMA-staged copy kernel */
#define BGR_KERNEL_STEPWISE_FLAT 2u      /* one kernel per request; k_checksum_column + k_copy_image */
#define BGR_KERNEL_BUNDLE 3u             /* the compiled particles kernel (k_particles_program) */
#define BGR_KERNEL_GENERIC_INTERPRETER 4u
#define BGR_KERNEL_GENERIC_NVRTC 5u
BGR_API int bgr_last_kernel(bgr_engine* e, uint32_t* kernel_out);
/* Held Saves of the bundle kernel (bit 27 above): out[0] in the last request vector, [1] in every request vector so
 * far, [2] with BGR_TUNE_HELD_SAVES=2 (verify) the active words and alive bytes, below the row count, in which a held
 * Save's target differed from what the Save would have stored, counted on the GPU (waits for it; 0 otherwise).
 * cap <= 3 */
BGR_API int bgr_held_saves(bgr_engine* e, uint64_t* out, uint32_t cap);
BGR_API int bgr_synchronize(bgr_engine* e);
BGR_API int bgr_stream(bgr_engine* e, void** stream_out);        /* the cudaStream_t the engine launches on (timing events) */
/* device-side launch trace: 4 x u64 per fused launch after the call, up to `capacity` launches (GPU globaltimer ns):
 * [0] first block started, [1] last block finished its tiles, [2] results + completion word written, [3] bundle:
 * 64-byte units of active planes the launch stored into slots and the live image (a word plane of 64 rows is 4 units,
 * its alive plane 1).
 * bgr_trace_read copies the rows out (waits for the GPU).  capacity 0 disables. */
BGR_API int bgr_trace_enable(bgr_engine* e, uint32_t capacity);
BGR_API int bgr_trace_read(bgr_engine* e, uint64_t* rows_out, uint32_t cap_launches, uint32_t* n_out);
/* cumulative host-side time of the hot loop: out[0] request vectors, [1] ns compiling requests, [2] ns enqueueing the
 * launch, [3] ns waiting for the completion word, [4] ns folding results (cap <= 8) */
BGR_API int bgr_host_profile(bgr_engine* e, uint64_t* out, uint32_t cap);

/* ---- host-side ring bookkeeping on its own ------------------------------------------------------
 * The frame -> HBM-slot queue the engine keeps for GgrsSnapshots (mod.rs:94-271), exposed without
 * an engine so the reference's 11 ring unit tests (mod.rs:365-508) run against it on a CPU-only
 * box.  Pure host logic, no GPU call. */
typedef struct bgr_ring bgr_ring;
BGR_API bgr_ring* bgr_ring_create(uint32_t n_slots);
BGR_API void bgr_ring_destroy(bgr_ring* r);
BGR_API uint32_t bgr_ring_depth(bgr_ring* r);
BGR_API int bgr_ring_set_depth(bgr_ring* r, uint32_t depth);
BGR_API int bgr_ring_push(bgr_ring* r, int32_t frame, uint32_t* slot_out);
BGR_API int bgr_ring_confirm(bgr_ring* r, int32_t frame);
BGR_API int bgr_ring_rollback(bgr_ring* r, int32_t frame, uint32_t* slot_out);
BGR_API int bgr_ring_get(bgr_ring* r, uint32_t* slot_out);
BGR_API int bgr_ring_peek(bgr_ring* r, int32_t frame, uint32_t* slot_out, int32_t* found);
/* the same ring with desync capture (BGR_CFG_DESYNC_CAPTURE): first(frame) = slot of the frame's retained first image */
BGR_API bgr_ring* bgr_ring_create_capture(uint32_t n_slots);
BGR_API int bgr_ring_first(bgr_ring* r, int32_t frame, uint32_t* slot_out, int32_t* found);
BGR_API int bgr_ring_slots_in_use(bgr_ring* r, uint32_t* n_out);  /* queued or pinned slots */
/* retention of confirmed frames on a standalone ring (bgr_retain_confirmed); count 0 turns it off */
BGR_API int bgr_ring_set_retention(bgr_ring* r, uint32_t interval, uint32_t count);
BGR_API int bgr_ring_retained(bgr_ring* r, int32_t* frames_out, uint32_t cap, uint32_t* n_out);  /* newest first */

#ifdef __cplusplus
}
#endif
#endif /* BEVY_GGRS_B200_H */
