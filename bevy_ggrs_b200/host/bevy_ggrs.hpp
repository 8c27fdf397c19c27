// C++ host-side mirror of the bevy_ggrs plugin surface for the rollback hot path, above the C ABI
// (include/bevy_ggrs_b200.h).  Same names, argument meaning and error behaviour as the reference:
//
//   App app(max_entities, max_depth);
//   app.add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})                 // lib.rs:198-258
//      .insert_resource(RollbackFrameRate{60})                         // time.rs:19-26
//      .add_systems(ReadInputs{}, read_local_inputs)                   // lib.rs:148-149
//      .rollback_component_with_clone<Transform>()                     // rollback_app.rs:178-183
//      .rollback_component_with_copy<Velocity>()                       // rollback_app.rs:157-162
//      .checksum_component<Transform>(hash_bytes(0, 12, true))         // rollback_app.rs:227-232
//      .add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_UPDATE, {col<Transform>, col<Velocity>}})
//      .insert_resource(Session::SyncTest(ggrs::SyncTestSession(2, 8, 9, 2)))
//      .add_observer([](const SyncTestMismatch& m) { ... });
//   app.update();                                                      // run_ggrs_schedules, schedule_systems.rs:19-83
//
// A Rust panic becomes a C++ exception carrying the same text (`Panic`).  The "World" is the engine:
// columns and the snapshot ring live in HBM, this layer holds no component data.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <typeindex>
#include <typeinfo>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "ggrs_standin.hpp"

namespace bevy_ggrs {

struct Panic : std::runtime_error {
    int status;
    Panic(int s, const std::string& text) : std::runtime_error(text), status(s) {}
};
inline void check(int status) {
    if (status != BGR_OK) throw Panic(status, bgr_last_error());
}

// ---- schedule labels / resources / events (lib.rs:73-149, snapshot/mod.rs:66-77) ----
struct GgrsSchedule {};
struct ReadInputs {};
struct Startup {};
struct RollbackFrameRate { size_t fps = 60; };
struct LocalPlayers { std::vector<ggrs::PlayerHandle> handles; };
struct LocalInputs { std::map<ggrs::PlayerHandle, uint8_t> inputs; };
struct SyncTestMismatch { ggrs::Frame current_frame; std::vector<ggrs::Frame> mismatched_frames; };
template <class Input = uint8_t> struct GgrsConfig { using input_type = Input; };
template <class Config> struct GgrsPlugin {};

struct Session {  // lib.rs:79-86: enum Session<T> { SyncTest(..), P2P(..), Spectator(..) }
    enum Kind { SyncTestKind, P2PKind, SpectatorKind } kind = SyncTestKind;
    std::shared_ptr<ggrs::SyncTestSession> synctest;
    std::shared_ptr<ggrs::P2PTraceSession> p2p;
    std::shared_ptr<ggrs::SpectatorTraceSession> spectator;
    static Session SyncTest(ggrs::SyncTestSession s) { Session r; r.kind = SyncTestKind; r.synctest = std::make_shared<ggrs::SyncTestSession>(std::move(s)); return r; }
    static Session P2P(ggrs::P2PTraceSession s) { Session r; r.kind = P2PKind; r.p2p = std::make_shared<ggrs::P2PTraceSession>(std::move(s)); return r; }
    static Session Spectator(ggrs::SpectatorTraceSession s) { Session r; r.kind = SpectatorKind; r.spectator = std::make_shared<ggrs::SpectatorTraceSession>(std::move(s)); return r; }
};

// a compiled-in GgrsSchedule system: id + bound columns + scalar parameters
struct System {
    uint32_t id;
    std::vector<uint32_t> columns;
    std::vector<uint32_t> params;
};

// A GgrsSchedule system that only touches host-side resources (box_game.rs:146-148 increase_frame_system).
// Resources are a few bytes and not data-parallel: they stay on the host, this layer rolls them back per frame
// (resource_snapshot.rs:65-93) and XORs their checksum parts into the engine's checksum (checksum.rs:88-99).
class App;
struct ResourceSystem { std::function<void(App&)> fn; };

// what a `fn(&T) -> u64` hasher becomes across the C ABI: seahash of a byte range of the element
struct ByteRangeHasher { uint32_t offset, len; bool assert_finite; };
inline ByteRangeHasher hash_bytes(uint32_t offset, uint32_t len, bool assert_finite = false) { return {offset, len, assert_finite}; }

class App {
public:
    App(uint32_t max_entities, uint32_t max_depth, int device = 0, uint32_t flags = 0) {
        bgr_config cfg;
        std::memset(&cfg, 0, sizeof cfg);
        cfg.abi_version = BGR_ABI_VERSION; cfg.device = device; cfg.max_entities = max_entities;
        cfg.max_depth = max_depth; cfg.fps = 60; cfg.flags = flags;
        cfg_ = cfg;
    }
    ~App() { if (engine_) bgr_engine_destroy(engine_); }
    App(const App&) = delete;

    template <class C> App& add_plugins(GgrsPlugin<C>) { return *this; }
    App& insert_resource(RollbackFrameRate r) { cfg_.fps = uint32_t(r.fps); return *this; }
    App& insert_resource(Session s) { session_ = std::move(s); return *this; }
    App& remove_session() { session_.reset(); return *this; }  // world.remove_resource::<Session<T>>()
    App& insert_resource(LocalInputs li) { local_inputs_ = std::move(li); return *this; }
    App& add_systems(ReadInputs, std::function<void(App&)> f) { read_inputs_.push_back(std::move(f)); return *this; }
    App& add_systems(Startup, std::function<void(App&)> f) { startup_.push_back(std::move(f)); return *this; }
    App& add_systems(GgrsSchedule, System s) { systems_.push_back(std::move(s)); return *this; }
    App& add_systems(GgrsSchedule, ResourceSystem s) { res_systems_.push_back(std::move(s.fn)); return *this; }
    App& add_observer(std::function<void(const SyncTestMismatch&)> f) { observers_.push_back(std::move(f)); return *this; }

    // ---- RollbackApp (rollback_app.rs:31-248) ----
    template <class T> App& rollback_component_with_copy() { return register_component<T>(BGR_STRATEGY_COPY); }
    // Clone of plain bytes -> an HBM column.  Clone of anything else (bevy's Sprite holds an Arc asset handle,
    // particles.rs:191) -> the type stays on the host in a side table keyed by row (= RollbackOrdered index, never
    // reused) and is rolled back there by the same request vectors: Save clones the table into a per-frame snapshot
    // (component_snapshot.rs:66-90), Load replaces it by a clone of the frame's snapshot = the four-way match of
    // component_snapshot.rs:99-115 for every entity at once; whether the entity exists is the alive mask in HBM.
    template <class T> App& rollback_component_with_clone() {
        if constexpr (std::is_trivially_copyable<T>::value) return register_component<T>(BGR_STRATEGY_CLONE);
        else { host_cols_[std::type_index(typeid(T))] = std::make_unique<HostColumn<T>>(); return *this; }
    }
    // commands.entity(row).insert(value) / .remove::<T>() / Query<&T> for a host-side component
    template <class T> void host_insert(uint32_t row, T value) {
        if (!entity_exists(row)) throw Panic(BGR_ERR_INVALID_ARGUMENT, "entity of row " + std::to_string(row) + " does not exist");
        host_col<T>().live.insert_or_assign(row, std::move(value));
    }
    template <class T> void host_remove(uint32_t row) { host_col<T>().live.erase(row); }
    template <class T> const T* host_get(uint32_t row) {
        auto& live = host_col<T>().live;
        auto it = live.find(row);
        return it != live.end() && entity_exists(row) ? &it->second : nullptr;
    }
    template <class T> std::vector<ggrs::Frame> host_snapshot_frames() {
        std::vector<ggrs::Frame> f;
        for (auto& kv : host_col<T>().snaps) f.push_back(kv.first);
        return f;
    }
    // a component single entities may lose / regain inside the window: Option<&mut T> in ComponentSnapshotPlugin::load
    // (component_snapshot.rs:99-115); see remove<T>() / insert<T>() below
    template <class T> App& rollback_optional_component_with_copy() { return register_component<T>(BGR_STRATEGY_COPY | BGR_STRATEGY_OPTIONAL); }
    template <class T> App& rollback_optional_component_with_clone() { return register_component<T>(BGR_STRATEGY_CLONE | BGR_STRATEGY_OPTIONAL); }
    template <class T> App& checksum_component(ByteRangeHasher h) { checksums_.push_back({col<T>(), h}); return *this; }
    template <class T> App& checksum_component_with_hash() { return checksum_component<T>(hash_bytes(0, uint32_t(sizeof(T)))); }

    // rollback_resource_with_copy / _with_clone (rollback_app.rs:171-176, 192-197) and
    // checksum_resource_with_hash (rollback_app.rs:213-218) for POD resources, host-side
    template <class R> App& rollback_resource_with_copy(const R& initial) {
        static_assert(std::is_trivially_copyable<R>::value, "POD resources only");
        std::vector<uint8_t> b(sizeof(R));
        std::memcpy(b.data(), &initial, sizeof(R));
        const std::type_index t(typeid(R));
        if (!resources_.count(t)) res_order_.push_back({t, uint32_t(sizeof(R))});
        resources_[t] = std::move(b);
        return *this;
    }
    template <class R> App& rollback_resource_with_clone(const R& initial) { return rollback_resource_with_copy<R>(initial); }
    template <class R> App& checksum_resource_with_hash() { res_checksummed_.push_back(std::type_index(typeid(R))); return *this; }
    template <class R> R& resource() {
        auto it = resources_.find(std::type_index(typeid(R)));
        if (it == resources_.end()) throw Panic(BGR_ERR_MISSING_RESOURCE, std::string("Requested resource does not exist: ") + typeid(R).name());
        return *reinterpret_cast<R*>(it->second.data());
    }

    template <class T> uint32_t col() const {
        auto it = columns_.find(std::type_index(typeid(T)));
        if (it == columns_.end()) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string("component not registered for rollback: ") + typeid(T).name());
        return it->second;
    }

    // ---- World access ----
    const LocalPlayers& local_players() const { return local_players_; }
    uint32_t spawn(uint32_t count) { finish(); uint32_t first = 0; check(bgr_spawn(engine_, count, &first)); return first; }
    // App(n, depth, device, BGR_CFG_GROWABLE): spawns grow the row capacity; reserve() grows it ahead of them
    void reserve(uint32_t rows) { finish(); check(bgr_reserve(engine_, rows)); }
    // {rows held without growing, most rows the engine can ever hold}
    std::pair<uint32_t, uint32_t> capacity() {
        finish();
        uint32_t cap = 0, ceiling = 0;
        check(bgr_capacity(engine_, &cap, &ceiling));
        return {cap, ceiling};
    }
    template <class T> void write(uint32_t first_row, const std::vector<T>& v) {
        finish();
        check(bgr_write_component(engine_, col<T>(), first_row, uint32_t(v.size()), v.data(), uint32_t(sizeof(T))));
    }
    template <class T> std::vector<T> read(uint32_t first_row, uint32_t count) {
        std::vector<T> v(count);
        check(bgr_read_component(engine_, col<T>(), first_row, count, v.data(), uint32_t(sizeof(T))));
        return v;
    }
    // commands.entity(row).remove::<T>() / .insert(value) / Query<Has<T>> for optional components
    template <class T> void remove(uint32_t row) { finish(); check(bgr_remove_component(engine_, col<T>(), row)); }
    template <class T> void insert(uint32_t row, const T& value) { finish(); check(bgr_insert_component(engine_, col<T>(), row, &value)); }
    template <class T> std::vector<uint8_t> has(uint32_t first_row, uint32_t count) {
        std::vector<uint8_t> v(count);
        check(bgr_has_component(engine_, col<T>(), first_row, count, v.data()));
        return v;
    }
    // Host edits (bgr_apply_edits): what an Update system or Commands do to rollback entities between frames, recorded
    // in order and sent as one queued batch by apply().  Equivalent to the single calls above in the same order.
    class Edits {
    public:
        explicit Edits(const App& app) : app_(app) {}
        template <class T> Edits& write(uint32_t first_row, const std::vector<T>& v) {
            for (const T& x : v) values_.insert(values_.end(), reinterpret_cast<const uint8_t*>(&x), reinterpret_cast<const uint8_t*>(&x) + sizeof(T));
            return add(BGR_EDIT_WRITE, app_.col<T>(), first_row, uint32_t(v.size()), 0, uint32_t(sizeof(T)), values_.size() - v.size() * sizeof(T));
        }
        // bytes [offset, offset + sizeof(F)) of T on `row`, e.g. write_field<Transform>(row, 0, translation)
        template <class T, class F> Edits& write_field(uint32_t row, uint32_t offset, const F& field) {
            const size_t at = push_bytes(&field, sizeof(F));
            return add(BGR_EDIT_WRITE, app_.col<T>(), row, 1, offset, uint32_t(sizeof(F)), at);
        }
        template <class T> Edits& insert(uint32_t row, const T& value) {
            const size_t at = push_bytes(&value, sizeof(T));
            return add(BGR_EDIT_INSERT, app_.col<T>(), row, 0, 0, 0, at);
        }
        template <class T> Edits& remove(uint32_t row) { return add(BGR_EDIT_REMOVE, app_.col<T>(), row, 0, 0, 0, 0); }
        Edits& despawn(uint32_t row) { return add(BGR_EDIT_DESPAWN, 0, row, 0, 0, 0, 0); }
        Edits& spawn(uint32_t count) { return add(BGR_EDIT_SPAWN, 0, 0, count, 0, 0, 0); }
        size_t size() const { return records_.size(); }

    private:
        friend class App;
        size_t push_bytes(const void* p, size_t n) {
            const size_t at = values_.size();
            values_.insert(values_.end(), static_cast<const uint8_t*>(p), static_cast<const uint8_t*>(p) + n);
            return at;
        }
        Edits& add(uint32_t kind, uint32_t column, uint32_t row, uint32_t count, uint32_t offset, uint32_t len, size_t at) {
            records_.push_back(bgr_edit{kind, column, row, count, offset, len, uint32_t(at), 0u});
            return *this;
        }
        const App& app_;
        std::vector<bgr_edit> records_;
        std::vector<uint8_t> values_;
    };
    // enqueues the batch behind the submitted request vectors and empties it; returns without waiting for the GPU
    void apply(Edits& edits) {
        finish();
        check(bgr_apply_edits(engine_, edits.records_.data(), uint32_t(edits.records_.size()), edits.values_.data(), edits.values_.size()));
        edits.records_.clear();
        edits.values_.clear();
    }
    // asynchronous host mirror of bytes [offset, offset+len) of every T in rows [first_row, first_row+count):
    // `dst` from bgr_host_alloc; readable after download_wait(ticket)
    template <class T> uint32_t download_begin(uint32_t offset, uint32_t len, uint32_t first_row, uint32_t count, void* dst) {
        uint32_t ticket = 0;
        check(bgr_download_begin(engine_, col<T>(), offset, len, first_row, count, dst, &ticket));
        return ticket;
    }
    void download_wait(uint32_t ticket) { check(bgr_download_wait(engine_, ticket)); }
    // change feed: only the rows whose existence, presence or tracked bytes changed since the last report
    // (include/bevy_ggrs_b200.h "change feed"); `dst` from bgr_host_alloc, records_cap * record_bytes bytes
    uint32_t feed_create(const std::vector<bgr_feed_field>& fields) {
        uint32_t feed = 0;
        check(bgr_feed_create(engine_, fields.data(), uint32_t(fields.size()), &feed));
        return feed;
    }
    void feed_reset(uint32_t feed) { check(bgr_feed_reset(engine_, feed)); }
    uint32_t feed_begin(uint32_t feed, void* dst, uint32_t records_cap) {
        uint32_t ticket = 0;
        check(bgr_feed_begin(engine_, feed, dst, records_cap, &ticket));
        return ticket;
    }
    bgr_feed_info feed_wait(uint32_t ticket) {
        bgr_feed_info info{};
        check(bgr_feed_wait(engine_, ticket, &info));
        return info;
    }
    // Applies the records of a feed whose field `field` is the whole of T to a row map: a record whose state has the
    // field's bit inserts or updates the row's T, any other record (despawned, un-spawned, component removed) erases it.
    // Rows that exist again after a rollback and rows spawned on the GPU come back as ordinary inserts.
    template <class T, class Map>
    static void apply_feed(const void* records, const bgr_feed_info& info, uint32_t field, uint32_t field_offset, Map& rows) {
        static_assert(std::is_trivially_copyable<T>::value, "rollback components are POD");
        const uint8_t* r = static_cast<const uint8_t*>(records);
        for (uint32_t i = 0; i < info.n_records; ++i, r += info.record_bytes) {
            uint32_t row = 0, state = 0;
            std::memcpy(&row, r, 4);
            std::memcpy(&state, r + 4, 4);
            if (state & (2u << field)) {
                T v;
                std::memcpy(&v, r + 8 + field_offset, sizeof(T));
                rows[row] = v;
            } else {
                rows.erase(row);
            }
        }
    }
    // GgrsComponentSnapshots<T>::peek(frame) (mod.rs:233-240)
    template <class T> std::optional<std::vector<T>> peek(ggrs::Frame frame, uint32_t first_row, uint32_t count) {
        std::vector<T> v(count);
        int32_t found = 0;
        check(bgr_peek(engine_, frame, col<T>(), first_row, count, v.data(), uint32_t(sizeof(T)), nullptr, &found));
        if (!found) return std::nullopt;
        return v;
    }
    uint64_t active_count() { uint64_t n = 0; check(bgr_active_count(engine_, &n)); return n; }
    int32_t rollback_frame_count() { int32_t f = 0; check(bgr_rollback_frame_count(engine_, &f)); return f; }
    int32_t confirmed_frame_count() { int32_t f = 0; check(bgr_confirmed_frame_count(engine_, &f)); return f; }
    uint64_t launch_count() { uint64_t n = 0; check(bgr_launch_count(engine_, &n)); return n; }
    bgr_engine* engine() { finish(); return engine_; }
    const std::vector<bgr_checksum>& last_checksums() const { return last_checksums_; }

    // ---- one Bevy frame: run_ggrs_schedules (schedule_systems.rs:19-83) ----
    void update() {
        finish();
        // bevy Time<Real>: zero delta on the first update, then TimeUpdateStrategy::ManualDuration(1/60 s)
        const uint64_t delta = first_update_ ? 0 : 16666667ull;
        first_update_ = false;
        const uint64_t fps_delta = run_slow_ ? 1000000000ull * 11 / (uint64_t(cfg_.fps) * 10) : 1000000000ull / cfg_.fps;
        accumulator_ns_ += delta;
        if (session_ && session_->kind == Session::P2PKind) session_->p2p->poll_remote_clients();             // :43-53
        if (session_ && session_->kind == Session::SpectatorKind) session_->spectator->poll_remote_clients();
        while (accumulator_ns_ >= fps_delta) {
            accumulator_ns_ -= fps_delta;
            if (!session_) {  // :70-79 "No session has been started yet, reset time data and snapshots"
                accumulator_ns_ = 0; run_slow_ = false;
                local_players_.handles.clear();
                check(bgr_reset_session(engine_));  // RollbackFrameCount(0), ConfirmedFrameCount(-1), MaxPredictionWindow(8)
                return;
            }
            tick();
        }
    }
    // exactly one GGRS tick (benches)
    void step() { finish(); tick(); }
    uint32_t max_prediction_window() { uint32_t v = 0; check(bgr_max_prediction_window(engine_, &v)); return v; }
    std::vector<int32_t> snapshot_frames() {
        int32_t f[128]; uint32_t n = 0;
        check(bgr_snapshot_frames(engine_, f, 128, &n));
        return std::vector<int32_t>(f, f + std::min<uint32_t>(n, 128));
    }

    // ---- desync capture (App(..., BGR_CFG_DESYNC_CAPTURE)) ----
    // Where a SyncTest re-simulation diverged: the frame's first-recorded image against its re-saved one, compared in HBM
    // (bgr_desync_diff).  Call it from a SyncTestMismatch observer with one of ev.mismatched_frames.  found == false: the
    // frame has no retained first image or no current snapshot.  An empty report for a mismatched frame means the
    // difference is in state the engine does not hold (resources, host-side component tables).
    struct DesyncReport {
        bool found = false;
        bgr_desync_summary summary{};
        std::vector<bgr_desync_column> columns;   // by column index (registration order)
        std::vector<std::string> column_names;    // typeid names, same index
        std::vector<bgr_desync_record> records;   // the first max_records, ascending (row, column, word)
    };
    DesyncReport desync_report(ggrs::Frame frame, uint32_t max_records = 64) {
        finish();
        DesyncReport r;
        r.columns.resize(pending_cols_.size());
        r.records.resize(max_records);
        uint32_t n = 0;
        int32_t found = 0;
        check(bgr_desync_diff(engine_, frame, &r.summary, r.columns.data(), uint32_t(r.columns.size()), r.records.data(),
                              max_records, &n, &found));
        r.found = found != 0;
        r.records.resize(n);
        for (auto& c : pending_cols_) r.column_names.push_back(c.name);
        return r;
    }

    // ---- P2P desync reports (GgrsEvent::DesyncDetected: the frame is confirmed and the other image is remote) ----
    // retain_confirmed before the first update keeps the confirmed multiples of the session's desync interval; the peers
    // exchange frame_digest results over the game's own channel, digest_mismatch (bgr_digest_mismatch, the one reader
    // of the format) names the blocks, the remote peer export_blocks those below its own header.n_blocks (possibly
    // none) and the local peer diff_remote's the blob, which also compares the local blocks the remote frame lacks.
    App& retain_confirmed(uint32_t interval, uint32_t count) {  // applied by the engine's build, like the registrations
        if (engine_) throw Panic(BGR_ERR_STATE, "retain_confirmed must be called before the App is built");
        retain_ = {interval, count};
        return *this;
    }
    std::vector<int32_t> retained_frames() {
        finish();
        int32_t f[64]; uint32_t n = 0;
        check(bgr_retained_frames(engine_, f, 64, &n));
        return std::vector<int32_t>(f, f + std::min<uint32_t>(n, 64));
    }
    struct FrameDigest {
        bool found = false;
        bgr_frame_digest_header header{};
        std::vector<uint64_t> words;  // header.n_blocks x (header.n_columns + 1)
    };
    FrameDigest frame_digest(ggrs::Frame frame) {
        finish();
        FrameDigest d;
        d.words.resize(size_t((capacity().first + BGR_DIGEST_BLOCK_ROWS - 1) / BGR_DIGEST_BLOCK_ROWS) * (pending_cols_.size() + 1));
        int32_t found = 0;
        check(bgr_frame_digest(engine_, frame, &d.header, d.words.data(), uint32_t(d.words.size()), &found));
        d.found = found != 0;
        d.words.resize(d.found ? size_t(d.header.n_blocks) * (d.header.n_columns + 1) : 0);
        return d;
    }
    // blocks whose digests differ, ascending; *host_state_differs: bit 0 ParticleRng, bit 1 Time<GgrsTime>
    static std::vector<uint32_t> digest_mismatch(const FrameDigest& local, const FrameDigest& remote,
                                                 uint32_t* host_state_differs = nullptr) {
        std::vector<uint32_t> blocks(std::max<uint32_t>(1, std::max(local.header.n_blocks, remote.header.n_blocks)));
        uint32_t n = 0, host = 0;
        check(bgr_digest_mismatch(&local.header, local.words.data(), &remote.header, remote.words.data(), blocks.data(),
                                  uint32_t(blocks.size()), &n, &host));
        blocks.resize(std::min<size_t>(n, blocks.size()));
        if (host_state_differs) *host_state_differs = host;
        return blocks;
    }
    // the export blob of `blocks` (ascending) of a queued or retained frame; empty when neither holds it
    std::vector<uint8_t> export_blocks(ggrs::Frame frame, const std::vector<uint32_t>& blocks) {
        finish();
        size_t bytes = 0;
        int32_t found = 0;
        check(bgr_frame_export(engine_, frame, blocks.data(), uint32_t(blocks.size()), nullptr, 0, &bytes, &found));
        if (!found) return {};
        std::vector<uint8_t> blob(bytes);
        check(bgr_frame_export(engine_, frame, blocks.data(), uint32_t(blocks.size()), blob.data(), blob.size(), &bytes, &found));
        return blob;
    }
    // the local image of `frame` ("first") against a peer's blob ("latest"): the records of desync_report
    DesyncReport diff_remote(ggrs::Frame frame, const std::vector<uint8_t>& blob, uint32_t max_records = 64) {
        finish();
        DesyncReport r;
        r.columns.resize(pending_cols_.size());
        r.records.resize(max_records);
        uint32_t n = 0;
        int32_t found = 0;
        check(bgr_desync_diff_remote(engine_, frame, blob.data(), blob.size(), &r.summary, r.columns.data(),
                                     uint32_t(r.columns.size()), r.records.data(), max_records, &n, &found));
        r.found = found != 0;
        r.records.resize(n);
        for (auto& c : pending_cols_) r.column_names.push_back(c.name);
        return r;
    }

    // ---- world checkpoints (bgr_checkpoint_save / bgr_checkpoint_restore; INTEGRATION.md "World checkpoints") ----
    // The engine blob followed by the App's rollback resources of the frame: u32 count, then per resource in
    // registration order u32 present, u32 len, the bytes, zero padding to a multiple of 4 (plugin.py writes the same).
    // Refused while host-side component tables are registered (their values are not plain bytes) and, with resources
    // registered, for a frame whose resource snapshot the App no longer holds (a retained frame).  Empty: the engine
    // holds neither a queued nor a retained snapshot of the frame.
    std::vector<uint8_t> checkpoint(ggrs::Frame frame) {
        checkpoint_args();
        auto rs = resource_snapshot(frame);
        size_t bytes = 0;
        int32_t found = 0;
        check(bgr_checkpoint_save(engine_, frame, nullptr, 0, &bytes, &found));
        if (!found) return {};
        std::vector<uint8_t> blob(bytes);  // an upper bound; the call reports the exact size
        check(bgr_checkpoint_save(engine_, frame, blob.data(), blob.size(), &bytes, &found));
        blob.resize(bytes);
        put_resources(rs == res_store_.end() ? Resources{} : rs->second, &blob);
        return blob;
    }
    // The engine's checkpoint delta of `frame` against `base_frame` (bgr_checkpoint_save_delta) followed by the App's
    // resources of `frame`, in checkpoint()'s section.  Refused where checkpoint(frame) is; empty: the engine holds either
    // frame neither queued nor retained.
    std::vector<uint8_t> checkpoint_delta(ggrs::Frame frame, ggrs::Frame base_frame) {
        checkpoint_args();
        auto rs = resource_snapshot(frame);
        size_t bytes = 0;
        int32_t found = 0;
        check(bgr_checkpoint_save_delta(engine_, frame, base_frame, nullptr, 0, &bytes, &found));
        if (!found) return {};
        std::vector<uint8_t> blob(bytes);  // an upper bound; the call reports the exact size
        check(bgr_checkpoint_save_delta(engine_, frame, base_frame, blob.data(), blob.size(), &bytes, &found));
        blob.resize(bytes);
        put_resources(rs == res_store_.end() ? Resources{} : rs->second, &blob);
        return blob;
    }
    // ---- replays (bgr_replay; INTEGRATION.md "Replays") ----
    // A recorded input log (inputs[j * n_players + h], n_players per frame) run from the current frame f0 in one call.  It
    // leaves the App as handle_requests of the stream [Save(f) if f % checksum_interval == 0, Advance(inputs[j])],
    // f = f0 + j, would leave it, except that no snapshot is pushed: the engine re-simulates the world, and the App steps
    // its rollback resources through the same frames on the host and XORs their checksum parts in.  The engine's ring is
    // not touched, so neither is the App's resource store.  Resource systems run at frames the world is not at: they must
    // not read the world.  Returns the checksums of the frames f with f % checksum_interval == 0, before they are
    // advanced, in order.  Refused while host-side component tables are registered.  A refused replay changes nothing; a
    // non-finite value at a checksum frame throws BGR_ERR_NON_FINITE after the whole log ran and the resources were
    // committed.
    std::vector<std::pair<ggrs::Frame, unsigned __int128>> replay(const std::vector<uint8_t>& inputs, uint32_t n_players,
                                                                  uint32_t checksum_interval) {
        const struct bgr_replay r = replay_args(inputs, n_players, checksum_interval);
        std::vector<bgr_checksum> cs(checksum_cap(r) + 1);
        uint32_t got = 0;
        ResourceSteps steps = step_resources(r.n_frames, checksum_interval, 0);
        commit_replay(steps, bgr_replay(engine_, &r, cs.data(), uint32_t(cs.size() - 1), &got));
        return fold_checksums(cs, got, steps);
    }

    // replay() that also writes an App checkpoint of every frame f with f % keyframe_interval == 0, before it is advanced,
    // to `keyframes` as (frame, blob), in order (bgr_replay_keyframes): the engine's keyframe followed by the App's
    // resources of the frame, byte for byte what checkpoint(f) writes on an App that ticked to f and saved it.  The
    // buffers are sized by the call's query, which runs nothing.
    std::vector<std::pair<ggrs::Frame, unsigned __int128>> replay_keyframes(
        const std::vector<uint8_t>& inputs, uint32_t n_players, uint32_t checksum_interval, uint32_t keyframe_interval,
        std::vector<std::pair<ggrs::Frame, std::vector<uint8_t>>>* keyframes) {
        const struct bgr_replay r = replay_args(inputs, n_players, checksum_interval);
        struct bgr_keyframes kf;
        std::memset(&kf, 0, sizeof kf);
        kf.interval = keyframe_interval;
        uint32_t got = 0, n_kf = 0;
        size_t bytes = 0;
        check(bgr_replay_keyframes(engine_, &r, &kf, nullptr, 0, &got, &n_kf, &bytes));  // the query
        std::vector<uint8_t> dst(std::max<size_t>(bytes, 1));
        std::vector<bgr_keyframe> index(std::max<uint32_t>(n_kf, 1));
        kf.dst = dst.data();
        kf.dst_cap = bytes;
        kf.index = index.data();
        kf.index_cap = n_kf;
        std::vector<bgr_checksum> cs(checksum_cap(r) + 1);
        ResourceSteps steps = step_resources(r.n_frames, checksum_interval, keyframe_interval);
        commit_replay(steps, bgr_replay_keyframes(engine_, &r, &kf, cs.data(), uint32_t(cs.size() - 1), &got, &n_kf, &bytes));
        keyframes->clear();
        for (uint32_t i = 0; i < n_kf && i < kf.index_cap; ++i) {
            keyframes->emplace_back(index[i].frame, std::vector<uint8_t>(dst.begin() + index[i].offset,
                                                                         dst.begin() + index[i].offset + index[i].bytes));
            auto snap = steps.snapshots.find(index[i].frame);
            put_resources(snap == steps.snapshots.end() ? Resources{} : snap->second, &keyframes->back().second);
        }
        return fold_checksums(cs, got, steps);
    }

    // replay() that also samples rows [first_row, first_row + n_rows) at every frame f with f % trace_interval == 0,
    // before it is advanced (bgr_replay_trace).  `samples` gets each sample's (frame, row count) and `records`
    // n_samples * n_rows change-feed records over `fields`, sample-major: engine fields only, while the checksums include
    // the resources' parts.  The buffers are sized by the call's query, which runs nothing.
    std::vector<std::pair<ggrs::Frame, unsigned __int128>> replay_trace(
        const std::vector<uint8_t>& inputs, uint32_t n_players, uint32_t checksum_interval, uint32_t trace_interval,
        const std::vector<bgr_feed_field>& fields, uint32_t first_row, uint32_t n_rows, std::vector<bgr_trace_sample>* samples,
        std::vector<uint8_t>* records) {
        const struct bgr_replay r = replay_args(inputs, n_players, checksum_interval);
        struct bgr_trace t;
        std::memset(&t, 0, sizeof t);
        t.interval = trace_interval;
        t.first_row = first_row;
        t.n_rows = n_rows;
        t.n_fields = uint32_t(fields.size());
        t.fields = fields.data();
        uint32_t got = 0, n_s = 0;
        size_t bytes = 0;
        check(bgr_replay_trace(engine_, &r, &t, nullptr, 0, &got, &n_s, &bytes));  // the query
        records->assign(std::max<size_t>(bytes, 1), 0);  // never a null dst, which is the query: a log may take no sample
        samples->assign(std::max<uint32_t>(n_s, 1), bgr_trace_sample{});
        t.dst = records->data();
        t.dst_cap = bytes;
        t.samples = samples->data();
        t.samples_cap = n_s;
        std::vector<bgr_checksum> cs(checksum_cap(r) + 1);
        ResourceSteps steps = step_resources(r.n_frames, checksum_interval, 0);
        commit_replay(steps, bgr_replay_trace(engine_, &r, &t, cs.data(), uint32_t(cs.size() - 1), &got, &n_s, &bytes));
        records->resize(bytes);
        samples->resize(n_s);
        return fold_checksums(cs, got, steps);
    }

    // Replaces the world and the App's resources with a checkpoint's.  The resource section is checked before the
    // engine restores, so a refused blob changes nothing.
    void restore_checkpoint(const std::vector<uint8_t>& blob) {
        checkpoint_args();
        bgr_checkpoint_header h;
        if (blob.size() < sizeof h) throw Panic(BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its header");
        std::memcpy(&h, blob.data(), sizeof h);
        const size_t engine_bytes = engine_part(blob, sizeof h, h.n_blocks, h.payload_bytes, "checkpoint");
        ResourceMap res = take_resources(blob, engine_bytes, "checkpoint");
        check(bgr_checkpoint_restore(engine_, blob.data(), engine_bytes));
        set_restored_resources(h.frame, res);
    }

    // Replaces the world and the App's resources with the target frame of `delta` (from checkpoint_delta()), given the
    // App checkpoint `base` it was written against.  Both resource sections are checked before the engine restores, so
    // a refused pair changes nothing.
    void restore_checkpoint_delta(const std::vector<uint8_t>& base, const std::vector<uint8_t>& delta) {
        checkpoint_args();
        bgr_checkpoint_header bh;
        bgr_checkpoint_delta_header dh;
        if (base.size() < sizeof bh) throw Panic(BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its header");
        if (delta.size() < sizeof dh) throw Panic(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta truncated: shorter than its header");
        std::memcpy(&bh, base.data(), sizeof bh);
        std::memcpy(&dh, delta.data(), sizeof dh);
        const size_t base_bytes = engine_part(base, sizeof bh, bh.n_blocks, bh.payload_bytes, "checkpoint");
        const size_t delta_bytes = engine_part(delta, sizeof dh, dh.n_blocks, dh.payload_bytes, "checkpoint delta");
        take_resources(base, base_bytes, "checkpoint");
        ResourceMap res = take_resources(delta, delta_bytes, "checkpoint delta");
        check(bgr_checkpoint_restore_delta(engine_, base.data(), base_bytes, delta.data(), delta_bytes));
        set_restored_resources(dh.frame, res);
    }

private:
    void checkpoint_args() {
        finish();
        if (!host_cols_.empty())
            throw Panic(BGR_ERR_UNSUPPORTED, "an App with host-side component tables cannot be checkpointed: their values are not plain bytes");
    }
    using Resources = std::map<std::type_index, std::vector<uint8_t>>;  // ResourceMap, declared below

    // checks that the App can replay `inputs` from its current frame and describes the log
    struct bgr_replay replay_args(const std::vector<uint8_t>& inputs, uint32_t n_players, uint32_t checksum_interval) {
        finish();
        if (!host_cols_.empty())
            throw Panic(BGR_ERR_UNSUPPORTED, "an App with host-side component tables cannot replay: their rows follow spawns and "
                                             "despawns a replay does not report frame by frame");
        if (n_players ? inputs.size() % n_players != 0 : !inputs.empty())
            throw Panic(BGR_ERR_INVALID_ARGUMENT, "the input log is not a whole number of frames of n_players bytes");
        if (!res_order_.empty() && res_frame_ != rollback_frame_count())
            throw Panic(BGR_ERR_STATE, "the App's resources are at frame " + std::to_string(res_frame_) + ", its world at frame " +
                                           std::to_string(rollback_frame_count()));
        struct bgr_replay r;
        std::memset(&r, 0, sizeof r);
        r.n_players = n_players;
        r.n_frames = n_players ? uint32_t(inputs.size() / n_players) : 0u;
        r.checksum_interval = checksum_interval;
        r.inputs = inputs.data();
        return r;
    }
    // the number of checksum frames of replay `r` from the current frame
    size_t checksum_cap(const struct bgr_replay& r) {
        const int64_t f0 = rollback_frame_count(), n = r.n_frames, k = r.checksum_interval;
        return k && f0 >= 0 ? size_t((f0 + n + k - 1) / k - (f0 + k - 1) / k) : 0u;
    }
    // The resources of a replay stepped through its frames: the resources and frame before it, the resource parts of the
    // checksum frames in order, and the resource snapshots of the keyframe frames.
    struct ResourceSteps {
        Resources before;
        ggrs::Frame frame_before = 0;
        std::vector<uint64_t> parts;
        std::map<ggrs::Frame, Resources> snapshots;
    };
    // The request-free counterpart of handle_resource_requests: steps resources_ and res_frame_ through the n_frames of a
    // replay as its Saves and Advances would, before the engine runs it.  At a checksum frame the resource part, at a
    // keyframe frame the resource snapshot, then the resource systems.  A throw (an absent checksummed resource, a
    // resource system) restores the resources first.
    ResourceSteps step_resources(uint32_t n_frames, uint32_t checksum_interval, uint32_t keyframe_interval) {
        ResourceSteps st;
        if (res_order_.empty()) return st;
        st.before = resources_;
        st.frame_before = res_frame_;
        try {
            for (uint32_t j = 0; j < n_frames; ++j) {
                if (checksum_interval && int64_t(res_frame_) % checksum_interval == 0) st.parts.push_back(resource_part());
                if (keyframe_interval && int64_t(res_frame_) % keyframe_interval == 0) st.snapshots[res_frame_] = resources_;
                res_frame_ += 1;
                for (auto& f : res_systems_) f(*this);
            }
        } catch (...) {
            resources_ = st.before;
            res_frame_ = st.frame_before;
            throw;
        }
        return st;
    }
    // Once the engine's replay call returned `rc`: BGR_OK or BGR_ERR_NON_FINITE (the log ran; thrown after this) keep the
    // stepped resources, any other status restores them and throws.
    void commit_replay(const ResourceSteps& st, int rc) {
        if (rc != BGR_OK && rc != BGR_ERR_NON_FINITE && !res_order_.empty()) {
            resources_ = st.before;
            res_frame_ = st.frame_before;
        }
        check(rc);
    }
    // the first `got` checksums of a replay with the resource parts XORed in
    static std::vector<std::pair<ggrs::Frame, unsigned __int128>> fold_checksums(std::vector<bgr_checksum>& cs, uint32_t got,
                                                                                const ResourceSteps& st) {
        std::vector<std::pair<ggrs::Frame, unsigned __int128>> out;
        for (uint32_t i = 0; i < got && i + 1 < cs.size(); ++i) {
            if (i < st.parts.size()) cs[i].lo ^= st.parts[i];
            out.emplace_back(cs[i].frame, (static_cast<unsigned __int128>(cs[i].hi) << 64) | cs[i].lo);
        }
        return out;
    }
    // the XOR of the checksummed resources' seahashes (resource_checksum.rs:63-82: the resource must exist)
    uint64_t resource_part() const {
        uint64_t part = 0;
        for (auto& t : res_checksummed_) { auto& b = resources_.at(t); part ^= bgr_seahash(b.data(), b.size()); }
        return part;
    }
    // the App's resource snapshot of `frame` (end(): none, and none is needed without registered resources)
    std::map<ggrs::Frame, Resources>::const_iterator resource_snapshot(ggrs::Frame frame) const {
        auto rs = res_store_.find(frame);
        if (!res_order_.empty() && rs == res_store_.end())
            throw Panic(BGR_ERR_NO_SNAPSHOT, "the App holds no resource snapshot of frame " + std::to_string(frame));
        return rs;
    }
    // appends the resource section of a resource snapshot to `blob`
    void put_resources(const Resources& snap, std::vector<uint8_t>* blob) const {
        auto put = [blob](uint32_t v) { const uint8_t* p = reinterpret_cast<const uint8_t*>(&v); blob->insert(blob->end(), p, p + 4); };
        put(uint32_t(res_order_.size()));
        for (const auto& r : res_order_) {
            auto it = snap.find(r.first);
            const bool present = it != snap.end();
            put(present ? 1u : 0u);
            put(present ? uint32_t(it->second.size()) : 0u);
            if (!present) continue;
            blob->insert(blob->end(), it->second.begin(), it->second.end());
            blob->resize(blob->size() + (4 - it->second.size() % 4) % 4, 0);
        }
    }
    // the bytes of the engine blob at the start of `blob` (`head`: its header's size), which a resource section follows
    static size_t engine_part(const std::vector<uint8_t>& blob, size_t head, uint32_t n_blocks, uint64_t payload_bytes,
                              const char* what) {
        const uint64_t prefix = head + 8ull * (uint64_t(n_blocks) + 1);
        if (payload_bytes > blob.size() || prefix + payload_bytes > blob.size())
            throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string(what) + " truncated: no resource section");
        return size_t(prefix + payload_bytes);
    }
    // the resource section of `blob` from byte `at` to its end, checked against the App's registration
    Resources take_resources(const std::vector<uint8_t>& blob, size_t at, const char* what) const {
        auto take = [&](size_t n) {
            if (n > blob.size() - at) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string(what) + " truncated: its resource section is incomplete");
            at += n;
            return blob.data() + at - n;
        };
        auto get = [&]() { uint32_t v; std::memcpy(&v, take(4), 4); return v; };
        if (get() != res_order_.size()) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string("the ") + what + "'s resources are not the App's");
        ResourceMap res;
        for (const auto& r : res_order_) {
            const uint32_t present = get(), n = get();
            if (present > 1 || n != (present ? r.second : 0u))
                throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string("resource ") + r.first.name() + ": bad presence or length");
            if (!present) continue;
            const uint8_t* p = take(n);
            res[r.first] = std::vector<uint8_t>(p, p + n);
            const uint8_t* pad = take((4 - n % 4) % 4);
            for (uint32_t i = 0; i < (4 - n % 4) % 4; ++i)
                if (pad[i]) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string("resource ") + r.first.name() + ": non-zero padding");
        }
        if (at != blob.size()) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string(what) + " overlong: bytes follow its resource section");
        return res;
    }
    void set_restored_resources(ggrs::Frame frame, const Resources& res) {
        resources_ = res;
        res_store_.clear();
        if (!res_order_.empty()) res_store_[frame] = res;
        res_frame_ = frame;
    }
    template <class T> App& register_component(uint32_t strategy) {
        static_assert(std::is_trivially_copyable<T>::value, "only POD components cross the C ABI");
        pending_cols_.push_back({std::type_index(typeid(T)), typeid(T).name(), uint32_t(sizeof(T)), strategy});
        columns_[std::type_index(typeid(T))] = uint32_t(pending_cols_.size() - 1);
        return *this;
    }
    void finish() {  // end of App::build
        if (engine_) return;
        check(bgr_engine_create(&cfg_, &engine_));
        for (auto& c : pending_cols_) { uint32_t id = 0; check(bgr_rollback_component(engine_, c.name.c_str(), c.bytes, c.strategy, &id)); }
        for (auto& ck : checksums_)
            check(bgr_checksum_component(engine_, ck.first, BGR_HASH_BYTES, ck.second.offset, ck.second.len,
                                         ck.second.assert_finite ? BGR_HASH_FLAG_ASSERT_FINITE_F32 : 0u));
        for (auto& s : systems_)
            check(bgr_add_system(engine_, s.id, s.columns.data(), uint32_t(s.columns.size()), s.params.data(), uint32_t(s.params.size())));
        if (retain_.second) check(bgr_retain_confirmed(engine_, retain_.first, retain_.second));
        check(bgr_build(engine_));
        for (auto& f : startup_) f(*this);
    }

    void tick() {  // :59-69: depending on the session type, doing a single update looks a bit different
        switch (session_->kind) {
        case Session::SyncTestKind: run_synctest(*session_->synctest); break;
        case Session::P2PKind: run_slow_ = session_->p2p->frames_ahead() > 0; run_p2p(*session_->p2p); break;
        case Session::SpectatorKind: run_spectator(*session_->spectator); break;
        }
    }

    // run_p2p (schedule_systems.rs:137-168)
    void run_p2p(ggrs::P2PTraceSession& sess) {
        local_players_.handles = sess.local_player_handles();
        if (sess.current_state() != ggrs::SessionState::Running) return;
        local_inputs_.reset();
        for (auto& f : read_inputs_) f(*this);
        if (!local_inputs_)
            throw Panic(BGR_ERR_MISSING_RESOURCE, "No local player inputs found. Did you insert systems into the ReadInputs schedule?");
        for (auto& kv : local_inputs_->inputs) sess.add_local_input(kv.first, kv.second);
        const auto requests = sess.advance_frame();
        // the numbers handle_requests reads from a P2P session before every request (:203-206)
        bgr_session_info info{BGR_SESSION_P2P, uint32_t(sess.max_prediction()), 0, sess.confirmed_frame()};
        handle_requests(requests, info, [&](ggrs::Frame f, unsigned __int128 c) { sess.save_cell(f, c); });
    }

    // run_spectator (schedule_systems.rs:120-135): only AdvanceFrame requests, several per tick when catching up
    void run_spectator(ggrs::SpectatorTraceSession& sess) {
        if (sess.current_state() != ggrs::SessionState::Running) return;
        const auto requests = sess.advance_frame();
        if (requests.empty()) return;  // PredictionThreshold: "Waiting for input from host."
        bgr_session_info info{BGR_SESSION_SPECTATOR, 0, 0, 0};  // max_prediction forced to 0, confirmed = current frame (:199-201, :209)
        handle_requests(requests, info, [](ggrs::Frame, unsigned __int128) {});
    }

    // run_synctest (schedule_systems.rs:85-118)
    void run_synctest(ggrs::SyncTestSession& sess) {
        local_players_.handles.clear();
        for (size_t i = 0; i < sess.num_players(); ++i) local_players_.handles.push_back(i);
        local_inputs_.reset();
        for (auto& f : read_inputs_) f(*this);  // world.run_schedule(ReadInputs)
        if (!local_inputs_)
            throw Panic(BGR_ERR_MISSING_RESOURCE, "No local player inputs found. Did you insert systems into the ReadInputs schedule?");
        for (auto& kv : local_inputs_->inputs) sess.add_local_input(kv.first, kv.second);
        std::vector<ggrs::GgrsRequest> requests;
        ggrs::MismatchedChecksum err;
        if (sess.advance_frame(requests, err)) {
            bgr_session_info info{BGR_SESSION_SYNCTEST, uint32_t(sess.max_prediction()), uint32_t(sess.check_distance()), 0};
            handle_requests(requests, info, [&](ggrs::Frame f, unsigned __int128 c) { sess.save_cell(f, c); });
        } else {  // :104-115
            SyncTestMismatch ev{err.current_frame, err.mismatched_frames};
            for (auto& o : observers_) o(ev);
        }
    }

    // handle_requests (schedule_systems.rs:170-289): ONE C-ABI call for the whole vector
    void handle_requests(const std::vector<ggrs::GgrsRequest>& requests, const bgr_session_info& info,
                         const std::function<void(ggrs::Frame, unsigned __int128)>& save_cell) {
        std::vector<bgr_request> reqs(requests.size());
        for (size_t i = 0; i < requests.size(); ++i) {
            bgr_request& q = reqs[i];
            std::memset(&q, 0, sizeof q);
            q.kind = uint32_t(requests[i].kind);
            q.frame = requests[i].frame;
            q.n_players = uint32_t(requests[i].inputs.size());
            for (size_t p = 0; p < requests[i].inputs.size() && p < BGR_MAX_PLAYERS; ++p) {
                q.inputs[p] = requests[i].inputs[p].first;
                q.status[p] = uint8_t(requests[i].inputs[p].second);
            }
        }
        last_checksums_.assign(BGR_MAX_REQUESTS, bgr_checksum{});
        uint32_t n = 0;
        check(bgr_handle_requests(engine_, &info, reqs.data(), uint32_t(reqs.size()), last_checksums_.data(), BGR_MAX_REQUESTS, &n));
        last_checksums_.resize(n);
        if (!resources_.empty()) handle_resource_requests(requests);
        if (!host_cols_.empty()) handle_host_component_requests(requests);
        for (auto& cs : last_checksums_)  // cell.save(frame, None, checksum) (:231-236)
            save_cell(cs.frame, (static_cast<unsigned __int128>(cs.hi) << 64) | cs.lo);
    }

    // host-side half of handle_requests for resources: the same request vector replayed on a few bytes
    void handle_resource_requests(const std::vector<ggrs::GgrsRequest>& requests) {
        size_t k = 0;
        for (const auto& r : requests) {
            if (r.kind == ggrs::GgrsRequest::SaveGameState) {
                res_store_[res_frame_] = resources_;
                const uint64_t part = resource_part();
                if (k < last_checksums_.size()) last_checksums_[k].lo ^= part;
                ++k;
            } else if (r.kind == ggrs::GgrsRequest::LoadGameState) {
                res_frame_ = r.frame;
                resources_ = res_store_.at(r.frame);
            } else {
                res_frame_ += 1;
                for (auto& f : res_systems_) f(*this);
            }
        }
        int32_t frames[128]; uint32_t nf = 0;
        check(bgr_snapshot_frames(engine_, frames, 128, &nf));
        for (auto it = res_store_.begin(); it != res_store_.end();) {
            bool alive = false;
            for (uint32_t i = 0; i < nf && i < 128; ++i) alive = alive || frames[i] == it->first;
            it = alive ? std::next(it) : res_store_.erase(it);
        }
    }

    // host-side half of handle_requests for non-POD components (see rollback_component_with_clone)
    struct HostColumnBase {
        virtual ~HostColumnBase() = default;
        virtual void save(ggrs::Frame f) = 0;
        virtual void load(ggrs::Frame f) = 0;
        virtual void prune(const std::vector<uint8_t>& alive, const std::vector<int32_t>& kept_frames) = 0;
        virtual bool empty() const = 0;
    };
    template <class T> struct HostColumn : HostColumnBase {
        std::map<uint32_t, T> live;
        std::map<ggrs::Frame, std::map<uint32_t, T>> snaps;
        void save(ggrs::Frame f) override { snaps[f] = live; }  // T's copy constructor is its Clone
        void load(ggrs::Frame f) override {
            auto it = snaps.find(f);
            if (it == snaps.end())  // mod.rs:209-212
                throw Panic(BGR_ERR_NO_SNAPSHOT, "Could not rollback to " + std::to_string(f) + ": no snapshot at that moment could be found.");
            live = it->second;
        }
        void prune(const std::vector<uint8_t>& alive, const std::vector<int32_t>& kept) override {
            for (auto it = live.begin(); it != live.end();)  // the components of despawned entities are gone with them
                it = it->first < alive.size() && alive[it->first] ? std::next(it) : live.erase(it);
            for (auto it = snaps.begin(); it != snaps.end();)  // what the engine's ring discarded (mod.rs:144-199)
                it = std::find(kept.begin(), kept.end(), it->first) != kept.end() ? std::next(it) : snaps.erase(it);
        }
        bool empty() const override { return live.empty(); }
    };
    template <class T> HostColumn<T>& host_col() {
        auto it = host_cols_.find(std::type_index(typeid(T)));
        if (it == host_cols_.end()) throw Panic(BGR_ERR_INVALID_ARGUMENT, std::string("not registered for rollback: ") + typeid(T).name());
        return static_cast<HostColumn<T>&>(*it->second);
    }
    bool entity_exists(uint32_t row) {
        finish();
        uint32_t rows = 0;
        check(bgr_row_count(engine_, &rows));
        if (row >= rows) return false;
        uint8_t a = 0;
        check(bgr_read_alive(engine_, row, 1, &a));
        return a != 0;
    }
    void handle_host_component_requests(const std::vector<ggrs::GgrsRequest>& requests) {
        for (const auto& r : requests) {
            if (r.kind == ggrs::GgrsRequest::SaveGameState) for (auto& c : host_cols_) c.second->save(r.frame);
            else if (r.kind == ggrs::GgrsRequest::LoadGameState) for (auto& c : host_cols_) c.second->load(r.frame);
        }
        std::vector<uint8_t> alive;
        bool any = false;
        for (auto& c : host_cols_) any = any || !c.second->empty();
        if (any) {
            uint32_t rows = 0;
            check(bgr_row_count(engine_, &rows));
            alive.resize(rows);
            if (rows) check(bgr_read_alive(engine_, 0, rows, alive.data()));
        }
        const std::vector<int32_t> kept = snapshot_frames();
        for (auto& c : host_cols_) c.second->prune(alive, kept);
    }
    std::map<std::type_index, std::unique_ptr<HostColumnBase>> host_cols_;

    struct PendingCol { std::type_index type; std::string name; uint32_t bytes, strategy; };
    using ResourceMap = std::map<std::type_index, std::vector<uint8_t>>;
    ResourceMap resources_;
    std::vector<std::pair<std::type_index, uint32_t>> res_order_;  // registered resources and their sizes, in order
    std::vector<std::type_index> res_checksummed_;
    std::vector<std::function<void(App&)>> res_systems_;
    std::map<ggrs::Frame, ResourceMap> res_store_;
    ggrs::Frame res_frame_ = 0;
    bgr_config cfg_{};
    bgr_engine* engine_ = nullptr;
    std::pair<uint32_t, uint32_t> retain_{0, 0};  // retain_confirmed(interval, count); count 0: off
    std::vector<PendingCol> pending_cols_;
    std::map<std::type_index, uint32_t> columns_;
    std::vector<std::pair<uint32_t, ByteRangeHasher>> checksums_;
    std::vector<System> systems_;
    std::vector<std::function<void(App&)>> read_inputs_, startup_;
    std::vector<std::function<void(const SyncTestMismatch&)>> observers_;
    std::optional<Session> session_;
    std::optional<LocalInputs> local_inputs_;
    LocalPlayers local_players_;
    std::vector<bgr_checksum> last_checksums_;
    uint64_t accumulator_ns_ = 0;
    bool run_slow_ = false, first_update_ = true;
};

}  // namespace bevy_ggrs
