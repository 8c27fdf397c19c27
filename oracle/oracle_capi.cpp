// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/seahash.hpp header).
// C ABI over the CPU restatement so that pytest / bench.py can drive it with ctypes using the
// same vocabulary as include/bevy_ggrs_b200.h (orc_* mirrors bgr_*).
#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>

#include "soa_baseline.hpp"
#include "world.hpp"

using namespace oracle;

#define ORC_API extern "C" __attribute__((visibility("default")))

static thread_local std::string g_err;

template <class F>
static int guarded(F&& f) {
    try {
        f();
        return BGR_OK;
    } catch (const RollbackPanic& e) {
        g_err = e.what();
        return BGR_ERR_NO_SNAPSHOT;
    } catch (const NonFinitePanic& e) {
        g_err = e.what();
        return BGR_ERR_NON_FINITE;
    } catch (const std::exception& e) {
        g_err = e.what();
        return BGR_ERR_INVALID_ARGUMENT;
    }
}

ORC_API const char* orc_last_error() { return g_err.c_str(); }

// ---- seahash -------------------------------------------------------------------------
ORC_API uint64_t orc_seahash(const void* p, uint64_t n) { return seahash(p, size_t(n)); }
// ChecksumPart::from_value(&v) for a u32 (checksum.rs:38-44)
ORC_API uint64_t orc_checksum_part_from_u32(uint32_t v) { SeaHasher h; h.write_u32(v); return h.finish(); }
// streaming interface check: hash fields appended one integer at a time
ORC_API uint64_t orc_seahash_u32_fields(const uint32_t* v, uint32_t n) { SeaHasher h; for (uint32_t i = 0; i < n; ++i) h.write_u32(v[i]); return h.finish(); }
ORC_API uint64_t orc_seahash_u64_fields(const uint64_t* v, uint32_t n) { SeaHasher h; for (uint32_t i = 0; i < n; ++i) h.write_u64(v[i]); return h.finish(); }

// ---- GgrsTime ------------------------------------------------------------------------
ORC_API uint32_t orc_ggrs_time_delta_bits(uint32_t fps, int32_t frame) {
    // delta of the AdvanceWorld step that ends at `frame` (time.rs:63-76)
    uint64_t f = uint64_t(int64_t(frame));
    uint64_t now = f * 1000000000ULL / fps, prev = (f - 1) * 1000000000ULL / fps;
    float s = duration_as_secs_f32(now - prev);
    uint32_t bits; std::memcpy(&bits, &s, 4); return bits;
}

// ---- GgrsSnapshots<u32,u32> ring KAT surface (mod.rs:353-508) -------------------------
using Snap = GgrsSnapshots<uint32_t>;
ORC_API Snap* orc_ring_new(uint32_t depth, int set_depth) { auto* s = new Snap(); if (set_depth) s->set_depth(depth); return s; }
ORC_API void orc_ring_free(Snap* s) { delete s; }
ORC_API void orc_ring_set_depth(Snap* s, uint32_t d) { s->set_depth(d); }
ORC_API uint32_t orc_ring_depth(Snap* s) { return uint32_t(s->depth); }
ORC_API void orc_ring_push(Snap* s, int32_t frame, uint32_t v) { s->push(frame, v); }
ORC_API void orc_ring_confirm(Snap* s, int32_t frame) { s->confirm(frame); }
ORC_API int orc_ring_rollback(Snap* s, int32_t frame) { return guarded([&] { s->rollback(frame); }); }
ORC_API int orc_ring_get(Snap* s, uint32_t* out) { return guarded([&] { *out = s->get(); }); }
ORC_API int orc_ring_peek(Snap* s, int32_t frame, uint32_t* out) { uint32_t* p = s->peek(frame); if (!p) return 0; *out = *p; return 1; }
ORC_API uint32_t orc_ring_len(Snap* s) { return uint32_t(s->frames.size()); }

// ---- RollbackOrdered KAT surface (rollback.rs:96-162) ---------------------------------
ORC_API RollbackOrdered* orc_ordered_new() { return new RollbackOrdered(); }
ORC_API RollbackOrdered* orc_ordered_clone(RollbackOrdered* o) { return new RollbackOrdered(*o); }
ORC_API void orc_ordered_free(RollbackOrdered* o) { delete o; }
ORC_API void orc_ordered_push(RollbackOrdered* o, uint64_t id) { o->push(id); }
ORC_API int orc_ordered_order(RollbackOrdered* o, uint64_t id, uint64_t* out) { return guarded([&] { *out = o->order_of(id); }); }
ORC_API uint64_t orc_ordered_len(RollbackOrdered* o) { return o->len(); }
ORC_API uint32_t orc_ordered_iter_sorted(RollbackOrdered* o, uint64_t* out, uint32_t cap) {
    uint32_t n = 0;
    for (uint64_t id : o->sorted) { if (n < cap) out[n] = id; ++n; }
    return n;
}

// ---- World ------------------------------------------------------------------------------
ORC_API World* orc_world_new(uint32_t fps, uint64_t order_base, uint32_t save_threads) {
    auto* w = new World();
    w->fps = fps; w->order_base = order_base; w->save_threads = save_threads ? save_threads : 1;
    return w;
}
ORC_API void orc_world_free(World* w) { delete w; }
ORC_API int orc_rollback_component(World* w, const char* name, uint32_t elem_bytes, uint32_t* col_out) {
    return guarded([&] { *col_out = w->add_column(name, elem_bytes); });
}
ORC_API int orc_checksum_component(World* w, uint32_t col, uint32_t kind, uint32_t off, uint32_t len, uint32_t flags) {
    return guarded([&] {
        if (col >= w->columns.size() || off + len > w->columns[col].elem_bytes) throw std::runtime_error("bad checksum range");
        auto& c = w->columns[col]; c.hash_kind = kind; c.hash_off = off; c.hash_len = len; c.hash_flags = flags;
    });
}
ORC_API int orc_rollback_resource(World* w, const char* name, const void* init, uint32_t bytes, int checksum, uint32_t* res_out) {
    return guarded([&] { *res_out = w->add_resource(name, init, bytes, checksum != 0); });
}
ORC_API int orc_add_system(World* w, uint32_t sys, const uint32_t* cols, uint32_t n_cols, const uint32_t* params, uint32_t n_params) {
    return guarded([&] {
        SystemDesc s; s.id = sys; s.cols.assign(cols, cols + n_cols); s.params.assign(params, params + n_params);
        if (sys == BGR_SYS_PARTICLES_SPAWN) {  // insert_resource(ParticleRng(GameRng::seed_from_u64(seed)))
            w->particle_rng.seed_from_u64(uint64_t(params[2]) | (uint64_t(params[3]) << 32));
            w->has_particle_rng = true;
        }
        w->systems.push_back(std::move(s));
    });
}
// add_systems(Startup, spawn_particles): the initial burst, outside the rollback loop
ORC_API int orc_run_startup_system(World* w, uint32_t sys) {
    return guarded([&] {
        for (const SystemDesc& s : w->systems)
            if (s.id == sys && sys == BGR_SYS_PARTICLES_SPAWN) { w->pending_spawns.clear(); w->spawn_particles(s); w->apply_spawns(); return; }
        throw std::runtime_error("startup system not registered");
    });
}
// raw RNG stream for the golden-vector test
ORC_API void orc_xoshiro_stream(uint64_t seed, uint32_t n, uint64_t* u64_out, float* f32_out, float low, float high) {
    Xoshiro256pp a, b;
    a.seed_from_u64(seed); b.seed_from_u64(seed);
    for (uint32_t i = 0; i < n; ++i) { u64_out[i] = a.next_u64(); f32_out[i] = b.random_range_f32(low, high); }
}
ORC_API void orc_xoshiro_from_state(const uint64_t* state4, uint32_t n, uint64_t* u64_out) {
    Xoshiro256pp a;
    for (int i = 0; i < 4; ++i) a.s[i] = state4[i];
    for (uint32_t i = 0; i < n; ++i) u64_out[i] = a.next_u64();
}
ORC_API void orc_xoshiro_seed_state(uint64_t seed, uint64_t* state4_out) {
    Xoshiro256pp a;
    a.seed_from_u64(seed);
    for (int i = 0; i < 4; ++i) state4_out[i] = a.s[i];
}
ORC_API int orc_spawn(World* w, uint32_t count, uint32_t* first_out) { return guarded([&] { *first_out = w->spawn(count); }); }
ORC_API uint32_t orc_row_count(World* w) { return uint32_t(w->rollback_ordered.len()); }
ORC_API uint64_t orc_active_count(World* w) { return w->rows(); }

// Component access is keyed by RollbackOrdered index (== engine row), not by table position.
ORC_API int orc_write_component(World* w, uint32_t col, uint32_t first, uint32_t count, const void* src, uint32_t stride) {
    return guarded([&] {
        uint32_t eb = w->columns.at(col).elem_bytes;
        // rows are still in spawn order before any despawn; locate through rollback id
        for (size_t r = 0; r < w->rows(); ++r) {
            uint64_t ord = w->rollback_ordered.order_of(w->rollback_id[r]);
            if (ord >= first && ord < uint64_t(first) + count)
                std::memcpy(&w->data[col][r * size_t(eb)], static_cast<const uint8_t*>(src) + (ord - first) * size_t(stride), eb);
        }
    });
}
// alive_out[i] = 1 if the entity with RollbackOrdered index first+i is alive and has the component
ORC_API int orc_read_component(World* w, uint32_t col, uint32_t first, uint32_t count, void* dst, uint32_t stride, uint8_t* alive_out) {
    return guarded([&] {
        uint32_t eb = w->columns.at(col).elem_bytes;
        if (alive_out) std::memset(alive_out, 0, count);
        for (size_t r = 0; r < w->rows(); ++r) {
            uint64_t ord = w->rollback_ordered.order_of(w->rollback_id[r]);
            if (ord >= first && ord < uint64_t(first) + count && w->has[col][r]) {
                std::memcpy(static_cast<uint8_t*>(dst) + (ord - first) * size_t(stride), &w->data[col][r * size_t(eb)], eb);
                if (alive_out) alive_out[ord - first] = 1;
            }
        }
    });
}
// alive_out[i] = 1 iff an entity with RollbackOrdered index first+i exists (whatever components it has)
ORC_API int orc_read_alive(World* w, uint32_t first, uint32_t count, uint8_t* alive_out) {
    return guarded([&] {
        std::memset(alive_out, 0, count);
        for (size_t r = 0; r < w->rows(); ++r) {
            uint64_t ord = w->rollback_ordered.order_of(w->rollback_id[r]);
            if (ord >= first && ord < uint64_t(first) + count) alive_out[ord - first] = 1;
        }
    });
}
// commands.entity(e).remove::<C>() / .insert(value) on the entity whose RollbackOrdered index is `order`
// (the other side of the Option<&mut S::Target> match in component_snapshot.rs:106-115)
static size_t row_of_order(World* w, uint64_t order) {
    for (size_t r = 0; r < w->rows(); ++r)
        if (w->rollback_ordered.order_of(w->rollback_id[r]) == order) return r;
    throw std::runtime_error("no live entity with that RollbackOrdered index");
}
ORC_API int orc_remove_component(World* w, uint32_t col, uint64_t order) {
    return guarded([&] { w->has.at(col).at(row_of_order(w, order)) = 0; });
}
// commands.entity(e).despawn() on the entity whose RollbackOrdered index is `order` (its index stays in RollbackOrdered)
ORC_API int orc_despawn(World* w, uint64_t order) {
    return guarded([&] {
        std::vector<size_t> rows{row_of_order(w, order)};
        w->apply_despawns(rows);
    });
}
ORC_API int orc_insert_component(World* w, uint32_t col, uint64_t order, const void* value) {
    return guarded([&] {
        size_t r = row_of_order(w, order);
        uint32_t eb = w->columns.at(col).elem_bytes;
        std::memcpy(&w->data[col][r * size_t(eb)], value, eb);
        w->has[col][r] = 1;
    });
}
// peek(frame) of GgrsComponentSnapshots<C> (mod.rs:233-240): returns 0 if no snapshot for the frame
ORC_API int orc_peek(World* w, int32_t frame, uint32_t col, uint32_t first, uint32_t count, void* dst, uint32_t stride, uint8_t* alive_out) {
    FlatTable* t = w->comp_snaps.at(col).peek(frame);
    if (!t) return 0;
    uint32_t eb = w->columns[col].elem_bytes;
    if (alive_out) std::memset(alive_out, 0, count);
    // RollbackOrdered as of that frame
    auto* ord_snap = w->ordered_snaps.peek(frame);
    const RollbackOrdered& ro = (ord_snap && *ord_snap) ? **ord_snap : w->rollback_ordered;
    t->for_each([&](uint64_t rid, const uint8_t* v) {
        uint64_t ord = ro.order_of(rid);
        if (ord >= first && ord < uint64_t(first) + count) {
            std::memcpy(static_cast<uint8_t*>(dst) + (ord - first) * size_t(stride), v, eb);
            if (alive_out) alive_out[ord - first] = 1;
        }
    });
    return 1;
}
ORC_API int orc_snapshot_frames(World* w, int32_t* out, uint32_t cap) {
    auto& fr = w->entity_snaps.frames;
    uint32_t n = 0;
    for (int32_t f : fr) { if (n < cap) out[n] = f; ++n; }
    return int(n);
}
ORC_API int orc_read_resource(World* w, uint32_t res, void* dst) {
    if (!w->res_present.at(res)) return 0;
    std::memcpy(dst, w->res_data[res].data(), w->res_data[res].size());
    return 1;
}
ORC_API int32_t orc_rollback_frame_count(World* w) { return w->rollback_frame_count; }
ORC_API void orc_set_rollback_frame_count(World* w, int32_t f) { w->rollback_frame_count = f; }
ORC_API int32_t orc_confirmed_frame_count(World* w) { return w->confirmed_frame_count; }
ORC_API void orc_set_max_prediction(World* w, uint32_t p) { w->max_prediction = p; }
// the session-less branch of run_ggrs_schedules (schedule_systems.rs:70-79)
ORC_API void orc_reset_session(World* w) { w->rollback_frame_count = 0; w->confirmed_frame_count = -1; w->max_prediction = 8; }
ORC_API uint32_t orc_last_dt_bits(World* w) { uint32_t b; std::memcpy(&b, &w->ggrs_time.delta_secs, 4); return b; }

ORC_API int orc_save_world(World* w, bgr_checksum* out) {
    return guarded([&] { w->save_world(); if (out) *out = bgr_checksum{w->rollback_frame_count, 1u, w->checksum_lo, 0}; });
}
// SaveWorld's Checksum half alone: the checksum of the current frame, no snapshot pushed (a replay's checksum frames)
ORC_API int orc_checksum_world(World* w, bgr_checksum* out) {
    return guarded([&] { w->checksum_world(); if (out) *out = bgr_checksum{w->rollback_frame_count, 1u, w->checksum_lo, 0}; });
}
// World::restore: `mask` one byte per row, `absent_bit` one per column, `cols[c]` rows * elem_bytes of column c
ORC_API int orc_restore(World* w, int32_t frame, uint32_t rows, const uint8_t* mask, const uint32_t* absent_bit,
                        const uint8_t* const* cols, uint64_t elapsed_ns, const uint64_t* rng) {
    return guarded([&] { w->restore(frame, rows, mask, absent_bit, cols, elapsed_ns, rng); });
}
ORC_API int orc_load_world(World* w) { return guarded([&] { w->load_world(); }); }
ORC_API int orc_advance_world(World* w, const uint8_t* inputs, uint32_t n_players) {
    return guarded([&] {
        w->n_players = n_players;
        std::memset(w->player_inputs, 0, sizeof w->player_inputs);
        if (inputs) std::memcpy(w->player_inputs, inputs, n_players);
        w->advance_world();
        w->n_players = 0;
    });
}
// per-column raw XOR (before the final hash) and parts of the last save — shard emulation / debugging
ORC_API int orc_last_partial(World* w, bgr_partial* out) {
    return guarded([&] {
        std::memset(out, 0, sizeof *out);
        out->frame = w->rollback_frame_count;
        out->active = w->rows();
        out->total = w->rollback_ordered.len();
        uint32_t n = 0;
        for (size_t c = 0; c < w->columns.size(); ++c)
            if (w->columns[c].hash_kind != BGR_HASH_NONE && n < BGR_MAX_CHECKSUM_COLUMNS) out->xor_[n++] = w->comp_xor_raw[c];
        out->n_columns = n;
    });
}

// handle_requests; also returns the wall time spent inside (ns) for the CPU baseline
ORC_API int orc_handle_requests(World* w, const bgr_session_info* sess, const bgr_request* reqs, uint32_t n,
                                bgr_checksum* out, uint32_t cap, uint32_t* n_out, uint64_t* elapsed_ns) {
    std::vector<bgr_checksum> cs;
    auto t0 = std::chrono::steady_clock::now();
    int rc = guarded([&] { w->handle_requests(*sess, reqs, n, cs); });
    auto t1 = std::chrono::steady_clock::now();
    if (elapsed_ns) *elapsed_ns = uint64_t(std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count());
    uint32_t k = 0;
    for (auto& c : cs) { if (k < cap) out[k] = c; ++k; }
    if (n_out) *n_out = k;
    return rc;
}

// ---- optimised SoA CPU bar (BASELINE.md §2(2)) -------------------------------------------------------------
ORC_API SoaWorld* orc_soa_new(uint32_t n, uint32_t depth, uint32_t fps, uint32_t threads) { return new SoaWorld(n, depth, fps, threads); }
ORC_API void orc_soa_free(SoaWorld* w) { delete w; }
ORC_API void orc_soa_set_columns(SoaWorld* w, const float* tf, const float* vel, const uint64_t* ttl) {
    std::memcpy(w->live.tf.data(), tf, w->n * 40);
    std::memcpy(w->live.vel.data(), vel, w->n * 12);
    std::memcpy(w->live.ttl.data(), ttl, w->n * 8);
    std::fill(w->live.alive.begin(), w->live.alive.end(), uint8_t(1));
}
ORC_API void orc_soa_get_columns(SoaWorld* w, float* tf, float* vel, uint64_t* ttl, uint8_t* alive) {
    std::memcpy(tf, w->live.tf.data(), w->n * 40);
    std::memcpy(vel, w->live.vel.data(), w->n * 12);
    std::memcpy(ttl, w->live.ttl.data(), w->n * 8);
    std::memcpy(alive, w->live.alive.data(), w->n);
}
ORC_API int orc_soa_handle_requests(SoaWorld* w, const bgr_session_info* sess, const bgr_request* reqs, uint32_t n,
                                    bgr_checksum* out, uint32_t cap, uint32_t* n_out, uint64_t* elapsed_ns) {
    std::vector<bgr_checksum> cs;
    auto t0 = std::chrono::steady_clock::now();
    int rc = guarded([&] { w->handle_requests(*sess, reqs, n, cs); });
    auto t1 = std::chrono::steady_clock::now();
    if (elapsed_ns) *elapsed_ns = uint64_t(std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count());
    uint32_t k = 0;
    for (auto& c : cs) { if (k < cap) out[k] = c; ++k; }
    if (n_out) *n_out = k;
    return rc;
}
