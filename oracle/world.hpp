// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/seahash.hpp header).
//
// CPU restatement of the reference's rollback hot path WITH THE REFERENCE'S DATA STRUCTURES
// (a fresh HashMap<RollbackId, T> per type per frame, hashed lookups on load, RollbackOrdered
// cloned on every save, serial per-type loops).  It is both the parity oracle and the timed
// "faithful CPU restatement" baseline of BASELINE.md §2(1).
//
// Reference items followed (paths relative to /root/reference):
//   RollbackOrdered                      src/snapshot/rollback.rs:57-94
//   GgrsComponentSnapshot (HashMap)      src/snapshot/mod.rs:274-312
//   ComponentSnapshotPlugin::save/load   src/snapshot/component_snapshot.rs:66-84, 95-123
//   EntitySnapshotPlugin::save/load      src/snapshot/entity.rs:39-51, 55-99
//   ResourceSnapshotPlugin::save/load    src/snapshot/resource_snapshot.rs:65-73, 77-93
//   ComponentChecksumPlugin              src/snapshot/component_checksum.rs:67-108
//   EntityChecksumPlugin::update         src/snapshot/entity_checksum.rs:29-52
//   ResourceChecksumPlugin               src/snapshot/resource_checksum.rs:63-82
//   ChecksumPlugin::update               src/snapshot/checksum.rs:88-99
//   schedule ordering                    src/snapshot/set.rs:85-127
//   GgrsTimePlugin::update               src/time.rs:63-76
//   handle_requests                      src/schedule_systems.rs:170-289
//   update_particles / despawn_particles examples/stress_tests/particles.rs:272-289
//   move_cube_system / increase_frame    examples/box_game/box_game.rs:146-206
//   increment_score / decrease_health    tests/component_rollback.rs:25-29, tests/synctest.rs:38-45
//
// PARITY STATUS: ring semantics and RollbackOrdered are pinned by the reference's own unit tests (ported in tests/);
// the third-party arithmetic is pinned by vectors that do not come from this restatement (tests/golden/
// third_party_kats.json, seahash_buffer_mode.json; tests/test_third_party_kats.py): seahash 4.1 by the crate's
// documented vector + 97 lengths of a buffer-form restatement, SplitMix64 / xoshiro256++ by the published reference
// vectors, Duration::as_secs_f32 (the dt sequence) by IEEE binary32 evaluation of the std formula, rand's f32 range by
// proof that its retry branch is unreachable for the example's range.  What remains "PARITY UNPINNED" in the strict
// sense is the COMPOSITION — how component_checksum.rs:67-108 / particles.rs combine those primitives, and therefore
// the numeric frame checksums and trajectories: the reference holds no numeric golden for them and no Rust toolchain
// exists here to produce one (SURVEY.md §8c).  oracle/ref_harness + scripts/gen_reference_goldens.sh generate such
// goldens from the UNMODIFIED crate on any box with cargo; tests/test_reference_goldens.py consumes them.
//
// Build with -ffp-contract=off: Rust/glam scalar Vec3 math rounds every mul and add.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <future>
#include <optional>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "../include/bevy_ggrs_b200.h"  // POD request / session / checksum structs and enums only
#include "ggrs_snapshots.hpp"
#include "seahash.hpp"

namespace oracle {

// oracle-only system id: a u32 resource += 1 (box_game.rs:146-148). Resources stay host-side in the product.
constexpr uint32_t ORC_SYS_RESOURCE_U32_ADD = 100;

// ---------------------------------------------------------------------------------------
// A flat open-addressing hash table with a runtime value size: stand-in for hashbrown's
// HashMap<RollbackId, As> (bevy::platform::collections::HashMap).  7/8 max load, power-of-two
// buckets, reserved up-front like `Iterator::collect` does from an exact size hint.
// ---------------------------------------------------------------------------------------
struct FlatTable {
    uint32_t stride = 0;
    size_t cap = 0, len = 0;
    std::vector<uint64_t> keys;
    std::vector<uint8_t> used;
    std::vector<uint8_t> vals;

    explicit FlatTable(uint32_t value_bytes = 8) : stride(value_bytes) {}

    static uint64_t mix(uint64_t k) {
        k ^= k >> 32;
        k *= 0x9E3779B97F4A7C15ULL;
        k ^= k >> 29;
        return k;
    }
    void reserve(size_t n) {
        size_t want = 8;
        while (want * 7 < n * 8) want <<= 1;
        if (want <= cap) return;
        FlatTable old = std::move(*this);
        stride = old.stride;
        cap = want; len = 0;
        keys.assign(cap, 0);
        used.assign(cap, 0);
        vals.assign(cap * size_t(stride), 0);
        for (size_t i = 0; i < old.cap; ++i)
            if (old.used[i]) std::memcpy(insert(old.keys[i]), &old.vals[i * size_t(old.stride)], stride);
    }
    uint8_t* insert(uint64_t key) {
        if ((len + 1) * 8 > cap * 7) reserve(len + 1);
        size_t m = cap - 1, i = mix(key) & m;
        while (used[i]) {
            if (keys[i] == key) return &vals[i * size_t(stride)];
            i = (i + 1) & m;
        }
        used[i] = 1; keys[i] = key; ++len;
        return &vals[i * size_t(stride)];
    }
    const uint8_t* find(uint64_t key) const {
        if (!cap) return nullptr;
        size_t m = cap - 1, i = mix(key) & m;
        while (used[i]) {
            if (keys[i] == key) return &vals[i * size_t(stride)];
            i = (i + 1) & m;
        }
        return nullptr;
    }
    template <class F> void for_each(F&& f) const {
        for (size_t i = 0; i < cap; ++i)
            if (used[i]) f(keys[i], &vals[i * size_t(stride)]);
    }
};

// rollback.rs:57-94
struct RollbackOrdered {
    FlatTable order{8};
    std::vector<uint64_t> sorted;
    void push(uint64_t rollback) {
        sorted.push_back(rollback);
        uint64_t idx = sorted.size() - 1;
        std::memcpy(order.insert(rollback), &idx, 8);
    }
    uint64_t order_of(uint64_t rollback) const {
        const uint8_t* p = order.find(rollback);
        if (!p) throw std::runtime_error("RollbackId was not registered in RollbackOrdered!");
        uint64_t v; std::memcpy(&v, p, 8); return v;
    }
    size_t len() const { return order.len; }
};

struct ColumnDesc {
    std::string name;
    uint32_t elem_bytes = 0;
    uint32_t hash_kind = BGR_HASH_NONE, hash_off = 0, hash_len = 0, hash_flags = 0;
};

struct ResourceDesc {
    std::string name;
    uint32_t bytes = 0;
    bool checksum = false;  // checksum_resource_with_hash (derive(Hash) over the POD bytes)
};

struct SystemDesc {
    uint32_t id = 0;
    std::vector<uint32_t> cols;
    std::vector<uint32_t> params;
};

// Time<GgrsTime> (time.rs:63-76; bevy Time::advance_to / Duration::as_secs_f32)
struct GgrsTimeState {
    uint64_t elapsed_ns = 0;
    uint64_t delta_ns = 0;
    float delta_secs = 0.0f;
};

inline float duration_as_secs_f32(uint64_t ns) {
    // core::time::Duration::as_secs_f32 = secs as f32 + nanos as f32 / 1e9f32
    uint64_t secs = ns / 1000000000ULL;
    uint32_t nanos = uint32_t(ns % 1000000000ULL);
    return float(secs) + float(nanos) / 1000000000.0f;
}

struct NonFinitePanic : std::runtime_error { using std::runtime_error::runtime_error; };

// ParticleRng(rand_xoshiro::Xoshiro256PlusPlus) (particles.rs:125-128) — third-party arithmetic, not under
// /root/reference; restated from the published algorithms, PARITY UNPINNED (no golden upstream, no cargo here):
//   rand_xoshiro 0.7  Xoshiro256PlusPlus::seed_from_u64(s): state = 4 outputs of SplitMix64(s)
//                     next_u64: rotl(s0 + s3, 23) + s0, then the xoshiro256 state update
//                     next_u32: upper 32 bits of next_u64
//   rand 0.9          random_range(low..high) for f32: v = f32::from_bits((next_u32 >> 9) | 0x3f800000) - 1.0;
//                     res = v * (high - low) + low   (mul then add, separately rounded); retried only if res >= high
struct Xoshiro256pp {
    uint64_t s[4] = {0, 0, 0, 0};
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    void seed_from_u64(uint64_t seed) {
        uint64_t x = seed;
        for (int i = 0; i < 4; ++i) {
            x += 0x9E3779B97F4A7C15ULL;
            uint64_t z = x;
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
            z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
            s[i] = z ^ (z >> 31);
        }
    }
    uint64_t next_u64() {
        uint64_t result = rotl(s[0] + s[3], 23) + s[0];
        uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return result;
    }
    uint32_t next_u32() { return uint32_t(next_u64() >> 32); }
    float random_range_f32(float low, float high) {
        const float scale = high - low;
        for (;;) {
            uint32_t bits = (next_u32() >> 9) | 0x3f800000u;
            float value1_2; std::memcpy(&value1_2, &bits, 4);
            float value0_1 = value1_2 - 1.0f;
            float res = value0_1 * scale + low;
            if (res < high) return res;
        }
    }
};

struct World {
    // ---- registration ----
    std::vector<ColumnDesc> columns;
    std::vector<ResourceDesc> resources;
    std::vector<SystemDesc> systems;
    uint32_t fps = 60;
    uint64_t order_base = 0;  // only used to emulate one shard of a sharded world
    unsigned save_threads = 1;  // SaveWorld runs per-type systems on Bevy's multithreaded executor

    // ---- single-archetype table (rows = live rollback entities) ----
    std::vector<uint64_t> rollback_id;            // RollbackId(Entity at first spawn)
    std::vector<uint64_t> entity;                 // current Entity bits
    std::vector<std::vector<uint8_t>> data;       // per column: AoS bytes, rows * elem_bytes
    std::vector<std::vector<uint8_t>> has;        // per column presence
    std::vector<std::vector<uint8_t>> res_data;   // per resource bytes
    std::vector<uint8_t> res_present;
    uint64_t next_entity = 0;
    uint32_t call_count = 0;  // the un-rolled-back atomic of tests/synctest.rs:83-125

    // ---- resources of the snapshot plugin ----
    RollbackOrdered rollback_ordered;
    int32_t rollback_frame_count = 0;   // mod.rs:66-67
    int32_t confirmed_frame_count = 0;  // mod.rs:76-77 (init_resource -> Default 0)
    std::optional<uint32_t> max_prediction;  // MaxPredictionWindow, lib.rs:116-117
    GgrsTimeState ggrs_time;
    Xoshiro256pp particle_rng;          // ParticleRng resource (particles.rs:128), rolled back with clone (:200)
    bool has_particle_rng = false;
    GgrsSnapshots<std::optional<Xoshiro256pp>> rng_snaps;
    uint8_t player_inputs[BGR_MAX_PLAYERS] = {0};
    uint32_t n_players = 0;

    // ---- snapshot storage: one GgrsSnapshots per registered type ----
    std::vector<GgrsSnapshots<FlatTable>> comp_snaps;                       // GgrsComponentSnapshots<C>
    GgrsSnapshots<FlatTable> entity_snaps;                                  // GgrsComponentSnapshots<Entity>
    GgrsSnapshots<std::optional<RollbackOrdered>> ordered_snaps;            // mod.rs:339
    GgrsSnapshots<std::optional<GgrsTimeState>> time_snaps;                 // time.rs:100
    std::vector<GgrsSnapshots<std::optional<std::vector<uint8_t>>>> res_snaps;

    // ---- checksum parts (ChecksumPart entities) ----
    std::vector<uint64_t> comp_parts;  // per column (only checksummed ones are folded)
    std::vector<uint64_t> res_parts;
    uint64_t entity_part = 0;
    uint64_t checksum_lo = 0;          // Checksum(u128): hi is always 0
    // raw per-column XOR before the final hash (for shard emulation / debugging)
    std::vector<uint64_t> comp_xor_raw;

    size_t rows() const { return rollback_id.size(); }

    uint32_t add_column(const std::string& name, uint32_t elem_bytes) {
        columns.push_back({name, elem_bytes});
        data.emplace_back(); has.emplace_back();
        comp_snaps.emplace_back();
        comp_parts.push_back(0); comp_xor_raw.push_back(0);
        return uint32_t(columns.size() - 1);
    }
    uint32_t add_resource(const std::string& name, const void* init, uint32_t bytes, bool checksum) {
        resources.push_back({name, bytes, checksum});
        res_data.emplace_back(static_cast<const uint8_t*>(init), static_cast<const uint8_t*>(init) + bytes);
        res_present.push_back(1);
        res_snaps.emplace_back();
        res_parts.push_back(0);
        return uint32_t(resources.size() - 1);
    }

    // commands.spawn((components..., Rollback)): on_add hook -> RollbackId + RollbackOrdered.push (rollback.rs:40-54)
    uint32_t spawn(uint32_t count) {
        // the caller addresses entities by RollbackOrdered index (== engine row): the first new one gets the next index.
        // (rows() — the dense table's length — is smaller once entities have been despawned; found by the request fuzz.)
        uint32_t first = uint32_t(rollback_ordered.len());
        for (uint32_t k = 0; k < count; ++k) {
            uint64_t e = next_entity++;
            rollback_id.push_back(e);
            entity.push_back(e);
            rollback_ordered.push(e);
            for (size_t c = 0; c < columns.size(); ++c) {
                data[c].resize(data[c].size() + columns[c].elem_bytes, 0);
                has[c].push_back(1);
            }
        }
        return first;
    }
    void swap_remove_row(size_t r) {
        size_t last = rows() - 1;
        for (size_t c = 0; c < columns.size(); ++c) {
            uint32_t eb = columns[c].elem_bytes;
            if (r != last) std::memcpy(&data[c][r * eb], &data[c][last * eb], eb);
            data[c].resize(last * size_t(eb));
            has[c][r] = has[c][last]; has[c].pop_back();
        }
        rollback_id[r] = rollback_id[last]; rollback_id.pop_back();
        entity[r] = entity[last]; entity.pop_back();
    }
    long find_row(uint64_t rid) const {
        for (size_t r = 0; r < rows(); ++r) if (rollback_id[r] == rid) return long(r);
        return -1;
    }

    // =====================================================================================
    // SaveWorld (set.rs:97-100; checksum.rs:119-124): Checksum set -> ChecksumPlugin::update -> Snapshot set
    // =====================================================================================
    uint64_t hash_element(const ColumnDesc& cd, const uint8_t* elem) const {
        if (cd.hash_flags & BGR_HASH_FLAG_ASSERT_FINITE_F32) {
            for (uint32_t o = 0; o + 4 <= cd.hash_len; o += 4) {
                float f; std::memcpy(&f, elem + cd.hash_off + o, 4);
                if (!std::isfinite(f)) throw NonFinitePanic("Hashing is not stable for NaN f32 values.");
            }
        }
        // custom_hasher(component): fresh checksum_hasher(), fields appended little-endian
        return seahash(elem + cd.hash_off, cd.hash_len);
    }
    void component_checksum(size_t c) {  // component_checksum.rs:67-108
        const ColumnDesc& cd = columns[c];
        uint64_t result = 0;
        for (size_t r = 0; r < rows(); ++r) {
            if (!has[c][r]) continue;
            SeaHasher h;  // `let mut hasher = hasher;` copy of a fresh hasher (:82)
            h.write_u64(order_base + rollback_ordered.order_of(rollback_id[r]));  // :85
            h.write_u64(hash_element(cd, &data[c][r * size_t(cd.elem_bytes)]));   // :86
            result ^= h.finish();                                                  // :89
        }
        comp_xor_raw[c] = result;
        SeaHasher outer;
        outer.write_u64(result);  // :93
        comp_parts[c] = outer.finish();
    }
    void entity_checksum() {  // entity_checksum.rs:29-52
        SeaHasher h;
        h.write_u64(uint64_t(rows()));
        h.write_u64(uint64_t(rollback_ordered.len()));
        entity_part = h.finish();
    }
    void component_save(size_t c) {  // component_snapshot.rs:66-84 (+ sync_depth, discard_old_snapshots, :135-144)
        auto& snaps = comp_snaps[c];
        if (max_prediction) snaps.set_depth(*max_prediction);  // mod.rs:260-270
        snaps.confirm(confirmed_frame_count);                   // mod.rs:243-255
        uint32_t eb = columns[c].elem_bytes;
        FlatTable t(eb);
        size_t n = 0;
        for (size_t r = 0; r < rows(); ++r) n += has[c][r];
        t.reserve(n);
        for (size_t r = 0; r < rows(); ++r)
            if (has[c][r]) std::memcpy(t.insert(rollback_id[r]), &data[c][r * size_t(eb)], eb);
        snaps.push(rollback_frame_count, std::move(t));
    }
    void entity_save() {  // entity.rs:39-51
        if (max_prediction) entity_snaps.set_depth(*max_prediction);
        entity_snaps.confirm(confirmed_frame_count);
        FlatTable t(8);
        t.reserve(rows());
        for (size_t r = 0; r < rows(); ++r) std::memcpy(t.insert(rollback_id[r]), &entity[r], 8);
        entity_snaps.push(rollback_frame_count, std::move(t));
    }
    void save_world() {
        checksum_world();
        snapshot_world();
    }
    // SaveWorldSystems::Checksum and ChecksumPlugin::update: the frame checksum without storing anything (what a
    // replay computes at its checksum frames)
    void checksum_world() {
        // --- SaveWorldSystems::Checksum: per-type systems, parallel-eligible ---
        std::vector<std::function<void()>> tasks;
        for (size_t c = 0; c < columns.size(); ++c)
            if (columns[c].hash_kind != BGR_HASH_NONE) tasks.push_back([this, c] { component_checksum(c); });
        tasks.push_back([this] { entity_checksum(); });
        for (size_t i = 0; i < resources.size(); ++i)
            if (resources[i].checksum)
                tasks.push_back([this, i] {  // resource_checksum.rs:63-82
                    res_parts[i] = res_present[i] ? seahash(res_data[i].data(), res_data[i].size()) : 0;
                });
        run_tasks(tasks);
        // --- ChecksumPlugin::update (checksum.rs:88-99): XOR of every ChecksumPart ---
        uint64_t x = entity_part;
        for (size_t c = 0; c < columns.size(); ++c)
            if (columns[c].hash_kind != BGR_HASH_NONE) x ^= comp_parts[c];
        for (size_t i = 0; i < resources.size(); ++i)
            if (resources[i].checksum) x ^= res_parts[i];
        checksum_lo = x;
    }
    void snapshot_world() {
        // --- SaveWorldSystems::Snapshot: per-type save systems ---
        std::vector<std::function<void()>> tasks;
        for (size_t c = 0; c < columns.size(); ++c) tasks.push_back([this, c] { component_save(c); });
        tasks.push_back([this] { entity_save(); });
        tasks.push_back([this] {  // ResourceSnapshotPlugin<CloneStrategy<RollbackOrdered>> (mod.rs:339)
            if (max_prediction) ordered_snaps.set_depth(*max_prediction);
            ordered_snaps.confirm(confirmed_frame_count);
            ordered_snaps.push(rollback_frame_count, std::optional<RollbackOrdered>(rollback_ordered));
        });
        tasks.push_back([this] {  // Time<GgrsTime> (time.rs:100)
            if (max_prediction) time_snaps.set_depth(*max_prediction);
            time_snaps.confirm(confirmed_frame_count);
            time_snaps.push(rollback_frame_count, std::optional<GgrsTimeState>(ggrs_time));
        });
        if (has_particle_rng)
            tasks.push_back([this] {  // rollback_resource_with_clone::<ParticleRng>() (particles.rs:200)
                if (max_prediction) rng_snaps.set_depth(*max_prediction);
                rng_snaps.confirm(confirmed_frame_count);
                rng_snaps.push(rollback_frame_count, std::optional<Xoshiro256pp>(particle_rng));
            });
        for (size_t i = 0; i < resources.size(); ++i)
            tasks.push_back([this, i] {  // resource_snapshot.rs:65-73
                if (max_prediction) res_snaps[i].set_depth(*max_prediction);
                res_snaps[i].confirm(confirmed_frame_count);
                std::optional<std::vector<uint8_t>> v;
                if (res_present[i]) v = res_data[i];
                res_snaps[i].push(rollback_frame_count, std::move(v));
            });
        run_tasks(tasks);
    }
    void run_tasks(std::vector<std::function<void()>>& tasks) {
        if (save_threads <= 1 || tasks.size() <= 1) {
            for (auto& t : tasks) t();
            return;
        }
        // Bevy's multithreaded executor may overlap *different* systems; each loop is serial.
        std::vector<std::future<void>> fs;
        size_t inflight_cap = save_threads;
        size_t next = 0;
        while (next < tasks.size()) {
            size_t batch_end = std::min(tasks.size(), next + inflight_cap);
            fs.clear();
            for (size_t i = next + 1; i < batch_end; ++i)
                fs.push_back(std::async(std::launch::async, tasks[i]));
            tasks[next]();
            for (auto& f : fs) f.get();
            next = batch_end;
        }
    }

    // =====================================================================================
    // LoadWorld (set.rs:86-96): Entity -> flush -> Data -> flush -> Mapping
    // =====================================================================================
    void load_world() {
        const int32_t frame = rollback_frame_count;
        // --- EntitySnapshotPlugin::load (entity.rs:55-99) ---
        FlatTable& esnap = entity_snaps.rollback(frame).get();
        {
            // rollback_mapping: RollbackId -> (current, old)
            struct Pair { uint64_t cur, old; uint8_t has_cur, has_old; };
            FlatTable mapping(sizeof(Pair));
            mapping.reserve(esnap.len);
            esnap.for_each([&](uint64_t rid, const uint8_t* v) {
                Pair p{0, 0, 0, 1}; std::memcpy(&p.old, v, 8);
                std::memcpy(mapping.insert(rid), &p, sizeof p);
            });
            for (size_t r = 0; r < rows(); ++r) {
                uint8_t* slot = mapping.insert(rollback_id[r]);
                Pair p; std::memcpy(&p, slot, sizeof p);
                p.cur = entity[r]; p.has_cur = 1;
                std::memcpy(slot, &p, sizeof p);
            }
            std::vector<size_t> to_despawn;
            std::vector<uint64_t> to_spawn;
            mapping.for_each([&](uint64_t rid, const uint8_t* v) {
                Pair p; std::memcpy(&p, v, sizeof p);
                if (!p.has_cur && p.has_old) to_spawn.push_back(rid);
            });
            for (size_t r = 0; r < rows(); ++r) {
                Pair p; std::memcpy(&p, mapping.find(rollback_id[r]), sizeof p);
                if (p.has_cur && !p.has_old) to_despawn.push_back(r);
            }
            // EntityFlush: apply commands
            apply_despawns(to_despawn);
            for (uint64_t rid : to_spawn) {
                // commands.spawn((rollback, Rollback)): RollbackId already present -> hook returns early (rollback.rs:43-47)
                rollback_id.push_back(rid);
                entity.push_back(next_entity++);
                for (size_t c = 0; c < columns.size(); ++c) {
                    data[c].resize(data[c].size() + columns[c].elem_bytes, 0);
                    has[c].push_back(0);
                }
            }
        }
        // --- LoadWorldSystems::Data ---
        for (size_t c = 0; c < columns.size(); ++c) {  // component_snapshot.rs:95-123
            FlatTable& snap = comp_snaps[c].rollback(frame).get();
            uint32_t eb = columns[c].elem_bytes;
            for (size_t r = 0; r < rows(); ++r) {
                const uint8_t* s = snap.find(rollback_id[r]);
                if (has[c][r] && s) std::memcpy(&data[c][r * size_t(eb)], s, eb);       // S::update
                else if (has[c][r] && !s) has[c][r] = 0;                                // remove
                else if (!has[c][r] && s) { std::memcpy(&data[c][r * size_t(eb)], s, eb); has[c][r] = 1; }  // insert
            }
        }
        {  // RollbackOrdered resource (resource_snapshot.rs:77-93)
            auto& s = ordered_snaps.rollback(frame).get();
            if (s) rollback_ordered = *s;
        }
        {
            auto& s = time_snaps.rollback(frame).get();
            if (s) ggrs_time = *s;
        }
        if (has_particle_rng) {
            auto& s = rng_snaps.rollback(frame).get();
            if (s) particle_rng = *s;
        }
        for (size_t i = 0; i < resources.size(); ++i) {
            auto& s = res_snaps[i].rollback(frame).get();
            if (s) { res_data[i] = *s; res_present[i] = 1; } else { res_present[i] = 0; }
        }
    }
    // A world checkpoint restored (bgr_checkpoint_restore): row r of the checkpoint gets RollbackOrdered index r, it
    // exists iff bit 0 of its mask byte is set, and column c is present on it unless mask & absent_bit[c].
    // RollbackFrameCount, Time<GgrsTime> and ParticleRng become the checkpoint's; every GgrsSnapshots is cleared and then
    // holds that frame's one snapshot.  The call counter, ConfirmedFrameCount and MaxPredictionWindow are left alone.
    void restore(int32_t frame, uint32_t n, const uint8_t* mask, const uint32_t* absent_bit,
                 const uint8_t* const* col_bytes, uint64_t elapsed_ns, const uint64_t rng[4]) {
        rollback_id.clear();
        entity.clear();
        for (auto& d : data) d.clear();
        for (auto& h : has) h.clear();
        rollback_ordered = RollbackOrdered{};
        pending_spawns.clear();
        for (uint32_t r = 0; r < n; ++r) {
            const uint64_t id = next_entity++;
            rollback_ordered.push(id);
            if (!(mask[r] & 1u)) continue;
            rollback_id.push_back(id);
            entity.push_back(id);
            for (size_t c = 0; c < columns.size(); ++c) {
                const uint32_t eb = columns[c].elem_bytes;
                const uint8_t* v = col_bytes[c] + size_t(r) * eb;
                data[c].insert(data[c].end(), v, v + eb);
                has[c].push_back((mask[r] & absent_bit[c]) ? 0 : 1);
            }
        }
        rollback_frame_count = frame;
        ggrs_time = GgrsTimeState{};
        ggrs_time.elapsed_ns = elapsed_ns;
        if (has_particle_rng)
            for (int i = 0; i < 4; ++i) particle_rng.s[i] = rng[i];
        for (auto& s : comp_snaps) s.clear();
        entity_snaps.clear();
        ordered_snaps.clear();
        time_snaps.clear();
        rng_snaps.clear();
        for (auto& s : res_snaps) s.clear();
        snapshot_world();
    }

    // despawn commands applied at a flush point; Bevy tables swap_remove, so process rows descending
    void apply_despawns(std::vector<size_t>& rows_to_kill) {
        std::sort(rows_to_kill.begin(), rows_to_kill.end());
        for (size_t i = rows_to_kill.size(); i-- > 0;) {
            if (i + 1 < rows_to_kill.size() && rows_to_kill[i] == rows_to_kill[i + 1]) continue;
            swap_remove_row(rows_to_kill[i]);
        }
    }

    // =====================================================================================
    // AdvanceWorld (set.rs:101-126; lib.rs:234-249; time.rs:98-111)
    // =====================================================================================
    void advance_world() {
        // First: GgrsTimePlugin::update (time.rs:63-76)
        uint64_t this_frame = uint64_t(int64_t(rollback_frame_count));  // `frame.0 as u64`
        uint64_t runtime = this_frame * 1000000000ULL / uint64_t(fps);
        if (runtime < ggrs_time.elapsed_ns) throw std::runtime_error("tried to move time backwards");
        ggrs_time.delta_ns = runtime - ggrs_time.elapsed_ns;   // Time::advance_to
        ggrs_time.elapsed_ns = runtime;
        ggrs_time.delta_secs = duration_as_secs_f32(ggrs_time.delta_ns);
        // Main: world.run_schedule(GgrsSchedule); commands apply at the end
        std::vector<size_t> despawn;
        pending_spawns.clear();
        for (const SystemDesc& s : systems) run_system(s, despawn);
        apply_despawns(despawn);
        apply_spawns();
    }

    // commands.spawn((Sprite, Velocity, Ttl, Rollback)) queued by spawn_particles; applied at the flush
    struct PendingSpawn { uint32_t tc, vc, lc; float vx, vy; uint64_t ttl; };
    std::vector<PendingSpawn> pending_spawns;
    void apply_spawns() {
        for (const PendingSpawn& ps : pending_spawns) {
            uint32_t r = spawn(1);  // Rollback on_add hook: RollbackId + RollbackOrdered.push
            size_t row = rows() - 1; (void)r;
            float tf[10] = {0, 0, 0, 0, 0, 0, 1.0f, 1.0f, 1.0f, 1.0f};  // Transform::default() (Sprite requires Transform)
            std::memcpy(&data[ps.tc][row * 40], tf, 40);
            float v[3] = {ps.vx, ps.vy, 0.0f};
            std::memcpy(&data[ps.vc][row * 12], v, 12);
            std::memcpy(&data[ps.lc][row * 8], &ps.ttl, 8);
        }
        pending_spawns.clear();
    }
    void spawn_particles(const SystemDesc& s) {  // particles.rs:258-270
        const float sp = 200.0f;
        for (uint32_t k = 0; k < s.params[0]; ++k) {
            PendingSpawn ps{s.cols[0], s.cols[1], s.cols[2], 0, 0, uint64_t(s.params[1])};
            ps.vx = particle_rng.random_range_f32(-sp, sp);
            ps.vy = particle_rng.random_range_f32(-sp, sp);
            pending_spawns.push_back(ps);
        }
    }

    void run_system(const SystemDesc& s, std::vector<size_t>& despawn) {
        const float dt = ggrs_time.delta_secs;
        switch (s.id) {
        case BGR_SYS_PARTICLES_SPAWN: {  // .run_if(spawn_pressed), particles.rs:254-256
            bool pressed = false;
            for (uint32_t i = 0; i < n_players; ++i) pressed = pressed || (player_inputs[i] & BGR_INPUT_SPAWN);
            if (pressed) spawn_particles(s);
            break;
        }
        case BGR_SYS_PARTICLES_UPDATE: {  // particles.rs:272-280
            uint32_t tc = s.cols[0], vc = s.cols[1];
            const float gx = 0.0f * 200.0f, gy = -1.0f * 200.0f, gz = 0.0f * 200.0f;  // Vec3::NEG_Y * 200.0
            for (size_t r = 0; r < rows(); ++r) {
                if (!has[tc][r] || !has[vc][r]) continue;
                float* t = reinterpret_cast<float*>(&data[tc][r * 40]);
                float* v = reinterpret_cast<float*>(&data[vc][r * 12]);
                // **velocity += gravity * time_step;  (each mul and add rounded separately)
                float ax = gx * dt, ay = gy * dt, az = gz * dt;
                v[0] = v[0] + ax; v[1] = v[1] + ay; v[2] = v[2] + az;
                // transform.translation += **velocity * time_step;
                float dx = v[0] * dt, dy = v[1] * dt, dz = v[2] * dt;
                t[0] = t[0] + dx; t[1] = t[1] + dy; t[2] = t[2] + dz;
            }
            break;
        }
        case BGR_SYS_PARTICLES_DESPAWN: {  // particles.rs:282-289
            uint32_t lc = s.cols[0];
            for (size_t r = 0; r < rows(); ++r) {
                if (!has[lc][r]) continue;
                uint64_t ttl; std::memcpy(&ttl, &data[lc][r * 8], 8);
                ttl -= 1;  // release-mode wrapping `**ttl -= 1`
                std::memcpy(&data[lc][r * 8], &ttl, 8);
                if (ttl == 0) despawn.push_back(r);
            }
            break;
        }
        case BGR_SYS_BOX_MOVE: {  // box_game.rs:154-206 ; player handle == RollbackOrdered index
            uint32_t tc = s.cols[0], vc = s.cols[1];
            const float ACCELERATION = 18.0f, MAX_SPEED = 3.0f, FRICTION = 0.0018f, PLANE_SIZE = 5.0f, CUBE_SIZE = 0.2f;
            for (size_t r = 0; r < rows(); ++r) {
                if (!has[tc][r] || !has[vc][r]) continue;  // Query<(&mut Transform, &mut Velocity, &Player)>
                float* t = reinterpret_cast<float*>(&data[tc][r * 40]);
                float* v = reinterpret_cast<float*>(&data[vc][r * 12]);
                uint64_t handle = rollback_ordered.order_of(rollback_id[r]);
                uint8_t input = handle < n_players ? player_inputs[handle] : 0;
                const uint8_t UP = 1, DOWN = 2, LEFT = 4, RIGHT = 8;
                if ((input & UP) && !(input & DOWN)) v[2] -= ACCELERATION * dt;
                if (!(input & UP) && (input & DOWN)) v[2] += ACCELERATION * dt;
                if ((input & LEFT) && !(input & RIGHT)) v[0] -= ACCELERATION * dt;
                if (!(input & LEFT) && (input & RIGHT)) v[0] += ACCELERATION * dt;
                if (!(input & UP) && !(input & DOWN)) v[2] *= std::pow(FRICTION, dt);
                if (!(input & LEFT) && !(input & RIGHT)) v[0] *= std::pow(FRICTION, dt);
                v[1] *= std::pow(FRICTION, dt);
                // glam Vec3::clamp_length_max
                float len_sq = (v[0] * v[0]) + (v[1] * v[1]) + (v[2] * v[2]);
                if (len_sq > MAX_SPEED * MAX_SPEED) {
                    float l = std::sqrt(len_sq);
                    v[0] = MAX_SPEED * (v[0] / l); v[1] = MAX_SPEED * (v[1] / l); v[2] = MAX_SPEED * (v[2] / l);
                }
                t[0] += v[0] * dt; t[1] += v[1] * dt; t[2] += v[2] * dt;
                float hw = (PLANE_SIZE - CUBE_SIZE) * 0.5f;
                auto clampf = [](float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); };
                t[0] = clampf(t[0], -hw, hw);
                t[2] = clampf(t[2], -hw, hw);
            }
            break;
        }
        case BGR_SYS_U32_ADD: {  // tests/component_rollback.rs:25-29
            uint32_t c = s.cols[0], off = s.params[0], k = s.params[1], eb = columns[c].elem_bytes;
            for (size_t r = 0; r < rows(); ++r) {
                if (!has[c][r]) continue;
                uint32_t x; std::memcpy(&x, &data[c][r * size_t(eb) + off], 4);
                x += k;
                std::memcpy(&data[c][r * size_t(eb) + off], &x, 4);
            }
            break;
        }
        case BGR_SYS_U32_SATSUB_DESPAWN: {  // tests/synctest.rs:38-45
            uint32_t c = s.cols[0], off = s.params[0], k = s.params[1], eb = columns[c].elem_bytes;
            for (size_t r = 0; r < rows(); ++r) {
                if (!has[c][r]) continue;
                uint32_t x; std::memcpy(&x, &data[c][r * size_t(eb) + off], 4);
                x = x > k ? x - k : 0;
                std::memcpy(&data[c][r * size_t(eb) + off], &x, 4);
                if (x == 0) despawn.push_back(r);
            }
            break;
        }
        case BGR_SYS_DESPAWN_ON_INPUT: {  // tests/hierarchy.rs:36-45 delete_child_system, keyed on the entity's own component
            uint32_t c = s.cols[0], player = s.params[0], value = s.params[1];
            uint8_t input = player < n_players ? player_inputs[player] : 0;
            if (input == value)
                for (size_t r = 0; r < rows(); ++r)
                    if (has[c][r]) despawn.push_back(r);
            break;
        }
        case BGR_SYS_U32_STORE_CALL_COUNT: {  // tests/synctest.rs:92-97
            uint32_t c = s.cols[0], off = s.params[0], eb = columns[c].elem_bytes;
            uint32_t count = call_count++;
            for (size_t r = 0; r < rows(); ++r)
                if (has[c][r]) std::memcpy(&data[c][r * size_t(eb) + off], &count, 4);
            break;
        }
        case ORC_SYS_RESOURCE_U32_ADD: {  // increase_frame_system, box_game.rs:146-148: FrameCount{frame:u32} resource
            uint32_t ri = s.params[0];
            if (res_present[ri]) { uint32_t f; std::memcpy(&f, res_data[ri].data(), 4); f += 1; std::memcpy(res_data[ri].data(), &f, 4); }
            break;
        }
        default: throw std::runtime_error("unknown system id");
        }
    }

    // =====================================================================================
    // handle_requests (schedule_systems.rs:170-289)
    // =====================================================================================
    void handle_requests(const bgr_session_info& sess, const bgr_request* reqs, uint32_t n,
                         std::vector<bgr_checksum>& out) {
        for (uint32_t i = 0; i < n; ++i) {
            const bgr_request& rq = reqs[i];
            int32_t current_frame = rollback_frame_count;  // :190-193
            std::optional<uint32_t> maxp;                  // :197-202
            std::optional<int32_t> confirmed;              // :204-212
            switch (sess.kind) {
            case BGR_SESSION_P2P: maxp = sess.max_prediction; confirmed = sess.confirmed_frame; break;
            case BGR_SESSION_SYNCTEST: {
                maxp = sess.max_prediction;
                int32_t cf = current_frame - int32_t(sess.check_distance);
                if (cf >= 0) confirmed = cf;
                break;
            }
            case BGR_SESSION_SPECTATOR: maxp = 0; confirmed = current_frame; break;
            default: break;
            }
            if (maxp) max_prediction = *maxp;              // :214-216
            if (confirmed) confirmed_frame_count = *confirmed;  // :218-220
            switch (rq.kind) {
            case BGR_REQ_SAVE: {                           // :223-237
                save_world();
                out.push_back(bgr_checksum{rq.frame, 1u, checksum_lo, 0});
                break;
            }
            case BGR_REQ_LOAD: {                           // :238-250
                rollback_frame_count = rq.frame;
                load_world();
                break;
            }
            case BGR_REQ_ADVANCE: {                        // :251-269
                rollback_frame_count += 1;
                n_players = rq.n_players;
                std::memcpy(player_inputs, rq.inputs, BGR_MAX_PLAYERS);
                advance_world();
                n_players = 0;
                break;
            }
            default: throw std::runtime_error("bad request kind");
            }
        }
    }
};

}  // namespace oracle
