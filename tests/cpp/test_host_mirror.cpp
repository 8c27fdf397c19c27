// The reference's SyncTest integration tests (tests/synctest.rs, tests/component_rollback.rs,
// tests/common/mod.rs) and the particles stress test, written against the C++ host mirror
// (bevy_ggrs_b200/host/bevy_ggrs.hpp) and therefore through the C ABI onto the GPU.
// Exit code 0 = all passed.  Needs an H100 (run by tests/test_gpu_cpp_host_mirror.py, -m gpu);
// `--no-gpu` only checks that the engine refuses to start without a device.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>

#include "../../bevy_ggrs_b200/host/bevy_ggrs.hpp"
#include "../../oracle/world.hpp"  // the checker: tests may link the oracle (never the product)

using namespace bevy_ggrs;

static int g_failed = 0;
#define EXPECT(cond)                                                                  \
    do {                                                                              \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failed; } \
    } while (0)

// ---- components of the reference tests / examples ----
struct Score { uint32_t v; };                                    // component_rollback.rs:22-23
struct Health { uint32_t v; };                                   // synctest.rs:24-31
struct Counter { uint32_t v; };                                  // synctest.rs:87-88
struct FrameCounter { uint32_t v; };
struct Transform { float translation[3]; float rotation[4]; float scale[3]; };  // 40 B payload
struct Velocity { float v[3]; };                                 // particles.rs:104-105
struct Ttl { uint64_t frames; };                                 // particles.rs:122-123

// tests/common/mod.rs:16-22
static void input_system(App& app) {
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = 0;
    app.insert_resource(li);
}
// tests/common/mod.rs:44-54
static void base_synctest_app(App& app, size_t check_distance) {
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(1, check_distance)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system);
}

static void copy_strategy_rolls_back_component_data() {  // component_rollback.rs:33-64
    std::printf("copy_strategy_rolls_back_component_data\n");
    App app(16, 8);
    base_synctest_app(app, 2);
    app.rollback_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.write<Score>(a.spawn(1), {Score{0}}); });
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    for (int i = 0; i < 20; ++i) app.update();
    EXPECT(!mismatch);
    EXPECT(app.rollback_frame_count() == 19);
    EXPECT(app.read<Score>(0, 1)[0].v == uint32_t(app.rollback_frame_count()));
}

static void despawn_and_rollback_does_not_panic() {  // synctest.rs:59-75
    std::printf("despawn_and_rollback_does_not_panic\n");
    App app(16, 8);
    base_synctest_app(app, 5);
    app.rollback_component_with_copy<Health>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_SATSUB_DESPAWN, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.write<Health>(a.spawn(1), {Health{10}}); });
    for (int i = 0; i < 60; ++i) app.update();
    EXPECT(app.active_count() == 0);
}

static void synctest_mismatch_fires_on_non_determinism() {  // synctest.rs:83-125
    std::printf("synctest_mismatch_fires_on_non_determinism\n");
    App app(16, 8);
    base_synctest_app(app, 2);
    app.rollback_component_with_copy<Counter>().checksum_component_with_hash<Counter>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_STORE_CALL_COUNT, {0}, {0}});
    app.add_systems(Startup{}, [](App& a) { a.spawn(1); });
    bool detected = false;
    app.add_observer([&](const SyncTestMismatch& m) { detected = true; EXPECT(!m.mismatched_frames.empty()); });
    for (int i = 0; i < 10; ++i) app.update();
    EXPECT(detected);
}

static void synctest_prunes_confirmed_snapshots() {  // synctest.rs:129-153
    std::printf("synctest_prunes_confirmed_snapshots\n");
    App app(16, 8);
    base_synctest_app(app, 5);
    app.rollback_component_with_clone<FrameCounter>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.spawn(1); });
    for (int i = 0; i < 20; ++i) app.update();
    EXPECT(app.confirmed_frame_count() > 0);
    EXPECT(!app.peek<FrameCounter>(0, 0, 1).has_value());
    auto newest = app.peek<FrameCounter>(app.rollback_frame_count() - 1, 0, 1);
    EXPECT(newest.has_value() && (*newest)[0].v == uint32_t(app.rollback_frame_count() - 1));
}

static void rollback_missing_frame_panics() {  // mod.rs:467-473 through the engine
    std::printf("rollback_missing_frame_panics\n");
    App app(16, 8);
    app.rollback_component_with_copy<Score>();
    app.spawn(1);
    bgr_checksum cs;
    check(bgr_save_world(app.engine(), &cs));
    check(bgr_set_rollback_frame_count(app.engine(), 99));
    bool panicked = false;
    try { check(bgr_load_world(app.engine())); }
    catch (const Panic& p) { panicked = std::string(p.what()).find("Could not rollback to 99") != std::string::npos && p.status == BGR_ERR_NO_SNAPSHOT; }
    EXPECT(panicked);
}

static void particles_stress_synctest() {  // examples/stress_tests/particles.rs as a SyncTest (BASELINE C2 shape, small)
    std::printf("particles_stress_synctest\n");
    const uint32_t n = 20000;
    App app(n, 9);
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(2, 8, 9, 2)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .insert_resource(RollbackFrameRate{60})
        .add_systems(ReadInputs{}, input_system)
        .rollback_component_with_clone<Transform>()
        .rollback_component_with_copy<Velocity>()
        .rollback_component_with_copy<Ttl>()
        .checksum_component<Velocity>(hash_bytes(0, 12, true))   // impl Hash for Velocity asserts is_finite (particles.rs:107-120)
        .checksum_component<Transform>(hash_bytes(0, 12, true));
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_UPDATE, {0, 1}, {}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_DESPAWN, {2}, {}});
    std::vector<Transform> t(n); std::vector<Velocity> v(n); std::vector<Ttl> l(n);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return float(double(s >> 11) / double(1ull << 53)); };
    for (uint32_t i = 0; i < n; ++i) {
        t[i] = Transform{{rnd() * 720.f - 360.f, rnd() * 720.f - 360.f, 0.f}, {0, 0, 0, 1}, {1, 1, 1}};
        v[i] = Velocity{{rnd() * 400.f - 200.f, rnd() * 400.f - 200.f, 0.f}};
        l[i] = Ttl{uint64_t(5 + (i % 40))};
    }
    uint32_t first = app.spawn(n);
    app.write<Transform>(first, t); app.write<Velocity>(first, v); app.write<Ttl>(first, l);
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    uint64_t l0 = app.launch_count();
    const int ticks = 30;
    for (int i = 0; i < ticks; ++i) app.step();
    EXPECT(!mismatch);
    EXPECT(app.rollback_frame_count() == ticks);
    EXPECT(app.launch_count() - l0 == uint64_t(ticks));  // one fused launch per handle_requests
    EXPECT(app.active_count() == uint64_t(std::count_if(l.begin(), l.end(), [&](const Ttl& x) { return x.frames > uint64_t(ticks); })));
    // rotation / scale are passive: bit-identical after 30 frames of save/load/advance
    auto t2 = app.read<Transform>(0, n);
    bool passive_ok = true;
    for (uint32_t i = 0; i < n; ++i)
        passive_ok = passive_ok && std::memcmp(t2[i].rotation, t[i].rotation, 28) == 0;
    EXPECT(passive_ok);
    // a survivor moved under gravity exactly 30 steps: y velocity decreased by ~ 200*0.5
    uint32_t k = n - 1;  // ttl 5 + (n-1)%40
    while (l[k].frames <= uint64_t(ticks)) --k;
    auto v2 = app.read<Velocity>(k, 1);
    EXPECT(std::fabs((v[k].v[1] - v2[0].v[1]) - 100.0f) < 0.01f);
}

// Option<&mut T> in ComponentSnapshotPlugin::load (component_snapshot.rs:99-115): a component removed by code outside
// GgrsSchedule is re-inserted by the next rollback, one inserted there is removed again; plus the async host mirror.
static void optional_component_is_reinserted_and_removed_by_rollback() {
    std::printf("optional_component_is_reinserted_and_removed_by_rollback\n");
    App app(16, 8);
    base_synctest_app(app, 3);
    app.rollback_optional_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.rollback_optional_component_with_copy<Health>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.spawn(2); a.remove<Health>(1); });
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    for (int i = 0; i < 10; ++i) app.update();
    EXPECT(app.has<Score>(0, 2) == (std::vector<uint8_t>{1, 1}));
    EXPECT(app.has<Health>(0, 2) == (std::vector<uint8_t>{1, 0}));
    app.remove<Score>(0);                 // (None, Some) at the next Load -> insert
    app.insert<Health>(1, Health{77});    // (Some, None) at the next Load -> remove
    EXPECT(app.has<Score>(0, 2) == (std::vector<uint8_t>{0, 1}));
    EXPECT(app.has<Health>(0, 2) == (std::vector<uint8_t>{1, 1}));
    app.update();
    EXPECT(app.has<Score>(0, 2) == (std::vector<uint8_t>{1, 1}));
    EXPECT(app.has<Health>(0, 2) == (std::vector<uint8_t>{1, 0}));
    auto sc = app.read<Score>(0, 2);
    EXPECT(sc[0].v == uint32_t(app.rollback_frame_count()) && sc[1].v == sc[0].v);  // resimulated from the snapshot
    EXPECT(!mismatch);
    // asynchronous mirror of Score for both rows
    void* pinned = nullptr;
    EXPECT(bgr_host_alloc(8, &pinned) == BGR_OK);
    uint32_t tk = app.download_begin<Score>(0, 4, 0, 2, pinned);
    app.update();                         // the next tick runs while the copy is in flight
    app.download_wait(tk);
    const uint32_t* m = static_cast<const uint32_t*>(pinned);
    EXPECT(m[0] == sc[0].v && m[1] == sc[1].v);
    bgr_host_free(pinned);
}

struct FrameCount { uint32_t frame; };  // box_game.rs:49-53

// BASELINE config C1: box_game SyncTest, 2 players, check_distance 8 (max_prediction 9), input_delay 2
// (examples/box_game/box_game_synctest.rs) — engine through the C++ mirror vs the oracle in the same process.
static void box_game_synctest_c1() {
    std::printf("box_game_synctest_c1\n");
    const uint8_t seq[8] = {1, 8, 5, 0, 2, 10, 4, 9};
    int tick_e = 0;
    App app(4, 9);
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(2, 8, 9, 2)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, [&](App& a) {
            LocalInputs li;
            for (auto h : a.local_players().handles) li.inputs[h] = seq[(tick_e + 3 * int(h)) % 8];
            a.insert_resource(li);
        })
        .rollback_resource_with_copy<FrameCount>(FrameCount{0})
        .rollback_component_with_copy<Velocity>()
        .rollback_component_with_clone<Transform>()
        .checksum_resource_with_hash<FrameCount>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_BOX_MOVE, {1, 0}, {}});
    app.add_systems(GgrsSchedule{}, ResourceSystem{[](App& a) { a.resource<FrameCount>().frame += 1; }});  // increase_frame_system
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    std::vector<Transform> t0(2);
    for (int h = 0; h < 2; ++h) {
        float rot = float(h) / 2.0f * 2.0f * 3.14159265358979323846f, r = 5.0f / 4.0f;
        t0[h] = Transform{{r * std::cos(rot), 0.1f, r * std::sin(rot)}, {0, 0, 0, 1}, {1, 1, 1}};
    }
    app.write<Transform>(app.spawn(2), t0);

    // the oracle, driven with the same request vectors
    oracle::World w;
    uint32_t ov = w.add_column("Velocity", 12), ot = w.add_column("Transform", 40);
    uint32_t zero = 0;
    uint32_t fc = w.add_resource("FrameCount", &zero, 4, true);
    w.systems.push_back({BGR_SYS_BOX_MOVE, {ot, ov}, {}});
    w.systems.push_back({oracle::ORC_SYS_RESOURCE_U32_ADD, {}, {fc}});
    w.spawn(2);
    std::memcpy(w.data[ot].data(), t0.data(), 80);
    ggrs::SyncTestSession osess(2, 8, 9, 2);
    bool all_equal = true;
    size_t n_cs = 0;
    for (int i = 0; i < 100; ++i) {
        app.step();
        for (size_t h = 0; h < 2; ++h) osess.add_local_input(h, seq[(tick_e + 3 * int(h)) % 8]);
        ++tick_e;
        std::vector<ggrs::GgrsRequest> reqs; ggrs::MismatchedChecksum err;
        if (!osess.advance_frame(reqs, err)) { mismatch = true; break; }
        std::vector<bgr_request> br(reqs.size());
        for (size_t k = 0; k < reqs.size(); ++k) {
            std::memset(&br[k], 0, sizeof(bgr_request));
            br[k].kind = uint32_t(reqs[k].kind); br[k].frame = reqs[k].frame; br[k].n_players = uint32_t(reqs[k].inputs.size());
            for (size_t p = 0; p < reqs[k].inputs.size(); ++p) br[k].inputs[p] = reqs[k].inputs[p].first;
        }
        bgr_session_info info{BGR_SESSION_SYNCTEST, 9, 8, 0};
        std::vector<bgr_checksum> ocs;
        w.handle_requests(info, br.data(), uint32_t(br.size()), ocs);
        for (auto& c : ocs) osess.save_cell(c.frame, (static_cast<unsigned __int128>(c.hi) << 64) | c.lo);
        const auto& ecs = app.last_checksums();
        all_equal = all_equal && ecs.size() == ocs.size();
        for (size_t k = 0; k < ocs.size() && k < ecs.size(); ++k, ++n_cs)
            all_equal = all_equal && ecs[k].lo == ocs[k].lo && ecs[k].frame == ocs[k].frame;
    }
    EXPECT(!mismatch);
    EXPECT(all_equal && n_cs > 400);  // FrameCount part ^ entity part: bit-identical
    EXPECT(app.resource<FrameCount>().frame == 100);
    auto te = app.read<Transform>(0, 2);
    auto ve = app.read<Velocity>(0, 2);
    bool equal = true, moved = false;
    for (int h = 0; h < 2; ++h) {
        size_t row = size_t(w.find_row(uint64_t(h)));
        equal = equal && std::memcmp(te[h].translation, &w.data[ot][row * 40], 12) == 0;
        equal = equal && std::memcmp(ve[h].v, &w.data[ov][row * 12], 12) == 0;
        for (int k = 0; k < 3; ++k) moved = moved || ve[h].v[k] != 0.0f;
    }
    EXPECT(equal);  // bit-identical: the friction factor is the C library's powf on both sides
    EXPECT(moved);
}

// tests/p2p.rs:268-304 (p2p_confirmed_frame_advances_and_prunes_snapshots), with the trace-driven P2P stand-in instead
// of two UDP peers: ConfirmedFrameCount follows the session's confirmed_frame, snapshots older than it are pruned, and
// the rollbacks the "remote" peer causes resimulate to the same state (score == frame, component_rollback.rs:54-64).
static void p2p_confirmed_frame_advances_and_prunes_snapshots() {
    std::printf("p2p_confirmed_frame_advances_and_prunes_snapshots\n");
    App app(16, 8);
    std::vector<int> depths;
    for (int t = 0; t < 60; ++t) depths.push_back((t * 7 + 3) % 5 == 0 ? 0 : (t * 5 + 1) % 4);  // 0..3 frames of misprediction
    app.insert_resource(Session::P2P(ggrs::P2PTraceSession(2, 8, depths, /*confirm_lag=*/3)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system);
    app.rollback_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.write<Score>(a.spawn(1), {Score{0}}); });
    for (int i = 0; i < 50; ++i) app.update();
    const int32_t confirmed = app.confirmed_frame_count(), frame = app.rollback_frame_count();
    EXPECT(confirmed > 0);                                  // advances once the session confirms frames
    EXPECT(frame == 49 && confirmed == frame - 3);
    EXPECT(!app.peek<Score>(0, 0, 1).has_value());          // the frame-0 snapshot was pruned (confirm, mod.rs:182-199)
    const auto frames = app.snapshot_frames();
    EXPECT(!frames.empty() && frames.size() <= 8);
    for (int32_t f : frames) EXPECT(f >= confirmed);        // nothing older than the confirmed frame survives
    EXPECT(app.read<Score>(0, 1)[0].v == uint32_t(frame));  // every rollback resimulated to the same state
    EXPECT(app.local_players().handles.size() == 1);        // local_player_handles(), not 0..num_players
    EXPECT(app.max_prediction_window() == 8);
}

// run_spectator (schedule_systems.rs:120-135) + the spectator arm of handle_requests (:199-201, :209): AdvanceFrame
// requests only — several per tick when catching up — MaxPredictionWindow 0, ConfirmedFrameCount = the frame in hand.
static void spectator_session_only_advances() {
    std::printf("spectator_session_only_advances\n");
    App app(16, 8);
    const std::vector<int> script = {1, 1, 3, 0, 2, 1, 0, 0, 4, 1};
    int total = 0;
    for (int k : script) total += k;
    app.insert_resource(Session::Spectator(ggrs::SpectatorTraceSession(2, script)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, [](App&) { std::printf("  FAILED: a spectator never reads local inputs\n"); ++g_failed; });
    app.rollback_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.write<Score>(a.spawn(1), {Score{0}}); });
    for (size_t i = 0; i <= script.size(); ++i) app.update();    // the first update has a zero delta
    EXPECT(app.rollback_frame_count() == total);
    EXPECT(app.read<Score>(0, 1)[0].v == uint32_t(total));
    EXPECT(app.snapshot_frames().empty());                       // no SaveGameState ever reaches a spectator
    EXPECT(app.max_prediction_window() == 0);
    EXPECT(app.confirmed_frame_count() == total - 1);            // = RollbackFrameCount when the last request was handled
    EXPECT(app.last_checksums().empty());
}

// tests/hierarchy.rs:125-188 (hierarchy): parent + child, both Rollback, linked by ChildOf; the child is despawned inside
// GgrsSchedule on one frame (delete_child_system, :36-45), rollbacks re-simulate that frame; afterwards the child is gone
// and the parent still exists.  ChildOf is an optional POD column holding the parent's RollbackOrdered index.
struct ParentEntity { uint8_t tag; };
struct ChildEntity { uint8_t tag; };
struct ChildOf { uint64_t parent; };
static void hierarchy_child_deleted_inside_the_schedule() {
    std::printf("hierarchy_child_deleted_inside_the_schedule\n");
    App app(8, 8);
    bool send_delete = false;
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(1, 2)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, [&](App& a) {
            LocalInputs li;
            li.inputs[0] = send_delete ? 1 : 0;   // hierarchy.rs:17-27
            send_delete = false;
            a.insert_resource(li);
        });
    app.rollback_optional_component_with_copy<ParentEntity>().rollback_optional_component_with_copy<ChildEntity>()
        .rollback_optional_component_with_copy<ChildOf>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_DESPAWN_ON_INPUT, {app.col<ChildOf>()}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) {
        const uint32_t first = a.spawn(2);
        a.remove<ChildEntity>(first); a.remove<ChildOf>(first);       // the parent
        a.remove<ParentEntity>(first + 1);                            // the child ...
        a.write<ChildOf>(first + 1, {ChildOf{first}});               // ... of the parent
    });
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    app.update();
    EXPECT(app.active_count() == 2 && app.has<ChildOf>(0, 2)[1] == 1 && app.read<ChildOf>(1, 1)[0].parent == 0);
    app.update();
    send_delete = true;
    for (int i = 0; i < 5; ++i) app.update();
    EXPECT(!mismatch);
    EXPECT(app.active_count() == 1);                                  // the child is gone ...
    EXPECT(app.has<ChildEntity>(0, 2)[1] == 0 && app.has<ChildOf>(0, 2)[1] == 0);
    EXPECT(app.has<ParentEntity>(0, 2)[0] == 1);                      // ... the parent still exists
}

// schedule_systems.rs:70-79: without a session the frame resources are reset
static void removed_session_resets_frame_resources() {
    std::printf("removed_session_resets_frame_resources\n");
    App app(16, 8);
    base_synctest_app(app, 2);
    app.rollback_component_with_copy<Score>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(Startup{}, [](App& a) { a.write<Score>(a.spawn(1), {Score{0}}); });
    for (int i = 0; i < 12; ++i) app.update();
    EXPECT(app.rollback_frame_count() == 11 && app.confirmed_frame_count() >= 0);
    app.remove_session();
    app.update();
    EXPECT(app.rollback_frame_count() == 0);
    EXPECT(app.confirmed_frame_count() == -1);
    EXPECT(app.max_prediction_window() == 8);
    EXPECT(app.local_players().handles.empty());
}

// particles.rs:191 `rollback_component_with_clone::<Sprite>()`: Sprite holds an Arc asset handle — Clone, not plain
// bytes.  It stays on the host (side table) and is rolled back by the same request vectors as the HBM columns.
struct Sprite {
    std::shared_ptr<int> image;  // the Arc
    int id;
};
static void non_pod_component_rolls_back_on_the_host_side_table() {
    std::printf("non_pod_component_rolls_back_on_the_host_side_table\n");
    App app(16, 8);
    base_synctest_app(app, 2);
    app.rollback_component_with_copy<Health>().checksum_component_with_hash<Health>();
    app.rollback_component_with_clone<Sprite>();   // not trivially copyable -> host side table
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_SATSUB_DESPAWN, {0}, {0, 1}});
    auto image = std::make_shared<int>(7);
    app.add_systems(Startup{}, [&](App& a) {
        a.write<Health>(a.spawn(3), {Health{1000}, Health{1000}, Health{9}});   // row 2 dies in frame 9
        for (uint32_t r = 0; r < 3; ++r) a.host_insert<Sprite>(r, Sprite{image, int(10 + r)});
    });
    bool mismatch = false;
    app.add_observer([&](const SyncTestMismatch&) { mismatch = true; });
    for (int i = 0; i < 6; ++i) app.update();
    EXPECT(!mismatch);
    EXPECT(app.host_get<Sprite>(0) && app.host_get<Sprite>(0)->id == 10 && app.host_get<Sprite>(2)->id == 12);
    EXPECT(app.host_get<Sprite>(1)->image.get() == image.get());      // clones share the asset
    EXPECT(image.use_count() > 4);                                     // ... and the snapshots hold clones
    EXPECT(app.host_snapshot_frames<Sprite>() == [&] { auto f = app.snapshot_frames(); std::sort(f.begin(), f.end()); return f; }());
    // an edit outside GgrsSchedule is undone by the next tick's Load of an older frame (any rollback component behaves so)
    app.host_remove<Sprite>(1);
    app.host_insert<Sprite>(0, Sprite{image, 99});
    EXPECT(!app.host_get<Sprite>(1) && app.host_get<Sprite>(0)->id == 99);
    app.update();
    EXPECT(app.host_get<Sprite>(1) && app.host_get<Sprite>(1)->id == 11 && app.host_get<Sprite>(0)->id == 10);
    // the entity of row 2 despawns inside the schedule (Health runs out): its Sprite goes with it
    for (int i = 0; i < 8; ++i) app.update();
    EXPECT(app.active_count() == 2);
    EXPECT(!app.host_get<Sprite>(2) && app.host_get<Sprite>(0) && app.host_get<Sprite>(1));
    bool threw = false;
    try { app.host_insert<Sprite>(2, Sprite{image, 1}); } catch (const Panic&) { threw = true; }
    EXPECT(threw);                                                      // no such entity any more
    EXPECT(!mismatch);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        // the library must refuse loudly (no CPU fallback) when no device is usable
        try {
            App app(16, 8);
            app.rollback_component_with_copy<Score>();
            app.spawn(1);
            std::printf("engine started: a GPU is present\n");
            return 0;
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
            return (p.status == BGR_ERR_CUDA) ? 0 : 1;
        }
    }
    try {
        copy_strategy_rolls_back_component_data();
        despawn_and_rollback_does_not_panic();
        synctest_mismatch_fires_on_non_determinism();
        synctest_prunes_confirmed_snapshots();
        rollback_missing_frame_panics();
        particles_stress_synctest();
        optional_component_is_reinserted_and_removed_by_rollback();
        box_game_synctest_c1();
        p2p_confirmed_frame_advances_and_prunes_snapshots();
        spectator_session_only_advances();
        removed_session_resets_frame_resources();
        hierarchy_child_deleted_inside_the_schedule();
        non_pod_component_rolls_back_on_the_host_side_table();
    } catch (const std::exception& e) {
        std::printf("unexpected exception: %s\n", e.what());
        return 2;
    }
    std::printf(g_failed ? "%d check(s) FAILED\n" : "all host-mirror tests passed\n", g_failed);
    return g_failed ? 1 : 0;
}
