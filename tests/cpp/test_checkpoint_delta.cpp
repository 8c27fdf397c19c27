// Checkpoint deltas through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): a box_game SyncTest App with a
// FrameCount resource takes a full checkpoint of a frame that the engine later retains, then a delta of a later frame
// against it.  One App restored from base plus delta and one restored from the later frame's full checkpoint both take
// over a copy of the session and continue with the source's checksums and resources, without a SyncTestMismatch.  A
// malformed resource section in either blob is refused, changing nothing, and both calls are refused while a host-side
// component table is registered.  Exit code 0 = passed.  Needs an H100 (tests/test_gpu_checkpoint_delta.py).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../bevy_ggrs_b200/host/bevy_ggrs.hpp"

using namespace bevy_ggrs;

static int g_failed = 0;
#define EXPECT(cond)                                                                  \
    do {                                                                              \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failed; } \
    } while (0)

struct Transform { float translation[3]; float rotation[4]; float scale[3]; };
struct Velocity { float v[3]; };
struct FrameCount { uint32_t frame; };  // box_game.rs:49-53
struct Sprite { std::string handle; };  // not plain bytes: a host-side component table

static const uint8_t kSeq[8] = {1, 8, 5, 0, 2, 10, 4, 9};
static const size_t kCheckDistance = 3;

// box_game as a SyncTest (examples/box_game/box_game_synctest.rs); inputs follow *tick
static void box_game(App& app, const Session& sess, int* tick, bool* mismatch) {
    app.insert_resource(sess)
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, [tick](App& a) {
            LocalInputs li;
            for (auto h : a.local_players().handles) li.inputs[h] = kSeq[(*tick + 3 * int(h)) % 8];
            a.insert_resource(li);
            *tick += 1;
        })
        .rollback_resource_with_copy<FrameCount>(FrameCount{0})
        .rollback_component_with_copy<Velocity>()
        .rollback_component_with_clone<Transform>()
        .checksum_resource_with_hash<FrameCount>()
        .checksum_component<Transform>(hash_bytes(0, 12))
        .retain_confirmed(4, 2);
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_BOX_MOVE, {1, 0}, {}});
    app.add_systems(GgrsSchedule{}, ResourceSystem{[](App& a) { a.resource<FrameCount>().frame += 1; }});  // increase_frame_system
    app.add_observer([mismatch](const SyncTestMismatch&) { *mismatch = true; });
}

static void spawn_players(App& app) {
    std::vector<Transform> t0(2);
    for (int h = 0; h < 2; ++h) {
        float rot = float(h) / 2.0f * 2.0f * 3.14159265358979323846f, r = 5.0f / 4.0f;
        t0[h] = Transform{{r * std::cos(rot), 0.1f, r * std::sin(rot)}, {0, 0, 0, 1}, {1, 1, 1}};
    }
    app.write<Transform>(app.spawn(2), t0);
}

static int status_of(const std::function<void()>& f) {
    try { f(); } catch (const Panic& p) { return p.status; }
    return BGR_OK;
}

static bool same_checksums(const std::vector<bgr_checksum>& x, const std::vector<bgr_checksum>& y) {
    if (x.size() != y.size()) return false;
    for (size_t k = 0; k < x.size(); ++k)
        if (x[k].frame != y[k].frame || x[k].lo != y[k].lo || x[k].hi != y[k].hi) return false;
    return true;
}

static void app_delta_continues_the_match() {
    std::printf("app_delta_continues_the_match\n");
    Session sa = Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2));
    int tick_a = 0, tick_b = 0, tick_c = 0;
    bool mis_a = false, mis_b = false, mis_c = false;
    App a(8, 9), b(8, 9), c(8, 9);
    box_game(a, sa, &tick_a, &mis_a);
    box_game(b, Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2)), &tick_b, &mis_b);
    box_game(c, Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2)), &tick_c, &mis_c);
    spawn_players(a);
    for (int i = 0; i < 40; ++i) a.step();
    // a base frame the engine retains once it is confirmed (a multiple of retain_confirmed's interval)
    while ((sa.synctest->current_frame() - ggrs::Frame(kCheckDistance)) % 4 != 0) a.step();
    const ggrs::Frame fb = sa.synctest->current_frame() - ggrs::Frame(kCheckDistance);
    const std::vector<uint8_t> base = a.checkpoint(fb);
    EXPECT(!base.empty());
    for (int i = 0; i < 5; ++i) a.step();
    const ggrs::Frame f = sa.synctest->current_frame() - ggrs::Frame(kCheckDistance);
    const std::vector<uint8_t> delta = a.checkpoint_delta(f, fb), full = a.checkpoint(f);
    EXPECT(!delta.empty() && delta == a.checkpoint_delta(f, fb));
    EXPECT(delta.size() < full.size() + sizeof(bgr_checkpoint_delta_header));
    // the App holds no resources of the retained base frame, so it cannot be a delta's target
    EXPECT(status_of([&] { a.checkpoint_delta(fb, f); }) == BGR_ERR_NO_SNAPSHOT);
    spawn_players(b);
    b.step();
    const auto frames_before = b.snapshot_frames();
    std::vector<uint8_t> shorter(delta.begin(), delta.end() - 1), longer = delta, bad_base = base;
    longer.push_back(0);
    bad_base[bad_base.size() - 8] = 8;  // the base's FrameCount length field
    EXPECT(status_of([&] { b.restore_checkpoint_delta(base, shorter); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(status_of([&] { b.restore_checkpoint_delta(base, longer); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(status_of([&] { b.restore_checkpoint_delta(bad_base, delta); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(status_of([&] { b.restore_checkpoint_delta(full, delta); }) == BGR_ERR_INVALID_ARGUMENT);  // another base
    EXPECT(b.snapshot_frames() == frames_before);
    b.restore_checkpoint_delta(base, delta);
    c.restore_checkpoint(full);
    b.insert_resource(Session::SyncTest(*sa.synctest));
    c.insert_resource(Session::SyncTest(*sa.synctest));
    EXPECT(b.snapshot_frames() == std::vector<int32_t>{f});
    EXPECT(b.checkpoint(f) == full);
    tick_b = tick_c = tick_a;
    bool same = true;
    size_t n = 0;
    for (int i = 0; i < 40; ++i) {
        a.step();
        b.step();
        c.step();
        same = same && same_checksums(a.last_checksums(), b.last_checksums()) && same_checksums(b.last_checksums(), c.last_checksums());
        n += a.last_checksums().size();
    }
    EXPECT(same && n >= 40);
    EXPECT(!mis_a && !mis_b && !mis_c);
    EXPECT(a.resource<FrameCount>().frame == b.resource<FrameCount>().frame);
    const auto ta = a.read<Transform>(0, 2), tb = b.read<Transform>(0, 2);
    EXPECT(std::memcmp(ta.data(), tb.data(), sizeof(Transform) * 2) == 0);
}

static void app_with_host_columns_refuses() {
    std::printf("app_with_host_columns_refuses\n");
    int tick = 0;
    bool mis = false;
    App app(8, 9);
    box_game(app, Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2)), &tick, &mis);
    app.rollback_component_with_clone<Sprite>();
    spawn_players(app);
    for (int i = 0; i < 10; ++i) app.step();
    const ggrs::Frame f = app.snapshot_frames()[0];
    EXPECT(status_of([&] { app.checkpoint_delta(f, f); }) == BGR_ERR_UNSUPPORTED);
    EXPECT(status_of([&] { app.restore_checkpoint_delta(std::vector<uint8_t>(200, 0), std::vector<uint8_t>(200, 0)); }) == BGR_ERR_UNSUPPORTED);
}

int main() {
    app_delta_continues_the_match();
    app_with_host_columns_refuses();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "checkpoint delta test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
