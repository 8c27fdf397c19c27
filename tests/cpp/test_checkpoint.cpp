// World checkpoints through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): a box_game SyncTest App with a
// FrameCount resource is checkpointed at the frame its next tick loads and restored into a second App that takes over a
// copy of the session.  Both continue with identical checksums and resources and no SyncTestMismatch.  The App refuses a
// frame whose resource snapshot it no longer holds, a malformed resource section (changing nothing), and both calls
// while a host-side component table is registered.  Exit code 0 = passed.  Needs an H100 (tests/test_cpp_checkpoint.py,
// -m gpu); `--no-gpu` only checks that the engine refuses to start without a device.
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

static void app_checkpoint_continues_the_match() {
    std::printf("app_checkpoint_continues_the_match\n");
    Session sa = Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2));  // the test keeps a handle on it
    int tick_a = 0, tick_b = 0;
    bool mis_a = false, mis_b = false;
    App a(8, 9), b(8, 9);
    box_game(a, sa, &tick_a, &mis_a);
    box_game(b, Session::SyncTest(ggrs::SyncTestSession(2, kCheckDistance, 9, 2)), &tick_b, &mis_b);
    spawn_players(a);
    for (int i = 0; i < 60; ++i) a.step();
    // the frame the next tick loads: the restored ring holds it alone
    const ggrs::Frame f = sa.synctest->current_frame() - ggrs::Frame(kCheckDistance);
    const std::vector<uint8_t> blob = a.checkpoint(f);
    EXPECT(!blob.empty());
    EXPECT(blob == a.checkpoint(f));
    // a retained frame: the engine has it, the App's resource snapshot of it is gone
    const auto retained = a.retained_frames();
    EXPECT(!retained.empty());
    if (!retained.empty()) EXPECT(status_of([&] { a.checkpoint(retained[0]); }) == BGR_ERR_NO_SNAPSHOT);
    // a malformed resource section is refused before the engine restores: b is untouched
    spawn_players(b);
    b.step();
    const auto frames_before = b.snapshot_frames();
    std::vector<uint8_t> shorter(blob.begin(), blob.end() - 1), longer = blob;
    longer.push_back(0);
    std::vector<uint8_t> wrong_len = blob;
    wrong_len[wrong_len.size() - 8] = 8;  // FrameCount's length field
    for (auto* x : {&shorter, &longer, &wrong_len}) EXPECT(status_of([&] { b.restore_checkpoint(*x); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(b.snapshot_frames() == frames_before);
    // restore, and let b take over a copy of a's session
    b.restore_checkpoint(blob);
    b.insert_resource(Session::SyncTest(*sa.synctest));
    EXPECT(b.snapshot_frames() == std::vector<int32_t>{f});
    EXPECT(b.rollback_frame_count() == f);
    EXPECT(b.resource<FrameCount>().frame == a.resource<FrameCount>().frame - uint32_t(kCheckDistance));
    tick_b = tick_a;
    bool same = true;
    size_t n = 0;
    for (int i = 0; i < 40; ++i) {
        a.step();
        b.step();
        const auto& ca = a.last_checksums();
        const auto& cb = b.last_checksums();
        same = same && ca.size() == cb.size();
        for (size_t k = 0; same && k < ca.size(); ++k) same = ca[k].frame == cb[k].frame && ca[k].lo == cb[k].lo && ca[k].hi == cb[k].hi;
        n += ca.size();
    }
    EXPECT(same && n >= 40);
    EXPECT(!mis_a && !mis_b);
    EXPECT(a.resource<FrameCount>().frame == b.resource<FrameCount>().frame);
    EXPECT(a.read<Transform>(0, 2).size() == 2);
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
    EXPECT(status_of([&] { app.checkpoint(app.snapshot_frames()[0]); }) == BGR_ERR_UNSUPPORTED);
    EXPECT(status_of([&] { app.restore_checkpoint(std::vector<uint8_t>(200, 0)); }) == BGR_ERR_UNSUPPORTED);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(16, 8);
            app.rollback_component_with_copy<Velocity>();
            app.spawn(1);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    app_checkpoint_continues_the_match();
    app_with_host_columns_refuses();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "checkpoint test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
