// The change feed through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): after every Bevy frame of a SyncTest
// session, a feed over Score is applied to a row map with App::apply_feed, and the map must hold exactly the rows that
// have a Score in the live world, with its value (read_component / has).  Health runs out on some rows (despawns,
// undone and redone by every re-simulation) and the host spawns rows between frames.
// Exit code 0 = passed.  Needs an H100 (tests/test_cpp_change_feed.py, -m gpu); `--no-gpu` only checks that the
// engine refuses to start without a device.
#include <cstdio>
#include <map>
#include <string>

#include "../../bevy_ggrs_b200/host/bevy_ggrs.hpp"

using namespace bevy_ggrs;

static int g_failed = 0;
#define EXPECT(cond)                                                                  \
    do {                                                                              \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failed; } \
    } while (0)

struct Score { uint32_t v; };   // +1 per frame
struct Health { uint32_t v; };  // -1 per frame, despawns at 0

static void input_system(App& app) {
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = 0;
    app.insert_resource(li);
}

static void feed_mirror_follows_the_live_world() {
    std::printf("feed_mirror_follows_the_live_world\n");
    const uint32_t rows = 1300, cap = 4096;
    App app(cap, 8);
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(1, 2)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system);
    app.rollback_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.rollback_component_with_copy<Health>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_SATSUB_DESPAWN, {1}, {0, 1}});
    app.add_systems(Startup{}, [&](App& a) {
        a.spawn(rows);
        std::vector<Health> h(rows);
        for (uint32_t r = 0; r < rows; ++r) h[r].v = 3 + r % 40;
        a.write<Health>(0, h);
    });
    app.update();  // builds the engine and runs Startup
    const uint32_t feed = app.feed_create({bgr_feed_field{app.col<Score>(), 0, 4}});
    void* buf = nullptr;
    if (bgr_host_alloc(size_t(cap) * 12, &buf) != BGR_OK) { EXPECT(false); return; }
    std::map<uint32_t, Score> mirror;
    size_t changed = 0;
    for (int i = 0; i < 40; ++i) {
        if (i % 9 == 4) app.spawn(5);
        app.update();
        const bgr_feed_info info = app.feed_wait(app.feed_begin(feed, buf, cap));
        EXPECT(info.pending == 0 && info.record_bytes == 12);
        App::apply_feed<Score>(buf, info, 0, 0, mirror);
        changed += info.n_records;
        const uint32_t n = info.rows;
        const std::vector<Score> score = app.read<Score>(0, n);
        const std::vector<uint8_t> has = app.has<Score>(0, n);
        std::map<uint32_t, Score> want;
        for (uint32_t r = 0; r < n; ++r)
            if (has[r]) want[r] = score[r];
        EXPECT(want.size() == mirror.size());
        bool same = want.size() == mirror.size();
        for (auto it = want.begin(), jt = mirror.begin(); same && it != want.end(); ++it, ++jt)
            same = it->first == jt->first && it->second.v == jt->second.v;
        EXPECT(same);
    }
    EXPECT(changed > rows && mirror.size() < rows);
    bgr_host_free(buf);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(16, 8);
            app.rollback_component_with_copy<Score>();
            app.spawn(1);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    feed_mirror_follows_the_live_world();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "change feed test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
