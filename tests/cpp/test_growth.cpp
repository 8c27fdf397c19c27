// Growable worlds through the C++ host mirror: the particles stress test created for 1024 rows with
// BGR_CFG_GROWABLE, the spawn input held until the world holds many times that, run as a SyncTest.  Every re-simulated
// frame must checksum as it did the first time, and the world must end as an engine created large enough from the
// start ends.  Exit code 0 = passed.  Needs an H100 (tests/test_cpp_growth.py, -m gpu); `--no-gpu` only checks that
// the engine refuses to start without a device.
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
struct Ttl { uint64_t frames; };

static void spawn_pressed(App& app) {  // the spawn input held by every local player (particles.rs:254-256)
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = BGR_INPUT_SPAWN;
    app.insert_resource(li);
}

// ticks of the particles world with the spawn input held; returns the checksums of every tick and the final state
struct Run { std::vector<bgr_checksum> checksums; std::vector<Velocity> velocity; uint32_t rows = 0, capacity = 0; uint64_t active = 0; bool mismatch = false; };

static Run run(uint32_t max_entities, uint32_t flags, int ticks) {
    App app(max_entities, 9, 0, flags);
    Run r;
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(2, 7)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .insert_resource(RollbackFrameRate{60})
        .add_systems(ReadInputs{}, spawn_pressed)
        .rollback_component_with_clone<Transform>()
        .rollback_component_with_copy<Velocity>()
        .rollback_component_with_copy<Ttl>()
        .checksum_component<Velocity>(hash_bytes(0, 12, true))
        .checksum_component<Transform>(hash_bytes(0, 12, true));
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_UPDATE, {0, 1}, {}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_DESPAWN, {2}, {}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_SPAWN, {0, 1, 2}, {1000, 100000, 7, 0}});
    app.add_observer([&](const SyncTestMismatch&) { r.mismatch = true; });
    for (int i = 0; i < ticks; ++i) {
        app.step();
        for (const bgr_checksum& c : app.last_checksums()) r.checksums.push_back(c);
    }
    check(bgr_row_count(app.engine(), &r.rows));
    r.active = app.active_count();
    r.velocity = app.read<Velocity>(0, r.rows);
    r.capacity = app.capacity().first;
    return r;
}

static void particles_grow_far_past_the_initial_capacity() {
    std::printf("particles_grow_far_past_the_initial_capacity\n");
    const int ticks = 60;  // 1000 rows per frame: ~60 000 rows, from a capacity of 1024
    Run g = run(1024, BGR_CFG_GROWABLE, ticks);
    EXPECT(!g.mismatch);
    EXPECT(g.rows > 50u * 1024u);
    EXPECT(g.capacity >= g.rows);
    Run f = run(g.capacity, 0, ticks);  // the twin: created with the final capacity, no growth
    EXPECT(!f.mismatch);
    EXPECT(f.rows == g.rows && f.active == g.active);
    bool same = g.checksums.size() == f.checksums.size();
    for (size_t i = 0; same && i < g.checksums.size(); ++i)
        same = g.checksums[i].frame == f.checksums[i].frame && g.checksums[i].lo == f.checksums[i].lo;
    EXPECT(same);
    EXPECT(g.velocity.size() == f.velocity.size() &&
           std::memcmp(g.velocity.data(), f.velocity.data(), g.velocity.size() * sizeof(Velocity)) == 0);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(1024, 8, 0, BGR_CFG_GROWABLE);
            app.rollback_component_with_copy<Velocity>();
            app.reserve(4096);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    particles_grow_far_past_the_initial_capacity();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "growth test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
