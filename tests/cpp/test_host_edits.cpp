// Host edits through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): two P2P runs of the particles world with
// optional Velocity and Ttl.  Between frames one App sends the game's edits as App::Edits batches (field and whole writes,
// inserts, removes, despawns, spawns followed by writes to the new rows), the other issues the same edits through the
// single calls, a field write as a read-modify-write of the element.  Every frame's checksums and the live world after
// it must be the same.  Exit code 0 = passed.  Needs an H100 (tests/test_cpp_host_edits.py, -m gpu); `--no-gpu` only
// checks that the engine refuses to start without a device.
#include <cstdio>
#include <cstring>
#include <random>
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
struct Vec3 { float x, y, z; };

static const uint32_t kRows = 6000, kCap = 16384;

static void input_system(App& app) {
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = 0;
    app.insert_resource(li);
}

static void setup(App& app) {
    std::vector<int> depths;
    for (int t = 0; t < 200; ++t) depths.push_back((t * 5 + 3) % 4);
    app.insert_resource(Session::P2P(ggrs::P2PTraceSession(2, 8, depths, /*confirm_lag=*/3)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system)
        .rollback_component_with_clone<Transform>()
        .rollback_optional_component_with_copy<Velocity>()
        .rollback_optional_component_with_copy<Ttl>()
        .checksum_component<Velocity>(hash_bytes(0, 12, true))
        .checksum_component<Transform>(hash_bytes(0, 12, true));
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_UPDATE, {0, 1}, {}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_PARTICLES_DESPAWN, {2}, {}});
    app.add_systems(Startup{}, [](App& a) {
        a.spawn(kRows);
        std::vector<Transform> t(kRows);
        std::vector<Velocity> v(kRows);
        std::vector<Ttl> l(kRows);
        for (uint32_t r = 0; r < kRows; ++r) {
            t[r] = Transform{{float(r), 1.0f, 2.0f}, {0, 0, 0, 1}, {1, 1, 1}};
            v[r] = Velocity{{0.5f, -0.25f, float(r % 7)}};
            l[r] = Ttl{40u + r % 300u};
        }
        a.write<Transform>(0, t);
        a.write<Velocity>(0, v);
        a.write<Ttl>(0, l);
    });
}

static bool same_world(App& a, App& b) {
    uint32_t ra = 0, rb = 0;
    check(bgr_row_count(a.engine(), &ra));
    check(bgr_row_count(b.engine(), &rb));
    if (ra != rb) return false;
    auto eq = [](const auto& x, const auto& y) { return x.size() == y.size() && std::memcmp(x.data(), y.data(), x.size() * sizeof(x[0])) == 0; };
    return eq(a.read<Transform>(0, ra), b.read<Transform>(0, rb)) && eq(a.read<Velocity>(0, ra), b.read<Velocity>(0, rb)) &&
           eq(a.read<Ttl>(0, ra), b.read<Ttl>(0, rb)) && eq(a.has<Velocity>(0, ra), b.has<Velocity>(0, rb)) &&
           eq(a.has<Ttl>(0, ra), b.has<Ttl>(0, rb)) && a.active_count() == b.active_count();
}

static void edits_match_the_single_calls() {
    std::printf("edits_match_the_single_calls\n");
    App a(kCap, 9), b(kCap, 9);
    setup(a);
    setup(b);
    std::mt19937 rng(12345);
    size_t records = 0;
    for (int frame = 0; frame < 40; ++frame) {
        a.step();
        b.step();
        const auto& ca = a.last_checksums();
        const auto& cb = b.last_checksums();
        bool same = ca.size() == cb.size();
        for (size_t i = 0; same && i < ca.size(); ++i) same = ca[i].frame == cb[i].frame && ca[i].lo == cb[i].lo;
        EXPECT(same);
        uint32_t rows = 0;
        check(bgr_row_count(a.engine(), &rows));
        App::Edits ed(a);
        for (int k = 0; k < 24; ++k) {
            const uint32_t row = rng() % rows;
            switch (rng() % 7) {
            case 0: {  // Transform.translation only: rotation and scale are passive planes
                const Vec3 t{float(rng() % 1000), -1.5f, 0.25f * float(k)};
                ed.write_field<Transform>(row, 0, t);
                Transform x = b.read<Transform>(row, 1)[0];
                std::memcpy(x.translation, &t, sizeof t);
                b.write<Transform>(row, {x});
                break;
            }
            case 1: {  // a band of whole Velocity elements across a segment boundary
                const uint32_t first = std::min(rows - 1, (row / 64u) * 64u + 60u), n = std::min(rows - first, 9u);
                std::vector<Velocity> v(n);
                for (uint32_t i = 0; i < n; ++i) v[i] = Velocity{{float(rng() % 50) - 25.0f, 0.0f, 1.0f}};
                ed.write<Velocity>(first, v);
                b.write<Velocity>(first, v);
                break;
            }
            case 2: {
                const Ttl t{5u + rng() % 90u};
                ed.insert<Ttl>(row, t);
                b.insert<Ttl>(row, t);
                break;
            }
            case 3:
                ed.remove<Velocity>(row);
                b.remove<Velocity>(row);
                break;
            case 4:
                ed.despawn(row);
                check(bgr_despawn(b.engine(), row));
                break;
            case 5: {  // overlapping records on one row: the later wins
                const float y = float(rng() % 100);
                ed.write_field<Velocity>(row, 4, y).write_field<Velocity>(row, 4, y + 1.0f);
                Velocity v = b.read<Velocity>(row, 1)[0];
                v.v[1] = y + 1.0f;
                b.write<Velocity>(row, {v});
                break;
            }
            default: {  // spawn, then write the new rows
                if (rows + 70 > kCap) break;
                const uint32_t n = 1 + rng() % 70;
                ed.spawn(n);
                const uint32_t first = b.spawn(n);
                std::vector<Velocity> v(n, Velocity{{1.0f, 2.0f, 3.0f}});
                std::vector<Ttl> l(n, Ttl{30});
                ed.write<Velocity>(first, v).write<Ttl>(first, l);
                b.write<Velocity>(first, v);
                b.write<Ttl>(first, l);
                rows += n;
                break;
            }
            }
        }
        records += ed.size();
        a.apply(ed);
        EXPECT(ed.size() == 0);
        if (frame % 8 == 7) EXPECT(same_world(a, b));
    }
    EXPECT(same_world(a, b));
    EXPECT(records > 500);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(16, 8);
            app.rollback_component_with_copy<Velocity>();
            App::Edits ed(app);
            ed.spawn(1);
            app.apply(ed);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    edits_match_the_single_calls();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "host edits test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
