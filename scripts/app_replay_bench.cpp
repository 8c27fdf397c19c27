// Host wall time of App::replay (the engine's replay plus the FrameCount resource stepped on the host) against the
// engine's bgr_replay alone, on box_game worlds of the C++ host mirror.  Built and run by scripts/app_replay_bench.py,
// which passes <frames> <checksum interval> <reps>; prints one JSON line.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../bevy_ggrs_b200/host/bevy_ggrs.hpp"

using namespace bevy_ggrs;

struct Transform { float translation[3]; float rotation[4]; float scale[3]; };
struct Velocity { float v[3]; };
struct FrameCount { uint32_t frame; };

static void box_game(App& app) {
    app.rollback_resource_with_copy<FrameCount>(FrameCount{0})
        .rollback_component_with_copy<Velocity>()
        .rollback_component_with_clone<Transform>()
        .checksum_resource_with_hash<FrameCount>()
        .checksum_component<Transform>(hash_bytes(0, 12, true));
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_BOX_MOVE, {1, 0}, {}});
    app.add_systems(GgrsSchedule{}, ResourceSystem{[](App& a) { a.resource<FrameCount>().frame += 1; }});
    std::vector<Transform> t0(2);
    for (int h = 0; h < 2; ++h) t0[h] = Transform{{1.25f * std::cos(3.14159265f * h), 0.1f, 1.25f * std::sin(3.14159265f * h)}, {0, 0, 0, 1}, {1, 1, 1}};
    app.write<Transform>(app.spawn(2), t0);
}

static double median(std::vector<double> v) {
    std::sort(v.begin(), v.end());
    return v[v.size() / 2];
}

int main(int argc, char** argv) {
    const uint32_t frames = argc > 1 ? uint32_t(std::atoi(argv[1])) : 3600u, k = argc > 2 ? uint32_t(std::atoi(argv[2])) : 10u;
    const int reps = argc > 3 ? std::atoi(argv[3]) : 5;
    App app(4, 4), eng(4, 4);
    box_game(app);
    box_game(eng);
    std::vector<uint8_t> log(2 * size_t(frames));
    uint32_t x = 7;
    std::vector<double> t_app, t_eng;
    std::vector<bgr_checksum> cs(frames / k + 2);
    for (int rep = 0; rep <= reps; ++rep) {
        for (auto& b : log) { x = x * 1664525u + 1013904223u; b = uint8_t(x >> 28); }
        auto t0 = std::chrono::steady_clock::now();
        const auto out = app.replay(log, 2, k);
        auto t1 = std::chrono::steady_clock::now();
        struct bgr_replay r;
        std::memset(&r, 0, sizeof r);
        r.n_frames = frames; r.n_players = 2; r.checksum_interval = k; r.inputs = log.data();
        uint32_t n = 0;
        check(bgr_replay(eng.engine(), &r, cs.data(), uint32_t(cs.size()), &n));
        auto t2 = std::chrono::steady_clock::now();
        if (n != out.size() || out.empty()) { std::fprintf(stderr, "checksum counts differ\n"); return 1; }
        if (rep) {
            t_app.push_back(std::chrono::duration<double, std::milli>(t1 - t0).count());
            t_eng.push_back(std::chrono::duration<double, std::milli>(t2 - t1).count());
        }
    }
    std::printf("{\"workload\": \"cpp_box_game_1\", \"frames\": %u, \"interval\": %u, \"app_replay_ms\": %.3f, "
                "\"engine_replay_ms\": %.3f}\n", frames, k, median(t_app), median(t_eng));
    return 0;
}
