// App replays through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): box_game with its FrameCount rollback
// resource, checksummed on the host as box_game_p2p.rs registers it.
//   - A P2P App plays a match.  An App restored from its checkpoint of frame 0 replays the match's input log, in two
//     calls, at the desync-detection interval: its checksums equal the P2P App's confirmed checksums at every interval
//     frame, and its world and FrameCount end equal.  The engine's replay alone gives other checksums.
//   - replay_keyframes writes the P2P App's checkpoint(f) byte for byte; restoring a keyframe and replaying the rest of
//     the log ends in the same checksums and state.
//   - A spectator App that advances the same frames through handle_requests ends like a replay of its inputs.
//   - Refusals change nothing: host-side component tables, resources out of step with the world, a log the engine
//     refuses.  A non-finite checksum still commits the stepped resources.
// Exit code 0 = passed.  `--stepwise` creates every engine with BGR_CFG_FORCE_STEPWISE.  Needs an H100
// (tests/test_cpp_app_replay.py).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
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

using Checksums = std::vector<std::pair<ggrs::Frame, unsigned __int128>>;
static const uint8_t kSeq[8] = {1, 8, 5, 0, 2, 10, 4, 9};
static const int kFrames = 120, kInterval = 10, kKeyframes = 16, kLag = 8;
static uint32_t g_flags = 0;

// box_game (examples/box_game/box_game_p2p.rs); handle 0's input follows *tick
static void box_game(App& app, int* tick) {
    app.add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
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
        .checksum_component<Transform>(hash_bytes(0, 12, true));
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_BOX_MOVE, {1, 0}, {}});
    app.add_systems(GgrsSchedule{}, ResourceSystem{[](App& a) { a.resource<FrameCount>().frame += 1; }});  // increase_frame_system
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

// the rollback frame, FrameCount and the bytes of both players' components
static std::vector<uint8_t> state_of(App& app) {
    std::vector<uint8_t> s(8);
    const int32_t f = app.rollback_frame_count();
    const uint32_t fc = app.resource<FrameCount>().frame;
    std::memcpy(s.data(), &f, 4);
    std::memcpy(s.data() + 4, &fc, 4);
    const auto t = app.read<Transform>(0, 2);
    const auto v = app.read<Velocity>(0, 2);
    s.insert(s.end(), reinterpret_cast<const uint8_t*>(t.data()), reinterpret_cast<const uint8_t*>(t.data() + 2));
    s.insert(s.end(), reinterpret_cast<const uint8_t*>(v.data()), reinterpret_cast<const uint8_t*>(v.data() + 2));
    return s;
}

// an App (no session) restored from an App checkpoint
struct Restored {
    int tick = 0;
    App app{4, 9, 0, g_flags};
    explicit Restored(const std::vector<uint8_t>& blob) {
        box_game(app, &tick);
        spawn_players(app);
        app.restore_checkpoint(blob);
    }
};

static void p2p_match_replays() {
    std::printf("p2p_match_replays\n");
    std::vector<int> depths(kFrames);
    uint32_t x = 12345;
    for (int& d : depths) { x = x * 1664525u + 1013904223u; d = (x >> 16) % 2 ? int((x >> 20) % 9) : 0; }
    int tick = 0;
    App a(4, 9, 0, g_flags);
    box_game(a, &tick);
    a.insert_resource(Session::P2P(ggrs::P2PTraceSession(2, 8, depths, kLag, 2)));
    spawn_players(a);
    std::map<ggrs::Frame, unsigned __int128> latest;  // each interval frame's latest checksum: re-saves replace predictions
    std::map<ggrs::Frame, std::vector<uint8_t>> saved;
    std::vector<uint8_t> first;
    for (int t = 0; t < kFrames; ++t) {
        a.step();
        for (const auto& cs : a.last_checksums())
            if (cs.frame % kInterval == 0) latest[cs.frame] = (static_cast<unsigned __int128>(cs.hi) << 64) | cs.lo;
        if (t == 0) first = a.checkpoint(0);
        if (t % kKeyframes == 0) saved[t] = a.checkpoint(t);  // the frame this tick saved last
    }
    // the input log: handle 0's input of tick t lands on frame t + input_delay; handle 1 is remote and never sent one
    std::vector<uint8_t> log(2 * kFrames, 0);
    for (int f = 2; f < kFrames; ++f) log[2 * f] = kSeq[(f - 2) % 8];
    std::map<ggrs::Frame, unsigned __int128> reports;
    for (const auto& kv : latest)
        if (kv.first <= kFrames - kLag) reports.insert(kv);
    EXPECT(reports.size() >= 10);

    Restored b(first);
    const std::vector<uint8_t> head(log.begin(), log.begin() + 2 * 47), tail(log.begin() + 2 * 47, log.end());
    Checksums cs = b.app.replay(head, 2, kInterval), rest = b.app.replay(tail, 2, kInterval);
    cs.insert(cs.end(), rest.begin(), rest.end());
    std::map<ggrs::Frame, unsigned __int128> got(cs.begin(), cs.end());
    bool equal = true;
    for (const auto& kv : reports) equal = equal && got.count(kv.first) && got[kv.first] == kv.second;
    EXPECT(equal);
    EXPECT(b.app.resource<FrameCount>().frame == uint32_t(kFrames) && state_of(b.app) == state_of(a));

    // the engine's replay alone leaves out FrameCount's part
    Restored c(first);
    struct bgr_replay r;
    std::memset(&r, 0, sizeof r);
    r.n_frames = kFrames; r.n_players = 2; r.checksum_interval = kInterval; r.inputs = log.data();
    std::vector<bgr_checksum> raw(kFrames / kInterval);
    uint32_t n = 0;
    check(bgr_replay(c.app.engine(), &r, raw.data(), uint32_t(raw.size()), &n));
    bool all_differ = n == raw.size();
    for (uint32_t i = 0; i < n; ++i)
        if (reports.count(raw[i].frame))
            all_differ = all_differ && ((static_cast<unsigned __int128>(raw[i].hi) << 64) | raw[i].lo) != reports[raw[i].frame];
    EXPECT(all_differ);

    // keyframes are the P2P App's checkpoints; seeking one and replaying the rest ends the same
    Restored d(first);
    std::vector<std::pair<ggrs::Frame, std::vector<uint8_t>>> kfs;
    EXPECT(d.app.replay_keyframes(log, 2, kInterval, kKeyframes, &kfs) == cs);
    EXPECT(kfs.size() == saved.size());
    bool same = true;
    for (const auto& kf : kfs) same = same && saved.count(kf.first) && saved[kf.first] == kf.second;
    EXPECT(same);
    EXPECT(state_of(d.app) == state_of(b.app));
    const auto& mid = kfs[kfs.size() / 2];
    Restored e(mid.second);
    const std::vector<uint8_t> after(log.begin() + 2 * mid.first, log.end());
    Checksums suffix;
    for (const auto& c2 : cs)
        if (c2.first >= mid.first) suffix.push_back(c2);
    EXPECT(e.app.replay(after, 2, kInterval) == suffix);
    EXPECT(state_of(e.app) == state_of(b.app));
}

// a spectator App advances frames through handle_requests; a replay of the same inputs ends the same
static void spectator_twin() {
    std::printf("spectator_twin\n");
    int tick_s = 0, tick_r = 0;
    App s(4, 9, 0, g_flags), r(4, 9, 0, g_flags);
    box_game(s, &tick_s);
    box_game(r, &tick_r);
    std::vector<int> script;
    int frames = 0;
    for (int i = 0; frames < 90; ++i) { script.push_back(1 + i % 4); frames += script.back(); }
    s.insert_resource(Session::Spectator(ggrs::SpectatorTraceSession(2, script)));
    spawn_players(s);
    spawn_players(r);
    for (size_t i = 0; i < script.size(); ++i) s.step();
    std::vector<uint8_t> log;
    for (int f = 0; f < frames; ++f)
        for (int p = 0; p < 2; ++p) log.push_back(uint8_t((f + p) & 3));  // the spectator session's inputs
    EXPECT(r.replay(std::vector<uint8_t>(log.begin(), log.begin() + 2 * 33), 2, 0).empty());
    EXPECT(r.replay(std::vector<uint8_t>(log.begin() + 2 * 33, log.end()), 2, 0).empty());
    EXPECT(s.rollback_frame_count() == frames && state_of(r) == state_of(s));
}

static void refusals_change_nothing() {
    std::printf("refusals_change_nothing\n");
    int tick = 0;
    App hosted(4, 9, 0, g_flags);
    box_game(hosted, &tick);
    hosted.rollback_component_with_clone<Sprite>();
    spawn_players(hosted);
    const std::vector<uint8_t> log(2 * 30, 5);
    std::vector<std::pair<ggrs::Frame, std::vector<uint8_t>>> kfs;
    std::vector<bgr_trace_sample> samples;
    std::vector<uint8_t> records;
    const std::vector<bgr_feed_field> fields{{1, 0, 12}};
    EXPECT(status_of([&] { hosted.replay(log, 2, 1); }) == BGR_ERR_UNSUPPORTED);
    EXPECT(status_of([&] { hosted.replay_keyframes(log, 2, 1, 4, &kfs); }) == BGR_ERR_UNSUPPORTED);
    EXPECT(status_of([&] { hosted.replay_trace(log, 2, 1, 4, fields, 0, 2, &samples, &records); }) == BGR_ERR_UNSUPPORTED);
    EXPECT(hosted.rollback_frame_count() == 0 && hosted.resource<FrameCount>().frame == 0);

    int t2 = 0;
    App app(4, 9, 0, g_flags);
    box_game(app, &t2);
    spawn_players(app);
    const auto before = state_of(app);
    check(bgr_set_rollback_frame_count(app.engine(), 3));  // the resources out of step with the world
    EXPECT(status_of([&] { app.replay(log, 2, 1); }) == BGR_ERR_STATE);
    check(bgr_set_rollback_frame_count(app.engine(), 0));
    EXPECT(state_of(app) == before);
    const std::vector<uint8_t> nine(9 * 4, 0);  // n_players > BGR_MAX_PLAYERS: refused by the engine after the stepping
    EXPECT(status_of([&] { app.replay(nine, 9, 1); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(status_of([&] { app.replay_keyframes(nine, 9, 1, 2, &kfs); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(status_of([&] { app.replay_trace(nine, 9, 1, 2, fields, 0, 2, &samples, &records); }) == BGR_ERR_INVALID_ARGUMENT);
    EXPECT(state_of(app) == before);

    // a non-finite translation at a checksum frame: the log ran, the resources are committed
    auto t = app.read<Transform>(0, 2);
    t[1].translation[0] = std::numeric_limits<float>::quiet_NaN();
    app.write<Transform>(0, t);
    EXPECT(status_of([&] { app.replay(log, 2, 1); }) == BGR_ERR_NON_FINITE);
    EXPECT(app.rollback_frame_count() == 30 && app.resource<FrameCount>().frame == 30);
    EXPECT(status_of([&] { app.replay(log, 2, 0); }) == BGR_OK);  // in step: no checksum frames, no refusal
    EXPECT(app.resource<FrameCount>().frame == 60);
}

int main(int argc, char** argv) {
    for (int i = 1; i < argc; ++i)
        if (std::strcmp(argv[i], "--stepwise") == 0) g_flags = BGR_CFG_FORCE_STEPWISE;
    p2p_match_replays();
    spectator_twin();
    refusals_change_nothing();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "app replay test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
