// The per-frame op of a replay (csrc/generic_program.cuh replay_op, which k_generic_jit_replay runs on the device) against
// the ADVANCE ops compile_requests builds for the same log, request by request: GgrsTime's step from the frame count
// (time.rs:63-76), friction from the C library's powf, the call counter of BGR_SYS_U32_STORE_CALL_COUNT, the inputs,
// and spawn_particles' first row, count and spawn-value offset.  The clock is built by replay_clock, the function the
// engine's replay_plan calls.  compile_requests itself lives inside the engine, which needs a GPU to exist, so its
// ADVANCE is restated here step by step as it applies to the HostState (advance() below); the GPU tests hold the
// engine's own request path to the replay on every registration.  The checksum frames (replay_first_point /
// replay_points_in, which place the SAVE ops of both the kernel and the chunked fallback) are checked against a scan
// of every frame, for segments starting anywhere in the log.  Random logs at 60, 7, 144 and 1000 fps, with and
// without a first step after bgr_set_rollback_frame_count / a checkpoint restore (Time<GgrsTime> not at the frame's
// runtime), counter systems and spawn frames.  Host only: exit code 0 = passed.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/generic_program.cuh"

using namespace bgr;

static int g_failed = 0;

static float secs_f32(uint64_t ns) {  // core::time::Duration::as_secs_f32
    return float(ns / 1000000000ULL) + float(uint32_t(ns % 1000000000ULL)) / 1000000000.0f;
}
static uint32_t bits(float f) { uint32_t b; std::memcpy(&b, &f, 4); return b; }

struct Host {  // the part of HostState an ADVANCE reads and writes
    int32_t frame;
    uint64_t elapsed;
    uint32_t call, rows, spawned;
};

// compile_requests' ADVANCE, with the vector's spawn-value offset running over the whole log
static Op advance(Host& s, uint32_t fps, uint32_t n_counter, bool spawn_sys, uint32_t rate, const uint8_t* in, uint32_t np) {
    Op op;
    std::memset(&op, 0, sizeof op);
    s.frame += 1;
    const uint64_t runtime = uint64_t(int64_t(s.frame)) * 1000000000ULL / fps;
    const uint64_t delta = runtime - s.elapsed;
    s.elapsed = runtime;
    op.kind = OP_ADVANCE;
    op.dt_bits = bits(secs_f32(delta));
    op.fr_bits = bits(powf(0.0018f, secs_f32(delta)));
    op.n_rows = s.rows;
    op.call_count = s.call;
    s.call += n_counter;
    for (uint32_t k = 0; k < 8 && k < np; ++k) op.inputs[k] = in[k];
    op.flags |= (np & 0xFu) << 8;
    bool pressed = false;
    for (uint32_t k = 0; k < np; ++k) pressed = pressed || (in[k] & 0x10u);
    if (spawn_sys && pressed) {
        op.flags |= OPF_SPAWN;
        op.image_off256 = s.rows;
        op.save_index = rate;
        op.call_count = s.spawned;
        s.spawned += rate;
        s.rows += rate;
    }
    return op;
}

static void run(uint32_t fps, int32_t f0, uint64_t elapsed0, uint32_t np, uint32_t n_counter, bool spawn_sys, uint32_t rate,
                uint32_t n, uint32_t seed) {
    std::mt19937 rng(seed);
    std::vector<uint8_t> log(size_t(n) * np);
    for (auto& v : log) v = uint8_t(rng() & 0x1F);  // direction bits and, now and then, INPUT_SPAWN
    Host s{f0, elapsed0, 1000u + seed, 300u, 0u};
    const ReplayClock c = replay_clock(f0, fps, elapsed0, np, s.call, n_counter, spawn_sys, rate, s.rows);
    uint32_t prefix = 0;
    for (uint32_t j = 0; j < n; ++j) {
        const uint8_t* in = log.data() + size_t(j) * np;
        const Op want = advance(s, fps, n_counter, spawn_sys, rate, in, np);
        const Op got = replay_op(c, j, in, prefix);
        if (std::memcmp(&want, &got, sizeof want) != 0) {
            std::printf("  FAILED fps %u f0 %d players %u counters %u spawn %d: frame %u differs (dt %08x/%08x fr %08x/%08x rows %u/%u "
                        "call %u/%u flags %x/%x)\n", fps, f0, np, n_counter, int(spawn_sys), j, want.dt_bits, got.dt_bits,
                        want.fr_bits, got.fr_bits, want.n_rows, got.n_rows, want.call_count, got.call_count, want.flags, got.flags);
            ++g_failed;
            return;
        }
        prefix += (got.flags & OPF_SPAWN) ? 1u : 0u;
    }
}

// the checksum frames of [a, b) against a scan of every frame
static void points(int32_t f0, uint32_t k, uint32_t n) {
    for (uint32_t a = 0; a <= n; a += 1 + a / 3)
        for (uint32_t b = a; b <= n; b += 1 + b / 5) {
            uint64_t first = ~0ULL;
            uint32_t count = 0;
            for (uint32_t j = a; j < b; ++j)
                if (k && (int64_t(f0) + j) % k == 0) { if (first == ~0ULL) first = j; ++count; }
            if (replay_first_point(f0, k, a, b) != first || replay_points_in(f0, k, a, b) != count) {
                std::printf("  FAILED checksum frames f0 %d k %u [%u, %u): first %llu/%llu count %u/%u\n", f0, k, a, b,
                            (unsigned long long)first, (unsigned long long)replay_first_point(f0, k, a, b), count,
                            replay_points_in(f0, k, a, b));
                ++g_failed;
                return;
            }
        }
}

int main() {
    for (int32_t f0 : {0, 1, 7, 10, 123456, 2147483000})
        for (uint32_t k : {0u, 1u, 2u, 7u, 10u, 1000u, 4294967295u}) points(f0, k, 400);
    uint32_t seed = 1;
    for (uint32_t fps : {60u, 7u, 144u, 1000u})
        for (int32_t f0 : {0, 7, 123456})
            for (int restored = 0; restored < 2; ++restored) {
                // restored: Time<GgrsTime> is not the frame's runtime (set_rollback_frame_count leaves it, a checkpoint
                // restore takes it from the blob)
                const uint64_t el = restored ? uint64_t(int64_t(f0)) * 1000000000ULL / fps / 3 : uint64_t(int64_t(f0)) * 1000000000ULL / fps;
                for (uint32_t np : {0u, 1u, 2u, 8u})
                    for (uint32_t counters : {0u, 2u})
                        for (int spawn = 0; spawn < 2; ++spawn) run(fps, f0, el, np, counters, spawn, spawn ? 25u : 0u, 3000, seed++);
            }
    if (g_failed) { std::printf("replay op test FAILED (%d)\n", g_failed); return 1; }
    std::printf("replay op test passed\n");
    return 0;
}
