// The keyframes of a replay (csrc/replay_keyframes.hpp plan_replay_keyframes, which bgr_replay_keyframes uses for the
// placement, the byte bound and every blob header's frame, rows, Time<GgrsTime> and ParticleRng) against the request
// stream restated frame by frame: at each frame f with f % K == 0 the state a SaveGameState{f} would snapshot, then the
// frame's AdvanceFrame (GgrsTimePlugin::update moves Time to (f + 1) * 1e9 / fps; a spawn frame adds `rate` rows and
// draws two random_range(-200, 200) per row, particles.rs:262-268).  The byte bound is restated from the blob format of
// include/bevy_ggrs_b200.h: header, u64 offsets[n_blocks + 1], per block the kind bytes and every vector RAW.
// Random logs at 60, 7 and 144 fps, from frame 0 and from a restored frame whose Time<GgrsTime> is not the frame's
// runtime (a checkpoint of another rate's engine or a bgr_set_rollback_frame_count), with and without spawns, at
// intervals 1, 7, 60 and past the log.  Host only: exit code 0 = passed.
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/replay_keyframes.hpp"

using namespace bgr;

static int g_failed = 0;

static size_t restated_bound(uint32_t rows, uint32_t words) {
    const size_t nb = (rows + 511) / 512;
    const size_t kinds = ((words + 1) + 3) / 4 * 4;                 // one kind byte per vector, padded to 4
    const size_t block = kinds + size_t(words) * 512 * 4 + 128 * 4; // every word plane and the mask plane RAW
    const size_t blob = 104 + 8 * (nb + 1) + nb * block;
    return (blob + 7) / 8 * 8;
}

int main() {
    static_assert(sizeof(bgr_checkpoint_header) == 104, "the blob header");
    std::mt19937_64 gen(0x4B45594652414D45ULL);
    int cases = 0;
    for (uint32_t fps : {60u, 7u, 144u})
        for (int restored = 0; restored < 2; ++restored)
            for (int spawn = 0; spawn < 2; ++spawn)
                for (uint32_t k : {1u, 7u, 60u, 5000u})
                    for (int rep = 0; rep < 4; ++rep) {
                        const uint32_t n = 1 + uint32_t(gen() % 700), words = 1 + uint32_t(gen() % 30);
                        const int32_t f0 = restored ? int32_t(gen() % 100000) : 0;
                        // a restore sets Time<GgrsTime> to the checkpoint's, which need not be f0's runtime at this rate
                        const uint64_t elapsed0 = restored ? uint64_t(f0) * 1000000000ULL / 61u : 0u;
                        const uint32_t rows0 = uint32_t(gen() % 5000), rate = spawn ? 1 + uint32_t(gen() % 300) : 0u;
                        ParticleRng rng0;
                        rng0.seed_from_u64(gen());
                        std::vector<uint8_t> pressed(n);
                        for (auto& p : pressed) p = spawn && gen() % 5 == 0;
                        std::vector<uint32_t> prefix;
                        if (spawn) {
                            prefix.assign(n + 1, 0);
                            for (uint32_t j = 0; j < n; ++j) prefix[j + 1] = prefix[j] + pressed[j];
                        }
                        const ReplayClock c = replay_clock(f0, fps, elapsed0, 2, 0, 0, spawn, rate, rows0);
                        const std::vector<KeyframePlan> got = plan_replay_keyframes(c, n, k, elapsed0, prefix, rng0, words);
                        // the stream, frame by frame
                        std::vector<KeyframePlan> want;
                        uint64_t elapsed = elapsed0;
                        uint32_t rows = rows0;
                        ParticleRng rng = rng0;
                        for (uint32_t j = 0; j < n; ++j) {
                            const int64_t f = int64_t(f0) + j;
                            if (f % k == 0) want.push_back(KeyframePlan{j, rows, elapsed, rng, restated_bound(rows, words)});
                            elapsed = uint64_t(f + 1) * 1000000000ULL / fps;
                            if (pressed[j]) {
                                rows += rate;
                                for (uint32_t i = 0; i < 2 * rate; ++i) rng.random_range(-200.0f, 200.0f);
                            }
                        }
                        ++cases;
                        bool ok = got.size() == want.size();
                        for (size_t q = 0; ok && q < got.size(); ++q)
                            ok = got[q].j == want[q].j && got[q].rows == want[q].rows && got[q].elapsed_ns == want[q].elapsed_ns &&
                                 std::memcmp(got[q].rng.s, want[q].rng.s, sizeof want[q].rng.s) == 0 &&
                                 got[q].max_bytes == want[q].max_bytes;
                        if (!ok && g_failed++ < 10)
                            std::printf("mismatch: fps %u f0 %d n %u k %u spawn %d rate %u: %zu keyframes, want %zu\n", fps, f0, n, k,
                                        spawn, rate, got.size(), want.size());
                    }
    if (g_failed) {
        std::printf("%d of %d cases failed\n", g_failed, cases);
        return 1;
    }
    std::printf("replay keyframe plan test passed (%d cases)\n", cases);
    return 0;
}
