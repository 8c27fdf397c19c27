// Replay keyframes (bgr_replay_keyframes): which frames of a replay are keyframes and what each blob's header says about
// its frame, planned on the host before anything runs.  Host only; tests/cpp/test_replay_keyframes.cpp holds it to a
// frame-by-frame restatement of the request stream.
#pragma once
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "checkpoint.cuh"      // ckpt_max_block_words
#include "generic_program.cuh" // ReplayClock, replay_first_point
#include "particle_rng.hpp"

namespace bgr {

// One keyframe: frame f0 + j, its RollbackOrdered::len(), Time<GgrsTime> and ParticleRng there, and the most bytes its
// blob can take in the output (every vector RAW) padded to the next blob's 8-byte boundary
struct KeyframePlan {
    uint32_t j, rows;
    uint64_t elapsed_ns;
    ParticleRng rng;
    size_t max_bytes;
};

// The keyframes of a replay of n frames from clock `c` at interval k (every frame f0 + j with (f0 + j) % k == 0), for
// an engine with `words` word planes whose Time<GgrsTime> is elapsed0 and ParticleRng rng0 before frame 0.  `prefix`
// holds the spawn frames before each frame ([n + 1]; empty without spawn_particles); each spawn frame draws c.rate
// particles of two random_range(-200, 200) (particles.rs:262-268), which is where ParticleRng moves.
inline std::vector<KeyframePlan> plan_replay_keyframes(const ReplayClock& c, uint32_t n, uint32_t k, uint64_t elapsed0,
                                                       const std::vector<uint32_t>& prefix, ParticleRng rng0, uint32_t words) {
    std::vector<KeyframePlan> out;
    const unsigned long long first = replay_first_point(c.f0, k, 0, n);
    if (first == ~0ULL) return out;
    ParticleRng rng = rng0;
    uint32_t drawn = 0;  // spawn frames whose draws `rng` has made
    for (unsigned long long j = first; j < n; j += k) {
        const uint32_t spawned = prefix.empty() ? 0u : prefix[j];
        for (; drawn < spawned; ++drawn)
            for (uint32_t i = 0; i < c.rate; ++i) {
                rng.random_range(-200.0f, 200.0f);
                rng.random_range(-200.0f, 200.0f);
            }
        KeyframePlan p;
        p.j = uint32_t(j);
        p.rows = c.rows0 + c.rate * spawned;
        p.elapsed_ns = j == 0 ? elapsed0 : uint64_t(int64_t(c.f0) + int64_t(j)) * 1000000000ULL / c.fps;
        p.rng = rng;
        const size_t nb = (p.rows + kTileRows - 1) / kTileRows;
        const size_t blob = sizeof(bgr_checkpoint_header) + sizeof(uint64_t) * (nb + 1) + nb * ckpt_max_block_words(words) * 4u;
        p.max_bytes = (blob + 7u) & ~size_t(7);
        out.push_back(p);
    }
    return out;
}

}  // namespace bgr
