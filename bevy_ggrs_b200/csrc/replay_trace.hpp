// Replay traces (bgr_replay_trace): the refusals of a trace, which frames of a replay are samples and each one's row
// count, where each record lands, how far a launch runs within the staging budget, and the field map of
// k_generic_jit_replay_trace, all on the host before anything runs.  Host only; tests/cpp/test_replay_trace.cpp holds
// it to a frame-by-frame scan of random logs.
#pragma once
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "feed_check.hpp"       // feed_fields, FeedParams
#include "generic_program.cuh"  // ReplayClock, replay_first_point, TraceMap

namespace bgr {

// The refusals of a trace besides the replay's and its field list's (feed_fields).  `row_limit`: the rows the engine can
// ever hold, max_entities (its ceiling when growable).  BGR_OK, or the status with *err = why.
inline int trace_check(const bgr_trace& t, uint64_t row_limit, std::string* err) {
    if (t.interval == 0) { *err = "bgr_trace.interval must be >= 1"; return BGR_ERR_INVALID_ARGUMENT; }
    if (t.reserved) { *err = "bgr_trace.reserved must be 0"; return BGR_ERR_INVALID_ARGUMENT; }
    if (t.n_rows == 0) { *err = "bgr_trace.n_rows must be >= 1"; return BGR_ERR_INVALID_ARGUMENT; }
    if (uint64_t(t.first_row) + t.n_rows > row_limit) {
        *err = "traced rows [" + std::to_string(t.first_row) + ", " + std::to_string(uint64_t(t.first_row) + t.n_rows) +
               ") exceed the engine's " + std::to_string(row_limit) + " rows";
        return BGR_ERR_INVALID_ARGUMENT;
    }
    return BGR_OK;
}

// The samples of a replay of n frames from clock `c` at interval T: every frame f0 + j, j < n, with (f0 + j) % T == 0,
// and RollbackOrdered::len() there (`prefix`: the spawn frames before each frame, [n + 1]; empty without spawn_particles)
inline std::vector<bgr_trace_sample> plan_trace_samples(const ReplayClock& c, uint32_t n, uint32_t T, const std::vector<uint32_t>& prefix) {
    std::vector<bgr_trace_sample> out;
    for (unsigned long long j = replay_first_point(c.f0, T, 0, n); j < n; j += T)
        out.push_back(bgr_trace_sample{int32_t(int64_t(c.f0) + int64_t(j)), c.rows0 + c.rate * (prefix.empty() ? 0u : prefix[j])});
    return out;
}

// bytes of one record: u32 row, u32 state, the field words
inline uint32_t trace_record_bytes(const FeedParams& p) { return 4u * p.record_words; }
// where sample s, traced row i lands in dst
inline size_t trace_record_offset(uint64_t s, uint32_t i, uint32_t n_rows, uint32_t record_bytes) {
    return size_t((s * n_rows + i) * record_bytes);
}

// The end of a launch that starts at frame a of a world whose log (or the checksum budget) ends the launch at b: the
// launch holds at most budget / stride samples of `stride` bytes, and at least one
inline uint32_t trace_launch_end(int32_t f0, uint32_t T, uint32_t a, uint32_t b, uint64_t budget, uint64_t stride) {
    const unsigned long long f = replay_first_point(f0, T, a, b);
    const uint64_t m = std::max<uint64_t>(1, budget / std::max<uint64_t>(1, stride));
    return (f != ~0ULL && f + m * T < b) ? uint32_t(f + m * T) : b;
}

// The field map of k_generic_jit_replay_trace for a field list mapped by feed_fields onto rows of at most kTraceMaxWords
// words: record slots grouped by word plane
inline TraceMap trace_map(const FeedParams& p) {
    TraceMap m{};
    m.n_fields = p.n_fields;
    m.record_words = p.record_words;
    for (uint32_t k = 0; k < p.n_fields; ++k) m.field_absent[k] = uint8_t(p.fields[k].absent);
    uint32_t at = 0;
    for (uint32_t j = 0; j < kTraceMaxWords; ++j) {
        m.word_first[j] = uint8_t(at);
        for (uint32_t k = 0; k < p.n_fields; ++k) {
            const FeedField& f = p.fields[k];
            if (j >= f.plane && j < f.plane + f.words) {
                m.word_absent[j] = uint8_t(f.absent);
                m.slot[at++] = uint8_t(f.rep_plane + (j - f.plane));
            }
        }
    }
    m.word_first[kTraceMaxWords] = uint8_t(at);
    return m;
}

}  // namespace bgr
