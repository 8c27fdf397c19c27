// The host plan of a replay trace (csrc/replay_trace.hpp, which bgr_replay_trace and bgr_batch_replay_trace run before
// anything executes) against a frame-by-frame scan of random logs: which frames are samples (from f0 != 0, at intervals
// 1, 7, 60 and past the log) and RollbackOrdered::len() at each under spawns; how the trace budget splits a replay into
// launches (every sample in exactly one launch, at most budget / stride of them and at least one per launch); where each
// record lands; the field map of k_generic_jit_replay_trace; and every refusal of a trace's row range and field list,
// with its status.  Host only: exit code 0 = passed.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/replay_trace.hpp"

using namespace bgr;

static int g_failed = 0, g_cases = 0;
#define EXPECT(cond, what)                                                                                   \
    do {                                                                                                     \
        ++g_cases;                                                                                           \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #cond, what); ++g_failed; } \
    } while (0)

// a registration: Transform (10 words, plane 0), Velocity (3 words, plane 10), Score (1 word, optional, absent bit 2)
static const FeedColumn kCols[] = {{0, 10, 0}, {10, 3, 0}, {13, 1, 2}};
static int fields_of(const std::vector<bgr_feed_field>& f, FeedParams& p, std::string* err) {
    return feed_fields(3u, [](uint32_t c) { return kCols[c]; }, 14u, f.data(), uint32_t(f.size()), p, err);
}

static void test_samples_and_launches(std::mt19937_64& gen) {
    for (uint32_t T : {1u, 7u, 60u, 5000u})
        for (int spawn = 0; spawn < 2; ++spawn)
            for (int rep = 0; rep < 6; ++rep) {
                const uint32_t n = 1 + uint32_t(gen() % 900);
                const int32_t f0 = rep % 3 == 0 ? 0 : int32_t(gen() % 100000);
                const uint32_t rows0 = uint32_t(gen() % 3000), rate = spawn ? 1 + uint32_t(gen() % 200) : 0u;
                std::vector<uint8_t> pressed(n);
                for (auto& p : pressed) p = spawn && gen() % 4 == 0;
                std::vector<uint32_t> prefix;
                if (spawn) {
                    prefix.assign(n + 1, 0);
                    for (uint32_t j = 0; j < n; ++j) prefix[j + 1] = prefix[j] + pressed[j];
                }
                const ReplayClock c = replay_clock(f0, 60, 0, 2, 0, 0, spawn, rate, rows0);
                const std::vector<bgr_trace_sample> got = plan_trace_samples(c, n, T, prefix);
                // the scan: at each frame, a sample before the frame's AdvanceFrame, which may spawn `rate` rows
                std::vector<bgr_trace_sample> want;
                std::vector<uint32_t> want_j;
                uint32_t rows = rows0;
                for (uint32_t j = 0; j < n; ++j) {
                    if ((int64_t(f0) + j) % T == 0) { want.push_back({int32_t(f0 + int32_t(j)), rows}); want_j.push_back(j); }
                    if (pressed[j]) rows += rate;
                }
                bool ok = got.size() == want.size();
                for (size_t q = 0; ok && q < got.size(); ++q) ok = got[q].frame == want[q].frame && got[q].rows == want[q].rows;
                EXPECT(ok, ("samples: f0 " + std::to_string(f0) + " n " + std::to_string(n) + " T " + std::to_string(T)).c_str());
                // launches under a budget of 1..5 samples of `stride` bytes (and a budget below one sample)
                const uint64_t stride = 8u + (gen() % 64) * 4u;
                for (uint64_t budget : {stride / 2, stride, 3 * stride + 1, 5 * stride}) {
                    const uint64_t per = std::max<uint64_t>(1, budget / stride);
                    std::vector<uint32_t> seen;
                    uint32_t a = 0, launches = 0;
                    bool ok2 = true;
                    while (a < n && launches < 100000) {
                        const uint32_t b = trace_launch_end(f0, T, a, n, budget, stride);
                        ok2 = ok2 && b > a && b <= n;
                        uint32_t in = 0;
                        for (uint32_t j : want_j) if (j >= a && j < b) { seen.push_back(j); ++in; }
                        ok2 = ok2 && in <= per && in == replay_points_in(f0, T, a, b);
                        // the launch ends right after its last sample only when the budget is full
                        ok2 = ok2 && (b == n || in == per);
                        a = b;
                        ++launches;
                    }
                    EXPECT(ok2 && seen == want_j, ("launches: T " + std::to_string(T) + " budget " + std::to_string(budget)).c_str());
                }
            }
}

static void test_offsets_and_map() {
    std::string err;
    FeedParams p{};
    // Transform's translation, Score, Velocity, and Transform words 1..2 again: plane 1 and 2 go to two record words
    const std::vector<bgr_feed_field> f = {{0, 0, 12}, {2, 0, 4}, {1, 0, 12}, {0, 4, 8}};
    EXPECT(fields_of(f, p, &err) == BGR_OK, err.c_str());
    EXPECT(p.record_words == 2u + 3u + 1u + 3u + 2u && trace_record_bytes(p) == 44u, "record bytes");
    EXPECT(p.keep == (1u | 2u), "mask bits of the state");
    EXPECT(trace_record_offset(0, 0, 100, 44) == 0 && trace_record_offset(0, 99, 100, 44) == 99u * 44u &&
               trace_record_offset(3, 7, 100, 44) == (3u * 100u + 7u) * 44u && trace_record_offset(70000, 99999, 100000, 44) == size_t(7000099999ull) * 44u,
           "record offsets");
    const TraceMap m = trace_map(p);
    EXPECT(m.n_fields == 4 && m.record_words == 11, "map sizes");
    EXPECT(m.field_absent[0] == 0 && m.field_absent[1] == 2 && m.field_absent[2] == 0, "field absent bits");
    // plane j -> record words: (plane, slots)
    const std::vector<std::vector<uint32_t>> want = {{0}, {1, 7}, {2, 8}, {}, {}, {}, {}, {}, {}, {}, {4}, {5}, {6}, {3}};
    bool ok = true;
    for (uint32_t j = 0; j < kTraceMaxWords; ++j) {
        std::vector<uint32_t> got;
        for (uint32_t s = m.word_first[j]; s < m.word_first[j + 1]; ++s) got.push_back(m.slot[s]);
        ok = ok && got == (j < want.size() ? want[j] : std::vector<uint32_t>{});
    }
    EXPECT(ok, "word -> record slots");
    EXPECT(m.word_absent[13] == 2 && m.word_absent[0] == 0, "word absent bits");
}

static void test_refusals() {
    std::string err;
    FeedParams p{};
    struct FieldCase { std::vector<bgr_feed_field> f; int status; const char* msg; };
    const FieldCase cases[] = {
        {{}, BGR_OK, ""},
        {{{0, 0, 40}}, BGR_OK, ""},
        {{{3, 0, 4}}, BGR_ERR_INVALID_ARGUMENT, "unknown column"},
        {{{0, 2, 4}}, BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element"},
        {{{0, 0, 6}}, BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element"},
        {{{0, 0, 0}}, BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element"},
        {{{1, 4, 12}}, BGR_ERR_INVALID_ARGUMENT, "field range must be 4-byte aligned and inside the element"},
        {std::vector<bgr_feed_field>(9, bgr_feed_field{1, 0, 4}), BGR_ERR_CAPACITY, "too many fields (BGR_MAX_FEED_FIELDS)"},
    };
    for (const FieldCase& c : cases) {
        err.clear();
        const int rc = fields_of(c.f, p, &err);
        EXPECT(rc == c.status && (rc == BGR_OK || err == c.msg), err.c_str());
    }
    err.clear();
    EXPECT(feed_fields(3u, [](uint32_t c) { return kCols[c]; }, 14u, nullptr, 1u, p, &err) == BGR_ERR_INVALID_ARGUMENT &&
               err == "null argument", "null field list");
    bgr_trace t{};
    t.interval = 7; t.first_row = 100; t.n_rows = 900;
    EXPECT(trace_check(t, 1000, &err) == BGR_OK, "the last row is the engine's last");
    t.n_rows = 901;
    EXPECT(trace_check(t, 1000, &err) == BGR_ERR_INVALID_ARGUMENT && err == "traced rows [100, 1001) exceed the engine's 1000 rows", err.c_str());
    t.first_row = 0xFFFFFFF0u; t.n_rows = 0x20u;  // first_row + n_rows wraps in 32 bits
    EXPECT(trace_check(t, 0xFFFFFFFFull, &err) == BGR_ERR_INVALID_ARGUMENT, "a range that wraps");
    t.first_row = 0; t.n_rows = 0;
    EXPECT(trace_check(t, 1000, &err) == BGR_ERR_INVALID_ARGUMENT && err == "bgr_trace.n_rows must be >= 1", err.c_str());
    t.n_rows = 1; t.interval = 0;
    EXPECT(trace_check(t, 1000, &err) == BGR_ERR_INVALID_ARGUMENT && err == "bgr_trace.interval must be >= 1", err.c_str());
    t.interval = 1; t.reserved = 1;
    EXPECT(trace_check(t, 1000, &err) == BGR_ERR_INVALID_ARGUMENT && err == "bgr_trace.reserved must be 0", err.c_str());
}

int main() {
    static_assert(sizeof(bgr_trace_sample) == 8 && sizeof(bgr_trace) == 56, "the header's trace structs");
    static_assert(sizeof(ReplayTrace) == 40 && sizeof(TraceMap) == 260, "the kernel's trace structs");
    std::mt19937_64 gen(0x5452414345ULL);
    test_samples_and_launches(gen);
    test_offsets_and_map();
    test_refusals();
    if (g_failed) {
        std::printf("%d of %d checks failed\n", g_failed, g_cases);
        return 1;
    }
    std::printf("replay trace plan test passed (%d checks)\n", g_cases);
    return 0;
}
