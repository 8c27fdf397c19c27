// The host side of a batched change-feed report (csrc/feed_check.hpp, run by bgr_batch_feed_begin before anything
// runs): every refusal of an entry (world out of range, listed twice, unknown feed, a report in flight, another field
// list) with its status, message and entry, in list order; a world listed again in a later call of a batch's list; and
// the table layout (first global tile, cap of at most the rows compared, staging size) against offsets computed by hand.
// Host only: exit code 0 = passed.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/feed_check.hpp"

using namespace bgr;

static int g_failed = 0, g_cases = 0;
#define EXPECT(cond, what)                                                                                   \
    do {                                                                                                     \
        ++g_cases;                                                                                           \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #cond, what); ++g_failed; } \
    } while (0)

// a registration's feed: fields of (plane, words, absent) as bgr_feed_create lays them out
static FeedParams feed_of(const std::vector<FeedField>& fields) {
    FeedParams p{};
    p.keep = 1u;
    for (const FeedField& f : fields) {
        p.fields[p.n_fields] = FeedField{f.plane, f.words, f.absent, p.rep_words};
        p.rep_words += f.words;
        p.keep |= f.absent;
        ++p.n_fields;
    }
    p.record_words = 2u + p.rep_words;
    return p;
}

// members x feeds: feeds[w][f] (nullptr: no such feed), busy[w][f]
struct Fleet {
    std::vector<std::vector<const FeedParams*>> feeds;
    std::vector<std::vector<bool>> busy;
    FeedView operator()(uint32_t w, uint32_t f) const {
        return f < feeds[w].size() && feeds[w][f] ? FeedView{feeds[w][f], busy[w][f]} : FeedView{nullptr, false};
    }
};

static void check(const Fleet& fl, const std::vector<bgr_batch_feed>& r, int status, uint32_t entry, const char* text) {
    uint32_t bad = 12345;
    std::string err;
    const int rc = feed_batch_check(uint32_t(fl.feeds.size()), r.data(), uint32_t(r.size()), fl, &bad, &err);
    EXPECT(rc == status, text);
    if (status != BGR_OK) {
        EXPECT(bad == entry, text);
        EXPECT(err == text, (err + " != " + text).c_str());
    }
}

int main() {
    const FeedParams a = feed_of({{3, 2, 0}, {7, 1, 4}});       // two fields, one of an optional column
    const FeedParams a2 = feed_of({{3, 2, 0}, {7, 1, 4}});      // the same list on another member
    const FeedParams b = feed_of({{3, 2, 0}});                  // a prefix of it: another record size
    const FeedParams c = feed_of({{3, 1, 0}, {7, 2, 4}});       // the same record size, other fields
    const FeedParams d = feed_of({{3, 2, 0}, {7, 1, 8}});       // the same words, another absent bit
    Fleet fl;
    fl.feeds = {{&a, &b}, {&a2, nullptr, &c}, {&a, &d}, {nullptr}};
    fl.busy = {{false, false}, {false, false, false}, {true, false}, {false}};
    EXPECT(feed_same_fields(a, a2) && !feed_same_fields(a, b) && !feed_same_fields(a, c) && !feed_same_fields(a, d), "field lists");

    check(fl, {}, BGR_OK, 0, "");
    check(fl, {{1, 0, 5}, {0, 0, 0}}, BGR_OK, 0, "");
    check(fl, {{0, 1, 5}}, BGR_OK, 0, "");
    check(fl, {{0, 0, 5}, {4, 0, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, "no such world in a batch of 4");
    check(fl, {{0, 0, 5}, {1, 0, 5}, {0, 0, 1}}, BGR_ERR_INVALID_ARGUMENT, 2, "listed twice in one call");
    check(fl, {{0, 0, 5}, {1, 1, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, "unknown feed");
    check(fl, {{3, 0, 5}}, BGR_ERR_INVALID_ARGUMENT, 0, "unknown feed");
    check(fl, {{1, 0, 5}, {0, BGR_MAX_FEEDS, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, "unknown feed");
    check(fl, {{1, 0, 5}, {2, 0, 5}}, BGR_ERR_STATE, 1, "a report of this feed is in flight");
    const char* other = "its feed's fields differ from those of entry 0's feed (a call has one record size)";
    check(fl, {{1, 0, 5}, {0, 1, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, other);
    check(fl, {{0, 0, 5}, {1, 2, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, other);
    check(fl, {{0, 0, 5}, {2, 1, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, other);
    check(fl, {{0, 1, 5}, {2, 1, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, other);
    // the first failing entry in list order is the one reported
    check(fl, {{0, 0, 5}, {2, 0, 5}, {9, 0, 5}}, BGR_ERR_STATE, 1, "a report of this feed is in flight");
    check(fl, {{0, 0, 5}, {0, 0, 5}, {2, 0, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, "listed twice in one call");

    // one list kept across calls, as a batch keeps it: a world listed in one call may be listed again in the next,
    // whether that call passed or was refused, and is still refused when listed twice in one call
    {
        WorldList list(4);
        auto call = [&](const std::vector<bgr_batch_feed>& r, int status, uint32_t entry, const char* text) {
            uint32_t bad = 12345;
            std::string err;
            list.begin();
            const int rc = feed_batch_check(list, r.data(), uint32_t(r.size()), fl, &bad, &err);
            EXPECT(rc == status, text);
            if (status != BGR_OK) EXPECT(bad == entry && err == text, (err + " != " + text).c_str());
        };
        call({{0, 0, 5}, {1, 0, 5}}, BGR_OK, 0, "second call");
        call({{1, 0, 5}, {0, 0, 5}}, BGR_OK, 0, "listed again in the next call");
        call({{0, 0, 5}, {1, 1, 5}}, BGR_ERR_INVALID_ARGUMENT, 1, "unknown feed");
        call({{1, 0, 5}, {0, 0, 5}}, BGR_OK, 0, "listed again after a refused call");
        call({{0, 0, 5}, {1, 0, 5}, {0, 0, 5}}, BGR_ERR_INVALID_ARGUMENT, 2, "listed twice in one call");
    }

    // the layout: tiles compared per world 3, 0, 1, 2048, 0; caps 10, 7, 9999, 2^32-1, 0
    std::vector<FeedWorld> tab(5);
    const uint32_t n_tiles[5] = {3, 0, 1, 2048, 0};
    for (int i = 0; i < 5; ++i) tab[i].n_tiles = n_tiles[i];
    const std::vector<bgr_batch_feed> r = {{4, 0, 10}, {2, 0, 7}, {0, 0, 9999}, {1, 0, 0xFFFFFFFFu}, {3, 0, 0}};
    uint64_t stage = 0;
    const uint32_t tiles = feed_layout(tab.data(), r.data(), 5, &stage);
    EXPECT(tiles == 3 + 0 + 1 + 2048 + 0, "total tiles");
    const uint32_t tile0[5] = {0, 3, 3, 4, 2052};
    const uint32_t cap[5] = {10, 0, 512, 2048 * 512, 0};  // a world without tiles reports nothing; no cap past its rows
    for (int i = 0; i < 5; ++i) {
        EXPECT(tab[i].tile0 == tile0[i], ("tile0 of entry " + std::to_string(i)).c_str());
        EXPECT(tab[i].cap == cap[i], ("cap of entry " + std::to_string(i)).c_str());
    }
    EXPECT(stage == 10u + 512u + 2048u * 512u, "staging records");
    feed_layout(tab.data(), r.data(), 0, &stage);
    EXPECT(stage == 0, "an empty call stages nothing");

    if (g_failed) {
        std::printf("%d of %d checks failed\n", g_failed, g_cases);
        return 1;
    }
    std::printf("feed host check test passed (%d checks)\n", g_cases);
    return 0;
}
