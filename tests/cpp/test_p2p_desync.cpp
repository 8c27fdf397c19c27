// P2P desync reports through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): two peers run the same game with
// different rollback patterns; peer B's initial population differs in one Tag word of block 0 and one Score of
// block 2.  Each keeps the confirmed multiples of the desync interval, the digests name exactly blocks 0 and 2, and
// B's exported blocks diffed on A show exactly those two words.  Then two peers whose frames differ in block count
// (512 vs 513 rows) run the documented exchange in both directions: each side reports the one row only B has.
// Exit code 0 = passed.  Needs an H100 (tests/test_cpp_p2p_desync.py, -m gpu); `--no-gpu` only checks that the engine
// refuses to start without a device.
#include <cstdio>
#include <set>
#include <string>

#include "../../bevy_ggrs_b200/host/bevy_ggrs.hpp"

using namespace bevy_ggrs;

static int g_failed = 0;
#define EXPECT(cond)                                                                  \
    do {                                                                              \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failed; } \
    } while (0)

struct Score { uint32_t v; };   // +1 per frame
struct Tag { uint32_t a, b; };  // written once, no system

static const uint32_t kRows = 1400;

static void input_system(App& app) {
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = 0;
    app.insert_resource(li);
}

static void setup(App& app, int seed, bool edited, uint32_t rows = kRows) {
    std::vector<int> depths;
    for (int t = 0; t < 80; ++t) depths.push_back((t * seed + 3) % 4);
    app.insert_resource(Session::P2P(ggrs::P2PTraceSession(2, 8, depths, /*confirm_lag=*/3)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system);
    app.rollback_component_with_copy<Score>().checksum_component_with_hash<Score>();
    app.rollback_component_with_copy<Tag>().checksum_component_with_hash<Tag>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.retain_confirmed(5, 4);
    app.add_systems(Startup{}, [edited, rows](App& a) {
        const uint32_t first = a.spawn(rows);
        std::vector<Score> s(rows);
        std::vector<Tag> t(rows);
        for (uint32_t i = 0; i < rows; ++i) { s[i].v = i * 7u; t[i] = Tag{i, i ^ 0x5a5au}; }
        if (edited) t[9].b ^= 1u;                                   // block 0
        if (edited) s[2 * BGR_DIGEST_BLOCK_ROWS + 17].v += 1000u;    // block 2
        a.write<Score>(first, s);
        a.write<Tag>(first, t);
    });
}

static void two_peers_find_and_diff_the_differing_blocks() {
    std::printf("two_peers_find_and_diff_the_differing_blocks\n");
    App a(kRows + 8, 8), b(kRows + 8, 8);
    setup(a, 5, false);
    setup(b, 3, true);
    for (int i = 0; i < 60; ++i) { a.update(); b.update(); }
    const auto ra = a.retained_frames(), rb = b.retained_frames();
    EXPECT(ra.size() == 4 && ra == rb);
    for (ggrs::Frame f : ra) {
        App::FrameDigest da = a.frame_digest(f), db = b.frame_digest(f);
        EXPECT(da.found && db.found && f % 5 == 0);
        uint32_t host = 0;
        const std::vector<uint32_t> blocks = App::digest_mismatch(da, db, &host);
        EXPECT((blocks == std::vector<uint32_t>{0, 2}) && host == 0);
        const std::vector<uint8_t> blob = b.export_blocks(f, blocks);
        EXPECT(!blob.empty());
        App::DesyncReport r = a.diff_remote(f, blob, 16);
        EXPECT(r.found && r.summary.frame == f);
        EXPECT(r.summary.rows_differing == 2 && r.summary.existence_differing == 0 && r.summary.words_differing == 2);
        EXPECT(r.columns[a.col<Tag>()].rows == 1 && r.columns[a.col<Score>()].rows == 1);
        EXPECT(r.records.size() == 2);
        if (r.records.size() == 2) {
            EXPECT(r.records[0].row == 9 && r.records[0].column == a.col<Tag>() && r.records[0].word == 1);
            EXPECT(r.records[0].first == (9u ^ 0x5a5au) && r.records[0].latest == (9u ^ 0x5a5au ^ 1u));
            EXPECT(r.records[1].row == 2 * BGR_DIGEST_BLOCK_ROWS + 17 && r.records[1].column == a.col<Score>());
            EXPECT(r.records[1].word == 0 && r.records[1].latest == r.records[1].first + 1000u);
        }
    }
    // a frame neither queued nor retained
    EXPECT(!a.frame_digest(3).found && a.export_blocks(3, {0}).empty());
}

// INTEGRATION.md's exchange: the local side asks for the mismatched blocks the peer has (below the peer digest's
// n_blocks, possibly none), the peer exports them, the local side diffs the blob.
static App::DesyncReport exchange(App& local, App& remote, ggrs::Frame f) {
    App::FrameDigest dl = local.frame_digest(f), dr = remote.frame_digest(f);
    std::vector<uint32_t> want;
    for (uint32_t b : App::digest_mismatch(dl, dr))
        if (b < dr.header.n_blocks) want.push_back(b);
    return local.diff_remote(f, remote.export_blocks(f, want), 16);
}

static void peers_with_different_block_counts_report_the_extra_row_both_ways() {
    std::printf("peers_with_different_block_counts_report_the_extra_row_both_ways\n");
    const uint32_t rows_a = BGR_DIGEST_BLOCK_ROWS, rows_b = BGR_DIGEST_BLOCK_ROWS + 1;
    App a(rows_b + 8, 8), b(rows_b + 8, 8);
    setup(a, 5, false, rows_a);
    setup(b, 3, false, rows_b);
    for (int i = 0; i < 60; ++i) { a.update(); b.update(); }
    const auto ra = a.retained_frames();
    EXPECT(!ra.empty() && ra == b.retained_frames());
    for (ggrs::Frame f : ra) {
        App::FrameDigest da = a.frame_digest(f), db = b.frame_digest(f);
        EXPECT(da.header.n_blocks == 1 && db.header.n_blocks == 2);
        EXPECT((App::digest_mismatch(da, db) == std::vector<uint32_t>{1}));
        const App::DesyncReport ab = exchange(a, b, f);   // A asks for block 1, B exports it
        const App::DesyncReport ba = exchange(b, a, f);   // B asks for nothing A has: A exports no block
        for (const App::DesyncReport* r : {&ab, &ba}) {
            EXPECT(r->found && r->summary.rows_differing == 1 && r->summary.existence_differing == 1);
            EXPECT(r->summary.words_differing == 0 && r->records.size() == 1);
            if (r->records.size() == 1) EXPECT(r->records[0].row == rows_a && r->records[0].column == 0xFFFFFFFFu);
        }
        EXPECT(ab.records.size() == 1 && ab.records[0].first == 0 && ab.records[0].latest != 0);
        EXPECT(ba.records.size() == 1 && ba.records[0].first != 0 && ba.records[0].latest == 0);
        EXPECT(ab.summary.rows_first == rows_a && ab.summary.rows_latest == rows_b);
        EXPECT(ba.summary.rows_first == rows_b && ba.summary.rows_latest == rows_a);
    }
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(16, 8);
            app.rollback_component_with_copy<Score>();
            app.retain_confirmed(5, 2);
            app.spawn(1);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    two_peers_find_and_diff_the_differing_blocks();
    peers_with_different_block_counts_report_the_extra_row_both_ways();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "p2p desync test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
