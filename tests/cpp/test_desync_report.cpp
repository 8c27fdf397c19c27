// The desync report through the C++ host mirror (bevy_ggrs_b200/host/bevy_ggrs.hpp): a SyncTestMismatch observer of
// the non-deterministic world of tests/synctest.rs:83-125 asks where the re-simulation diverged, and the report must
// name the Counter column, its one word, and every entity: 1400 of them, so the records come from many warps of three
// 512-row tiles.
// Exit code 0 = passed.  Needs an H100 (tests/test_cpp_desync_report.py, -m gpu); `--no-gpu` only checks that the
// engine refuses to start without a device.
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

struct Score { uint32_t v; };    // deterministic, +1 per frame
struct Counter { uint32_t v; };  // synctest.rs:87-88: written from a counter that is not rolled back

static void input_system(App& app) {
    LocalInputs li;
    for (auto h : app.local_players().handles) li.inputs[h] = 0;
    app.insert_resource(li);
}

static void mismatch_observer_reports_the_counter_column() {
    std::printf("mismatch_observer_reports_the_counter_column\n");
    const uint32_t rows = 1400;
    App app(rows + 64, 8, 0, BGR_CFG_DESYNC_CAPTURE);
    app.insert_resource(Session::SyncTest(ggrs::SyncTestSession(1, 2)))
        .add_plugins(GgrsPlugin<GgrsConfig<uint8_t>>{})
        .add_systems(ReadInputs{}, input_system);
    app.rollback_component_with_copy<Score>();
    app.rollback_component_with_copy<Counter>().checksum_component_with_hash<Counter>();
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_ADD, {0}, {0, 1}});
    app.add_systems(GgrsSchedule{}, System{BGR_SYS_U32_STORE_CALL_COUNT, {1}, {0}});
    app.add_systems(Startup{}, [&](App& a) { a.spawn(rows); });
    int reports = 0;
    app.add_observer([&](const SyncTestMismatch& m) {
        if (reports) return;
        for (ggrs::Frame f : m.mismatched_frames) {
            App::DesyncReport r = app.desync_report(f, 2 * rows);
            EXPECT(r.found);
            if (!r.found) continue;
            ++reports;
            const uint32_t counter = app.col<Counter>();
            EXPECT(r.summary.frame == f);
            EXPECT(r.summary.rows_differing == rows && r.summary.words_differing == rows);
            EXPECT(r.summary.existence_differing == 0 && r.summary.host_state_differs == 0);
            EXPECT(r.columns[counter].rows == rows && r.columns[counter].rows_in_checksum == rows);
            EXPECT(r.columns[app.col<Score>()].rows == 0);
            EXPECT(r.column_names[counter].find("Counter") != std::string::npos);
            EXPECT(r.records.size() == rows);
            std::set<uint32_t> seen;
            for (const bgr_desync_record& rec : r.records) {
                EXPECT(rec.column == counter && rec.word == 0 && rec.first != rec.latest);
                seen.insert(rec.row);
            }
            EXPECT(seen.size() == rows);
            for (size_t i = 1; i < r.records.size(); ++i) EXPECT(r.records[i - 1].row < r.records[i].row);
            // a cap that ends inside the second tile returns exactly the leading records
            App::DesyncReport head = app.desync_report(f, 700);
            EXPECT(head.records.size() == 700);
            for (size_t i = 0; i < head.records.size() && i < r.records.size(); ++i)
                EXPECT(head.records[i].row == r.records[i].row && head.records[i].latest == r.records[i].latest);
        }
    });
    for (int i = 0; i < 10 && !reports; ++i) app.update();
    EXPECT(reports > 0);
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "--no-gpu") {
        try {
            App app(16, 8, 0, BGR_CFG_DESYNC_CAPTURE);
            app.rollback_component_with_copy<Counter>();
            app.spawn(1);
            std::printf("engine started: a GPU is present\n");
        } catch (const Panic& p) {
            std::printf("refused: %s\n", p.what());
        }
        return 0;
    }
    mismatch_observer_reports_the_counter_column();
    std::printf(g_failed ? "%d check(s) FAILED\n" : "desync report test passed\n", g_failed);
    return g_failed ? 1 : 0;
}
