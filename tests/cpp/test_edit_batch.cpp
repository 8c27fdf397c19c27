// The host side of a batched edit call (csrc/edit_batch.hpp, run by bgr_batch_apply_edits before anything runs): every
// refusal of an entry (world out of range, listed twice, null pointers, a record the single call refuses, a spawn past
// a member's ceiling) with its status, message and entry, in list order; and the layout of a call's patch (each world's
// offsets in the flat word, mask and spawn spaces, the tables, the staging bytes) against offsets computed by hand.
// Host only: exit code 0 = passed.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/edit_batch.hpp"

using namespace bgr;

static int g_failed = 0, g_cases = 0;
#define EXPECT(cond, what)                                                                                   \
    do {                                                                                                     \
        ++g_cases;                                                                                           \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #cond, what); ++g_failed; } \
    } while (0)

// Members as the checks see them: their row count, capacity and ceiling.  `validate` stands in for the engine's
// validate_edits: records of kind BGR_EDIT_SPAWN append rows, a record with row >= the row count so far is refused
// with the single call's text, and a fixed member refuses spawns past its capacity.
struct Member { uint64_t rows, cap, ceiling; };
struct Fleet {
    std::vector<Member> m;
    int validate(uint32_t w, const bgr_batch_edits& x, uint64_t* rows, std::string* err) const {
        uint64_t r = m[w].rows;
        for (uint32_t i = 0; i < x.n_edits; ++i) {
            const bgr_edit& d = x.edits[i];
            if (d.kind == BGR_EDIT_SPAWN) { r += d.count; continue; }
            if (d.row >= r) { *err = "edit " + std::to_string(i) + ": row out of range"; return BGR_ERR_INVALID_ARGUMENT; }
        }
        if (r > m[w].cap && m[w].ceiling == m[w].cap) { *err = "spawn exceeds max_entities"; return BGR_ERR_CAPACITY; }
        *rows = r;
        return BGR_OK;
    }
};

static int check(const Fleet& f, const std::vector<bgr_batch_edits>& x, std::vector<uint64_t>& rows, uint32_t* bad, std::string* err) {
    rows.assign(x.size(), ~0ull);
    return edit_batch_check(uint32_t(f.m.size()), x.data(), uint32_t(x.size()),
                            [&](uint32_t w, const bgr_batch_edits& e, uint64_t* r, std::string* s) { return f.validate(w, e, r, s); },
                            [&](uint32_t w) { return f.m[w].rows; }, [&](uint32_t w) { return f.m[w].ceiling; },
                            rows.data(), bad, err);
}

static bgr_edit write_at(uint32_t row) { bgr_edit d{}; d.kind = BGR_EDIT_WRITE; d.row = row; d.count = 1; d.byte_len = 4; return d; }
static bgr_edit spawn(uint32_t n) { bgr_edit d{}; d.kind = BGR_EDIT_SPAWN; d.count = n; return d; }

static void test_checks() {
    // 0: fixed, 10 rows of 16; 1: growable, 10 of 16, ceiling 100; 2: fixed, 0 of 4
    Fleet f{{{10, 16, 16}, {10, 16, 100}, {0, 4, 4}}};
    const bgr_edit ok[2] = {write_at(3), write_at(9)};
    const bgr_edit bad_row[4] = {write_at(0), write_at(1), write_at(2), write_at(10)};
    const bgr_edit grow[2] = {spawn(50), write_at(59)};
    const bgr_edit huge[1] = {spawn(91)};
    const bgr_edit past_cap[1] = {spawn(5)};
    const uint8_t vals[4] = {};
    std::vector<uint64_t> rows;
    uint32_t bad = 99;
    std::string err;

    // every entry passes: rows afterwards, an empty entry keeps its member's rows; a growable member may pass its cap
    int rc = check(f, {{0, 2, ok, vals, 4}, {1, 2, grow, nullptr, 0}, {2, 0, nullptr, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_OK, err.c_str());
    EXPECT(rows[0] == 10 && rows[1] == 60 && rows[2] == 0, "rows after each entry");

    // out of range, at entry 1
    rc = check(f, {{0, 2, ok, vals, 4}, {3, 0, nullptr, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 1 && err == "no such world in a batch of 3", err.c_str());
    // listed twice, at the second listing, even with no edits
    rc = check(f, {{2, 0, nullptr, nullptr, 0}, {0, 2, ok, vals, 4}, {2, 0, nullptr, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 2 && err == "listed twice in one call", err.c_str());
    // null pointers: records without a pointer, values_bytes without values (even with no records, as the single call)
    rc = check(f, {{0, 2, nullptr, vals, 4}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 0 && err == "null argument", err.c_str());
    rc = check(f, {{1, 0, nullptr, nullptr, 0}, {0, 0, nullptr, nullptr, 8}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 1 && err == "null argument", err.c_str());
    // a bad record in entry 2: the single call's text, the entry's index
    rc = check(f, {{2, 0, nullptr, nullptr, 0}, {1, 2, ok, vals, 4}, {0, 4, bad_row, vals, 4}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 2 && err == "edit 3: row out of range", err.c_str());
    // a fixed member past its capacity, with a growable member that grows listed before it
    rc = check(f, {{1, 2, grow, nullptr, 0}, {2, 1, past_cap, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_CAPACITY && bad == 1 && err == "spawn exceeds max_entities", err.c_str());
    // a growable member past its ceiling
    rc = check(f, {{0, 2, ok, vals, 4}, {1, 1, huge, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_CAPACITY && bad == 1 && err == "101 rows exceed the engine's ceiling of 100 rows (BGR_CFG_GROWABLE)", err.c_str());
    // the first failure in list order wins
    rc = check(f, {{0, 4, bad_row, vals, 4}, {5, 0, nullptr, nullptr, 0}}, rows, &bad, &err);
    EXPECT(rc == BGR_ERR_INVALID_ARGUMENT && bad == 0 && err == "edit 3: row out of range", err.c_str());
}

static void test_layout() {
    // entry: words, masks, first_row, spawned.  0: a patch; 1: no edits; 2: spawn only (empty patch); 3: masks only and a
    // spawn; 4: words and masks
    const EditCounts c[5] = {{5, 2, 100, 0}, {0, 0, 7, 0}, {0, 0, 30, 4}, {0, 3, 0, 2}, {6, 1, 9, 0}};
    EditLayout L;
    uint32_t bad = 99;
    std::string err;
    int rc = edit_layout(c, 5, &L, &bad, &err);
    EXPECT(rc == BGR_OK, err.c_str());
    EXPECT(L.n_words == 11 && L.n_masks == 6 && L.n_spawned == 6, "totals");
    EXPECT(L.patch.size() == 3 && L.patch_entry == std::vector<uint32_t>({0, 3, 4}), "patch entries");
    // t0 = earlier words + masks; word0 / mask0 = earlier words / masks
    EXPECT(L.patch[0].t0 == 0 && L.patch[0].n_words == 5 && L.patch[0].word0 == 0 && L.patch[0].mask0 == 0, "entry 0");
    EXPECT(L.patch[1].t0 == 7 && L.patch[1].n_words == 0 && L.patch[1].word0 == 5 && L.patch[1].mask0 == 2, "entry 3");
    EXPECT(L.patch[2].t0 == 10 && L.patch[2].n_words == 6 && L.patch[2].word0 == 5 && L.patch[2].mask0 == 5, "entry 4");
    EXPECT(L.spawn.size() == 2 && L.spawn_entry == std::vector<uint32_t>({2, 3}), "spawn entries");
    EXPECT(L.spawn[0].row0 == 0 && L.spawn[0].first_row == 30 && L.spawn[0].count == 4, "spawn of entry 2");
    EXPECT(L.spawn[1].row0 == 4 && L.spawn[1].first_row == 0 && L.spawn[1].count == 2, "spawn of entry 3");
    // staging: 11 words of 16 B, 6 masks of 8 B, 3 EditWorlds and 2 SpawnWorlds of 24 B
    EXPECT(L.off_masks == 176 && L.off_patch == 224 && L.off_spawn == 296 && L.bytes == 344, "staging offsets");

    // nothing to do: no tables, no bytes
    const EditCounts none[2] = {{0, 0, 5, 0}, {0, 0, 0, 0}};
    rc = edit_layout(none, 2, &L, &bad, &err);
    EXPECT(rc == BGR_OK && L.patch.empty() && L.spawn.empty() && L.bytes == 0, "empty call");

    // one launch's index space: 2^31 - 1 words and masks, or spawned rows
    const EditCounts big[3] = {{1u << 30, 0, 0, 0}, {(1u << 30) - 2, 1, 0, 0}, {0, 1, 0, 0}};
    rc = edit_layout(big, 3, &L, &bad, &err);
    EXPECT(rc == BGR_ERR_CAPACITY && bad == 2 && err == "edit batch too large", err.c_str());
    const EditCounts spawns[2] = {{0, 0, 0, 0x40000000u}, {0, 0, 0, 0x40000000u}};
    rc = edit_layout(spawns, 2, &L, &bad, &err);
    EXPECT(rc == BGR_ERR_CAPACITY && bad == 1, err.c_str());
}

int main() {
    test_checks();
    test_layout();
    if (g_failed) {
        std::printf("%d of %d checks failed\n", g_failed, g_cases);
        return 1;
    }
    std::printf("edit batch host check test passed (%d checks)\n", g_cases);
    return 0;
}
