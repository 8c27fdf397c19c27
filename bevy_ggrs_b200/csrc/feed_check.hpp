// Batched change feed (bgr_batch_feed_begin): the host checks of a call's entries, made before anything runs, and the
// table layout of a report (each world's first global tile and cap, the staging size).  Host only;
// tests/cpp/test_feed_check.cpp holds it to every refusal and to hand-computed offsets.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>

#include "../../include/bevy_ggrs_b200.h"
#include "batch_call.hpp"
#include "change_feed.cuh"  // FeedParams, FeedWorld

namespace bgr {

// A registered column as a change feed's field list sees it: its word planes and its absent bit (0: not optional)
struct FeedColumn {
    uint32_t first_plane, words, absent;
};

// The field list of a change feed (bgr_feed_create) or a replay trace (bgr_replay_trace) checked and mapped onto the
// image: each field's word plane, words, absent bit and record words, the mask bits its records' state is made of and the
// record size.  `col_at(c)` gives column c of the n_cols registered.  BGR_OK, or the status with *err = why; p is then
// unspecified.
template <class ColAt>
int feed_fields(uint32_t n_cols, ColAt col_at, uint32_t words, const bgr_feed_field* fields, uint32_t n_fields, FeedParams& p,
                std::string* err) {
    if (n_fields > BGR_MAX_FEED_FIELDS) { *err = "too many fields (BGR_MAX_FEED_FIELDS)"; return BGR_ERR_CAPACITY; }
    if (n_fields && !fields) { *err = "null argument"; return BGR_ERR_INVALID_ARGUMENT; }
    p.keep = 1u;
    p.rep_words = 0;
    for (uint32_t k = 0; k < n_fields; ++k) {
        const bgr_feed_field& f = fields[k];
        if (f.column >= n_cols) { *err = "unknown column"; return BGR_ERR_INVALID_ARGUMENT; }
        const FeedColumn c = col_at(f.column);
        if ((f.byte_offset & 3u) || (f.byte_len & 3u) || f.byte_len == 0 || uint64_t(f.byte_offset) + f.byte_len > uint64_t(c.words) * 4u) {
            *err = "field range must be 4-byte aligned and inside the element";
            return BGR_ERR_INVALID_ARGUMENT;
        }
        p.fields[k] = FeedField{c.first_plane + f.byte_offset / 4u, f.byte_len / 4u, c.absent, p.rep_words};
        p.rep_words += f.byte_len / 4u;
        p.keep |= c.absent;
    }
    p.n_fields = n_fields;
    p.words = words;
    p.record_words = 2u + p.rep_words;
    return BGR_OK;
}

// A feed as the checks see it: its registration (the fields, mask bits and record size in `reg`) and whether a report
// of it is in flight
struct FeedView {
    const FeedParams* reg;  // nullptr: no such feed
    bool busy;
};

// the same field list (so the same record layout) as another feed of the same registration
inline bool feed_same_fields(const FeedParams& a, const FeedParams& b) {
    if (a.n_fields != b.n_fields || a.keep != b.keep || a.record_words != b.record_words) return false;
    return std::memcmp(a.fields, b.fields, sizeof(FeedField) * a.n_fields) == 0;
}

// Checks the entries of one call in list order: world admitted to the call's `list` (begun by the caller), the feed known
// and idle, its fields those of entry 0's feed.  `view(world, feed)` gives the feed.  BGR_OK, or the status with *bad = the
// failing entry and *err = why (the single call's message where it has one).
template <class View>
int feed_batch_check(WorldList& list, const bgr_batch_feed* reports, uint32_t n, View view, uint32_t* bad, std::string* err) {
    const FeedParams* first = nullptr;
    for (uint32_t i = 0; i < n; ++i) {
        *bad = i;
        const bgr_batch_feed& r = reports[i];
        if (const int rc = list.admit(r.world, err); rc != BGR_OK) return rc;
        const FeedView f = view(r.world, r.feed);
        if (!f.reg) { *err = "unknown feed"; return BGR_ERR_INVALID_ARGUMENT; }
        if (f.busy) { *err = "a report of this feed is in flight"; return BGR_ERR_STATE; }
        if (!first) first = f.reg;
        else if (!feed_same_fields(*f.reg, *first)) {
            *err = "its feed's fields differ from those of entry 0's feed (a call has one record size)";
            return BGR_ERR_INVALID_ARGUMENT;
        }
    }
    return BGR_OK;
}

// The same checks as one call to a batch of n_members that keeps no listing state between calls
template <class View>
int feed_batch_check(uint32_t n_members, const bgr_batch_feed* reports, uint32_t n, View view, uint32_t* bad, std::string* err) {
    WorldList list(n_members);
    list.begin();
    return feed_batch_check(list, reports, n, view, bad, err);
}

// Fills tile0 and cap of every entry of `tab` (img, rep, rows and n_tiles set) in list order: consecutive global tiles,
// and a cap of at most every row compared.  Returns the global tile count; *stage_records = the records the staging
// must hold, the sum of the caps.
inline uint32_t feed_layout(FeedWorld* tab, const bgr_batch_feed* reports, uint32_t n, uint64_t* stage_records) {
    uint32_t tiles = 0;
    uint64_t recs = 0;
    for (uint32_t i = 0; i < n; ++i) {
        tab[i].tile0 = tiles;
        tab[i].cap = uint32_t(std::min<uint64_t>(reports[i].records_cap, uint64_t(tab[i].n_tiles) * kTileRows));
        tiles += tab[i].n_tiles;
        recs += tab[i].cap;
    }
    *stage_records = recs;
    return tiles;
}

}  // namespace bgr
