// Batched host edits (bgr_batch_apply_edits): the host checks of a call's entries, made before anything runs, and the
// layout of a call's patch (each world's offsets in the flat word, mask and spawn spaces, and the staging bytes).  Host
// only; tests/cpp/test_edit_batch.cpp holds it to every refusal and to hand-computed offsets.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "batch_call.hpp"
#include "kernels.cuh"  // EditWorld, SpawnWorld

namespace bgr {

// Checks the entries of one call in list order: world admitted to the call's `list` (begun by the caller), no null
// pointer, every record by the single call's checks, and the row count after the entry's spawns within the member's
// ceiling.
//   validate(world, entry, &rows, &err): bgr_apply_edits' own checks of a non-empty entry (status, err = its message,
//                                        rows = the row count after the entry);
//   ceiling(world):                      the most rows the member can hold (a growable member's BGR_CFG_GROWABLE
//                                        ceiling; a fixed member's own check in `validate` already refused more than
//                                        its max_entities).
// BGR_OK with rows[i] = entry i's row count afterwards (its member's rows(world) for an empty entry), or the status with
// *bad = the failing entry and *err = why.  Nothing is grown here, so a refusal leaves every member as it was.
template <class Validate, class Rows, class Ceiling>
int edit_batch_check(WorldList& list, const bgr_batch_edits* entries, uint32_t n, Validate validate, Rows rows_of,
                     Ceiling ceiling, uint64_t* rows, uint32_t* bad, std::string* err) {
    for (uint32_t i = 0; i < n; ++i) {
        *bad = i;
        const bgr_batch_edits& x = entries[i];
        if (const int rc = list.admit(x.world, err); rc != BGR_OK) return rc;
        if ((x.n_edits && !x.edits) || (x.values_bytes && !x.values)) { *err = "null argument"; return BGR_ERR_INVALID_ARGUMENT; }
        rows[i] = rows_of(x.world);
        if (x.n_edits == 0) continue;
        const int rc = validate(x.world, x, &rows[i], err);
        if (rc != BGR_OK) return rc;
        if (rows[i] > ceiling(x.world)) {
            *err = std::to_string(rows[i]) + " rows exceed the engine's ceiling of " + std::to_string(ceiling(x.world)) +
                   " rows (BGR_CFG_GROWABLE)";
            return BGR_ERR_CAPACITY;
        }
    }
    return BGR_OK;
}

// The same checks as one call to a batch of n_members that keeps no listing state between calls
template <class Validate, class Rows, class Ceiling>
int edit_batch_check(uint32_t n_members, const bgr_batch_edits* entries, uint32_t n, Validate validate, Rows rows_of,
                     Ceiling ceiling, uint64_t* rows, uint32_t* bad, std::string* err) {
    WorldList list(n_members);
    list.begin();
    return edit_batch_check(list, entries, n, validate, rows_of, ceiling, rows, bad, err);
}

// What one entry's folded patch holds: its stored words and presence masks, and the rows it spawns after first_row
// (the member's row count before the call)
struct EditCounts {
    uint64_t n_words, n_masks;
    uint32_t first_row, spawned;
};

// A call's patch in one page-locked staging buffer, read in place by the kernels except for the two tables, which go to
// the device with one copy:
//   [words: uint4 x n_words][masks: uint2 x n_masks][patch: EditWorld x patch.size()][spawn: SpawnWorld x spawn.size()]
// `patch` has one entry per world with a non-empty patch and `spawn` one per spawning world, both in list order (so in
// ascending t0 / row0, as the kernels' binary search needs); their img is left for the caller.
struct EditLayout {
    std::vector<EditWorld> patch;
    std::vector<SpawnWorld> spawn;
    std::vector<uint32_t> patch_entry, spawn_entry;  // the list entry of each table row
    uint32_t n_words = 0, n_masks = 0, n_spawned = 0;
    size_t off_masks = 0, off_patch = 0, off_spawn = 0, bytes = 0;
};

// BGR_OK, or BGR_ERR_CAPACITY with *bad = the entry at which one launch's index space (words and masks, or spawned
// rows, 2^31 - 1 at most, as for one bgr_apply_edits) would overflow.
inline int edit_layout(const EditCounts* c, uint32_t n, EditLayout* L, uint32_t* bad, std::string* err) {
    *L = EditLayout{};
    uint64_t words = 0, masks = 0, spawned = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (c[i].n_words + c[i].n_masks) {
            L->patch.push_back(EditWorld{nullptr, uint32_t(words + masks), uint32_t(c[i].n_words), uint32_t(words), uint32_t(masks)});
            L->patch_entry.push_back(i);
        }
        if (c[i].spawned) {
            L->spawn.push_back(SpawnWorld{nullptr, uint32_t(spawned), c[i].first_row, c[i].spawned, 0u});
            L->spawn_entry.push_back(i);
        }
        words += c[i].n_words;
        masks += c[i].n_masks;
        spawned += c[i].spawned;
        if (words + masks > 0x7FFFFFFFull || spawned > 0x7FFFFFFFull) {
            *bad = i;
            *err = "edit batch too large";
            return BGR_ERR_CAPACITY;
        }
    }
    L->n_words = uint32_t(words);
    L->n_masks = uint32_t(masks);
    L->n_spawned = uint32_t(spawned);
    L->off_masks = words * sizeof(uint4);
    L->off_patch = L->off_masks + masks * sizeof(uint2);
    L->off_spawn = L->off_patch + L->patch.size() * sizeof(EditWorld);
    L->bytes = L->off_spawn + L->spawn.size() * sizeof(SpawnWorld);
    return BGR_OK;
}

}  // namespace bgr
