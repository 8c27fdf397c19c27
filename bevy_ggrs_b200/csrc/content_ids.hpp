// Content ids of the bundle kernel's active planes and alive byte, derived on the host (the invariant and every writer
// of an image are listed in engine.cu HostState).  Pure host code: no CUDA header, so tests compile it on its own.
//
// An id names one content exactly, never a hash of it: two images get the same id only when one was derived from the
// same content by the same ADVANCE as the other, or is a copy of it.  The kernels are bit-deterministic, so equal
// derivations give equal bytes, and a Save of content the target slot already holds can skip its stores.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <type_traits>

namespace bgr {

// The fields of an ADVANCE op its result depends on; everything else of the op is zeroed (engine.cu advance_key).
struct AdvanceKey {
    uint32_t dt_bits = 0, fr_bits = 0;  // frame time and friction factor
    uint32_t n_rows = 0;                // rows that exist while it runs
    uint32_t call_count = 0;            // the un-rolled-back counter of the call-count systems
    uint32_t n_players = 0;
    uint8_t inputs[8] = {};
    bool operator==(const AdvanceKey& o) const { return std::memcmp(this, &o, sizeof *this) == 0; }
};
static_assert(sizeof(AdvanceKey) == 28, "AdvanceKey has no padding: operator== compares every byte");

// How an image's content came about: its id (0 = unknown), the id of the content an ADVANCE with `key` made it from
// (0: it was not made by an ADVANCE of known content, so no other derivation matches it), and its row count.
struct ContentRecord {
    uint64_t cid = 0, parent = 0;
    AdvanceKey key;
    uint32_t rows = 0;
};

template <uint32_t kSlots>
struct ContentIds {
    ContentRecord live;                          // image 0, a deferred live image taken as materialised
    std::array<ContentRecord, kSlots> slot{};    // image s + 1
    uint64_t counter = 0;                        // ids handed out so far; an id is never handed out twice
    uint64_t epoch = 0;                          // the engine's stamp-table clears this table has seen

    // content nothing else is known to equal (a host write, a spawn)
    ContentRecord fresh(uint32_t rows) {
        ContentRecord r;
        r.cid = ++counter;
        r.rows = rows;
        return r;
    }
    // ADVANCE `k` applied to content `from`: the id of an image's content derived the same way (a slot's, or the live
    // image's, which a deferred live image's replay derives again), else a fresh one
    ContentRecord advance(const ContentRecord& from, const AdvanceKey& k) {
        ContentRecord r;
        r.parent = from.cid;
        r.key = k;
        r.rows = k.n_rows;
        auto same = [&](const ContentRecord& s) { return s.cid && s.parent == from.cid && s.key == k; };
        if (from.cid) {
            if (same(live)) { r.cid = live.cid; return r; }
            for (const ContentRecord& s : slot)
                if (same(s)) { r.cid = s.cid; return r; }
        }
        r.cid = ++counter;
        return r;
    }
    // A SAVE of content `reg` with `rows` rows into slot s.  True: it is held, the slot already holds exactly that
    // content (only when `may_hold`).  The slot takes the record either way.
    bool save(uint32_t s, const ContentRecord& reg, uint32_t rows, bool may_hold) {
        ContentRecord& t = slot[s];
        const bool held = may_hold && reg.cid != 0 && t.cid == reg.cid && t.rows == rows;
        t = reg;
        t.rows = rows;
        return held;
    }
    void forget() {
        live = ContentRecord{};
        slot.fill(ContentRecord{});
    }
    // `epoch` counts the clears of the engine's stamp table: one since the last call forgets every id
    void sync_epoch(uint64_t e) {
        if (epoch != e) forget();
        epoch = e;
    }
};
static_assert(std::is_trivially_copyable<ContentIds<4>>::value, "HostState copies it on every call");

}  // namespace bgr
