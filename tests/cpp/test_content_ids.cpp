// Content ids on their own (bevy_ggrs_b200/csrc/content_ids.hpp) with the engine's snapshot ring (ring.hpp): the
// host-side derivation that lets the bundle kernel hold a Save whose slot already holds the content.  Built and run by
// tests/test_content_ids.py; no GPU, no engine.
#include <cstdio>
#include <cstdlib>
#include <type_traits>

#include <string>

#include "../../bevy_ggrs_b200/csrc/content_ids.hpp"
#include "../../bevy_ggrs_b200/csrc/ring.hpp"

using namespace bgr;

static int g_failed = 0;
#define CHECK(cond)                                                              \
    do {                                                                         \
        if (!(cond)) {                                                           \
            std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond);        \
            ++g_failed;                                                          \
        }                                                                        \
    } while (0)

static_assert(std::is_trivially_copyable<ContentIds<64>>::value, "the engine's HostState copies it on every call");
static_assert(std::is_trivially_copyable<ContentRecord>::value, "records are plain data");

static AdvanceKey key(int32_t frame, uint32_t rows = 1000, uint32_t call_count = 0, uint8_t input = 0) {
    AdvanceKey k;
    k.dt_bits = 0x3c888889u;  // 1/60 s
    k.fr_bits = 0x3f7c0000u + uint32_t(frame % 7);  // stands for a per-frame friction factor
    k.n_rows = rows;
    k.call_count = call_count;
    k.n_players = 2;
    k.inputs[0] = input;
    k.inputs[1] = uint8_t(frame);  // the second player's input changes every frame
    return k;
}

// A SyncTest engine as engine.cu compile_requests / derive_content_ids drive the ring and the ids: the ring decides
// which slot each Save gets, ContentIds::save decides whether it is held.  Every Save skips the passive planes (the
// steady state) unless `passive_changed`.
struct SyncTestModel {
    SlotRing ring;
    ContentIds<SlotRing::kMaxSlots> c;
    int32_t frame = 0;
    int32_t d;
    bool passive_changed = false;
    uint64_t epoch = 0;
    SyncTestModel(int32_t d_, uint32_t slots) : ring(slots), d(d_) {
        ring.set_depth(slots);
        c.live = c.fresh(1000);
    }
    int save(ContentRecord& reg) {
        const uint32_t s = ring.push(frame);
        CHECK(s < SlotRing::kMaxSlots);
        return c.save(s, reg, reg.rows, !passive_changed) ? 1 : 0;
    }
    void advance(ContentRecord& reg) { reg = c.advance(reg, key(++frame)); }
    // one tick: [Load(f-d), Adv, Save, ..., Adv, Save(f), Adv] once f > d > 0, else [Save(f), Adv].  Returns held Saves.
    int tick() {
        c.sync_epoch(epoch);
        int held = 0;
        ContentRecord reg = c.live;
        if (d > 0 && frame > d) {
            ring.confirm(frame - d);
            std::string err;
            CHECK(ring.rollback(frame - d, &err));
            uint32_t s = 0;
            CHECK(ring.get(&s, &err));
            reg = c.slot[s];
            frame -= d;
            for (int32_t i = 0; i < d; ++i) {
                if (i > 0) held += save(reg);
                advance(reg);
            }
        }
        held += save(reg);
        advance(reg);
        c.live = reg;
        return held;
    }
};

int main() {
    // LIFO reuse through the engine's own ring: every re-save gets back the slot that holds its frame, and holds
    for (int32_t d = 1; d <= 8; ++d) {
        SyncTestModel m(d, uint32_t(d) + 1);
        for (int t = 0; t <= d; ++t) CHECK(m.tick() == 0);       // the first ticks save new frames only
        for (int t = 0; t < 20; ++t) CHECK(m.tick() == d - 1);   // Save(f) is new, the d - 1 re-saves are held
        // a host write of the live image: a fresh id.  The next tick's Load(f-d) rolls it back, so it still holds
        m.c.live = m.c.fresh(1000);
        CHECK(m.tick() == d - 1);
        // a slot written from the host (checkpoint restore, an edit of a slot): the re-saves derived from it store
        m.c.slot[0] = m.c.fresh(1000);
        for (uint32_t s = 1; s < uint32_t(d) + 1; ++s) m.c.slot[s] = m.c.fresh(1000);
        CHECK(m.tick() == 0);
        CHECK(m.tick() == d - 1);
        // a clear of the stamp table forgets every id: the next tick holds nothing, the one after holds again
        m.epoch += 1;
        CHECK(m.tick() == 0);
        CHECK(m.tick() == d - 1);
        // a Save that must store passive planes is never held
        m.passive_changed = true;
        CHECK(m.tick() == 0);
        m.passive_changed = false;
        CHECK(m.tick() == d - 1);
    }
    // clean P2P ticks (Save(f), Advance) never hold: each Save is a new frame into the slot of the evicted oldest one
    {
        SyncTestModel m(0, 8);
        for (int t = 0; t < 30; ++t) CHECK(m.tick() == 0);
    }
    // equal derivations get equal ids; any key field the result depends on gives a new one
    {
        ContentIds<8> c;
        const ContentRecord base = c.fresh(1000);
        c.slot[0] = base;
        const ContentRecord a = c.advance(base, key(5));
        c.slot[1] = a;
        CHECK(a.cid != 0 && a.cid != base.cid && a.parent == base.cid);
        CHECK(c.advance(base, key(5)).cid == a.cid);  // found through slot 1's record
        AdvanceKey k = key(5);
        k.inputs[0] = 1;
        CHECK(c.advance(base, k).cid != a.cid);  // a different input
        k = key(5);
        k.dt_bits ^= 1u;
        CHECK(c.advance(base, k).cid != a.cid);  // a different frame time
        CHECK(c.advance(base, key(5, 1000, 3)).cid != a.cid);  // a different call count
        CHECK(c.advance(base, key(5, 999)).cid != a.cid);      // a different row count
        k = key(5);
        k.fr_bits ^= 1u;
        CHECK(c.advance(base, k).cid != a.cid);  // a different friction factor (box_game)
        k = key(5);
        k.n_players = 3;
        CHECK(c.advance(base, k).cid != a.cid);
        // the same key from other content
        const ContentRecord other = c.fresh(1000);
        CHECK(c.advance(other, key(5)).cid != a.cid);
        // unknown content derives nothing known: fresh every time, and never matched later
        const ContentRecord u1 = c.advance(ContentRecord{}, key(5)), u2 = c.advance(ContentRecord{}, key(5));
        CHECK(u1.cid != 0 && u2.cid != 0 && u1.cid != u2.cid && u1.parent == 0);
    }
    // a spawn (or a host write) gives a fresh id, never one an image already has
    {
        ContentIds<8> c;
        const ContentRecord x = c.fresh(10), y = c.fresh(10), z = c.fresh(14);
        CHECK(x.cid != y.cid && y.cid != z.cid && x.cid != z.cid && z.rows == 14);
        CHECK(x.parent == 0 && y.parent == 0);
    }
    // forgetting clears every image's id but never hands an id out twice
    {
        ContentIds<8> c;
        c.live = c.fresh(5);
        c.slot[3] = c.advance(c.live, key(1, 5));
        const uint64_t before = c.slot[3].cid;
        c.forget();
        CHECK(c.live.cid == 0 && c.slot[3].cid == 0);
        CHECK(c.fresh(5).cid > before);
        CHECK(c.advance(c.live, key(1, 5)).cid > before);
    }
    if (g_failed) {
        std::printf("%d checks failed\n", g_failed);
        return 1;
    }
    std::printf("content id tests passed\n");
    return 0;
}
