// Host-side bookkeeping of the snapshot ring: which frame lives in which HBM slot.
//
// Behaviour contract = GgrsSnapshots<For, As> (reference src/snapshot/mod.rs:94-271):
// a newest-first queue of (frame -> snapshot) with
//   push(frame)     :144-178  drop every stored frame that is not older than `frame`
//                              (i32 wrap-around aware), prepend, then evict beyond `depth`
//   confirm(frame)  :182-199  drop from the old end while stored < frame
//   rollback(frame) :207-223  drop from the new end until the newest == frame, else fail with
//                              "Could not rollback to {frame}: no snapshot at that moment could be found."
//   get()/peek()    :226-240
// Only the *payload* differs: instead of owning a HashMap per frame, an entry names a slot of
// pre-allocated HBM; freed slots go back to a free list, so no allocation ever happens on the
// hot path.  All per-type rings of the reference move in lock-step (every SaveWorld pushes
// the same frame into each of them, every LoadWorld rolls each back to the same frame), so one
// ring serves every registered column.
//
// Desync capture (BGR_CFG_DESYNC_CAPTURE, reset(n, true)): the ring also keeps, per frame, a WITNESS — the slot of the
// frame's first push since its previous witness was released.  A witness slot is pinned: when the queue drops the
// entry (rollback, or a push of an older / equal frame) the slot does not go back on the free list, so a re-save of
// the frame lands in another slot and the first image survives for bgr_desync_diff.  The queue itself (get / peek /
// frames) is exactly the plain ring's.  A witness is released when
//   - confirm(c) runs with its frame < c (whether or not the frame is still queued),
//   - the queue evicts its frame from the OLD end for depth,
//   - release_witnesses() runs (bgr_reset_session),
//   - a push finds no free slot: the witness recorded first is released, and so on until a slot is free.
// Bound: a SyncTest of check distance d (d < max_prediction <= depth) needs at most 2(d+1) slots.  A re-save of frame
// f inside a rollback confirms only f-d, so while tick `cur` re-saves frame cur-1 the queue holds cur-d-1 .. cur-1
// (d+1 images) and the witnesses of those d+1 frames sit in other slots.  d+1 <= max_prediction <= max_depth, so the
// engine's 2*max_depth slots always suffice (tests/test_desync_capture.py walks every d in 1..7, max_prediction in
// d+1..8 and sees exactly 2(d+1) for d >= 2).  Deeper P2P rollbacks can exceed that; the shortage rule then trades
// witnesses for slots, so capture never makes a push fail that the plain ring would have served.
//
// Retention (bgr_retain_confirmed, set_retention(interval, count)): P2P desync detection compares the checksums of the
// confirmed frames 0, interval, 2*interval, ... between peers, and the report arrives a round trip after confirm() has
// dropped the frame.  So a frame f >= 0 with f % interval == 0 that leaves the queue from the OLD end (confirm, or the
// depth eviction in push) keeps its slot as a RETAINED frame instead of freeing it.
//   - Only the old end counts: a frame dropped from the new end (rollback, the re-save of an equal or older frame) was
//     not final.
//   - At most `count` frames are retained; the one retained first is released first.
//   - A push of a retained frame's number releases the stale copy; release_retained() (bgr_reset_session) releases all.
//   - The queue (get / peek / frames) is exactly the plain ring's, and a push never fails where the plain ring would
//     succeed: the engine allocates `count` extra slots and at most `count` are ever retained.
//   - slot_rows / slot_elapsed_ns / slot_rng are indexed by slot, so a retained frame keeps its row count, time and RNG.
// A retained slot is never handed to a Save, so it is never written again until it is released.  That is why the
// deferred live image (BGR_TUNE_DEFER_LIVE) may keep reading the base slot of the last Save even when that Save's own
// frame gets retained (a depth-1 ring retains it at the next push): the bytes the deferred image is rebuilt from stay
// as they were, exactly as if the slot had been freed and not yet reused.
#pragma once
#include <array>
#include <cstdint>
#include <string>
#include <vector>

namespace bgr {

// Fixed capacity (kMaxSlots), trivially copyable: handle_requests validates a request vector against a COPY of
// the host state, so copying the ring must not allocate on the hot path.
class SlotRing {
public:
    static constexpr uint32_t kNoSlot = 0xFFFFFFFFu;
    static constexpr uint32_t kMaxSlots = 64;

    explicit SlotRing(uint32_t n_slots = 0) { reset(n_slots); }

    void reset(uint32_t n_slots, bool capture = false) {
        n_slots_ = n_slots > kMaxSlots ? kMaxSlots : n_slots;
        capture_ = capture;
        entries_.n = 0;
        free_.n = 0;
        witnesses_.n = 0;
        retained_.n = 0;
        retain_interval_ = 0;
        retain_count_ = 0;
        for (uint32_t s = n_slots_; s-- > 0;) free_.push_back(s);
        depth_ = 60;  // DEFAULT_FPS until sync_depth runs (mod.rs:112)
    }

    uint32_t depth() const { return depth_; }
    void set_depth(uint32_t d) { depth_ = d; }  // mod.rs:120-135 (no eviction until the next push)
    uint32_t len() const { return entries_.size(); }
    uint32_t n_slots() const { return n_slots_; }

    // Returns the slot that now holds `frame`, or kNoSlot if more than n_slots snapshots would
    // have to be alive at once (configuration error, reported by the caller).
    uint32_t push(int32_t frame) {
        for (uint32_t i = 0; i < retained_.size(); ++i)  // the stale retained copy of this frame
            if (retained_[i].frame == frame) { release_retained_at(i); break; }
        // entries_ is oldest-first; the reference's "front" is our back()
        while (!entries_.empty() && !is_older(entries_.back().frame, frame)) release_back();
        // the entries that `while len > depth` would evict after the insert can go first:
        // the final queue is identical and their slots become reusable for this push
        while (!entries_.empty() && entries_.size() + 1 > depth_) release_front();
        if (depth_ == 0) return kNoSlot - 1;  // pushed and immediately evicted: nothing is stored
        while (free_.empty() && !witnesses_.empty()) release_witness(0);  // capture only: shortage rule
        if (free_.empty()) return kNoSlot;
        uint32_t s = free_.back();
        free_.pop_back();
        entries_.push_back({frame, s});
        if (capture_ && find_witness(frame) == kNoSlot) witnesses_.push_back({frame, s});
        return s;
    }

    void confirm(int32_t confirmed_frame) {
        while (!entries_.empty() && entries_.front().frame < confirmed_frame) release_front();
        for (uint32_t i = 0; i < witnesses_.size();) {
            if (witnesses_[i].frame < confirmed_frame) release_witness(i);
            else ++i;
        }
    }

    bool capture() const { return capture_; }
    void release_witnesses() { while (!witnesses_.empty()) release_witness(0); }
    // the slot of `frame`'s first-recorded image (capture rings only)
    bool first(int32_t frame, uint32_t* slot) const {
        uint32_t i = find_witness(frame);
        if (i == kNoSlot) return false;
        *slot = witnesses_[i].slot;
        return true;
    }
    // queued frames whose first-recorded image is a different slot (re-saved since), newest first
    void desync_frames(std::vector<int32_t>* out) const {
        out->clear();
        for (uint32_t i = entries_.size(); i-- > 0;) {
            uint32_t w = find_witness(entries_[i].frame);
            if (w != kNoSlot && witnesses_[w].slot != entries_[i].slot) out->push_back(entries_[i].frame);
        }
    }
    uint32_t slots_in_use() const { return n_slots_ - free_.size(); }

    // retention (see the header comment); count == 0 turns it off
    void set_retention(uint32_t interval, uint32_t count) {
        release_retained();
        retain_interval_ = interval;
        retain_count_ = count;
    }
    uint32_t retain_count() const { return retain_count_; }
    void release_retained() { while (!retained_.empty()) release_retained_at(0); }
    bool retained(int32_t frame, uint32_t* slot) const {
        for (uint32_t i = 0; i < retained_.size(); ++i)
            if (retained_[i].frame == frame) { *slot = retained_[i].slot; return true; }
        return false;
    }
    // retained frames, the most recently retained first
    void retained_frames(std::vector<int32_t>* out) const {
        out->clear();
        for (uint32_t i = retained_.size(); i-- > 0;) out->push_back(retained_[i].frame);
    }

    // bgr_checkpoint_restore: forget every queued frame, witness and retained frame, then push `frame` alone.  Depth,
    // capture and the retention setting stay.  Returns push()'s slot.
    uint32_t restart(int32_t frame) {
        entries_.n = 0;
        witnesses_.n = 0;
        retained_.n = 0;
        free_.n = 0;
        for (uint32_t s = n_slots_; s-- > 0;) free_.push_back(s);
        return push(frame);
    }

    // false => the reference would panic; `error` gets the same text
    bool rollback(int32_t frame, std::string* error) {
        for (;;) {
            if (entries_.empty()) {
                if (error)
                    *error = "Could not rollback to " + std::to_string(frame) +
                             ": no snapshot at that moment could be found.";
                return false;
            }
            if (entries_.back().frame != frame) release_back();
            else return true;
        }
    }

    bool get(uint32_t* slot, std::string* error) const {
        if (entries_.empty()) {
            if (error) *error = "no snapshot available — call rollback(frame) before get()";
            return false;
        }
        *slot = entries_.back().slot;
        return true;
    }

    bool peek(int32_t frame, uint32_t* slot) const {
        for (uint32_t i = entries_.size(); i-- > 0;)  // newest first, like the reference's iter()
            if (entries_[i].frame == frame) { *slot = entries_[i].slot; return true; }
        return false;
    }

    // newest first
    void frames(std::vector<int32_t>* out) const {
        out->clear();
        for (uint32_t i = entries_.size(); i-- > 0;) out->push_back(entries_[i].frame);
    }

private:
    struct Entry { int32_t frame; uint32_t slot; };

    // "stored is strictly older than incoming" == NOT (current_after_frame || current_after_frame_wrapped), mod.rs:156-161
    static bool is_older(int32_t stored, int32_t incoming) {
        int64_t diff = int64_t(stored) - int64_t(incoming);
        uint32_t ad = uint32_t(diff < 0 ? -diff : diff);
        bool wrapped = ad > (UINT32_MAX / 2);
        bool after = stored >= incoming && !wrapped;
        bool after_wrapped = incoming >= stored && wrapped;
        return !(after || after_wrapped);
    }
    // tiny inline vector: no heap, trivially copyable
    template <class T>
    struct Small {
        std::array<T, kMaxSlots> a;
        uint32_t n = 0;
        bool empty() const { return n == 0; }
        uint32_t size() const { return n; }
        T& back() { return a[n - 1]; }
        const T& back() const { return a[n - 1]; }
        T& front() { return a[0]; }
        const T& front() const { return a[0]; }
        T& operator[](uint32_t i) { return a[i]; }
        const T& operator[](uint32_t i) const { return a[i]; }
        void push_back(const T& v) { a[n++] = v; }
        void pop_back() { --n; }
        void pop_front() { for (uint32_t i = 1; i < n; ++i) a[i - 1] = a[i]; --n; }
        void erase(uint32_t k) { for (uint32_t i = k + 1; i < n; ++i) a[i - 1] = a[i]; --n; }
    };
    uint32_t find_witness(int32_t frame) const {
        for (uint32_t i = 0; i < witnesses_.size(); ++i)
            if (witnesses_[i].frame == frame) return i;
        return kNoSlot;
    }
    bool pinned(uint32_t slot) const {  // a witness or a retained frame holds the slot
        for (uint32_t i = 0; i < witnesses_.size(); ++i)
            if (witnesses_[i].slot == slot) return true;
        for (uint32_t i = 0; i < retained_.size(); ++i)
            if (retained_[i].slot == slot) return true;
        return false;
    }
    bool queued(uint32_t slot) const {
        for (uint32_t i = 0; i < entries_.size(); ++i)
            if (entries_[i].slot == slot) return true;
        return false;
    }
    void release_witness(uint32_t i) {
        const uint32_t s = witnesses_[i].slot;
        witnesses_.erase(i);
        if (!queued(s)) free_.push_back(s);
    }
    // dropping from the new end keeps the frame's witness (a SyncTest Load and its re-saves do exactly that)
    void release_back() {
        const uint32_t s = entries_.back().slot;
        entries_.pop_back();
        if (!pinned(s)) free_.push_back(s);
    }
    // dropping from the old end (depth, confirm) releases the frame's witness too
    void release_front() {
        const Entry e = entries_.front();
        entries_.pop_front();
        const uint32_t w = find_witness(e.frame);
        if (w != kNoSlot && witnesses_[w].slot != e.slot) release_witness(w);
        else if (w != kNoSlot) witnesses_.erase(w);  // the witness is this entry's own slot, freed below
        if (retain_count_ && e.frame >= 0 && e.frame % int64_t(retain_interval_) == 0) {
            retained_.push_back(e);
            if (retained_.size() > retain_count_) release_retained_at(0);
            return;
        }
        if (!pinned(e.slot)) free_.push_back(e.slot);
    }
    void release_retained_at(uint32_t i) {
        const uint32_t s = retained_[i].slot;
        retained_.erase(i);
        if (!queued(s) && !pinned(s)) free_.push_back(s);
    }

    Small<Entry> entries_;  // oldest first; depth is small (<= 64), O(depth) per operation
    Small<uint32_t> free_;
    Small<Entry> witnesses_;  // capture rings: (frame, slot of its first-recorded image), in the order recorded
    Small<Entry> retained_;   // retention: (frame, slot) that left from the old end, in the order retained
    uint32_t retain_interval_ = 0, retain_count_ = 0;
    uint32_t n_slots_ = 0;
    uint32_t depth_ = 60;
    bool capture_ = false;
};

}  // namespace bgr
