// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/seahash.hpp header).
//
// CPU restatement of `GgrsSnapshots<For, As>` — the newest-first ring of per-frame
// snapshots (reference src/snapshot/mod.rs:94-271).
//   push      mod.rs:144-178   (pops stored frames >= frame, i32-wrap aware, then evicts beyond depth)
//   confirm   mod.rs:182-199   (pops oldest while frame < confirmed)
//   rollback  mod.rs:207-223   (pops newest until == frame, else panics
//                               "Could not rollback to {frame}: no snapshot at that moment could be found.")
//   get       mod.rs:226-230
//   peek      mod.rs:233-240
//   set_depth mod.rs:120-135, default depth = DEFAULT_FPS = 60 (mod.rs:112, lib.rs:58)
// PINNING: the reference's own 11 unit tests (mod.rs:365-508) are ported verbatim in
// tests/test_ring_kats.py and run against this class through oracle_capi.
#pragma once
#include <cstdint>
#include <cstdlib>
#include <deque>
#include <stdexcept>
#include <string>

namespace oracle {

struct RollbackPanic : std::runtime_error {
    using std::runtime_error::runtime_error;
};

template <class As>
struct GgrsSnapshots {
    std::deque<As> snapshots;     // newest at the front
    std::deque<int32_t> frames;   // newest at the front
    size_t depth = 60;

    GgrsSnapshots& set_depth(size_t d) { depth = d; return *this; }
    // every stored frame dropped, the depth kept (a checkpoint restore starts the ring again)
    GgrsSnapshots& clear() { snapshots.clear(); frames.clear(); return *this; }

    static uint32_t abs_diff(int32_t a, int32_t b) {
        int64_t x = int64_t(a) - int64_t(b);
        return uint32_t(x < 0 ? -x : x);
    }

    GgrsSnapshots& push(int32_t frame, As snapshot) {
        while (!frames.empty()) {
            int32_t current = frames.front();
            bool wrapped = abs_diff(current, frame) > (UINT32_MAX / 2);
            bool current_after_frame = current >= frame && !wrapped;
            bool current_after_frame_wrapped = frame >= current && wrapped;
            if (current_after_frame || current_after_frame_wrapped) {
                snapshots.pop_front();
                frames.pop_front();
            } else {
                break;
            }
        }
        snapshots.push_front(std::move(snapshot));
        frames.push_front(frame);
        while (snapshots.size() > depth) {
            snapshots.pop_back();
            frames.pop_back();
        }
        return *this;
    }

    GgrsSnapshots& confirm(int32_t confirmed_frame) {
        while (!frames.empty() && frames.back() < confirmed_frame) {
            snapshots.pop_back();
            frames.pop_back();
        }
        return *this;
    }

    GgrsSnapshots& rollback(int32_t frame) {
        for (;;) {
            if (frames.empty())
                throw RollbackPanic("Could not rollback to " + std::to_string(frame) +
                                    ": no snapshot at that moment could be found.");
            if (frames.front() != frame) {
                snapshots.pop_front();
                frames.pop_front();
            } else {
                break;
            }
        }
        return *this;
    }

    As& get() {
        if (snapshots.empty())
            throw RollbackPanic("no snapshot available — call rollback(frame) before get()");
        return snapshots.front();
    }

    As* peek(int32_t frame) {
        for (size_t i = 0; i < frames.size(); ++i)
            if (frames[i] == frame) return &snapshots[i];
        return nullptr;
    }
};

}  // namespace oracle
