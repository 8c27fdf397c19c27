// World batches: the rule every bgr_batch_* call applies to the worlds it lists, each index in range and listed at most
// once per call.  Host only; tests/cpp/test_feed_check.cpp and tests/cpp/test_edit_batch.cpp hold it to its messages.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"

namespace bgr {

// The members of a batch a call has listed so far: member w is listed in the current call when listed[w] == calls, so
// beginning a call clears nothing.
class WorldList {
public:
    explicit WorldList(uint32_t n_members = 0) : listed_(n_members, 0u) {}

    // Starts a call: no member is listed in it yet
    void begin() {
        if (++calls_ == 0) {  // wrapped: a stamp from 2^32 calls ago must not read as this call's
            std::fill(listed_.begin(), listed_.end(), 0u);
            calls_ = 1;
        }
    }

    // Lists member w in the current call: BGR_OK, or BGR_ERR_INVALID_ARGUMENT with *err = why
    int admit(uint32_t w, std::string* err) {
        if (w >= listed_.size()) {
            *err = "no such world in a batch of " + std::to_string(listed_.size());
            return BGR_ERR_INVALID_ARGUMENT;
        }
        if (listed_[w] == calls_) { *err = "listed twice in one call"; return BGR_ERR_INVALID_ARGUMENT; }
        listed_[w] = calls_;
        return BGR_OK;
    }

private:
    std::vector<uint32_t> listed_;
    uint32_t calls_ = 0;
};

}  // namespace bgr
