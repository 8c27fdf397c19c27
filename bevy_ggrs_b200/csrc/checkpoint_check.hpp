// World checkpoints: the host checks of a blob's header and block offsets against the engine it is restored into, made
// before anything is uploaded (bgr_checkpoint_restore and bgr_batch_checkpoint_restore), and those of a checkpoint delta
// against the engine and its base checkpoint (bgr_checkpoint_restore_delta).  Host only;
// tests/cpp/test_checkpoint_check.cpp and tests/cpp/test_checkpoint_delta_check.cpp hold them to every refusal of the
// restores with its status.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/bevy_ggrs_b200.h"
#include "checkpoint.cuh"  // ckpt_kind_words, ckpt_max_block_words

namespace bgr {

// What a blob has to match: the registration layout (with order_base), fps and capacity of the engine restored into
struct CkptTarget {
    uint64_t layout;
    uint32_t words, n_columns, fps;
    uint64_t ceiling;  // the most rows the engine can hold (a growable engine's ceiling)
    bool growable;
};

// bytes ahead of the payload: the header and the offsets
inline size_t checkpoint_prefix(uint32_t n_blocks) {
    return sizeof(bgr_checkpoint_header) + sizeof(uint64_t) * (size_t(n_blocks) + 1u);
}

// The block offsets of a blob (`what`: "checkpoint" or "checkpoint delta"), read from `in`: they start at 0, end at
// payload_bytes, and each block lies within a block's size bounds in multiples of 4.
inline int checkpoint_offsets_check(uint32_t words, uint32_t n_blocks, uint64_t payload_bytes, const uint8_t* in,
                                    const char* what, std::vector<uint64_t>* offsets, std::string* err) {
    offsets->resize(size_t(n_blocks) + 1u);
    std::memcpy(offsets->data(), in, sizeof(uint64_t) * offsets->size());
    const std::vector<uint64_t>& o = *offsets;
    // a block is at least its kind bytes and one u32 per vector (every vector CONST) and at most every vector RAW.  The
    // lower bound also bounds the scratch image the decoding allocates by the blob's size: a tile of the image is at
    // most tile_bytes / min_block times the smallest block (390x for the stress schema), and only a world that is
    // constant in every tile gets there.
    const uint64_t max_block = uint64_t(ckpt_max_block_words(words)) * 4u;
    const uint64_t min_block = uint64_t(ckpt_kind_words(words) + words + 1u) * 4u;
    if (o[0] != 0 || o[n_blocks] != payload_bytes) {
        *err = std::string(what) + " offsets do not span the payload";
        return BGR_ERR_INVALID_ARGUMENT;
    }
    for (uint32_t b = 0; b < n_blocks; ++b)
        if (o[b + 1] < o[b] + min_block || o[b + 1] % 4u || o[b + 1] - o[b] > max_block) {
            *err = std::string(what) + " offset " + std::to_string(b + 1) + " is not ascending, aligned or within a block's size";
            return BGR_ERR_INVALID_ARGUMENT;
        }
    return BGR_OK;
}

// Checks `bytes` bytes of `blob` (untrusted input from disk or another machine) field by field.  BGR_OK: *h and
// *offsets ([n_blocks + 1]) hold the blob's, and its payload lies at blob + checkpoint_prefix(h->n_blocks).  Otherwise
// the status and *err say why.
inline int checkpoint_check(const CkptTarget& t, const void* blob, size_t bytes, bgr_checkpoint_header* h,
                            std::vector<uint64_t>* offsets, std::string* err) {
    auto refuse = [err](int status, const std::string& why) { *err = why; return status; };
    const uint8_t* in = static_cast<const uint8_t*>(blob);
    if (bytes < sizeof *h) return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its header");
    std::memcpy(h, in, sizeof *h);
    if (h->magic != BGR_CHECKPOINT_MAGIC) return refuse(BGR_ERR_INVALID_ARGUMENT, "not a world checkpoint (bad magic)");
    if (h->version != BGR_CHECKPOINT_VERSION)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "unsupported checkpoint format version " + std::to_string(h->version));
    if (h->layout != t.layout || h->words != t.words || h->n_columns != t.n_columns)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "the checkpoint comes from an engine with a different registration (layout differs)");
    if (h->fps != t.fps)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "the checkpoint was taken at " + std::to_string(h->fps) + " fps, this engine runs at " +
                                                    std::to_string(t.fps));
    if (h->n_blocks != (h->rows + kTileRows - 1) / kTileRows)  // u32, as bgr_engine::tiles_for
        return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint header: n_blocks does not match rows");
    if (h->rows > t.ceiling)
        return refuse(BGR_ERR_CAPACITY, "the checkpoint holds " + std::to_string(h->rows) + " rows, more than this engine's " +
                                            (t.growable ? "ceiling of " : "capacity of ") + std::to_string(t.ceiling));
    const uint32_t n_blocks = h->n_blocks;
    const size_t prefix = checkpoint_prefix(n_blocks);
    if (bytes < prefix) return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint truncated: shorter than its block offsets");
    if (bytes - prefix != h->payload_bytes)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint length " + std::to_string(bytes) +
                                                    " does not match its payload (truncated or overlong)");
    return checkpoint_offsets_check(t.words, n_blocks, h->payload_bytes, in + sizeof *h, "checkpoint", offsets, err);
}

// bytes ahead of a delta's payload: the header and the offsets
inline size_t checkpoint_delta_prefix(uint32_t n_blocks) {
    return sizeof(bgr_checkpoint_delta_header) + sizeof(uint64_t) * (size_t(n_blocks) + 1u);
}

// Checks `bytes` bytes of the delta `blob` against the engine and the header of the base checkpoint it is applied to
// (which checkpoint_check has accepted for the same engine).  BGR_OK: *h and *offsets ([n_blocks + 1]) hold the delta's,
// and its payload lies at blob + checkpoint_delta_prefix(h->n_blocks).  Otherwise the status and *err say why.
inline int checkpoint_delta_check(const CkptTarget& t, const bgr_checkpoint_header& base, const void* blob, size_t bytes,
                                  bgr_checkpoint_delta_header* h, std::vector<uint64_t>* offsets, std::string* err) {
    auto refuse = [err](int status, const std::string& why) { *err = why; return status; };
    const uint8_t* in = static_cast<const uint8_t*>(blob);
    if (bytes < sizeof *h) return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta truncated: shorter than its header");
    std::memcpy(h, in, sizeof *h);
    if (h->magic != BGR_CHECKPOINT_DELTA_MAGIC) return refuse(BGR_ERR_INVALID_ARGUMENT, "not a checkpoint delta (bad magic)");
    if (h->version != BGR_CHECKPOINT_DELTA_VERSION)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "unsupported checkpoint delta format version " + std::to_string(h->version));
    if (h->layout != t.layout || h->words != t.words || h->n_columns != t.n_columns)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "the checkpoint delta comes from an engine with a different registration (layout differs)");
    if (h->fps != t.fps)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "the checkpoint delta was taken at " + std::to_string(h->fps) + " fps, this engine runs at " +
                                                    std::to_string(t.fps));
    if (h->base_frame != base.frame || h->base_rows != base.rows || h->base_root != base.digest_root)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "the checkpoint delta was written against another base (base frame " +
                                                    std::to_string(h->base_frame) + ", the base checkpoint holds frame " +
                                                    std::to_string(base.frame) + ")");
    if (h->n_blocks != (std::max(h->rows, h->base_rows) + kTileRows - 1) / kTileRows)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta header: n_blocks does not match rows and base_rows");
    if (h->rows > t.ceiling)
        return refuse(BGR_ERR_CAPACITY, "the checkpoint delta holds " + std::to_string(h->rows) + " rows, more than this engine's " +
                                            (t.growable ? "ceiling of " : "capacity of ") + std::to_string(t.ceiling));
    const size_t prefix = checkpoint_delta_prefix(h->n_blocks);
    if (bytes < prefix) return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta truncated: shorter than its block offsets");
    if (bytes - prefix != h->payload_bytes)
        return refuse(BGR_ERR_INVALID_ARGUMENT, "checkpoint delta length " + std::to_string(bytes) +
                                                    " does not match its payload (truncated or overlong)");
    return checkpoint_offsets_check(t.words, h->n_blocks, h->payload_bytes, in + sizeof *h, "checkpoint delta", offsets, err);
}

}  // namespace bgr
