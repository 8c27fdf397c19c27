// The host checks of a checkpoint delta (csrc/checkpoint_check.hpp checkpoint_delta_check, which
// bgr_checkpoint_restore_delta runs before anything is uploaded): every malformed header and offsets case is refused
// with the status and message the restore gives, and well-formed deltas (written here in the delta format of
// include/bevy_ggrs_b200.h: header, u64 offsets[n_blocks + 1], payload) are accepted with their header and offsets.
// Host only: exit code 0 = passed.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../bevy_ggrs_b200/csrc/checkpoint_check.hpp"

using namespace bgr;

static int g_failed = 0, g_cases = 0;
#define EXPECT(cond, what)                                                                                   \
    do {                                                                                                     \
        ++g_cases;                                                                                           \
        if (!(cond)) { std::printf("  FAILED %s:%d: %s (%s)\n", __FILE__, __LINE__, #cond, what); ++g_failed; } \
    } while (0)

static const uint64_t kLayout = 0x1234567890ABCDEFull;

// the header of the base checkpoint the deltas below are written against
static bgr_checkpoint_header base_header(uint32_t words, uint32_t rows) {
    bgr_checkpoint_header h{};
    h.magic = BGR_CHECKPOINT_MAGIC;
    h.version = BGR_CHECKPOINT_VERSION;
    h.layout = kLayout;
    h.frame = 40;
    h.rows = rows;
    h.words = words;
    h.n_blocks = (rows + 511) / 512;
    h.n_columns = 3;
    h.fps = 60;
    h.digest_root = 0xFEEDFACECAFEBEEFull;
    return h;
}

// a delta of `rows` rows against `base` whose blocks take `block_bytes[b]` payload bytes (the payload is never read)
static std::vector<uint8_t> delta(const bgr_checkpoint_header& base, uint32_t rows, const std::vector<uint64_t>& block_bytes,
                                  uint32_t fps = 60) {
    bgr_checkpoint_delta_header h{};
    h.magic = BGR_CHECKPOINT_DELTA_MAGIC;
    h.version = BGR_CHECKPOINT_DELTA_VERSION;
    h.layout = kLayout;
    h.frame = 44;
    h.rows = rows;
    h.base_frame = base.frame;
    h.base_rows = base.rows;
    h.words = base.words;
    h.n_blocks = uint32_t(block_bytes.size());
    h.n_columns = 3;
    h.fps = fps;
    h.base_root = base.digest_root;
    std::vector<uint64_t> off{0};
    for (uint64_t b : block_bytes) off.push_back(off.back() + b);
    h.payload_bytes = off.back();
    std::vector<uint8_t> out(sizeof h + sizeof(uint64_t) * off.size() + h.payload_bytes, 0);
    std::memcpy(out.data(), &h, sizeof h);
    std::memcpy(out.data() + sizeof h, off.data(), sizeof(uint64_t) * off.size());
    return out;
}

static bgr_checkpoint_delta_header* hdr(std::vector<uint8_t>& b) { return reinterpret_cast<bgr_checkpoint_delta_header*>(b.data()); }
static uint64_t* offs(std::vector<uint8_t>& b) { return reinterpret_cast<uint64_t*>(b.data() + sizeof(bgr_checkpoint_delta_header)); }

static void refused(const CkptTarget& t, const bgr_checkpoint_header& base, const std::vector<uint8_t>& b, size_t bytes,
                    int status, const char* text) {
    bgr_checkpoint_delta_header h;
    std::vector<uint64_t> o;
    std::string err;
    const int rc = checkpoint_delta_check(t, base, b.data(), bytes, &h, &o, &err);
    EXPECT(rc == status, text);
    EXPECT(err.find(text) != std::string::npos, (err + " lacks: " + text).c_str());
}

static void accepted(const CkptTarget& t, const bgr_checkpoint_header& base, std::vector<uint8_t> b) {
    bgr_checkpoint_delta_header h;
    std::vector<uint64_t> o;
    std::string err;
    const int rc = checkpoint_delta_check(t, base, b.data(), b.size(), &h, &o, &err);
    EXPECT(rc == BGR_OK, err.c_str());
    EXPECT(std::memcmp(&h, b.data(), sizeof h) == 0, "the header");
    EXPECT(o.size() == size_t(h.n_blocks) + 1u && std::memcmp(o.data(), offs(b), sizeof(uint64_t) * o.size()) == 0, "the offsets");
    EXPECT(checkpoint_delta_prefix(h.n_blocks) + h.payload_bytes == b.size(), "the prefix");
}

int main() {
    static_assert(sizeof(bgr_checkpoint_delta_header) == 120, "the delta header is 120 bytes");
    for (uint32_t words : {1u, 3u, 15u}) {
        const uint64_t min_block = uint64_t(ckpt_kind_words(words) + words + 1u) * 4u;
        const uint64_t max_block = uint64_t(ckpt_max_block_words(words)) * 4u;
        const CkptTarget fixed{kLayout, words, 3u, 60u, 4096u, false}, growable{kLayout, words, 3u, 60u, 1u << 20, true};
        const bgr_checkpoint_header base = base_header(words, 1500), empty = base_header(words, 0);
        // accepted: fewer, equal and more rows than the base, an empty base or target, both bounds of a block's size
        accepted(fixed, base, delta(base, 1500, {max_block, min_block, min_block + 4u * words}));
        accepted(fixed, base, delta(base, 0, {min_block, min_block, min_block}));
        accepted(fixed, base, delta(base, 700, {min_block, max_block, min_block}));
        accepted(fixed, base, delta(base, 4096, std::vector<uint64_t>(8, max_block)));
        accepted(fixed, empty, delta(empty, 0, {}));
        accepted(fixed, empty, delta(empty, 513, {min_block, min_block}));
        accepted(growable, base, delta(base, 5000, std::vector<uint64_t>(10, min_block)));

        const std::vector<uint8_t> good = delta(base, 1200, {max_block, min_block, min_block + 8u});
        std::vector<uint8_t> b;
        refused(fixed, base, good, sizeof(bgr_checkpoint_delta_header) - 1, BGR_ERR_INVALID_ARGUMENT, "shorter than its header");
        refused(fixed, base, good, 0, BGR_ERR_INVALID_ARGUMENT, "shorter than its header");
        b = good; hdr(b)->magic = BGR_CHECKPOINT_MAGIC;  // a full checkpoint is not a delta
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "not a checkpoint delta (bad magic)");
        b = good; hdr(b)->version = 2;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "unsupported checkpoint delta format version 2");
        b = good; hdr(b)->layout ^= 1u;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "different registration (layout differs)");
        b = good; hdr(b)->words += 1;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "different registration (layout differs)");
        b = good; hdr(b)->n_columns = 4;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "different registration (layout differs)");
        b = delta(base, 1200, {max_block, min_block, min_block}, 144);
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "the checkpoint delta was taken at 144 fps, this engine runs at 60");
        b = good; hdr(b)->base_frame += 1;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "written against another base");
        b = good; hdr(b)->base_root ^= 1u;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "written against another base");
        b = good; hdr(b)->base_rows = 1400;  // same block count, another base
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "written against another base");
        b = good; hdr(b)->rows = 1537;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "n_blocks does not match rows and base_rows");
        b = good; hdr(b)->n_blocks = 2;  // the target's own block count: the base's third block is missing
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "n_blocks does not match rows and base_rows");
        b = delta(base, 4097, std::vector<uint64_t>(9, min_block));
        refused(fixed, base, b, b.size(), BGR_ERR_CAPACITY, "holds 4097 rows, more than this engine's capacity of 4096");
        b = delta(base, (1u << 20) + 1u, std::vector<uint64_t>(2049, min_block));
        refused(growable, base, b, b.size(), BGR_ERR_CAPACITY, "more than this engine's ceiling of 1048576");
        b = good;
        refused(fixed, base, b, sizeof(bgr_checkpoint_delta_header) + 8u * 3u, BGR_ERR_INVALID_ARGUMENT, "shorter than its block offsets");
        refused(fixed, base, b, b.size() - 4u, BGR_ERR_INVALID_ARGUMENT, "does not match its payload (truncated or overlong)");
        b.resize(b.size() + 8u);
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "does not match its payload (truncated or overlong)");
        b = good; offs(b)[0] = 4;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offsets do not span the payload");
        b = good; offs(b)[3] -= 4;
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offsets do not span the payload");
        b = good; offs(b)[1] += 2;  // unaligned
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offset 1 is not ascending, aligned or within a block's size");
        b = good; offs(b)[2] = offs(b)[1] + min_block - 4u;  // a block below every vector CONST
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offset 2 is not ascending");
        b = good; offs(b)[2] = offs(b)[1] - 4u;  // descending
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offset 2 is not ascending");
        b = delta(base, 1200, {max_block + 4u, min_block, min_block});  // a block past every vector RAW
        refused(fixed, base, b, b.size(), BGR_ERR_INVALID_ARGUMENT, "checkpoint delta offset 1 is not ascending");
    }
    if (g_failed) {
        std::printf("%d of %d checks failed\n", g_failed, g_cases);
        return 1;
    }
    std::printf("checkpoint delta host check test passed (%d checks)\n", g_cases);
    return 0;
}
