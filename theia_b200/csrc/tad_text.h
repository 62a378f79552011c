// Text key slots of streamed host blocks (tad_stream_push_text): ClickHouse Native String column bytes decoded and
// dictionary-encoded on the device into job-stable u32 ids (implemented in tad_text.cu; DESIGN.md section 10).
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

#include <cuda_runtime.h>

namespace tad {

// The device dictionary of one text slot.  Open addressing over a 64-bit FNV-1a hash of the bytes: a slot holds
// (high 32 hash bits << 32) | ref, where ref is a name id, or kTextPending | row for a name first seen in the chunk being
// encoded.  A lookup compares the bytes whenever the tag matches.  Names are kept once each in `arena`, in id order:
// name k is arena[off[k], off[k + 1]).  state[0] = names, state[1] = arena bytes, state[2] = decode error flag,
// state[3..4] = the current chunk's new names / bytes, state[5] = a name was missing from a frozen dictionary.
struct TextDict {
    unsigned long long *slots;   // cap
    uint32_t *minrow;            // cap: smallest row of the chunk that reached a pending slot (UINT32_MAX: none)
    uint32_t *slot_id;           // cap: the id a pending slot's first row published
    uint32_t cap;                // power of two
    uint8_t *arena;
    uint64_t *off;               // names + 1
    uint64_t *hash;              // names: each name's hash, for the rehash
    unsigned long long *state;   // 8 words
    uint32_t frozen;             // the dictionary is complete: a name not in it sets state[5] and is not added
    uint64_t hash_mask;          // ANDed into every name's hash: ~0, or narrower to make hashes collide (TAD_DEBUG_TEXT_MASK)
};

// Scratch of one chunk of `n` rows: per row (offset, length) into the staged text, the pending slot it reached, and the
// (new-name count << 40 | bytes) scan.  text_scratch_bytes(n) sizes it.
size_t text_scratch_bytes(uint64_t n);

// A fresh table of `cap` slots (every slot empty, minrow all ones).  Two launches.
cudaError_t launch_text_clear(cudaStream_t st, const TextDict &d);
// Every name of `old` (its `names` ids) re-inserted into the empty table `d` (same arena).  One launch.
cudaError_t launch_text_rehash(cudaStream_t st, const TextDict &old, const TextDict &d, uint64_t names);

// Rows [lo, lo + n) of a block, as the bytes of its 32-row segments s0 .. s0 + nseg - 1: `text` holds the span from
// the start of segment s0 (span_bytes), `marks` the block's marks of those segments (absolute, marks[0] = the span's
// start), block_rows the block's rows.  Each row's id (order of first appearance over the dictionary's life) goes to
// ids[0, n).  A segment whose VarUInt lengths do not end exactly at the next mark (or the span's end), or that would read
// past the span, sets state[2] and encodes its rows as the empty name.  Seven launches (two of them the CUB scan).
cudaError_t launch_text_encode(cudaStream_t st, const TextDict &d, const uint8_t *text, uint64_t span_bytes,
                               const uint64_t *marks, uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo,
                               uint64_t n, void *scratch, size_t scratch_bytes, uint32_t *ids);

constexpr uint32_t kTextPending = 0x80000000u;
constexpr int kTextLaunches = 7;

// Row predicates of a filtered streamed job (tad_stream_filter).  Name ops, as TAD_NAME_* of include/theia_tad.h:
constexpr int kNameAny = 0, kNameEq = 1, kNameNonEmpty = 2, kNameIContains = 3;
// A dropped row carries this bit in the id of the job's first text slot (ids are < 2^30); the split and pack kernels'
// marked instances drop it.
constexpr uint32_t kTextDropped = 0x80000000u;

// keep[id] = the predicate `op` / pattern (device memory) on name id, for the names the chunk just encoded added to `d`
// (ids [state[0] - state[3], state[0]); `n`, the chunk's rows, bounds their count).  Only while the dictionary is open.
// One launch.
cudaError_t launch_text_match(cudaStream_t st, const TextDict &d, uint8_t *keep, int op, const uint8_t *pat,
                              uint32_t pat_len, uint64_t n);

// One chunk's row predicates: a slot with keep[t] set fails a row whose name's keep byte is 0; proto_eq >= 0 fails a row
// whose proto byte differs.  A failed row gets kTextDropped in mark[i] (the first text slot's ids).  One launch.
struct TextMark {
    const uint32_t *ids[2];
    const uint8_t *keep[2];
    const uint8_t *proto;
    int32_t proto_eq;
    uint32_t *mark;
};
cudaError_t launch_text_mark(cudaStream_t st, const TextMark &m, uint64_t n);

// The namespace ignore list of a job whose namespace slots are text (tad_submit_stream_filtered_ns).  Its device image,
// built once per job on the host: kNsStateWords state words (slot t's decode error flag at word 8t + 2, as a TextDict's
// state[2]), then the names' 64-bit hashes in ascending order, the u32 offsets of their bytes (names + 1) and the bytes,
// padded to 8 bytes.  The kernel holds everything after the state words in shared memory.
constexpr uint32_t kNsMaxNames = 1024, kNsMaxBytes = 32768;
constexpr int kNsStateWords = 16;
// The verdict a namespace slot stages per row: the row filter's one-entry ignore list {kNsListed} drops listed rows.
constexpr uint32_t kNsListed = 1;
// `hash_mask` is ANDed into every hash (~0 in the engine; a narrow mask makes hashes collide, for the tests).
std::vector<uint8_t> ns_list_image(const uint8_t *bytes, const uint64_t *off, uint32_t names, uint64_t hash_mask);

// Rows [lo, lo + n) of a block's namespace text slot (staged as for launch_text_encode) -> verdict[i] = kNsListed when
// the row's name is in the list `image` (device memory, `names` names, `image_bytes` long), else 0.  A segment that does
// not decode sets state[2] (the slot's state words) and its rows read as the empty name.  Two launches; `scratch` as
// for launch_text_encode; `hash_mask` as the image was built with.
cudaError_t launch_ns_match(cudaStream_t st, const void *image, uint32_t names, size_t image_bytes, uint64_t hash_mask,
                            unsigned long long *state,
                            const uint8_t *text, uint64_t span_bytes, const uint64_t *marks, uint32_t nseg, uint64_t seg0_row,
                            uint64_t block_rows, uint64_t lo, uint64_t n, void *scratch, size_t scratch_bytes,
                            uint32_t *verdict);
constexpr int kNsLaunches = 2;

}  // namespace tad
