// Text key slots on the device (tad_text.h): decode of Native String column bytes, the job's dictionary of names, and
// the namespace ignore list tested on namespace text.
// A translation unit of its own, so that no existing kernel's unit gains a CUB instance or a constant.
#include <algorithm>
#include <cstring>

#include <cub/device/device_scan.cuh>

#include "../../include/theia_tad.h"
#include "tad_text.h"

namespace tad {

namespace {

constexpr unsigned long long kEmpty = ~0ull;
constexpr uint32_t kNone = 0xffffffffu;
constexpr uint64_t kByteBits = 40;           // scan word: new names << 40 | their bytes (a chunk has < 2^24 rows)
constexpr int kThreads = 256;

__host__ __device__ __forceinline__ uint64_t name_hash(const uint8_t *s, uint32_t len)
{
    uint64_t h = 1469598103934665603ull;     // FNV-1a, then a fold so that the low (slot) bits see the high bytes
    for (uint32_t k = 0; k < len; k++) h = (h ^ s[k]) * 1099511628211ull;
    return h ^ (h >> 29);
}

__host__ __device__ __forceinline__ bool same_bytes(const uint8_t *a, uint32_t na, const uint8_t *b, uint32_t nb)
{
    if (na != nb) return false;
    for (uint32_t k = 0; k < na; k++)
        if (a[k] != b[k]) return false;
    return true;
}

struct ChunkScratch {
    uint32_t *off, *len, *slot_of;
    unsigned long long *scan_in, *scan_out;
    void *cub_tmp;
    size_t cub_bytes;
};

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

size_t cub_scan_bytes(uint64_t n)
{
    size_t b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, b, (const unsigned long long *)nullptr, (unsigned long long *)nullptr, (int)n);
    return b;
}

ChunkScratch carve(void *scratch, uint64_t n)
{
    char *p = static_cast<char *>(scratch);
    ChunkScratch c;
    c.off = reinterpret_cast<uint32_t *>(p); p += align256(n * 4);
    c.len = reinterpret_cast<uint32_t *>(p); p += align256(n * 4);
    c.slot_of = reinterpret_cast<uint32_t *>(p); p += align256(n * 4);
    c.scan_in = reinterpret_cast<unsigned long long *>(p); p += align256(n * 8);
    c.scan_out = reinterpret_cast<unsigned long long *>(p); p += align256(n * 8);
    c.cub_tmp = p;
    c.cub_bytes = cub_scan_bytes(n);
    return c;
}

// One thread per 32-row segment: walk its rows' VarUInt lengths inside [mark, next mark) and record the (offset,
// length) of the rows in [lo, lo + n).  Every byte read is checked against the segment's end, which is checked against
// the span: a malformed column can set the error flag, never read outside the span.
__global__ void text_decode_kernel(const uint8_t *__restrict__ text, uint64_t span, const uint64_t *__restrict__ marks,
                                   uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo, uint64_t n,
                                   uint32_t *__restrict__ off, uint32_t *__restrict__ len, unsigned long long *state)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= nseg) return;
    const uint64_t base = marks[0];
    const uint64_t r0 = seg0_row + 32ull * k, r1 = min(r0 + 32, block_rows);
    uint64_t pos = marks[k] - base;
    const uint64_t end = k + 1 < nseg ? marks[k + 1] - base : span;
    bool ok = pos <= end && end <= span;
    for (uint64_t r = r0; ok && r < r1; r++) {
        uint64_t v = 0;
        int shift = 0;
        for (;;) {                                   // VarUInt: 7 bits per byte, least significant group first
            if (pos >= end || shift > 63) { ok = false; break; }
            const uint8_t b = text[pos++];
            v |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (!ok || v > end - pos) { ok = false; break; }
        if (r >= lo && r < lo + n) {
            off[r - lo] = (uint32_t)pos;
            len[r - lo] = (uint32_t)v;
        }
        pos += v;
    }
    ok = ok && pos == end;
    if (!ok) {
        atomicOr(state + 2, 1ull);
        for (uint64_t r = max(r0, lo); r < min(r1, lo + n); r++) {
            off[r - lo] = 0;
            len[r - lo] = 0;
        }
    }
}

// One thread per row: find the row's name.  A name with an id writes it; a new name claims an empty slot (or meets the
// row that claimed it in this chunk) and records its smallest row there.
__global__ void text_probe_kernel(TextDict d, const uint8_t *__restrict__ text, const uint32_t *__restrict__ off,
                                  const uint32_t *__restrict__ len, uint64_t n, uint32_t *__restrict__ slot_of,
                                  uint32_t *__restrict__ ids)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *s = text + off[i];
    const uint32_t m = len[i];
    const uint64_t h = name_hash(s, m) & d.hash_mask;
    const uint32_t tag = (uint32_t)(h >> 32), mask = d.cap - 1;
    uint32_t p = (uint32_t)h & mask;
    for (;;) {
        unsigned long long cur = *(volatile unsigned long long *)(d.slots + p);
        if (cur == kEmpty && d.frozen) {             // a later round's name the first round did not bring
            atomicOr(d.state + 5, 1ull);
            slot_of[i] = kNone;
            ids[i] = 0;
            return;
        }
        if (cur == kEmpty) {
            const unsigned long long mine = (unsigned long long)tag << 32 | kTextPending | (uint32_t)i;
            cur = atomicCAS(d.slots + p, kEmpty, mine);
            if (cur == kEmpty) {
                slot_of[i] = p;
                atomicMin(d.minrow + p, (uint32_t)i);
                return;
            }
        }
        if ((uint32_t)(cur >> 32) == tag) {
            const uint32_t ref = (uint32_t)cur;
            if (ref & kTextPending) {
                const uint32_t r = ref & ~kTextPending;
                if (same_bytes(s, m, text + off[r], len[r])) {
                    slot_of[i] = p;
                    atomicMin(d.minrow + p, (uint32_t)i);
                    return;
                }
            } else if (same_bytes(s, m, d.arena + d.off[ref], (uint32_t)(d.off[ref + 1] - d.off[ref]))) {
                slot_of[i] = kNone;
                ids[i] = ref;
                return;
            }
        }
        p = (p + 1) & mask;
    }
}

// The first row of each new name: (1 << 40 | its length), every other row 0.
__global__ void text_first_kernel(TextDict d, const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ len,
                                  uint64_t n, unsigned long long *__restrict__ scan_in)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t p = slot_of[i];
    scan_in[i] = p != kNone && d.minrow[p] == (uint32_t)i ? (1ull << kByteBits) | len[i] : 0ull;
}

// The first row of each new name takes id names + rank, copies its bytes to the arena and publishes the id in its slot.
__global__ void text_assign_kernel(TextDict d, const uint8_t *__restrict__ text, const uint32_t *__restrict__ off,
                                   const uint32_t *__restrict__ len, const uint32_t *__restrict__ slot_of,
                                   const unsigned long long *__restrict__ scan_in,
                                   const unsigned long long *__restrict__ scan_out, uint64_t n)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long x = scan_out[i], v = scan_in[i];
    if (i == n - 1) {
        d.state[3] = (x + v) >> kByteBits;
        d.state[4] = (x + v) & ((1ull << kByteBits) - 1);
    }
    if (!v) return;
    const uint32_t id = (uint32_t)(d.state[0] + (x >> kByteBits));
    const uint64_t at = d.state[1] + (x & ((1ull << kByteBits) - 1));
    const uint8_t *s = text + off[i];
    const uint32_t m = len[i];
    for (uint32_t k = 0; k < m; k++) d.arena[at + k] = s[k];
    d.off[id] = at;
    const uint64_t h = name_hash(s, m) & d.hash_mask;
    d.hash[id] = h;
    const uint32_t p = slot_of[i];
    d.slot_id[p] = id;
    d.slots[p] = (h >> 32) << 32 | id;
}

// Every row that reached a pending slot reads the id published there; the slot is reset for the next chunk.
__global__ void text_resolve_kernel(TextDict d, const uint32_t *__restrict__ slot_of, uint64_t n, uint32_t *__restrict__ ids)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        d.state[0] += d.state[3];
        d.state[1] += d.state[4];
        d.off[d.state[0]] = d.state[1];
    }
    if (i >= n) return;
    const uint32_t p = slot_of[i];
    if (p == kNone) return;
    ids[i] = d.slot_id[p];
    d.minrow[p] = kNone;
}

__global__ void text_rehash_kernel(TextDict d, const uint64_t *__restrict__ hash, uint64_t names)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= names) return;
    const uint64_t h = hash[k];
    const uint32_t mask = d.cap - 1;
    uint32_t p = (uint32_t)h & mask;
    const unsigned long long e = (h >> 32) << 32 | k;
    while (atomicCAS(d.slots + p, kEmpty, e) != kEmpty) p = (p + 1) & mask;
}

// Folded unit of s at byte k for the case-insensitive test (Python's str.lower() as far as it can meet an ASCII
// pattern): A-Z -> a-z; U+0130 (C4 B0) -> 'i' and then a non-ASCII unit (its U+0307); U+212A (E2 84 AA) -> 'k'; every
// other byte as it is.  `adv` = the bytes consumed; `last` = the unit ends the ASCII run (U+0130's combining dot follows).
__host__ __device__ __forceinline__ uint8_t fold_unit(const uint8_t *s, uint32_t n, uint32_t k, uint32_t &adv, bool &last)
{
    const uint8_t c = s[k];
    adv = 1;
    last = false;
    if (c >= 'A' && c <= 'Z') return (uint8_t)(c + 32);
    if (c == 0xC4 && k + 1 < n && s[k + 1] == 0xB0) { adv = 2; last = true; return 'i'; }
    if (c == 0xE2 && k + 2 < n && s[k + 1] == 0x84 && s[k + 2] == 0xAA) { adv = 3; return 'k'; }
    return c;
}

// pattern.lower() in name.lower() for a UTF-8 name and an ASCII pattern.  Lower-cased non-ASCII code points other than
// U+0130 and U+212A stay non-ASCII, so they can never meet a pattern byte and compare exactly.
__host__ __device__ __forceinline__ bool name_icontains(const uint8_t *s, uint32_t n, const uint8_t *p, uint32_t m)
{
    if (m == 0) return true;
    for (uint32_t start = 0; start < n; start++) {
        uint32_t k = start, j = 0;
        while (j < m && k < n) {
            uint32_t adv;
            bool last;
            const uint8_t u = fold_unit(s, n, k, adv, last);
            const uint8_t q = p[j] >= 'A' && p[j] <= 'Z' ? (uint8_t)(p[j] + 32) : p[j];
            if (u != q) break;
            j++;
            k += adv;
            if (last) break;
        }
        if (j == m) return true;
    }
    return false;
}

// The name predicate of a text slot (tad_stream_filter): TAD_NAME_ANY / EQ / NONEMPTY / ICONTAINS.
__host__ __device__ __forceinline__ bool name_match(int op, const uint8_t *s, uint32_t n, const uint8_t *p, uint32_t m)
{
    switch (op) {
    case kNameEq: return same_bytes(s, n, p, m);
    case kNameNonEmpty: return n > 0;
    case kNameIContains: return name_icontains(s, n, p, m);
    default: return true;
    }
}

// One thread per name the chunk may have added: the chunk's new names are ids [state[0] - state[3], state[0]).
__global__ void text_match_kernel(TextDict d, uint8_t *__restrict__ keep, int op, const uint8_t *__restrict__ pat,
                                  uint32_t pat_len, uint64_t n)
{
    const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint64_t names = d.state[0], added = d.state[3];
    if (k >= added) return;
    const uint64_t id = names - added + k;
    const uint64_t a = d.off[id];
    keep[id] = name_match(op, d.arena + a, (uint32_t)(d.off[id + 1] - a), pat, pat_len) ? 1 : 0;
}

__global__ void text_mark_kernel(TextMark m, uint64_t n)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool keep = m.proto_eq < 0 || m.proto[i] == (uint8_t)m.proto_eq;
    for (int t = 0; t < 2; t++)
        if (m.keep[t]) keep = keep && m.keep[t][m.ids[t][i]];
    if (!keep) m.mark[i] |= kTextDropped;
}

// Whether the name s (m bytes, hash h) is in an ignore list of `names` names sorted by hash: every entry whose hash
// equals h is compared byte for byte, so a hash collision never lists a name.
__host__ __device__ __forceinline__ bool ns_listed(uint32_t names, const uint64_t *hash, const uint32_t *off,
                                                   const uint8_t *bytes, const uint8_t *s, uint32_t m, uint64_t h)
{
    uint32_t lo = 0, hi = names;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (hash[mid] < h) lo = mid + 1; else hi = mid;
    }
    for (; lo < names && hash[lo] == h; lo++)
        if (same_bytes(s, m, bytes + off[lo], off[lo + 1] - off[lo])) return true;
    return false;
}

// Where an ignore list image's parts start, past its state words.
struct NsParts {
    size_t hash, off, bytes, end;
};
__host__ __device__ __forceinline__ NsParts ns_parts(uint32_t names, size_t nbytes)
{
    NsParts p;
    p.hash = 0;
    p.off = p.hash + (size_t)names * 8;
    p.bytes = p.off + ((size_t)names + 1) * 4;
    p.end = (p.bytes + nbytes + 7) & ~size_t(7);
    return p;
}

// One thread per row: the row's namespace (decoded into off / len) tested against the list, held in shared memory.
__global__ void ns_match_kernel(const uint64_t *__restrict__ list, uint32_t words, uint32_t names, uint64_t hash_mask,
                                const uint8_t *__restrict__ text, const uint32_t *__restrict__ off,
                                const uint32_t *__restrict__ len, uint64_t n, uint32_t *__restrict__ verdict)
{
    extern __shared__ uint64_t sh[];
    for (uint32_t k = threadIdx.x; k < words; k += blockDim.x) sh[k] = list[k];
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const NsParts p = ns_parts(names, 0);
    const char *b = reinterpret_cast<const char *>(sh);
    const uint8_t *s = text + off[i];
    const uint32_t m = len[i];
    const bool hit = ns_listed(names, reinterpret_cast<const uint64_t *>(b + p.hash), reinterpret_cast<const uint32_t *>(b + p.off),
                               reinterpret_cast<const uint8_t *>(b + p.bytes), s, m, name_hash(s, m) & hash_mask);
    verdict[i] = hit ? kNsListed : 0u;
}

unsigned grid(uint64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

}  // namespace

cudaError_t launch_text_match(cudaStream_t st, const TextDict &d, uint8_t *keep, int op, const uint8_t *pat,
                              uint32_t pat_len, uint64_t n)
{
    if (n == 0) return cudaSuccess;
    text_match_kernel<<<grid(n), kThreads, 0, st>>>(d, keep, op, pat, pat_len, n);
    return cudaGetLastError();
}

cudaError_t launch_text_mark(cudaStream_t st, const TextMark &m, uint64_t n)
{
    if (n == 0) return cudaSuccess;
    text_mark_kernel<<<grid(n), kThreads, 0, st>>>(m, n);
    return cudaGetLastError();
}

size_t text_scratch_bytes(uint64_t n)
{
    n = n ? n : 1;
    return 3 * align256(n * 4) + 2 * align256(n * 8) + align256(cub_scan_bytes(n));
}

cudaError_t launch_text_clear(cudaStream_t st, const TextDict &d)
{
    cudaError_t e = cudaMemsetAsync(d.slots, 0xff, (size_t)d.cap * sizeof(unsigned long long), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d.minrow, 0xff, (size_t)d.cap * sizeof(uint32_t), st);
    return e;
}

cudaError_t launch_text_rehash(cudaStream_t st, const TextDict &old, const TextDict &d, uint64_t names)
{
    if (!names) return cudaSuccess;
    text_rehash_kernel<<<grid(names), kThreads, 0, st>>>(d, old.hash, names);
    return cudaGetLastError();
}

cudaError_t launch_text_encode(cudaStream_t st, const TextDict &d, const uint8_t *text, uint64_t span_bytes,
                               const uint64_t *marks, uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo,
                               uint64_t n, void *scratch, size_t scratch_bytes, uint32_t *ids)
{
    if (n == 0) return cudaSuccess;
    if (scratch_bytes < text_scratch_bytes(n) || n >= (1ull << 24)) return cudaErrorInvalidValue;
    ChunkScratch c = carve(scratch, n);
    text_decode_kernel<<<(nseg + 127) / 128, 128, 0, st>>>(text, span_bytes, marks, nseg, seg0_row, block_rows, lo, n, c.off,
                                                          c.len, d.state);
    text_probe_kernel<<<grid(n), kThreads, 0, st>>>(d, text, c.off, c.len, n, c.slot_of, ids);
    text_first_kernel<<<grid(n), kThreads, 0, st>>>(d, c.slot_of, c.len, n, c.scan_in);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(c.cub_tmp, c.cub_bytes, c.scan_in, c.scan_out, (int)n, st);
    if (e != cudaSuccess) return e;
    text_assign_kernel<<<grid(n), kThreads, 0, st>>>(d, text, c.off, c.len, c.slot_of, c.scan_in, c.scan_out, n);
    text_resolve_kernel<<<grid(n), kThreads, 0, st>>>(d, c.slot_of, n, ids);
    return cudaGetLastError();
}

std::vector<uint8_t> ns_list_image(const uint8_t *bytes, const uint64_t *off, uint32_t names, uint64_t hash_mask)
{
    std::vector<uint32_t> order(names);
    std::vector<uint64_t> h(names);
    for (uint32_t k = 0; k < names; k++) {
        order[k] = k;
        h[k] = name_hash(bytes + off[k], (uint32_t)(off[k + 1] - off[k])) & hash_mask;
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return h[a] < h[b]; });
    const NsParts p = ns_parts(names, off[names] - off[0]);
    std::vector<uint8_t> img(kNsStateWords * 8 + p.end, 0);
    uint8_t *q = img.data() + kNsStateWords * 8;
    uint32_t at = 0;
    for (uint32_t j = 0; j < names; j++) {
        const uint32_t k = order[j], m = (uint32_t)(off[k + 1] - off[k]);
        memcpy(q + p.hash + 8 * j, &h[k], 8);
        memcpy(q + p.off + 4 * j, &at, 4);
        if (m) memcpy(q + p.bytes + at, bytes + off[k], m);
        at += m;
    }
    memcpy(q + p.off + 4 * names, &at, 4);
    return img;
}

cudaError_t launch_ns_match(cudaStream_t st, const void *image, uint32_t names, size_t image_bytes, uint64_t hash_mask,
                            unsigned long long *state,
                            const uint8_t *text, uint64_t span_bytes, const uint64_t *marks, uint32_t nseg, uint64_t seg0_row,
                            uint64_t block_rows, uint64_t lo, uint64_t n, void *scratch, size_t scratch_bytes,
                            uint32_t *verdict)
{
    if (n == 0) return cudaSuccess;
    const size_t held = image_bytes - kNsStateWords * 8;      // the hashes, offsets and bytes: a multiple of 8
    if (scratch_bytes < text_scratch_bytes(n) || n >= (1ull << 24) || names > kNsMaxNames ||
        held > ns_parts(kNsMaxNames, kNsMaxBytes).end)
        return cudaErrorInvalidValue;
    ChunkScratch c = carve(scratch, n);
    text_decode_kernel<<<(nseg + 127) / 128, 128, 0, st>>>(text, span_bytes, marks, nseg, seg0_row, block_rows, lo, n, c.off,
                                                          c.len, state);
    const uint64_t *list = reinterpret_cast<const uint64_t *>(static_cast<const char *>(image) + kNsStateWords * 8);
    ns_match_kernel<<<grid(n), kThreads, held, st>>>(list, (uint32_t)(held / 8), names, hash_mask, text, c.off, c.len, n,
                                                     verdict);
    return cudaGetLastError();
}

}  // namespace tad

// The device's name predicate run on the host, for the tests: 1 when `name` passes op / pattern, 0 when not, -1 for a bad op.
extern "C" int tad_debug_name_match(int op, const uint8_t *name, uint32_t name_len, const uint8_t *pattern,
                                    uint32_t pattern_len)
{
    if (op < tad::kNameAny || op > tad::kNameIContains) return -1;
    return tad::name_match(op, name, name_len, pattern, pattern_len) ? 1 : 0;
}

// The device's namespace ignore-list test run on the host, for the tests: 1 when `name` is one of the `names` names of
// the list (name k = bytes[offsets[k] .. offsets[k + 1])), else 0.  `hash_mask` is ANDed into every hash (~0: as the
// engine hashes; a narrow mask forces collisions).
extern "C" int tad_debug_ns_match(const uint8_t *name, uint32_t name_len, const uint8_t *bytes, const uint64_t *offsets,
                                  uint32_t names, uint64_t hash_mask)
{
    const std::vector<uint8_t> img = tad::ns_list_image(bytes, offsets, names, hash_mask);
    const uint8_t *q = img.data() + tad::kNsStateWords * 8;
    const tad::NsParts p = tad::ns_parts(names, 0);
    return tad::ns_listed(names, reinterpret_cast<const uint64_t *>(q + p.hash), reinterpret_cast<const uint32_t *>(q + p.off),
                          q + p.bytes, name, name_len, tad::name_hash(name, name_len) & hash_mask) ? 1 : 0;
}

// ---- the text kernels on one device, for the tests ---------------------------------------------------------------------
// A dictionary driven through launch_text_* as TextKeys drives it, with its own buffers and a hash mask, and the ignore
// list's device lookup with an explicit mask.  Every call synchronises before it returns.  Error codes as theia_tad.h:
// 0, -1 (TAD_ERR_INVALID_ARG: an argument the kernels cannot take safely), -2 (a CUDA error).

// The hash the dictionaries and the ignore list use.
extern "C" uint64_t tad_debug_name_hash(const uint8_t *bytes, uint32_t len) { return tad::name_hash(bytes, len); }

namespace {

struct DebugDict {
    int device;
    tad::TextDict d;
    uint64_t names = 0, bytes = 0;               // state[0], state[1] after the last encode
    uint64_t arena_cap = 0, names_cap = 0;       // arena bytes; names the off / hash arrays hold
};

cudaError_t debug_alloc_slots(tad::TextDict &d, uint32_t cap)
{
    d.slots = nullptr;
    d.minrow = d.slot_id = nullptr;
    d.cap = cap;
    cudaError_t e = cudaMalloc(&d.slots, (size_t)cap * 8);
    if (e == cudaSuccess) e = cudaMalloc(&d.minrow, (size_t)cap * 4);
    if (e == cudaSuccess) e = cudaMalloc(&d.slot_id, (size_t)cap * 4);
    if (e == cudaSuccess) e = tad::launch_text_clear(0, d);
    return e;
}

void debug_free_slots(tad::TextDict &d)
{
    cudaFree(d.slots);
    cudaFree(d.minrow);
    cudaFree(d.slot_id);
}

// *p (have bytes, of which `keep` are live) grown to at least `need` bytes
template <typename T> cudaError_t debug_grow(T *&p, size_t have, size_t need, size_t keep)
{
    if (need <= have) return cudaSuccess;
    T *q = nullptr;
    cudaError_t e = cudaMalloc(&q, need);
    if (e == cudaSuccess && keep) e = cudaMemcpy(q, p, keep, cudaMemcpyDeviceToDevice);
    if (e != cudaSuccess) {
        cudaFree(q);
        return e;
    }
    cudaFree(p);
    p = q;
    return cudaSuccess;
}

// The rows [lo, lo + n) lie inside the segments' rows and the block, and the offsets fit the kernels' u32.
bool debug_rows_ok(uint64_t span, uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo, uint64_t n)
{
    return n < (1ull << 24) && span < (1ull << 32) && seg0_row % 32 == 0 && lo >= seg0_row &&
           lo + n <= std::min<uint64_t>(seg0_row + 32ull * nseg, block_rows);
}

// The segments' marks and bytes copied to the device (marks first, text after, as the text staging holds them).
cudaError_t debug_stage(const uint8_t *text, uint64_t span, const uint64_t *marks, uint32_t nseg, uint64_t n, char *&buf,
                        void *&scratch, size_t &scratch_bytes)
{
    scratch_bytes = tad::text_scratch_bytes(n);
    const size_t at = tad::align256((size_t)nseg * 8 + 8);
    cudaError_t e = cudaMalloc(&buf, at + span + 1);
    if (e == cudaSuccess) e = cudaMalloc(&scratch, scratch_bytes);
    if (e == cudaSuccess && nseg) e = cudaMemcpy(buf, marks, (size_t)nseg * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && span) e = cudaMemcpy(buf + at, text, span, cudaMemcpyHostToDevice);
    return e;
}

}  // namespace

// A dictionary of `cap` slots (a power of two, >= 2) on `device`, every name's hash ANDed with hash_mask.
extern "C" int tad_debug_text_dict_new(int device, uint32_t cap, uint64_t hash_mask, void **out)
{
    if (!out || cap < 2 || (cap & (cap - 1))) return TAD_ERR_INVALID_ARG;
    *out = nullptr;
    if (cudaSetDevice(device) != cudaSuccess) return TAD_ERR_CUDA;
    DebugDict *h = new DebugDict();
    h->device = device;
    tad::TextDict &d = h->d;
    d.arena = nullptr;
    d.off = d.hash = nullptr;
    d.state = nullptr;
    d.frozen = 0;
    d.hash_mask = hash_mask;
    cudaError_t e = debug_alloc_slots(d, cap);
    if (e == cudaSuccess) e = cudaMalloc(&d.state, 64);
    if (e == cudaSuccess) e = cudaMemset(d.state, 0, 64);
    if (e == cudaSuccess) e = cudaMalloc(&d.off, 8);
    if (e == cudaSuccess) e = cudaMemset(d.off, 0, 8);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        debug_free_slots(d);
        cudaFree(d.state);
        cudaFree(d.off);
        delete h;
        return TAD_ERR_CUDA;
    }
    *out = h;
    return TAD_OK;
}

// One chunk through launch_text_encode (arguments as there; text / marks in host memory): ids_out[0, n) and the state
// words after it (state_out[8]).  An open dictionary refuses a chunk that could take it past half full,
// 2 * (names + n) > cap, as the engine grows before that.
extern "C" int tad_debug_text_dict_encode(void *handle, const uint8_t *text, uint64_t span, const uint64_t *marks,
                                          uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo, uint64_t n,
                                          uint32_t *ids_out, uint64_t *state_out)
{
    DebugDict *h = static_cast<DebugDict *>(handle);
    if (!h || !state_out || (n && (!ids_out || !marks || !nseg)) || (span && !text)) return TAD_ERR_INVALID_ARG;
    if (n && !debug_rows_ok(span, nseg, seg0_row, block_rows, lo, n)) return TAD_ERR_INVALID_ARG;
    tad::TextDict &d = h->d;
    if (!d.frozen && 2 * (h->names + n) > d.cap) return TAD_ERR_INVALID_ARG;
    if (cudaSetDevice(h->device) != cudaSuccess) return TAD_ERR_CUDA;
    const uint64_t nn = h->names + n;
    cudaError_t e = debug_grow(d.arena, h->arena_cap, std::max<uint64_t>(h->bytes + span, 1), h->bytes);
    if (e == cudaSuccess) h->arena_cap = std::max<uint64_t>(h->arena_cap, std::max<uint64_t>(h->bytes + span, 1));
    if (e == cudaSuccess) e = debug_grow(d.off, (h->names_cap + 1) * 8, (nn + 1) * 8, (h->names + 1) * 8);
    if (e == cudaSuccess) e = debug_grow(d.hash, h->names_cap * 8, std::max<uint64_t>(nn, 1) * 8, h->names * 8);
    if (e == cudaSuccess) h->names_cap = std::max(h->names_cap, std::max<uint64_t>(nn, 1));
    char *buf = nullptr;
    void *scratch = nullptr;
    uint32_t *ids = nullptr;
    size_t scratch_bytes = 0;
    if (e == cudaSuccess) e = debug_stage(text, span, marks, nseg, n, buf, scratch, scratch_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&ids, std::max<uint64_t>(n, 1) * 4);
    if (e == cudaSuccess)
        e = tad::launch_text_encode(0, d, reinterpret_cast<const uint8_t *>(buf + tad::align256((size_t)nseg * 8 + 8)), span,
                                    reinterpret_cast<const uint64_t *>(buf), nseg, seg0_row, block_rows, lo, n, scratch,
                                    scratch_bytes, ids);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && n) e = cudaMemcpy(ids_out, ids, n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(state_out, d.state, 64, cudaMemcpyDeviceToHost);
    cudaFree(buf);
    cudaFree(scratch);
    cudaFree(ids);
    if (e != cudaSuccess) return TAD_ERR_CUDA;
    h->names = state_out[0];
    h->bytes = state_out[1];
    return TAD_OK;
}

// A table of new_cap slots (a power of two holding the names at most half full): cleared and every name re-inserted
// from its stored hash, as TextKeys::grow does.
extern "C" int tad_debug_text_dict_grow(void *handle, uint32_t new_cap)
{
    DebugDict *h = static_cast<DebugDict *>(handle);
    if (!h || new_cap < 2 || (new_cap & (new_cap - 1)) || 2 * h->names > new_cap) return TAD_ERR_INVALID_ARG;
    if (cudaSetDevice(h->device) != cudaSuccess) return TAD_ERR_CUDA;
    tad::TextDict nd = h->d;
    cudaError_t e = debug_alloc_slots(nd, new_cap);
    if (e == cudaSuccess) e = tad::launch_text_rehash(0, h->d, nd, h->names);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        debug_free_slots(nd);
        return TAD_ERR_CUDA;
    }
    debug_free_slots(h->d);
    h->d = nd;
    return TAD_OK;
}

// Later chunks look names up and add none; a name the dictionary lacks sets state[5] and gets id 0.
extern "C" int tad_debug_text_dict_freeze(void *handle)
{
    DebugDict *h = static_cast<DebugDict *>(handle);
    if (!h) return TAD_ERR_INVALID_ARG;
    h->d.frozen = 1;
    return TAD_OK;
}

// The dictionary's name and byte counts; with non-null buffers also its arena (bytes), offsets (names + 1) and the
// stored hash of every name (names).
extern "C" int tad_debug_text_dict_names(void *handle, uint64_t *names, uint64_t *bytes, uint8_t *arena_out,
                                         uint64_t *off_out, uint64_t *hash_out)
{
    DebugDict *h = static_cast<DebugDict *>(handle);
    if (!h || !names || !bytes) return TAD_ERR_INVALID_ARG;
    *names = h->names;
    *bytes = h->bytes;
    if (cudaSetDevice(h->device) != cudaSuccess) return TAD_ERR_CUDA;
    cudaError_t e = cudaSuccess;
    if (arena_out && h->bytes) e = cudaMemcpy(arena_out, h->d.arena, h->bytes, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && off_out) e = cudaMemcpy(off_out, h->d.off, (h->names + 1) * 8, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && hash_out && h->names) e = cudaMemcpy(hash_out, h->d.hash, h->names * 8, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? TAD_OK : TAD_ERR_CUDA;
}

extern "C" int tad_debug_text_dict_free(void *handle)
{
    DebugDict *h = static_cast<DebugDict *>(handle);
    if (!h) return TAD_ERR_INVALID_ARG;
    cudaSetDevice(h->device);
    debug_free_slots(h->d);
    cudaFree(h->d.arena);
    cudaFree(h->d.off);
    cudaFree(h->d.hash);
    cudaFree(h->d.state);
    delete h;
    return TAD_OK;
}

// The device twin of tad_debug_ns_match: rows [lo, lo + n) of a namespace text column (arguments as for
// tad_debug_text_dict_encode) tested by launch_ns_match against the list, image and lookup both under hash_mask.
// verdict_out[0, n): 1 = listed; *error = the decode error flag (state word 2).
extern "C" int tad_debug_ns_match_device(int device, const uint8_t *list_bytes, const uint64_t *list_off, uint32_t names,
                                         uint64_t hash_mask, const uint8_t *text, uint64_t span, const uint64_t *marks,
                                         uint32_t nseg, uint64_t seg0_row, uint64_t block_rows, uint64_t lo, uint64_t n,
                                         uint32_t *verdict_out, uint64_t *error)
{
    if (!list_off || (names && !list_bytes) || !error || (span && !text) || (n && (!verdict_out || !marks || !nseg)))
        return TAD_ERR_INVALID_ARG;
    if (names > tad::kNsMaxNames || list_off[names] - list_off[0] > tad::kNsMaxBytes) return TAD_ERR_INVALID_ARG;
    if (n && !debug_rows_ok(span, nseg, seg0_row, block_rows, lo, n)) return TAD_ERR_INVALID_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return TAD_ERR_CUDA;
    const std::vector<uint8_t> img = tad::ns_list_image(list_bytes, list_off, names, hash_mask);
    void *dimg = nullptr, *scratch = nullptr;
    char *buf = nullptr;
    uint32_t *verdict = nullptr;
    size_t scratch_bytes = 0;
    cudaError_t e = cudaMalloc(&dimg, img.size());
    if (e == cudaSuccess) e = cudaMemcpy(dimg, img.data(), img.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = debug_stage(text, span, marks, nseg, n, buf, scratch, scratch_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&verdict, std::max<uint64_t>(n, 1) * 4);
    if (e == cudaSuccess)
        e = tad::launch_ns_match(0, dimg, names, img.size(), hash_mask, static_cast<unsigned long long *>(dimg),
                                 reinterpret_cast<const uint8_t *>(buf + tad::align256((size_t)nseg * 8 + 8)), span,
                                 reinterpret_cast<const uint64_t *>(buf), nseg, seg0_row, block_rows, lo, n, scratch,
                                 scratch_bytes, verdict);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess && n) e = cudaMemcpy(verdict_out, verdict, n * 4, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(error, static_cast<uint64_t *>(dimg) + 2, 8, cudaMemcpyDeviceToHost);
    cudaFree(dimg);
    cudaFree(buf);
    cudaFree(scratch);
    cudaFree(verdict);
    return e == cudaSuccess ? TAD_OK : TAD_ERR_CUDA;
}
