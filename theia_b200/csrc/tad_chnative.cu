// Host-only helpers for ClickHouse Native-format String columns (include/theia_tad.h, last section).
// No CUDA calls: usable without a GPU; lives in the library so that the Go / C / Python shims share one decoder.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/theia_tad.h"

extern "C" {

int tad_ch_string_index(const uint8_t *buf, size_t len, uint64_t rows, uint64_t *offsets, uint32_t *lengths, size_t *consumed)
{
    if ((!buf && len) || !offsets || !lengths) return TAD_ERR_INVALID_ARG;
    size_t p = 0;
    for (uint64_t i = 0; i < rows; i++) {
        uint64_t n = 0;
        int shift = 0;
        for (;;) {                                   // VarUInt: 7 bits per byte, least significant group first
            if (p >= len || shift > 63) return TAD_ERR_INVALID_ARG;
            const uint8_t b = buf[p++];
            n |= (uint64_t)(b & 0x7f) << shift;
            if (!(b & 0x80)) break;
            shift += 7;
        }
        if (n >= (1ull << 32) || n > len - p) return TAD_ERR_INVALID_ARG;
        offsets[i] = p;
        lengths[i] = (uint32_t)n;
        p += (size_t)n;
    }
    if (consumed) *consumed = p;
    return TAD_OK;
}

static void parse_ipv4_range(const uint8_t *buf, const uint64_t *offsets, const uint32_t *lengths, uint64_t lo, uint64_t hi,
                             uint32_t *out, uint8_t *is_v4)
{
    for (uint64_t i = lo; i < hi; i++) {
        const uint8_t *s = buf + offsets[i];
        const uint32_t n = lengths[i];
        uint32_t v = 0, part = 0, digits = 0, dots = 0;
        bool ok = n >= 7 && n <= 15;
        for (uint32_t k = 0; ok && k < n; k++) {
            const uint8_t c = s[k];
            if (c >= '0' && c <= '9') {
                ok = !(digits > 0 && part == 0);     // no leading zeros: the text must be what tad_ch_format_ipv4 writes back
                part = part * 10 + (c - '0');
                ok = ok && ++digits <= 3 && part <= 255;
            } else if (c == '.') {
                ok = digits > 0 && ++dots <= 3;
                v = (v << 8) | part;
                part = 0;
                digits = 0;
            } else {
                ok = false;
            }
        }
        ok = ok && dots == 3 && digits > 0;
        out[i] = ok ? ((v << 8) | part) : 0u;
        is_v4[i] = ok ? 1 : 0;
    }
}

int tad_ch_parse_ipv4(const uint8_t *buf, const uint64_t *offsets, const uint32_t *lengths, uint64_t rows, uint32_t *out,
                      uint8_t *is_v4)
{
    if (!buf || !offsets || !lengths || !out || !is_v4) return TAD_ERR_INVALID_ARG;
    // rows are independent: large columns are split over a few host threads (the index pass before is sequential)
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const uint64_t nt = rows < (1u << 16) ? 1 : std::min<uint64_t>({(uint64_t)hw, 16, rows >> 15});
    if (nt <= 1) {
        parse_ipv4_range(buf, offsets, lengths, 0, rows, out, is_v4);
        return TAD_OK;
    }
    std::vector<std::thread> th;
    for (uint64_t t = 0; t < nt; t++)
        th.emplace_back(parse_ipv4_range, buf, offsets, lengths, rows * t / nt, rows * (t + 1) / nt, out, is_v4);
    for (auto &x : th) x.join();
    return TAD_OK;
}

int tad_ch_format_ipv4(const uint32_t *ips, uint64_t rows, uint8_t *out, size_t out_cap, size_t *written)
{
    if (!ips || !out || !written) return TAD_ERR_INVALID_ARG;
    size_t p = 0;
    for (uint64_t i = 0; i < rows; i++) {
        if (out_cap - p < 16) return TAD_ERR_INVALID_ARG;
        uint8_t *len_at = out + p++;
        const size_t start = p;
        for (int k = 3; k >= 0; k--) {
            const uint32_t b = (ips[i] >> (8 * k)) & 255u;
            if (b >= 100) out[p++] = (uint8_t)('0' + b / 100);
            if (b >= 10) out[p++] = (uint8_t)('0' + (b / 10) % 10);
            out[p++] = (uint8_t)('0' + b % 10);
            if (k) out[p++] = '.';
        }
        *len_at = (uint8_t)(p - start);              // 7..15 < 128: a one-byte VarUInt
    }
    *written = p;
    return TAD_OK;
}

int tad_ch_format_names(const uint8_t *bytes, const uint64_t *offsets, uint32_t count, const uint32_t *ids, uint64_t rows,
                        uint8_t *out, size_t out_cap, size_t *written)
{
    if ((rows && (!ids || !offsets || !bytes)) || (!out && out_cap) || !written) return TAD_ERR_INVALID_ARG;
    size_t p = 0;
    for (uint64_t i = 0; i < rows; i++) {
        const uint32_t id = ids[i];
        if (id >= count || offsets[id + 1] < offsets[id]) return TAD_ERR_INVALID_ARG;
        uint64_t n = offsets[id + 1] - offsets[id];
        uint8_t len[10];
        int k = 0;
        do {
            len[k++] = (uint8_t)((n & 0x7f) | (n >= 0x80 ? 0x80 : 0));
            n >>= 7;
        } while (n);
        n = offsets[id + 1] - offsets[id];
        if (out_cap - p < k || out_cap - p - k < n) return TAD_ERR_INVALID_ARG;
        memcpy(out + p, len, k);
        if (n) memcpy(out + p + k, bytes + offsets[id], n);
        p += k + n;
    }
    *written = p;
    return TAD_OK;
}

int tad_ch_dictionary(const uint8_t *buf, const uint64_t *offsets, const uint32_t *lengths, uint64_t rows, uint32_t *ids,
                      uint64_t *first_row, uint32_t *n_unique)
{
    if ((!buf && rows) || !offsets || !lengths || !ids || !first_row || !n_unique) return TAD_ERR_INVALID_ARG;
    if (rows >= (1ull << 32)) return TAD_ERR_INVALID_ARG;
    // open addressing over (hash, id); the table doubles when half full.  FNV-1a over the value bytes.
    size_t cap = 1024;
    std::vector<uint32_t> slot_id(cap, 0xffffffffu);
    std::vector<uint64_t> slot_hash(cap, 0);
    uint32_t n = 0;
    for (uint64_t i = 0; i < rows; i++) {
        const uint8_t *s = buf + offsets[i];
        const uint32_t len = lengths[i];
        uint64_t h = 1469598103934665603ull;
        for (uint32_t k = 0; k < len; k++) h = (h ^ s[k]) * 1099511628211ull;
        h ^= h >> 29;
        size_t p = (size_t)h & (cap - 1);
        for (;;) {
            const uint32_t id = slot_id[p];
            if (id == 0xffffffffu) {                        // new value
                slot_id[p] = n;
                slot_hash[p] = h;
                first_row[n] = i;
                ids[i] = n++;
                break;
            }
            const uint64_t r = first_row[id];
            if (slot_hash[p] == h && lengths[r] == len && memcmp(buf + offsets[r], s, len) == 0) { ids[i] = id; break; }
            p = (p + 1) & (cap - 1);
        }
        if ((size_t)n * 2 > cap) {                          // grow and re-insert (ids are stable)
            cap *= 2;
            std::vector<uint32_t> nid(cap, 0xffffffffu);
            std::vector<uint64_t> nh(cap, 0);
            for (size_t q = 0; q < slot_id.size(); q++) {
                if (slot_id[q] == 0xffffffffu) continue;
                size_t t = (size_t)slot_hash[q] & (cap - 1);
                while (nid[t] != 0xffffffffu) t = (t + 1) & (cap - 1);
                nid[t] = slot_id[q];
                nh[t] = slot_hash[q];
            }
            slot_id.swap(nid);
            slot_hash.swap(nh);
        }
    }
    *n_unique = n;
    return TAD_OK;
}

}  // extern "C"
