// pcd_binary.h -- the PCD header reader and the stages of the binary / binary_compressed reader (DESIGN.md section 12.1).
// pcd_kernels.cu runs the stages as kernels; host_selftest.cpp runs the very same functions serially, so the CPU test-suite
// checks the parallel LZF decoder (speculative token discovery, composition of the chunks' entry maps, token records, pointer
// jumping over back-references) before any GPU run.
//
// Field rules restated from PCL 1.8 (PCDReader::readHeader, readBodyBinary, fromPCLPointCloud2<PointXYZI>); PCL is not built
// here, so parity with it is unpinned:
//   - FIELDS, SIZE, TYPE and COUNT (optional, default 1) have one entry per field; TYPE/SIZE is F 4/8 or I/U 1/2/4;
//   - WIDTH x HEIGHT == POINTS (both absent: WIDTH = POINTS, HEIGHT = 1);
//   - x, y, z are F 4 COUNT 1; intensity is taken when it is F 4 COUNT 1 and is 0 otherwise (PCL finds no match for it);
//   - binary: AoS, point_step = sum of SIZE x COUNT over every field ("_" padding included);
//   - binary_compressed: uint32 compressed_size, uint32 uncompressed_size, then one LZF stream whose output is SoA: one block of
//     POINTS x SIZE x COUNT bytes per field not named "_", in header order.  uncompressed_size must be POINTS x point_step.
// LZF restated from liblzf's lzf_d.c: control byte c < 32 copies the next c + 1 bytes; otherwise L = c >> 5 (+ the next byte when
// L == 7) + 2 bytes are copied one at a time from D = ((c & 31) << 8) + the following byte + 1 bytes back in the output.
#pragma once
#include <stdint.h>

#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/erasor_b200.h"
#include "pcd_codec.h"

namespace pcd {

// ---- the header, read on the host ----------------------------------------------------------------------------------------
struct Header {
    std::vector<std::string> fields, sizes, types, counts;
    unsigned long long points = 0, width = 0, height = 0;
    bool have_points = false, have_width = false, have_height = false, have_data = false;
    std::string data;
    uint64_t data_off = 0;       // first byte after the DATA line
    uint64_t lines = 0;          // lines before data_off
};

inline bool header_uint(const std::string& s, unsigned long long& v) {
    char* end = nullptr;
    v = std::strtoull(s.c_str(), &end, 10);
    return end && *end == 0 && s[0] != '-';
}

// header lines up to and including DATA; false when the text ends before a DATA line
inline bool parse_header(const char* s, uint64_t n, Header& h) {
    uint64_t p = 0;
    while (p < n) {
        uint64_t e = p;                              // the line ends at '\n', "\r\n" or a lone '\r' (universal newlines)
        while (e < n && s[e] != '\n' && s[e] != '\r') ++e;
        std::vector<std::string> tok;
        for (uint64_t q = p; q < e;) {
            while (q < e && is_ws((uint8_t)s[q])) ++q;
            const uint64_t a = q;
            while (q < e && !is_ws((uint8_t)s[q])) ++q;
            if (q > a) tok.emplace_back(s + a, q - a);
        }
        ++h.lines;
        const uint64_t next = e >= n ? n : (s[e] == '\r' && e + 1 < n && s[e + 1] == '\n') ? e + 2 : e + 1;
        if (!tok.empty()) {
            if (tok[0] == "FIELDS") h.fields.assign(tok.begin() + 1, tok.end());
            else if (tok[0] == "SIZE") h.sizes.assign(tok.begin() + 1, tok.end());
            else if (tok[0] == "TYPE") h.types.assign(tok.begin() + 1, tok.end());
            else if (tok[0] == "COUNT") h.counts.assign(tok.begin() + 1, tok.end());
            else if (tok[0] == "POINTS" && tok.size() > 1) h.have_points = header_uint(tok[1], h.points);
            else if (tok[0] == "WIDTH" && tok.size() > 1) h.have_width = header_uint(tok[1], h.width);
            else if (tok[0] == "HEIGHT" && tok.size() > 1) h.have_height = header_uint(tok[1], h.height);
            else if (tok[0] == "DATA") {
                h.have_data = true;
                h.data = tok.size() > 1 ? tok[1] : std::string();
                h.data_off = next;
                return true;
            }
        }
        p = next;
    }
    return false;
}

// ---- layout of a binary file ---------------------------------------------------------------------------------------------
enum { DATA_ASCII = 0, DATA_BINARY = 1, DATA_COMPRESSED = 2 };

// where point i's value of slot s (x y z intensity) lies: off[s] + i * stride bytes into the body (binary) or the decompressed
// buffer (binary_compressed); slots whose bit is clear in fields read as 0
struct Gather {
    uint64_t stride;
    uint64_t off[4];
    uint32_t fields;
};

struct Layout {
    uint32_t mode = DATA_ASCII;
    uint32_t zero_intensity = 0;     // FIELDS names intensity, but not as F 4 COUNT 1
    uint64_t point_step = 0;         // binary: the AoS stride; binary_compressed: the bytes of the non-"_" fields
    uint64_t points = 0, width = 0, height = 0;
    uint64_t keep_end = 0;           // binary_compressed: the end of the last block the gather reads
    Gather g{0, {0, 0, 0, 0}, 0};
};

// The header's rules for the binary modes (ascii is left to erasor_pcd_parse_ascii: only mode is set).  ERASOR_OK, or an error
// code with msg.
inline int resolve_layout(const Header& h, Layout& L, std::string& msg) {
    L = Layout();
    L.points = h.points;
    L.width = h.width;
    L.height = h.height;
    if (h.data == "ascii") { L.mode = DATA_ASCII; return ERASOR_OK; }
    if (h.data == "binary") L.mode = DATA_BINARY;
    else if (h.data == "binary_compressed") L.mode = DATA_COMPRESSED;
    else { msg = "DATA " + h.data + ": not a PCD data mode (ascii, binary or binary_compressed)"; return ERASOR_E_UNSUPPORTED; }
    if (h.sizes.empty() || h.types.empty()) { msg = "no SIZE or TYPE line: PCD versions before 0.7 are not read"; return ERASOR_E_UNSUPPORTED; }
    const size_t nf = h.fields.size();
    if (h.sizes.size() != nf || h.types.size() != nf || (!h.counts.empty() && h.counts.size() != nf)) {
        msg = "FIELDS, SIZE, TYPE and COUNT list different numbers of fields";
        return ERASOR_E_INVALID;
    }
    if (!h.have_points) { msg = "no valid POINTS line in the PCD header"; return ERASOR_E_INVALID; }
    if (!h.have_width && !h.have_height) { L.width = h.points; L.height = 1; }           // PCL's rule for older files
    if (L.height ? (L.width > h.points / L.height || L.width * L.height != h.points) : h.points != 0) {
        msg = "WIDTH x HEIGHT differs from POINTS";
        return ERASOR_E_INVALID;
    }
    const uint64_t kMaxStep = 0xFFFFFFFFull;         // point_step is a uint32 in erasor_pcd_load_info_t; no real point is near it
    int slot_field[4] = {-1, -1, -1, -1};
    std::vector<uint64_t> bytes(nf), at(nf);
    uint64_t aos = 0, soa = 0;
    for (size_t k = 0; k < nf; ++k) {
        unsigned long long size = 0, count = 1;
        if (!header_uint(h.sizes[k], size) || (!h.counts.empty() && (!header_uint(h.counts[k], count) || count == 0)) || count > kMaxStep) {
            msg = "field " + h.fields[k] + ": SIZE or COUNT is not a positive integer";
            return ERASOR_E_INVALID;
        }
        const std::string& t = h.types[k];
        const bool ok = (t == "F" && (size == 4 || size == 8)) || ((t == "I" || t == "U") && (size == 1 || size == 2 || size == 4));
        if (!ok) { msg = "field " + h.fields[k] + ": TYPE " + t + " SIZE " + h.sizes[k] + " is not a PCD type"; return ERASOR_E_UNSUPPORTED; }
        bytes[k] = size * count;
        const bool pad = h.fields[k] == "_";
        at[k] = L.mode == DATA_BINARY ? aos : soa;
        aos += bytes[k];
        if (!pad) soa += bytes[k];
        if (aos > kMaxStep) { msg = "a point of 2^32 bytes or more"; return ERASOR_E_UNSUPPORTED; }
        const std::string& f = h.fields[k];
        const int s = f == "x" ? 0 : f == "y" ? 1 : f == "z" ? 2 : f == "intensity" ? 3 : -1;
        if (s >= 0 && slot_field[s] < 0) {
            slot_field[s] = (int)k;
            const bool f4 = t == "F" && size == 4 && count == 1;
            if (f4) L.g.fields |= 1u << s;
            else if (s < 3) { msg = "field " + f + ": x, y and z must be TYPE F SIZE 4 COUNT 1"; return ERASOR_E_UNSUPPORTED; }
            else L.zero_intensity = 1;
        }
    }
    if (slot_field[0] < 0 || slot_field[1] < 0 || slot_field[2] < 0) { msg = "the PCD's FIELDS lack x, y or z"; return ERASOR_E_INVALID; }
    L.point_step = L.mode == DATA_BINARY ? aos : soa;
    if (L.point_step && h.points > ~0ull / L.point_step) { msg = "POINTS x point_step exceeds 2^64 bytes"; return ERASOR_E_INVALID; }
    for (int s = 0; s < 4; ++s) {
        if (!((L.g.fields >> s) & 1u)) continue;
        const uint64_t o = at[slot_field[s]];
        L.g.off[s] = L.mode == DATA_BINARY ? o : o * h.points;
        if (L.mode == DATA_COMPRESSED && L.g.off[s] + 4 * h.points > L.keep_end) L.keep_end = L.g.off[s] + 4 * h.points;
    }
    L.g.stride = L.mode == DATA_BINARY ? L.point_step : 4;
    return ERASOR_OK;
}

// binary: the file holds its POINTS x point_step bytes after the header
inline int check_binary_body(const Layout& L, uint64_t data_off, uint64_t len, std::string& msg) {
    if (len < data_off || len - data_off < L.points * L.point_step) {
        msg = "the file ends before its POINTS x point_step bytes of binary data";
        return ERASOR_E_INVALID;
    }
    return ERASOR_OK;
}

// binary_compressed: the two sizes after the header, and the stream they announce
inline int check_compressed_sizes(const Layout& L, uint64_t data_off, uint64_t len, uint64_t csize, uint64_t usize, std::string& msg) {
    if (len - data_off - 8 < csize) { msg = "the file ends before its compressed_size bytes of LZF data"; return ERASOR_E_INVALID; }
    if (usize != L.points * L.point_step) {
        msg = "uncompressed_size " + std::to_string(usize) + " differs from POINTS x point_step = " + std::to_string(L.points * L.point_step);
        return ERASOR_E_INVALID;
    }
    return ERASOR_OK;
}

PCD_HD uint32_t le32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// point i's four values as bit patterns (copied, never converted: NaN payloads survive)
PCD_HD void gather_point(const uint8_t* base, const Gather& g, uint64_t i, uint32_t v[4]) {
    for (int s = 0; s < 4; ++s) v[s] = ((g.fields >> s) & 1u) ? le32(base + g.off[s] + i * g.stride) : 0u;
}

// ---- LZF ---------------------------------------------------------------------------------------------------------------
// A token is at most 33 bytes (control byte + 32 literals), so the first token that starts in a chunk starts at one of its first
// kLzfEntries bytes, and the walk from any of them leaves the chunk at most 32 bytes past its end.
constexpr int kLzfEntries = 33;

enum { LZF_PAST_STREAM = 1, LZF_BEFORE_START = 2, LZF_OVERRUN = 3 };

// bytes of the stream the token with control byte c takes
PCD_HD uint32_t lzf_token_size(uint8_t c) { return c < 32 ? (uint32_t)c + 2u : ((c >> 5) == 7 ? 3u : 2u); }

// Stage A: the walk from byte `begin + e` of the chunk [begin, end) to the first token start at or past end.
struct LzfWalk {
    uint32_t exit;               // that start - end, 0..32: the entry of the next chunk along this chain
    uint32_t tokens;             // tokens that start in the chunk along this chain
    uint32_t bytes;              // their output bytes (a token whose length byte lies past the stream counts 0; stage B rejects it)
};

PCD_HD LzfWalk lzf_walk(const uint8_t* s, uint64_t csize, uint64_t begin, uint64_t end, uint32_t e) {
    LzfWalk w{0, 0, 0};
    uint64_t pos = begin + e;
    while (pos < end) {
        const uint8_t c = s[pos];
        uint32_t len = c < 32 ? (uint32_t)c + 1u : (uint32_t)(c >> 5) + 2u;
        if (c >= 32 && (c >> 5) == 7) len = pos + 1 < csize ? len + s[pos + 1] : 0u;
        w.bytes += len;
        ++w.tokens;
        pos += lzf_token_size(c);
    }
    w.exit = (uint32_t)(pos - end);
    return w;
}

// the map of a chunk after the maps of earlier chunks: out[e] = later[earlier[e]]
PCD_HD uint8_t lzf_compose(const uint8_t* later, const uint8_t* earlier, int e) { return later[earlier[e]]; }

// Stage B: one token as a record.  kind_len: the output length, bit 31 set for a back-reference; arg: the literal's first byte in
// the stream, or the distance.
struct LzfToken {
    uint32_t dst, arg, kind_len;
};
constexpr uint32_t kLzfRef = 0x80000000u;

// The token at pos whose output starts at dst; returns 0, or the first rule of section 3 it breaks.  Every bound is checked
// before the byte it guards is read.
PCD_HD int lzf_token(const uint8_t* s, uint64_t csize, uint64_t usize, uint64_t pos, uint64_t dst, LzfToken& t, uint32_t& size) {
    const uint8_t c = s[pos];
    size = lzf_token_size(c);
    t.dst = (uint32_t)dst;
    if (pos + size > csize) { t.arg = 0; t.kind_len = 0; return LZF_PAST_STREAM; }
    if (c < 32) {
        t.arg = (uint32_t)(pos + 1);
        t.kind_len = (uint32_t)c + 1u;
    } else {
        uint32_t len = (uint32_t)(c >> 5);
        if (len == 7) len += s[pos + 1];
        len += 2;
        const uint32_t d = ((uint32_t)(c & 31) << 8) + s[pos + size - 1] + 1u;
        t.arg = d;
        t.kind_len = kLzfRef | len;
        if (d > dst) return LZF_BEFORE_START;
    }
    if (dst + (t.kind_len & ~kLzfRef) > usize) return LZF_OVERRUN;
    return 0;
}

// Stage B over one chunk from its true entry: records from rec[0], the first broken rule as (stream offset << 2) | rule in *err
// (~0 when none).  Returns the tokens walked.
PCD_HD uint64_t lzf_records(const uint8_t* s, uint64_t csize, uint64_t usize, uint64_t begin, uint64_t end, uint32_t entry, uint64_t dst,
                            LzfToken* rec, uint64_t* err) {
    uint64_t pos = begin + entry, k = 0;
    *err = ~0ull;
    while (pos < end) {
        uint32_t size;
        const int bad = lzf_token(s, csize, usize, pos, dst, rec[k], size);
        if (bad && *err == ~0ull) *err = (pos << 2) | (uint64_t)bad;
        dst += rec[k].kind_len & ~kLzfRef;
        pos += size;
        ++k;
    }
    return k;
}

// Stage C: a record's bytes below keep.  Literal bytes are copied and point at themselves in src; byte j of a back-reference points
// at j - D.
PCD_HD void lzf_expand(const LzfToken& t, const uint8_t* s, uint8_t* out, uint32_t* src, uint64_t keep) {
    const uint32_t len = t.kind_len & ~kLzfRef;
    const uint64_t end = (uint64_t)t.dst + len < keep ? (uint64_t)t.dst + len : keep;
    if (t.kind_len & kLzfRef) {
        for (uint64_t j = t.dst; j < end; ++j) src[j] = (uint32_t)(j - t.arg);
    } else {
        for (uint64_t j = t.dst; j < end; ++j) { out[j] = s[t.arg + (j - t.dst)]; src[j] = (uint32_t)j; }
    }
}

// one pointer-jumping step of byte j: src[j] <- src[src[j]]; true when it moved
PCD_HD bool lzf_jump(uint32_t* src, uint64_t j) {
    const uint32_t a = src[j];
    if (a == j) return false;
    const uint32_t b = src[a];
    if (b == a) return false;
    src[j] = b;
    return true;
}

// after the jumps every byte points at the literal byte it copies
PCD_HD void lzf_fill(const uint32_t* src, uint8_t* out, uint64_t j) {
    const uint32_t a = src[j];
    if (a != j) out[j] = out[a];
}

inline std::string lzf_error_message(uint64_t err) {
    const uint64_t pos = err >> 2;
    const int rule = (int)(err & 3);
    const char* what = rule == LZF_PAST_STREAM ? "reads past compressed_size" : rule == LZF_BEFORE_START ? "refers before the start of the output"
                                                                                                            : "writes past uncompressed_size";
    return "malformed LZF stream: the token at stream byte " + std::to_string(pos) + " " + what;
}

inline void fill_load_info(const Header& h, const Layout& L, erasor_pcd_load_info_t& inf) {
    inf.data_mode = L.mode;
    inf.fields = L.g.fields;
    inf.intensity_zero_filled = L.zero_intensity;
    inf.point_step = (uint32_t)L.point_step;
    inf.width = L.width;
    inf.height = L.height;
    inf.points = h.points;
    inf.data_offset = h.data_off;
}

}  // namespace pcd
