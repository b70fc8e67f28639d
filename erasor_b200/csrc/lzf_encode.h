// lzf_encode.h -- the segmented LZF encoder behind erasor_pcd_format's binary_compressed mode (DESIGN.md section 12.3).
// pcd_kernels.cu runs it one warp per segment; host_selftest.cpp runs lzf_encode_segment serially; tests/lzf_encode_model.py
// restates the rule in Python.  All three give the same stream byte for byte, because the stream is a pure function of the input:
//   - the input is cut into segments of kLzfSeg bytes (the last one may be shorter), each encoded on its own: no reference reaches
//     before its segment's start, so the segments' token streams concatenate into one valid LZF stream (a decoder's only state is
//     its output position);
//   - every position i of a segment with three bytes left enters a table keyed by lzf_hash(bytes i..i+2), whatever the parse does.
//     cand(i) is the last earlier position of the segment with the same hash; it counts when its three bytes equal those at i and
//     i - cand(i) <= kLzfMaxDist.  cand(i) does not depend on the parse, so it can be found for all positions at once;
//   - a match is extended to at most kLzfMaxRef bytes, never past the segment's end;
//   - the parse is greedy from the segment's start: a match where one counts, else one literal byte; literal runs are cut at 32.
// This is not tests/pcd_binary_model.py's lzf_compress (which inserts only the positions its parse visits, so it is serial).
#pragma once
#include <stdint.h>

#include <cstdio>

#include "../../include/erasor_b200.h"
#include "pcd_codec.h"

namespace pcd {

// The header of every file erasor_pcd_format writes (pcl::io::savePCDFileASCII's for PointXYZI); only the DATA word differs
// between the modes.  Returns its length.
inline int format_header(char* buf, size_t cap, uint64_t n, int data_mode) {
    const char* word = data_mode == ERASOR_PCD_BINARY ? "binary" : data_mode == ERASOR_PCD_BINARY_COMPRESSED ? "binary_compressed" : "ascii";
    return std::snprintf(buf, cap,
                         "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\n"
                         "COUNT 1 1 1 1\nWIDTH %llu\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %llu\nDATA %s\n",
                         (unsigned long long)n, (unsigned long long)n, word);
}

constexpr uint32_t kLzfSeg = 16384;          // bytes per segment (S)
constexpr int kLzfHashLog = 13;              // the table holds 2^13 positions per segment
constexpr uint32_t kLzfHashSize = 1u << kLzfHashLog;
constexpr uint32_t kLzfMaxLit = 32;          // bytes per literal token
constexpr uint32_t kLzfMaxRef = 264;         // bytes per back-reference (7 + 255 + 2)
constexpr uint32_t kLzfMaxDist = 8192;       // 13 distance bits + 1

// the table key of the three bytes at p
PCD_HD uint32_t lzf_hash(const uint8_t* p) {
    const uint32_t v = ((uint32_t)p[0] << 16) | ((uint32_t)p[1] << 8) | (uint32_t)p[2];
    return (v * 2654435761u) >> (32 - kLzfHashLog);
}

// positions of a segment of len bytes that enter the table (three bytes left)
PCD_HD uint32_t lzf_positions(uint32_t len) { return len >= 3 ? len - 2 : 0; }

// the most bytes a segment of len bytes can take: all literals cost len + ceil(len / 32); a back-reference saves at least one byte
// and can add at most one literal run, so no mix costs more than that plus 1
PCD_HD uint64_t lzf_segment_cap(uint64_t len) { return len + (len + kLzfMaxLit - 1) / kLzfMaxLit + 1; }

// cand c (< i) counts for position i
PCD_HD bool lzf_cand_ok(const uint8_t* s, uint32_t i, uint32_t c) {
    return i - c <= kLzfMaxDist && s[c] == s[i] && s[c + 1] == s[i + 1] && s[c + 2] == s[i + 2];
}

// the match at i from c, at most kLzfMaxRef bytes and never past len (the first three bytes are known to be equal)
PCD_HD uint32_t lzf_match_len(const uint8_t* s, uint32_t len, uint32_t i, uint32_t c) {
    const uint32_t most = len - i < kLzfMaxRef ? len - i : kLzfMaxRef;
    uint32_t l = 3;
    while (l < most && s[c + l] == s[i + l]) ++l;
    return l;
}

// the back-reference token copying length (3..264) bytes from dist (1..8192) back; returns its bytes (2 or 3)
PCD_HD uint32_t lzf_put_ref(uint8_t* o, uint32_t length, uint32_t dist) {
    const uint32_t l = length - 2, d = dist - 1;
    if (l < 7) {
        o[0] = (uint8_t)((l << 5) | (d >> 8));
        o[1] = (uint8_t)(d & 255);
        return 2;
    }
    o[0] = (uint8_t)((7u << 5) | (d >> 8));
    o[1] = (uint8_t)(l - 7);
    o[2] = (uint8_t)(d & 255);
    return 3;
}

// literal runs of n bytes: the token count
PCD_HD uint32_t lzf_lit_runs(uint32_t n) { return (n + kLzfMaxLit - 1) / kLzfMaxLit; }

// byte k (0..n-1) of a literal stretch of n bytes goes to o + lzf_lit_at(k); run r's control byte to o + r * 33
PCD_HD uint32_t lzf_lit_at(uint32_t k) { return k + k / kLzfMaxLit + 1; }
PCD_HD uint8_t lzf_lit_control(uint32_t n, uint32_t r) {
    const uint32_t m = n - r * kLzfMaxLit;
    return (uint8_t)((m < kLzfMaxLit ? m : kLzfMaxLit) - 1);
}

// serially: the literal stretch s[0, n) as tokens at o; returns the bytes written
PCD_HD uint32_t lzf_put_lits(uint8_t* o, const uint8_t* s, uint32_t n) {
    const uint32_t runs = lzf_lit_runs(n);
    for (uint32_t r = 0; r < runs; ++r) o[r * (kLzfMaxLit + 1)] = lzf_lit_control(n, r);
    for (uint32_t k = 0; k < n; ++k) o[lzf_lit_at(k)] = s[k];
    return n + runs;
}

// One segment s[0, len) serially (table: kLzfHashSize entries of scratch, position + 1, 0 = empty).  Writes at most
// lzf_segment_cap(len) bytes at out; returns them, *tokens = the tokens.
inline uint32_t lzf_encode_segment(const uint8_t* s, uint32_t len, uint16_t* table, uint8_t* out, uint32_t* tokens) {
    for (uint32_t h = 0; h < kLzfHashSize; ++h) table[h] = 0;
    const uint32_t npos = lzf_positions(len);
    uint32_t o = 0, ntok = 0, lit = 0, p = 0;
    for (uint32_t i = 0; i < npos; ++i) {
        const uint32_t h = lzf_hash(s + i);
        const uint32_t t = table[h];
        table[h] = (uint16_t)(i + 1);
        if (i < p || !t || !lzf_cand_ok(s, i, t - 1)) continue;       // inside the last match, or no candidate
        const uint32_t c = t - 1, l = lzf_match_len(s, len, i, c);
        o += lzf_put_lits(out + o, s + lit, i - lit);
        ntok += lzf_lit_runs(i - lit);
        o += lzf_put_ref(out + o, l, i - c);
        ++ntok;
        p = lit = i + l;
    }
    o += lzf_put_lits(out + o, s + lit, len - lit);
    ntok += lzf_lit_runs(len - lit);
    *tokens = ntok;
    return o;
}

// ERASOR_OK, or ERASOR_E_UNSUPPORTED when a binary_compressed file cannot state a size in its uint32 fields: usize = POINTS x 16
// uncompressed bytes, csize the stream's bytes
PCD_HD int compressed_sizes_fit(uint64_t usize, uint64_t csize) {
    return usize > 0xFFFFFFFFull || csize > 0xFFFFFFFFull ? ERASOR_E_UNSUPPORTED : ERASOR_OK;
}

}  // namespace pcd
