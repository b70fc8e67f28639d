// lz4_frame.h -- the LZ4 frame and block format as erasor_bag_index reads LZ4-compressed bag chunks (DESIGN.md section 12.2.1).
// pcd_kernels.cu runs the block walk with one warp per block and XXH32 with one thread per block or frame; host_selftest.cpp runs
// the very same functions serially, so the CPU test-suite checks the decoder before any GPU run.
//
// Rules [3P], restated from the public LZ4 frame and block format descriptions and from what roslz4 writes (rosbag is not built
// here, so parity with it is unpinned):
//   - frame: magic 0x184D2204 (LE), FLG, BD, [content size u64], [dict id u32], HC = (XXH32(FLG .. last descriptor byte, 0) >> 8)
//     & 0xFF; then blocks, each a u32 whose high bit means "stored" and whose low 31 bits are the data size, the data, and a u32
//     XXH32(data, 0) when FLG's block-checksum bit is set; then the end mark 0 and a u32 XXH32(content, 0) when FLG's
//     content-checksum bit is set;
//   - FLG: version (bits 7-6) 01, block independence (bit 5) 1, block checksum (4), content size (3), content checksum (2),
//     reserved (1) 0, dict id (0) 0.  BD: block max id (bits 6-4) 4..7 = 64 KB, 256 KB, 1 MB, 4 MB; the other bits 0;
//   - a sequence: a token whose high nibble is the literal length and low nibble the match length - 4, each 15 extended by bytes
//     added until one is below 255; the literals; a u16 LE offset (1..65535 back in the block's own output); the match, copied
//     byte after byte (so an offset below the length repeats the last `offset` bytes).  The last sequence of a block has literals
//     only: the block ends right after them.
// Not enforced (a known divergence from liblz4's safe decoder): the last 5 bytes of a block being literals, and the last match
// starting 12 bytes or more before the block's end.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

#include "pcd_codec.h"

namespace lz4 {

constexpr uint32_t kMagic = 0x184D2204u;

// why a block walk stopped (0: it did not)
enum : uint32_t {
    R_OK = 0,
    R_OFFSET0 = 1,          // a match offset of 0
    R_OFFSET_BEFORE = 2,    // a match offset reaching before the block's own output
    R_LITERALS_PAST = 3,    // a literal run reading past the block
    R_LENGTH_PAST = 4,      // a length extension reading past the block
    R_OUTPUT_PAST = 5,      // output past the block max
    R_ENDS_IN_SEQ = 6,      // the block ends inside a sequence (before its offset)
    R_BLOCK_SUM = 7,        // a block checksum mismatch
    R_CONTENT_SUM = 8,      // the content checksum mismatch
    R_SIZE = 9,             // the frame does not decode to the chunk's size
};

PCD_HD const char* reason_text(uint32_t r) {
    switch (r) {
    case R_OFFSET0: return "a match offset of 0";
    case R_OFFSET_BEFORE: return "a match offset reaching before the block's own output";
    case R_LITERALS_PAST: return "a literal run reading past the block";
    case R_LENGTH_PAST: return "a length extension reading past the block";
    case R_OUTPUT_PAST: return "output past the block max";
    case R_ENDS_IN_SEQ: return "the block ends inside a sequence";
    case R_BLOCK_SUM: return "the block checksum does not match";
    case R_CONTENT_SUM: return "the content checksum does not match";
    case R_SIZE: return "the frame does not decode to the chunk's 'size'";
    default: return "no error";
    }
}

PCD_HD uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
PCD_HD uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

constexpr uint32_t kP1 = 2654435761u, kP2 = 2246822519u, kP3 = 3266489917u, kP4 = 668265263u, kP5 = 374761393u;

// the word at p: one 32-bit load when p is 4-byte aligned (the device's decoded chunks are 16-byte aligned), else byte by byte
PCD_HD uint32_t ld32(const uint8_t* p) {
#ifdef __CUDA_ARCH__
    if (!(reinterpret_cast<uintptr_t>(p) & 3u)) return *reinterpret_cast<const uint32_t*>(p);
#endif
    return rd32(p);
}

// XXH32's accumulator j (0..3) of [p, p + n) after every whole 16-byte stripe: the four accumulators are independent chains, so
// four threads can run them at once and xxh32_merge combines them
PCD_HD uint32_t xxh32_lane(const uint8_t* p, uint64_t n, uint32_t seed, uint32_t j) {
    uint32_t v = j == 0 ? seed + kP1 + kP2 : j == 1 ? seed + kP2 : j == 2 ? seed : seed - kP1;
    for (uint64_t i = 4 * j; i + 16 - 4 * j <= n; i += 16) v = rotl(v + ld32(p + i) * kP2, 13) * kP1;
    return v;
}

// XXH32 of [p, p + n) from its four accumulators (ignored when n < 16): the merge, the tail and the avalanche
PCD_HD uint32_t xxh32_merge(const uint32_t v[4], const uint8_t* p, uint64_t n, uint32_t seed) {
    uint64_t i = n & ~15ull;
    uint32_t h = n >= 16 ? rotl(v[0], 1) + rotl(v[1], 7) + rotl(v[2], 12) + rotl(v[3], 18) : seed + kP5;
    h += (uint32_t)n;
    for (; i + 4 <= n; i += 4) h = rotl(h + ld32(p + i) * kP3, 17) * kP4;
    for (; i < n; ++i) h = rotl(h + p[i] * kP5, 11) * kP1;
    h ^= h >> 15;
    h *= kP2;
    h ^= h >> 13;
    h *= kP3;
    h ^= h >> 16;
    return h;
}

// XXH32 of [p, p + n) with seed, by one thread
PCD_HD uint32_t xxh32(const uint8_t* p, uint64_t n, uint32_t seed) {
    uint32_t v[4];
    for (uint32_t j = 0; j < 4; ++j) v[j] = xxh32_lane(p, n, seed, j);
    return xxh32_merge(v, p, n, seed);
}

// One sequence at s[i]: its literal run [*lit0, *lit0 + *lit), then (when *last is false) a match of *mlen bytes *off back.  o: the
// block's output so far; cap: the block max.  Returns R_OK, or the broken rule with *at the byte it guards.
PCD_HD uint32_t sequence(const uint8_t* s, uint32_t n, uint32_t i, uint32_t o, uint32_t cap, uint32_t* lit0, uint32_t* lit, uint32_t* off,
                         uint32_t* mlen, uint32_t* next, bool* last, uint32_t* at) {
    const uint32_t tok = s[i++];
    uint32_t L = tok >> 4;
    if (L == 15) {
        uint32_t b;
        do {
            if (i >= n) { *at = i; return R_LENGTH_PAST; }
            b = s[i++];
            L += b;
        } while (b == 255);
    }
    if (L > n - i) { *at = i; return R_LITERALS_PAST; }
    if (L > cap - o) { *at = i; return R_OUTPUT_PAST; }
    *lit0 = i;
    *lit = L;
    i += L;
    o += L;
    if (i == n) { *last = true; *next = i; return R_OK; }
    *last = false;
    if (n - i < 2) { *at = i; return R_ENDS_IN_SEQ; }
    const uint32_t d = (uint32_t)s[i] | (uint32_t)s[i + 1] << 8;
    if (d == 0) { *at = i; return R_OFFSET0; }
    if (d > o) { *at = i; return R_OFFSET_BEFORE; }
    i += 2;
    uint32_t M = tok & 15u;
    if (M == 15) {
        uint32_t b;
        do {
            if (i >= n) { *at = i; return R_LENGTH_PAST; }
            b = s[i++];
            M += b;
        } while (b == 255);
    }
    M += 4;
    if (M > cap - o) { *at = i; return R_OUTPUT_PAST; }
    *off = d;
    *mlen = M;
    *next = i;
    return R_OK;
}

// The lanes that walk one block together.  Serial is one lane (the host, and the device's size pass); pcd_kernels.cu defines a
// warp of 32 whose lane 0 parses each sequence and broadcasts it.
struct Serial {
    PCD_HD uint32_t lane() const { return 0; }
    PCD_HD uint32_t lanes() const { return 1; }
    PCD_HD void sync() const {}
    PCD_HD uint32_t bcast(uint32_t v) const { return v; }
};

// The compressed block s[0, n) into dst (nullptr: the size alone), at most cap bytes.  Returns R_OK with *out the decoded size, or
// the first broken rule with *at its byte in s.  Every rule is checked before the byte it guards is read.  A match whose offset is
// below its length is copied in rounds of `offset` bytes: byte k of the match is byte (k mod offset) of the `offset` bytes before
// it, so every lane reads output that is already complete.
template <class W>
PCD_HD uint32_t block(const W& w, const uint8_t* s, uint32_t n, uint8_t* dst, uint32_t cap, uint32_t* out, uint32_t* at) {
    uint32_t i = 0, o = 0;
    while (true) {
        uint32_t r = R_OK, lit0 = 0, lit = 0, off = 0, mlen = 0, next = 0, a = 0;
        bool last = false;
        if (w.lane() == 0) {
            if (i >= n) r = R_ENDS_IN_SEQ, a = i;   // an empty block, or one whose last sequence carries a match
            else r = sequence(s, n, i, o, cap, &lit0, &lit, &off, &mlen, &next, &last, &a);
        }
        r = w.bcast(r);
        if (r != R_OK) { *at = w.bcast(a); return r; }
        lit0 = w.bcast(lit0); lit = w.bcast(lit); off = w.bcast(off); mlen = w.bcast(mlen); next = w.bcast(next);
        last = w.bcast(last ? 1u : 0u) != 0;
        if (dst) {
            for (uint32_t k = w.lane(); k < lit; k += w.lanes()) dst[o + k] = s[lit0 + k];
            o += lit;
            if (!last) {
                w.sync();
                const uint8_t* src = dst + o - off;
                if (off >= mlen) for (uint32_t k = w.lane(); k < mlen; k += w.lanes()) dst[o + k] = src[k];
                else for (uint32_t k = w.lane(); k < mlen; k += w.lanes()) dst[o + k] = src[k % off];
                o += mlen;
            }
            w.sync();
        } else {
            o += lit + (last ? 0 : mlen);
        }
        i = next;
        if (last) { *out = o; return R_OK; }
    }
}

// ---- the frame, read on the host (no decoding: the block table comes from the size prefixes) ------------------------------
struct Block {
    uint64_t off;                    // its data, from the start of the frame
    uint32_t csize;                  // its data's length
    uint32_t stored;                 // 1: the data is the output
    uint32_t sum;                    // its checksum, when the frame has block checksums
};

struct Frame {
    uint32_t block_max = 0;
    bool block_sums = false, content_sum = false;
    uint32_t sum = 0;                // the content checksum, when present
    std::vector<Block> blocks;
};

enum { F_OK = 0, F_UNSUPPORTED = 1, F_INVALID = 2 };

// The frame that must fill d[0, n) exactly and decode to `size` bytes: F_OK, or F_UNSUPPORTED / F_INVALID with msg (the byte in
// the frame named by the caller's prefix).
inline int parse_frame(const uint8_t* d, uint64_t n, uint64_t size, Frame& fr, std::string& msg) {
    fr = Frame();
    auto at = [](uint64_t p) { return " (byte " + std::to_string(p) + " of the frame)"; };
    if (n < 4 || rd32(d) != kMagic) { msg = "it does not start with the LZ4 frame magic 0x184D2204 (a legacy or skippable frame?)"; return F_UNSUPPORTED; }
    if (n < 7) { msg = "the frame descriptor runs past the chunk"; return F_INVALID; }
    const uint8_t flg = d[4], bd = d[5];
    if ((flg >> 6) != 1) { msg = "frame version " + std::to_string(flg >> 6) + ", not 1" + at(4); return F_UNSUPPORTED; }
    if (flg & 0x02u) { msg = "a reserved FLG bit is set" + at(4); return F_INVALID; }
    if (flg & 0x01u) { msg = "the frame names a dictionary" + at(4); return F_UNSUPPORTED; }
    if (!(flg & 0x20u)) { msg = "linked blocks (block independence 0) cannot be decoded in parallel" + at(4); return F_UNSUPPORTED; }
    if (bd & 0x8Fu) { msg = "a reserved BD bit is set" + at(5); return F_INVALID; }
    const uint32_t id = (bd >> 4) & 7u;
    if (id < 4) { msg = "block max id " + std::to_string(id) + " (only 4..7 exist)" + at(5); return F_INVALID; }
    fr.block_max = 1u << (8 + 2 * id);
    fr.block_sums = (flg & 0x10u) != 0;
    fr.content_sum = (flg & 0x04u) != 0;
    const bool has_size = (flg & 0x08u) != 0;
    const uint64_t hc = 6 + (has_size ? 8 : 0);
    if (n < hc + 1) { msg = "the frame descriptor runs past the chunk"; return F_INVALID; }
    if (((xxh32(d + 4, hc - 4, 0) >> 8) & 0xFFu) != d[hc]) { msg = "the header checksum does not match" + at(hc); return F_INVALID; }
    if (has_size) {
        uint64_t cs = 0;
        for (int k = 7; k >= 0; --k) cs = cs << 8 | d[6 + k];
        if (cs != size) { msg = "its content size " + std::to_string(cs) + " differs from the chunk's 'size' " + std::to_string(size) + at(6); return F_INVALID; }
    }
    uint64_t p = hc + 1;
    for (;;) {
        if (n - p < 4) { msg = "a block size runs past the chunk" + at(p); return F_INVALID; }
        const uint32_t v = rd32(d + p);
        if (v == 0) { p += 4; break; }
        const uint32_t bs = v & 0x7FFFFFFFu;
        if (bs > fr.block_max) {
            msg = "block " + std::to_string(fr.blocks.size()) + " holds " + std::to_string(bs) + " bytes, above the block max " + std::to_string(fr.block_max) + at(p);
            return F_INVALID;
        }
        const uint64_t need = (uint64_t)bs + (fr.block_sums ? 4 : 0);
        if (n - p - 4 < need) { msg = "block " + std::to_string(fr.blocks.size()) + " runs past the chunk" + at(p); return F_INVALID; }
        fr.blocks.push_back(Block{p + 4, bs, v >> 31, fr.block_sums ? rd32(d + p + 4 + bs) : 0u});
        p += 4 + need;
    }
    if (fr.content_sum) {
        if (n - p < 4) { msg = "the content checksum runs past the chunk" + at(p); return F_INVALID; }
        fr.sum = rd32(d + p);
        p += 4;
    }
    if (p != n) { msg = "the chunk's data goes on " + std::to_string(n - p) + " bytes past the end of its LZ4 frame" + at(p); return F_INVALID; }
    if (fr.blocks.empty() && size) { msg = "the frame holds no block, the chunk's 'size' is " + std::to_string(size); return F_INVALID; }
    return F_OK;
}

}  // namespace lz4
