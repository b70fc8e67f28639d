// bz2_stream.h -- the bzip2 stream format as erasor_bag_index reads bz2-compressed bag chunks (DESIGN.md section 12.2.2).
// pcd_kernels.cu runs these functions on the device (a thread per candidate block for the walk and the decode, a CTA per block for
// the inverse BWT, a thread per block for RLE1 and the CRC); host_selftest.cpp runs the very same functions serially, so the CPU
// test-suite checks the decoder against Python's bz2 (libbz2) before any GPU run.
//
// Rules [3P], restated from the public bzip2 format (no libbz2 source is used; rosbag is not built here, so parity with it is
// unpinned).  Bits are read most significant first.
//   - stream: "BZh", a level digit '1'..'9' (blocks of at most level x 100 000 bytes before RLE1), then blocks, each starting with
//     the 48-bit magic 0x314159265359, then the end-of-stream magic 0x177245385090, the 32-bit stream CRC and padding to a byte;
//   - block: CRC (32), randomised (1; must be 0 here), origPtr (24); the symbol map (16 bits of used 16-byte ranges, then 16 bits per
//     used range); nGroups (3, 2..6); nSelectors (15, at least 1; libbz2 keeps the first 18002), each selector a unary MTF index
//     below nGroups; per group a code length of 5 bits and per symbol a delta walk (1 then 0: +1, 1 then 1: -1, 0: next symbol),
//     every length 1..20; then Huffman symbols, a new group every 50: RUNA (0) and RUNB (1) spell a run of the front MTF byte in
//     bijective base 2, symbol k + 1 moves MTF entry k to the front and emits it, nInUse + 1 ends the block;
//   - inverse BWT: T[cftab[L[i]]++] = i, p = T[origPtr], then n times: emit L[p], p = T[p].  A periodic block's T is several
//     cycles; the walk then goes round origPtr's cycle more than once, as libbz2's does;
//   - RLE1: four equal bytes are followed by a count 0..255 of further copies;
//   - CRC: CRC-32, polynomial 0x04C11DB7, most significant bit first, initial and final xor 0xFFFFFFFF; the stream CRC is
//     rotl1(c) ^ blockCRC over the blocks in order.
// Known divergences from libbz2 (streams it may accept and these rules refuse; no bzip2 encoder writes them): randomised blocks,
// concatenated streams, trailing bytes after the stream's padding, over-subscribed or incomplete Huffman codes.
#pragma once
#include <stdint.h>

#include "pcd_codec.h"

namespace bz2 {

constexpr uint64_t kBlockMagic = 0x314159265359ull, kEosMagic = 0x177245385090ull;
constexpr uint32_t kMaxGroups = 6, kMaxAlpha = 258, kMaxLen = 20, kGroupSize = 50, kMaxSelectors = 18002;
constexpr uint32_t kSplit = 256;                         // inverse BWT: every kSplit-th position is a splitter
constexpr uint32_t kMaxSplitters = 900000 / kSplit + 2;  // of the largest block, origPtr's start included

// why a walk, a chain or a later stage stopped (0: it did not)
enum : uint32_t {
    R_OK = 0,
    R_RANDOMISED,           // (unsupported) a randomised block
    R_SECOND_STREAM,        // (unsupported) a second stream after the first
    R_PAST,                 // the stream runs past the chunk
    R_NO_MAGIC,             // neither a block magic nor the end-of-stream magic where the previous block ended
    R_MAP_EMPTY,            // an empty symbol map
    R_GROUPS,               // nGroups outside 2..6
    R_SELECTORS0,           // nSelectors of 0
    R_SELECTOR,             // a selector MTF index >= nGroups
    R_CODE_LEN,             // a code length outside 1..20
    R_CODE_OVER,            // an over-subscribed code
    R_CODE_INCOMPLETE,      // an incomplete code
    R_NO_SYMBOL,            // a bit pattern that decodes to no symbol
    R_RUN_LONG,             // a RUNA/RUNB run longer than the block max
    R_BLOCK_LONG,           // a block longer than the block max
    R_NO_EOB,               // the selectors run out before the end-of-block symbol
    R_ORIGPTR,              // origPtr >= the block length
    R_RLE_END,              // four equal bytes end the block without their count
    R_BLOCK_CRC,            // a block CRC mismatch
    R_STREAM_CRC,           // the stream CRC mismatch
    R_TRAILING,             // bytes after the stream's padding
    R_SIZE,                 // the stream does not decode to the chunk's size
};

PCD_HD const char* reason_text(uint32_t r) {
    switch (r) {
    case R_RANDOMISED: return "a randomised block (bzip2 before 0.9.5) is not read";
    case R_SECOND_STREAM: return "a second bzip2 stream follows the first: concatenated streams are not read";
    case R_PAST: return "the stream runs past the chunk";
    case R_NO_MAGIC: return "neither a block magic nor the end-of-stream magic where the previous block ended";
    case R_MAP_EMPTY: return "an empty symbol map";
    case R_GROUPS: return "nGroups outside 2..6";
    case R_SELECTORS0: return "nSelectors of 0";
    case R_SELECTOR: return "a selector MTF index at or above nGroups";
    case R_CODE_LEN: return "a code length outside 1..20";
    case R_CODE_OVER: return "an over-subscribed Huffman code";
    case R_CODE_INCOMPLETE: return "an incomplete Huffman code";
    case R_NO_SYMBOL: return "a bit pattern that decodes to no symbol";
    case R_RUN_LONG: return "a RUNA/RUNB run longer than the block max";
    case R_BLOCK_LONG: return "a block longer than the block max";
    case R_NO_EOB: return "no end-of-block symbol before the selectors run out";
    case R_ORIGPTR: return "origPtr at or past the block length";
    case R_RLE_END: return "four equal bytes end the block without their RLE1 count";
    case R_BLOCK_CRC: return "the block CRC does not match";
    case R_STREAM_CRC: return "the stream CRC does not match";
    case R_TRAILING: return "the chunk's data goes on past the end of its bzip2 stream";
    case R_SIZE: return "the stream does not decode to the chunk's 'size'";
    default: return "no error";
    }
}

PCD_HD bool unsupported(uint32_t r) { return r == R_RANDOMISED || r == R_SECOND_STREAM; }

// the bits [0, end) of a chunk's data d, read most significant first; nothing at or past `end` is ever read
struct Bits {
    const uint8_t* d;
    uint64_t pos, end;
    PCD_HD bool have(uint32_t k) const { return end - pos >= k; }
    // the k (<= 32) bits at pos, bits past end read as 0
    PCD_HD uint32_t peek(uint32_t k) const {
        const uint64_t b0 = pos >> 3, nbytes = (end + 7) >> 3;
        const uint32_t sh = (uint32_t)(pos & 7u), nb = (sh + k + 7) >> 3;
        uint64_t w = 0;
        for (uint32_t i = 0; i < nb; ++i) w = w << 8 | (b0 + i < nbytes ? d[b0 + i] : 0u);
        w >>= nb * 8 - sh - k;
        if (end - pos < k) w &= ~((1ull << (k - (end - pos))) - 1);   // a partial last byte: its bits past end are not data
        return (uint32_t)(w & ((1ull << k) - 1));
    }
    PCD_HD uint32_t get(uint32_t k) { const uint32_t v = peek(k); pos += k; return v; }
};

// the 48 bits at bit `at` of d[0, nbytes) (at + 48 <= 8 nbytes)
PCD_HD uint64_t magic_at(const uint8_t* d, uint64_t at) {
    const uint64_t b0 = at >> 3;
    const uint32_t sh = (uint32_t)(at & 7u);
    uint64_t w = 0;
    for (uint32_t i = 0; i < (sh ? 7u : 6u); ++i) w = w << 8 | d[b0 + i];
    return (sh ? w >> (8 - sh) : w) & 0xFFFFFFFFFFFFull;
}

// one block's Huffman tables and symbol map, built by the walk
struct Tables {
    int32_t limit[kMaxGroups][kMaxLen + 1];   // the largest code of each length (first - 1 when none)
    int32_t base[kMaxGroups][kMaxLen + 1];    // code - base = the symbol's index in perm
    uint16_t perm[kMaxGroups][kMaxAlpha];     // symbols by (length, symbol)
    uint8_t min_len[kMaxGroups];
    uint8_t unseq[256];                       // MTF index -> byte
};

// the canonical code of group g from its lengths: R_OK, or over-subscribed / incomplete
PCD_HD uint32_t make_code(Tables& T, uint32_t g, const uint8_t* len, uint32_t alpha) {
    uint32_t count[kMaxLen + 1] = {0};
    uint32_t lo = kMaxLen, hi = 1;
    for (uint32_t s = 0; s < alpha; ++s) { ++count[len[s]]; lo = len[s] < lo ? len[s] : lo; hi = len[s] > hi ? len[s] : hi; }
    uint32_t pp = 0;
    for (uint32_t L = lo; L <= hi; ++L)
        for (uint32_t s = 0; s < alpha; ++s)
            if (len[s] == L) T.perm[g][pp++] = (uint16_t)s;
    int64_t code = 0;
    uint32_t idx = 0;
    for (uint32_t L = 1; L <= kMaxLen; ++L) {
        if (code + count[L] > (1ll << L)) return R_CODE_OVER;
        T.base[g][L] = (int32_t)(code - idx);
        T.limit[g][L] = (int32_t)(code + count[L]) - 1;
        idx += count[L];
        code = (code + count[L]) << 1;
    }
    if (code != (1ll << (kMaxLen + 1))) return R_CODE_INCOMPLETE;
    T.min_len[g] = (uint8_t)lo;
    return R_OK;
}

// what a walk found out about the block at its candidate's bit
struct Walk {
    uint64_t end;                    // the bit after its last symbol
    uint64_t where;                  // the bit where the rule broke (reason != 0)
    uint32_t n, crc, orig, reason;   // its length before RLE1, its stored CRC, origPtr
};

// The block whose magic is at bit `at` of a chunk's data bits [0, nbits) in a stream of `level`: the header, the tables, then the
// symbols to the end-of-block symbol.  tt == nullptr: the walk alone (length and end bit).  Else the BWT's last column is written to
// tt[0, n) (the MTF and run output) and its byte histogram to hist[256] (zeroed here).  Every rule is checked before the bits it
// guards are used; nothing is written past tt[level x 100 000).
PCD_HD Walk block(const uint8_t* d, uint64_t nbits, uint64_t at, uint32_t level, Tables& T, uint8_t* tt, uint32_t* hist) {
    Walk w{0, 0, 0, 0, 0, R_OK};
    Bits b{d, at + 48, nbits};
    const uint32_t nmax = level * 100000u;
    auto fail = [&](uint32_t r, uint64_t where) { w.reason = r; w.where = where; return w; };
    if (!b.have(57)) return fail(R_PAST, b.pos);
    w.crc = b.get(32);
    if (b.get(1)) return fail(R_RANDOMISED, b.pos - 1);
    w.orig = b.get(24);
    if (!b.have(16)) return fail(R_PAST, b.pos);
    const uint32_t used16 = b.get(16);
    uint32_t n_in_use = 0;
    for (uint32_t i = 0; i < 16; ++i) {
        if (!(used16 >> (15 - i) & 1u)) continue;
        if (!b.have(16)) return fail(R_PAST, b.pos);
        const uint32_t m = b.get(16);
        for (uint32_t j = 0; j < 16; ++j)
            if (m >> (15 - j) & 1u) T.unseq[n_in_use++] = (uint8_t)(16 * i + j);
    }
    if (!n_in_use) return fail(R_MAP_EMPTY, b.pos);
    const uint32_t alpha = n_in_use + 2;
    if (!b.have(3)) return fail(R_PAST, b.pos);
    const uint32_t ng = b.get(3);
    if (ng < 2 || ng > kMaxGroups) return fail(R_GROUPS, b.pos - 3);
    if (!b.have(15)) return fail(R_PAST, b.pos);
    const uint32_t nsel_all = b.get(15);
    if (!nsel_all) return fail(R_SELECTORS0, b.pos - 15);
    const uint32_t nsel = nsel_all < kMaxSelectors ? nsel_all : kMaxSelectors;
    const uint64_t sel0 = b.pos;
    for (uint32_t i = 0; i < nsel_all; ++i) {
        uint32_t j = 0;
        for (;;) {
            if (!b.have(1)) return fail(R_PAST, b.pos);
            if (!b.get(1)) break;
            if (++j >= ng) return fail(R_SELECTOR, b.pos - 1);
        }
    }
    uint8_t len[kMaxAlpha];
    for (uint32_t g = 0; g < ng; ++g) {
        if (!b.have(5)) return fail(R_PAST, b.pos);
        const uint64_t g0 = b.pos;
        uint32_t cur = b.get(5);
        for (uint32_t s = 0; s < alpha; ++s) {
            for (;;) {
                if (cur < 1 || cur > kMaxLen) return fail(R_CODE_LEN, b.pos);
                if (!b.have(1)) return fail(R_PAST, b.pos);
                if (!b.get(1)) break;
                if (!b.have(1)) return fail(R_PAST, b.pos);
                cur = b.get(1) ? cur - 1 : cur + 1;
            }
            len[s] = (uint8_t)cur;
        }
        const uint32_t r = make_code(T, g, len, alpha);
        if (r != R_OK) return fail(r, g0);
    }
    // the symbols; the selectors are read again, one per group of 50, from sel0 (already checked)
    Bits sb{d, sel0, nbits};
    uint8_t smtf[kMaxGroups] = {0, 1, 2, 3, 4, 5};
    uint8_t mtf[256];
    if (tt) {
        for (uint32_t i = 0; i < 256; ++i) { mtf[i] = (uint8_t)i; hist[i] = 0; }
    }
    const uint32_t eob = n_in_use + 1;
    uint32_t n = 0, groups = 0, left = 0, g = 0, run = 0, N = 1;
    for (;;) {
        if (!left) {
            if (groups == nsel) return fail(R_NO_EOB, b.pos);
            uint32_t j = 0;
            while (sb.get(1)) ++j;
            const uint8_t v = smtf[j];
            for (; j > 0; --j) smtf[j] = smtf[j - 1];
            smtf[0] = v;
            g = v;
            ++groups;
            left = kGroupSize;
        }
        --left;
        const uint64_t s0 = b.pos;
        const uint32_t v = b.peek(kMaxLen);
        uint32_t zn = T.min_len[g];
        while (zn <= kMaxLen && (int32_t)(v >> (kMaxLen - zn)) > T.limit[g][zn]) ++zn;
        if (zn > kMaxLen) return fail(R_NO_SYMBOL, s0);
        if (!b.have(zn)) return fail(R_PAST, s0);
        b.pos += zn;
        const uint32_t sym = T.perm[g][(int32_t)(v >> (kMaxLen - zn)) - T.base[g][zn]];
        if (sym <= 1) {                                   // RUNA / RUNB
            run += (sym + 1) * N;
            N <<= 1;
            if (run > nmax) return fail(R_RUN_LONG, s0);
            continue;
        }
        if (run) {
            if (run > nmax - n) return fail(R_RUN_LONG, s0);
            if (tt) {
                const uint8_t c = T.unseq[mtf[0]];
                for (uint32_t k = 0; k < run; ++k) tt[n + k] = c;
                hist[c] += run;
            }
            n += run;
            run = 0;
            N = 1;
        }
        if (sym == eob) break;
        if (n >= nmax) return fail(R_BLOCK_LONG, s0);
        if (tt) {
            uint32_t k = sym - 1;
            const uint8_t u = mtf[k];
            for (; k > 0; --k) mtf[k] = mtf[k - 1];
            mtf[0] = u;
            const uint8_t c = T.unseq[u];
            tt[n] = c;
            ++hist[c];
        }
        ++n;
    }
    if (w.orig >= n) return fail(R_ORIGPTR, at + 48 + 33);
    w.n = n;
    w.end = b.pos;
    return w;
}

// T of the inverse BWT from the last column L[0, n) and its histogram: T[cftab[L[i]]++] = i
PCD_HD void lf_vector(const uint8_t* L, uint32_t n, const uint32_t* hist, uint32_t* T) {
    uint32_t cf[256];
    uint32_t s = 0;
    for (uint32_t c = 0; c < 256; ++c) { cf[c] = s; s += hist[c]; }
    for (uint32_t i = 0; i < n; ++i) T[cf[L[i]]++] = i;
}

// the inverse BWT by one thread: out[k] = L[p_k], p_0 = T[orig], p_{k+1} = T[p_k]
PCD_HD void unbwt_serial(const uint8_t* L, const uint32_t* T, uint32_t n, uint32_t orig, uint8_t* out) {
    uint32_t p = T[orig];
    for (uint32_t k = 0; k < n; ++k) {
        out[k] = L[p];
        p = T[p];
    }
}

// The splitters of a block for the parallel inverse BWT: positions j = kSplit i (ids 0 .. ceil(n / kSplit) - 1), and p_0 = T[orig]
// when it is not one of them (id ceil(n / kSplit)).  The sublists from the splitters on p_0's cycle, ranked from p_0's, give
// out[0, m) for that cycle's length m; when m < n (a periodic block) out[k] = out[k mod m], which is the serial walk's output.
PCD_HD uint32_t split_count(uint32_t n) { return (n + kSplit - 1) / kSplit + 1; }
PCD_HD bool is_split(uint32_t p, uint32_t p0) { return p % kSplit == 0 || p == p0; }
PCD_HD uint32_t split_id(uint32_t p, uint32_t p0, uint32_t n) { return p % kSplit == 0 ? p / kSplit : (n + kSplit - 1) / kSplit; }
PCD_HD uint32_t split_pos(uint32_t id, uint32_t p0, uint32_t n) { return id == (n + kSplit - 1) / kSplit ? p0 : id * kSplit; }
// the sublist from splitter position s: its length to the next splitter, whose id goes to *next
PCD_HD uint32_t split_walk(const uint32_t* T, uint32_t s, uint32_t p0, uint32_t n, uint32_t* next) {
    uint32_t q = s, len = 0;
    do { q = T[q]; ++len; } while (!is_split(q, p0));
    *next = split_id(q, p0, n);
    return len;
}

// CRC-32 as bzip2 computes it
PCD_HD void crc_table(uint32_t t[256]) {
    for (uint32_t i = 0; i < 256; ++i) {
        uint32_t c = i << 24;
        for (int k = 0; k < 8; ++k) c = (c & 0x80000000u) ? (c << 1) ^ 0x04C11DB7u : c << 1;
        t[i] = c;
    }
}
PCD_HD uint32_t crc_byte(const uint32_t* t, uint32_t c, uint8_t b) { return (c << 8) ^ t[(c >> 24) ^ b]; }

// RLE1 of a block's BWT output x[0, n): out != nullptr writes the output; *osize its length, *crc its CRC.  R_OK or R_RLE_END.
PCD_HD uint32_t rle1(const uint8_t* x, uint32_t n, const uint32_t* t, uint8_t* out, uint64_t* osize, uint32_t* crc) {
    uint64_t o = 0;
    uint32_t c = 0xFFFFFFFFu, i = 0;
    while (i < n) {
        const uint8_t v = x[i];
        uint32_t r = 1;
        while (r < 4 && i + r < n && x[i + r] == v) ++r;
        uint32_t copies = r;
        if (r == 4) {
            if (i + 4 >= n) return R_RLE_END;
            copies += x[i + 4];
            ++i;
        }
        i += r;
        for (uint32_t k = 0; k < copies; ++k) {
            if (out) out[o + k] = v;
            c = crc_byte(t, c, v);
        }
        o += copies;
    }
    *osize = o;
    *crc = ~c;
    return R_OK;
}

// the candidates: every bit at or after 32 (the stream header) where the block magic starts and fits in the chunk's len bytes.
// The magic overlaps itself only at shifts of 45 or more, so byte p holds at most one start: 1 + its bit in the byte, or 0.
PCD_HD uint32_t candidate_at(const uint8_t* d, uint64_t len, uint64_t p) {
    for (uint32_t j = 0; j < 8; ++j) {
        const uint64_t bit = 8 * p + j;
        if (bit < 32 || bit + 48 > 8 * len) continue;
        if (magic_at(d, bit) == kBlockMagic) return j + 1;
    }
    return 0;
}

// the candidates a chunk of len bytes can hold at most (starts 45 bits apart at least)
PCD_HD uint64_t max_candidates(uint64_t len) { return 8 * len >= 48 ? (8 * len - 48) / 45 + 1 : 0; }

}  // namespace bz2
