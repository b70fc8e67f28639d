// pcd_kernels.cu -- the ASCII PCD codec on the device (DESIGN.md section 12): erasor_pcd_parse_ascii turns the text of a PCD file
// into float4 x y z intensity, erasor_pcd_format_ascii turns a cloud into the text write_pcd_ascii / save_pcd_ascii write.  The
// per-token arithmetic is pcd_codec.h, which the CPU test-suite also runs on the host.
//
// Parse: the header (a few hundred bytes) is read on the host.  On the device, over the data bytes:
//   1. k_pcd_nl_count     line ends per 64 KB chunk (16-byte loads; '\n' or a lone '\r', as Python's universal newlines read
//                         them), then an exclusive scan of the chunk counts;
//   2. k_pcd_nl_scatter   the start of every line, in order (a CTA-wide scan per 4 KB tile);
//   3. k_pcd_classify     1 for a data line (anything but blanks before the end or a '#'), then an exclusive scan: the row of a line;
//   4. k_pcd_parse        one thread per line: split on blanks, check every token against numpy's loadtxt grammar and the token count
//                         against FIELDS, parse the kept columns on the fast path; the first bad line wins an atomicMin;
//   5. k_pcd_parse_slow   one thread per row holding a token the fast path left (limbs in local memory), only when there is one.
// Format: k_pcd_fmt_len gives every line's length, an exclusive scan its offset, k_pcd_fmt_write writes it after the header.
// Load (erasor_pcd_load, DESIGN.md section 12.1): ascii goes to the parse above; binary is one pass of k_pcd_gather_tile; a
// binary_compressed stream is decoded by k_lzf_walk (speculative token discovery), k_lzf_compose (scan of the chunks' entry maps),
// k_lzf_records, k_lzf_expand / k_lzf_jump / k_lzf_fill (pointer jumping over back-references), then gathered by k_pcd_gather.
// Write (erasor_pcd_format, DESIGN.md section 12.3): binary is the header and the cloud copied; binary_compressed is k_pcd_soa, then
// k_lzf_encode (lzf_encode.h's segmented rule, one warp per segment) and k_lzf_compact after a scan of the segments' sizes.
// Bags (erasor_bag_*, DESIGN.md section 12.2): the index is bag_index.h, on the host; one k_bag_gather launch decodes the clouds of a
// load from the selected blobs.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/erasor_b200.h"
#include "bag_index.h"
#include "buffers.h"
#include "lzf_encode.h"
#include "pcd_binary.h"
#include "pcd_codec.h"

namespace {
constexpr int kThreads = 256;
constexpr uint64_t kTile = 16ull * kThreads;          // bytes per CTA iteration of the newline passes
constexpr uint64_t kChunk = 16ull * kTile;            // bytes per CTA of the newline passes
constexpr int kScanItems = 4;
constexpr uint64_t kScanTile = (uint64_t)kScanItems * kThreads;
constexpr int kMaxFields = 64;
constexpr int kSlowThreads = 64;
constexpr int kMaxLine = 4 * 15 + 4;                  // "-1.2345678e-45" is the longest value: 4 values, 3 blanks and '\n'

struct Fields {
    int n;
    int8_t slot[kMaxFields];                          // field k -> 0..3 (x, y, z, intensity) or -1 (validated, not kept)
};

struct PcdStats {
    unsigned long long err;                           // (0-based data line << 1) | (1: wrong token count), ~0 when none
    unsigned long long slow_tokens;
    unsigned long long slow_rows;
    unsigned long long total;                         // scan totals read back by the host
};

// the data bytes in a 16-byte aligned frame: byte j of the data is base[j + o], o = the data pointer's misalignment
struct Text {
    const uint8_t* base;
    uint64_t o, len;
    __device__ __forceinline__ uint8_t at(uint64_t j) const { return base[j + o]; }
};

// CTA-wide exclusive scan of one value per thread; *total gets the sum.  s: 32 + 1 entries.
__device__ __forceinline__ uint64_t cta_excl_scan(uint64_t v, uint64_t* s, uint64_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint64_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) s[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = lane < nw ? s[lane] : 0;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, w, d);
            if (lane >= d) w += y;
        }
        if (lane < nw) s[lane] = w;
        if (lane == 31) s[32] = w;
    }
    __syncthreads();
    const uint64_t r = x - v + (warp ? s[warp - 1] : 0);
    total = s[32];
    __syncthreads();
    return r;
}

// the 16 bytes of the frame at f (f % 16 == 0); bytes outside the data read as 0
__device__ __forceinline__ void load16(const Text& t, uint64_t f, uint8_t b[16]) {
    if (f >= t.o && f + 16 <= t.o + t.len) {
        const uint4 v = *reinterpret_cast<const uint4*>(t.base + f);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        for (int k = 0; k < 16; ++k) b[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    } else {
        for (int k = 0; k < 16; ++k) b[k] = (f + k >= t.o && f + k < t.o + t.len) ? t.base[f + k] : 0;
    }
}

__device__ __forceinline__ uint8_t byte_at(const Text& t, uint64_t f) { return (f >= t.o && f < t.o + t.len) ? t.base[f] : 0; }

// Line ends as Python's universal newlines read them (read_pcd_ascii opens the file in text mode): '\n', and a '\r' that no '\n'
// follows.  The '\r' of "\r\n" stays in its line as a blank.  after: the byte following the 16.
__device__ __forceinline__ bool ends_line(const uint8_t b[16], int k, uint8_t after) {
    return b[k] == '\n' || (b[k] == '\r' && (k < 15 ? b[k + 1] : after) != '\n');
}

__global__ void __launch_bounds__(kThreads) k_pcd_nl_count(Text t, uint32_t* cnt) {
    __shared__ uint32_t s;
    if (threadIdx.x == 0) s = 0;
    __syncthreads();
    const uint64_t end = t.o + t.len;
    uint32_t c = 0;
    for (uint64_t f = (uint64_t)blockIdx.x * kChunk + 16ull * threadIdx.x; f < (uint64_t)(blockIdx.x + 1) * kChunk && f < end; f += kTile) {
        uint8_t b[16];
        load16(t, f, b);
        const uint8_t after = byte_at(t, f + 16);
        for (int k = 0; k < 16; ++k) c += ends_line(b, k, after);
    }
    atomicAdd(&s, c);
    __syncthreads();
    if (threadIdx.x == 0) cnt[blockIdx.x] = s;
}

// line_start[1 + k] = the data offset after the k-th line end
__global__ void __launch_bounds__(kThreads) k_pcd_nl_scatter(Text t, const uint64_t* chunk_off, uint64_t* line_start) {
    __shared__ uint64_t s[33];
    const uint64_t end = t.o + t.len;
    uint64_t run = chunk_off[blockIdx.x];
    for (uint64_t tile = (uint64_t)blockIdx.x * kChunk; tile < (uint64_t)(blockIdx.x + 1) * kChunk && tile < end; tile += kTile) {
        const uint64_t f = tile + 16ull * threadIdx.x;
        uint8_t b[16];
        if (f < end) load16(t, f, b); else for (int k = 0; k < 16; ++k) b[k] = 0;
        const uint8_t after = f < end ? byte_at(t, f + 16) : 0;
        uint32_t c = 0;
        for (int k = 0; k < 16; ++k) c += ends_line(b, k, after);
        uint64_t tot;
        uint64_t at = run + cta_excl_scan(c, s, tot);
        for (int k = 0; k < 16; ++k)
            if (ends_line(b, k, after)) line_start[1 + at++] = f + k - t.o + 1;
        run += tot;
    }
}

__device__ __forceinline__ uint64_t line_end(const Text& t, const uint64_t* line_start, uint64_t nlines, uint64_t i) {
    return i + 1 < nlines ? line_start[i + 1] - 1 : t.len;
}

__global__ void __launch_bounds__(kThreads) k_pcd_classify(Text t, const uint64_t* line_start, uint64_t nlines, uint32_t* flag) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t p = line_start[i];
        const uint64_t e = line_end(t, line_start, nlines, i);
        while (p < e && pcd::is_ws(t.at(p))) ++p;
        flag[i] = (p < e && t.at(p) != '#') ? 1u : 0u;
    }
}

// exclusive scan of n uint32 into uint64: per-tile sums, one CTA over the tile sums (sums[ntiles] = total), per-tile apply
__global__ void __launch_bounds__(kThreads) k_pcd_scan_tiles(const uint32_t* in, uint64_t n, uint64_t* sums) {
    __shared__ uint64_t s[33];
    const uint64_t i0 = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    uint64_t v = 0;
    for (int k = 0; k < kScanItems; ++k) if (i0 + k < n) v += in[i0 + k];
    uint64_t tot;
    cta_excl_scan(v, s, tot);
    if (threadIdx.x == 0) sums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kThreads) k_pcd_scan_top(uint64_t* sums, uint64_t ntiles) {
    __shared__ uint64_t s[33];
    uint64_t run = 0;
    for (uint64_t b = 0; b < ntiles; b += kThreads) {
        const uint64_t i = b + threadIdx.x;
        const uint64_t v = i < ntiles ? sums[i] : 0;
        uint64_t tot;
        const uint64_t x = cta_excl_scan(v, s, tot);
        if (i < ntiles) sums[i] = run + x;
        run += tot;
    }
    if (threadIdx.x == 0) sums[ntiles] = run;
}

__global__ void __launch_bounds__(kThreads) k_pcd_scan_apply(const uint32_t* in, uint64_t n, const uint64_t* sums, uint64_t* out) {
    __shared__ uint64_t s[33];
    const uint64_t i0 = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
    uint32_t v[kScanItems];
    uint64_t sum = 0;
    for (int k = 0; k < kScanItems; ++k) { v[k] = i0 + k < n ? in[i0 + k] : 0u; sum += v[k]; }
    uint64_t tot;
    uint64_t at = sums[blockIdx.x] + cta_excl_scan(sum, s, tot);
    for (int k = 0; k < kScanItems; ++k) {
        if (i0 + k < n) out[i0 + k] = at;
        at += v[k];
    }
}

// One data line: its tokens through scan_token.  Returns false when the line is invalid (*wrong_count: the token count is not
// f.n); vals gets the kept columns that the fast path settled, *n_slow the kept tokens it left to the slow path.
__device__ __forceinline__ bool parse_line(const Text& t, uint64_t p, uint64_t e, const Fields& f, float vals[4], int* n_slow,
                                           bool* wrong_count) {
    int k = 0;
    *n_slow = 0;
    *wrong_count = false;
    uint8_t tok[32];
    while (true) {
        while (p < e && pcd::is_ws(t.at(p))) ++p;
        if (p >= e || t.at(p) == '#') break;
        const uint64_t a = p;
        while (p < e && !pcd::is_ws(t.at(p)) && t.at(p) != '#') ++p;
        if (k >= f.n) { *wrong_count = true; return false; }
        const int slot = f.slot[k];
        const uint64_t len = p - a;
        pcd::TokenScan r;
        if (len <= sizeof(tok)) {
            for (uint64_t j = 0; j < len; ++j) tok[j] = t.at(a + j);
            r = pcd::scan_token(tok, len, slot >= 0);
        } else {
            r = pcd::scan_token(t.base + t.o + a, len, slot >= 0);
        }
        if (r.kind == pcd::TOK_INVALID) return false;
        if (slot >= 0) {
            if (r.kind == pcd::TOK_SLOW) ++*n_slow;
            else vals[slot] = (float)r.value;
        }
        ++k;
    }
    if (k != f.n) { *wrong_count = true; return false; }
    return true;
}

__global__ void __launch_bounds__(kThreads) k_pcd_parse(Text t, const uint64_t* line_start, uint64_t nlines, uint32_t* flag,
                                                        const uint64_t* row_of_line, uint64_t points, Fields f, float4* out, PcdStats* st) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += (uint64_t)gridDim.x * blockDim.x) {
        if (!flag[i]) continue;
        const uint64_t row = row_of_line[i];
        if (row >= points) continue;                  // np.loadtxt(max_rows = POINTS) neither reads nor checks the rest
        float v[4] = {0.0f, 0.0f, 0.0f, 0.0f};
        int n_slow;
        bool wrong;
        if (!parse_line(t, line_start[i], line_end(t, line_start, nlines, i), f, v, &n_slow, &wrong)) {
            atomicMin(&st->err, (unsigned long long)((i << 1) | (wrong ? 1u : 0u)));
            continue;
        }
        out[row] = make_float4(v[0], v[1], v[2], v[3]);
        if (n_slow) {
            flag[i] = 2;
            atomicAdd(&st->slow_tokens, (unsigned long long)n_slow);
            atomicAdd(&st->slow_rows, 1ull);
        }
    }
}

// the rows k_pcd_parse flagged 2: their kept tokens that the fast path left, by exact big-integer arithmetic
__global__ void __launch_bounds__(kSlowThreads) k_pcd_parse_slow(Text t, const uint64_t* line_start, uint64_t nlines, const uint32_t* flag,
                                                                 const uint64_t* row_of_line, Fields f, float4* out) {
    pcd::Big D, A, B;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nlines; i += (uint64_t)gridDim.x * blockDim.x) {
        if (flag[i] != 2) continue;
        float* o = reinterpret_cast<float*>(out + row_of_line[i]);
        uint64_t p = line_start[i];
        const uint64_t e = line_end(t, line_start, nlines, i);
        for (int k = 0; k < f.n; ++k) {
            while (p < e && pcd::is_ws(t.at(p))) ++p;
            const uint64_t a = p;
            while (p < e && !pcd::is_ws(t.at(p)) && t.at(p) != '#') ++p;
            const int slot = f.slot[k];
            if (slot < 0) continue;
            const uint8_t* s = t.base + t.o + a;
            const pcd::TokenScan r = pcd::scan_token(s, p - a, true);
            if (r.kind != pcd::TOK_SLOW) continue;
            const double v = pcd::parse_slow_abs(s, p - a, D, A, B);
            o[slot] = (float)(r.neg ? -v : v);
        }
    }
}

__device__ __forceinline__ int format_point(float4 q, char* buf) {
    int n = pcd::format_g8(q.x, buf);
    buf[n++] = ' ';
    n += pcd::format_g8(q.y, buf + n);
    buf[n++] = ' ';
    n += pcd::format_g8(q.z, buf + n);
    buf[n++] = ' ';
    n += pcd::format_g8(q.w, buf + n);
    buf[n++] = '\n';
    return n;
}

__global__ void __launch_bounds__(kThreads) k_pcd_fmt_len(const float4* pts, uint64_t n, uint32_t* len) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        char buf[kMaxLine];
        len[i] = (uint32_t)format_point(pts[i], buf);
    }
}

__global__ void __launch_bounds__(kThreads) k_pcd_fmt_write(const float4* pts, uint64_t n, const uint64_t* off, uint8_t* text) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        char buf[kMaxLine];
        const int m = format_point(pts[i], buf);
        uint8_t* d = text + off[i];
        for (int k = 0; k < m; ++k) d[k] = (uint8_t)buf[k];
    }
}

thread_local std::string g_pcd_err;

using erasor::DeviceBuffer;
using erasor::PinnedBuffer;
using pcd::Header;
using pcd::parse_header;

// ---- binary and binary_compressed (DESIGN.md section 12.1; the per-item logic is pcd_binary.h) ----------------------------
constexpr int kGatherThreads = 256;
constexpr uint32_t kGatherTile = 16384;              // file bytes a CTA stages in shared memory per iteration
constexpr uint64_t kLzfChunk = 4096;                  // compressed bytes per chunk of the token discovery

// binary: a tile of points is staged with 16-byte aligned loads (bytes of a 16-byte block that lie outside the body are read one by
// one, so nothing outside [body, body + points * stride) is touched), then every thread extracts its points' four fields at any
// offset and stride and writes one 16-byte value per point
__global__ void __launch_bounds__(kGatherThreads) k_pcd_gather_tile(const uint8_t* body, uint64_t points, pcd::Gather g, uint32_t per_tile,
                                                                      uint4* out) {
    __shared__ __align__(16) uint8_t tile[kGatherTile + 32];
    const uintptr_t b = reinterpret_cast<uintptr_t>(body);
    for (uint64_t p0 = (uint64_t)blockIdx.x * per_tile; p0 < points; p0 += (uint64_t)gridDim.x * per_tile) {
        const uint64_t np = min((uint64_t)per_tile, points - p0);
        const uintptr_t lo = b + p0 * g.stride, hi = b + (p0 + np) * g.stride;
        const uintptr_t a0 = lo & ~uintptr_t(15), a1 = (hi + 15) & ~uintptr_t(15);
        for (uintptr_t a = a0 + 16u * threadIdx.x; a < a1; a += 16u * blockDim.x) {
            uint8_t* d = tile + (a - a0);
            if (a >= lo && a + 16 <= hi) {
                *reinterpret_cast<uint4*>(d) = *reinterpret_cast<const uint4*>(a);
            } else {
                for (int k = 0; k < 16; ++k) d[k] = (a + k >= lo && a + k < hi) ? *reinterpret_cast<const uint8_t*>(a + k) : 0;
            }
        }
        __syncthreads();
        const uint8_t* t = tile + (lo - a0);
        for (uint32_t i = threadIdx.x; i < np; i += blockDim.x) {
            uint32_t v[4];
            pcd::gather_point(t, g, i, v);
            out[p0 + i] = make_uint4(v[0], v[1], v[2], v[3]);
        }
        __syncthreads();
    }
}

// one thread per point, straight from global memory: the decompressed SoA blocks, and binary points wider than a tile
__global__ void __launch_bounds__(kGatherThreads) k_pcd_gather(const uint8_t* base, uint64_t points, pcd::Gather g, uint4* out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < points; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t v[4];
        pcd::gather_point(base, g, i, v);
        out[i] = make_uint4(v[0], v[1], v[2], v[3]);
    }
}

// Stage A: one thread per (chunk, entry)
__global__ void __launch_bounds__(kThreads) k_lzf_walk(const uint8_t* s, uint64_t csize, uint64_t nchunks, uint8_t* map, uint32_t* tokens,
                                                       uint32_t* bytes) {
    const uint64_t total = nchunks * pcd::kLzfEntries;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k = i / pcd::kLzfEntries;
        const uint64_t begin = k * kLzfChunk, end = min(begin + kLzfChunk, csize);
        const pcd::LzfWalk w = pcd::lzf_walk(s, csize, begin, end, (uint32_t)(i - k * pcd::kLzfEntries));
        map[i] = (uint8_t)w.exit;
        tokens[i] = w.tokens;
        bytes[i] = w.bytes;
    }
}

// one round of the inclusive scan of the chunks' entry maps under composition: out_k = in_k o in_(k-d) (k >= d)
__global__ void __launch_bounds__(kThreads) k_lzf_compose(const uint8_t* in, uint8_t* out, uint64_t nchunks, uint64_t d) {
    const uint64_t total = nchunks * pcd::kLzfEntries;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k = i / pcd::kLzfEntries;
        const int e = (int)(i - k * pcd::kLzfEntries);
        out[i] = k >= d ? pcd::lzf_compose(in + k * pcd::kLzfEntries, in + (k - d) * pcd::kLzfEntries, e) : in[i];
    }
}

// the true entry of every chunk (chunk 0 starts at its first byte) and its chain's token and byte counts
__global__ void __launch_bounds__(kThreads) k_lzf_true(const uint8_t* scanned, const uint32_t* tokens, const uint32_t* bytes, uint64_t nchunks,
                                                       uint32_t* entry, uint32_t* ctok, uint32_t* cbyt) {
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nchunks; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t e = k ? scanned[(k - 1) * pcd::kLzfEntries] : 0u;
        entry[k] = e;
        ctok[k] = tokens[k * pcd::kLzfEntries + e];
        cbyt[k] = bytes[k * pcd::kLzfEntries + e];
    }
}

// Stage B: one thread per chunk; the first broken rule of the stream wins an atomicMin
__global__ void __launch_bounds__(kThreads) k_lzf_records(const uint8_t* s, uint64_t csize, uint64_t usize, uint64_t nchunks, const uint32_t* entry,
                                                          const uint64_t* tok_off, const uint64_t* byte_off, pcd::LzfToken* rec,
                                                          unsigned long long* err) {
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nchunks; k += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t begin = k * kLzfChunk, end = min(begin + kLzfChunk, csize);
        uint64_t e;
        pcd::lzf_records(s, csize, usize, begin, end, entry[k], byte_off[k], rec + tok_off[k], &e);
        if (e != ~0ull) atomicMin(err, (unsigned long long)e);
    }
}

// Stage C
__global__ void __launch_bounds__(kThreads) k_lzf_expand(const pcd::LzfToken* rec, uint64_t ntok, const uint8_t* s, uint8_t* out, uint32_t* src,
                                                         uint64_t keep) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ntok; i += (uint64_t)gridDim.x * blockDim.x)
        if (rec[i].dst < keep) pcd::lzf_expand(rec[i], s, out, src, keep);
}

__global__ void __launch_bounds__(kThreads) k_lzf_jump(uint32_t* src, uint64_t keep, unsigned int* moved) {
    bool any = false;
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < keep; j += (uint64_t)gridDim.x * blockDim.x)
        any |= pcd::lzf_jump(src, j);
    if (__syncthreads_or(any) && threadIdx.x == 0) atomicOr(moved, 1u);
}

__global__ void __launch_bounds__(kThreads) k_lzf_fill(const uint32_t* src, uint8_t* out, uint64_t keep) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < keep; j += (uint64_t)gridDim.x * blockDim.x)
        pcd::lzf_fill(src, out, j);
}

// ---- the binary_compressed writer (DESIGN.md section 12.3; the rule is lzf_encode.h) ---------------------------------------
// the float4 cloud as x[n] | y[n] | z[n] | intensity[n]
__global__ void __launch_bounds__(kThreads) k_pcd_soa(const uint4* pts, uint64_t n, uint32_t* soa) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 v = pts[i];
        soa[i] = v.x;
        soa[n + i] = v.y;
        soa[2 * n + i] = v.z;
        soa[3 * n + i] = v.w;
    }
}

// warp-wide literal stretch s[0, n) as tokens at o (the byte layout of pcd::lzf_put_lits)
__device__ __forceinline__ void warp_put_lits(uint8_t* o, const uint8_t* s, uint32_t n, int lane) {
    for (uint32_t r = lane; r < pcd::lzf_lit_runs(n); r += 32) o[r * (pcd::kLzfMaxLit + 1)] = pcd::lzf_lit_control(n, r);
    for (uint32_t k = lane; k < n; k += 32) o[pcd::lzf_lit_at(k)] = s[k];
}

// pcd::lzf_match_len, 32 byte pairs per step: the first pair that differs, or the end, ends the match
__device__ __forceinline__ uint32_t warp_match_len(const uint8_t* s, uint32_t len, uint32_t i, uint32_t c, int lane) {
    const uint32_t most = min(len - i, pcd::kLzfMaxRef);
    for (uint32_t b = 3;; b += 32) {
        const uint32_t j = b + lane;
        const unsigned stop = __ballot_sync(0xFFFFFFFFu, j >= most || s[c + j] != s[i + j]);
        if (stop) return b + __ffs(stop) - 1;
    }
}

// One warp per segment.  The table sweep goes 32 positions a step: lanes whose three bytes hash alike (__match_any_sync) take
// the nearest lower such lane as their candidate, the lowest of them the table's entry; then the highest of them enters the table.
// This is cand(i) of lzf_encode.h for every position.  The greedy parse trails the sweep: in each step's window it takes the first
// position at or past its own whose candidate counts (a ballot), extends the match 32 bytes at a time, and writes the literals
// before it and the reference.  Tokens go to the segment's slot of pcd::lzf_segment_cap(kLzfSeg) bytes.
__global__ void __launch_bounds__(32) k_lzf_encode(const uint8_t* soa, uint64_t usize, uint8_t* slots, uint64_t slot_cap, uint32_t* seg_len,
                                                     uint32_t* seg_tok) {
    __shared__ uint16_t table[pcd::kLzfHashSize];
    const int lane = threadIdx.x;
    const uint64_t seg = blockIdx.x, base0 = seg * pcd::kLzfSeg;
    const uint32_t len = (uint32_t)min((uint64_t)pcd::kLzfSeg, usize - base0);
    const uint8_t* s = soa + base0;
    uint8_t* o = slots + seg * slot_cap;
    for (uint32_t h = lane; h < pcd::kLzfHashSize; h += 32) table[h] = 0;
    __syncwarp();
    const uint32_t npos = pcd::lzf_positions(len);
    uint32_t olen = 0, ntok = 0, lit = 0, p = 0;                        // warp-uniform
    for (uint32_t base = 0; base < npos; base += 32) {
        const uint32_t i = base + lane;
        const bool act = i < npos;
        const uint32_t h = act ? pcd::lzf_hash(s + i) : pcd::kLzfHashSize + lane;   // idle lanes match nobody
        const unsigned same = __match_any_sync(0xFFFFFFFFu, h);
        const unsigned lower = same & ((1u << lane) - 1u);
        uint32_t c = 0;
        bool has = false;
        if (lower) { c = base + 31 - __clz(lower); has = true; }
        else if (act) { const uint32_t t = table[h]; has = t != 0; c = t - 1; }
        const bool ok = act && has && pcd::lzf_cand_ok(s, i, c);
        __syncwarp();
        if (act && (same >> lane) == 1u) table[h] = (uint16_t)(i + 1);   // the group's highest lane
        __syncwarp();
        const unsigned valid = __ballot_sync(0xFFFFFFFFu, ok);
        while (p < base + 32) {
            const unsigned m = valid & (~0u << (p - base));
            if (!m) { p = base + 32; break; }
            const uint32_t q = base + __ffs(m) - 1;
            const uint32_t cq = __shfl_sync(0xFFFFFFFFu, c, q - base);
            const uint32_t l = warp_match_len(s, len, q, cq, lane);
            warp_put_lits(o + olen, s + lit, q - lit, lane);
            olen += q - lit + pcd::lzf_lit_runs(q - lit);
            ntok += pcd::lzf_lit_runs(q - lit) + 1;
            if (lane == 0) pcd::lzf_put_ref(o + olen, l, q - cq);
            olen += l - 2 < 7 ? 2 : 3;
            p = lit = q + l;
        }
    }
    warp_put_lits(o + olen, s + lit, len - lit, lane);
    olen += len - lit + pcd::lzf_lit_runs(len - lit);
    ntok += pcd::lzf_lit_runs(len - lit);
    if (lane == 0) { seg_len[seg] = olen; seg_tok[seg] = ntok; }
}

// segment k's tokens from its slot to the stream at off[k]
__global__ void __launch_bounds__(kThreads) k_lzf_compact(const uint8_t* slots, uint64_t slot_cap, const uint32_t* seg_len, const uint64_t* off,
                                                          uint8_t* stream) {
    const uint64_t k = blockIdx.x;
    const uint8_t* src = slots + k * slot_cap;
    uint8_t* dst = stream + off[k];
    for (uint32_t j = threadIdx.x; j < seg_len[k]; j += blockDim.x) dst[j] = src[j];
}

// ---- erasor/node bags (DESIGN.md section 12.2; the index and the per-point decode are bag_index.h) --------------------------
// One cloud of a erasor_bag_load call.  A cloud whose rows are contiguous (row_step == width x point_step, or one row) is one row
// of n points; otherwise each of its rows is tiled on its own, so that a tile never spans row padding.
struct BagDesc {
    uint64_t src;                    // the cloud's data in the device copy of the blobs (16-byte aligned), or in the decoded chunks
    uint64_t out;                    // its first output point
    uint64_t tile0;                  // its first tile
    uint64_t cols;                   // points per row as tiled
    uint64_t tiles_per_row;
    uint32_t per_tile;               // points per tile
    uint32_t staged;                 // 1: a tile's bytes are staged in shared memory; 0: read from global memory point by point
    uint32_t reach;                  // bag::point_reach
    uint32_t lz4;                    // 1: src is in the decoded chunks (lz4 or bz2)
    bag::Cloud c;
};

// one CTA per tile: the cloud by binary search over tile0, then as k_pcd_gather_tile, at the cloud's row_step and point_step
__global__ void __launch_bounds__(kGatherThreads) k_bag_gather(const uint8_t* blobs, const uint8_t* dec, const BagDesc* d, int nclouds, uint64_t ntiles,
                                                                uint4* out) {
    __shared__ __align__(16) uint8_t tile[kGatherTile + 32];
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int lo = 0, hi = nclouds - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (d[mid].tile0 <= t) lo = mid; else hi = mid - 1;
        }
        const BagDesc& D = d[lo];
        const uint64_t lt = t - D.tile0, r = lt / D.tiles_per_row, c0 = (lt - r * D.tiles_per_row) * D.per_tile;
        const uint32_t np = (uint32_t)min((uint64_t)D.per_tile, D.cols - c0);
        const uint32_t step = D.c.point_step;
        const uint8_t* src = (D.lz4 ? dec : blobs) + D.src + r * D.c.row_step + c0 * step;
        uint4* o = out + D.out + r * D.cols + c0;
        if (D.staged) {
            const uintptr_t lo_a = reinterpret_cast<uintptr_t>(src), hi_a = lo_a + (uint64_t)(np - 1) * step + D.reach;
            const uintptr_t a0 = lo_a & ~uintptr_t(15), a1 = (hi_a + 15) & ~uintptr_t(15);
            for (uintptr_t a = a0 + 16u * threadIdx.x; a < a1; a += 16u * blockDim.x) {
                uint8_t* dst = tile + (a - a0);
                if (a >= lo_a && a + 16 <= hi_a) {
                    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(a);
                } else {
                    for (int k = 0; k < 16; ++k) dst[k] = (a + k >= lo_a && a + k < hi_a) ? *reinterpret_cast<const uint8_t*>(a + k) : 0;
                }
            }
            __syncthreads();
            const uint8_t* s = tile + (lo_a - a0);
            for (uint32_t j = threadIdx.x; j < np; j += blockDim.x) {
                uint32_t v[4];
                bag::point_values(s + (uint64_t)j * step, D.c, v);
                o[j] = make_uint4(v[0], v[1], v[2], v[3]);
            }
            __syncthreads();
        } else {
            for (uint32_t j = threadIdx.x; j < np; j += blockDim.x) {
                uint32_t v[4];
                bag::point_values(src + (uint64_t)j * step, D.c, v);
                o[j] = make_uint4(v[0], v[1], v[2], v[3]);
            }
        }
    }
}

// ---- lz4 chunks of a bag (DESIGN.md section 12.2.1; the rules are lz4_frame.h, the plan and the node layout bag_index.h) --------
// A warp walking one block: lane 0 parses each sequence and broadcasts it, the copies use all 32 lanes
struct Warp {
    PCD_HD uint32_t lane() const {
#ifdef __CUDA_ARCH__
        return threadIdx.x & 31u;
#else
        return 0;
#endif
    }
    PCD_HD uint32_t lanes() const { return 32; }
    PCD_HD void sync() const {
#ifdef __CUDA_ARCH__
        __syncwarp();
#endif
    }
    PCD_HD uint32_t bcast(uint32_t v) const {
#ifdef __CUDA_ARCH__
        return __shfl_sync(0xFFFFFFFFu, v, 0);
#else
        return v;
#endif
    }
};

// 1. one thread per block: its decoded size, from the token walk without copies (every rule checked)
__global__ void __launch_bounds__(kThreads) k_lz4_size(const uint8_t* src, const bag::Lz4Block* blk, uint64_t nb, uint32_t* bsize,
                                                       unsigned long long* err) {
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Lz4Block B = blk[b];
        uint32_t o = B.csize, at = 0, r = lz4::R_OK;
        if (!B.stored) r = lz4::block(lz4::Serial{}, src + B.src, B.csize, nullptr, B.cap, &o, &at);
        if (r != lz4::R_OK) atomicMin(err, (unsigned long long)bag::block_key(B, b, at, r));
        bsize[b] = r == lz4::R_OK ? o : 0u;
    }
}

// 2. one thread per chunk: its blocks' places in the decoded buffer (a serial scan: a chunk holds a few blocks), ~0 for every block
// of a chunk that does not decode to its size
__global__ void __launch_bounds__(kThreads) k_lz4_place(const bag::Lz4ChunkDesc* cd, uint64_t nc, const uint32_t* bsize, uint64_t* boff,
                                                        unsigned long long* err) {
    for (uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Lz4ChunkDesc d = cd[c];
        uint64_t s = 0;
        for (uint32_t b = d.block0; b < d.block0 + d.nblocks; ++b) s += bsize[b];
        const bool ok = s == d.size;
        if (!ok) atomicMin(err, (unsigned long long)bag::chunk_key(d, c, lz4::R_SIZE));
        s = 0;
        for (uint32_t b = d.block0; b < d.block0 + d.nblocks; ++b) { boff[b] = ok ? d.dec + s : ~0ull; s += bsize[b]; }
    }
}

// 3. one warp per block: the decode straight into place
__global__ void __launch_bounds__(kThreads) k_lz4_decode(const uint8_t* src, const bag::Lz4Block* blk, uint64_t nb, const uint32_t* bsize,
                                                         const uint64_t* boff, uint8_t* dec) {
    const uint64_t nw = (uint64_t)gridDim.x * (blockDim.x >> 5);
    for (uint64_t b = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; b < nb; b += nw) {
        const uint64_t at = boff[b];
        if (at == ~0ull) continue;
        const bag::Lz4Block B = blk[b];
        if (B.stored) {
            for (uint32_t k = threadIdx.x & 31u; k < B.csize; k += 32) dec[at + k] = src[B.src + k];
        } else {
            uint32_t o, e;
            lz4::block(Warp{}, src + B.src, B.csize, dec + at, bsize[b], &o, &e);
        }
    }
}

// 4. XXH32 is one serial chain per input: one thread per block checksum (blocks are small)
__global__ void __launch_bounds__(kThreads) k_lz4_sums(const uint8_t* src, const bag::Lz4Block* blk, uint64_t nb, unsigned long long* err) {
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Lz4Block B = blk[b];
        if (B.has_sum && lz4::xxh32(src + B.src, B.csize, 0) != B.sum) atomicMin(err, (unsigned long long)bag::block_key(B, b, B.csize, lz4::R_BLOCK_SUM));
    }
}

// ... and four threads per content checksum, one per XXH32 accumulator (independent chains over the 16-byte stripes of the chunk,
// 16-byte aligned in the decoded buffer, so each reads aligned words); CTAs of kContentThreads spread the chunks over the SMs
constexpr int kContentThreads = 32;
__global__ void __launch_bounds__(kContentThreads) k_lz4_content(const bag::Lz4ChunkDesc* cd, uint64_t nc, const uint8_t* dec, unsigned long long* err) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, c = t >> 2;
    const uint32_t j = (uint32_t)(t & 3u);
    const bool live = c < nc;
    const bag::Lz4ChunkDesc d = live ? cd[c] : bag::Lz4ChunkDesc{};
    const uint8_t* p = dec + d.dec;
    uint32_t v[4];
    const uint32_t mine = live && d.has_sum ? lz4::xxh32_lane(p, d.size, 0, j) : 0u;
    const uint32_t q = threadIdx.x & ~3u;
    for (uint32_t k = 0; k < 4; ++k) v[k] = __shfl_sync(0xFFFFFFFFu, mine, q + k);
    if (live && j == 0 && d.has_sum && lz4::xxh32_merge(v, p, d.size, 0) != d.sum)
        atomicMin(err, (unsigned long long)bag::chunk_key(d, c, lz4::R_CONTENT_SUM));
}

// 5. one thread per kept node in an LZ4 chunk: the record its index entry points to, then the node layout (bag::parse_node_core)
__global__ void __launch_bounds__(kThreads) k_bag_parse(const uint8_t* dec, const bag::Lz4NodeIn* in, uint64_t n, bag::NodeOut* out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Lz4NodeIn q = in[i];
        bag::NodeOut r{};
        uint64_t d0 = 0, d1 = 0;
        r.code = bag::record_core(dec + q.dec, q.len, q.rec, q.conn, q.time_ns, &d0, &d1, &r.a);
        if (r.code == bag::NF_OK) r.code = bag::parse_node_core(dec + q.dec, d0, d1, &r.seq, r.odom, r.cloud, &r.a, &r.b);
        out[i] = r;
    }
}

// ---- bz2 chunks of a bag (DESIGN.md section 12.2.2; the rules are bz2_stream.h, the plan, chain and placement bag_index.h) -----
constexpr int kBzWalkThreads = 8;                    // walk and decode: one bz2::Tables per thread in shared memory
constexpr int kBzBwtThreads = 512;                   // inverse BWT: one CTA per block

// the decoded bz2 chunk holding byte q of the device copy
__device__ uint32_t bz2_chunk_of(const bag::Bz2ChunkDesc* bd, uint32_t nc, uint64_t q) {
    uint32_t lo = 0, hi = nc - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (bd[mid].src <= q) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// 1a. one thread per byte of the copy: 1 when the block magic starts at one of its bits, else 0
__global__ void __launch_bounds__(kThreads) k_bz2_scan(const uint8_t* src, uint64_t nbytes, const bag::Bz2ChunkDesc* bd, uint32_t nc, uint32_t* flag) {
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nbytes; q += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Bz2ChunkDesc& D = bd[bz2_chunk_of(bd, nc, q)];
        const uint64_t p = q - D.src;
        flag[q] = p < D.len && bz2::candidate_at(src + D.src, D.len, p) ? 1u : 0u;
    }
}

// 1b. ... and after the scan of the flags, the candidates in bit order
__global__ void __launch_bounds__(kThreads) k_bz2_emit(const uint8_t* src, uint64_t nbytes, const bag::Bz2ChunkDesc* bd, uint32_t nc, const uint32_t* flag,
                                                       const uint64_t* off, bag::Bz2Cand* cand) {
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nbytes; q += (uint64_t)gridDim.x * blockDim.x) {
        if (!flag[q]) continue;
        const uint32_t c = bz2_chunk_of(bd, nc, q);
        const bag::Bz2ChunkDesc& D = bd[c];
        const uint64_t p = q - D.src;
        cand[off[q]] = bag::Bz2Cand{8 * p + bz2::candidate_at(src + D.src, D.len, p) - 1, c, 0};
    }
}

// 2. one thread per candidate: the speculative walk (header, tables, symbols to the end-of-block symbol; no writes)
__global__ void __launch_bounds__(kBzWalkThreads) k_bz2_walk(const uint8_t* src, const bag::Bz2ChunkDesc* bd, const bag::Bz2Cand* cand,
                                                             const uint64_t* ncand, bz2::Walk* walk) {
    extern __shared__ __align__(16) uint8_t bz_sh[];
    bz2::Tables& T = reinterpret_cast<bz2::Tables*>(bz_sh)[threadIdx.x];
    const uint64_t n = *ncand;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const bag::Bz2Cand C = cand[i];
        const bag::Bz2ChunkDesc& D = bd[C.chunk];
        walk[i] = bz2::block(src + D.src, 8 * D.len, C.bit, D.level, T, nullptr, nullptr);
    }
}

// 3. one thread per chunk: the chain of true blocks (bag::bz2_chain)
__global__ void __launch_bounds__(kThreads) k_bz2_chain(const uint8_t* src, const bag::Bz2ChunkDesc* bd, uint32_t nc, const bag::Bz2Cand* cand,
                                                        const uint64_t* off, const uint64_t* ncand, const bz2::Walk* walk, int32_t* blkno,
                                                        uint64_t* tt_off, uint32_t* nblocks, unsigned long long* err) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += gridDim.x * blockDim.x) {
        const bag::Bz2ChunkDesc& D = bd[c];
        const uint64_t c0 = off[D.src], c1 = c + 1 < nc ? off[bd[c + 1].src] : *ncand;
        const uint64_t k = bag::bz2_chain(c, D, src + D.src, cand, c0, c1, walk, blkno, tt_off, nblocks + c);
        if (k != ~0ull) atomicMin(err, (unsigned long long)k);
    }
}

// 4. one thread per true block: the walk again, now with the MTF and run output into its tt slot, then its LF vector
__global__ void __launch_bounds__(kBzWalkThreads) k_bz2_decode(const uint8_t* src, const bag::Bz2ChunkDesc* bd, const bag::Bz2Cand* cand,
                                                               const uint64_t* ncand, const uint64_t* tt_off, uint8_t* tt, uint32_t* lf) {
    extern __shared__ __align__(16) uint8_t bz_sh[];
    bz2::Tables& T = reinterpret_cast<bz2::Tables*>(bz_sh)[threadIdx.x];
    const uint64_t n = *ncand;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t at = tt_off[i];
        if (at == ~0ull) continue;
        const bag::Bz2Cand C = cand[i];
        const bag::Bz2ChunkDesc& D = bd[C.chunk];
        uint32_t hist[256];
        const bz2::Walk w = bz2::block(src + D.src, 8 * D.len, C.bit, D.level, T, tt + at, hist);
        bz2::lf_vector(tt + at, w.n, hist, lf + at);
    }
}

// 5. one CTA per true block: the inverse BWT by splitters (bz2_stream.h): every thread walks sublists to the next splitter, thread
// 0 ranks the splitters from origPtr's, every thread walks its sublists again, writing each byte at its rank, and a periodic
// block's cycle is repeated to its length
__global__ void __launch_bounds__(kBzBwtThreads) k_bz2_bwt(const uint64_t* ncand, const bz2::Walk* walk, const uint64_t* tt_off, const uint8_t* tt,
                                                           const uint32_t* lf, uint8_t* bw) {
    __shared__ uint32_t nxt[bz2::kMaxSplitters], len[bz2::kMaxSplitters], rank[bz2::kMaxSplitters];
    __shared__ uint32_t cycle;
    const uint64_t nc = *ncand;
    for (uint64_t i = blockIdx.x; i < nc; i += gridDim.x) {
        const uint64_t at = tt_off[i];
        if (at == ~0ull) continue;
        const uint32_t n = walk[i].n;
        const uint8_t* L = tt + at;
        const uint32_t* T = lf + at;
        const uint32_t p0 = T[walk[i].orig], ns = bz2::split_count(n);
        for (uint32_t s = threadIdx.x; s < ns; s += blockDim.x) {
            rank[s] = ~0u;
            if (s + 1 < ns || p0 % bz2::kSplit) len[s] = bz2::split_walk(T, bz2::split_pos(s, p0, n), p0, n, &nxt[s]);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t id0 = bz2::split_id(p0, p0, n);
            uint32_t s = id0, r = 0;
            do { rank[s] = r; r += len[s]; s = nxt[s]; } while (s != id0);
            cycle = r;
        }
        __syncthreads();
        for (uint32_t s = threadIdx.x; s < ns; s += blockDim.x) {
            if (rank[s] == ~0u) continue;
            uint32_t q = bz2::split_pos(s, p0, n), r = rank[s];
            for (uint32_t k = 0; k < len[s]; ++k) { bw[at + r + k] = L[q]; q = T[q]; }
        }
        __syncthreads();
        const uint32_t m = cycle;
        for (uint32_t k = m + threadIdx.x; k < n; k += blockDim.x) bw[at + k] = bw[at + k % m];
        __syncthreads();
    }
}

// 6. one thread per true block: RLE1's output length and the block CRC over it, checked
__global__ void __launch_bounds__(kThreads) k_bz2_rle(const bag::Bz2Cand* cand, const uint64_t* ncand, const bz2::Walk* walk, const uint64_t* tt_off,
                                                      const uint8_t* bw, uint64_t* osize, unsigned long long* err) {
    __shared__ uint32_t tab[256];
    if (threadIdx.x == 0) bz2::crc_table(tab);
    __syncthreads();
    const uint64_t nc = *ncand;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t at = tt_off[i];
        if (at == ~0ull) continue;
        uint64_t os = 0;
        uint32_t crc = 0;
        uint32_t r = bz2::rle1(bw + at, walk[i].n, tab, nullptr, &os, &crc);
        if (r == bz2::R_OK && crc != walk[i].crc) r = bz2::R_BLOCK_CRC;
        if (r != bz2::R_OK) atomicMin(err, (unsigned long long)bag::bz2_key(cand[i].chunk, cand[i].bit, r));
        osize[i] = r == bz2::R_OK ? os : ~0ull;
    }
}

// 7. one thread per chunk: the blocks' places in the decoded buffer (bag::bz2_place)
__global__ void __launch_bounds__(kThreads) k_bz2_place(const bag::Bz2ChunkDesc* bd, uint32_t nc, const uint64_t* off, const uint64_t* ncand,
                                                        const uint64_t* tt_off, const uint64_t* osize, uint64_t* out_off, unsigned long long* err) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < nc; c += gridDim.x * blockDim.x) {
        const bag::Bz2ChunkDesc& D = bd[c];
        const uint64_t c0 = off[D.src], c1 = c + 1 < nc ? off[bd[c + 1].src] : *ncand;
        const uint64_t k = bag::bz2_place(c, D, c0, c1, tt_off, osize, out_off);
        if (k != ~0ull) atomicMin(err, (unsigned long long)k);
    }
}

// 8. one thread per true block: RLE1 into place
__global__ void __launch_bounds__(kThreads) k_bz2_expand(const uint64_t* ncand, const bz2::Walk* walk, const uint64_t* tt_off, const uint64_t* out_off,
                                                         const uint8_t* bw, uint8_t* dec) {
    __shared__ uint32_t tab[256];
    if (threadIdx.x == 0) bz2::crc_table(tab);
    __syncthreads();
    const uint64_t nc = *ncand;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += (uint64_t)gridDim.x * blockDim.x) {
        if (out_off[i] == ~0ull) continue;
        uint64_t os = 0;
        uint32_t crc = 0;
        bz2::rle1(bw + tt_off[i], walk[i].n, tab, dec + out_off[i], &os, &crc);
    }
}

// 9. the block an error key names: the last block of its chunk starting at or before its bit
__global__ void __launch_bounds__(kThreads) k_bz2_errblock(const bag::Bz2Cand* cand, const uint64_t* ncand, const int32_t* blkno,
                                                           const unsigned long long* err, int* blk) {
    const uint64_t key = *err, nc = *ncand;
    if (key == ~0ull) return;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += (uint64_t)gridDim.x * blockDim.x)
        if (blkno[i] >= 0 && cand[i].chunk == key >> 44 && cand[i].bit <= ((key >> 8) & 0xFFFFFFFFFull)) atomicMax(blk, blkno[i]);
}

constexpr uint64_t kBagStage = 32ull << 20;          // bytes per pinned staging buffer (two) for a pageable file

uint32_t blocks_for(uint64_t n, int per, int cap) { return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((n + per - 1) / per, (uint64_t)cap)); }
}  // namespace

struct erasor_pcd_ctx {
    int device = 0;
    cudaStream_t st = nullptr;
    std::string err;
    DeviceBuffer text, chunk_cnt, chunk_off, lines, flags, rows, sums, out, stats;   // parse
    DeviceBuffer pts, lens, offs, ftext;                                              // format
    DeviceBuffer soa, lz_slots, lz_seglen, lz_segtok, lz_segoff, lz_segtokoff;          // format, binary_compressed
    DeviceBuffer lz_map0, lz_map1, lz_tok, lz_byt, lz_entry, lz_ctok, lz_cbyt, lz_tokoff, lz_byteoff, lz_rec, lz_src, lz_dec, lz_flags;   // load
    DeviceBuffer bag_blobs, bag_desc;                                                 // erasor_bag_load
    PinnedBuffer h_stats;                                                             // PcdStats
    int sm_count = 132;
    // erasor_bag_index's index and file (the caller's memory), and the pinned staging of a pageable file
    bag::Index bag;
    bool bag_ok = false, bag_pinned = false;
    const uint8_t* bag_file = nullptr;
    PinnedBuffer bag_stage[2];
    cudaEvent_t bag_ev[2] = {nullptr, nullptr};
    // the LZ4 chunks of the index: the plan, the decoded chunks (kept until the next erasor_bag_index), the decode's scratch (the
    // compressed copy z4_src is released when the index returns)
    bag::ChunkPlan z4;
    DeviceBuffer z4_src, z4_dec, z4_blk, z4_cd, z4_in, z4_bsize, z4_boff, z4_res;
    cudaEvent_t z4_ev[3] = {nullptr, nullptr, nullptr};
    double z4_decode_ms = 0, z4_sums_ms = 0;
    // the bz2 chunks' decode scratch (all of it released when the index returns), what it found and its stage times
    DeviceBuffer z2_src, z2_bd, z2_flag, z2_off, z2_cand, z2_walk, z2_blkno, z2_tt_off, z2_osize, z2_out_off, z2_tt, z2_lf, z2_bw;
    cudaEvent_t z2_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    bag::Bz2Found z2_found;
    uint64_t z2_scratch = 0;
    double z2_ms[4] = {0, 0, 0, 0};
    // erasor_pcd_format(_ascii)'s file of its last call (in ftext), kept for a following call with the same input and mode
    bool cached = false;
    const float* c_ptr = nullptr;
    size_t c_n = 0;
    int c_kind = -1, c_mode = -1;
    uint64_t c_len = 0;
    erasor_pcd_format_info_t c_info{};
};

namespace {
#define PCK(call) ERASOR_CUDA_TRY(p->err, call, #call)

int fail(erasor_pcd_t p, int rc, const std::string& msg) { p->err = msg; return rc; }

// exclusive scan of n uint32 at in into out (n uint64); *total = the sum (synchronous read-back when total != nullptr)
int scan_u32(erasor_pcd_t p, const uint32_t* in, uint64_t n, uint64_t* out, uint64_t* total) {
    const uint64_t ntiles = (n + kScanTile - 1) / kScanTile;
    PCK(p->sums.ensure(sizeof(uint64_t) * (ntiles + 1)));
    uint64_t* sums = p->sums.as<uint64_t>();
    k_pcd_scan_tiles<<<(unsigned)ntiles, kThreads, 0, p->st>>>(in, n, sums);
    k_pcd_scan_top<<<1, kThreads, 0, p->st>>>(sums, ntiles);
    k_pcd_scan_apply<<<(unsigned)ntiles, kThreads, 0, p->st>>>(in, n, sums, out);
    PCK(cudaGetLastError());
    if (total) {
        PCK(cudaMemcpyAsync(total, sums + ntiles, sizeof(uint64_t), cudaMemcpyDeviceToHost, p->st));
        PCK(cudaStreamSynchronize(p->st));
    }
    return ERASOR_OK;
}

// The header of a host or device file (from a device file, growing prefixes until the DATA line is in)
int read_header(erasor_pcd_t p, const char* text, uint64_t len, int text_kind, Header& h, bool& found) {
    found = false;
    if (text_kind == ERASOR_PTR_HOST) {
        found = parse_header(text, len, h);
        return ERASOR_OK;
    }
    std::vector<char> pre;
    for (uint64_t m = std::min<uint64_t>(len, 1 << 16);; m = std::min<uint64_t>(len, 4 * m)) {
        pre.resize(m);
        PCK(cudaMemcpy(pre.data(), text, m, cudaMemcpyDeviceToHost));
        h = Header();
        found = parse_header(pre.data(), m, h) && (h.data_off < m || m == len);   // the DATA line's end lies inside the prefix
        if (found || m == len) break;
    }
    return ERASOR_OK;
}

// The LZF stream s (device) -> p->lz_dec, of which the first keep bytes are materialised; the whole stream is validated.
int lzf_decode(erasor_pcd_t p, const uint8_t* s, uint64_t csize, uint64_t usize, uint64_t keep, uint64_t* ntok) {
    const uint64_t nchunks = (csize + kLzfChunk - 1) / kLzfChunk;
    const uint64_t nent = nchunks * pcd::kLzfEntries;
    const uint32_t g_ent = blocks_for(nent, kThreads, p->sm_count * 16), g_ch = blocks_for(nchunks, kThreads, p->sm_count * 16);
    *ntok = 0;
    if (!nchunks) return usize ? fail(p, ERASOR_E_INVALID, "malformed LZF stream: it ends after 0 of " + std::to_string(usize) + " bytes") : ERASOR_OK;
    // A. every chunk walked from each of its 33 possible entries, then the entry maps composed (log2(chunks) rounds)
    PCK(p->lz_map0.ensure(nent));
    PCK(p->lz_map1.ensure(nent));
    PCK(p->lz_tok.ensure(sizeof(uint32_t) * nent));
    PCK(p->lz_byt.ensure(sizeof(uint32_t) * nent));
    k_lzf_walk<<<g_ent, kThreads, 0, p->st>>>(s, csize, nchunks, p->lz_map0.as<uint8_t>(), p->lz_tok.as<uint32_t>(), p->lz_byt.as<uint32_t>());
    uint8_t *m_in = p->lz_map0.as<uint8_t>(), *m_out = p->lz_map1.as<uint8_t>();
    for (uint64_t d = 1; d < nchunks; d *= 2) {
        k_lzf_compose<<<g_ent, kThreads, 0, p->st>>>(m_in, m_out, nchunks, d);
        std::swap(m_in, m_out);
    }
    PCK(p->lz_entry.ensure(sizeof(uint32_t) * nchunks));
    PCK(p->lz_ctok.ensure(sizeof(uint32_t) * nchunks));
    PCK(p->lz_cbyt.ensure(sizeof(uint32_t) * nchunks));
    PCK(p->lz_tokoff.ensure(sizeof(uint64_t) * nchunks));
    PCK(p->lz_byteoff.ensure(sizeof(uint64_t) * nchunks));
    k_lzf_true<<<g_ch, kThreads, 0, p->st>>>(m_in, p->lz_tok.as<uint32_t>(), p->lz_byt.as<uint32_t>(), nchunks, p->lz_entry.as<uint32_t>(),
                                             p->lz_ctok.as<uint32_t>(), p->lz_cbyt.as<uint32_t>());
    PCK(cudaGetLastError());
    uint64_t tokens = 0, bytes = 0;
    int rc = scan_u32(p, p->lz_ctok.as<uint32_t>(), nchunks, p->lz_tokoff.as<uint64_t>(), &tokens);
    if (rc == ERASOR_OK) rc = scan_u32(p, p->lz_cbyt.as<uint32_t>(), nchunks, p->lz_byteoff.as<uint64_t>(), &bytes);
    if (rc != ERASOR_OK) return rc;
    *ntok = tokens;
    // B. token records along the true chain, every rule checked
    PCK(p->lz_rec.ensure(sizeof(pcd::LzfToken) * tokens));
    PCK(p->lz_flags.ensure(2 * sizeof(unsigned long long)));
    unsigned long long* flags = p->lz_flags.as<unsigned long long>();
    PCK(cudaMemsetAsync(flags, 0xFF, sizeof(unsigned long long), p->st));
    k_lzf_records<<<g_ch, kThreads, 0, p->st>>>(s, csize, usize, nchunks, p->lz_entry.as<uint32_t>(), p->lz_tokoff.as<uint64_t>(),
                                                p->lz_byteoff.as<uint64_t>(), p->lz_rec.as<pcd::LzfToken>(), flags);
    PCK(cudaGetLastError());
    unsigned long long err = 0;
    PCK(cudaMemcpyAsync(&err, flags, sizeof(err), cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    if (err != ~0ull) return fail(p, ERASOR_E_INVALID, pcd::lzf_error_message(err));
    if (bytes != usize)
        return fail(p, ERASOR_E_INVALID, "malformed LZF stream: it ends after " + std::to_string(bytes) + " of " + std::to_string(usize) + " bytes");
    // C. literals copied, every other byte resolved to the literal it copies by pointer jumping
    PCK(p->lz_dec.ensure(std::max<uint64_t>(keep, 1)));
    PCK(p->lz_src.ensure(sizeof(uint32_t) * std::max<uint64_t>(keep, 1)));
    uint8_t* dec = p->lz_dec.as<uint8_t>();
    uint32_t* src = p->lz_src.as<uint32_t>();
    const uint32_t g_keep = blocks_for(keep, kThreads, p->sm_count * 16);
    k_lzf_expand<<<blocks_for(tokens, kThreads, p->sm_count * 16), kThreads, 0, p->st>>>(p->lz_rec.as<pcd::LzfToken>(), tokens, s, dec, src, keep);
    PCK(cudaGetLastError());
    unsigned int* moved = reinterpret_cast<unsigned int*>(flags + 1);
    for (;;) {
        unsigned int h_moved = 0;
        PCK(cudaMemsetAsync(moved, 0, sizeof(unsigned int), p->st));
        k_lzf_jump<<<g_keep, kThreads, 0, p->st>>>(src, keep, moved);
        PCK(cudaMemcpyAsync(&h_moved, moved, sizeof(h_moved), cudaMemcpyDeviceToHost, p->st));
        PCK(cudaStreamSynchronize(p->st));
        if (!h_moved) break;
    }
    k_lzf_fill<<<g_keep, kThreads, 0, p->st>>>(src, dec, keep);
    PCK(cudaGetLastError());
    return ERASOR_OK;
}

// Bytes of the bag file to the device: span k is host[k][0, len) -> d + at (at increasing).  From a pinned file each span is one
// cudaMemcpyAsync; from a pageable one a window of the device layout at a time is filled on the host in one pinned buffer while
// the other one's copy runs.
struct Span { const uint8_t* host; uint64_t len, at; };

int upload_spans(erasor_pcd_t p, uint8_t* d, const std::vector<Span>& spans) {
    if (p->bag_pinned) {
        for (const Span& s : spans) PCK(cudaMemcpyAsync(d + s.at, s.host, s.len, cudaMemcpyHostToDevice, p->st));
        return ERASOR_OK;
    }
    for (int k = 0; k < 2; ++k) {
        if (!p->bag_stage[k].p()) PCK(p->bag_stage[k].allocate(kBagStage));
        if (!p->bag_ev[k]) PCK(cudaEventCreateWithFlags(&p->bag_ev[k], cudaEventDisableTiming));
    }
    int cur = 0;
    uint64_t w0 = 0, filled = 0;                      // the window [w0, w0 + kBagStage) of the device layout; bytes of it filled
    auto flush = [&]() -> cudaError_t {
        cudaError_t e = cudaMemcpyAsync(d + w0, p->bag_stage[cur].p(), filled, cudaMemcpyHostToDevice, p->st);
        if (e == cudaSuccess) e = cudaEventRecord(p->bag_ev[cur], p->st);
        cur ^= 1;
        w0 += filled;
        filled = 0;
        return e == cudaSuccess ? cudaEventSynchronize(p->bag_ev[cur]) : e;    // the buffer filled next is free again
    };
    PCK(cudaEventSynchronize(p->bag_ev[0]));
    PCK(cudaEventSynchronize(p->bag_ev[1]));
    for (const Span& s : spans) {
        uint64_t done = 0;
        while (done < s.len) {
            const uint64_t at = s.at + done;          // device offset of the next byte
            if (at - w0 >= kBagStage) PCK(flush());
            const uint64_t take = std::min(s.len - done, kBagStage - (at - w0));
            std::memcpy(p->bag_stage[cur].as<uint8_t>() + (at - w0), s.host + done, take);
            filled = at - w0 + take;
            done += take;
        }
    }
    if (filled) PCK(flush());
    return ERASOR_OK;
}

// The bz2 chunks of p->z4 into dec, launched on p->st after the LZ4 stages (no read-back): err gets the first broken rule's key,
// res[0] the total of candidates, blk the block the key names and nblocks each chunk's true blocks
int bz2_launch(erasor_pcd_t p, uint8_t* dec, unsigned long long* err, uint64_t* d_ncand_out, int* d_blk, uint32_t* d_nblocks) {
    const bag::ChunkPlan& P = p->z4;
    const uint32_t nc = (uint32_t)P.bd.size();
    const uint64_t nbytes = P.bz_src_bytes, cap_c = std::max<uint64_t>(P.bz_cands, 1), tt_bytes = std::max<uint64_t>(P.bz_tt_bytes, 16);
    const uint64_t ntiles = (nbytes + kScanTile - 1) / kScanTile;
    // every buffer sized from what the host has: the streams' bytes, the candidate bound and the BWT bound (bag_index.h)
    PCK(p->z2_src.ensure(nbytes));
    PCK(p->z2_bd.ensure(sizeof(bag::Bz2ChunkDesc) * nc));
    PCK(p->z2_flag.ensure(sizeof(uint32_t) * nbytes));
    PCK(p->z2_off.ensure(sizeof(uint64_t) * nbytes));
    PCK(p->z2_cand.ensure(sizeof(bag::Bz2Cand) * cap_c));
    PCK(p->z2_walk.ensure(sizeof(bz2::Walk) * cap_c));
    PCK(p->z2_blkno.ensure(sizeof(int32_t) * cap_c));
    PCK(p->z2_tt_off.ensure(sizeof(uint64_t) * cap_c));
    PCK(p->z2_osize.ensure(sizeof(uint64_t) * cap_c));
    PCK(p->z2_out_off.ensure(sizeof(uint64_t) * cap_c));
    PCK(p->z2_tt.ensure(tt_bytes));
    PCK(p->z2_lf.ensure(sizeof(uint32_t) * tt_bytes));
    PCK(p->z2_bw.ensure(tt_bytes));
    PCK(p->sums.ensure(sizeof(uint64_t) * (ntiles + 1)));
    p->z2_scratch = nbytes * (1 + sizeof(uint32_t) + sizeof(uint64_t)) + sizeof(bag::Bz2ChunkDesc) * nc + sizeof(uint64_t) * (ntiles + 1) +
                    cap_c * (sizeof(bag::Bz2Cand) + sizeof(bz2::Walk) + sizeof(int32_t) + 3 * sizeof(uint64_t)) + tt_bytes * (2 + sizeof(uint32_t));
    for (cudaEvent_t& ev : p->z2_ev)
        if (!ev) PCK(cudaEventCreate(&ev));
    std::vector<Span> spans;
    for (uint32_t c = 0; c < nc; ++c) spans.push_back(Span{p->bag_file + p->bag.bz2[P.bz_chunks[c]].data, P.bd[c].len, P.bd[c].src});
    uint8_t* src = p->z2_src.as<uint8_t>();
    int rc = upload_spans(p, src, spans);
    if (rc != ERASOR_OK) return rc;
    PCK(cudaMemcpyAsync(p->z2_bd.p(), P.bd.data(), sizeof(bag::Bz2ChunkDesc) * nc, cudaMemcpyHostToDevice, p->st));
    PCK(cudaMemsetAsync(p->z2_blkno.p(), 0xFF, sizeof(int32_t) * cap_c, p->st));
    PCK(cudaMemsetAsync(p->z2_tt_off.p(), 0xFF, sizeof(uint64_t) * cap_c, p->st));
    PCK(cudaMemsetAsync(p->z2_out_off.p(), 0xFF, sizeof(uint64_t) * cap_c, p->st));
    PCK(cudaMemsetAsync(d_nblocks, 0, sizeof(uint32_t) * nc, p->st));
    PCK(cudaMemsetAsync(d_blk, 0xFF, sizeof(int), p->st));
    const bag::Bz2ChunkDesc* bd = p->z2_bd.as<bag::Bz2ChunkDesc>();
    uint32_t* flag = p->z2_flag.as<uint32_t>();
    uint64_t* off = p->z2_off.as<uint64_t>();
    bag::Bz2Cand* cand = p->z2_cand.as<bag::Bz2Cand>();
    bz2::Walk* walk = p->z2_walk.as<bz2::Walk>();
    int32_t* blkno = p->z2_blkno.as<int32_t>();
    uint64_t *tt_off = p->z2_tt_off.as<uint64_t>(), *osize = p->z2_osize.as<uint64_t>(), *out_off = p->z2_out_off.as<uint64_t>();
    uint8_t *tt = p->z2_tt.as<uint8_t>(), *bw = p->z2_bw.as<uint8_t>();
    uint32_t* lf = p->z2_lf.as<uint32_t>();
    const uint64_t* ncand = p->sums.as<uint64_t>() + ntiles;          // the scan's total
    const int cap = p->sm_count * 16;
    const size_t sh_walk = sizeof(bz2::Tables) * kBzWalkThreads;
    const uint32_t g_walk = blocks_for(cap_c, kBzWalkThreads, p->sm_count * 32);
    PCK(cudaEventRecord(p->z2_ev[0], p->st));
    k_bz2_scan<<<blocks_for(nbytes, kThreads, cap), kThreads, 0, p->st>>>(src, nbytes, bd, nc, flag);
    rc = scan_u32(p, flag, nbytes, off, nullptr);
    if (rc != ERASOR_OK) return rc;
    k_bz2_emit<<<blocks_for(nbytes, kThreads, cap), kThreads, 0, p->st>>>(src, nbytes, bd, nc, flag, off, cand);
    k_bz2_walk<<<g_walk, kBzWalkThreads, sh_walk, p->st>>>(src, bd, cand, ncand, walk);
    k_bz2_chain<<<blocks_for(nc, kThreads, cap), kThreads, 0, p->st>>>(src, bd, nc, cand, off, ncand, walk, blkno, tt_off, d_nblocks, err);
    PCK(cudaEventRecord(p->z2_ev[1], p->st));
    k_bz2_decode<<<g_walk, kBzWalkThreads, sh_walk, p->st>>>(src, bd, cand, ncand, tt_off, tt, lf);
    PCK(cudaEventRecord(p->z2_ev[2], p->st));
    k_bz2_bwt<<<blocks_for(cap_c, 1, p->sm_count * 4), kBzBwtThreads, 0, p->st>>>(ncand, walk, tt_off, tt, lf, bw);
    PCK(cudaEventRecord(p->z2_ev[3], p->st));
    k_bz2_rle<<<blocks_for(cap_c, kThreads, cap), kThreads, 0, p->st>>>(cand, ncand, walk, tt_off, bw, osize, err);
    k_bz2_place<<<blocks_for(nc, kThreads, cap), kThreads, 0, p->st>>>(bd, nc, off, ncand, tt_off, osize, out_off, err);
    k_bz2_expand<<<blocks_for(cap_c, kThreads, cap), kThreads, 0, p->st>>>(ncand, walk, tt_off, out_off, bw, dec);
    PCK(cudaEventRecord(p->z2_ev[4], p->st));
    k_bz2_errblock<<<blocks_for(cap_c, kThreads, cap), kThreads, 0, p->st>>>(cand, ncand, blkno, err, d_blk);
    PCK(cudaMemcpyAsync(d_ncand_out, ncand, sizeof(uint64_t), cudaMemcpyDeviceToDevice, p->st));
    PCK(cudaGetLastError());
    return ERASOR_OK;
}

// erasor_bag_index's nodes in compressed chunks: the chunks holding one uploaded, decoded and checked in one submission (the LZ4
// stages, then the bz2 stages, into one decoded buffer), the nodes parsed, one read-back; then bag::finish_chunks
int bag_decode(erasor_pcd_t p, std::string& msg) {
    bag::ChunkPlan& P = p->z4;
    bag::plan_chunks(p->bag, P);
    const uint64_t nb = P.blocks.size(), nc = P.cd.size(), nn = P.nodes.size(), nz = P.bd.size();
    if (nz > bag::kMaxBz2Chunks) { msg = "more than 2^20 bz2 chunks hold kept nodes"; return ERASOR_E_CAPACITY; }
    if (nc) PCK(p->z4_src.ensure(std::max<uint64_t>(P.src_bytes, 16)));
    PCK(p->z4_dec.ensure(std::max<uint64_t>(P.dec_bytes, 16)));
    if (nc) {
        PCK(p->z4_blk.ensure(sizeof(bag::Lz4Block) * std::max<uint64_t>(nb, 1)));
        PCK(p->z4_cd.ensure(sizeof(bag::Lz4ChunkDesc) * nc));
        PCK(p->z4_bsize.ensure(sizeof(uint32_t) * std::max<uint64_t>(nb, 1)));
        PCK(p->z4_boff.ensure(sizeof(uint64_t) * std::max<uint64_t>(nb, 1)));
    }
    PCK(p->z4_in.ensure(sizeof(bag::Lz4NodeIn) * nn));
    // the node results, then the LZ4 key, the bz2 key, the bz2 candidates, the block the bz2 key names, the bz2 chunks' blocks
    const size_t res_bytes = sizeof(bag::NodeOut) * nn + 3 * sizeof(unsigned long long) + sizeof(int) + sizeof(uint32_t) * nz;
    PCK(p->z4_res.ensure(res_bytes));
    for (cudaEvent_t& ev : p->z4_ev)
        if (!ev) PCK(cudaEventCreate(&ev));
    uint8_t* dec = p->z4_dec.as<uint8_t>();
    bag::NodeOut* d_res = p->z4_res.as<bag::NodeOut>();
    unsigned long long* d_err = reinterpret_cast<unsigned long long*>(d_res + nn);
    PCK(cudaMemsetAsync(d_err, 0xFF, 2 * sizeof(unsigned long long), p->st));
    if (nc) {
        std::vector<Span> spans;
        for (size_t c = 0; c < nc; ++c) {
            const bag::Lz4Chunk& k = p->bag.lz4[P.chunks[c]];
            spans.push_back(Span{p->bag_file + k.data, k.len, P.cd[c].src});
        }
        uint8_t* src = p->z4_src.as<uint8_t>();
        const int rc = upload_spans(p, src, spans);
        if (rc != ERASOR_OK) return rc;
        if (nb) PCK(cudaMemcpyAsync(p->z4_blk.p(), P.blocks.data(), sizeof(bag::Lz4Block) * nb, cudaMemcpyHostToDevice, p->st));
        PCK(cudaMemcpyAsync(p->z4_cd.p(), P.cd.data(), sizeof(bag::Lz4ChunkDesc) * nc, cudaMemcpyHostToDevice, p->st));
        PCK(cudaMemcpyAsync(p->z4_in.p(), P.nodes.data(), sizeof(bag::Lz4NodeIn) * nn, cudaMemcpyHostToDevice, p->st));
        const bag::Lz4Block* blk = p->z4_blk.as<bag::Lz4Block>();
        const bag::Lz4ChunkDesc* cd = p->z4_cd.as<bag::Lz4ChunkDesc>();
        uint32_t* bsize = p->z4_bsize.as<uint32_t>();
        uint64_t* boff = p->z4_boff.as<uint64_t>();
        const int cap = p->sm_count * 16;
        PCK(cudaEventRecord(p->z4_ev[0], p->st));
        if (nb) k_lz4_size<<<blocks_for(nb, kThreads, cap), kThreads, 0, p->st>>>(src, blk, nb, bsize, d_err);
        k_lz4_place<<<blocks_for(nc, kThreads, cap), kThreads, 0, p->st>>>(cd, nc, bsize, boff, d_err);
        if (nb) k_lz4_decode<<<blocks_for(nb, kThreads / 32, cap), kThreads, 0, p->st>>>(src, blk, nb, bsize, boff, dec);
        PCK(cudaEventRecord(p->z4_ev[1], p->st));
        if (nb) k_lz4_sums<<<blocks_for(nb, kThreads, cap), kThreads, 0, p->st>>>(src, blk, nb, d_err);
        k_lz4_content<<<(unsigned)((4 * nc + kContentThreads - 1) / kContentThreads), kContentThreads, 0, p->st>>>(cd, nc, dec, d_err);
        PCK(cudaEventRecord(p->z4_ev[2], p->st));
    } else {
        PCK(cudaMemcpyAsync(p->z4_in.p(), P.nodes.data(), sizeof(bag::Lz4NodeIn) * nn, cudaMemcpyHostToDevice, p->st));
    }
    uint64_t* d_ncand = reinterpret_cast<uint64_t*>(d_err + 2);
    int* d_blk = reinterpret_cast<int*>(d_err + 3);
    uint32_t* d_nblocks = reinterpret_cast<uint32_t*>(d_blk + 1);
    if (nz) {
        const int rc = bz2_launch(p, dec, d_err + 1, d_ncand, d_blk, d_nblocks);
        if (rc != ERASOR_OK) return rc;
    }
    k_bag_parse<<<blocks_for(nn, kThreads, p->sm_count * 16), kThreads, 0, p->st>>>(dec, p->z4_in.as<bag::Lz4NodeIn>(), nn, d_res);
    PCK(cudaGetLastError());
    std::vector<uint8_t> res(res_bytes);
    PCK(cudaMemcpyAsync(res.data(), d_res, res_bytes, cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    if (nc) {
        float t0 = 0, t1 = 0;
        PCK(cudaEventElapsedTime(&t0, p->z4_ev[0], p->z4_ev[1]));
        PCK(cudaEventElapsedTime(&t1, p->z4_ev[1], p->z4_ev[2]));
        p->z4_decode_ms = t0;
        p->z4_sums_ms = t1;
    }
    const uint8_t* tail = res.data() + sizeof(bag::NodeOut) * nn;
    uint64_t keys[3];
    int blk = -1;
    std::memcpy(keys, tail, sizeof(keys));
    std::memcpy(&blk, tail + sizeof(keys), sizeof(int));
    if (nz) {
        p->z2_found.blocks.resize(nz);
        std::memcpy(p->z2_found.blocks.data(), tail + sizeof(keys) + sizeof(int), sizeof(uint32_t) * nz);
        p->z2_found.candidates = keys[2];
        for (int k = 0; k < 4; ++k) {
            float t = 0;
            PCK(cudaEventElapsedTime(&t, p->z2_ev[k], p->z2_ev[k + 1]));
            p->z2_ms[k] = t;
        }
    }
    const int rc = bag::decode_error(p->bag, P, keys[0], nz ? keys[1] : ~0ull, blk, msg);
    if (rc != ERASOR_OK) return rc;
    return bag::finish_chunks(p->bag, reinterpret_cast<const bag::NodeOut*>(res.data()), msg);
}

}  // namespace

extern "C" {

int erasor_pcd_create(int device, erasor_pcd_t* out) {
    if (!out) { g_pcd_err = "null argument"; return ERASOR_E_INVALID; }
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); g_pcd_err = "no CUDA device"; return ERASOR_E_CUDA; }
    if (device < 0 || device >= ndev) { g_pcd_err = "device index out of range"; return ERASOR_E_INVALID; }
    erasor_pcd_ctx* p = new erasor_pcd_ctx();
    p->device = device;
    cudaError_t c = cudaSetDevice(device);
    if (c == cudaSuccess) c = cudaStreamCreateWithFlags(&p->st, cudaStreamNonBlocking);
    if (c == cudaSuccess) c = p->h_stats.allocate(sizeof(PcdStats));
    if (c == cudaSuccess) c = p->stats.ensure(sizeof(PcdStats));
    if (c == cudaSuccess) c = cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, device);
    if (c != cudaSuccess) {
        g_pcd_err = std::string("erasor_pcd_create: ") + cudaGetErrorString(c);
        erasor_pcd_destroy(p);
        return ERASOR_E_CUDA;
    }
    *out = p;
    return ERASOR_OK;
}

void erasor_pcd_destroy(erasor_pcd_t p) {
    if (!p) return;
    cudaSetDevice(p->device);
    if (p->st) cudaStreamSynchronize(p->st);
    for (cudaEvent_t ev : p->bag_ev)
        if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : p->z4_ev)
        if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : p->z2_ev)
        if (ev) cudaEventDestroy(ev);
    if (p->st) cudaStreamDestroy(p->st);
    delete p;
}

const char* erasor_pcd_last_error(erasor_pcd_t p) { return p ? p->err.c_str() : g_pcd_err.c_str(); }

int erasor_pcd_parse_ascii(erasor_pcd_t p, const char* text, size_t len, int text_kind, float* out_xyzi, size_t cap, int out_kind,
                           size_t* n, erasor_pcd_info_t* info) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    p->cached = false;
    if (info) *info = erasor_pcd_info_t{};
    if (!n || (len && !text)) return fail(p, ERASOR_E_INVALID, "null argument");
    if ((text_kind != ERASOR_PTR_HOST && text_kind != ERASOR_PTR_DEVICE) || (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE))
        return fail(p, ERASOR_E_INVALID, "text_kind and out_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    PCK(cudaSetDevice(p->device));
    *n = 0;
    erasor_pcd_info_t inf{};
    // 1. the header, on the host
    Header h;
    bool found = false;
    const int hrc = read_header(p, text, len, text_kind, h, found);
    if (hrc != ERASOR_OK) return hrc;
    if (!found) return fail(p, ERASOR_E_INVALID, "no DATA line in the PCD header");
    for (size_t k = 0; k < h.fields.size(); ++k) {
        const std::string& f = h.fields[k];
        if (f == "x") inf.fields |= 1u; else if (f == "y") inf.fields |= 2u; else if (f == "z") inf.fields |= 4u; else if (f == "intensity") inf.fields |= 8u;
    }
    inf.has_intensity = (inf.fields & 8u) ? 1u : 0u;
    inf.points = h.points;
    inf.header_lines = h.lines;
    if (info) *info = inf;
    if (h.data != "ascii") return fail(p, ERASOR_E_UNSUPPORTED, "DATA " + h.data + ": only ASCII PCDs are parsed on the device");
    for (const std::string& c : h.counts)
        if (c != "1") return fail(p, ERASOR_E_UNSUPPORTED, "COUNT " + c + ": only fields with COUNT 1 are supported");
    if ((inf.fields & 7u) != 7u) return fail(p, ERASOR_E_INVALID, "the PCD's FIELDS lack x, y or z");
    if (h.fields.size() > (size_t)kMaxFields) return fail(p, ERASOR_E_UNSUPPORTED, "more than 64 FIELDS");
    if (!h.have_points) return fail(p, ERASOR_E_INVALID, "no valid POINTS line in the PCD header");
    if (!out_xyzi) { *n = (size_t)h.points; return ERASOR_OK; }
    if (cap < h.points) return fail(p, ERASOR_E_CAPACITY, "out_xyzi holds fewer points than the header's POINTS");
    if (out_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(out_xyzi) & 15u))
        return fail(p, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)");
    Fields f{};
    f.n = (int)h.fields.size();
    for (int k = 0; k < f.n; ++k) {
        const std::string& s = h.fields[k];
        f.slot[k] = s == "x" ? 0 : s == "y" ? 1 : s == "z" ? 2 : s == "intensity" ? 3 : -1;
    }
    const uint64_t dlen = len - h.data_off;
    if (!dlen || !h.points) { if (info) *info = inf; return ERASOR_OK; }

    // 2. the data bytes on the device, in a 16-byte aligned frame
    Text t{};
    if (text_kind == ERASOR_PTR_HOST) {
        PCK(p->text.ensure(dlen));
        PCK(cudaMemcpyAsync(p->text.p(), text + h.data_off, dlen, cudaMemcpyHostToDevice, p->st));
        t.base = p->text.as<uint8_t>();
        t.o = 0;
    } else {
        const uintptr_t a = reinterpret_cast<uintptr_t>(text) + h.data_off;
        t.base = reinterpret_cast<const uint8_t*>(a & ~uintptr_t(15));
        t.o = a & 15u;
    }
    t.len = dlen;

    // 3. line structure
    const uint64_t nchunks = (t.o + dlen + kChunk - 1) / kChunk;
    PCK(p->chunk_cnt.ensure(sizeof(uint32_t) * nchunks));
    PCK(p->chunk_off.ensure(sizeof(uint64_t) * nchunks));
    k_pcd_nl_count<<<(unsigned)nchunks, kThreads, 0, p->st>>>(t, p->chunk_cnt.as<uint32_t>());
    PCK(cudaGetLastError());
    uint64_t nl = 0;
    int rc = scan_u32(p, p->chunk_cnt.as<uint32_t>(), nchunks, p->chunk_off.as<uint64_t>(), &nl);
    if (rc != ERASOR_OK) return rc;
    const uint64_t nlines = nl + 1;
    if (nlines >= 0xFFFFFFFFull) return fail(p, ERASOR_E_UNSUPPORTED, "2^32 or more lines");
    PCK(p->lines.ensure(sizeof(uint64_t) * nlines));
    PCK(p->flags.ensure(sizeof(uint32_t) * nlines));
    PCK(p->rows.ensure(sizeof(uint64_t) * nlines));
    uint64_t* line_start = p->lines.as<uint64_t>();
    PCK(cudaMemsetAsync(line_start, 0, sizeof(uint64_t), p->st));
    k_pcd_nl_scatter<<<(unsigned)nchunks, kThreads, 0, p->st>>>(t, p->chunk_off.as<uint64_t>(), line_start);
    const uint32_t g_lines = blocks_for(nlines, kThreads, p->sm_count * 16);
    k_pcd_classify<<<g_lines, kThreads, 0, p->st>>>(t, line_start, nlines, p->flags.as<uint32_t>());
    PCK(cudaGetLastError());
    uint64_t data_rows = 0;
    rc = scan_u32(p, p->flags.as<uint32_t>(), nlines, p->rows.as<uint64_t>(), &data_rows);
    if (rc != ERASOR_OK) return rc;

    // 4. rows
    const uint64_t rows = std::min<uint64_t>(data_rows, h.points);
    float4* d_out = reinterpret_cast<float4*>(out_xyzi);
    if (out_kind == ERASOR_PTR_HOST) { PCK(p->out.ensure(sizeof(float4) * std::max<uint64_t>(rows, 1))); d_out = p->out.as<float4>(); }
    PcdStats* d_st = p->stats.as<PcdStats>();
    PcdStats* hs = p->h_stats.as<PcdStats>();
    std::memset(hs, 0, sizeof(PcdStats));
    hs->err = ~0ull;
    PCK(cudaMemcpyAsync(d_st, hs, sizeof(PcdStats), cudaMemcpyHostToDevice, p->st));
    k_pcd_parse<<<g_lines, kThreads, 0, p->st>>>(t, line_start, nlines, p->flags.as<uint32_t>(), p->rows.as<uint64_t>(), h.points, f, d_out, d_st);
    PCK(cudaGetLastError());
    PCK(cudaMemcpyAsync(hs, d_st, sizeof(PcdStats), cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    if (hs->err != ~0ull) {
        const unsigned long long line = h.lines + (hs->err >> 1) + 1;
        char msg[160];
        if (hs->err & 1u) std::snprintf(msg, sizeof(msg), "line %llu: the row does not hold exactly %d values (one per FIELDS entry)", line, f.n);
        else std::snprintf(msg, sizeof(msg), "line %llu: a value that is not a number", line);
        inf.error_line = line;
        if (info) *info = inf;
        return fail(p, ERASOR_E_INVALID, msg);
    }
    if (hs->slow_rows) {
        k_pcd_parse_slow<<<blocks_for(nlines, kSlowThreads, p->sm_count * 16), kSlowThreads, 0, p->st>>>(t, line_start, nlines, p->flags.as<uint32_t>(),
                                                                                                         p->rows.as<uint64_t>(), f, d_out);
        PCK(cudaGetLastError());
    }
    if (out_kind == ERASOR_PTR_HOST && rows) PCK(cudaMemcpyAsync(out_xyzi, d_out, sizeof(float4) * rows, cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    inf.rows = rows;
    inf.slow_tokens = hs->slow_tokens;
    if (info) *info = inf;
    *n = (size_t)rows;
    return ERASOR_OK;
}

int erasor_pcd_format_ascii(erasor_pcd_t p, const float* xyzi, size_t n, int in_kind, char* out, size_t cap, int out_kind, size_t* len) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (!len || (n && !xyzi)) return fail(p, ERASOR_E_INVALID, "null argument");
    if ((in_kind != ERASOR_PTR_HOST && in_kind != ERASOR_PTR_DEVICE) || (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE))
        return fail(p, ERASOR_E_INVALID, "in_kind and out_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    if (in_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(xyzi) & 15u))
        return fail(p, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)");
    PCK(cudaSetDevice(p->device));
    const bool hit = p->cached && p->c_ptr == xyzi && p->c_n == n && p->c_kind == in_kind && p->c_mode == ERASOR_PCD_ASCII;
    p->cached = false;
    if (!hit) {
        char head[512];
        const int hl = pcd::format_header(head, sizeof(head), n, ERASOR_PCD_ASCII);
        const float4* d_pts = reinterpret_cast<const float4*>(xyzi);
        if (in_kind == ERASOR_PTR_HOST && n) {
            PCK(p->pts.ensure(sizeof(float4) * n));
            PCK(cudaMemcpyAsync(p->pts.p(), xyzi, sizeof(float4) * n, cudaMemcpyHostToDevice, p->st));
            d_pts = p->pts.as<float4>();
        }
        uint64_t body = 0;
        if (n) {
            PCK(p->lens.ensure(sizeof(uint32_t) * n));
            PCK(p->offs.ensure(sizeof(uint64_t) * n));
            const uint32_t g = blocks_for(n, kThreads, p->sm_count * 16);
            k_pcd_fmt_len<<<g, kThreads, 0, p->st>>>(d_pts, n, p->lens.as<uint32_t>());
            PCK(cudaGetLastError());
            const int rc = scan_u32(p, p->lens.as<uint32_t>(), n, p->offs.as<uint64_t>(), &body);
            if (rc != ERASOR_OK) return rc;
        }
        const uint64_t total = (uint64_t)hl + body;
        PCK(p->ftext.ensure(total));
        PCK(cudaMemcpyAsync(p->ftext.p(), head, hl, cudaMemcpyHostToDevice, p->st));
        if (n) {
            k_pcd_fmt_write<<<blocks_for(n, kThreads, p->sm_count * 16), kThreads, 0, p->st>>>(d_pts, n, p->offs.as<uint64_t>(), p->ftext.as<uint8_t>() + hl);
            PCK(cudaGetLastError());
        }
        PCK(cudaStreamSynchronize(p->st));
        p->c_ptr = xyzi; p->c_n = n; p->c_kind = in_kind; p->c_mode = ERASOR_PCD_ASCII; p->c_len = total;
        p->c_info = erasor_pcd_format_info_t{};
        p->c_info.header_bytes = (uint64_t)hl;
    }
    *len = (size_t)p->c_len;
    if (!out || cap < p->c_len) {
        p->cached = true;                             // the following call with the same input fetches this text
        return out ? fail(p, ERASOR_E_CAPACITY, "out holds fewer bytes than the formatted text") : ERASOR_OK;
    }
    PCK(cudaMemcpyAsync(out, p->ftext.p(), p->c_len, out_kind == ERASOR_PTR_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, p->st));
    PCK(cudaStreamSynchronize(p->st));
    return ERASOR_OK;
}

int erasor_pcd_format(erasor_pcd_t p, const float* xyzi, size_t n, int in_kind, int data_mode, char* out, size_t cap, int out_kind,
                      size_t* len, erasor_pcd_format_info_t* info) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (data_mode == ERASOR_PCD_ASCII) {
        const int rc = erasor_pcd_format_ascii(p, xyzi, n, in_kind, out, cap, out_kind, len);
        if ((rc == ERASOR_OK || rc == ERASOR_E_CAPACITY) && info) *info = p->c_info;
        return rc;
    }
    if (data_mode != ERASOR_PCD_BINARY && data_mode != ERASOR_PCD_BINARY_COMPRESSED)
        return fail(p, ERASOR_E_INVALID, "data_mode must be ERASOR_PCD_ASCII, ERASOR_PCD_BINARY or ERASOR_PCD_BINARY_COMPRESSED");
    if (!len || (n && !xyzi)) return fail(p, ERASOR_E_INVALID, "null argument");
    if ((in_kind != ERASOR_PTR_HOST && in_kind != ERASOR_PTR_DEVICE) || (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE))
        return fail(p, ERASOR_E_INVALID, "in_kind and out_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    if (in_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(xyzi) & 15u))
        return fail(p, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)");
    const bool compressed = data_mode == ERASOR_PCD_BINARY_COMPRESSED;
    if (compressed && (n > 0xFFFFFFFFull / 16 || pcd::compressed_sizes_fit(16ull * n, 0) != ERASOR_OK))
        return fail(p, ERASOR_E_UNSUPPORTED, "binary_compressed: POINTS x 16 exceeds the format's uint32 uncompressed_size");
    PCK(cudaSetDevice(p->device));
    const bool hit = p->cached && p->c_ptr == xyzi && p->c_n == n && p->c_kind == in_kind && p->c_mode == data_mode;
    p->cached = false;
    if (!hit) {
        p->c_mode = -1;                               // ftext is about to change
        char head[512];
        const int hl = pcd::format_header(head, sizeof(head), n, data_mode);
        erasor_pcd_format_info_t inf{};
        inf.data_mode = (uint32_t)data_mode;
        inf.header_bytes = (uint64_t)hl;
        const uint64_t body = 16ull * n;
        if (!compressed) {                            // the points as they are
            PCK(p->ftext.ensure(hl + body));
            PCK(cudaMemcpyAsync(p->ftext.p(), head, hl, cudaMemcpyHostToDevice, p->st));
            if (n) PCK(cudaMemcpyAsync(p->ftext.as<uint8_t>() + hl, xyzi, body, in_kind == ERASOR_PTR_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, p->st));
            PCK(cudaStreamSynchronize(p->st));
            p->c_len = hl + body;
        } else {
            // the cloud as SoA, one warp per segment into worst-case slots, a scan of the segment sizes, then the slots compacted
            const uint64_t nseg = (body + pcd::kLzfSeg - 1) / pcd::kLzfSeg;
            const uint64_t slot = pcd::lzf_segment_cap(pcd::kLzfSeg);
            uint64_t csize = 0, ntok = 0;
            if (n) {
                const uint4* d_pts = reinterpret_cast<const uint4*>(xyzi);
                if (in_kind == ERASOR_PTR_HOST) {
                    PCK(p->pts.ensure(body));
                    PCK(cudaMemcpyAsync(p->pts.p(), xyzi, body, cudaMemcpyHostToDevice, p->st));
                    d_pts = p->pts.as<uint4>();
                }
                PCK(p->soa.ensure(body));
                PCK(p->lz_slots.ensure(nseg * slot));
                PCK(p->lz_seglen.ensure(sizeof(uint32_t) * nseg));
                PCK(p->lz_segtok.ensure(sizeof(uint32_t) * nseg));
                PCK(p->lz_segoff.ensure(sizeof(uint64_t) * nseg));
                PCK(p->lz_segtokoff.ensure(sizeof(uint64_t) * nseg));
                k_pcd_soa<<<blocks_for(n, kThreads, p->sm_count * 16), kThreads, 0, p->st>>>(d_pts, n, p->soa.as<uint32_t>());
                k_lzf_encode<<<(unsigned)nseg, 32, 0, p->st>>>(p->soa.as<uint8_t>(), body, p->lz_slots.as<uint8_t>(), slot, p->lz_seglen.as<uint32_t>(),
                                                              p->lz_segtok.as<uint32_t>());
                PCK(cudaGetLastError());
                int rc = scan_u32(p, p->lz_segtok.as<uint32_t>(), nseg, p->lz_segtokoff.as<uint64_t>(), nullptr);
                if (rc == ERASOR_OK) rc = scan_u32(p, p->lz_seglen.as<uint32_t>(), nseg, p->lz_segoff.as<uint64_t>(), &csize);
                if (rc != ERASOR_OK) return rc;
                PCK(cudaMemcpyAsync(&ntok, p->lz_segtokoff.as<uint64_t>() + (nseg - 1), sizeof(uint64_t), cudaMemcpyDeviceToHost, p->st));
                uint32_t last = 0;
                PCK(cudaMemcpyAsync(&last, p->lz_segtok.as<uint32_t>() + (nseg - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, p->st));
                PCK(cudaStreamSynchronize(p->st));
                ntok += last;
                if (pcd::compressed_sizes_fit(body, csize) != ERASOR_OK)
                    return fail(p, ERASOR_E_UNSUPPORTED, "binary_compressed: the LZF stream exceeds the format's uint32 compressed_size");
            }
            const uint64_t total = (uint64_t)hl + 8 + csize;
            PCK(p->ftext.ensure(total));
            const uint32_t sizes[2] = {(uint32_t)csize, (uint32_t)body};   // little-endian, as the device is
            PCK(cudaMemcpyAsync(p->ftext.p(), head, hl, cudaMemcpyHostToDevice, p->st));
            PCK(cudaMemcpyAsync(p->ftext.as<uint8_t>() + hl, sizes, 8, cudaMemcpyHostToDevice, p->st));
            if (n) {
                k_lzf_compact<<<(unsigned)nseg, kThreads, 0, p->st>>>(p->lz_slots.as<uint8_t>(), slot, p->lz_seglen.as<uint32_t>(), p->lz_segoff.as<uint64_t>(),
                                                                     p->ftext.as<uint8_t>() + hl + 8);
                PCK(cudaGetLastError());
            }
            PCK(cudaStreamSynchronize(p->st));
            p->c_len = total;
            inf.segments = (uint32_t)nseg;
            inf.uncompressed_size = body;
            inf.compressed_size = csize;
            inf.lzf_tokens = ntok;
        }
        p->c_ptr = xyzi; p->c_n = n; p->c_kind = in_kind; p->c_mode = data_mode; p->c_info = inf;
    }
    *len = (size_t)p->c_len;
    if (info) *info = p->c_info;
    if (!out || cap < p->c_len) {
        p->cached = true;                             // the following call with the same input and mode fetches this file
        return out ? fail(p, ERASOR_E_CAPACITY, "out holds fewer bytes than the formatted file") : ERASOR_OK;
    }
    PCK(cudaMemcpyAsync(out, p->ftext.p(), p->c_len, out_kind == ERASOR_PTR_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice, p->st));
    PCK(cudaStreamSynchronize(p->st));
    return ERASOR_OK;
}

int erasor_pcd_load(erasor_pcd_t p, const char* file, size_t len, int file_kind, float* out_xyzi, size_t cap, int out_kind, size_t* n,
                    erasor_pcd_load_info_t* info) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    p->cached = false;
    erasor_pcd_load_info_t inf{};
    if (info) *info = inf;
    auto done = [&](int rc) { if (info) *info = inf; return rc; };
    if (!n || (len && !file)) return fail(p, ERASOR_E_INVALID, "null argument");
    if ((file_kind != ERASOR_PTR_HOST && file_kind != ERASOR_PTR_DEVICE) || (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE))
        return fail(p, ERASOR_E_INVALID, "file_kind and out_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    PCK(cudaSetDevice(p->device));
    *n = 0;
    Header h;
    bool found = false;
    int rc = read_header(p, file, len, file_kind, h, found);
    if (rc != ERASOR_OK) return rc;
    if (!found) return fail(p, ERASOR_E_INVALID, "no DATA line in the PCD header");
    pcd::Layout L;
    std::string msg;
    rc = pcd::resolve_layout(h, L, msg);
    pcd::fill_load_info(h, L, inf);
    if (rc != ERASOR_OK) return done(fail(p, rc, msg));
    if (L.mode == pcd::DATA_ASCII) {
        rc = erasor_pcd_parse_ascii(p, file, len, file_kind, out_xyzi, cap, out_kind, n, &inf.ascii);
        inf.fields = inf.ascii.fields;
        return done(rc);
    }
    if (L.mode == pcd::DATA_BINARY && (rc = pcd::check_binary_body(L, h.data_off, len, msg)) != ERASOR_OK) return done(fail(p, rc, msg));
    if (!L.points) return done(ERASOR_OK);                                          // reads no data
    uint64_t csize = 0, usize = 0;
    if (L.mode == pcd::DATA_COMPRESSED) {
        if (len - h.data_off < 8) return done(fail(p, ERASOR_E_INVALID, "the file ends before compressed_size and uncompressed_size"));
        uint8_t sz[8];
        if (file_kind == ERASOR_PTR_HOST) std::memcpy(sz, file + h.data_off, 8);
        else PCK(cudaMemcpy(sz, file + h.data_off, 8, cudaMemcpyDeviceToHost));
        csize = pcd::le32(sz);
        usize = pcd::le32(sz + 4);
        inf.compressed_size = csize;
        inf.uncompressed_size = usize;
        if ((rc = pcd::check_compressed_sizes(L, h.data_off, len, csize, usize, msg)) != ERASOR_OK) return done(fail(p, rc, msg));
    }
    if (!out_xyzi) { *n = (size_t)L.points; return done(ERASOR_OK); }
    if (cap < L.points) return done(fail(p, ERASOR_E_CAPACITY, "out_xyzi holds fewer points than the header's POINTS"));
    if (out_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(out_xyzi) & 15u))
        return done(fail(p, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)"));

    // the body (binary) or the stream (binary_compressed) on the device
    const uint64_t body = L.mode == pcd::DATA_BINARY ? L.points * L.point_step : csize;
    const uint64_t at = h.data_off + (L.mode == pcd::DATA_BINARY ? 0 : 8);
    const uint8_t* d_in = reinterpret_cast<const uint8_t*>(file) + at;
    if (file_kind == ERASOR_PTR_HOST) {
        PCK(p->text.ensure(std::max<uint64_t>(body, 1)));
        PCK(cudaMemcpyAsync(p->text.p(), file + at, body, cudaMemcpyHostToDevice, p->st));
        d_in = p->text.as<uint8_t>();
    }
    uint4* d_out = reinterpret_cast<uint4*>(out_xyzi);
    if (out_kind == ERASOR_PTR_HOST) { PCK(p->out.ensure(sizeof(uint4) * L.points)); d_out = p->out.as<uint4>(); }
    const uint32_t g_pts = blocks_for(L.points, kGatherThreads, p->sm_count * 16);
    if (L.mode == pcd::DATA_BINARY) {
        if (L.point_step <= kGatherTile) {
            const uint32_t per_tile = (uint32_t)std::min<uint64_t>(4 * kGatherThreads, kGatherTile / L.point_step);
            k_pcd_gather_tile<<<blocks_for(L.points, per_tile, p->sm_count * 8), kGatherThreads, 0, p->st>>>(d_in, L.points, L.g, per_tile, d_out);
        } else {
            k_pcd_gather<<<g_pts, kGatherThreads, 0, p->st>>>(d_in, L.points, L.g, d_out);
        }
    } else {
        uint64_t ntok = 0;
        rc = lzf_decode(p, d_in, csize, usize, L.keep_end, &ntok);
        inf.lzf_tokens = ntok;
        if (rc != ERASOR_OK) { cudaStreamSynchronize(p->st); return done(rc); }
        k_pcd_gather<<<g_pts, kGatherThreads, 0, p->st>>>(p->lz_dec.as<uint8_t>(), L.points, L.g, d_out);
    }
    PCK(cudaGetLastError());
    if (out_kind == ERASOR_PTR_HOST) PCK(cudaMemcpyAsync(out_xyzi, d_out, sizeof(uint4) * L.points, cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    *n = (size_t)L.points;
    return done(ERASOR_OK);
}

int erasor_bag_index(erasor_pcd_t p, const char* file, size_t len, const char* topic, int keep_first, size_t* n_nodes, erasor_bag_info_t* info) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    p->cached = false;
    p->bag_ok = false;
    p->bag = bag::Index();
    p->z4 = bag::ChunkPlan();
    p->z4_decode_ms = p->z4_sums_ms = 0;
    p->z2_found = bag::Bz2Found();
    p->z2_scratch = 0;
    for (double& t : p->z2_ms) t = 0;
    p->bag_file = nullptr;
    if (info) *info = erasor_bag_info_t{};
    if (!n_nodes || (len && !file)) return fail(p, ERASOR_E_INVALID, "null argument");
    *n_nodes = 0;
    PCK(cudaSetDevice(p->device));
    std::string msg;
    int rc = bag::build_index(reinterpret_cast<const uint8_t*>(file), len, topic ? topic : "/node/combined/optimized", keep_first != 0, p->bag, msg);
    if (rc != ERASOR_OK) { p->bag = bag::Index(); return fail(p, rc, msg); }
    cudaPointerAttributes a{};
    p->bag_pinned = cudaPointerGetAttributes(&a, file) == cudaSuccess && a.type == cudaMemoryTypeHost;
    cudaGetLastError();
    p->bag_file = reinterpret_cast<const uint8_t*>(file);
    if (!p->bag.pending.empty()) {
        rc = bag_decode(p, msg);
        p->z4_src = DeviceBuffer();                  // the compressed copy is not needed past the index: only the decoded chunks stay
        for (DeviceBuffer* b : {&p->z2_src, &p->z2_bd, &p->z2_flag, &p->z2_off, &p->z2_cand, &p->z2_walk, &p->z2_blkno, &p->z2_tt_off,
                                &p->z2_osize, &p->z2_out_off, &p->z2_tt, &p->z2_lf, &p->z2_bw})
            *b = DeviceBuffer();                     // nor is any of the bz2 scratch
        if (rc != ERASOR_OK) {
            p->bag = bag::Index();
            p->z4 = bag::ChunkPlan();
            p->z2_found = bag::Bz2Found();
            p->bag_file = nullptr;
            return rc == ERASOR_E_CUDA ? rc : fail(p, rc, msg);
        }
    }
    p->bag_ok = true;
    *n_nodes = p->bag.nodes.size();
    if (info) bag::fill_info(p->bag, *info);
    return ERASOR_OK;
}

int erasor_bag_nodes(erasor_pcd_t p, size_t first, size_t count, uint32_t* seq, uint64_t* stamp_ns, double* odom7, erasor_bag_cloud_t* clouds) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (!p->bag_ok) return fail(p, ERASOR_E_STATE, "no bag indexed: call erasor_bag_index first");
    std::string msg;
    const int rc = bag::check_range(p->bag, first, count, msg);
    if (rc != ERASOR_OK) return fail(p, rc, msg);
    for (size_t k = 0; k < count; ++k) {
        const bag::Node& nd = p->bag.nodes[first + k];
        if (seq) seq[k] = nd.seq;
        if (stamp_ns) stamp_ns[k] = nd.stamp_ns;
        if (odom7) std::memcpy(odom7 + 7 * k, nd.odom, sizeof(nd.odom));
        if (clouds) bag::fill_cloud(nd.cloud, clouds[k]);
    }
    return ERASOR_OK;
}

int erasor_bag_load(erasor_pcd_t p, size_t first, size_t count, float* out_xyzi, size_t cap, int out_kind, uint64_t* offsets) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (!p->bag_ok) return fail(p, ERASOR_E_STATE, "no bag indexed: call erasor_bag_index first");
    std::string msg;
    const int rc = bag::check_range(p->bag, first, count, msg);
    if (rc != ERASOR_OK) return fail(p, rc, msg);
    std::vector<uint64_t> list(count);
    for (size_t k = 0; k < count; ++k) list[k] = first + k;
    return erasor_bag_load_list(p, list.data(), count, out_xyzi, cap, out_kind, offsets);
}

int erasor_bag_load_list(erasor_pcd_t p, const uint64_t* nodes, size_t count, float* out_xyzi, size_t cap, int out_kind, uint64_t* offsets) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    p->cached = false;
    if (!p->bag_ok) return fail(p, ERASOR_E_STATE, "no bag indexed: call erasor_bag_index first");
    if (!offsets || (count && !nodes)) return fail(p, ERASOR_E_INVALID, "null argument");
    if (out_kind != ERASOR_PTR_HOST && out_kind != ERASOR_PTR_DEVICE) return fail(p, ERASOR_E_INVALID, "out_kind must be ERASOR_PTR_HOST or ERASOR_PTR_DEVICE");
    uint64_t total = 0;
    std::string msg;
    int rc = bag::check_list(p->bag, nodes, count, &total, msg);
    if (rc != ERASOR_OK) return fail(p, rc, msg);
    offsets[0] = 0;
    for (size_t k = 0; k < count; ++k) offsets[k + 1] = offsets[k] + bag::cloud_points(p->bag.nodes[nodes[k]].cloud);
    if (!out_xyzi) return ERASOR_OK;
    if (cap < total) return fail(p, ERASOR_E_CAPACITY, "out_xyzi holds fewer points than the nodes' clouds");
    if (out_kind == ERASOR_PTR_DEVICE && (reinterpret_cast<uintptr_t>(out_xyzi) & 15u))
        return fail(p, ERASOR_E_INVALID, "device clouds must be 16-byte aligned (one float4 per point)");
    if (!total) return ERASOR_OK;
    PCK(cudaSetDevice(p->device));

    // the clouds' descriptors and the device copy of their data, each blob at a 16-byte aligned offset (a node in an LZ4 chunk is
    // read where its chunk was decoded)
    std::vector<BagDesc> desc;
    std::vector<Span> spans;
    uint64_t blob_bytes = 0, ntiles = 0;
    for (size_t k = 0; k < count; ++k) {
        const bag::Node& nd = p->bag.nodes[nodes[k]];
        const bag::Cloud& c = nd.cloud;
        const uint64_t n = bag::cloud_points(c);
        if (!n) continue;
        BagDesc D{};
        D.c = c;
        D.lz4 = nd.decoded();
        D.src = D.lz4 ? bag::dec_of(p->z4, nd) + c.data_off : blob_bytes;
        D.out = offsets[k];
        D.tile0 = ntiles;
        D.reach = bag::point_reach(c);
        const bool rows_contiguous = c.height == 1 || (uint64_t)c.row_step == (uint64_t)c.width * c.point_step;
        D.cols = rows_contiguous ? n : c.width;
        const uint64_t rows = rows_contiguous ? 1 : c.height;
        D.staged = D.reach <= kGatherTile;
        D.per_tile = D.staged ? (uint32_t)std::min<uint64_t>(4 * kGatherThreads, 1 + (kGatherTile - D.reach) / std::max<uint32_t>(c.point_step, 1))
                              : 4 * kGatherThreads;
        D.tiles_per_row = (D.cols + D.per_tile - 1) / D.per_tile;
        ntiles += rows * D.tiles_per_row;
        if (!D.lz4) {
            spans.push_back(Span{p->bag_file + c.data_off, c.data_len, blob_bytes});
            blob_bytes += (c.data_len + 15) & ~15ull;
        }
        desc.push_back(D);
    }
    PCK(p->bag_blobs.ensure(blob_bytes));
    PCK(p->bag_desc.ensure(sizeof(BagDesc) * desc.size()));
    uint8_t* d_blobs = p->bag_blobs.as<uint8_t>();
    rc = upload_spans(p, d_blobs, spans);
    if (rc != ERASOR_OK) return rc;
    PCK(cudaMemcpyAsync(p->bag_desc.p(), desc.data(), sizeof(BagDesc) * desc.size(), cudaMemcpyHostToDevice, p->st));
    uint4* d_out = reinterpret_cast<uint4*>(out_xyzi);
    if (out_kind == ERASOR_PTR_HOST) { PCK(p->out.ensure(sizeof(uint4) * total)); d_out = p->out.as<uint4>(); }
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(ntiles, (uint64_t)p->sm_count * 8));
    k_bag_gather<<<grid, kGatherThreads, 0, p->st>>>(d_blobs, p->z4_dec.as<uint8_t>(), p->bag_desc.as<BagDesc>(), (int)desc.size(), ntiles, d_out);
    PCK(cudaGetLastError());
    if (out_kind == ERASOR_PTR_HOST) PCK(cudaMemcpyAsync(out_xyzi, d_out, sizeof(uint4) * total, cudaMemcpyDeviceToHost, p->st));
    PCK(cudaStreamSynchronize(p->st));
    return ERASOR_OK;
}

int erasor_bag_lz4_stats(erasor_pcd_t p, erasor_bag_lz4_stats_t* stats) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (!stats) return fail(p, ERASOR_E_INVALID, "null argument");
    bag::fill_lz4_stats(p->bag, p->z4, *stats);
    stats->decode_ms = p->z4_decode_ms;
    stats->checksum_ms = p->z4_sums_ms;
    return ERASOR_OK;
}

int erasor_bag_bz2_stats(erasor_pcd_t p, erasor_bag_bz2_stats_t* stats) {
    if (!p) return ERASOR_E_INVALID;
    p->err.clear();
    if (!stats) return fail(p, ERASOR_E_INVALID, "null argument");
    if (!p->bag_ok) { *stats = erasor_bag_bz2_stats_t{}; return ERASOR_OK; }
    bag::fill_bz2_stats(p->bag, p->z4, p->z2_found, *stats);
    stats->scratch_bytes = p->z2_scratch;
    stats->scan_ms = p->z2_ms[0];
    stats->decode_ms = p->z2_ms[1];
    stats->bwt_ms = p->z2_ms[2];
    stats->rle_ms = p->z2_ms[3];
    return ERASOR_OK;
}

}  // extern "C"
