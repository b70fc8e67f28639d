// host_selftest.cpp -- compiles binning.h, pcd_codec.h and pcd_binary.h for the HOST so that the CPU test-suite (-m "not gpu")
// can check the exact-threshold bin arithmetic against the oracle, and the ASCII PCD codec's per-token arithmetic against
// numpy and Python, the binary PCD reader with its parallel LZF decoder run serially, and the erasor/node bag index with its
// per-point decode, without a GPU.
// This library is loaded by tests only; the product API (erasor_capi.cu) has no host compute path.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "bag_index.h"
#include "binning_tables.h"
#include "pcd_binary.h"
#include "pcd_codec.h"
#include "pose_math.h"

extern "C" {

// bins[i] = bin id or -1; stats = {negzero, ambiguous, slow}; qerr_max = max |q_float - q_double| over binned points
int erasor_hostcheck_bin_points(const erasor_params_t* p, const float* xyzi, size_t n, int32_t* bins,
                                uint64_t* stats3, double* qerr_max, double* eps_q) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    const erasor::BinTablesView v = T.host_view();
    erasor::BinFenceCounters fc{0, 0, 0};
    uint64_t s0 = 0, s1 = 0, s2 = 0;
    double qe = 0.0;
    for (size_t i = 0; i < n; ++i) {
        fc = erasor::BinFenceCounters{0, 0, 0};
        const float x = xyzi[4 * i], y = xyzi[4 * i + 1], z = xyzi[4 * i + 2];
        bins[i] = erasor::bin_of_point(v, v.ring_thr, x, y, z, &fc);
        s0 += fc.negzero; s1 += fc.ambiguous; s2 += fc.slow;
        if (bins[i] >= 0 && y != 0.0f) {
            // replicate the float guess and compare with the double-precision coordinate
            const float ax = std::fabs(x), ay = std::fabs(y);
            const float mx = std::fmax(ax, ay), mn = std::fmin(ax, ay);
            float a = erasor::atan_unit(mn / mx);
            if (ay > ax) a = 1.57079637f - a;
            if (x < 0.0f) a = 3.14159274f - a;
            if (y < 0.0f) a = 6.28318548f - a;
            const float  q  = a * v.inv_ss;
            const double th = (y >= 0) ? std::atan2((double)y, (double)x) : 2 * 3.1415926535 + std::atan2((double)y, (double)x);
            const double e  = std::fabs((double)q - th / T.sector_size);
            if (e > qe) qe = e;
        }
    }
    stats3[0] = s0; stats3[1] = s1; stats3[2] = s2;
    *qerr_max = qe;
    *eps_q = T.eps_q;
    return 0;
}

// expose the tables for inspection: ring thresholds (R+1 doubles), s_max, z window
int erasor_hostcheck_tables(const erasor_params_t* p, double* ring_thr, double* s_max, float* z_lo, float* z_hi, int* sec_of_pi) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    std::memcpy(ring_thr, T.ring_thr.data(), sizeof(double) * (T.R + 1));
    *s_max = T.s_max; *z_lo = T.z_lo; *z_hi = T.z_hi; *sec_of_pi = T.sec_of_pi;
    return 0;
}

// what erasor_process_nodes hands the device for one node (pose_math.h): criterion point, squared radius, origin -> body rows and the
// float guard band of the radius pre-test
int erasor_hostcheck_node_pose(const double* odom7, double voi_max_range, double* px_py_limit, float* T12, float* guards4) {
    erasor::NodePose np;
    erasor::node_pose_of(odom7, voi_max_range, np);
    px_py_limit[0] = np.px; px_py_limit[1] = np.py; px_py_limit[2] = np.limit;
    for (int i = 0; i < 12; ++i) T12[i] = np.T[i];
    guards4[0] = np.pxf; guards4[1] = np.pyf; guards4[2] = np.lim_lo; guards4[3] = np.lim_hi;
    return 0;
}

// byte offset of each bin's region in K4b's global scratch (device_types.h): bin bins[k] with scatter offsets dsq[k], dsm[k]
int erasor_hostcheck_k4b_scratch_offset(const uint32_t* dsq, const uint32_t* dsm, const uint32_t* bins, size_t n, uint64_t* out) {
    for (size_t k = 0; k < n; ++k) out[k] = erasor::k4b_scratch_offset(dsq[k], dsm[k], bins[k]);
    return 0;
}

// the float guard bands of the device's fast path (binning_tables.cpp): {up_k, dn_k} per ring threshold and around s_max
int erasor_hostcheck_guards(const erasor_params_t* p, float* ring_guard, float* smax_lo_hi) {
    erasor::HostBinTables T;
    std::string err;
    if (erasor::build_bin_tables(*p, T, err) != 0) return -1;
    std::memcpy(ring_guard, T.ring_guard.data(), sizeof(float) * T.ring_guard.size());
    smax_lo_hi[0] = T.smax_lo; smax_lo_hi[1] = T.smax_hi;
    return 0;
}

// pcd_codec.h's parse on n tokens, token k = text[offs[k] .. offs[k + 1]): bits[k] = the float's bit pattern (0 when invalid),
// kind[k] = 0 fast path, 1 big-integer path, 2 invalid.  want_value = 0 runs the check alone, as the kernel does for a column it
// does not keep (kind 0 or 2, bits 0).
int erasor_hostcheck_pcd_parse(const uint8_t* text, const uint64_t* offs, size_t n, int want_value, uint32_t* bits, int32_t* kind) {
    pcd::Big D, A, B;
    for (size_t k = 0; k < n; ++k) {
        const uint8_t* s = text + offs[k];
        const uint64_t len = offs[k + 1] - offs[k];
        const pcd::TokenScan r = pcd::scan_token(s, len, want_value != 0);
        kind[k] = r.kind;
        float f = 0.0f;
        if (r.kind == pcd::TOK_OK && want_value) f = (float)r.value;
        else if (r.kind == pcd::TOK_SLOW) {
            const double v = pcd::parse_slow_abs(s, len, D, A, B);
            f = (float)(r.neg ? -v : v);
        }
        bits[k] = pcd::float_to_bits(f);
    }
    return 0;
}

// pcd_codec.h's "%.8g" on n floats: value k's text at out[16 k ..], its length in lens[k]
int erasor_hostcheck_pcd_format(const float* vals, size_t n, char* out, int32_t* lens) {
    for (size_t k = 0; k < n; ++k) lens[k] = pcd::format_g8(vals[k], out + 16 * k);
    return 0;
}
}

namespace {
void set_err(char* err, size_t cap, const std::string& m) {
    if (err && cap) { std::strncpy(err, m.c_str(), cap - 1); err[cap - 1] = 0; }
}

// pcd_kernels.cu's lzf_decode with every kernel run serially, over chunks of `chunk` bytes
int lzf_decode_stages(const uint8_t* s, uint64_t csize, uint64_t usize, uint8_t* out, uint64_t keep, uint64_t chunk, uint64_t* ntok, std::string& msg) {
    const uint64_t nchunks = (csize + chunk - 1) / chunk;
    const int E = pcd::kLzfEntries;
    *ntok = 0;
    if (!nchunks) {
        if (usize) { msg = "malformed LZF stream: it ends after 0 of " + std::to_string(usize) + " bytes"; return ERASOR_E_INVALID; }
        return ERASOR_OK;
    }
    // A
    std::vector<uint8_t> m_in(nchunks * E), m_out(nchunks * E);
    std::vector<uint32_t> tok(nchunks * E), byt(nchunks * E);
    for (uint64_t k = 0; k < nchunks; ++k)
        for (int e = 0; e < E; ++e) {
            const pcd::LzfWalk w = pcd::lzf_walk(s, csize, k * chunk, std::min(k * chunk + chunk, csize), (uint32_t)e);
            m_in[k * E + e] = (uint8_t)w.exit;
            tok[k * E + e] = w.tokens;
            byt[k * E + e] = w.bytes;
        }
    for (uint64_t d = 1; d < nchunks; d *= 2) {
        for (uint64_t k = 0; k < nchunks; ++k)
            for (int e = 0; e < E; ++e)
                m_out[k * E + e] = k >= d ? pcd::lzf_compose(&m_in[k * E], &m_in[(k - d) * E], e) : m_in[k * E + e];
        m_in.swap(m_out);
    }
    std::vector<uint32_t> entry(nchunks);
    std::vector<uint64_t> tok_off(nchunks), byte_off(nchunks);
    uint64_t tokens = 0, bytes = 0;
    for (uint64_t k = 0; k < nchunks; ++k) {
        entry[k] = k ? m_in[(k - 1) * E] : 0u;
        tok_off[k] = tokens;
        byte_off[k] = bytes;
        tokens += tok[k * E + entry[k]];
        bytes += byt[k * E + entry[k]];
    }
    *ntok = tokens;
    // B
    std::vector<pcd::LzfToken> rec(tokens);
    uint64_t err = ~0ull;
    for (uint64_t k = 0; k < nchunks; ++k) {
        uint64_t e;
        pcd::lzf_records(s, csize, usize, k * chunk, std::min(k * chunk + chunk, csize), entry[k], byte_off[k], rec.data() + tok_off[k], &e);
        err = std::min(err, e);
    }
    if (err != ~0ull) { msg = pcd::lzf_error_message(err); return ERASOR_E_INVALID; }
    if (bytes != usize) { msg = "malformed LZF stream: it ends after " + std::to_string(bytes) + " of " + std::to_string(usize) + " bytes"; return ERASOR_E_INVALID; }
    // C
    std::vector<uint32_t> src(keep);
    for (uint64_t i = 0; i < tokens; ++i)
        if (rec[i].dst < keep) pcd::lzf_expand(rec[i], s, out, src.data(), keep);
    for (bool moved = true; moved;) {
        moved = false;
        for (uint64_t j = 0; j < keep; ++j) moved |= pcd::lzf_jump(src.data(), j);
    }
    for (uint64_t j = 0; j < keep; ++j) pcd::lzf_fill(src.data(), out, j);
    return ERASOR_OK;
}
}  // namespace

extern "C" {

// erasor_pcd_load's binary and binary_compressed branches on the host (the same header reader, layout rules and stages, run
// serially, the LZF stream cut into chunks of `chunk` bytes).  Returns 1 for an ascii file (erasor_pcd_parse_ascii's, not checked
// here), else what erasor_pcd_load returns; err gets the message.
int erasor_hostcheck_pcd_load(const char* file, size_t len, float* out, size_t cap, size_t* n, erasor_pcd_load_info_t* info, uint64_t chunk,
                              char* err, size_t errcap) {
    erasor_pcd_load_info_t inf{};
    *info = inf;
    *n = 0;
    set_err(err, errcap, "");
    pcd::Header h;
    if (!pcd::parse_header(file, len, h)) { set_err(err, errcap, "no DATA line in the PCD header"); return ERASOR_E_INVALID; }
    pcd::Layout L;
    std::string msg;
    int rc = pcd::resolve_layout(h, L, msg);
    pcd::fill_load_info(h, L, inf);
    *info = inf;
    if (rc != ERASOR_OK) { set_err(err, errcap, msg); return rc; }
    if (L.mode == pcd::DATA_ASCII) return 1;
    if (L.mode == pcd::DATA_BINARY && (rc = pcd::check_binary_body(L, h.data_off, len, msg)) != ERASOR_OK) { set_err(err, errcap, msg); return rc; }
    if (!L.points) return ERASOR_OK;
    uint64_t csize = 0, usize = 0;
    if (L.mode == pcd::DATA_COMPRESSED) {
        if (len - h.data_off < 8) { set_err(err, errcap, "the file ends before compressed_size and uncompressed_size"); return ERASOR_E_INVALID; }
        csize = pcd::le32(reinterpret_cast<const uint8_t*>(file) + h.data_off);
        usize = pcd::le32(reinterpret_cast<const uint8_t*>(file) + h.data_off + 4);
        info->compressed_size = csize;
        info->uncompressed_size = usize;
        if ((rc = pcd::check_compressed_sizes(L, h.data_off, len, csize, usize, msg)) != ERASOR_OK) { set_err(err, errcap, msg); return rc; }
    }
    if (!out) { *n = L.points; return ERASOR_OK; }
    if (cap < L.points) { set_err(err, errcap, "out holds fewer points than the header's POINTS"); return ERASOR_E_CAPACITY; }
    const uint8_t* base = reinterpret_cast<const uint8_t*>(file) + h.data_off;
    std::vector<uint8_t> dec;
    if (L.mode == pcd::DATA_COMPRESSED) {
        dec.resize(L.keep_end);
        uint64_t ntok = 0;
        rc = lzf_decode_stages(base + 8, csize, usize, dec.data(), L.keep_end, chunk, &ntok, msg);
        info->lzf_tokens = ntok;
        if (rc != ERASOR_OK) { set_err(err, errcap, msg); return rc; }
        base = dec.data();
    }
    for (uint64_t i = 0; i < L.points; ++i) pcd::gather_point(base, L.g, i, reinterpret_cast<uint32_t*>(out) + 4 * i);
    *n = L.points;
    return ERASOR_OK;
}

// the stages A-C alone on an LZF stream: out gets the first keep of usize bytes; ntok the tokens of the true chain
int erasor_hostcheck_lzf_decode(const uint8_t* s, uint64_t csize, uint8_t* out, uint64_t usize, uint64_t keep, uint64_t chunk, uint64_t* ntok,
                                char* err, size_t errcap) {
    std::string msg;
    const int rc = lzf_decode_stages(s, csize, usize, out, keep, chunk, ntok, msg);
    set_err(err, errcap, msg);
    return rc;
}

// ---- erasor/node bags: bag_index.h's index, and its per-point decode run serially (what erasor_bag_load's gather computes) ----
static bag::Index g_bag;

// erasor_bag_index on the host; the index is kept for the two calls below
int erasor_hostcheck_bag_index(const char* file, size_t len, const char* topic, int keep_first, size_t* n_nodes, erasor_bag_info_t* info,
                               char* err, size_t errcap) {
    std::string msg;
    *n_nodes = 0;
    *info = erasor_bag_info_t{};
    const int rc = bag::build_index(reinterpret_cast<const uint8_t*>(file), len, topic ? topic : "/node/combined/optimized", keep_first != 0, g_bag, msg);
    set_err(err, errcap, msg);
    if (rc != ERASOR_OK) return rc;
    *n_nodes = g_bag.nodes.size();
    bag::fill_info(g_bag, *info);
    return ERASOR_OK;
}

int erasor_hostcheck_bag_nodes(size_t first, size_t count, uint32_t* seq, uint64_t* stamp_ns, double* odom7, erasor_bag_cloud_t* clouds) {
    if (first > g_bag.nodes.size() || count > g_bag.nodes.size() - first) return ERASOR_E_INVALID;
    for (size_t k = 0; k < count; ++k) {
        const bag::Node& nd = g_bag.nodes[first + k];
        seq[k] = nd.seq;
        stamp_ns[k] = nd.stamp_ns;
        std::memcpy(odom7 + 7 * k, nd.odom, sizeof(nd.odom));
        bag::fill_cloud(nd.cloud, clouds[k]);
    }
    return ERASOR_OK;
}

// the clouds of nodes [first, first + count) of the indexed file, back to back; offsets: count + 1
int erasor_hostcheck_bag_decode(const char* file, size_t first, size_t count, float* out, uint64_t* offsets, char* err, size_t errcap) {
    uint64_t total = 0;
    std::string msg;
    std::vector<uint64_t> list(count);
    for (size_t k = 0; k < count; ++k) list[k] = first + k;
    int rc = bag::check_range(g_bag, first, count, msg);
    if (rc == ERASOR_OK) rc = bag::check_list(g_bag, list.data(), count, &total, msg);
    set_err(err, errcap, msg);
    if (rc != ERASOR_OK) return rc;
    offsets[0] = 0;
    for (size_t k = 0; k < count; ++k) {
        const bag::Cloud& c = g_bag.nodes[first + k].cloud;
        const uint8_t* d = reinterpret_cast<const uint8_t*>(file) + c.data_off;
        const uint64_t n = bag::cloud_points(c);
        uint32_t* o = reinterpret_cast<uint32_t*>(out) + 4 * offsets[k];
        for (uint64_t i = 0; i < n; ++i) bag::point_values(d + bag::point_offset(c, i), c, o + 4 * i);
        offsets[k + 1] = offsets[k] + n;
    }
    return ERASOR_OK;
}

// A serial liblzf-style decoder (one token after the other, bytes copied one at a time): 0, or -1 for a malformed stream
int erasor_hostcheck_lzf_serial(const uint8_t* s, uint64_t csize, uint8_t* out, uint64_t usize) {
    uint64_t i = 0, o = 0;
    while (i < csize) {
        const uint32_t c = s[i++];
        if (c < 32) {
            const uint64_t len = c + 1;
            if (i + len > csize || o + len > usize) return -1;
            std::memcpy(out + o, s + i, len);
            i += len;
            o += len;
        } else {
            uint64_t len = c >> 5;
            if (len == 7) { if (i >= csize) return -1; len += s[i++]; }
            len += 2;
            if (i >= csize) return -1;
            const uint64_t d = ((uint64_t)(c & 31) << 8) + s[i++] + 1;
            if (d > o || o + len > usize) return -1;
            for (uint64_t k = 0; k < len; ++k, ++o) out[o] = out[o - d];
        }
    }
    return o == usize ? 0 : -1;
}

// The greedy LZF encoder of tests/pcd_binary_model.py (lzf_compress), for inputs too large for Python: a table keyed by the exact
// three bytes at each position holds the last position they were seen at; a match within 8192 bytes is extended to at most 264
// bytes; literal runs are cut at 32.  Only the position where a match starts enters the table.  -1 when out is too small.
int erasor_hostcheck_lzf_compress(const uint8_t* in, uint64_t n, uint8_t* out, uint64_t cap, uint64_t* clen) {
    std::vector<uint32_t> last(1u << 24, 0);         // position + 1, 0 = never seen
    uint64_t o = 0, lit = 0, i = 0;
    auto flush = [&](uint64_t end) -> bool {
        while (lit < end) {
            const uint64_t m = std::min<uint64_t>(32, end - lit);
            if (o + 1 + m > cap) return false;
            out[o++] = (uint8_t)(m - 1);
            std::memcpy(out + o, in + lit, m);
            o += m;
            lit += m;
        }
        return true;
    };
    while (i + 2 < n) {
        const uint32_t key = ((uint32_t)in[i] << 16) | ((uint32_t)in[i + 1] << 8) | in[i + 2];
        const uint64_t cand = last[key];
        last[key] = (uint32_t)(i + 1);
        if (cand && i - (cand - 1) <= 8192) {
            const uint64_t p = cand - 1;
            uint64_t len = 3;
            while (len < 264 && i + len < n && in[p + len] == in[i + len]) ++len;
            if (!flush(i)) return -1;
            const uint64_t off = i - p - 1, l = len - 2;
            if (o + 3 > cap) return -1;
            if (l < 7) out[o++] = (uint8_t)((l << 5) | (off >> 8));
            else { out[o++] = (uint8_t)((7u << 5) | (off >> 8)); out[o++] = (uint8_t)(l - 7); }
            out[o++] = (uint8_t)(off & 255);
            i += len;
            lit = i;
        } else {
            ++i;
        }
    }
    if (!flush(n)) return -1;
    *clen = o;
    return 0;
}
}
