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
#include "lzf_encode.h"
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
static bag::ChunkPlan g_plan;
static bag::Bz2Found g_found;
static std::vector<uint8_t> g_dec;                   // the decoded lz4 and bz2 chunks, laid out as the device's decoded buffer

// The stages of erasor_bag_index's LZ4 decode (pcd_kernels.cu), serially, into dec (sized here): the key of the first broken rule
// or ~0
static uint64_t lz4_stages(const uint8_t* file, const bag::Index& x, const bag::ChunkPlan& p, std::vector<uint8_t>& dec) {
    std::vector<uint8_t> src(std::max<uint64_t>(p.src_bytes, 1));
    for (size_t c = 0; c < p.chunks.size(); ++c) {
        const bag::Lz4Chunk& k = x.lz4[p.chunks[c]];
        std::memcpy(src.data() + p.cd[c].src, file + k.data, k.len);
    }
    dec.assign(std::max<uint64_t>(p.dec_bytes, 1), 0);
    uint64_t err = ~0ull;
    const size_t nb = p.blocks.size();
    std::vector<uint32_t> bsize(nb, 0);
    std::vector<uint64_t> boff(nb, ~0ull);
    for (size_t b = 0; b < nb; ++b) {                 // k_lz4_size
        const bag::Lz4Block& B = p.blocks[b];
        uint32_t o = B.csize, at = 0, r = lz4::R_OK;
        if (!B.stored) r = lz4::block(lz4::Serial{}, src.data() + B.src, B.csize, nullptr, B.cap, &o, &at);
        if (r != lz4::R_OK) err = std::min(err, bag::block_key(B, b, at, r));
        bsize[b] = r == lz4::R_OK ? o : 0;
    }
    for (size_t c = 0; c < p.cd.size(); ++c) {       // k_lz4_place
        const bag::Lz4ChunkDesc& d = p.cd[c];
        uint64_t s = 0;
        for (uint32_t b = d.block0; b < d.block0 + d.nblocks; ++b) s += bsize[b];
        if (s != d.size) { err = std::min(err, bag::chunk_key(d, c, lz4::R_SIZE)); continue; }
        s = 0;
        for (uint32_t b = d.block0; b < d.block0 + d.nblocks; ++b) { boff[b] = d.dec + s; s += bsize[b]; }
    }
    for (size_t b = 0; b < nb; ++b) {                 // k_lz4_decode
        const bag::Lz4Block& B = p.blocks[b];
        if (boff[b] == ~0ull) continue;
        uint32_t o = 0, at = 0;
        if (B.stored) std::memcpy(dec.data() + boff[b], src.data() + B.src, B.csize);
        else lz4::block(lz4::Serial{}, src.data() + B.src, B.csize, dec.data() + boff[b], bsize[b], &o, &at);
    }
    for (size_t b = 0; b < nb; ++b) {                 // k_lz4_sums
        const bag::Lz4Block& B = p.blocks[b];
        if (B.has_sum && lz4::xxh32(src.data() + B.src, B.csize, 0) != B.sum) err = std::min(err, bag::block_key(B, b, B.csize, lz4::R_BLOCK_SUM));
    }
    for (size_t c = 0; c < p.cd.size(); ++c) {       // k_lz4_content
        const bag::Lz4ChunkDesc& d = p.cd[c];
        if (d.has_sum && lz4::xxh32(dec.data() + d.dec, d.size, 0) != d.sum) err = std::min(err, bag::chunk_key(d, c, lz4::R_CONTENT_SUM));
    }
    return err;
}

// The stages of erasor_bag_index's bz2 decode (pcd_kernels.cu), serially, into dec: the bz2 key of the first broken rule or ~0, *blk
// the block it names; found gets the blocks and candidates
static uint64_t bz2_stages(const uint8_t* file, const bag::Index& x, const bag::ChunkPlan& p, std::vector<uint8_t>& dec, int64_t* blk, bag::Bz2Found& found) {
    const size_t nc = p.bd.size();
    std::vector<uint8_t> src(std::max<uint64_t>(p.bz_src_bytes, 1));
    for (size_t c = 0; c < nc; ++c) std::memcpy(src.data() + p.bd[c].src, file + x.bz2[p.bz_chunks[c]].data, p.bd[c].len);
    std::vector<bag::Bz2Cand> cand;                   // k_bz2_scan, the scan, k_bz2_emit
    std::vector<uint64_t> c0(nc + 1);
    for (size_t c = 0; c < nc; ++c) {
        const bag::Bz2ChunkDesc& D = p.bd[c];
        c0[c] = cand.size();
        for (uint64_t q = 0; q < D.len; ++q)
            if (const uint32_t j = bz2::candidate_at(src.data() + D.src, D.len, q)) cand.push_back(bag::Bz2Cand{8 * q + j - 1, (uint32_t)c, 0});
    }
    c0[nc] = cand.size();
    const size_t n = cand.size();
    found.candidates = n;
    found.blocks.assign(nc, 0);
    static bz2::Tables T;
    std::vector<bz2::Walk> walk(n);                   // k_bz2_walk
    for (size_t i = 0; i < n; ++i) {
        const bag::Bz2ChunkDesc& D = p.bd[cand[i].chunk];
        walk[i] = bz2::block(src.data() + D.src, 8 * D.len, cand[i].bit, D.level, T, nullptr, nullptr);
    }
    std::vector<int32_t> blkno(n, -1);
    std::vector<uint64_t> tt_off(n, ~0ull), osize(n, ~0ull), out_off(n, ~0ull);
    uint64_t err = ~0ull;
    for (size_t c = 0; c < nc; ++c)                   // k_bz2_chain
        err = std::min(err, bag::bz2_chain(c, p.bd[c], src.data() + p.bd[c].src, cand.data(), c0[c], c0[c + 1], walk.data(), blkno.data(), tt_off.data(),
                                           &found.blocks[c]));
    std::vector<uint8_t> tt(std::max<uint64_t>(p.bz_tt_bytes, 1)), bw(tt.size());
    std::vector<uint32_t> lf(tt.size());
    uint32_t tab[256];
    bz2::crc_table(tab);
    for (size_t i = 0; i < n; ++i) {
        if (tt_off[i] == ~0ull) continue;
        const bag::Bz2ChunkDesc& D = p.bd[cand[i].chunk];
        uint32_t hist[256];                           // k_bz2_decode
        const bz2::Walk w = bz2::block(src.data() + D.src, 8 * D.len, cand[i].bit, D.level, T, tt.data() + tt_off[i], hist);
        bz2::lf_vector(tt.data() + tt_off[i], w.n, hist, lf.data() + tt_off[i]);
        bz2::unbwt_serial(tt.data() + tt_off[i], lf.data() + tt_off[i], w.n, w.orig, bw.data() + tt_off[i]);               // k_bz2_bwt
        uint64_t os = 0;
        uint32_t crc = 0;
        uint32_t r = bz2::rle1(bw.data() + tt_off[i], w.n, tab, nullptr, &os, &crc);                                     // k_bz2_rle
        if (r == bz2::R_OK && crc != w.crc) r = bz2::R_BLOCK_CRC;
        if (r != bz2::R_OK) err = std::min(err, bag::bz2_key(cand[i].chunk, cand[i].bit, r));
        osize[i] = r == bz2::R_OK ? os : ~0ull;
    }
    for (size_t c = 0; c < nc; ++c)                   // k_bz2_place
        err = std::min(err, bag::bz2_place(c, p.bd[c], c0[c], c0[c + 1], tt_off.data(), osize.data(), out_off.data()));
    for (size_t i = 0; i < n; ++i) {                  // k_bz2_expand
        if (out_off[i] == ~0ull) continue;
        uint64_t os = 0;
        uint32_t crc = 0;
        bz2::rle1(bw.data() + tt_off[i], walk[i].n, tab, dec.data() + out_off[i], &os, &crc);
    }
    *blk = -1;                                        // k_bz2_errblock
    if (err != ~0ull)
        for (size_t i = 0; i < n; ++i)
            if (blkno[i] >= 0 && cand[i].chunk == err >> 44 && cand[i].bit <= ((err >> 8) & 0xFFFFFFFFFull)) *blk = std::max<int64_t>(*blk, blkno[i]);
    return err;
}

// k_bag_parse, serially
static void parse_stage(const bag::ChunkPlan& p, const std::vector<uint8_t>& dec, std::vector<bag::NodeOut>& res) {
    res.assign(p.nodes.size(), bag::NodeOut{});
    for (size_t i = 0; i < p.nodes.size(); ++i) {     // k_bag_parse
        const bag::Lz4NodeIn& n = p.nodes[i];
        bag::NodeOut& r = res[i];
        uint64_t d0 = 0, d1 = 0;
        r.code = bag::record_core(dec.data() + n.dec, n.len, n.rec, n.conn, n.time_ns, &d0, &d1, &r.a);
        if (r.code == bag::NF_OK) r.code = bag::parse_node_core(dec.data() + n.dec, d0, d1, &r.seq, r.odom, r.cloud, &r.a, &r.b);
    }
}

// erasor_bag_index on the host; the index is kept for the two calls below
int erasor_hostcheck_bag_index(const char* file, size_t len, const char* topic, int keep_first, size_t* n_nodes, erasor_bag_info_t* info,
                               char* err, size_t errcap) {
    std::string msg;
    *n_nodes = 0;
    *info = erasor_bag_info_t{};
    g_plan = bag::ChunkPlan();
    g_found = bag::Bz2Found();
    g_dec.clear();
    const uint8_t* f = reinterpret_cast<const uint8_t*>(file);
    int rc = bag::build_index(f, len, topic ? topic : "/node/combined/optimized", keep_first != 0, g_bag, msg);
    if (rc == ERASOR_OK && !g_bag.pending.empty()) {
        bag::plan_chunks(g_bag, g_plan);
        std::vector<bag::NodeOut> res;
        const uint64_t key = lz4_stages(f, g_bag, g_plan, g_dec);
        int64_t blk = -1;
        const uint64_t bz_key = bz2_stages(f, g_bag, g_plan, g_dec, &blk, g_found);
        parse_stage(g_plan, g_dec, res);
        rc = bag::decode_error(g_bag, g_plan, key, bz_key, blk, msg);
        if (rc == ERASOR_OK) rc = bag::finish_chunks(g_bag, res.data(), msg);
    }
    set_err(err, errcap, msg);
    if (rc != ERASOR_OK) { g_bag = bag::Index(); g_plan = bag::ChunkPlan(); g_found = bag::Bz2Found(); return rc; }
    *n_nodes = g_bag.nodes.size();
    bag::fill_info(g_bag, *info);
    return ERASOR_OK;
}

// erasor_bag_lz4_stats of the last erasor_hostcheck_bag_index
int erasor_hostcheck_bag_lz4_stats(erasor_bag_lz4_stats_t* s) {
    bag::fill_lz4_stats(g_bag, g_plan, *s);
    return ERASOR_OK;
}

// One bzip2 stream s[0, len) of decoded length `size` through the bz2 stages, as a bz2 chunk at byte 0 of a file: out (size bytes)
// gets the decoded data; the return is what erasor_bag_index returns for such a chunk, err its message
int erasor_hostcheck_bz2_stream(const uint8_t* s, uint64_t len, uint32_t size, uint8_t* out, char* err, size_t errcap) {
    bag::Index x;
    uint32_t level = 0;
    std::string msg;
    int rc = bag::detail::bz2_header(s, len, &level, msg);
    if (rc != ERASOR_OK) { set_err(err, errcap, "bz2 chunk at byte 0: " + msg); return rc; }
    x.bz2.push_back(bag::Bz2Chunk{0, 0, len, size, level});
    x.nodes.resize(1);
    x.nodes[0].bz = 0;
    x.pending.push_back(0);
    bag::ChunkPlan p;
    bag::plan_chunks(x, p);
    std::vector<uint8_t> dec(std::max<uint64_t>(p.dec_bytes, 1));
    bag::Bz2Found found;
    int64_t blk = -1;
    const uint64_t key = bz2_stages(s, x, p, dec, &blk, found);
    rc = bag::decode_error(x, p, ~0ull, key, blk, msg);
    set_err(err, errcap, msg);
    if (rc == ERASOR_OK) std::memcpy(out, dec.data(), size);
    return rc;
}

// erasor_bag_bz2_stats of the last erasor_hostcheck_bag_index, without the times and the scratch
int erasor_hostcheck_bag_bz2_stats(erasor_bag_bz2_stats_t* s) {
    bag::fill_bz2_stats(g_bag, g_plan, g_found, *s);
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
        const bag::Node& nd = g_bag.nodes[first + k];
        const bag::Cloud& c = nd.cloud;
        const uint8_t* d = (nd.decoded() ? g_dec.data() + bag::dec_of(g_plan, nd) : reinterpret_cast<const uint8_t*>(file)) + c.data_off;
        const uint64_t n = bag::cloud_points(c);
        uint32_t* o = reinterpret_cast<uint32_t*>(out) + 4 * offsets[k];
        for (uint64_t i = 0; i < n; ++i) bag::point_values(d + bag::point_offset(c, i), c, o + 4 * i);
        offsets[k + 1] = offsets[k] + n;
    }
    return ERASOR_OK;
}

// A greedy LZ4 block encoder for inputs too large for tests/lz4_model.py: a table keyed by a hash of the four bytes at each
// position holds the last position they were seen at; a match within 65535 bytes is extended while it lasts.  As liblz4 requires of
// its input, the last match starts 12 bytes or more before the end and the last 5 bytes are literals.
static uint64_t lz4_block_greedy(const uint8_t* in, uint32_t n, uint8_t* out) {
    std::vector<int64_t> table(1u << 16, -1);
    uint64_t o = 0;
    auto len_ext = [&](uint32_t v) { for (; v >= 255; v -= 255) out[o++] = 255; out[o++] = (uint8_t)v; };
    auto emit = [&](uint32_t a, uint32_t lit, uint32_t off, uint32_t mlen) {
        out[o++] = (uint8_t)((std::min<uint32_t>(lit, 15) << 4) | (off ? std::min<uint32_t>(mlen - 4, 15) : 0));
        if (lit >= 15) len_ext(lit - 15);
        std::memcpy(out + o, in + a, lit);
        o += lit;
        if (!off) return;
        out[o++] = (uint8_t)off;
        out[o++] = (uint8_t)(off >> 8);
        if (mlen - 4 >= 15) len_ext(mlen - 4 - 15);
    };
    uint32_t i = 0, anchor = 0;
    const uint32_t limit = n >= 13 ? n - 12 : 0, mend = n >= 5 ? n - 5 : 0;
    while (i < limit) {
        uint32_t v;
        std::memcpy(&v, in + i, 4);
        const uint32_t h = (v * 2654435761u) >> 16;
        const int64_t cand = table[h];
        table[h] = i;
        uint32_t w = 0;
        if (cand >= 0) std::memcpy(&w, in + cand, 4);
        if (cand >= 0 && i - cand <= 65535 && w == v) {
            uint32_t len = 4;
            while (i + len < mend && in[cand + len] == in[i + len]) ++len;
            emit(anchor, i - anchor, (uint32_t)(i - cand), len);
            i += len;
            anchor = i;
        } else {
            ++i;
        }
    }
    emit(anchor, n - anchor, 0, 0);
    return o;
}

// The LZ4 frame of in[0, n) with block max id bsid (4..7), block checksums and a content checksum when asked; a block that does
// not shrink is stored.  *clen = the frame's length; -1 when out (cap bytes) is too small.
int erasor_hostcheck_lz4_frame(const uint8_t* in, uint64_t n, int bsid, int block_sums, int content_sum, uint8_t* out, uint64_t cap, uint64_t* clen) {
    const uint64_t bmax = 1ull << (8 + 2 * bsid);
    if (cap < 15 + n + (n / bmax + 1) * (8 + bmax / 255 + 16)) return -1;
    uint64_t o = 0;
    auto put32 = [&](uint32_t v) { for (int k = 0; k < 4; ++k) out[o++] = (uint8_t)(v >> (8 * k)); };
    put32(lz4::kMagic);
    out[o++] = (uint8_t)(0x60 | (block_sums ? 0x10 : 0) | (content_sum ? 0x04 : 0));
    out[o++] = (uint8_t)(bsid << 4);
    out[o] = (uint8_t)((lz4::xxh32(out + 4, 2, 0) >> 8) & 0xFF);
    ++o;
    for (uint64_t a = 0; a < n; a += bmax) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(bmax, n - a);
        const uint64_t c = lz4_block_greedy(in + a, m, out + o + 4);
        const bool stored = c >= m;
        if (stored) std::memcpy(out + o + 4, in + a, m);
        const uint32_t bs = stored ? m : (uint32_t)c;
        put32(bs | (stored ? 0x80000000u : 0u));
        o += bs;
        if (block_sums) put32(lz4::xxh32(out + o - bs, bs, 0));
    }
    put32(0);
    if (content_sum) put32(lz4::xxh32(in, n, 0));
    *clen = o;
    return 0;
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

// lzf_encode.h's segmented encoder run serially over n bytes: the stream at out (cap bytes; -1 when it does not fit), its length
// in *clen, its tokens in *tokens and its segments in *segments
int erasor_hostcheck_lzf_encode(const uint8_t* in, uint64_t n, uint8_t* out, uint64_t cap, uint64_t* clen, uint64_t* tokens, uint64_t* segments) {
    std::vector<uint16_t> table(pcd::kLzfHashSize);
    std::vector<uint8_t> slot(pcd::lzf_segment_cap(pcd::kLzfSeg));
    uint64_t o = 0, ntok = 0, nseg = 0;
    for (uint64_t b = 0; b < n; b += pcd::kLzfSeg, ++nseg) {
        const uint32_t len = (uint32_t)std::min<uint64_t>(pcd::kLzfSeg, n - b);
        uint32_t t = 0;
        const uint32_t m = pcd::lzf_encode_segment(in + b, len, table.data(), slot.data(), &t);
        if (o + m > cap) return -1;
        std::memcpy(out + o, slot.data(), m);
        o += m;
        ntok += t;
    }
    *clen = o;
    *tokens = ntok;
    *segments = nseg;
    return 0;
}

// erasor_pcd_format's size rule for binary_compressed: POINTS x 16 uncompressed bytes and a stream of csize bytes
int erasor_hostcheck_pcd_sizes_fit(uint64_t usize, uint64_t csize) { return pcd::compressed_sizes_fit(usize, csize); }

// erasor_pcd_format's binary and binary_compressed files on the host (the same header, SoA and encoder, run serially); ascii is
// ERASOR_E_INVALID here (erasor_pcd_format_ascii's text is checked elsewhere).  out == NULL or cap too small gives the size
// (ERASOR_E_CAPACITY for the latter).
int erasor_hostcheck_pcd_format_file(const float* xyzi, size_t n, int data_mode, char* out, size_t cap, size_t* len, erasor_pcd_format_info_t* info) {
    erasor_pcd_format_info_t inf{};
    if (data_mode != ERASOR_PCD_BINARY && data_mode != ERASOR_PCD_BINARY_COMPRESSED) return ERASOR_E_INVALID;
    const bool compressed = data_mode == ERASOR_PCD_BINARY_COMPRESSED;
    if (compressed && (n > 0xFFFFFFFFull / 16 || pcd::compressed_sizes_fit(16ull * n, 0) != ERASOR_OK)) return ERASOR_E_UNSUPPORTED;
    char head[512];
    const int hl = pcd::format_header(head, sizeof(head), n, data_mode);
    inf.data_mode = (uint32_t)data_mode;
    inf.header_bytes = (uint64_t)hl;
    const uint64_t body = 16ull * n;
    std::vector<uint8_t> file(head, head + hl);
    if (!compressed) {
        file.resize(hl + body);
        if (n) std::memcpy(file.data() + hl, xyzi, body);
    } else {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(xyzi);
        std::vector<uint32_t> soa(4 * n);
        for (size_t i = 0; i < n; ++i)
            for (int s = 0; s < 4; ++s) soa[s * n + i] = w[4 * i + s];
        const uint64_t nseg = (body + pcd::kLzfSeg - 1) / pcd::kLzfSeg;
        std::vector<uint8_t> stream(nseg * pcd::lzf_segment_cap(pcd::kLzfSeg));
        uint64_t csize = 0, ntok = 0, segs = 0;
        erasor_hostcheck_lzf_encode(reinterpret_cast<const uint8_t*>(soa.data()), body, stream.data(), stream.size(), &csize, &ntok, &segs);
        if (pcd::compressed_sizes_fit(body, csize) != ERASOR_OK) return ERASOR_E_UNSUPPORTED;
        const uint32_t sizes[2] = {(uint32_t)csize, (uint32_t)body};
        file.resize(hl + 8 + csize);
        std::memcpy(file.data() + hl, sizes, 8);
        if (csize) std::memcpy(file.data() + hl + 8, stream.data(), csize);
        inf.segments = (uint32_t)segs;
        inf.uncompressed_size = body;
        inf.compressed_size = csize;
        inf.lzf_tokens = ntok;
    }
    *len = file.size();
    if (info) *info = inf;
    if (!out) return ERASOR_OK;
    if (cap < file.size()) return ERASOR_E_CAPACITY;
    std::memcpy(out, file.data(), file.size());
    return ERASOR_OK;
}
}
