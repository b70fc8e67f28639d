// bag_index.h -- the index of a ROS bag 2.0 file of erasor/node messages, read on the host, and the per-point decode of their
// PointCloud2 clouds (DESIGN.md section 12.2).  pcd_kernels.cu runs the decode in its gather kernel; host_selftest.cpp builds the
// same index and runs the same decode serially, so the CPU test-suite checks both before any GPU run.
//
// Format restated from the public ROS bag 2.0 description (no ROS is built here: parity with rosbag is unpinned).  After the
// line "#ROSBAG V2.0\n" the file is a sequence of records: uint32 header_len, the header's fields, uint32 data_len, the data.
// A field is uint32 len, then name=value (name up to the first '='; the value binary, little-endian).  Ops: 0x03 bag header,
// 0x05 chunk (its data holds further records), 0x07 connection, 0x02 message data, 0x04 index data, 0x06 chunk info.  The
// records are walked in file order, chunks included; the index section is checked for structure only.
//
// An lz4 chunk (DESIGN.md section 12.2.1) is not walked: its frame descriptor and block table are read (lz4_frame.h), and its
// messages are the entries (time, offset in the decoded chunk) of the index data records that follow it.  A bz2 chunk (section
// 12.2.2, bz2_stream.h) is indexed the same way; the host reads only its 4-byte stream header.  The nodes in compressed chunks are
// parsed after the chunks that hold a kept node are decoded, by the same parse_node_core, on the device (or serially by the host
// build): plan_chunks lays the decode out, finish_chunks takes the parsed nodes back.
//
// An erasor/node message serialises, in order: header (seq, stamp, frame_id); odom, a Pose of 7 doubles (position x y z, then
// orientation x y z w); odomCov, 36 doubles; lidar, a PointCloud2 (header; height, width; the field list, each a name string,
// offset, datatype byte and count; is_bigendian; point_step, row_step; data as a length-prefixed byte array; is_dense);
// lidarOdom, a Pose; image, a CompressedImage (header, format string, byte array); gps, a NavSatFix (header; status as int8 +
// uint16; latitude, longitude, altitude; 9 covariance doubles; covariance type byte).  Strings and arrays carry a uint32 length.
//
// PointXYZI decode restated from PCL 1.8's fromPCLPointCloud2 (unpinned): point (r, c) starts at r row_step + c point_step in data;
// a field serves x, y, z or intensity when its name matches, datatype is 7 (FLOAT32) and count is 0 or 1, the first such field in
// order; values are copied bit for bit; is_bigendian is ignored.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/erasor_b200.h"
#include "bz2_stream.h"
#include "lz4_frame.h"
#include "pcd_binary.h"

namespace bag {

constexpr uint8_t OP_MSG = 0x02, OP_BAG_HEADER = 0x03, OP_INDEX = 0x04, OP_CHUNK = 0x05, OP_CHUNK_INFO = 0x06, OP_CONNECTION = 0x07;
constexpr uint8_t kFloat32 = 7;
constexpr uint64_t kMaxCloudPoints = 1ull << 31;          // the limits of erasor_voxelize_batch
constexpr uint64_t kMaxCallPoints = 0xFFFFFFFFull;

// one cloud as the device gather reads it: point (r, c) at data + r row_step + c point_step; slot s (x y z intensity) at off[s]
// when bit s of fields is set, else 0
struct Cloud {
    uint64_t data_off, data_len;     // the data blob in the file
    uint32_t width, height, point_step, row_step;
    uint32_t fields;
    uint32_t off[4];
    uint32_t big_endian;
};

struct Node {
    uint32_t seq;                    // header.seq
    uint64_t stamp_ns;               // the record's time
    double odom[7];
    Cloud cloud;                     // data_off: in the file, or in the decoded chunk when lz >= 0 or bz >= 0
    int64_t lz = -1;                 // the LZ4 chunk (Index::lz4) holding the node, else -1
    int64_t bz = -1;                 // the bz2 chunk (Index::bz2) holding the node, else -1
    uint64_t rec = 0;                // in a compressed chunk: the index entry's offset of the message record in the decoded chunk
    uint32_t conn = 0;               // in a compressed chunk: the index entry's connection
    bool decoded() const { return lz >= 0 || bz >= 0; }
};

// an LZ4 chunk: the record, its data in the file, its decoded length and its frame's block table
struct Lz4Chunk {
    uint64_t rec, data, len;
    uint32_t size;
    lz4::Frame frame;
};

// a bz2 chunk: the record, its data in the file, its decoded length and its stream's level (the host reads the 4-byte header only)
struct Bz2Chunk {
    uint64_t rec, data, len;
    uint32_t size, level;
};

struct Index {
    std::vector<Node> nodes;         // selected, in delivery order, the first dropped unless keep_first
    std::string md5sum;
    uint64_t chunks = 0, connections = 0, messages = 0, selected = 0, unknown = 0;
    uint64_t total_points = 0, intensity_zero_filled = 0, big_endian = 0;
    std::vector<Lz4Chunk> lz4;       // every LZ4 chunk of the file, in file order
    std::vector<Bz2Chunk> bz2;       // every bz2 chunk of the file, in file order
    std::vector<uint64_t> pending;   // the nodes in compressed chunks, parsed after their chunks are decoded (finish_chunks)
    int fail_rc = 0;                 // the first node parsed on the host that failed, when it follows a pending one
    std::string fail_msg;
};

// ---- the node layout, shared by the host walk and the device parse of nodes in LZ4 chunks ----------------------------------
// why a message is not an erasor/node (0: it is); a and b carry the numbers the message names
enum : uint32_t {
    NF_OK = 0, NF_HEADER, NF_ODOM, NF_ODOMCOV, NF_LIDAR, NF_FIELDS, NF_DATA_PAST, NF_LIDARODOM, NF_IMAGE, NF_GPS,
    NF_LONGER,                       // a: the bytes past the structure
    NF_NO_FIELD,                     // a: the slot (x y z), b: 1 when a field of that name exists
    NF_CAPACITY,                     // 2^31 points or more
    NF_POINT_PAST,                   // a: the byte the last point reads up to, b: lidar.data's length
    NF_REC_PAST,                     // (LZ4) the index entry's record runs past the decoded chunk
    NF_REC_OP,                       // (LZ4) the record there is not a message data record
    NF_REC_CONN,                     // (LZ4) a: its connection
    NF_REC_TIME,                     // (LZ4) a: its time in ns
};

struct Rd {
    const uint8_t* f;
    uint64_t pos, end;
    PCD_HD bool take(uint64_t n) { if (n > end - pos) return false; pos += n; return true; }
    PCD_HD bool u8(uint8_t& v) { if (end - pos < 1) return false; v = f[pos++]; return true; }
    PCD_HD bool u32(uint32_t& v) { if (end - pos < 4) return false; v = pcd::le32(f + pos); pos += 4; return true; }
    PCD_HD bool f64(double& v) {
        if (end - pos < 8) return false;
        const uint64_t u = (uint64_t)pcd::le32(f + pos) | (uint64_t)pcd::le32(f + pos + 4) << 32;
        memcpy(&v, &u, 8);
        pos += 8;
        return true;
    }
    PCD_HD bool skip_str() { uint32_t n; return u32(n) && take(n); }
    PCD_HD bool header(uint32_t* seq) { uint32_t s, t0, t1; if (!u32(s) || !u32(t0) || !u32(t1) || !skip_str()) return false; if (seq) *seq = s; return true; }
};

// The erasor/node message f[d0, end): seq, odom and the cloud layout (data_off from f), or the first broken rule.  Only the
// rules; detail::parse_node turns a code back into its message.
PCD_HD uint32_t parse_node_core(const uint8_t* f, uint64_t d0, uint64_t end, uint32_t* seq, double odom[7], Cloud& cl, uint64_t* a, uint64_t* b) {
    Rd c{f, d0, end};
    if (!c.header(seq)) return NF_HEADER;
    for (int i = 0; i < 7; ++i) if (!c.f64(odom[i])) return NF_ODOM;
    if (!c.take(36 * 8)) return NF_ODOMCOV;
    cl = Cloud{};
    uint32_t nf;
    if (!c.header(nullptr) || !c.u32(cl.height) || !c.u32(cl.width) || !c.u32(nf)) return NF_LIDAR;
    bool taken[4] = {false, false, false, false}, named[4] = {false, false, false, false};
    const char* kNames[4] = {"x", "y", "z", "intensity"};
    for (uint32_t j = 0; j < nf; ++j) {
        uint32_t len, off, count;
        uint8_t dt;
        if (!c.u32(len) || len > c.end - c.pos) return NF_FIELDS;
        const uint8_t* name = f + c.pos;
        c.pos += len;
        if (!c.u32(off) || !c.u8(dt) || !c.u32(count)) return NF_FIELDS;
        for (int s = 0; s < 4; ++s) {
            uint32_t k = 0;
            while (kNames[s][k] && k < len && (uint8_t)kNames[s][k] == name[k]) ++k;
            if (kNames[s][k] || k != len) continue;
            named[s] = true;
            if (!taken[s] && dt == kFloat32 && count <= 1) { taken[s] = true; cl.off[s] = off; cl.fields |= 1u << s; }
        }
    }
    uint8_t be, dense;
    uint32_t dlen;
    if (!c.u8(be) || !c.u32(cl.point_step) || !c.u32(cl.row_step) || !c.u32(dlen)) return NF_LIDAR;
    cl.big_endian = be ? 1u : 0u;
    cl.data_off = c.pos;
    cl.data_len = dlen;
    if (!c.take(dlen)) return NF_DATA_PAST;
    if (!c.u8(dense)) return NF_LIDAR;
    for (int i = 0; i < 7; ++i) { double d; if (!c.f64(d)) return NF_LIDARODOM; }
    if (!c.header(nullptr) || !c.skip_str() || !c.skip_str()) return NF_IMAGE;
    uint8_t st, ct;                  // gps: status (int8 status + uint16 service), latitude .. covariance, covariance type
    if (!c.header(nullptr) || !c.u8(st) || !c.take(2) || !c.take(3 * 8 + 9 * 8) || !c.u8(ct)) return NF_GPS;
    if (c.pos != c.end) { *a = c.end - c.pos; return NF_LONGER; }
    for (int s = 0; s < 3; ++s)
        if (!(cl.fields >> s & 1u)) { *a = s; *b = named[s] ? 1 : 0; return NF_NO_FIELD; }
    const uint64_t n = (uint64_t)cl.width * cl.height;
    if (n >= kMaxCloudPoints) return NF_CAPACITY;
    if (n) {
        uint64_t hi = 0;             // in 64 bits: once this check passes, point_reach's 32-bit sum cannot wrap (data_len < 2^32)
        for (int s = 0; s < 4; ++s)
            if (cl.fields >> s & 1u) hi = hi > (uint64_t)cl.off[s] + 4u ? hi : (uint64_t)cl.off[s] + 4u;
        const uint64_t last = (uint64_t)(cl.height - 1) * cl.row_step + (uint64_t)(cl.width - 1) * cl.point_step;
        if (last + hi > cl.data_len) { *a = last + hi; *b = cl.data_len; return NF_POINT_PAST; }
    }
    return NF_OK;
}

// The message data record at offset `off` of a decoded chunk f[0, len) that an index entry (conn, time_ns) points to: [*d0, *d1)
// its data, or the broken rule
PCD_HD uint32_t record_core(const uint8_t* f, uint64_t len, uint64_t off, uint32_t conn, uint64_t time_ns, uint64_t* d0, uint64_t* d1, uint64_t* a) {
    if (off > len || len - off < 4) return NF_REC_PAST;
    const uint32_t hl = pcd::le32(f + off);
    const uint64_t h0 = off + 4, h1 = h0 + hl;
    if (hl > len - h0 || len - h1 < 4) return NF_REC_PAST;
    const uint32_t dl = pcd::le32(f + h1);
    if (dl > len - h1 - 4) return NF_REC_PAST;
    int have = 0;
    uint32_t c = 0;
    uint64_t t = 0;
    for (uint64_t p = h0; p < h1;) {
        if (h1 - p < 4) return NF_REC_OP;
        const uint32_t n = pcd::le32(f + p);
        if (n > h1 - p - 4) return NF_REC_OP;
        const uint8_t* s = f + p + 4;
        uint32_t k = 0;
        while (k < n && s[k] != '=') ++k;
        if (k == n) return NF_REC_OP;
        const uint8_t* v = s + k + 1;
        const uint32_t vl = n - k - 1;
        if (k == 2 && s[0] == 'o' && s[1] == 'p' && vl == 1 && v[0] == OP_MSG) have |= 1;
        if (k == 4 && s[0] == 'c' && s[1] == 'o' && s[2] == 'n' && s[3] == 'n' && vl == 4) { c = pcd::le32(v); have |= 2; }
        if (k == 4 && s[0] == 't' && s[1] == 'i' && s[2] == 'm' && s[3] == 'e' && vl == 8) { t = (uint64_t)pcd::le32(v) * 1000000000ull + pcd::le32(v + 4); have |= 4; }
        p += 4ull + n;
    }
    if (have != 7) return NF_REC_OP;
    if (c != conn) { *a = c; return NF_REC_CONN; }
    if (t != time_ns) { *a = t; return NF_REC_TIME; }
    *d0 = h1 + 4;
    *d1 = h1 + 4 + dl;
    return NF_OK;
}

PCD_HD uint64_t cloud_points(const Cloud& c) { return (uint64_t)c.width * c.height; }

// where point i (row-major) of cloud c starts in its data
PCD_HD uint64_t point_offset(const Cloud& c, uint64_t i) {
    const uint64_t r = i / c.width;
    return r * c.row_step + (i - r * c.width) * c.point_step;
}

// the four values of the point that starts at p, as bit patterns (copied, never converted: NaN payloads survive)
PCD_HD void point_values(const uint8_t* p, const Cloud& c, uint32_t v[4]) {
    for (int s = 0; s < 4; ++s) v[s] = ((c.fields >> s) & 1u) ? pcd::le32(p + c.off[s]) : 0u;
}

// the bytes a point reads from its start: past the end of the last value it takes
PCD_HD uint32_t point_reach(const Cloud& c) {
    uint32_t hi = 0;
    for (int s = 0; s < 4; ++s)
        if ((c.fields >> s) & 1u) hi = hi > c.off[s] + 4u ? hi : c.off[s] + 4u;
    return hi;
}

// ---- the walk ------------------------------------------------------------------------------------------------------------
namespace detail {

struct Err {
    int rc = ERASOR_OK;
    std::string msg;
    bool set(int code, const std::string& m) { if (rc == ERASOR_OK) { rc = code; msg = m; } return false; }
};

inline uint32_t rd32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
inline std::string at(uint64_t pos) { return " at byte " + std::to_string(pos); }

// header fields (name -> [value offset, length]) of the field block [pos, end)
struct Field { std::string name; uint64_t off, len; };

inline bool read_fields(const uint8_t* f, uint64_t pos, uint64_t end, std::vector<Field>& out, Err& e, const char* what) {
    out.clear();
    while (pos < end) {
        if (end - pos < 4) return e.set(ERASOR_E_INVALID, std::string(what) + ": a header field length runs past the header" + at(pos));
        const uint32_t n = rd32(f + pos);
        if (n > end - pos - 4) return e.set(ERASOR_E_INVALID, std::string(what) + ": a header field runs past the header" + at(pos));
        const uint8_t* s = f + pos + 4;
        const uint8_t* eq = static_cast<const uint8_t*>(std::memchr(s, '=', n));
        if (!eq) return e.set(ERASOR_E_INVALID, std::string(what) + ": a header field without '='" + at(pos));
        out.push_back(Field{std::string(reinterpret_cast<const char*>(s), eq - s), (uint64_t)(eq + 1 - f), (uint64_t)(s + n - eq - 1)});
        pos += 4ull + n;
    }
    return true;
}

inline const Field* find(const std::vector<Field>& fs, const char* name) {
    for (const Field& x : fs) if (x.name == name) return &x;
    return nullptr;
}

// a required field of exactly `len` bytes (0: any length)
inline const Field* need(const std::vector<Field>& fs, const char* name, uint64_t len, uint64_t rec, const char* what, Err& e) {
    const Field* x = find(fs, name);
    if (!x) { e.set(ERASOR_E_INVALID, std::string(what) + " record" + at(rec) + " lacks its '" + name + "' header field"); return nullptr; }
    if (len && x->len != len) {
        e.set(ERASOR_E_INVALID, std::string(what) + " record" + at(rec) + ": header field '" + name + "' has " + std::to_string(x->len) +
                                    " bytes, not " + std::to_string(len));
        return nullptr;
    }
    return x;
}

// the 4-byte header of the bzip2 stream b[0, len): ERASOR_OK with *level, or the code with msg
inline int bz2_header(const uint8_t* b, uint64_t len, uint32_t* level, std::string& msg) {
    if (len < 3 || b[0] != 'B' || b[1] != 'Z' || b[2] != 'h') { msg = "its data does not start with 'BZh' (a bzip1 or other stream?)"; return ERASOR_E_UNSUPPORTED; }
    if (len < 4) { msg = "the stream runs past the chunk (bit 24 of the chunk data)"; return ERASOR_E_INVALID; }
    if (b[3] < '1' || b[3] > '9') { msg = "level digit " + std::to_string(b[3]) + " is not '1'..'9' (bit 24 of the chunk data)"; return ERASOR_E_INVALID; }
    *level = (uint32_t)(b[3] - '0');
    return ERASOR_OK;
}

struct Conn { std::string topic, type, md5sum; bool defined = false; };
// a message: its record and data in the file; or (lz >= 0 / bz >= 0) an index entry of LZ4 chunk lz / bz2 chunk bz, rec its offset
// in the decoded chunk
struct Msg { uint32_t conn; uint64_t time_ns, rec, data, len; int64_t lz = -1, bz = -1; };

struct Walk {
    const uint8_t* f;
    std::vector<Conn> conns;          // by conn id (dense: rosbag numbers them from 0)
    std::vector<uint32_t> conn_ids;   // ids seen, in first-definition order
    std::vector<Msg> msgs;
    uint64_t chunks = 0, unknown = 0;
    std::vector<Lz4Chunk> lz4;
    std::vector<Bz2Chunk> bz2;
    std::vector<Msg> entries;         // the index entries of the last compressed chunk, while its index data records follow it
    Err e;

    // the last compressed chunk's messages, from the index data records that followed it: in file order, by offset in the chunk
    bool close_lz4() {
        if (!open) return true;
        if (entries.empty())
            return e.set(ERASOR_E_UNSUPPORTED, "chunk" + at(open_bz2 ? bz2.back().rec : lz4.back().rec) + " is " + (open_bz2 ? "bz2" : "lz4") +
                                                   "-compressed and no index data record follows it: an unindexed bag is not read");
        std::stable_sort(entries.begin(), entries.end(), [](const Msg& a, const Msg& b) { return a.rec < b.rec; });
        msgs.insert(msgs.end(), entries.begin(), entries.end());
        entries.clear();
        open = false;
        return true;
    }
    bool open = false;                // a compressed chunk was the last chunk and its index data records are being read
    bool open_bz2 = false;            // ... and it is a bz2 chunk

    Conn& conn(uint32_t id) {
        if (id >= conns.size()) conns.resize((size_t)id + 1);
        return conns[id];
    }

    // the records of [pos, end); in_chunk: the records of one chunk's data
    bool records(uint64_t pos, uint64_t end, bool in_chunk) {
        std::vector<Field> fs;
        while (pos < end) {
            const uint64_t rec = pos;
            if (end - pos < 4) return e.set(ERASOR_E_INVALID, "a record's header length runs past its container" + at(rec));
            const uint32_t hl = rd32(f + pos);
            if (hl > end - pos - 4) return e.set(ERASOR_E_INVALID, "a record's header runs past its container" + at(rec));
            const uint64_t h0 = pos + 4, h1 = h0 + hl;
            if (end - h1 < 4) return e.set(ERASOR_E_INVALID, "a record's data length runs past its container" + at(rec));
            const uint32_t dl = rd32(f + h1);
            if (dl > end - h1 - 4) return e.set(ERASOR_E_INVALID, "a record's data runs past its container" + at(rec));
            const uint64_t d0 = h1 + 4, d1 = d0 + dl;
            if (!read_fields(f, h0, h1, fs, e, "record")) return false;
            const Field* op = find(fs, "op");
            if (!op || op->len != 1) return e.set(ERASOR_E_INVALID, "a record without a one-byte 'op' header field" + at(rec));
            const uint8_t o = f[op->off];
            if (!one(o, fs, rec, d0, dl, in_chunk)) return false;
            pos = d1;
        }
        return true;
    }

    bool one(uint8_t o, const std::vector<Field>& fs, uint64_t rec, uint64_t d0, uint32_t dl, bool in_chunk) {
        switch (o) {
        case OP_BAG_HEADER:
            if (in_chunk) return e.set(ERASOR_E_INVALID, "a bag header record inside a chunk" + at(rec));
            return need(fs, "index_pos", 8, rec, "bag header", e) && need(fs, "conn_count", 4, rec, "bag header", e) &&
                   need(fs, "chunk_count", 4, rec, "bag header", e);
        case OP_CHUNK: {
            if (in_chunk) return e.set(ERASOR_E_INVALID, "a chunk record inside a chunk" + at(rec));
            const Field* c = need(fs, "compression", 0, rec, "chunk", e);
            const Field* s = c ? need(fs, "size", 4, rec, "chunk", e) : nullptr;
            if (!s) return false;
            if (!close_lz4()) return false;
            const std::string comp(reinterpret_cast<const char*>(f + c->off), c->len);
            if (comp == "lz4") {
                Lz4Chunk k{rec, d0, dl, rd32(f + s->off), lz4::Frame()};
                std::string m;
                const int fr = lz4::parse_frame(f + d0, dl, k.size, k.frame, m);
                if (fr != lz4::F_OK) return e.set(fr == lz4::F_UNSUPPORTED ? ERASOR_E_UNSUPPORTED : ERASOR_E_INVALID, "lz4 chunk" + at(rec) + ": " + m);
                ++chunks;
                lz4.push_back(std::move(k));
                open = true;
                open_bz2 = false;
                return true;
            }
            if (comp == "bz2") {             // the stream header only: the device finds the blocks (DESIGN.md section 12.2.2)
                uint32_t level = 0;
                std::string m;
                const int hr = bz2_header(f + d0, dl, &level, m);
                if (hr != ERASOR_OK) return e.set(hr, "bz2 chunk" + at(rec) + ": " + m);
                ++chunks;
                bz2.push_back(Bz2Chunk{rec, d0, dl, rd32(f + s->off), level});
                open = true;
                open_bz2 = true;
                return true;
            }
            if (comp != "none")
                return e.set(ERASOR_E_UNSUPPORTED, "chunk" + at(rec) + " is compressed with '" + comp + "': only uncompressed, lz4 and bz2 chunks are read");
            if (rd32(f + s->off) != dl)
                return e.set(ERASOR_E_INVALID, "chunk" + at(rec) + " holds " + std::to_string(dl) + " bytes of data, its 'size' says " +
                                                   std::to_string(rd32(f + s->off)));
            ++chunks;
            return records(d0, d0 + dl, true);
        }
        case OP_CONNECTION: {
            const Field* id = need(fs, "conn", 4, rec, "connection", e);
            const Field* tp = id ? need(fs, "topic", 0, rec, "connection", e) : nullptr;
            if (!tp) return false;
            std::vector<Field> ch;
            if (!read_fields(f, d0, d0 + dl, ch, e, "connection header")) return false;
            const Field* ty = need(ch, "type", 0, rec, "connection", e);
            const Field* md = ty ? need(ch, "md5sum", 0, rec, "connection", e) : nullptr;
            if (!md) return false;
            const uint32_t k = rd32(f + id->off);
            Conn& c = conn(k);
            if (!c.defined) conn_ids.push_back(k);
            c.defined = true;
            c.topic.assign(reinterpret_cast<const char*>(f + tp->off), tp->len);
            c.type.assign(reinterpret_cast<const char*>(f + ty->off), ty->len);
            c.md5sum.assign(reinterpret_cast<const char*>(f + md->off), md->len);
            return true;
        }
        case OP_MSG: {
            const Field* id = need(fs, "conn", 4, rec, "message data", e);
            const Field* t = id ? need(fs, "time", 8, rec, "message data", e) : nullptr;
            if (!t) return false;
            const uint64_t ns = (uint64_t)rd32(f + t->off) * 1000000000ull + rd32(f + t->off + 4);
            msgs.push_back(Msg{rd32(f + id->off), ns, rec, d0, dl});
            return true;
        }
        case OP_INDEX: {
            const Field* v = need(fs, "ver", 4, rec, "index data", e);
            const Field* c = v && need(fs, "conn", 4, rec, "index data", e) ? need(fs, "count", 4, rec, "index data", e) : nullptr;
            if (!c) return false;
            if ((uint64_t)rd32(f + c->off) * 12u != dl)
                return e.set(ERASOR_E_INVALID, "index data record" + at(rec) + ": " + std::to_string(dl) + " bytes of data for " +
                                                   std::to_string(rd32(f + c->off)) + " entries of 12");
            if (open && !in_chunk) {
                const Field* cn = find(fs, "conn");
                for (uint64_t q = d0; q < d0 + dl; q += 12)
                    entries.push_back(Msg{rd32(f + cn->off), (uint64_t)rd32(f + q) * 1000000000ull + rd32(f + q + 4), rd32(f + q + 8), 0, 0,
                                          open_bz2 ? -1 : (int64_t)lz4.size() - 1, open_bz2 ? (int64_t)bz2.size() - 1 : -1});
            }
            return true;
        }
        case OP_CHUNK_INFO: {
            const char* w = "chunk info";
            const Field* c = need(fs, "ver", 4, rec, w, e) && need(fs, "chunk_pos", 8, rec, w, e) && need(fs, "start_time", 8, rec, w, e) &&
                                     need(fs, "end_time", 8, rec, w, e) ? need(fs, "count", 4, rec, w, e) : nullptr;
            if (!c) return false;
            if ((uint64_t)rd32(f + c->off) * 8u != dl)
                return e.set(ERASOR_E_INVALID, "chunk info record" + at(rec) + ": " + std::to_string(dl) + " bytes of data for " +
                                                   std::to_string(rd32(f + c->off)) + " entries of 8");
            return true;
        }
        default:
            ++unknown;
            return true;
        }
    }
};

// the message of a parse_node_core / record_core code for the node `who`; false with e set (true for NF_OK)
inline bool node_fail(uint32_t code, uint64_t a, uint64_t b, const std::string& who, Err& e) {
    static const char* kNames[4] = {"x", "y", "z", "intensity"};
    auto bad = [&](const std::string& what) { return e.set(ERASOR_E_INVALID, who + ": " + what); };
    switch (code) {
    case NF_OK: return true;
    case NF_HEADER: return bad("the message ends inside its header");
    case NF_ODOM: return bad("the message ends inside odom");
    case NF_ODOMCOV: return bad("the message ends inside odomCov");
    case NF_LIDAR: return bad("the message ends inside lidar");
    case NF_FIELDS: return bad("the message ends inside lidar.fields");
    case NF_DATA_PAST: return bad("lidar.data runs past the message");
    case NF_LIDARODOM: return bad("the message ends inside lidarOdom");
    case NF_IMAGE: return bad("the message ends inside image");
    case NF_GPS: return bad("the message ends inside gps");
    case NF_LONGER: return bad("the message is " + std::to_string(a) + " bytes longer than an erasor/node");
    case NF_NO_FIELD:
        return e.set(ERASOR_E_UNSUPPORTED, who + ": lidar has no field '" + kNames[a] + (b ? "' of datatype FLOAT32 and count 1" : "'"));
    case NF_CAPACITY: return e.set(ERASOR_E_CAPACITY, who + ": a cloud of 2^31 points or more");
    case NF_POINT_PAST:
        return bad("its last point reads up to byte " + std::to_string(a) + " of lidar.data, which holds " + std::to_string(b));
    case NF_REC_PAST: return bad("the index entry's record runs past the decoded chunk");
    case NF_REC_OP: return bad("the index entry does not point to a message data record");
    case NF_REC_CONN: return bad("the record there is on connection " + std::to_string(a) + ", not the index entry's");
    case NF_REC_TIME: return bad("the record there has time " + std::to_string(a) + " ns, not the index entry's");
    default: return bad("unknown node error");
    }
}

// one erasor/node message -> node; false with e set when it is malformed or its cloud cannot be decoded
inline bool parse_node(const uint8_t* f, const Msg& m, uint64_t k, Node& nd, Err& e, uint64_t& zero_filled) {
    nd.stamp_ns = m.time_ns;
    uint64_t a = 0, b = 0;
    const uint32_t code = parse_node_core(f, m.data, m.data + m.len, &nd.seq, nd.odom, nd.cloud, &a, &b);
    if (!node_fail(code, a, b, "node " + std::to_string(k) + " (message record" + at(m.rec) + ")", e)) return false;
    if (!(nd.cloud.fields & 8u)) ++zero_filled;
    return true;
}

}  // namespace detail

// The index of the bag in file[0, len): every message on `topic`, in delivery order (a stable sort by record time), parsed as an
// erasor/node; the first one dropped unless keep_first.  ERASOR_OK, or an error code with msg.
inline int build_index(const uint8_t* file, uint64_t len, const std::string& topic, bool keep_first, Index& out, std::string& msg) {
    out = Index();
    static const char kMagic[] = "#ROSBAG V";
    if (len < 13 || std::memcmp(file, kMagic, 9) != 0) { msg = "not a ROS bag: the file does not start with '#ROSBAG V'"; return ERASOR_E_INVALID; }
    if (std::memcmp(file, "#ROSBAG V2.0\n", 13) != 0) {
        const uint8_t* nl = static_cast<const uint8_t*>(std::memchr(file, '\n', std::min<uint64_t>(len, 64)));
        msg = "'" + std::string(reinterpret_cast<const char*>(file), nl ? nl - file : 12) + "': only ROS bag version 2.0 is read";
        return ERASOR_E_UNSUPPORTED;
    }
    detail::Walk w{file};
    if (!w.records(13, len, false) || !w.close_lz4()) { msg = w.e.msg; return w.e.rc; }
    out.lz4 = std::move(w.lz4);
    out.bz2 = std::move(w.bz2);
    out.chunks = w.chunks;
    out.unknown = w.unknown;
    out.connections = w.conn_ids.size();
    out.messages = w.msgs.size();
    std::vector<detail::Msg> sel;
    for (const detail::Msg& m : w.msgs) {
        if (m.conn >= w.conns.size() || !w.conns[m.conn].defined) {
            msg = "message record" + detail::at(m.rec) + " is on connection " + std::to_string(m.conn) + ", which the bag never defines";
            return ERASOR_E_INVALID;
        }
        if (w.conns[m.conn].topic == topic) sel.push_back(m);
    }
    for (uint32_t id : w.conn_ids) {
        const detail::Conn& c = w.conns[id];
        if (c.topic != topic) continue;
        if (c.type != "erasor/node") { msg = "topic " + topic + " carries '" + c.type + "' messages, not erasor/node"; return ERASOR_E_UNSUPPORTED; }
        if (out.md5sum.empty()) out.md5sum = c.md5sum;
    }
    out.selected = sel.size();
    std::stable_sort(sel.begin(), sel.end(), [](const detail::Msg& a, const detail::Msg& b) { return a.time_ns < b.time_ns; });
    const size_t first = keep_first || sel.empty() ? 0 : 1;
    out.nodes.resize(sel.size() - first);
    detail::Err e;
    for (size_t k = first; k < sel.size(); ++k) {
        Node& nd = out.nodes[k - first];
        if (sel[k].lz >= 0 || sel[k].bz >= 0) {       // parsed once its chunk is decoded (finish_chunks)
            nd.lz = sel[k].lz;
            nd.bz = sel[k].bz;
            nd.rec = sel[k].rec;
            nd.conn = sel[k].conn;
            nd.stamp_ns = sel[k].time_ns;
            out.pending.push_back(k - first);
            continue;
        }
        if (!detail::parse_node(file, sel[k], k - first, nd, e, out.intensity_zero_filled)) {
            if (!out.pending.empty()) { out.fail_rc = e.rc; out.fail_msg = e.msg; out.nodes.resize(k - first + 1); break; }
            msg = e.msg; const int rc = e.rc; out.nodes.clear(); return rc;
        }
        out.total_points += cloud_points(nd.cloud);
        out.big_endian += nd.cloud.big_endian;
    }
    return ERASOR_OK;
}

// ---- nodes in compressed chunks: what the device (or the host build, serially) decodes and parses --------------------------------
// A block of the LZ4 decode, an LZ4 chunk, a bz2 chunk, and a node to parse, as the kernels read them
struct Lz4Block {
    uint64_t src;                    // its data in the device copy of the compressed chunks
    uint32_t csize, stored, cap;     // cap: the frame's block max
    uint32_t chunk;                  // its chunk in ChunkPlan::chunks
    uint32_t has_sum, sum;
};
struct Lz4ChunkDesc {
    uint64_t src, dec;               // its compressed data in the device copy, its decoded data in the decoded buffer
    uint32_t size, block0, nblocks, has_sum, sum, pad_;
};
struct Bz2ChunkDesc {
    uint64_t src, len;               // its stream in the device copy of the bz2 chunks, its length
    uint64_t dec;                    // its decoded data in the decoded buffer
    uint64_t tt;                     // its blocks' slots in the BWT buffers: ceil(5 size / 4) bytes
    uint64_t cand_cap;               // max_candidates(len)
    uint32_t size, level;
};
struct Lz4NodeIn { uint64_t dec, len, rec, time_ns; uint32_t conn, pad_; };   // the decoded chunk [dec, dec + len), the index entry
struct NodeOut {
    uint32_t code, seq;
    uint64_t a, b;
    double odom[7];
    Cloud cloud;
};

// the BWT buffers of a bz2 chunk of decoded length `size`: the tt bytes of its true blocks total at most ceil(5 size / 4), as RLE1
// turns at most 5 bytes into 4
PCD_HD uint64_t tt_cap(uint32_t size) { return (5ull * size + 3) / 4; }

struct ChunkPlan {
    std::vector<uint32_t> chunks;    // Index::lz4 ids holding a kept node, in file order
    std::vector<Lz4ChunkDesc> cd;
    std::vector<Lz4Block> blocks;
    std::vector<uint32_t> bz_chunks; // Index::bz2 ids holding a kept node, in file order
    std::vector<Bz2ChunkDesc> bd;
    std::vector<Lz4NodeIn> nodes;    // Index::pending, in order
    std::vector<int64_t> slot;       // Index::lz4 id -> its entry of chunks / cd, or -1
    std::vector<int64_t> bz_slot;    // Index::bz2 id -> its entry of bz_chunks / bd, or -1
    uint64_t src_bytes = 0, dec_bytes = 0, stored = 0, block_sums = 0, content_sums = 0;
    uint64_t bz_src_bytes = 0, bz_tt_bytes = 0, bz_cands = 0;   // bz2: the bounds every buffer is sized from
};

// where node nd (in a compressed chunk) has its decoded chunk in the decoded buffer
inline uint64_t dec_of(const ChunkPlan& p, const Node& nd) { return nd.lz >= 0 ? p.cd[p.slot[nd.lz]].dec : p.bd[p.bz_slot[nd.bz]].dec; }

inline void fill_lz4_stats(const Index& x, const ChunkPlan& p, erasor_bag_lz4_stats_t& s) {
    s = erasor_bag_lz4_stats_t{};
    s.chunks = x.lz4.size();
    s.decoded_chunks = p.chunks.size();
    for (uint32_t c : p.chunks) { s.compressed_bytes += x.lz4[c].len; s.decoded_bytes += x.lz4[c].size; }
    s.blocks = p.blocks.size();
    s.stored_blocks = p.stored;
    s.block_checksums = p.block_sums;
    s.content_checksums = p.content_sums;
}

// what the bz2 decode found: per decoded chunk its true blocks; the candidates of all
struct Bz2Found {
    std::vector<uint32_t> blocks;
    uint64_t candidates = 0;
};

inline void fill_bz2_stats(const Index& x, const ChunkPlan& p, const Bz2Found& f, erasor_bag_bz2_stats_t& s) {
    s = erasor_bag_bz2_stats_t{};
    s.chunks = x.bz2.size();
    for (const Bz2Chunk& k : x.bz2) ++s.streams_by_level[k.level - 1];
    s.decoded_chunks = p.bz_chunks.size();
    for (uint32_t c : p.bz_chunks) { s.compressed_bytes += x.bz2[c].len; s.decoded_bytes += x.bz2[c].size; }
    for (uint32_t b : f.blocks) s.blocks += b;
    s.candidates = f.candidates;
}

// the decode error key: the first broken rule in (block, byte) order wins an atomicMin
// unit: the position in file order of what broke, counting each decoded chunk's blocks, then one unit for the chunk as a whole
// (its decoded length and content checksum); block b of chunk c is unit b + c, chunk c's own unit block0 + nblocks + c, so a
// chunk without blocks still has a unit of its own
PCD_HD uint64_t err_key(uint64_t unit, uint32_t byte, uint32_t reason) { return unit << 28 | (uint64_t)(byte & 0x7FFFFFu) << 5 | reason; }
PCD_HD uint64_t block_key(const Lz4Block& B, uint64_t b, uint32_t byte, uint32_t reason) { return err_key(b + B.chunk, byte, reason); }
PCD_HD uint64_t chunk_key(const Lz4ChunkDesc& d, uint64_t c, uint32_t reason) {
    return err_key((uint64_t)d.block0 + d.nblocks + c, reason == lz4::R_SIZE ? 0 : 1, reason);    // a short frame before its checksum
}
// the bz2 error key, its own atomicMin: the decoded bz2 chunk (file order), then the bit of its data where the rule broke (the
// block's magic for a rule checked after the walk, the chunk's end for its decoded length), then the reason
PCD_HD uint64_t bz2_key(uint64_t c, uint64_t bit, uint32_t reason) { return c << 44 | (bit & 0xFFFFFFFFFull) << 8 | reason; }
constexpr uint64_t kMaxBz2Chunks = 1ull << 20;

// a candidate block of the bz2 decode: the bit of its chunk's data holding the block magic, and the chunk (ChunkPlan::bd)
struct Bz2Cand { uint64_t bit; uint32_t chunk, pad_; };

// The chain of decoded bz2 chunk c (data d, candidates [c0, c1) in bit order, walked): from bit 32, each position must hold a
// candidate whose walk succeeded (a true block, given block number blkno and, while the blocks' lengths fit tt_cap, its BWT slot
// tt_off) or the end-of-stream magic, its stream CRC and the chunk's end.  The key of the first broken rule, or ~0 with *nblocks.
PCD_HD uint64_t bz2_chain(uint64_t c, const Bz2ChunkDesc& D, const uint8_t* d, const Bz2Cand* cand, uint64_t c0, uint64_t c1,
                          const bz2::Walk* walk, int32_t* blkno, uint64_t* tt_off, uint32_t* nblocks) {
    const uint64_t nbits = 8 * D.len, cap = tt_cap(D.size);
    uint64_t pos = 32, tt = 0, i = c0, key = ~0ull;
    uint32_t blk = 0, comb = 0;
    for (;;) {
        while (i < c1 && cand[i].bit < pos) ++i;
        if (i < c1 && cand[i].bit == pos) {
            const bz2::Walk w = walk[i];
            blkno[i] = (int32_t)blk;
            if (w.reason != bz2::R_OK) return bz2_key(c, w.where, w.reason);
            if (key == ~0ull && w.n <= cap - tt) { tt_off[i] = D.tt + tt; tt += w.n; }
            else key = bz2_key(c, nbits, bz2::R_SIZE);        // more than the chunk's size can need: decode no further block
            comb = (comb << 1 | comb >> 31) ^ w.crc;
            pos = w.end;
            ++blk;
            continue;
        }
        uint64_t k;
        if (nbits - pos < 48) k = bz2_key(c, pos, bz2::R_PAST);
        else if (bz2::magic_at(d, pos) != bz2::kEosMagic) k = bz2_key(c, pos, bz2::R_NO_MAGIC);
        else if (nbits - pos - 48 < 32) k = bz2_key(c, pos + 48, bz2::R_PAST);
        else {
            bz2::Bits b{d, pos + 48, nbits};
            const uint32_t stored = b.get(32);
            const uint64_t end = (pos + 80 + 7) / 8;
            if (end != D.len) {
                const bool bzh = D.len - end >= 3 && d[end] == 'B' && d[end + 1] == 'Z' && d[end + 2] == 'h';
                k = bz2_key(c, 8 * end, bzh ? bz2::R_SECOND_STREAM : bz2::R_TRAILING);
            } else if (stored != comb) {
                k = bz2_key(c, pos + 48, bz2::R_STREAM_CRC);
            } else {
                *nblocks = blk;
                return key;
            }
        }
        return k < key ? k : key;
    }
}

// The placement of decoded bz2 chunk c's blocks (RLE1 output lengths osize, ~0 for a block that failed): their offsets in the
// decoded buffer, or ~0 for all unless they add up to the chunk's size.  The key of a wrong decoded length, or ~0.
PCD_HD uint64_t bz2_place(uint64_t c, const Bz2ChunkDesc& D, uint64_t c0, uint64_t c1, const uint64_t* tt_off, const uint64_t* osize, uint64_t* out_off) {
    uint64_t s = 0;
    bool failed = false;
    for (uint64_t i = c0; i < c1; ++i)
        if (tt_off[i] != ~0ull) { if (osize[i] == ~0ull) failed = true; else s += osize[i]; }
    const bool ok = !failed && s == D.size;
    s = 0;
    for (uint64_t i = c0; i < c1; ++i)
        if (tt_off[i] != ~0ull) { out_off[i] = ok ? D.dec + s : ~0ull; s += ok ? osize[i] : 0; }
    return ok || failed ? ~0ull : bz2_key(c, 8 * D.len, bz2::R_SIZE);
}

inline void plan_chunks(const Index& x, ChunkPlan& p) {
    p = ChunkPlan();
    p.slot.assign(x.lz4.size(), -1);
    p.bz_slot.assign(x.bz2.size(), -1);
    for (uint64_t k : x.pending) {
        const Node& nd = x.nodes[k];
        if (nd.lz >= 0) p.slot[nd.lz] = 0;
        else p.bz_slot[nd.bz] = 0;
    }
    // the kept chunks of both kinds in file order: the decoded buffer holds their slots in that order
    std::vector<std::pair<uint64_t, int64_t>> order;      // (record, lz4 id or -1 - bz2 id)
    for (size_t c = 0; c < x.lz4.size(); ++c) if (p.slot[c] >= 0) order.push_back({x.lz4[c].rec, (int64_t)c});
    for (size_t c = 0; c < x.bz2.size(); ++c) if (p.bz_slot[c] >= 0) order.push_back({x.bz2[c].rec, -1 - (int64_t)c});
    std::sort(order.begin(), order.end());
    for (const auto& o : order) {
        if (o.second < 0) {
            const size_t c = (size_t)(-1 - o.second);
            const Bz2Chunk& k = x.bz2[c];
            p.bz_slot[c] = (int64_t)p.bz_chunks.size();
            p.bz_chunks.push_back((uint32_t)c);
            const uint64_t cands = bz2::max_candidates(k.len);
            p.bd.push_back(Bz2ChunkDesc{p.bz_src_bytes, k.len, p.dec_bytes, p.bz_tt_bytes, cands, k.size, k.level});
            p.bz_src_bytes += (k.len + 15) & ~15ull;
            p.bz_tt_bytes += (tt_cap(k.size) + 15) & ~15ull;
            p.bz_cands += cands;
            p.dec_bytes += ((uint64_t)k.size + 15) & ~15ull;
            continue;
        }
        const size_t c = (size_t)o.second;
        p.slot[c] = (int64_t)p.chunks.size();
        p.chunks.push_back((uint32_t)c);
        const Lz4Chunk& k = x.lz4[c];
        Lz4ChunkDesc d{p.src_bytes, p.dec_bytes, k.size, (uint32_t)p.blocks.size(), (uint32_t)k.frame.blocks.size(), k.frame.content_sum, k.frame.sum, 0};
        for (const lz4::Block& b : k.frame.blocks) {
            p.blocks.push_back(Lz4Block{d.src + b.off, b.csize, b.stored, k.frame.block_max, (uint32_t)(p.cd.size()), k.frame.block_sums, b.sum});
            p.stored += b.stored;
            p.block_sums += k.frame.block_sums;
        }
        p.content_sums += k.frame.content_sum;
        p.cd.push_back(d);
        p.src_bytes += (k.len + 15) & ~15ull;
        p.dec_bytes += ((uint64_t)k.size + 15) & ~15ull;
    }
    for (uint64_t k : x.pending) {
        const Node& nd = x.nodes[k];
        const uint64_t dec = dec_of(p, nd), size = nd.lz >= 0 ? x.lz4[nd.lz].size : x.bz2[nd.bz].size;
        p.nodes.push_back(Lz4NodeIn{dec, size, nd.rec, nd.stamp_ns, nd.conn, 0});
    }
}

// the message of an LZ4 decode error key
inline std::string lz4_error(const Index& x, const ChunkPlan& p, uint64_t key) {
    const uint64_t u = key >> 28;
    const uint32_t byte = (uint32_t)(key >> 5) & 0x7FFFFFu, r = (uint32_t)key & 31u;
    size_t c = 0;                                    // the chunk whose units [block0 + c, block0 + c + nblocks] hold u
    while (c + 1 < p.cd.size() && (uint64_t)p.cd[c + 1].block0 + c + 1 <= u) ++c;
    const Lz4Chunk& k = x.lz4[p.chunks[c]];
    const uint64_t blk = u - p.cd[c].block0 - c;     // == nblocks: the chunk as a whole
    const std::string m = "lz4 chunk" + detail::at(k.rec) + ": ";
    if (r == lz4::R_SIZE) return m + "its frame does not decode to the chunk's 'size' of " + std::to_string(k.size) + " bytes";
    if (r == lz4::R_CONTENT_SUM) return m + "the content checksum does not match";
    if (r == lz4::R_BLOCK_SUM) return m + "block " + std::to_string(blk) + ": the block checksum does not match";
    return m + "malformed block " + std::to_string(blk) + ": " + lz4::reason_text(r) + " (byte " + std::to_string(k.frame.blocks[blk].off + byte) +
           " of the frame)";
}

// the message of a bz2 decode error key; blk: the last block of the chunk starting at or before the key's bit (-1: none)
inline std::string bz2_error(const Index& x, const ChunkPlan& p, uint64_t key, int64_t blk, int* rc) {
    const uint64_t c = key >> 44, bit = (key >> 8) & 0xFFFFFFFFFull;
    const uint32_t r = (uint32_t)key & 0xFFu;
    const Bz2Chunk& k = x.bz2[p.bz_chunks[c]];
    *rc = bz2::unsupported(r) ? ERASOR_E_UNSUPPORTED : ERASOR_E_INVALID;
    const std::string m = "bz2 chunk" + detail::at(k.rec) + ": ";
    if (r == bz2::R_SIZE) return m + "its stream does not decode to the chunk's 'size' of " + std::to_string(k.size) + " bytes";
    if (r == bz2::R_TRAILING || r == bz2::R_SECOND_STREAM) return m + bz2::reason_text(r) + " (byte " + std::to_string(bit / 8) + " of the chunk data)";
    const std::string where = " (bit " + std::to_string(bit) + " of the chunk data)";
    if (r == bz2::R_STREAM_CRC) return m + bz2::reason_text(r) + where;
    if (r == bz2::R_NO_MAGIC || (r == bz2::R_PAST && blk < 0))
        return m + bz2::reason_text(r) + (blk < 0 ? " after the stream header" : " after block " + std::to_string(blk)) + where;
    return m + "block " + std::to_string(blk) + ": " + bz2::reason_text(r) + where;
}

// the first of the two decode errors in file order (an LZ4 key and a bz2 key, ~0 for none): its code and message, or ERASOR_OK
inline int decode_error(const Index& x, const ChunkPlan& p, uint64_t lz_key, uint64_t bz_key, int64_t bz_blk, std::string& msg) {
    if (lz_key == ~0ull && bz_key == ~0ull) return ERASOR_OK;
    uint64_t lz_rec = ~0ull, bz_rec = ~0ull;
    if (lz_key != ~0ull) {
        const uint64_t u = lz_key >> 28;
        size_t c = 0;
        while (c + 1 < p.cd.size() && (uint64_t)p.cd[c + 1].block0 + c + 1 <= u) ++c;
        lz_rec = x.lz4[p.chunks[c]].rec;
    }
    if (bz_key != ~0ull) bz_rec = x.bz2[p.bz_chunks[bz_key >> 44]].rec;
    if (lz_rec < bz_rec) { msg = lz4_error(x, p, lz_key); return ERASOR_E_INVALID; }
    int rc = ERASOR_E_INVALID;
    msg = bz2_error(x, p, bz_key, bz_blk, &rc);
    return rc;
}

// The nodes of x.pending from their parse (res, in x.pending's order), then the first failure in delivery order: ERASOR_OK or an
// error code with msg (the index is then cleared)
inline int finish_chunks(Index& x, const NodeOut* res, std::string& msg) {
    detail::Err e;
    for (size_t i = 0; i < x.pending.size() && e.rc == ERASOR_OK; ++i) {
        const uint64_t k = x.pending[i];
        Node& nd = x.nodes[k];
        const NodeOut& r = res[i];
        const std::string who = "node " + std::to_string(k) + " (message record at byte " + std::to_string(nd.rec) + " of " +
                                (nd.lz >= 0 ? "lz4 chunk" + detail::at(x.lz4[nd.lz].rec) : "bz2 chunk" + detail::at(x.bz2[nd.bz].rec)) + ")";
        if (!detail::node_fail(r.code, r.a, r.b, who, e)) break;
        nd.seq = r.seq;
        std::memcpy(nd.odom, r.odom, sizeof(nd.odom));
        nd.cloud = r.cloud;
    }
    if (e.rc == ERASOR_OK && x.fail_rc) e.set(x.fail_rc, x.fail_msg);
    if (e.rc != ERASOR_OK) { msg = e.msg; x.nodes.clear(); return e.rc; }
    for (uint64_t k : x.pending) {
        const Cloud& c = x.nodes[k].cloud;
        x.total_points += cloud_points(c);
        x.big_endian += c.big_endian;
        x.intensity_zero_filled += (c.fields & 8u) ? 0 : 1;
    }
    return ERASOR_OK;
}

inline void fill_cloud(const Cloud& c, erasor_bag_cloud_t& o) {
    o.data_offset = c.data_off;
    o.data_len = c.data_len;
    o.width = c.width;
    o.height = c.height;
    o.point_step = c.point_step;
    o.row_step = c.row_step;
    o.fields = c.fields;
    o.big_endian = c.big_endian;
    for (int s = 0; s < 4; ++s) o.offset[s] = c.off[s];
}

inline void fill_info(const Index& x, erasor_bag_info_t& o) {
    o = erasor_bag_info_t{};
    o.version = 200;
    o.chunks = x.chunks;
    o.connections = x.connections;
    o.messages = x.messages;
    o.selected = x.selected;
    o.unknown_records = x.unknown;
    o.nodes = x.nodes.size();
    o.total_points = x.total_points;
    o.intensity_zero_filled = x.intensity_zero_filled;
    o.big_endian = x.big_endian;
    std::strncpy(o.md5sum, x.md5sum.c_str(), sizeof(o.md5sum) - 1);
}

// the node range [first, first + count) of x: ERASOR_OK, or ERASOR_E_INVALID with msg
inline int check_range(const Index& x, uint64_t first, uint64_t count, std::string& msg) {
    if (first > x.nodes.size() || count > x.nodes.size() - first) {
        msg = "nodes [" + std::to_string(first) + ", " + std::to_string(first + count) + ") lie outside the bag's " + std::to_string(x.nodes.size());
        return ERASOR_E_INVALID;
    }
    return ERASOR_OK;
}

// the nodes list[0 .. count) of x: ERASOR_OK, or ERASOR_E_INVALID / ERASOR_E_CAPACITY with msg; *points = their points
inline int check_list(const Index& x, const uint64_t* list, uint64_t count, uint64_t* points, std::string& msg) {
    uint64_t n = 0;
    for (uint64_t k = 0; k < count; ++k) {
        if (list[k] >= x.nodes.size()) {
            msg = "node " + std::to_string(list[k]) + " lies outside the bag's " + std::to_string(x.nodes.size());
            return ERASOR_E_INVALID;
        }
        n += cloud_points(x.nodes[list[k]].cloud);
    }
    *points = n;
    if (n >= kMaxCallPoints) { msg = "2^32 - 1 points or more in one call"; return ERASOR_E_CAPACITY; }
    return ERASOR_OK;
}

}  // namespace bag
