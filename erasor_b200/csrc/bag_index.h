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
    Cloud cloud;
};

struct Index {
    std::vector<Node> nodes;         // selected, in delivery order, the first dropped unless keep_first
    std::string md5sum;
    uint64_t chunks = 0, connections = 0, messages = 0, selected = 0, unknown = 0;
    uint64_t total_points = 0, intensity_zero_filled = 0, big_endian = 0;
};

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

// a bounded reader over [pos, end) of the file
struct Cur {
    const uint8_t* f;
    uint64_t pos, end;
    bool take(uint64_t n) { if (n > end - pos) return false; pos += n; return true; }
    bool u8(uint8_t& v) { if (end - pos < 1) return false; v = f[pos++]; return true; }
    bool u32(uint32_t& v) { if (end - pos < 4) return false; v = rd32(f + pos); pos += 4; return true; }
    bool f64(double& v) { if (end - pos < 8) return false; std::memcpy(&v, f + pos, 8); pos += 8; return true; }
    bool str(std::string& s) {
        uint32_t n;
        if (!u32(n) || n > end - pos) return false;
        s.assign(reinterpret_cast<const char*>(f + pos), n);
        pos += n;
        return true;
    }
    bool skip_str() { uint32_t n; return u32(n) && take(n); }
};

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

struct Conn { std::string topic, type, md5sum; bool defined = false; };
struct Msg { uint32_t conn; uint64_t time_ns, rec, data, len; };

struct Walk {
    const uint8_t* f;
    std::vector<Conn> conns;          // by conn id (dense: rosbag numbers them from 0)
    std::vector<uint32_t> conn_ids;   // ids seen, in first-definition order
    std::vector<Msg> msgs;
    uint64_t chunks = 0, unknown = 0;
    Err e;

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
            const std::string comp(reinterpret_cast<const char*>(f + c->off), c->len);
            if (comp != "none")
                return e.set(ERASOR_E_UNSUPPORTED, "chunk" + at(rec) + " is compressed with '" + comp + "': only uncompressed chunks are read");
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

// a std_msgs/Header: seq, stamp, frame_id
inline bool skip_header(Cur& c, uint32_t* seq) {
    uint32_t s, t0, t1;
    if (!c.u32(s) || !c.u32(t0) || !c.u32(t1) || !c.skip_str()) return false;
    if (seq) *seq = s;
    return true;
}

// one erasor/node message -> node; false with e set when it is malformed or its cloud cannot be decoded
inline bool parse_node(const uint8_t* f, const Msg& m, uint64_t k, Node& nd, Err& e, uint64_t& zero_filled) {
    const std::string who = "node " + std::to_string(k) + " (message record" + at(m.rec) + ")";
    Cur c{f, m.data, m.data + m.len};
    auto bad = [&](const char* what) { return e.set(ERASOR_E_INVALID, who + ": " + what); };
    nd.stamp_ns = m.time_ns;
    if (!skip_header(c, &nd.seq)) return bad("the message ends inside its header");
    for (int i = 0; i < 7; ++i) if (!c.f64(nd.odom[i])) return bad("the message ends inside odom");
    if (!c.take(36 * 8)) return bad("the message ends inside odomCov");
    // lidar: sensor_msgs/PointCloud2
    Cloud& cl = nd.cloud;
    cl = Cloud{};
    uint32_t nf;
    if (!skip_header(c, nullptr) || !c.u32(cl.height) || !c.u32(cl.width) || !c.u32(nf)) return bad("the message ends inside lidar");
    int slot_field[4] = {-1, -1, -1, -1};
    bool named[4] = {false, false, false, false};
    static const char* kNames[4] = {"x", "y", "z", "intensity"};
    for (uint32_t j = 0; j < nf; ++j) {
        std::string name;
        uint32_t off, count;
        uint8_t dt;
        if (!c.str(name) || !c.u32(off) || !c.u8(dt) || !c.u32(count)) return bad("the message ends inside lidar.fields");
        for (int s = 0; s < 4; ++s) {
            if (name != kNames[s]) continue;
            named[s] = true;
            if (slot_field[s] < 0 && dt == kFloat32 && count <= 1) { slot_field[s] = (int)j; cl.off[s] = off; cl.fields |= 1u << s; }
        }
    }
    uint8_t be, dense;
    uint32_t dlen;
    if (!c.u8(be) || !c.u32(cl.point_step) || !c.u32(cl.row_step) || !c.u32(dlen)) return bad("the message ends inside lidar");
    cl.big_endian = be ? 1u : 0u;
    cl.data_off = c.pos;
    cl.data_len = dlen;
    if (!c.take(dlen)) return bad("lidar.data runs past the message");
    if (!c.u8(dense)) return bad("the message ends inside lidar");
    for (int i = 0; i < 7; ++i) { double d; if (!c.f64(d)) return bad("the message ends inside lidarOdom"); }
    if (!skip_header(c, nullptr) || !c.skip_str() || !c.skip_str()) return bad("the message ends inside image");
    uint8_t st, ct;                  // gps: status (int8 status + uint16 service), latitude .. covariance, covariance type
    if (!skip_header(c, nullptr) || !c.u8(st) || !c.take(2) || !c.take(3 * 8 + 9 * 8) || !c.u8(ct)) return bad("the message ends inside gps");
    if (c.pos != c.end) return e.set(ERASOR_E_INVALID, who + ": the message is " + std::to_string(c.end - c.pos) + " bytes longer than an erasor/node");
    for (int s = 0; s < 3; ++s)
        if (!(cl.fields >> s & 1u))
            return e.set(ERASOR_E_UNSUPPORTED, who + ": lidar has no field '" + kNames[s] + (named[s] ? "' of datatype FLOAT32 and count 1" : "'"));
    if (!(cl.fields & 8u)) ++zero_filled;
    const uint64_t n = cloud_points(cl);
    if (n >= kMaxCloudPoints) return e.set(ERASOR_E_CAPACITY, who + ": a cloud of 2^31 points or more");
    if (n) {
        uint64_t hi = 0;             // in 64 bits: once this check passes, point_reach's 32-bit sum cannot wrap (data_len < 2^32)
        for (int s = 0; s < 4; ++s)
            if (cl.fields >> s & 1u) hi = std::max<uint64_t>(hi, (uint64_t)cl.off[s] + 4u);
        const uint64_t last = (uint64_t)(cl.height - 1) * cl.row_step + (uint64_t)(cl.width - 1) * cl.point_step;
        if (last + hi > cl.data_len)
            return e.set(ERASOR_E_INVALID, who + ": its last point reads up to byte " + std::to_string(last + hi) + " of lidar.data, which holds " +
                                               std::to_string(cl.data_len));
    }
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
    if (!w.records(13, len, false)) { msg = w.e.msg; return w.e.rc; }
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
        if (!detail::parse_node(file, sel[k], k - first, nd, e, out.intensity_zero_filled)) { msg = e.msg; const int rc = e.rc; out.nodes.clear(); return rc; }
        out.total_points += cloud_points(nd.cloud);
        out.big_endian += nd.cloud.big_endian;
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
