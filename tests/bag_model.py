"""Test-side model of ROS bag 2.0 files of erasor/node messages, written from the public format description (no ROS here): a numpy
writer that lays a bag out as the reference's kitti2node does, and an independent numpy reader of what erasor_bag_index /
erasor_bag_load must give.  It shares no code with the committed fixture's generator (tests/golden/make_bag_golden.py), so one
misreading of the format cannot pass both.

The writer (write_bag) takes (topic, (sec, nsec), payload) messages in write order and produces:
  - "#ROSBAG V2.0\\n", then a bag header record padded to 4096 bytes (index_pos, conn_count, chunk_count);
  - uncompressed chunks closed once their data passes chunk_bytes, so frames split across chunk boundaries; in each chunk a
    connection record precedes the first message of that connection, and the chunk is followed by one index-data record per
    connection it holds (time, offset of the message record in the chunk's data);
  - at index_pos, every connection record, then one chunk-info record per chunk.
kitti2node_messages gives a frame's four messages (/tf, /node/combined/optimized, /debug/pc_raw, /debug/pc_label) per node, the
first frame written twice.  The connection headers carry a placeholder message_definition: nothing reads it.
"""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")
TOPIC = "/node/combined/optimized"
NODE_MD5 = "0123456789abcdef0123456789abcdef"
FLOAT32, FLOAT64, UINT16, UINT8 = 7, 8, 4, 2
TYPES = {TOPIC: "erasor/node", "/tf": "tf2_msgs/TFMessage", "/debug/pc_raw": "sensor_msgs/PointCloud2",
         "/debug/pc_label": "sensor_msgs/PointCloud2"}
NP_OF = {FLOAT32: "<f4", FLOAT64: "<f8", UINT16: "<u2", UINT8: "u1"}


def u8(v): return np.array([v], dtype="u1").tobytes()
def u16(v): return np.array([v], dtype="<u2").tobytes()
def u32(v): return np.array([v], dtype="<u4").tobytes()
def u64(v): return np.array([v], dtype="<u8").tobytes()
def f64s(vals): return np.asarray(vals, dtype="<f8").tobytes()
def string(s): b = s.encode() if isinstance(s, str) else bytes(s); return u32(len(b)) + b
def header(seq, stamp, frame_id): return u32(seq) + u32(stamp[0]) + u32(stamp[1]) + string(frame_id)


# ---- PointCloud2 layouts -------------------------------------------------------------------------------------------------------
# fields: (name, offset, datatype, count); a field takes the column of its name (x y z intensity), "_" is padding
LAYOUTS = {
    "pcl_xyzi": dict(fields=[("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 16, FLOAT32, 1)], point_step=32),
    "packed": dict(fields=[("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 12, FLOAT32, 1)], point_step=16),
    "odd_step": dict(fields=[("intensity", 0, FLOAT32, 1), ("z", 5, FLOAT32, 1), ("y", 9, FLOAT32, 1), ("x", 13, FLOAT32, 1)], point_step=22),
    "i_uint16": dict(fields=[("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 12, UINT16, 1)], point_step=14),
    "i_float64": dict(fields=[("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 16, FLOAT64, 1)], point_step=24),
    "no_intensity": dict(fields=[("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1)], point_step=12),
    # the first x is FLOAT64 and does not match; the second x and the first intensity win
    "duplicates": dict(fields=[("x", 0, FLOAT64, 1), ("y", 8, FLOAT32, 1), ("x", 12, FLOAT32, 1), ("z", 16, FLOAT32, 1),
                               ("intensity", 20, FLOAT32, 1), ("intensity", 24, FLOAT32, 1)], point_step=28),
    "count0": dict(fields=[("x", 0, FLOAT32, 0), ("y", 4, FLOAT32, 0), ("z", 8, FLOAT32, 0), ("intensity", 12, FLOAT32, 0)], point_step=16),
    "x_float64": dict(fields=[("x", 0, FLOAT64, 1), ("y", 8, FLOAT32, 1), ("z", 12, FLOAT32, 1)], point_step=16),
}


def pack_cloud(xyzi, layout, height=1, row_pad=0, seed=0):
    """(data bytes, PointCloud2 dict) of an [n, 4] float32 cloud in a layout; height > 1 makes an organised cloud of rows of
    n / height points, each row followed by row_pad bytes.  Bytes no field covers are random."""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    n = len(xyzi)
    width = n // height if height else 0
    assert width * height == n
    ps = layout["point_step"]
    row_step = width * ps + row_pad
    rng = np.random.default_rng(seed)
    buf = np.frombuffer(rng.bytes(row_step * height), dtype=np.uint8).copy()
    col = {"x": 0, "y": 1, "z": 2, "intensity": 3}
    r, c = np.divmod(np.arange(n), max(width, 1))
    base = r * row_step + c * ps
    for name, off, dt, _ in layout["fields"]:
        if name not in col or not n:
            continue
        vals = xyzi[:, col[name]]
        raw = np.ascontiguousarray(vals.astype(NP_OF[dt]) if dt != FLOAT32 else vals).view(np.uint8).reshape(n, -1)
        for k in range(raw.shape[1]):
            buf[base + off + k] = raw[:, k]
    return buf.tobytes(), dict(height=height, width=width, fields=layout["fields"], point_step=ps, row_step=row_step, is_bigendian=0)


def pointcloud2(pc, data, seq=0, stamp=(0, 0), frame_id="velodyne", is_dense=1):
    b = header(seq, stamp, frame_id) + u32(pc["height"]) + u32(pc["width"]) + u32(len(pc["fields"]))
    for name, off, dt, cnt in pc["fields"]:
        b += string(name) + u32(off) + u8(dt) + u32(cnt)
    return b + u8(pc["is_bigendian"]) + u32(pc["point_step"]) + u32(pc["row_step"]) + string(data) + u8(is_dense)


def node_payload(seq, stamp, odom, pc, data, frame_id="map", lidar_frame="velodyne", extra=b""):
    """one serialised erasor/node; extra is appended (a message longer than its structure)"""
    b = header(seq, stamp, frame_id) + f64s(odom) + f64s(np.arange(36) * 0.5)
    b += pointcloud2(pc, data, seq, stamp, lidar_frame)
    b += f64s([1, 2, 3, 0, 0, 0, 1])                                      # lidarOdom
    b += header(seq, stamp, "cam") + string("jpeg") + string(b"\xff\xd8\x00")   # image
    b += header(seq, stamp, "gps") + u8(0) + u16(1) + f64s([37.5, 127.0, 30.0]) + f64s(np.zeros(9)) + u8(0)   # gps
    return b + extra


def kitti2node_messages(nodes, debug=True, layout="pcl_xyzi", frame_ids=None):
    """nodes: (seq, odom7, cloud) -> the messages kitti2node writes, per frame /tf, the node, /debug/pc_raw, /debug/pc_label; the
    first frame twice.  Frame k (0 = the duplicate) has time (1000 + k // 10, (k % 10) 10^8)."""
    frames = [nodes[0]] + list(nodes)
    out = []
    for k, (seq, odom, cloud) in enumerate(frames):
        t = (1000 + k // 10, (k % 10) * 100000000)
        fid = frame_ids[k % len(frame_ids)] if frame_ids else "velodyne"
        data, pc = pack_cloud(cloud, LAYOUTS[layout], seed=k)
        out.append(("/tf", t, u32(1) + header(seq, t, "map") + string("body") + f64s([0, 0, 0, 0, 0, 0, 1])))
        out.append((TOPIC, t, node_payload(seq, t, odom, pc, data, lidar_frame=fid)))
        if debug:
            out.append(("/debug/pc_raw", t, pointcloud2(pc, data, seq, t)))
            out.append(("/debug/pc_label", t, pointcloud2(pc, data, seq, t)))
    return out


# ---- records -------------------------------------------------------------------------------------------------------------------
def record(fields, data):
    h = b"".join(u32(len(name) + 1 + len(v)) + name.encode() + b"=" + v for name, v in fields)
    return u32(len(h)) + h + u32(len(data)) + data


def conn_record(cid, topic, types):
    ch = [("topic", topic.encode()), ("type", types[topic].encode()), ("md5sum", NODE_MD5.encode()),
          ("message_definition", b"# placeholder\n"), ("callerid", b"/kitti2node")]
    return record([("op", u8(7)), ("conn", u32(cid)), ("topic", topic.encode())], b"".join(u32(len(k) + 1 + len(v)) + k.encode() + b"=" + v for k, v in ch))


def time_bytes(t): return u32(t[0]) + u32(t[1])


def write_bag(messages, chunk_bytes=1 << 20, compression="none", types=None, version=b"2.0"):
    """messages: (topic, (sec, nsec), payload) in write order -> the bag's bytes"""
    types = dict(TYPES, **(types or {}))
    conn_of = {}
    for topic, _, _ in messages:
        conn_of.setdefault(topic, len(conn_of))
    out = [b"#ROSBAG V" + version + b"\n", b""]          # [1]: the bag header, written last
    pos = 4096 + len(out[0])
    chunk_infos = []
    i = 0
    while i < len(messages):
        body, seen, idx = [], set(), {}
        size = 0
        t_lo, t_hi = None, None
        while i < len(messages) and size <= chunk_bytes:
            topic, t, payload = messages[i]
            cid = conn_of[topic]
            if cid not in seen:
                seen.add(cid)
                r = conn_record(cid, topic, types)
                body.append(r)
                size += len(r)
            idx.setdefault(cid, []).append((t, size))
            r = record([("op", u8(2)), ("conn", u32(cid)), ("time", time_bytes(t))], payload)
            body.append(r)
            size += len(r)
            t_lo = t if t_lo is None or t < t_lo else t_lo
            t_hi = t if t_hi is None or t > t_hi else t_hi
            i += 1
        data = b"".join(body)
        rec = record([("op", u8(5)), ("compression", compression.encode()), ("size", u32(len(data)))], data)
        chunk_infos.append((pos, t_lo, t_hi, {c: len(v) for c, v in idx.items()}))
        out.append(rec)
        pos += len(rec)
        for cid in sorted(idx):
            r = record([("op", u8(4)), ("ver", u32(1)), ("conn", u32(cid)), ("count", u32(len(idx[cid])))],
                       b"".join(time_bytes(t) + u32(off) for t, off in idx[cid]))
            out.append(r)
            pos += len(r)
    index_pos = pos
    for topic, cid in conn_of.items():
        out.append(conn_record(cid, topic, types))
    for cpos, lo, hi, counts in chunk_infos:
        out.append(record([("op", u8(6)), ("ver", u32(1)), ("chunk_pos", u64(cpos)), ("start_time", time_bytes(lo)), ("end_time", time_bytes(hi)),
                           ("count", u32(len(counts)))], b"".join(u32(c) + u32(k) for c, k in sorted(counts.items()))))
    h = [("op", u8(3)), ("index_pos", u64(index_pos)), ("conn_count", u32(len(conn_of))), ("chunk_count", u32(len(chunk_infos)))]
    hb = record(h, b"")
    out[1] = record(h, b" " * (4096 - len(hb)))
    assert len(out[1]) == 4096
    return b"".join(out)


# ---- the reader ----------------------------------------------------------------------------------------------------------------
class BagError(ValueError):
    pass


def _fields(buf, a, b):
    out = {}
    while a < b:
        n = int(np.frombuffer(buf, "<u4", 1, a)[0])
        s = bytes(buf[a + 4:a + 4 + n])
        k = s.index(b"=")
        out[s[:k].decode()] = (a + 4 + k + 1, s[k + 1:])
        a += 4 + n
    return out


def _walk(buf, a, b, conns, msgs):
    while a < b:
        hl = int(np.frombuffer(buf, "<u4", 1, a)[0])
        h = _fields(buf, a + 4, a + 4 + hl)
        d0 = a + 4 + hl + 4
        dl = int(np.frombuffer(buf, "<u4", 1, a + 4 + hl)[0])
        op = h["op"][1][0]
        if op == 5:
            if h["compression"][1] != b"none":
                raise BagError("compressed chunk")
            _walk(buf, d0, d0 + dl, conns, msgs)
        elif op == 7:
            ch = _fields(buf, d0, d0 + dl)
            conns[int(np.frombuffer(h["conn"][1], "<u4")[0])] = (h["topic"][1].decode(), ch["type"][1].decode(), ch["md5sum"][1].decode())
        elif op == 2:
            sec, nsec = np.frombuffer(h["time"][1], "<u4")
            msgs.append((int(np.frombuffer(h["conn"][1], "<u4")[0]), int(sec) * 10**9 + int(nsec), d0, dl))
        a = d0 + dl


class _R:
    def __init__(self, buf, a):
        self.buf, self.a = buf, a

    def get(self, dt, n=1):
        v = np.frombuffer(self.buf, dt, n, self.a)
        self.a += v.nbytes
        return v

    def u32(self): return int(self.get("<u4")[0])
    def skip(self, n): self.a += n
    def string(self): n = self.u32(); s = bytes(self.buf[self.a:self.a + n]); self.a += n; return s
    def header(self): seq = self.u32(); self.skip(8); self.string(); return seq


def read_bag(data, topic=TOPIC, keep_first=False, decode=True):
    """-> list of dicts per node: seq, stamp_ns, odom (float64[7]), layout (erasor_bag_cloud_t's fields), cloud (float32 [n, 4],
    the device's output bit for bit) -- in delivery order, the first dropped unless keep_first"""
    buf = memoryview(data)
    if bytes(buf[:13]) != b"#ROSBAG V2.0\n":
        raise BagError("version")
    conns, msgs = {}, []
    _walk(buf, 13, len(buf), conns, msgs)
    sel = [m for m in msgs if conns[m[0]][0] == topic]
    sel.sort(key=lambda m: m[1])                      # Python's sort is stable
    out = []
    for conn, t, d0, dl in (sel if keep_first else sel[1:]):
        r = _R(buf, d0)
        seq = r.header()
        odom = r.get("<f8", 7).copy()
        r.skip(36 * 8)
        r.header()
        height, width, nf = r.u32(), r.u32(), r.u32()
        flds = []
        for _ in range(nf):
            name = r.string().decode()
            off = r.u32()
            dt = int(r.get("u1")[0])
            flds.append((name, off, dt, r.u32()))
        be = int(r.get("u1")[0])
        ps, rs, dlen = r.u32(), r.u32(), r.u32()
        doff = r.a
        r.skip(dlen + 1)
        r.skip(7 * 8)
        r.header(); r.string(); r.string()
        r.header(); r.skip(1 + 2 + 3 * 8 + 9 * 8 + 1)
        if r.a != d0 + dl:
            raise BagError("length")
        fields, offs = 0, [0, 0, 0, 0]
        for s, nm in enumerate(("x", "y", "z", "intensity")):
            for name, off, dt, cnt in flds:
                if name == nm and dt == FLOAT32 and cnt <= 1:
                    fields |= 1 << s
                    offs[s] = off
                    break
        lay = dict(data_offset=doff, data_len=dlen, width=width, height=height, point_step=ps, row_step=rs, fields=fields, big_endian=be,
                   offset=offs)
        nd = dict(seq=seq, stamp_ns=t, odom=odom, layout=lay)
        if decode:
            n = width * height
            bits = np.zeros((n, 4), dtype=np.uint32)
            rr, cc = np.divmod(np.arange(n, dtype=np.int64), max(width, 1))
            base = doff + rr * rs + cc * ps
            raw = np.frombuffer(buf, dtype=np.uint8)
            for s in range(4):
                if fields >> s & 1:
                    i = base + offs[s]
                    bits[:, s] = raw[i] | raw[i + 1].astype(np.uint32) << 8 | raw[i + 2].astype(np.uint32) << 16 | raw[i + 3].astype(np.uint32) << 24
            nd["cloud"] = bits.view(np.float32)
        out.append(nd)
    return out


# ---- the host build (liberasor_b200_hostcheck.so) -------------------------------------------------------------------------------
class BagInfo(ctypes.Structure):
    """erasor_bag_info_t"""
    _fields_ = [("version", ctypes.c_uint32), ("pad_", ctypes.c_uint32)] + \
               [(k, ctypes.c_uint64) for k in ("chunks", "connections", "messages", "selected", "unknown_records", "nodes", "total_points",
                                                "intensity_zero_filled", "big_endian")] + [("md5sum", ctypes.c_char * 40)]


class BagCloud(ctypes.Structure):
    """erasor_bag_cloud_t"""
    _fields_ = [("data_offset", ctypes.c_uint64), ("data_len", ctypes.c_uint64)] + \
               [(k, ctypes.c_uint32) for k in ("width", "height", "point_step", "row_step", "fields", "big_endian")] + [("offset", ctypes.c_uint32 * 4)]


def info_dict(info):
    d = {k: int(getattr(info, k)) for k, _ in BagInfo._fields_ if k not in ("md5sum", "pad_")}
    d["md5sum"] = info.md5sum.decode()
    return d


def cloud_dict(c):
    d = {k: int(getattr(c, k)) for k, _ in BagCloud._fields_ if k != "offset"}
    d["offset"] = [int(v) for v in c.offset]
    return d


_HC = None


def hostcheck():
    global _HC
    if _HC is None:
        L = ctypes.CDLL(HOSTCHECK)
        vp, sz = ctypes.c_void_p, ctypes.c_size_t
        L.erasor_hostcheck_bag_index.argtypes = [vp, sz, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(sz), ctypes.POINTER(BagInfo), ctypes.c_char_p, sz]
        L.erasor_hostcheck_bag_nodes.argtypes = [sz, sz, vp, vp, vp, vp]
        L.erasor_hostcheck_bag_decode.argtypes = [vp, sz, sz, vp, vp, ctypes.c_char_p, sz]
        _HC = L
    return _HC


def hc_read(data, topic=TOPIC, keep_first=False):
    """(rc, message, info dict, nodes as read_bag gives them) of the host build of erasor_bag_index + erasor_bag_nodes + the decode"""
    L = hostcheck()
    a = np.frombuffer(data, dtype=np.uint8) if len(data) else np.zeros(1, np.uint8)
    n, info, err = ctypes.c_size_t(0), BagInfo(), ctypes.create_string_buffer(1024)
    rc = L.erasor_hostcheck_bag_index(a.ctypes.data, len(data), topic.encode(), int(keep_first), ctypes.byref(n), ctypes.byref(info), err, 1024)
    if rc != 0:
        return rc, err.value.decode(), None, None
    k = n.value
    seq, stamp, odom, clouds = np.zeros(k, np.uint32), np.zeros(k, np.uint64), np.zeros((k, 7)), (BagCloud * max(k, 1))()
    assert L.erasor_hostcheck_bag_nodes(0, k, seq.ctypes.data, stamp.ctypes.data, odom.ctypes.data, ctypes.addressof(clouds)) == 0
    off = np.zeros(k + 1, np.uint64)
    out = np.zeros((max(info.total_points, 1), 4), np.float32)
    rc = L.erasor_hostcheck_bag_decode(a.ctypes.data, 0, k, out.ctypes.data, off.ctypes.data, err, 1024)
    if rc != 0:
        return rc, err.value.decode(), info_dict(info), None
    nodes = [dict(seq=int(seq[i]), stamp_ns=int(stamp[i]), odom=odom[i], layout=cloud_dict(clouds[i]), cloud=out[int(off[i]):int(off[i + 1])])
             for i in range(k)]
    return 0, "", info_dict(info), nodes
