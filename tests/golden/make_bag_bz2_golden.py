"""Writes tests/golden/node_tiny_bz2.bag: a ROS bag 2.0 file of three erasor/node messages and one interleaved /tf message in two
bz2 chunks, assembled field by field with struct.pack and compressed with the standard library's bz2, independently of
tests/bag_model.py and tests/bz2_model.py, so that one misreading of the bag or bzip2 format cannot pass both the fixture and the
model.

  chunk 1 (level 1): node 0 (50 points), a /tf message, node 1 (20 000 points of a 7-byte pattern: 320 000 bytes without a run of
           four, so the stream holds four blocks of at most 100 000 RLE1 bytes, each a few hundred bytes compressed)
  chunk 2 (level 9): node 2 (200 random points)
Each chunk is followed by its index data records; then the connections, the chunk infos and the bag header's index_pos.  Run with
python3 to rewrite the file.
"""
import bz2
import os
import struct

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "node_tiny_bz2.bag")
NODE, TF = "/node/combined/optimized", "/tf"


def nodes():
    """(seq, odom7, cloud float32 [n][4]) of the three nodes"""
    rng = np.random.default_rng(2026)
    pattern = np.frombuffer((b"\x11\x22\x33\x44\x55\x66\x77" * 45715)[:320000], np.float32).reshape(-1, 4)
    return [(100, np.array([1.0, 2.0, 0.5, 0, 0, 0, 1.0]), rng.normal(size=(50, 4)).astype(np.float32)),
            (101, np.array([1.5, 2.5, 0.5, 0, 0, 0.6, 0.8]), pattern.copy()),
            (102, np.array([2.0, 3.0, 0.5, 0, 0, 1.0, 0]), rng.normal(size=(200, 4)).astype(np.float32))]


def string(b):
    return struct.pack("<I", len(b)) + b


def header(seq, sec, frame):
    return struct.pack("<III", seq, sec, 0) + string(frame)


def node_msg(seq, odom, cloud, sec):
    out = header(seq, sec, b"map") + struct.pack("<7d", *odom) + struct.pack("<36d", *([0.0] * 36))
    out += header(seq, sec, b"velodyne") + struct.pack("<II", 1, len(cloud)) + struct.pack("<I", 4)
    for k, name in enumerate((b"x", b"y", b"z", b"intensity")):
        out += string(name) + struct.pack("<IBI", 4 * k, 7, 1)
    data = cloud.astype("<f4").tobytes()
    out += struct.pack("<BII", 0, 16, len(data)) + string(data) + struct.pack("<B", 1)
    out += struct.pack("<7d", *odom)                                 # lidarOdom
    out += header(seq, sec, b"camera") + string(b"jpeg") + string(b"")
    out += header(seq, sec, b"gps") + struct.pack("<bH", 0, 1) + struct.pack("<12d", *([0.0] * 12)) + struct.pack("<B", 0)
    return out


def field(name, value):
    return struct.pack("<I", len(name) + 1 + len(value)) + name + b"=" + value


def record(fields, data):
    h = b"".join(field(n, v) for n, v in fields)
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def conn_record(cid, topic, typ):
    data = field(b"topic", topic.encode()) + field(b"type", typ) + field(b"md5sum", b"0" * 32) + field(b"message_definition", b"")
    return record([(b"op", b"\x07"), (b"conn", struct.pack("<I", cid)), (b"topic", topic.encode())], data)


def build():
    ns = nodes()
    conns = [(0, TF, b"tf2_msgs/TFMessage"), (1, NODE, b"erasor/node")]
    # (chunk level, [(conn, sec, payload)])
    chunks = [(1, [(1, 10, node_msg(*ns[0], 10)), (0, 11, b"\x01\x02\x03\x04"), (1, 12, node_msg(*ns[1], 12))]),
              (9, [(1, 13, node_msg(*ns[2], 13))])]
    body, infos, pos = b"", [], 13 + 4096 + 8 + 0
    head_len = len(record([(b"op", b"\x03"), (b"index_pos", bytes(8)), (b"conn_count", bytes(4)), (b"chunk_count", bytes(4))], b""))
    pos = 13 + head_len + 4096 - head_len                            # the bag header record is padded to 4096 bytes
    for level, msgs in chunks:
        inner, offsets = b"", []
        for cid, topic, typ in conns:
            inner += conn_record(cid, topic, typ)
        for cid, sec, payload in msgs:
            offsets.append((cid, sec, len(inner)))
            inner += record([(b"op", b"\x02"), (b"conn", struct.pack("<I", cid)), (b"time", struct.pack("<II", sec, 0))], payload)
        chunk = record([(b"op", b"\x05"), (b"compression", b"bz2"), (b"size", struct.pack("<I", len(inner)))], bz2.compress(inner, level))
        index = b""
        for cid, _, _ in conns:
            entries = [struct.pack("<III", sec, 0, off) for c, sec, off in offsets if c == cid]
            if entries:
                index += record([(b"op", b"\x04"), (b"ver", struct.pack("<I", 1)), (b"conn", struct.pack("<I", cid)),
                                 (b"count", struct.pack("<I", len(entries)))], b"".join(entries))
        counts = [(cid, sum(1 for c, _, _ in offsets if c == cid)) for cid, _, _ in conns]
        infos.append((pos, min(s for _, s, _ in offsets), max(s for _, s, _ in offsets), [c for c in counts if c[1]]))
        body += chunk + index
        pos += len(chunk) + len(index)
    index_pos = pos
    tail = b"".join(conn_record(cid, topic, typ) for cid, topic, typ in conns)
    for cpos, t0, t1, counts in infos:
        tail += record([(b"op", b"\x06"), (b"ver", struct.pack("<I", 1)), (b"chunk_pos", struct.pack("<Q", cpos)),
                        (b"start_time", struct.pack("<II", t0, 0)), (b"end_time", struct.pack("<II", t1, 0)),
                        (b"count", struct.pack("<I", len(counts)))], b"".join(struct.pack("<II", c, n) for c, n in counts))
    hfields = [(b"op", b"\x03"), (b"index_pos", struct.pack("<Q", index_pos)), (b"conn_count", struct.pack("<I", len(conns))),
               (b"chunk_count", struct.pack("<I", len(chunks)))]
    bag_header = record(hfields, b" " * (4096 - head_len))
    return b"#ROSBAG V2.0\n" + bag_header + body + tail


if __name__ == "__main__":
    with open(PATH, "wb") as f:
        f.write(build())
    print(PATH)
