"""Writes tests/golden/node_tiny.bag: a ROS bag 2.0 file assembled field by field with explicit struct.pack calls, independently of
tests/bag_model.py, so that one misreading of the format cannot pass both the fixture and the model.

Layout (times as sec.nsec):
  "#ROSBAG V2.0\\n", bag header record padded to 4096 bytes
  chunk 1: conn 0 (/tf), /tf @10.0, conn 1 (/node/combined/optimized), node @10.0 (seq 7: the first frame, written twice),
           /tf @10.5, node @10.5 (seq 7 again)
  index data for conn 0 and conn 1
  chunk 2: conn 0, /tf @11.0, conn 1, node @11.0 (seq 9)
  index data for conn 0 and conn 1
  index section: conn 0, conn 1, chunk info x 2
The seq-7 node's cloud is pcl::toROSMsg's PointXYZI layout (x@0 y@4 z@8 intensity@16, point_step 32, one row of 3); the seq-9
node's cloud is organised, 2 rows of 2 points, point_step 16, row_step 40 (8 bytes of padding after each row).  Run with python3 to
rewrite the file; EXPECTED holds what a reader must give after dropping the first node.
"""
import os
import struct

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "node_tiny.bag")
MD5 = b"4dd8a3d1d6b0b1d4c26d0c4fc1e3bd55"

ODOM7 = (1.5, -2.25, 0.125, 0.0, 0.0, 0.38268343236508978, 0.92387953251128674)
ODOM9 = (3.0, 4.0, -0.5, 0.0, 0.0, -0.70710678118654757, 0.70710678118654757)
PTS7 = ((1.0, 2.0, 3.0, 40.0), (-1.5, 0.25, 7.75, 252.0), (100.0, -200.0, 0.5, 65536.0))
PTS9 = ((0.5, 0.5, 0.5, 1.0), (1.5, 1.5, 1.5, 2.0), (2.5, 2.5, 2.5, 3.0), (3.5, 3.5, 3.5, 4.0))
EXPECTED = [(7, ODOM7, PTS7), (9, ODOM9, PTS9)]


def field(name, value):
    body = name + b"=" + value
    return struct.pack("<I", len(body)) + body


def record(header_fields, data):
    h = b"".join(header_fields)
    return struct.pack("<I", len(h)) + h + struct.pack("<I", len(data)) + data


def connection(conn, topic, msg_type):
    ch = (field(b"topic", topic) + field(b"type", msg_type) + field(b"md5sum", MD5 if msg_type == b"erasor/node" else b"*")
          + field(b"message_definition", b"(placeholder)") + field(b"callerid", b"/golden"))
    return record([field(b"op", b"\x07"), field(b"conn", struct.pack("<I", conn)), field(b"topic", topic)], ch)


def message(conn, sec, nsec, payload):
    return record([field(b"op", b"\x02"), field(b"conn", struct.pack("<I", conn)), field(b"time", struct.pack("<II", sec, nsec))], payload)


def ros_header(seq, sec, nsec, frame_id):
    return struct.pack("<III", seq, sec, nsec) + struct.pack("<I", len(frame_id)) + frame_id


def tf_payload(seq, sec, nsec):
    return struct.pack("<I", 1) + ros_header(seq, sec, nsec, b"map") + struct.pack("<I", 4) + b"body" + struct.pack("<7d", 0, 0, 0, 0, 0, 0, 1)


def cloud_pcl(points):
    """x y z at 0 4 8, intensity at 16, point_step 32; bytes 12..15 and 20..31 of a point are 0xAB filler"""
    data = b""
    for x, y, z, i in points:
        data += struct.pack("<fff", x, y, z) + b"\xab" * 4 + struct.pack("<f", i) + b"\xab" * 12
    fields = [(b"x", 0), (b"y", 4), (b"z", 8), (b"intensity", 16)]
    return 1, len(points), fields, 32, 32 * len(points), data


def cloud_organised(points):
    """2 x 2 points, x y z intensity at 0 4 8 12, point_step 16, row_step 40"""
    data = b""
    for r in range(2):
        for c in range(2):
            data += struct.pack("<4f", *points[2 * r + c])
        data += b"\xcd" * 8
    fields = [(b"x", 0), (b"y", 4), (b"z", 8), (b"intensity", 12)]
    return 2, 2, fields, 16, 40, data


def node_payload(seq, sec, nsec, odom, cloud):
    height, width, fields, point_step, row_step, data = cloud
    b = ros_header(seq, sec, nsec, b"map")
    b += struct.pack("<7d", *odom)                                     # odom
    b += struct.pack("<36d", *[0.01 * k for k in range(36)])           # odomCov
    b += ros_header(seq, sec, nsec, b"velodyne")                       # lidar
    b += struct.pack("<II", height, width) + struct.pack("<I", len(fields))
    for name, off in fields:
        b += struct.pack("<I", len(name)) + name + struct.pack("<IBI", off, 7, 1)
    b += struct.pack("<B", 0) + struct.pack("<II", point_step, row_step) + struct.pack("<I", len(data)) + data + struct.pack("<B", 1)
    b += struct.pack("<7d", 0, 0, 0, 0, 0, 0, 1)                        # lidarOdom
    b += ros_header(seq, sec, nsec, b"camera") + struct.pack("<I", 4) + b"jpeg" + struct.pack("<I", 2) + b"\xff\xd8"   # image
    b += ros_header(seq, sec, nsec, b"gps") + struct.pack("<bH", 0, 1) + struct.pack("<3d", 37.0, 127.0, 50.0) + struct.pack("<9d", *([0.0] * 9))
    b += struct.pack("<B", 0)                                           # position_covariance_type
    return b


def index_data(conn, entries):
    data = b"".join(struct.pack("<III", sec, nsec, off) for sec, nsec, off in entries)
    return record([field(b"op", b"\x04"), field(b"ver", struct.pack("<I", 1)), field(b"conn", struct.pack("<I", conn)),
                   field(b"count", struct.pack("<I", len(entries)))], data)


def chunk(parts):
    """(chunk record, [(conn, sec, nsec, offset of the message record in the chunk data)])"""
    data, idx = b"", []
    for kind, conn, sec, nsec, payload in parts:
        if kind == "conn":
            data += payload
        else:
            idx.append((conn, sec, nsec, len(data)))
            data += message(conn, sec, nsec, payload)
    rec = record([field(b"op", b"\x05"), field(b"compression", b"none"), field(b"size", struct.pack("<I", len(data)))], data)
    return rec, idx


def build():
    tf, node = b"/tf", b"/node/combined/optimized"
    c_tf, c_node = connection(0, tf, b"tf2_msgs/TFMessage"), connection(1, node, b"erasor/node")
    ch1, i1 = chunk([("conn", 0, 0, 0, c_tf), ("msg", 0, 10, 0, tf_payload(7, 10, 0)),
                     ("conn", 1, 0, 0, c_node), ("msg", 1, 10, 0, node_payload(7, 10, 0, ODOM7, cloud_pcl(PTS7))),
                     ("msg", 0, 10, 500000000, tf_payload(7, 10, 500000000)),
                     ("msg", 1, 10, 500000000, node_payload(7, 10, 500000000, ODOM7, cloud_pcl(PTS7)))])
    ch2, i2 = chunk([("conn", 0, 0, 0, c_tf), ("msg", 0, 11, 0, tf_payload(9, 11, 0)),
                     ("conn", 1, 0, 0, c_node), ("msg", 1, 11, 0, node_payload(9, 11, 0, ODOM9, cloud_organised(PTS9)))])
    magic = b"#ROSBAG V2.0\n"
    pos1 = len(magic) + 4096
    body = ch1 + b"".join(index_data(c, [(s, n, o) for cc, s, n, o in i1 if cc == c]) for c in (0, 1))
    pos2 = pos1 + len(body)
    body += ch2 + b"".join(index_data(c, [(s, n, o) for cc, s, n, o in i2 if cc == c]) for c in (0, 1))
    index_pos = pos1 + len(body)
    infos = b""
    for pos, lo, hi in ((pos1, (10, 0), (10, 500000000)), (pos2, (11, 0), (11, 0))):
        infos += record([field(b"op", b"\x06"), field(b"ver", struct.pack("<I", 1)), field(b"chunk_pos", struct.pack("<Q", pos)),
                         field(b"start_time", struct.pack("<II", *lo)), field(b"end_time", struct.pack("<II", *hi)),
                         field(b"count", struct.pack("<I", 2))], struct.pack("<IIII", 0, 2, 1, 2) if pos == pos1 else struct.pack("<IIII", 0, 1, 1, 1))
    hfields = [field(b"op", b"\x03"), field(b"index_pos", struct.pack("<Q", index_pos)), field(b"conn_count", struct.pack("<I", 2)),
               field(b"chunk_count", struct.pack("<I", 2))]
    hlen = sum(len(f) for f in hfields)
    bag_header = record(hfields, b" " * (4096 - 8 - hlen))
    assert len(bag_header) == 4096
    return magic + bag_header + body + c_tf + c_node + infos


if __name__ == "__main__":
    with open(PATH, "wb") as f:
        f.write(build())
    print(PATH)
