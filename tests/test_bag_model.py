"""CPU: the erasor/node bag reader (erasor_b200/csrc/bag_index.h, compiled for the host into liberasor_b200_hostcheck.so, its decode
run serially) against the numpy model of tests/bag_model.py and the struct-built fixture tests/golden/node_tiny.bag: node lists,
seqs, record times, odom bit patterns, blob offsets, resolved layouts and decoded clouds, then every fence."""
import os
import struct
import sys

import numpy as np
import pytest

import bag_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_bag_golden as G  # noqa: E402

OK, E_INVALID, E_CAPACITY, E_UNSUPPORTED = 0, -1, -4, -5

pytestmark = pytest.mark.skipif(not os.path.exists(M.HOSTCHECK), reason="build with erasor_b200/csrc/build.sh")


def nodes_of(n_nodes, n_pts=50, seed=0, empty=(), nan=False):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_nodes):
        m = 0 if k in empty else n_pts + k
        c = rng.normal(size=(m, 4)).astype(np.float32) * 20
        c[:, 3] = rng.integers(0, 1 << 20, m).astype(np.float32)
        if nan and m:
            bits = c.view(np.uint32)
            bits[::3, 0] = 0x7FC00001 + np.arange(len(bits[::3]), dtype=np.uint32)      # quiet NaNs with payloads
            bits[1::5, 2] = 0xFF800123                                                   # negative NaN, payload 0x123
        pose = np.concatenate([rng.normal(size=3) * 100, rng.normal(size=4)])
        out.append((100 + 2 * k, pose / np.r_[1, 1, 1, [np.linalg.norm(pose[3:])] * 4], c))
    return out


def same_nodes(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g["seq"] == w["seq"] and g["stamp_ns"] == w["stamp_ns"]
        assert np.array_equal(np.asarray(g["odom"]).view(np.uint64), np.asarray(w["odom"]).view(np.uint64))
        assert g["layout"] == w["layout"]
        assert g["cloud"].shape == w["cloud"].shape and np.array_equal(g["cloud"].view(np.uint32), w["cloud"].view(np.uint32))


def check(data, keep_first=False, topic=M.TOPIC):
    rc, msg, info, got = M.hc_read(data, topic, keep_first)
    assert rc == OK, msg
    want = M.read_bag(data, topic, keep_first)
    same_nodes(got, want)
    assert info["nodes"] == len(want) and info["total_points"] == sum(len(w["cloud"]) for w in want)
    return info, got


def rc_of(data, **kw):
    rc, msg, _, _ = M.hc_read(data, **kw)
    return rc, msg


# ---- the fixture -----------------------------------------------------------------------------------------------------------------
def test_golden_fixture_is_the_generators():
    with open(G.PATH, "rb") as f:
        assert f.read() == G.build()


@pytest.mark.parametrize("reader", ["hostcheck", "model"])
def test_golden_fixture_reads_as_expected(reader):
    data = open(G.PATH, "rb").read()
    nodes = M.hc_read(data)[3] if reader == "hostcheck" else M.read_bag(data)
    assert [n["seq"] for n in nodes] == [7, 9]
    for n, (seq, odom, pts) in zip(nodes, G.EXPECTED):
        assert np.array_equal(np.asarray(n["odom"]), np.array(odom))
        assert np.array_equal(n["cloud"], np.array(pts, dtype=np.float32))
    assert nodes[1]["layout"]["row_step"] == 40 and nodes[1]["layout"]["height"] == 2
    assert nodes[0]["layout"]["point_step"] == 32 and nodes[0]["layout"]["offset"] == [0, 4, 8, 16]


def test_golden_fixture_counts_and_keep_first():
    data = open(G.PATH, "rb").read()
    info, got = check(data, keep_first=True)
    assert [n["seq"] for n in got] == [7, 7, 9]
    assert [n["stamp_ns"] for n in got] == [10 * 10**9, 10 * 10**9 + 500000000, 11 * 10**9]
    assert (info["chunks"], info["connections"], info["messages"], info["selected"], info["unknown_records"]) == (2, 2, 6, 3, 0)
    assert info["md5sum"] == G.MD5.decode()
    assert rc_of(data, topic="/tf")[0] == E_UNSUPPORTED          # tf2_msgs/TFMessage is not erasor/node


# ---- the model's kitti2node layout ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep_first", [False, True])
@pytest.mark.parametrize("chunk_bytes", [1, 3000, 1 << 20])
def test_kitti2node_layout(keep_first, chunk_bytes):
    nodes = nodes_of(9)
    data = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=chunk_bytes)
    info, got = check(data, keep_first)
    seqs = [s for s, _, _ in nodes]
    assert [n["seq"] for n in got] == ([seqs[0]] + seqs if keep_first else seqs)
    assert info["messages"] == 4 * 10 and info["selected"] == 10 and info["connections"] == 4
    for n, (_, odom, cloud) in zip(got[1:] if keep_first else got, nodes):
        assert np.array_equal(n["odom"], odom) and np.array_equal(n["cloud"].view(np.uint32), cloud.view(np.uint32))
    if chunk_bytes == 1:
        assert info["chunks"] == 40


def test_equal_timestamps_keep_file_order():
    nodes = nodes_of(6)
    msgs = [(t, (5, 0), p) for t, _, p in M.kitti2node_messages(nodes)]
    _, got = check(M.write_bag(msgs, chunk_bytes=2000), keep_first=True)
    assert [n["seq"] for n in got] == [nodes[0][0]] + [s for s, _, _ in nodes]


def test_out_of_order_times_across_chunks():
    nodes = nodes_of(8)
    msgs = M.kitti2node_messages(nodes)
    # frames written newest first in the second half: delivery order is by record time
    frames = [msgs[4 * k:4 * k + 4] for k in range(len(msgs) // 4)]
    data = M.write_bag([m for f in frames[:4] + frames[4:][::-1] for m in f], chunk_bytes=2500)
    _, got = check(data, keep_first=True)
    assert [n["seq"] for n in got] == [nodes[0][0]] + [s for s, _, _ in nodes]


@pytest.mark.parametrize("layout", [k for k in M.LAYOUTS if k != "x_float64"])
def test_layouts(layout):
    nodes = nodes_of(4, n_pts=37)
    info, got = check(M.write_bag(M.kitti2node_messages(nodes, layout=layout), chunk_bytes=4000))
    takes_i = layout not in ("i_uint16", "i_float64", "no_intensity")
    assert info["intensity_zero_filled"] == (0 if takes_i else len(got))
    for n, (_, _, cloud) in zip(got, nodes):
        assert n["layout"]["fields"] == (15 if takes_i else 7)
        assert np.array_equal(n["cloud"][:, :3].view(np.uint32), cloud[:, :3].view(np.uint32))
        want_i = cloud[:, 3] if takes_i else np.zeros(len(cloud), np.float32)
        assert np.array_equal(n["cloud"][:, 3].view(np.uint32), want_i.view(np.uint32))
    if layout == "duplicates":
        assert got[0]["layout"]["offset"] == [12, 8, 16, 20]


def test_frame_id_lengths_shift_the_blob():
    nodes = nodes_of(16, n_pts=9)
    data = M.write_bag(M.kitti2node_messages(nodes, frame_ids=["v" * k for k in range(16)]), chunk_bytes=5000)
    _, got = check(data, keep_first=True)
    assert len({n["layout"]["data_offset"] % 16 for n in got}) >= 8


def test_empty_clouds_and_nan_payloads():
    nodes = nodes_of(7, empty=(0, 3, 6), nan=True)
    info, got = check(M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=3000))
    assert [len(n["cloud"]) for n in got] == [len(c) for _, _, c in nodes]
    for n, (_, _, cloud) in zip(got, nodes):
        assert np.array_equal(n["cloud"].view(np.uint32), cloud.view(np.uint32))


def test_organised_cloud_with_row_padding():
    rng = np.random.default_rng(2)
    msgs = []
    for k, (h, pad) in enumerate([(2, 0), (4, 12), (8, 3), (1, 7)]):
        c = rng.normal(size=(8 * 3, 4)).astype(np.float32)
        data, pc = M.pack_cloud(c, M.LAYOUTS["odd_step"], height=h, row_pad=pad, seed=k)
        msgs.append((M.TOPIC, (10 + k, 0), M.node_payload(k, (10 + k, 0), np.arange(7.0), pc, data)))
    _, got = check(M.write_bag(msgs), keep_first=True)
    assert [n["layout"]["height"] for n in got] == [2, 4, 8, 1]


def test_big_endian_flag_is_counted_and_ignored():
    c = np.arange(40, dtype=np.float32).reshape(10, 4)
    data, pc = M.pack_cloud(c, M.LAYOUTS["packed"])
    pc["is_bigendian"] = 1
    msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), pc, data)) for k in range(3)]
    info, got = check(M.write_bag(msgs))
    assert info["big_endian"] == 2 and np.array_equal(got[0]["cloud"], c)


def test_unknown_records_are_skipped_and_counted():
    nodes = nodes_of(3)
    data = M.write_bag(M.kitti2node_messages(nodes))
    extra = M.record([("op", M.u8(0x09)), ("x", b"1")], b"abc")
    info, _ = check(data + extra + extra)
    assert info["unknown_records"] == 2


def test_hostcheck_decode_ranges():
    nodes = nodes_of(5)
    data = M.write_bag(M.kitti2node_messages(nodes))
    L = M.hostcheck()
    assert M.hc_read(data)[0] == OK
    a = np.frombuffer(data, np.uint8)
    off = np.zeros(4, np.uint64)
    out = np.zeros((1000, 4), np.float32)
    assert L.erasor_hostcheck_bag_decode(a.ctypes.data, 2, 3, out.ctypes.data, off.ctypes.data, None, 0) == OK
    assert np.array_equal(out[:int(off[-1])], np.concatenate([c for _, _, c in nodes[2:5]]))
    assert L.erasor_hostcheck_bag_decode(a.ctypes.data, 3, 3, out.ctypes.data, off.ctypes.data, None, 0) == E_INVALID


# ---- fences ----------------------------------------------------------------------------------------------------------------------
def records(data, a=13, b=None, in_chunk=False, out=None):
    """(pos, op, end, in_chunk) of every record"""
    out = [] if out is None else out
    b = len(data) if b is None else b
    while a < b:
        hl = struct.unpack_from("<I", data, a)[0]
        dl = struct.unpack_from("<I", data, a + 4 + hl)[0]
        h = M._fields(memoryview(data), a + 4, a + 4 + hl)
        op = h["op"][1][0]
        out.append((a, op, a + 8 + hl + dl, in_chunk))
        if op == 5:
            records(data, a + 8 + hl, a + 8 + hl + dl, True, out)
        a += 8 + hl + dl
    return out


def small_bag():
    return M.write_bag(M.kitti2node_messages(nodes_of(4, n_pts=10)), chunk_bytes=1500)


@pytest.mark.parametrize("op", [3, 5, 7, 2, 4, 6])
def test_truncation_inside_each_record_kind(op):
    data = small_bag()
    recs = [r for r in records(data) if r[1] == op]
    assert recs
    pos, _, end, _ = recs[-1]
    for cut in sorted({pos + 1, pos + 4, pos + 9, (pos + end) // 2, end - 1}):
        rc, msg = rc_of(data[:cut])
        assert rc == E_INVALID, (cut, msg)
        assert "byte" in msg


@pytest.mark.parametrize("op", [7, 2])
def test_records_running_past_their_chunk(op):
    data = bytearray(small_bag())
    pos = [r for r in records(bytes(data)) if r[1] == op and r[3]][0][0]
    hl = struct.unpack_from("<I", data, pos)[0]
    struct.pack_into("<I", data, pos + 4 + hl, struct.unpack_from("<I", data, pos + 4 + hl)[0] + 100000)
    rc, msg = rc_of(bytes(data))
    assert rc == E_INVALID and "past its container" in msg and f"byte {pos}" in msg


def test_chunk_size_mismatch():
    data = bytearray(small_bag())
    pos = [r for r in records(bytes(data)) if r[1] == 5][0][0]
    i = bytes(data).index(b"size=", pos) + 5
    struct.pack_into("<I", data, i, struct.unpack_from("<I", data, i)[0] + 1)
    rc, msg = rc_of(bytes(data))
    assert rc == E_INVALID and f"chunk at byte {pos}" in msg


@pytest.mark.parametrize("comp", ["bz2", "lz4"])
def test_compressed_chunks(comp):
    data = M.write_bag(M.kitti2node_messages(nodes_of(3)), compression=comp)
    rc, msg = rc_of(data)
    assert rc == E_UNSUPPORTED and comp in msg and f"byte {13 + 4096}" in msg


def test_undefined_connection():
    msgs = M.kitti2node_messages(nodes_of(2))
    data = M.write_bag(msgs)
    # a message record on connection 9 appended in a chunk of its own
    rec = M.record([("op", M.u8(2)), ("conn", M.u32(9)), ("time", M.time_bytes((1, 0)))], b"x")
    chunk = M.record([("op", M.u8(5)), ("compression", b"none"), ("size", M.u32(len(rec)))], rec)
    rc, msg = rc_of(data + chunk)
    assert rc == E_INVALID and "connection 9" in msg


def test_wrong_type_on_topic():
    data = M.write_bag(M.kitti2node_messages(nodes_of(2)), types={M.TOPIC: "sensor_msgs/PointCloud2"})
    rc, msg = rc_of(data)
    assert rc == E_UNSUPPORTED and "sensor_msgs/PointCloud2" in msg


def test_missing_header_field():
    data = bytearray(small_bag())
    i = bytes(data).index(b"compression=")
    data[i:i + 11] = b"compressioX"
    rc, msg = rc_of(bytes(data))
    assert rc == E_INVALID and "compression" in msg


@pytest.mark.parametrize("delta", [1, -1, 8])
def test_message_longer_or_shorter_than_its_structure(delta):
    c = np.ones((5, 4), np.float32)
    data, pc = M.pack_cloud(c, M.LAYOUTS["packed"])
    good = M.node_payload(1, (1, 0), np.arange(7.0), pc, data)
    bad = good + b"\0" * delta if delta > 0 else good[:delta]
    msgs = [(M.TOPIC, (1, 0), good), (M.TOPIC, (2, 0), good), (M.TOPIC, (3, 0), bad)]
    rc, msg = rc_of(M.write_bag(msgs))
    assert rc == E_INVALID and "node 1" in msg


def test_field_read_past_data():
    c = np.ones((6, 4), np.float32)
    data, pc = M.pack_cloud(c, M.LAYOUTS["packed"])
    for change in ({"width": 7}, {"point_step": 17}, {"fields": [("x", 0, 7, 1), ("y", 4, 7, 1), ("z", 8, 7, 1), ("intensity", 13, 7, 1)]},
                   {"height": 2, "width": 3, "row_step": 49}):
        q = dict(pc, **change)
        msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), q, data)) for k in range(2)]
        rc, msg = rc_of(M.write_bag(msgs))
        assert rc == E_INVALID and "lidar.data" in msg, change


def test_x_as_float64():
    msgs = M.kitti2node_messages(nodes_of(2), layout="x_float64")
    rc, msg = rc_of(M.write_bag(msgs))
    assert rc == E_UNSUPPORTED and "'x'" in msg and "node 0" in msg


def test_other_bag_versions():
    data = M.write_bag(M.kitti2node_messages(nodes_of(2)), version=b"1.2")
    rc, msg = rc_of(data)
    assert rc == E_UNSUPPORTED and "V1.2" in msg
    assert rc_of(b"not a bag at all")[0] == E_INVALID


def test_capacity_of_one_cloud():
    data, pc = M.pack_cloud(np.ones((1, 4), np.float32), M.LAYOUTS["packed"])
    q = dict(pc, width=1 << 16, height=1 << 15, point_step=0, row_step=0)
    msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), q, data)) for k in range(2)]
    rc, msg = rc_of(M.write_bag(msgs))
    assert rc == E_CAPACITY and "2^31" in msg
