"""CPU: bags with lz4 chunks (DESIGN.md section 12.2.1).  The model of tests/lz4_model.py against the published XXH32 vectors and a
system liblz4 (both ways, when ctypes can load one); the host build (erasor_b200/csrc/lz4_frame.h and bag_index.h compiled into
liberasor_b200_hostcheck.so, the decode stages run serially) against the uncompressed twin of every bag and the fixture
tests/golden/node_tiny_lz4.bag; adversarial block streams embedded as cloud data, so that every decoded byte comes back through
the load; and every fence, with its code and offset."""
import os
import struct
import sys

import numpy as np
import pytest

import bag_model as M
import lz4_model as Z
from test_bag_model import nodes_of, same_nodes

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_bag_lz4_golden as G  # noqa: E402

OK, E_INVALID, E_UNSUPPORTED = 0, -1, -5
LIB = Z.liblz4()
needs_hostcheck = pytest.mark.skipif(not os.path.exists(M.HOSTCHECK), reason="build with erasor_b200/csrc/build.sh")
needs_liblz4 = pytest.mark.skipif(LIB is None, reason="no system liblz4 to cross-check against")


# ---- the model -------------------------------------------------------------------------------------------------------------------
def test_xxh32_published_vectors():
    assert Z.xxh32(b"") == 0x02CC5D05
    assert Z.xxh32(b"", 0x9E3779B1) == 0x36B78AE7


def sample(n, seed):
    rng = np.random.default_rng(seed)
    parts = [rng.integers(0, 256, n // 4, dtype=np.uint8).tobytes(), bytes(n // 4), rng.integers(0, 3, n // 4, dtype=np.uint8).tobytes()]
    parts.append((parts[0][:777] * (n // 3000 + 1))[:n - 3 * (n // 4)])
    return b"".join(parts)


@needs_liblz4
@pytest.mark.parametrize("bsid", [4, 5, 6, 7])
@pytest.mark.parametrize("sums", [(False, False), (True, True), (True, False)])
def test_model_and_liblz4_read_each_other(bsid, sums):
    data = sample(300000, bsid)
    assert Z.decode_frame(Z.lib_compress(LIB, data, bsid, *sums)) == data
    mine = Z.compress(data[:150000], bsid, *sums, stored=(1,))
    out, ok = Z.lib_decompress(LIB, mine, 150000)
    assert ok and out == data[:150000]


@needs_hostcheck
def test_host_encoder_frames_decode():
    data = sample(1 << 20, 1)
    for bsid in (4, 7):
        f = Z.hc_frame(data, bsid, True, True)
        assert Z.decode_frame(f) == data
        if LIB is not None:
            out, ok = Z.lib_decompress(LIB, f, len(data))
            assert ok and out == data


# ---- the host build against the uncompressed twin ------------------------------------------------------------------------------------
def strip(nodes):
    return [dict(n, layout=dict(n["layout"], data_offset=0)) for n in nodes]


def twin_check(plain, twin, keep_first=False):
    r0, r1 = M.hc_read(plain, keep_first=keep_first), M.hc_read(twin, keep_first=keep_first)
    assert r0[0] == OK and r1[0] == OK, r1[1]
    assert r1[2] == r0[2]
    same_nodes(strip(r1[3]), strip(r0[3]))
    return r1


@needs_hostcheck
def test_golden_fixture_is_the_generators():
    assert open(G.PATH, "rb").read() == G.build()


@needs_hostcheck
@pytest.mark.parametrize("keep_first", [False, True])
def test_golden_fixture_equals_its_uncompressed_twin(keep_first):
    twin = open(G.PATH, "rb").read()
    twin_check(open(G.SRC, "rb").read(), twin, keep_first)
    chunks = [twin[d0:d0 + dl] for pos, end, fs, d0, dl in Z.top_records(twin) if fs["op"][1][0] == 5]
    assert Z.hc_stats() == dict(chunks=2, decoded_chunks=2, compressed_bytes=sum(len(f) for f in chunks),
                                decoded_bytes=sum(len(Z.decode_frame(f)) for f in chunks), blocks=4, stored_blocks=1, block_checksums=3,
                                content_checksums=2)


@needs_hostcheck
@pytest.mark.parametrize("keep_first", [False, True])
@pytest.mark.parametrize("chunk_bytes,bsid,block_sums", [(1, 4, False), (3000, 4, True), (70000, 4, False), (300000, 5, True), (1 << 20, 7, False)])
def test_kitti2node_twins(keep_first, chunk_bytes, bsid, block_sums):
    plain = M.write_bag(M.kitti2node_messages(nodes_of(9, n_pts=300)), chunk_bytes=chunk_bytes)
    twin_check(plain, Z.lz4_twin(plain, lambda d: Z.compress(d, bsid, block_sums, True, stored=(1,))), keep_first)


@needs_hostcheck
def test_mixed_chunks_and_equal_times_keep_file_order():
    nodes = nodes_of(8)
    msgs = [(t, (5, 0), p) for t, _, p in M.kitti2node_messages(nodes)]      # every record at the same time
    plain = M.write_bag(msgs, chunk_bytes=2000)
    twin = Z.lz4_twin(plain, which=lambda k: k % 3 != 1)
    _, _, info, got = twin_check(plain, twin, keep_first=True)
    assert [n["seq"] for n in got] == [nodes[0][0]] + [s for s, _, _ in nodes]
    st = Z.hc_stats()
    assert 0 < st["chunks"] < info["chunks"]


@needs_hostcheck
def test_layouts_and_organised_clouds():
    for layout in ("packed", "odd_step", "i_uint16", "no_intensity", "duplicates", "count0"):
        plain = M.write_bag(M.kitti2node_messages(nodes_of(4, n_pts=37), layout=layout), chunk_bytes=4000)
        twin_check(plain, Z.lz4_twin(plain))
    rng = np.random.default_rng(2)
    msgs = []
    for k, (h, pad) in enumerate([(2, 0), (4, 12), (8, 3)]):
        d, pc = M.pack_cloud(rng.normal(size=(24, 4)).astype(np.float32), M.LAYOUTS["odd_step"], height=h, row_pad=pad, seed=k)
        msgs.append((M.TOPIC, (10 + k, 0), M.node_payload(k, (10 + k, 0), np.arange(7.0), pc, d)))
    plain = M.write_bag(msgs)
    twin_check(plain, Z.lz4_twin(plain), keep_first=True)


# ---- adversarial streams, embedded as cloud data ---------------------------------------------------------------------------------
def embedded(seqs, tail=64, bsid=5, seed=0):
    """a bag of one node (twice: the first is dropped) whose cloud data D is what the parse seqs produces; the chunk is the frame
    [prefix (greedy), D (the parse), suffix (literals only)]"""
    rng = np.random.default_rng(seed)
    D = Z.data_of_seqs(seqs, tail, rng)
    D += bytes(-len(D) % 16)
    seqs = list(seqs)
    pc = dict(height=1, width=len(D) // 16, fields=M.LAYOUTS["packed"]["fields"], point_step=16, row_step=len(D), is_bigendian=0)
    msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), pc, D)) for k in range(2)]
    plain = M.write_bag(msgs, chunk_bytes=1 << 30)

    def frame_of(data):
        a = data.rindex(D)
        return Z.frame([(data[:a], "lz"), (D, seqs), (data[a + len(D):], [])], bsid, True, True)
    return plain, Z.lz4_twin(plain, frame_of), D


@needs_hostcheck
@pytest.mark.parametrize("name,seqs", [
    ("literals_only", []),
    ("extensions", [(1, 1, 4), (15, 2, 19), (16, 1, 20), (269, 7, 273), (270, 3, 274), (15 + 255 * 3 + 7, 5, 19 + 255 * 4 + 3)]),
    ("offsets", [(40, 1, 300), (3, 2, 77), (40, 31, 100), (9, 32, 64), (50, 33, 34), (1, 33, 4)]),
    ("offset_65535", [(70000, 65535, 65540), (4, 1, 4)]),
])
def test_adversarial_streams(name, seqs):
    plain, twin, D = embedded(seqs)
    _, _, _, got = twin_check(plain, twin)
    assert got[0]["cloud"].tobytes() == D                            # every decoded byte, bit for bit


@needs_hostcheck
def test_a_block_of_exactly_the_block_max():
    plain = M.write_bag(M.kitti2node_messages(nodes_of(2, n_pts=3000)), chunk_bytes=1 << 30)
    frames = []
    twin = Z.lz4_twin(plain, lambda d: frames.append(Z.compress(d, 4, True, True)) or frames[-1])
    twin_check(plain, twin)
    first = struct.unpack_from("<I", frames[0], 7)[0] & 0x7FFFFFFF
    assert Z.decode_block(frames[0][11:11 + first], 1 << 16).__len__() == 1 << 16 and Z.hc_stats()["blocks"] >= 3


# ---- fences ----------------------------------------------------------------------------------------------------------------------
def base():
    return M.write_bag(M.kitti2node_messages(nodes_of(3, n_pts=20), debug=False), chunk_bytes=1 << 20)


def raw_frame(*blocks, bsid=4):
    """a frame of raw compressed blocks, with a content checksum of nothing (the decode fails first)"""
    desc = bytes([0x64, bsid << 4])
    out = struct.pack("<I", Z.MAGIC) + desc + bytes([(Z.xxh32(desc) >> 8) & 0xFF])
    for b in blocks:
        out += struct.pack("<I", len(b)) + b
    return out + struct.pack("<I", 0) + struct.pack("<I", 0)


def flip(f, at):
    at %= len(f)
    return f[:at] + bytes([f[at] ^ 1]) + f[at + 1:]


FRAME_FENCES = {
    # name: (frame_of, code, text)
    "magic": (lambda d: d, E_UNSUPPORTED, "frame magic"),
    "version": (lambda d: Z.frame([(d, "lz")], flg=0x24), E_UNSUPPORTED, "frame version 0"),
    "reserved_flg": (lambda d: Z.frame([(d, "lz")], flg=0x66), E_INVALID, "reserved FLG bit"),
    "dictionary": (lambda d: Z.frame([(d, "lz")], flg=0x65), E_UNSUPPORTED, "dictionary"),
    "linked": (lambda d: Z.frame([(d, "lz")], flg=0x44), E_UNSUPPORTED, "linked blocks"),
    "reserved_bd": (lambda d: Z.frame([(d, "lz")], bd=0x41), E_INVALID, "reserved BD bit"),
    "block_max_id": (lambda d: Z.frame([(d, "lz")], bd=0x30), E_INVALID, "block max id 3"),
    "content_size": (lambda d: Z.frame([(d, "lz")], content_size=len(d) + 1), E_INVALID, "content size"),
    "header_checksum": (lambda d: flip(Z.frame([(d, "lz")]), 6), E_INVALID, "header checksum"),
    "block_above_max": (lambda d: Z.frame([(d + bytes(70000), "stored")]), E_INVALID, "above the block max"),
    "block_past_chunk": (lambda d: Z.frame([(d, "lz")])[:-12], E_INVALID, "runs past the chunk"),
    "trailing_bytes": (lambda d: Z.frame([(d, "lz")]) + b"\0", E_INVALID, "past the end of its LZ4 frame"),
    "block_checksum": (lambda d: flip(Z.frame([(d, "lz")], block_sums=True), -9), E_INVALID, "block checksum does not match"),
    "content_checksum": (lambda d: flip(Z.frame([(d, "lz")]), -1), E_INVALID, "content checksum does not match"),
    "decoded_length": (lambda d: Z.frame([(d[:-1], "lz")]), E_INVALID, "does not decode to the chunk's 'size'"),
    "offset_0": (lambda d: raw_frame(b"\x40abcd\x00\x00\x10x"), E_INVALID, "offset of 0 (byte 16 of the frame)"),
    "offset_before": (lambda d: raw_frame(b"\x40abcd\x05\x00\x10x"), E_INVALID, "before the block's own output (byte 16"),
    "offset_before_2nd_block": (lambda d: raw_frame(b"\x40abcd", b"\x00\x01\x00\x10x"), E_INVALID, "malformed block 1"),
    "literals_past": (lambda d: raw_frame(b"\xf0\x10abc"), E_INVALID, "literal run reading past the block"),
    "extension_past": (lambda d: raw_frame(b"\xf0\xff"), E_INVALID, "length extension reading past"),
    "output_past": (lambda d: raw_frame(b"\x4fabcd\x01\x00" + b"\xff" * 300 + b"\x00\x10x"), E_INVALID, "output past the block max"),
    "ends_in_sequence": (lambda d: raw_frame(b"\x40abcd\x01"), E_INVALID, "ends inside a sequence"),
    "ends_after_match": (lambda d: raw_frame(b"\x40abcd\x01\x00"), E_INVALID, "ends inside a sequence"),
}


@needs_hostcheck
@pytest.mark.parametrize("name", list(FRAME_FENCES))
def test_frame_fences(name):
    frame_of, code, text = FRAME_FENCES[name]
    twin = Z.lz4_twin(base(), frame_of)
    rc, msg = M.hc_read(twin)[:2]
    assert rc == code and text in msg and f"lz4 chunk at byte {13 + 4096}" in msg, msg
    assert Z.hc_stats()["chunks"] == 0


def index_entries(data):
    """(position of the entry, conn) of every index data entry"""
    out = []
    for pos, end, fs, d0, dl in Z.top_records(data):
        if fs["op"][1][0] == 4:
            out += [(q, struct.unpack("<I", fs["conn"][1])[0]) for q in range(d0, d0 + dl, 12)]
    return out


def index_fence_bags():
    """name -> (bag, code, texts) of the index fences: an unindexed bag, then index entries of the last node that miss its record,
    reach past the decoded chunk, point to a record of another op, or carry another time"""
    twin = Z.lz4_twin(base())
    entries = [q for q, c in index_entries(twin) if c == 1]       # kitti2node's second connection is the node topic
    recs = [r for r in Z.top_records(twin) if r[2]["op"][1][0] == 4]
    out = {"unindexed": (twin[:recs[0][0]] + twin[recs[-1][1]:], E_UNSUPPORTED, ["unindexed", f"chunk at byte {13 + 4096}"])}
    for name, at, value, texts in (("missed_record", 8, lambda v: v + 1, [f"lz4 chunk at byte {13 + 4096}"]),
                                   ("past_chunk", 8, lambda v: 1 << 30, ["runs past the decoded chunk"]),
                                   ("other_op", 8, lambda v: 0, ["does not point to a message data record"]),   # a connection record
                                   ("time", 4, lambda v: v + 1, ["has time"])):
        b = bytearray(twin)
        struct.pack_into("<I", b, entries[-1] + at, value(struct.unpack_from("<I", b, entries[-1] + at)[0]))
        out[name] = (bytes(b), E_INVALID, ["node 2"] + texts)
    return out


def empty_chunk_bags():
    """name -> (bag, code, texts): a node's chunk rewritten as size 0 and a frame without blocks, its content checksum wrong or
    right, as the first decoded chunk or the last; the message names that chunk"""
    plain = M.write_bag(M.kitti2node_messages(nodes_of(4, n_pts=20), debug=False), chunk_bytes=1)   # /tf, node, /tf, node, ...
    empty = Z.frame([])
    out = {}
    for where, target in (("first", 3), ("last", 9)):               # chunk 3: the first kept node (chunk 1's is dropped)
        for name, f, text in (("bad_sum", flip(empty, -1), "content checksum does not match"), ("good_sum", empty, "runs past the decoded chunk")):
            k = iter(range(100))
            twin = bytearray(Z.lz4_twin(plain, lambda d: f if next(k) == target else Z.compress(d)))
            pos, _, fs, _, _ = [r for r in Z.top_records(bytes(twin)) if r[2]["op"][1][0] == 5][target]
            struct.pack_into("<I", twin, fs["size"][0], 0)
            out[f"{where}_{name}"] = (bytes(twin), E_INVALID, [text, f"lz4 chunk at byte {pos}"])
    return out


def bad_node_bags():
    """the uncompressed bag and its twins with a node one byte too long (node 1) and one too short (node 2), each in an lz4 or
    a none chunk"""
    c = np.ones((5, 4), np.float32)
    data, pc = M.pack_cloud(c, M.LAYOUTS["packed"])
    good = M.node_payload(1, (1, 0), np.arange(7.0), pc, data)
    msgs = [(M.TOPIC, (1, 0), good), (M.TOPIC, (2, 0), good), (M.TOPIC, (3, 0), good + b"\0"), (M.TOPIC, (4, 0), good[:-1])]
    plain = M.write_bag(msgs, chunk_bytes=1)
    return plain, [Z.lz4_twin(plain, which=w) for w in (lambda k: True, lambda k: k == 2, lambda k: k == 3, lambda k: k != 2)]


@needs_hostcheck
@pytest.mark.parametrize("name", ["unindexed", "missed_record", "past_chunk", "other_op", "time"])
def test_index_fences(name):
    data, code, texts = index_fence_bags()[name]
    rc, msg = M.hc_read(data)[:2]
    assert rc == code and all(t in msg for t in texts), msg


@needs_hostcheck
@pytest.mark.parametrize("name", ["first_bad_sum", "first_good_sum", "last_bad_sum", "last_good_sum"])
def test_a_chunk_without_blocks(name):
    data, code, texts = empty_chunk_bags()[name]
    rc, msg = M.hc_read(data)[:2]
    assert rc == code and all(t in msg for t in texts), msg
    assert Z.hc_stats()["chunks"] == 0


@needs_hostcheck
def test_a_bad_node_in_an_lz4_chunk_is_reported_in_delivery_order():
    plain, twins = bad_node_bags()
    want = M.hc_read(plain)[:2]
    for twin in twins:
        rc, msg = M.hc_read(twin)[:2]
        assert rc == want[0] == E_INVALID and "node 1" in msg and "1 bytes longer" in msg, msg
