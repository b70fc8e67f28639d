"""CPU: bags with bz2 chunks (DESIGN.md section 12.2.2).  The host build (erasor_b200/csrc/bz2_stream.h and bag_index.h compiled into
liberasor_b200_hostcheck.so, the decode stages run serially) against Python's bz2 (libbz2) and the uncompressed twin of every bag,
the fixture tests/golden/node_tiny_bz2.bag, every fence with its code, chunk, block and bit, and a seeded differential test of
mutated streams against libbz2."""
import bz2
import ctypes
import os
import sys

import numpy as np
import pytest

import bag_model as M
import bz2_model as B
from lz4_model import top_records
from test_bag_model import nodes_of
from test_lz4_bag_model import strip

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_bag_bz2_golden as G  # noqa: E402

OK, E_INVALID, E_UNSUPPORTED = 0, -1, -5
CHUNK = 13 + 4096                                   # the first chunk record of base()
needs_hostcheck = pytest.mark.skipif(not os.path.exists(M.HOSTCHECK), reason="build with erasor_b200/csrc/build.sh")
# libbz2 accepts these and the device refuses them (bz2_stream.h)
DIVERGENCES = ("randomised block", "second bzip2 stream", "goes on past the end of its bzip2 stream", "over-subscribed", "incomplete Huffman")


def hc_stream(stream, size):
    """erasor_hostcheck_bz2_stream: (rc, message, decoded bytes)"""
    L = M.hostcheck()
    L.erasor_hostcheck_bz2_stream.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t]
    src = np.frombuffer(stream, np.uint8) if stream else np.zeros(1, np.uint8)
    out = np.zeros(max(size, 1), np.uint8)
    err = ctypes.create_string_buffer(1024)
    rc = L.erasor_hostcheck_bz2_stream(src.ctypes.data, len(stream), size, out.ctypes.data, err, 1024)
    return rc, err.value.decode(), out[:size].tobytes()


def twin_check(plain, twin, keep_first=False):
    r0, r1 = M.hc_read(plain, keep_first=keep_first), M.hc_read(twin, keep_first=keep_first)
    assert r0[0] == OK and r1[0] == OK, r1[1]
    assert r1[2] == r0[2]
    from test_bag_model import same_nodes
    same_nodes(strip(r1[3]), strip(r0[3]))
    return r1


# ---- streams through the host build against libbz2 -----------------------------------------------------------------------------------
def sample(n, seed):
    rng = np.random.default_rng(seed)
    return b"".join([rng.integers(0, 256, n // 3, dtype=np.uint8).tobytes(), bytes(n // 3), (b"xyz" * n)[:n - 2 * (n // 3)]])


@needs_hostcheck
@pytest.mark.parametrize("level", range(1, 10))
def test_every_level_decodes_as_libbz2(level):
    data = sample(150000 * level, level)
    s = bz2.compress(data, level)
    rc, msg, out = hc_stream(s, len(data))
    assert rc == OK and out == data, msg


@needs_hostcheck
@pytest.mark.parametrize("name", ["empty", "one_byte", "runs_0_and_251", "run_at_block_end", "long_runa_runb", "periodic", "five_blocks",
                                  "full_block"])
def test_edge_streams(name):
    rng = np.random.default_rng(7)
    if name == "empty":
        data, s = b"", bz2.compress(b"")
    elif name == "one_byte":
        data, s = b"q", bz2.compress(b"q", 1)
    elif name == "runs_0_and_251":
        data = b"ab" + b"c" * 4 + b"d" + b"e" * 255 + b"f"          # RLE1 counts 0 and 251
        s = B.encode(data)
    elif name == "run_at_block_end":
        data = b"xy" + b"z" * 300                                    # block 0 ends with the run's count
        r = B.rle1(data)
        s = B.encode(data, split=[len(r) - 10, 10])
    elif name == "long_runa_runb":
        data = b"\x00" * 1000000 + b"\x01"                           # RUNA/RUNB spell runs of thousands of MTF zeros
        s = bz2.compress(data, 9)
    elif name == "periodic":
        data = b"abcdefg" * 200000                                   # several BWT cycles per block
        s = bz2.compress(data, 3)
    elif name == "five_blocks":
        data = rng.integers(0, 256, 520000, dtype=np.uint8).tobytes()
        s = bz2.compress(data, 1)
        assert len(B.fields(s)[0]) >= 5
    else:                                                            # blocks of exactly level x 100 000 RLE1 bytes
        data = rng.integers(0, 200, 250000, dtype=np.uint8).tobytes()
        s = bz2.compress(data, 1)
    rc, msg, out = hc_stream(s, len(data))
    assert rc == OK and out == data, msg


def planted_bag():
    """a bag whose node 1 carries planted()'s data as its cloud, and its bz2 twin whose chunk holds the planted block"""
    _, P = B.planted()
    D = P + bytes(-len(P) % 16)
    pc = dict(height=1, width=len(D) // 16, fields=M.LAYOUTS["packed"]["fields"], point_step=16, row_step=len(D), is_bigendian=0)
    msgs = [(M.TOPIC, (1, k), M.node_payload(k, (1, k), np.arange(7.0), pc, D)) for k in range(2)]
    plain = M.write_bag(msgs, chunk_bytes=1 << 30)
    return plain, B.bz2_twin(plain, B.with_planted), D


@needs_hostcheck
def test_a_planted_block_magic_is_a_false_candidate():
    plain, twin, D = planted_bag()
    _, _, _, got = twin_check(plain, twin)
    assert got[0]["cloud"].tobytes() == D
    st = B.hc_stats()
    assert st["blocks"] == 3 and st["candidates"] == 4


# ---- bags ----------------------------------------------------------------------------------------------------------------------------
@needs_hostcheck
@pytest.mark.parametrize("keep_first", [False, True])
@pytest.mark.parametrize("level", [1, 5, 9])
def test_kitti2node_twins(keep_first, level):
    plain = M.write_bag(M.kitti2node_messages(nodes_of(9, n_pts=300)), chunk_bytes=3000)
    twin_check(plain, B.bz2_twin(plain, level=level), keep_first)
    st = B.hc_stats()
    assert st["streams_by_level"][level - 1] == st["chunks"] > 0 and st["blocks"] == st["decoded_chunks"]


@needs_hostcheck
def test_mixed_none_lz4_bz2_chunks_and_equal_times():
    import lz4_model as Z
    nodes = nodes_of(9)
    msgs = [(t, (5, 0), p) for t, _, p in M.kitti2node_messages(nodes)]      # every record at the same time
    plain = M.write_bag(msgs, chunk_bytes=2000)
    twin = B.bz2_twin(Z.lz4_twin(plain, which=lambda k: k % 3 == 1), which=lambda k: k % 3 == 2, level=2)
    _, _, info, got = twin_check(plain, twin, keep_first=True)
    assert [n["seq"] for n in got] == [nodes[0][0]] + [s for s, _, _ in nodes]
    assert 0 < B.hc_stats()["chunks"] < info["chunks"] and 0 < Z.hc_stats()["chunks"]


@needs_hostcheck
def test_golden_fixture_is_the_generators():
    assert open(G.PATH, "rb").read() == G.build()


@needs_hostcheck
@pytest.mark.parametrize("keep_first", [False, True])
def test_golden_fixture(keep_first):
    data = open(G.PATH, "rb").read()
    rc, msg, info, nodes = M.hc_read(data, keep_first=keep_first)
    assert rc == OK, msg
    want = G.nodes()
    want = want if keep_first else want[1:]
    assert [n["seq"] for n in nodes] == [w[0] for w in want]
    for n, (_, odom, cloud) in zip(nodes, want):
        assert np.array_equal(n["cloud"].view(np.uint32), cloud.view(np.uint32)) and np.array_equal(n["odom"], odom)
    st = B.hc_stats()
    assert st["chunks"] == 2 and st["streams_by_level"][0] == 1 and st["streams_by_level"][8] == 1 and st["blocks"] >= 4
    assert os.path.getsize(G.PATH) < 64 * 1024


# ---- fences --------------------------------------------------------------------------------------------------------------------------
def base():
    return M.write_bag(M.kitti2node_messages(nodes_of(3, n_pts=20), debug=False), chunk_bytes=1 << 20)


def _f(s):
    return B.fields(s)


def fence_streams():
    """name -> (stream_of(chunk data), code, texts)"""
    c = lambda d: bz2.compress(d, 9)                                 # noqa: E731
    blk = lambda d: _f(c(d))[0][0]                                   # noqa: E731
    eos = lambda d: _f(c(d))[1]                                      # noqa: E731
    return {
        "bzip1": (lambda d: b"BZ0" + c(d)[3:], E_UNSUPPORTED, ["does not start with 'BZh'"]),
        "level_0": (lambda d: b"BZh0" + c(d)[4:], E_INVALID, ["level digit 48", "bit 24"]),
        "randomised": (lambda d: B.set_field(c(d), blk(d)["rand"], 1, 1), E_UNSUPPORTED, ["block 0: a randomised block", "bit 112 "]),
        "second_stream": (lambda d: c(d) + bz2.compress(b"x"), E_UNSUPPORTED, ["second bzip2 stream"]),
        "trailing_byte": (lambda d: c(d) + b"\0", E_INVALID, ["goes on past the end of its bzip2 stream"]),
        "truncated": (lambda d: c(d)[:-4], E_INVALID, ["stream runs past the chunk"]),
        "truncated_in_block": (lambda d: c(d)[:40], E_INVALID, ["block 0: the stream runs past the chunk"]),
        "no_magic": (lambda d: B.set_field(c(d), eos(d), 48, 0x123456789ABC), E_INVALID, ["neither a block magic", "after block 0"]),
        "no_block_at_all": (lambda d: b"BZh9" + b"\x12" * 20, E_INVALID, ["neither a block magic", "after the stream header", "bit 32 "]),
        "empty_map": (lambda d: B.splice(c(d), blk(d)["map"], blk(d)["groups"] - blk(d)["map"], "0" * 16), E_INVALID, ["an empty symbol map"]),
        "groups_1": (lambda d: B.set_field(c(d), blk(d)["groups"], 3, 1), E_INVALID, ["nGroups outside 2..6"]),
        "groups_7": (lambda d: B.set_field(c(d), blk(d)["groups"], 3, 7), E_INVALID, ["nGroups outside 2..6"]),
        "selectors_0": (lambda d: B.set_field(c(d), blk(d)["nsel"], 15, 0), E_INVALID, ["nSelectors of 0"]),
        "selector_index": (lambda d: B.splice(c(d), blk(d)["sel"], 0, "1" * blk(d)["ng"]), E_INVALID, ["selector MTF index"]),
        "code_length_0": (lambda d: B.set_field(c(d), blk(d)["lens"], 5, 0), E_INVALID, ["code length outside 1..20"]),
        "code_length_21": (lambda d: B.set_field(c(d), blk(d)["lens"], 5, 21), E_INVALID, ["code length outside 1..20"]),
        "over_subscribed": (lambda d: B.encode(d, lens=[1] * (len(set(B.rle1(d))) + 2), check=False), E_INVALID, ["over-subscribed"]),
        "incomplete": (lambda d: B.encode(d, lens=[10] * (len(set(B.rle1(d))) + 2), check=False), E_INVALID, ["incomplete Huffman"]),
        "origptr": (lambda d: B.set_field(c(d), blk(d)["orig"], 24, 0xFFFFFF), E_INVALID, ["origPtr at or past", f"bit {32 + 48 + 33}"]),
        "block_crc": (lambda d: B.flip_bit(c(d), blk(d)["crc"]), E_INVALID, ["block 0: the block CRC does not match", "bit 32 "]),
        "stream_crc": (lambda d: B.flip_bit(c(d), eos(d) + 60), E_INVALID, ["the stream CRC does not match"]),
        "size": (lambda d: c(d[:-1]), E_INVALID, ["does not decode to the chunk's 'size'"]),
        "run_too_long": (lambda d: B.encode(d, 1, parts=[b"a" * 100001], check=False), E_INVALID, ["RUNA/RUNB run longer"]),
        "block_too_long": (lambda d: B.stream_of_blocks([B.block_of_symbols(B.mtf_symbols(b"b" + b"a" * 99999 + b"c", b"abc"), b"abc", 0)], 1),
                           E_INVALID, ["block longer than the block max"]),
        "rle_end": (lambda d: B.encode(d, parts=[b"xyzzzz"], check=False), E_INVALID, ["four equal bytes end the block"]),
    }


def fence_bags():
    return {k: (B.bz2_twin(base(), v[0]), v[1], v[2]) for k, v in fence_streams().items()}


@needs_hostcheck
@pytest.mark.parametrize("name", list(fence_streams()))
def test_fences(name):
    data, code, texts = fence_bags()[name]
    rc, msg = M.hc_read(data)[:2]
    assert rc == code and f"bz2 chunk at byte {CHUNK}" in msg and all(t in msg for t in texts), msg
    assert B.hc_stats()["chunks"] == 0


@needs_hostcheck
def test_second_block_fences_name_block_1():
    data = np.random.default_rng(1).integers(0, 256, 150000, dtype=np.uint8).tobytes()
    s = bz2.compress(data, 1)
    blocks, _ = B.fields(s)
    bad = B.set_field(s, blocks[1]["groups"], 3, 0)
    rc, msg, _ = hc_stream(bad, len(data))
    assert rc == E_INVALID and "block 1: nGroups" in msg and f"bit {blocks[1]['groups']} " in msg, msg


@needs_hostcheck
def test_unindexed_bz2_chunk():
    twin = B.bz2_twin(base())
    recs = [r for r in top_records(twin) if r[2]["op"][1][0] == 4]
    rc, msg = M.hc_read(twin[:recs[0][0]] + twin[recs[-1][1]:])[:2]
    assert rc == E_UNSUPPORTED and "bz2-compressed" in msg and "unindexed" in msg, msg


# ---- differential test against libbz2 ---------------------------------------------------------------------------------------------
def libbz2(s):
    try:
        return bz2.decompress(s)
    except (OSError, ValueError, EOFError):
        return None


@needs_hostcheck
@pytest.mark.parametrize("seed", range(4))
def test_differential_against_libbz2(seed):
    rng = np.random.default_rng(seed)
    data = sample(3000 + 1000 * seed, seed) + b"a" * 300 + (b"periodic" * 50)
    s = bz2.compress(data, 1 + 3 * seed % 9)
    blocks, eos = B.fields(s)
    cases = [B.flip_bit(s, int(b)) for b in rng.integers(0, 8 * len(s), 150)]
    cases += [B.flip_bit(s, int(b)) for b in rng.integers(32, blocks[0]["syms"] + 64, 100)]     # the header and the tables
    cases += [s[:int(k)] for k in rng.integers(0, len(s), 30)]
    cases += [B.set_field(s, blocks[0][f], w, int(rng.integers(0, 1 << w))) for f, w in (("orig", 24), ("groups", 3), ("nsel", 15)) for _ in range(5)]
    cases += [s, s + b"\0", s + bz2.compress(b"z"), B.set_field(s, blocks[0]["rand"], 1, 1)]
    tally = {"both": 0, "neither": 0, "divergence": 0}
    for m in cases:
        ref = libbz2(m)
        rc, msg, out = hc_stream(m, len(ref) if ref is not None else len(data))
        if rc == OK:
            assert ref is not None and out == ref, msg                  # whatever we accept, libbz2 accepts with the same bytes
            tally["both"] += 1
        elif ref is None:
            tally["neither"] += 1                                        # whatever libbz2 rejects, we reject
        else:
            assert any(t in msg for t in DIVERGENCES), msg               # and every other refusal is a documented divergence
            tally["divergence"] += 1
    assert tally["both"] > 0 and tally["neither"] > 0 and tally["divergence"] >= 2, tally
