"""CPU: the segmented LZF encoder and the binary / binary_compressed PCD writer of erasor_pcd_format, host build
(liberasor_b200_hostcheck.so, the same lzf_encode.h the device runs) against the Python restatement in tests/lzf_encode_model.py,
byte for byte; every stream decoded back through the serial decoder and the parallel decoder's stages; whole files read back by
the numpy reader and the host build of erasor_pcd_load; and the uint32 size rule at its edges."""
import struct

import numpy as np
import pytest

import lzf_encode_model as E
import pcd_binary_model as M
from erasor_b200 import synth

S = E.SEG


def rnd(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def check_stream(data, chunks=(33, 64, 4096)):
    """host == model; the stream decodes to data serially and through stages A-C at several chunk sizes; returns the stream"""
    data = bytes(data)
    got, tok, seg = E.hc_encode(data)
    want, mtok, mseg = E.encode(data)
    assert got == want
    assert (tok, seg) == (mtok, mseg) == (tok, -(-len(data) // S))
    assert M.lzf_decompress(got, len(data)) == data
    for ch in chunks:
        rc, out, ntok, msg = M.hc_lzf_decode(got, len(data), ch)
        assert rc == 0, msg
        assert out == data and ntok == tok
    return got


def collision_keys(k=4):
    """k three-byte keys with one hash and different bytes"""
    v = np.arange(1 << 20, dtype=np.uint64)
    h = E.lzf_hash(v >> np.uint64(16), (v >> np.uint64(8)) & np.uint64(255), v & np.uint64(255))
    keys = v[h == h[0x12345]][:k]
    assert len(keys) == k
    return [bytes([int(x) >> 16, (int(x) >> 8) & 255, int(x) & 255]) for x in keys]


@pytest.mark.parametrize("n", [0, 1, 2, 3, 4, 5])
def test_tiny_inputs(n):
    s = check_stream(rnd(n, n))
    assert len(s) == (n + 1 if n else 0)


def test_all_equal_bytes_are_distance_one_references_of_264():
    data = b"\x07" * (3 * S + 5)
    s = check_stream(data)
    seg0 = E.encode_segment(data[:S])[0]
    assert seg0.startswith(M.lit_token(b"\x07") + M.ref_token(264, 1) * 5)     # each segment starts again with one literal


@pytest.mark.parametrize("period", [8191, 8192, 8193])
def test_the_distance_limit(period):
    base = rnd(period, period)
    data = (base * 2)[:S]
    s = check_stream(data)
    if period <= 8192:
        assert len(s) < 0.6 * len(data)                        # the second copy is references at distance period
    else:
        assert len(s) > len(data) - 64                         # out of reach: literals


def test_hash_collisions_with_different_bytes():
    keys = collision_keys()
    rng = np.random.default_rng(3)
    parts = []
    for k in range(400):
        parts.append(keys[rng.integers(0, len(keys))])
        if rng.random() < 0.3:
            parts.append(rnd(int(rng.integers(1, 6)), k))
    data = b"".join(parts)
    check_stream(data)
    # a colliding key in between hides an earlier equal one: cand is the last position with the same hash, not the same bytes
    a, b = keys[0], keys[1]
    data = a + b"\x00\x01" + b + b"\x02" + a
    cand = E.candidates(data)
    assert (cand < 0).all()
    check_stream(data)


@pytest.mark.parametrize("tail", [0, 1, 2, 3, 263, 264, 265])
def test_matches_at_a_segment_end(tail):
    """a long repeat ending exactly at the segment end, or one that would run past it into the next segment"""
    pre = rnd(S - 300 - tail, 11)
    rep = rnd(300, 12)
    data = pre[:S - 600 - tail] + rep + rep + b"\xAA" * tail + rep[:50] + rnd(700, 13)
    check_stream(data)
    segs = [E.encode_segment(data[b:b + S])[0] for b in range(0, len(data), S)]
    assert b"".join(segs) == E.hc_encode(data)[0]


@pytest.mark.parametrize("phase", range(33))
def test_segment_boundary_at_every_literal_phase(phase):
    """a literal stretch that the segment boundary cuts after `phase` bytes of its last run"""
    head = b"\x55" * (S - 64 - phase)                         # compresses; the literals start 64 + phase bytes before the end
    data = head + rnd(64 + phase + 100, phase) + b"\x55" * 40
    s = check_stream(data)
    assert M.lzf_decompress(s, len(data)) == data


@pytest.mark.parametrize("run", [31, 32, 33, 64, 65])
def test_literal_run_lengths(run):
    blk = rnd(40, 99)
    data = blk + rnd(run, run) + blk + rnd(run, run + 1) + blk
    s = check_stream(data)
    assert M.lit_token(data[:32]) == s[:33]


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("d", [-1, 0, 1])
def test_sizes_around_segment_multiples(k, d):
    n = k * S + d
    rng = np.random.default_rng(n)
    data = (rng.integers(0, 4, n, dtype=np.uint8) * 17).tobytes()      # compressible, with references everywhere
    check_stream(data, chunks=(4096,))


def test_random_bytes_stay_within_the_worst_case():
    data = rnd(5 * S + 777, 5)
    s = check_stream(data, chunks=(4096,))
    bound = sum(m + -(-m // 32) for m in (min(S, len(data) - b) for b in range(0, len(data), S)))
    assert len(s) <= bound


def labelled_map():
    sc = synth.Scene(seed=12, length=30.0, n_nodes=4, n_dynamic=3)
    return sc.build_map([0, 1, 2, 3], voxel=0.2, n_beams=16, n_az=400)


def test_soa_of_the_labelled_map():
    c = labelled_map()
    data = E.soa(c)
    s = check_stream(data, chunks=(4096,))
    assert len(s) < len(data)


def special_cloud():
    bits = np.array([0x7FC01234, 0xFFBFFFFF, 0x7F800001, 0xFF800000, 0x7F800000, 0x80000000, 0x00000000, 0x00000001, 0x807FFFFF,
                     0x3F800000, 0xFFFFFFFF, 0x7FFFFFFF], dtype=np.uint32)
    rng = np.random.default_rng(8)
    return bits[rng.integers(0, len(bits), (3001, 4))].view(np.float32)


@pytest.mark.parametrize("mode", ["binary", "binary_compressed"])
@pytest.mark.parametrize("which", ["empty", "one", "two", "specials", "labelled"])
def test_whole_files(mode, which):
    c = {"empty": np.zeros((0, 4), np.float32), "one": np.array([[1.5, -2.0, 3.25, 40.0]], np.float32),
         "two": np.array([[1.5, -2.0, 3.25, 40.0], [np.nan, -0.0, 1e-45, 252.0]], np.float32), "specials": special_cloud(),
         "labelled": labelled_map()}[which]
    rc, got, info = E.hc_format(c, mode)
    assert rc == 0
    assert got == E.write_file(c, mode)
    head = M.header(M.XYZI, len(c), mode)
    assert got.startswith(head) and info["header_bytes"] == len(head) and info["data_mode"] == E.MODES[mode]
    if mode == "binary_compressed":
        stream, tok, seg = E.encode(E.soa(c))
        assert info == dict(info, uncompressed_size=16 * len(c), compressed_size=len(stream), lzf_tokens=tok, segments=seg)
        assert got[len(head):len(head) + 8] == struct.pack("<II", len(stream), 16 * len(c))
    else:
        assert len(got) == len(head) + 16 * len(c)
    ref, flag = M.read_reference(got)
    assert flag == 0 and np.array_equal(ref.view(np.uint32), c.view(np.uint32))
    rc, out, linfo, msg = M.hc_load(got, chunk=64)
    assert rc == 0, msg
    assert np.array_equal(out.view(np.uint32), c.view(np.uint32))


def test_unknown_mode_and_capacity():
    L = E.hostcheck()
    import ctypes
    c = np.ones((3, 4), np.float32)
    n, info = ctypes.c_size_t(0), E.FormatInfo()
    assert L.erasor_hostcheck_pcd_format_file(c.ctypes.data_as(ctypes.c_void_p), 3, 3, None, 0, ctypes.byref(n), ctypes.byref(info)) == -1
    assert L.erasor_hostcheck_pcd_format_file(c.ctypes.data_as(ctypes.c_void_p), 3, 1, None, 0, ctypes.byref(n), ctypes.byref(info)) == 0
    buf = np.zeros(n.value - 1, np.uint8)
    assert L.erasor_hostcheck_pcd_format_file(c.ctypes.data_as(ctypes.c_void_p), 3, 1, buf.ctypes.data_as(ctypes.c_void_p), len(buf),
                                              ctypes.byref(n), ctypes.byref(info)) == -4


def test_uint32_size_limit_edges():
    top = 0xFFFFFFFF
    assert E.hc_sizes_fit(0, 0) == 0
    assert E.hc_sizes_fit(16 * (top // 16), top) == 0
    assert E.hc_sizes_fit(top, top) == 0
    assert E.hc_sizes_fit(top + 1, 0) == -5
    assert E.hc_sizes_fit(16 * (top // 16 + 1), 0) == -5
    assert E.hc_sizes_fit(16, top + 1) == -5
    assert top // 16 == 268435455                              # the most points a binary_compressed file can hold
