"""CPU: the binary / binary_compressed PCD reader of erasor_pcd_load (erasor_b200/csrc/pcd_binary.h, compiled for the host into
liberasor_b200_hostcheck.so, its stages run serially) against the numpy reference and the serial LZF decoder of
tests/pcd_binary_model.py: PCL's header and field rules, and the parallel LZF decoder (speculative token discovery over chunks,
composition of the chunks' entry maps, token records, pointer jumping) on streams built to break it."""
import os
import struct

import numpy as np
import pytest

import pcd_binary_model as M

HERE = os.path.dirname(os.path.abspath(__file__))
OK, E_INVALID, E_UNSUPPORTED = 0, -1, -5
CHUNKS = [1, 2, 5, 7, 16, 33, 40, 64, 100, 4096]

pytestmark = pytest.mark.skipif(not os.path.exists(M.HOSTCHECK), reason="build with erasor_b200/csrc/build.sh")


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check_file(data, chunks=(4096, 7)):
    ref, flag = M.read_reference(data)
    for c in chunks:
        rc, got, info, msg = M.hc_load(data, chunk=c)
        assert rc == OK, msg
        assert same_bits(got, ref)
        assert info["intensity_zero_filled"] == flag
    return info


def check_stream(stream, want, chunks=CHUNKS):
    assert M.lzf_decompress(stream, len(want)) == want
    assert M.hc_lzf_serial(stream, len(want)) == (0, want)
    for c in chunks:
        rc, got, _, msg = M.hc_lzf_decode(stream, len(want), c)
        assert rc == OK, (c, msg)
        assert got == want, c


# ---- header and field rules ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["binary", "binary_compressed"])
@pytest.mark.parametrize("layout", sorted(M.LAYOUTS))
def test_layouts_equal_numpy_reference(layout, mode):
    spec = M.LAYOUTS[layout]
    rec = M.random_records(spec, 257, seed=len(layout))
    info = check_file(M.write_pcd(spec, rec, mode))
    assert info["data_mode"] == (1 if mode == "binary" else 2)
    assert info["point_step"] == M.point_step(spec, compressed=mode != "binary")
    takes_i = any(f[0] == "intensity" and f[1:] == ("F", 4, 1) for f in spec)
    has_i = any(f[0] == "intensity" for f in spec)
    assert info["fields"] == (15 if takes_i else 7)
    assert info["intensity_zero_filled"] == int(has_i and not takes_i)


def test_non_float_intensity_is_zero():
    for layout in ("u2_intensity", "f8_intensity", "count2_intensity", "xyz"):
        spec = M.LAYOUTS[layout]
        rec = M.random_records(spec, 40, seed=3)
        for mode in ("binary", "binary_compressed"):
            rc, got, info, _ = M.hc_load(M.write_pcd(spec, rec, mode))
            assert rc == OK and np.all(got[:, 3].view(np.uint32) == 0)
            assert info["intensity_zero_filled"] == int(layout != "xyz")


def test_padding_fields_are_skipped_in_both_modes():
    spec = M.WIDE
    rec = M.random_records(spec, 33, seed=9)
    assert M.point_step(spec) == 50 and M.point_step(spec, compressed=True) == 46
    for mode in ("binary", "binary_compressed"):
        ref, _ = M.read_reference(M.write_pcd(spec, rec, mode))
        assert same_bits(ref[:, 3], rec["intensity"].astype(np.float32))
        check_file(M.write_pcd(spec, rec, mode))


def test_organized_cloud_is_row_major():
    spec = M.WIDE
    rec = M.random_records(spec, 8 * 5, seed=4)
    for mode in ("binary", "binary_compressed"):
        info = check_file(M.write_pcd(spec, rec, mode, width=8, height=5))
        assert (info["width"], info["height"], info["points"]) == (8, 5, 40)


@pytest.mark.parametrize("residue", range(16))
def test_header_length_at_every_residue(residue):
    spec = M.WIDE
    rec = M.random_records(spec, 21, seed=residue)
    base = len(M.header(spec, 21, "binary"))
    pad = (residue - base) % 16
    for mode in ("binary", "binary_compressed"):
        data = M.write_pcd(spec, rec, mode, comment=" " + "p" * pad if pad else "")
        info = check_file(data)
        assert data[info["data_offset"] - 1:info["data_offset"]] == b"\n"


def test_header_offsets_cover_all_residues():
    spec = M.XYZI
    seen = set()
    for pad in range(16):
        data = M.write_pcd(spec, M.random_records(spec, 3), "binary", comment=" " + "p" * pad)
        seen.add(M.hc_load(data)[2]["data_offset"] % 16)
    assert seen == set(range(16))


def test_missing_count_defaults_to_one_and_missing_width_height():
    spec = M.XYZI
    rec = M.random_records(spec, 10, seed=1)
    check_file(M.write_pcd(spec, rec, "binary", counts=False))
    data = M.write_pcd(spec, rec, "binary").replace(b"WIDTH 10\nHEIGHT 1\n", b"")
    info = check_file(data)
    assert (info["width"], info["height"]) == (10, 1)


def test_empty_cloud_reads_no_data():
    for mode in ("binary", "binary_compressed"):
        data = M.header(M.XYZI, 0, mode)
        rc, got, info, _ = M.hc_load(data)
        assert rc == OK and got.shape == (0, 4)


def _mutate(data, old, new):
    assert old in data
    return data.replace(old, new, 1)


def rejections():
    spec = M.XYZI
    rec = M.random_records(spec, 12, seed=2)
    b = M.write_pcd(spec, rec, "binary")
    c = M.write_pcd(spec, rec, "binary_compressed")
    off = M.parse_header(c)[1]
    csize, usize = struct.unpack_from("<II", c, off)
    cases = {
        "size_list_short": (_mutate(b, b"SIZE 4 4 4 4", b"SIZE 4 4 4"), E_INVALID),
        "type_list_long": (_mutate(b, b"TYPE F F F F", b"TYPE F F F F F"), E_INVALID),
        "count_list_short": (_mutate(c, b"COUNT 1 1 1 1", b"COUNT 1 1 1"), E_INVALID),
        "width_height": (_mutate(b, b"WIDTH 12\nHEIGHT 1", b"WIDTH 5\nHEIGHT 2"), E_INVALID),
        "height_only": (_mutate(b, b"WIDTH 12\n", b""), E_INVALID),
        "count_zero": (_mutate(b, b"COUNT 1 1 1 1", b"COUNT 1 1 1 0"), E_INVALID),
        "no_x": (_mutate(b, b"FIELDS x y z intensity", b"FIELDS a y z intensity"), E_INVALID),
        "no_points": (_mutate(b, b"POINTS 12", b"POINTS x"), E_INVALID),
        "binary_truncated": (b[:-1], E_INVALID),
        "compressed_truncated": (c[:-1], E_INVALID),
        "compressed_no_sizes": (c[:off + 7], E_INVALID),
        "uncompressed_size_mismatch": (c[:off] + struct.pack("<II", csize, usize + 16) + c[off + 8:], E_INVALID),
        "f2": (_mutate(b, b"SIZE 4 4 4 4", b"SIZE 4 4 4 2"), E_UNSUPPORTED),
        "u8": (_mutate(_mutate(b, b"SIZE 4 4 4 4", b"SIZE 4 4 4 8"), b"TYPE F F F F", b"TYPE F F F U"), E_UNSUPPORTED),
        "type_x": (_mutate(b, b"TYPE F F F F", b"TYPE F F F X"), E_UNSUPPORTED),
        "x_f8": (_mutate(b, b"SIZE 4 4 4 4", b"SIZE 8 4 4 4"), E_UNSUPPORTED),
        "y_count2": (_mutate(b, b"COUNT 1 1 1 1", b"COUNT 1 2 1 1"), E_UNSUPPORTED),
        "z_u4": (_mutate(b, b"TYPE F F F F", b"TYPE F F U F"), E_UNSUPPORTED),
        "no_size_type": (_mutate(_mutate(b, b"SIZE 4 4 4 4\n", b""), b"TYPE F F F F\n", b""), E_UNSUPPORTED),
        "data_mode": (_mutate(b, b"DATA binary", b"DATA binary_lz4"), E_UNSUPPORTED),
    }
    return cases


@pytest.mark.parametrize("case", sorted(rejections()))
def test_header_rejections(case):
    data, code = rejections()[case]
    rc, _, _, msg = M.hc_load(data)
    assert rc == code, msg
    assert msg


def test_rejection_names_the_field():
    b = M.write_pcd(M.XYZI, M.random_records(M.XYZI, 4), "binary")
    rc, _, _, msg = M.hc_load(_mutate(b, b"TYPE F F F F", b"TYPE F F U F"))
    assert rc == E_UNSUPPORTED and "field z" in msg


def test_ascii_is_left_to_the_ascii_parser():
    data = M.header(M.XYZI, 1, "ascii") + b"1 2 3 4\n"
    assert M.hc_load(data)[0] == 1


# ---- LZF --------------------------------------------------------------------------------------------------------------------
def test_golden_fixture():
    """tests/golden/xyzi_2pts_binary_compressed.pcd: two points (1, 1, 2, 0) as PCL lays them out, SoA blocks x | y | z | intensity
    of 8 bytes each (32 bytes: 00 00 80 3F twice, twice; 00 00 00 40 twice; eight zeros).  After the header come
    compressed_size = 19 (13 00 00 00) and uncompressed_size = 32 (20 00 00 00), then six tokens:
      03 00 00 80 3F   literal run of 3 + 1 = 4 bytes: out[0:4] = 00 00 80 3F
      E0 03 03         back-reference, c >> 5 = 7 so L = 7 + 03 + 2 = 12, D = ((E0 & 31) << 8) + 03 + 1 = 4: out[4:16] repeats out[0:4]
      03 00 00 00 40   literal run of 4 bytes: out[16:20] = 00 00 00 40
      40 03            back-reference, L = 2 + 2 = 4, D = 3 + 1 = 4: out[20:24] = out[16:20]
      00 00            literal run of 1 byte: out[24] = 00
      A0 00            back-reference, L = 5 + 2 = 7, D = 1: out[25:32] = seven copies of out[24]"""
    data = open(os.path.join(HERE, "golden", "xyzi_2pts_binary_compressed.pcd"), "rb").read()
    want = np.array([[1, 1, 2, 0], [1, 1, 2, 0]], dtype=np.float32)
    for c in CHUNKS:
        rc, got, info, msg = M.hc_load(data, chunk=c)
        assert rc == OK, msg
        assert same_bits(got, want)
        assert (info["compressed_size"], info["uncompressed_size"], info["lzf_tokens"]) == (19, 32, 6)
    ref, _ = M.read_reference(data)
    assert same_bits(ref, want)


def test_encoder_round_trips_and_cpp_encoder_matches():
    rng = np.random.default_rng(7)
    inputs = [b"", b"a", b"ab", b"abc", b"aaaa", bytes(1000), rng.integers(0, 256, 3000, dtype=np.uint8).tobytes(),
              rng.integers(0, 4, 20000, dtype=np.uint8).tobytes(), (b"0123456789abcdef" * 700) + bytes(9000) + b"xyz" * 400,
              np.repeat(rng.integers(0, 256, 500, dtype=np.uint8), rng.integers(1, 300, 500)).tobytes()]
    for data in inputs:
        s = M.lzf_compress(data)
        assert M.lzf_decompress(s, len(data)) == data
        assert M.hc_lzf_compress(data) == s
        if data:
            check_stream(s, data, chunks=(1, 33, 64, 4096))


def _filler(n):
    """tokens of literals taking exactly n >= 2 stream bytes"""
    toks = []
    while n:
        size = min(n, 33) if n - min(n, 33) != 1 else 32
        toks.append(("lit", bytes(range(size - 1))))
        n -= size
    return toks


@pytest.mark.parametrize("phase", range(33))
def test_literal_run_straddles_chunk_boundary(phase):
    lit = bytes(range(100, 132))
    start = 64 - phase                               # the 33-byte token covers [start, start + 33), chunk boundary at 64
    toks = _filler(start) + [("lit", lit), ("ref", 10, 3)] + _filler(40)
    s, want = M.build_stream(toks)
    assert s[start] == 31
    check_stream(s, want, chunks=(64, 32, 31, 33, 65))


def test_reference_lengths_and_distances():
    rng = np.random.default_rng(3)
    toks = [("lit", rng.integers(0, 256, 32, dtype=np.uint8).tobytes()) for _ in range(260)]
    for ln in (3, 9, 10, 264):
        for d in (1, 2, 31, 8192):
            toks.append(("ref", ln, d))
            toks.append(("lit", b"z"))
    s, want = M.build_stream(toks)
    check_stream(s, want)


def test_overlapping_copies():
    toks = [("lit", b"abc"), ("ref", 264, 3), ("ref", 100, 2), ("ref", 7, 1), ("lit", b"q" * 32), ("ref", 50, 33)]
    s, want = M.build_stream(toks)
    assert want[3:267] == (b"abc" * 89)[:264]
    check_stream(s, want)


def test_entries_whose_chains_never_converge():
    # "00 AA" then "20 00" tokens (length 3, D = 1): walked from an odd offset the bytes parse as "00 20" one-byte literals, which
    # stay on the odd grid, so entries of different parity never meet inside any chunk
    toks = [("lit", b"\xaa")] + [("ref", 3, 1)] * 3000
    s, want = M.build_stream(toks)
    assert s[2:8] == b"\x20\x00" * 3
    check_stream(s, want)


def test_one_token_and_empty_streams():
    check_stream(*M.build_stream([("lit", b"x")]))
    check_stream(*M.build_stream([("lit", bytes(range(32)))]))
    for c in CHUNKS:
        assert M.hc_lzf_decode(b"", 0, c)[0] == OK
        assert M.hc_lzf_decode(b"", 5, c)[0] == E_INVALID


def test_periodic_stream_builder():
    for usize in (40, 35, 32 + 265, 32 + 266, 32 + 264 * 3 + 1, 10000):
        s = M.periodic_stream(bytes(range(32)), usize)
        want = (bytes(range(32)) * (usize // 32 + 1))[:usize]
        check_stream(s, want, chunks=(7, 4096))


def test_partial_materialisation_still_validates_the_whole_stream():
    s, want = M.build_stream([("lit", b"abcdefgh"), ("ref", 100, 8), ("lit", b"z")])
    rc, got, _, _ = M.hc_lzf_decode(s, len(want), 5, keep=20)
    assert rc == OK and got == want[:20]
    bad = s + M.ref_token(3, 5000)
    assert M.hc_lzf_decode(bad, len(want) + 3, 5, keep=20)[0] == E_INVALID


def malformed():
    s, want = M.build_stream([("lit", b"abcd"), ("ref", 20, 4)])
    return {
        "literal_past_end": (s + b"\x05\x01\x02", len(want) + 6),
        "length_byte_past_end": (s + b"\xe0", len(want) + 9),
        "distance_byte_past_end": (s + b"\x20", len(want) + 3),
        "reference_first": (M.ref_token(3, 1) + s, len(want) + 3),
        "reference_before_start": (M.lit_token(b"ab") + M.ref_token(3, 3), 5),
        "far_reference": (s + M.ref_token(5, 8192), len(want) + 5),
        "overrun": (s, len(want) - 1),
        "overrun_by_literal": (s + M.lit_token(b"xyz"), len(want) + 2),
        "short": (s, len(want) + 1),
        "empty_stream": (b"", 16),
    }


@pytest.mark.parametrize("case", sorted(malformed()))
def test_malformed_streams_are_invalid(case):
    stream, usize = malformed()[case]
    with pytest.raises(M.LzfError):
        M.lzf_decompress(stream, usize)
    assert M.hc_lzf_serial(stream, usize)[0] == -1
    for c in CHUNKS:
        rc, _, _, msg = M.hc_lzf_decode(stream, usize, c)
        assert rc == E_INVALID and msg.startswith("malformed LZF stream"), (c, msg)


@pytest.mark.parametrize("case", sorted(malformed()))
def test_malformed_streams_in_files_are_invalid(case):
    stream, usize = malformed()[case]
    n = -(-usize // 16)                               # a XYZI file whose uncompressed_size is 16 n: every stream stays malformed
    head = M.header(M.XYZI, n, "binary_compressed")
    data = head + struct.pack("<II", len(stream), 16 * n) + stream
    rc, _, _, msg = M.hc_load(data)
    assert rc == E_INVALID, msg
