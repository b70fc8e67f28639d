"""GPU: the ASCII PCD codec on the device (capi.PcdCodec over erasor_pcd_parse_ascii / erasor_pcd_format_ascii) against the host
reader and writer of erasor_b200.evaluate.  Parsed clouds must equal read_pcd_ascii's float32 arrays bit for bit, formatted files
must equal write_pcd_ascii's bytes, and every file read_pcd_ascii rejects must be rejected with the line of the bad row."""
import ctypes

import numpy as np
import pytest

from erasor_b200 import capi
from erasor_b200 import evaluate as E
from erasor_b200 import synth
from test_pcd_codec_model import adversarial_tokens, format_values

pytestmark = pytest.mark.gpu
HEAD = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS {f}\nSIZE {s}\nTYPE {t}\nCOUNT {c}\nWIDTH {n}\nHEIGHT 1\n"
        "VIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA ascii\n")   # 11 lines: the first data row is line 12


def header(fields, n):
    k = len(fields)
    return HEAD.format(f=" ".join(fields), s=" ".join(["4"] * k), t=" ".join(["F"] * k), c=" ".join(["1"] * k), n=n)


@pytest.fixture(scope="module")
def codec():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    with capi.PcdCodec(0) as c:
        yield c


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check_file(codec, path):
    """device parse == read_pcd_ascii, through all four pointer-kind combinations"""
    import torch
    ref = E.read_pcd_ascii(path)
    raw = open(path, "rb").read()
    assert same_bits(codec.read(path), ref)
    assert same_bits(codec.parse(raw, device_out=True).cpu().numpy(), ref)
    dtext = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    assert same_bits(codec.parse(dtext).reshape(-1, 4), ref)
    assert same_bits(codec.parse(dtext, device_out=True).cpu().numpy(), ref)
    return ref


def check_format(codec, tmp_path, cloud):
    """device format == write_pcd_ascii's bytes (host and device input), and parse(format(x)) == read_pcd_ascii(write_pcd_ascii(x))"""
    import torch
    p = str(tmp_path / "w.pcd")
    E.write_pcd_ascii(p, cloud)
    want = open(p, "rb").read()
    got = codec.format(cloud)
    assert got == want
    assert codec.format(torch.from_numpy(np.ascontiguousarray(cloud, dtype=np.float32)).cuda()) == want
    assert same_bits(codec.parse(got), E.read_pcd_ascii(p))
    q = str(tmp_path / "d.pcd")
    codec.write(q, cloud)
    assert open(q, "rb").read() == want


def labelled_cloud(n, seed):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-80, 80, (n, 3)).astype(np.float32)
    xyz[:, 2] = rng.uniform(-3, 6, n)
    lab = rng.choice(np.array([0, 40, 44, 48, 50, 70, 252, 253, 254, 255, 256, 257, 258, 259], dtype=np.float32), n)
    return np.concatenate([xyz, lab[:, None]], axis=1).astype(np.float32)


def test_golden_seed41_pair(codec, tmp_path, oracle_mod):
    from test_eval_grid_model import seed41_pass
    gt, est = seed41_pass(oracle_mod)
    for name, c in (("gt", gt), ("est", est)):
        p = str(tmp_path / f"{name}.pcd")
        E.write_pcd_ascii(p, c)
        check_file(codec, p)
        check_format(codec, tmp_path, c)
    assert codec.last_info()["rows"] > 0


def test_driver_layout(codec, tmp_path):
    """the map and scans of the C++ driver's file layout"""
    sc = synth.Scene(seed=43, length=40.0, n_nodes=15, n_dynamic=6)
    kw = dict(n_beams=24, n_az=480)
    m = sc.build_map(list(range(15)), voxel=0.2, **kw)
    E.write_pcd_ascii(str(tmp_path / "dense_global_map.pcd"), m)
    check_file(codec, str(tmp_path / "dense_global_map.pcd"))
    for k in (0, 7, 14):
        s = sc.scan(k, seed_offset=9, **kw)
        p = str(tmp_path / f"{k:06d}.pcd")
        E.write_pcd_ascii(p, s)
        check_file(codec, p)
        check_format(codec, tmp_path, s)


def test_two_million_point_labelled_cloud(codec, tmp_path):
    c = labelled_cloud(2_000_000, 5)
    p = str(tmp_path / "big.pcd")
    E.write_pcd_ascii(p, c)
    check_file(codec, p)
    check_format(codec, tmp_path, c)


def test_adversarial_tokens_file(codec, tmp_path):
    toks = adversarial_tokens()
    toks += ["0"] * (-len(toks) % 4)
    rows = [" ".join(toks[i:i + 4]) for i in range(0, len(toks), 4)]
    p = str(tmp_path / "adv.pcd")
    with open(p, "w") as f:
        f.write(header(["x", "y", "z", "intensity"], len(rows)) + "\n".join(rows) + "\n")
    with np.errstate(over="ignore"):
        check_file(codec, p)
    assert codec.last_info()["slow_tokens"] > 100


def test_adversarial_values_format(codec, tmp_path):
    v = format_values(per_binade=32)
    v = np.concatenate([v, np.zeros(-len(v) % 4, dtype=np.float32)]).reshape(-1, 4)
    check_format(codec, tmp_path, v)


def test_layout_variants(codec, tmp_path):
    """CRLF, comments, blank and whitespace-only lines, reordered and extra fields, fewer rows than POINTS"""
    body = ["1.5 2 3 7", "# a comment line", "", "  \t ", "-4e-3\t5.25 6 8  # trailing comment", "\v7 8\f 9 1e1", "10 11 12 13"]
    cases = {
        "crlf": header(["x", "y", "z", "intensity"], 5).replace("\n", "\r\n") + "\r\n".join(body) + "\r\n",
        "reordered": header(["intensity", "z", "x", "y"], 5) + "\n".join(body) + "\n",
        "fewer_rows": header(["x", "y", "z", "intensity"], 9) + "\n".join(body) + "\n",
        "no_final_newline": header(["x", "y", "z", "intensity"], 5) + "\n".join(body),
        "stops_at_points": header(["x", "y", "z", "intensity"], 3) + "\n".join(body) + "\nnot numbers at all\n",
        "lone_cr": header(["x", "y", "z", "intensity"], 5).replace("\n", "\r") + "\r".join(body) + "\r",
        "mixed_ends": header(["x", "y", "z", "intensity"], 5) + "\r".join(body[:3]) + "\r\n" + "\n".join(body[3:]) + "\r",
    }
    extra = ["1 2 3 4 5 6", "# c", "7 8 9 10 11 12"]
    cases["extra_fields"] = header(["normal_x", "x", "y", "rgb", "z", "intensity"], 2) + "\n".join(extra) + "\n"
    for name, text in cases.items():
        p = str(tmp_path / f"{name}.pcd")
        with open(p, "w", newline="") as f:
            f.write(text)
        ref = check_file(codec, p)
        assert len(ref) == codec.last_info()["rows"], name
    assert codec.last_info()["points"] == 2


def test_missing_intensity(codec, tmp_path):
    p = str(tmp_path / "xyz.pcd")
    with open(p, "w") as f:
        f.write(header(["x", "y", "z"], 2) + "1 2 3\n4 5 6\n")
    with pytest.raises(KeyError):
        E.read_pcd_ascii(p)
    with pytest.raises(KeyError):
        codec.read(p)
    out = codec.read(p, require_intensity=False)
    assert same_bits(out, np.array([[1, 2, 3, 0], [4, 5, 6, 0]], dtype=np.float32))
    assert codec.last_info()["has_intensity"] == 0
    q = str(tmp_path / "noy.pcd")
    with open(q, "w") as f:
        f.write(header(["x", "z", "intensity"], 1) + "1 2 3\n")
    with pytest.raises(KeyError):
        codec.read(q, require_intensity=False)


@pytest.mark.parametrize("bad_row,line", [("1 2 3 0x10", 14), ("1 2 3", 14), ("1 2 3 4 5", 14), ("1 2 3 1d5", 14), ("1_0 2 3 4", 14),
                                          ("1 2 3 4 # ok\n--1 0 0 0", 15), (". 1 1 1", 14), ("1 2 e5 4", 14), ("1 2 3 4 #\n1e 2 3 4", 15)])
def test_invalid_rows(codec, tmp_path, bad_row, line):
    p = str(tmp_path / "bad.pcd")
    with open(p, "w") as f:
        f.write(header(["x", "y", "z", "intensity"], 6) + "0 0 0 0\n1 1 1 1\n" + bad_row + "\n2 2 2 2\nnan 1 1 1\n")
    with pytest.raises(ValueError):
        E.read_pcd_ascii(p)
    with pytest.raises(capi.ErasorError) as ei:
        codec.read(p)
    assert ei.value.code == capi.E_INVALID
    assert f"line {line}:" in str(ei.value)
    assert codec.last_info()["error_line"] == line


@pytest.mark.parametrize("bad_row", ["0x10 1 2 3 4 5", "1 2 3 1_0 4 5", "1 2 3 nan(1) 4 5", "e5 1 2 3 4 5"])
def test_invalid_token_in_a_column_that_is_not_kept(codec, tmp_path, bad_row):
    """normal_x and rgb are not kept, but every token is checked, as np.loadtxt checks every column"""
    p = str(tmp_path / "bad_extra.pcd")
    with open(p, "w") as f:
        f.write(header(["normal_x", "x", "y", "rgb", "z", "intensity"], 3) + "1 2 3 4 5 6\n# c\n" + bad_row + "\n7 8 9 10 11 12\n")
    with pytest.raises(ValueError):
        E.read_pcd_ascii(p)
    with pytest.raises(capi.ErasorError) as ei:
        codec.read(p)
    assert ei.value.code == capi.E_INVALID and "line 14:" in str(ei.value)


def test_invalid_lone_cr_row_reports_its_line(codec, tmp_path):
    """with lone '\r' line ends, the line numbers are Python's universal-newline lines, which read_pcd_ascii also sees"""
    p = str(tmp_path / "mac_bad.pcd")
    with open(p, "w", newline="") as f:
        f.write((header(["x", "y", "z", "intensity"], 4) + "0 0 0 0\n1 1 1 1\n1 2 3\n2 2 2 2\n").replace("\n", "\r"))
    with pytest.raises(ValueError):
        E.read_pcd_ascii(p)
    with pytest.raises(capi.ErasorError) as ei:
        codec.read(p)
    assert "line 14:" in str(ei.value) and codec.last_info()["error_line"] == 14


@pytest.mark.parametrize("text", [b"", b"not a pcd\n", b"FIELDS x y z intensity\nPOINTS 1\n", b"\r\n\r"])
def test_text_without_a_header_is_invalid_not_a_missing_field(codec, text):
    with pytest.raises(capi.ErasorError) as ei:
        codec.parse(text)
    assert ei.value.code == capi.E_INVALID and "DATA" in str(ei.value)
    assert codec.last_info()["header_lines"] == 0 and codec.last_info()["points"] == 0


def test_unsupported_headers(codec):
    binary = header(["x", "y", "z", "intensity"], 1).replace("DATA ascii", "DATA binary").encode() + b"\0" * 16
    with pytest.raises(capi.ErasorError) as ei:
        codec.parse(binary)
    assert ei.value.code == capi.E_UNSUPPORTED
    count2 = header(["x", "y", "z", "intensity"], 1).replace("COUNT 1 1 1 1", "COUNT 1 1 1 2").encode() + b"1 2 3 4 5\n"
    with pytest.raises(capi.ErasorError) as ei:
        codec.parse(count2)
    assert ei.value.code == capi.E_UNSUPPORTED


def test_device_parsed_map_feeds_the_evaluator(codec, tmp_path, oracle_mod):
    from test_eval_grid_model import seed41_pass
    gt, est = seed41_pass(oracle_mod)
    gp, ep_ = str(tmp_path / "gt.pcd"), str(tmp_path / "est.pcd")
    E.write_pcd_ascii(gp, gt)
    E.write_pcd_ascii(ep_, est)
    dg, de = codec.read(gp, device_out=True), codec.read(ep_, device_out=True)
    with capi.Evaluator(0) as ev:
        dev = ev.evaluate_ptr(dg.data_ptr(), len(dg), de.data_ptr(), len(de))
        host = ev.evaluate(E.read_pcd_ascii(gp), E.read_pcd_ascii(ep_))
    assert dev == host


def test_format_size_query_then_fetch(codec):
    """the raw ABI: a size query keeps the text for the following call with the same input; a short buffer is E_CAPACITY"""
    c = labelled_cloud(1000, 2)
    L = codec.L
    n = ctypes.c_size_t(0)
    assert L.erasor_pcd_format_ascii(codec.h, c.ctypes.data, len(c), capi.PTR_HOST, None, 0, capi.PTR_HOST, ctypes.byref(n)) == 0
    buf = np.empty(n.value, dtype=np.uint8)
    assert L.erasor_pcd_format_ascii(codec.h, c.ctypes.data, len(c), capi.PTR_HOST, buf.ctypes.data, 10, capi.PTR_HOST, ctypes.byref(n)) == capi.E_CAPACITY
    assert L.erasor_pcd_format_ascii(codec.h, c.ctypes.data, len(c), capi.PTR_HOST, buf.ctypes.data, len(buf), capi.PTR_HOST, ctypes.byref(n)) == 0
    assert buf.tobytes() == codec.format(c)


def test_text_above_two_gib_round_trips(codec):
    """a cloud whose text exceeds 2^31 bytes: device format -> device parse; sampled rows checked against Python's "%.8g" and
    float()"""
    import torch
    n = 37_000_000
    g = torch.Generator(device="cuda").manual_seed(3)
    x = -(1.0 + 9.0 * torch.rand((n, 4), device="cuda", generator=g)) * 1e-6            # "-1.2345678e-06": 14 bytes per value
    x = x.contiguous()
    L = codec.L
    size = ctypes.c_size_t(0)
    assert L.erasor_pcd_format_ascii(codec.h, x.data_ptr(), n, capi.PTR_DEVICE, None, 0, capi.PTR_DEVICE, ctypes.byref(size)) == 0
    assert size.value > 2 ** 31
    text = torch.empty(size.value, dtype=torch.uint8, device="cuda")
    assert L.erasor_pcd_format_ascii(codec.h, x.data_ptr(), n, capi.PTR_DEVICE, text.data_ptr(), size.value, capi.PTR_DEVICE,
                                     ctypes.byref(size)) == 0
    y = codec.parse(text, device_out=True)
    assert y.shape == (n, 4)
    del text
    rng = np.random.default_rng(0)
    idx = np.concatenate([rng.integers(0, n, 2000), [0, n - 1]])
    xs, ys = x[idx].cpu().numpy(), y[idx].cpu().numpy()
    want = np.array([[np.float32(float("%.8g" % float(v))) for v in row] for row in xs], dtype=np.float32)
    assert same_bits(ys, want)
