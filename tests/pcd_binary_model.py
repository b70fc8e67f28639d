"""Test-side reference for binary and binary_compressed PCD files (not part of the library):

- writers for both layouts: a numpy structured array (one record per point, any fields) -> the file's bytes, AoS for binary and
  one LZF-compressed block per non-"_" field for binary_compressed, as PCL 1.8's writers lay them out;
- a numpy structured-dtype reader for both, with PCL's PointXYZI rules (x y z intensity taken when F 4 COUNT 1; any other
  intensity, or none, is 0);
- a serial pure-Python LZF decoder (liblzf's lzf_d.c, restated);
- an independent greedy LZF encoder: a table keyed by the exact three bytes at a position holds the last position they were seen
  at, a match within 8192 bytes is extended to at most 264 bytes, literal runs are cut at 32, and only the position where a match
  starts enters the table (erasor_hostcheck_lzf_compress is the same encoder in C++, for large inputs);
- a token-level stream builder for adversarial and very large streams.
"""
import ctypes
import os
import struct

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTCHECK = os.path.join(ROOT, "erasor_b200", "_lib", "liberasor_b200_hostcheck.so")

NP_TYPES = {("F", 4): "<f4", ("F", 8): "<f8", ("U", 1): "u1", ("U", 2): "<u2", ("U", 4): "<u4", ("I", 1): "i1", ("I", 2): "<i2",
            ("I", 4): "<i4"}
BITS_TYPES = {("F", 4): "<u4", ("F", 8): "<u8"}      # the reader reads floats as their bit patterns

# (name, TYPE, SIZE, COUNT) per field
XYZI = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "F", 4, 1)]
# padding, non-float fields and COUNT > 1 around the four, point_step 50 (intensity at byte 15)
WIDE = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("_", "U", 1, 3), ("intensity", "F", 4, 1), ("ring", "U", 2, 1),
        ("t", "U", 4, 1), ("normal", "F", 4, 3), ("rgb", "U", 1, 4), ("_", "U", 1, 1), ("curvature", "F", 8, 1)]
XYZ = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1)]
U2_INTENSITY = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "U", 2, 1), ("ring", "U", 2, 1)]
F8_INTENSITY = [("z", "F", 4, 1), ("intensity", "F", 8, 1), ("x", "F", 4, 1), ("y", "F", 4, 1)]
COUNT2_INTENSITY = [("x", "F", 4, 1), ("y", "F", 4, 1), ("z", "F", 4, 1), ("intensity", "F", 4, 2), ("_", "I", 1, 1)]
LAYOUTS = {"xyzi": XYZI, "wide": WIDE, "xyz": XYZ, "u2_intensity": U2_INTENSITY, "f8_intensity": F8_INTENSITY,
           "count2_intensity": COUNT2_INTENSITY}


def _names(spec):
    out, k = [], 0
    for f in spec:
        if f[0] == "_":
            out.append(f"_pad{k}")
            k += 1
        else:
            out.append(f[0])
    return out


def record_dtype(spec, bits=False):
    """the packed numpy dtype of one point (AoS)"""
    formats = []
    for name, t, size, count in spec:
        fmt = (BITS_TYPES.get((t, size)) if bits else None) or NP_TYPES[(t, size)]
        formats.append(fmt if count == 1 else (fmt, (count,)))
    return np.dtype({"names": _names(spec), "formats": formats})


def point_step(spec, compressed=False):
    return sum(size * count for name, _, size, count in spec if not (compressed and name == "_"))


def random_records(spec, n, seed=0, xyzi=None):
    """n points of layout spec with seeded random bytes everywhere; x y z intensity from xyzi ([n, 4] float32) when given"""
    dt = record_dtype(spec)
    rng = np.random.default_rng(seed)
    rec = np.frombuffer(rng.integers(0, 256, n * dt.itemsize, dtype=np.uint8).tobytes(), dtype=dt).copy()
    for name, t, size, count in spec:
        if (t, size) in (("F", 4), ("F", 8)) and name != "_":
            rec[name] = rng.uniform(-100, 100, rec[name].shape)
    if xyzi is not None:
        xyzi = np.ascontiguousarray(xyzi, dtype=np.float32)
        for s, name in enumerate(("x", "y", "z", "intensity")):
            for f in spec:
                if f[0] == name and f[1:] == ("F", 4, 1):
                    rec[name] = xyzi[:, s]
    return rec


def header(spec, n, mode, width=None, height=None, comment="", counts=True):
    w = n if width is None else width
    h = 1 if height is None else height
    lines = ["# .PCD v0.7 - Point Cloud Data file format" + comment, "VERSION 0.7",
             "FIELDS " + " ".join(f[0] for f in spec), "SIZE " + " ".join(str(f[2]) for f in spec),
             "TYPE " + " ".join(f[1] for f in spec)]
    if counts:
        lines.append("COUNT " + " ".join(str(f[3]) for f in spec))
    lines += [f"WIDTH {w}", f"HEIGHT {h}", "VIEWPOINT 0 0 0 1 0 0 0", f"POINTS {n}", f"DATA {mode}"]
    return ("\n".join(lines) + "\n").encode()


def soa_bytes(spec, rec):
    """PCL 1.8 writeBinaryCompressed's buffer: one block per field not named "_", in header order"""
    names = _names(spec)
    return b"".join(np.ascontiguousarray(rec[nm]).tobytes() for nm, f in zip(names, spec) if f[0] != "_")


def write_pcd(spec, rec, mode, compress=None, **head):
    """the file's bytes; compress(bytes) -> LZF stream (default: the Python greedy encoder)"""
    n = len(rec)
    h = header(spec, n, mode, **head)
    if mode == "binary":
        return h + rec.tobytes()
    raw = soa_bytes(spec, rec)
    stream = (compress or lzf_compress)(raw)
    return h + struct.pack("<II", len(stream), len(raw)) + stream


def parse_header(data):
    """(dict of header keys -> token lists, data offset)"""
    keys, p = {}, 0
    while True:
        e = data.index(b"\n", p)
        tok = data[p:e].decode().split()
        p = e + 1
        if tok and not tok[0].startswith("#"):
            keys[tok[0]] = tok[1:]
            if tok[0] == "DATA":
                return keys, p


def read_reference(data, decompress=None):
    """float32 [n, 4] x y z intensity of a binary or binary_compressed file (numpy structured dtypes), and the intensity flag"""
    keys, off = parse_header(data)
    n = int(keys["POINTS"][0])
    spec = [(f, t, int(s), int(c)) for f, t, s, c in zip(keys["FIELDS"], keys["TYPE"], keys["SIZE"], keys.get("COUNT", ["1"] * len(keys["FIELDS"])))]
    names = _names(spec)
    out = np.zeros((n, 4), dtype=np.uint32)
    zero_flag = 0
    if keys["DATA"][0] == "binary":
        rec = np.frombuffer(data, dtype=record_dtype(spec, bits=True), count=n, offset=off)
        cols = {nm: rec[nm] for nm in names}
    else:
        csize, usize = struct.unpack_from("<II", data, off)
        raw = (decompress or lzf_decompress)(data[off + 8: off + 8 + csize], usize)
        cols, at = {}, 0
        for nm, (f, t, size, count) in zip(names, spec):
            if f == "_":
                continue
            fmt = BITS_TYPES.get((t, size)) or NP_TYPES[(t, size)]
            cols[nm] = np.frombuffer(raw, dtype=np.dtype(fmt), count=n * count, offset=at).reshape((n, count) if count > 1 else (n,))
            at += n * size * count
    for s, name in enumerate(("x", "y", "z", "intensity")):
        for nm, f in zip(names, spec):
            if f[0] == name:
                if f[1:] == ("F", 4, 1):
                    out[:, s] = cols[nm]
                else:
                    zero_flag = 1
                break
    return out.view(np.float32), zero_flag


# ---- LZF ------------------------------------------------------------------------------------------------------------------
class LzfError(ValueError):
    pass


def lzf_decompress(stream, usize):
    """liblzf's lzf_d.c, one token after the other; raises LzfError for every malformed case"""
    s, out, i = bytes(stream), bytearray(), 0
    while i < len(s):
        c = s[i]
        i += 1
        if c < 32:
            if i + c + 1 > len(s):
                raise LzfError("literal run past the end of the stream")
            if len(out) + c + 1 > usize:
                raise LzfError("output overrun")
            out += s[i:i + c + 1]
            i += c + 1
        else:
            ln = c >> 5
            if ln == 7:
                if i >= len(s):
                    raise LzfError("length byte past the end of the stream")
                ln += s[i]
                i += 1
            ln += 2
            if i >= len(s):
                raise LzfError("distance byte past the end of the stream")
            d = ((c & 31) << 8) + s[i] + 1
            i += 1
            if d > len(out):
                raise LzfError("reference before the output start")
            if len(out) + ln > usize:
                raise LzfError("output overrun")
            for _ in range(ln):
                out.append(out[-d])
    if len(out) != usize:
        raise LzfError("stream ends short of uncompressed_size")
    return bytes(out)


def lzf_compress(data):
    """the greedy encoder described in the module docstring"""
    data = bytes(data)
    n, out, last, lit, i = len(data), bytearray(), {}, 0, 0

    def flush(end):
        nonlocal lit
        while lit < end:
            m = min(32, end - lit)
            out.append(m - 1)
            out.extend(data[lit:lit + m])
            lit += m

    while i + 2 < n:
        key = data[i:i + 3]
        p = last.get(key)
        last[key] = i
        if p is not None and i - p <= 8192:
            ln = 3
            while ln < 264 and i + ln < n and data[p + ln] == data[i + ln]:
                ln += 1
            flush(i)
            out.extend(ref_token(ln, i - p))
            i += ln
            lit = i
        else:
            i += 1
    flush(n)
    return bytes(out)


def lit_token(b):
    assert 1 <= len(b) <= 32
    return bytes([len(b) - 1]) + bytes(b)


def ref_token(length, dist):
    """the bytes of a back-reference copying `length` (3..264) bytes from `dist` (1..8192) back"""
    assert 3 <= length <= 264 and 1 <= dist <= 8192
    l, o = length - 2, dist - 1
    if l < 7:
        return bytes([(l << 5) | (o >> 8), o & 255])
    return bytes([(7 << 5) | (o >> 8), l - 7, o & 255])


def build_stream(tokens):
    """tokens: ("lit", bytes) or ("ref", length, dist) -> (stream, decoded bytes)"""
    s, out = bytearray(), bytearray()
    for t in tokens:
        if t[0] == "lit":
            s += lit_token(t[1])
            out += t[1]
        else:
            s += ref_token(t[1], t[2])
            for _ in range(t[1]):
                out.append(out[-t[2]])
    return bytes(s), bytes(out)


def periodic_stream(prefix, usize):
    """A stream of usize bytes: `prefix` (1..32 bytes) as a literal, then maximal references at distance len(prefix), so the output
    repeats prefix.  Built with numpy, so streams near the uint32 limit take a moment."""
    d, n_full = len(prefix), (usize - len(prefix)) // 264
    rest = usize - len(prefix) - 264 * n_full
    tail = b""
    if rest:
        if rest < 3:                                 # fold the remainder into the last reference
            n_full -= 1
            rest += 264
            tail = ref_token(rest - 132, d) + ref_token(132, d)
        else:
            tail = ref_token(rest, d)
    body = np.tile(np.frombuffer(ref_token(264, d), dtype=np.uint8), n_full).tobytes()
    return lit_token(prefix) + body + tail


# ---- the host build (liberasor_b200_hostcheck.so) -------------------------------------------------------------------------
class LoadInfo(ctypes.Structure):
    """erasor_pcd_load_info_t"""
    _fields_ = [(name, ctypes.c_uint32) for name in ("data_mode", "fields", "intensity_zero_filled", "point_step")] + \
               [(name, ctypes.c_uint64) for name in ("width", "height", "points", "data_offset", "compressed_size", "uncompressed_size",
                                                     "lzf_tokens")] + \
               [("ascii", ctypes.c_uint64 * 5), ("ascii_fields", ctypes.c_uint32 * 2)]


_HC = None


def hostcheck():
    global _HC
    if _HC is None:
        L = ctypes.CDLL(HOSTCHECK)
        vp, u64, sz = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_size_t
        L.erasor_hostcheck_pcd_load.argtypes = [vp, sz, vp, sz, ctypes.POINTER(sz), ctypes.POINTER(LoadInfo), u64, ctypes.c_char_p, sz]
        L.erasor_hostcheck_lzf_decode.argtypes = [vp, u64, vp, u64, u64, u64, ctypes.POINTER(u64), ctypes.c_char_p, sz]
        L.erasor_hostcheck_lzf_serial.argtypes = [vp, u64, vp, u64]
        L.erasor_hostcheck_lzf_compress.argtypes = [vp, u64, vp, u64, ctypes.POINTER(u64)]
        _HC = L
    return _HC


def _ptr(b):
    a = np.frombuffer(b, dtype=np.uint8) if len(b) else np.zeros(1, np.uint8)
    return a, a.ctypes.data_as(ctypes.c_void_p)


def hc_load(data, chunk=4096):
    """(rc, float32 [n, 4] or None, info dict, message) of the host build of erasor_pcd_load"""
    L = hostcheck()
    keep, p = _ptr(data)
    n, info, err = ctypes.c_size_t(0), LoadInfo(), ctypes.create_string_buffer(512)
    rc = L.erasor_hostcheck_pcd_load(p, len(data), None, 0, ctypes.byref(n), ctypes.byref(info), chunk, err, 512)
    out = None
    if rc == 0:
        out = np.zeros((max(n.value, 1), 4), dtype=np.float32)
        rc = L.erasor_hostcheck_pcd_load(p, len(data), out.ctypes.data_as(ctypes.c_void_p), n.value, ctypes.byref(n), ctypes.byref(info), chunk, err, 512)
        out = out[:n.value]
    d = {name: int(getattr(info, name)) for name, _ in LoadInfo._fields_ if not name.startswith("ascii")}
    return rc, out, d, err.value.decode()


def hc_lzf_decode(stream, usize, chunk, keep=None):
    """(rc, decoded bytes, tokens, message) of stages A-C run serially"""
    L = hostcheck()
    keep_n = usize if keep is None else keep
    ks, ps = _ptr(stream)
    out = np.zeros(max(keep_n, 1), dtype=np.uint8)
    ntok, err = ctypes.c_uint64(0), ctypes.create_string_buffer(512)
    rc = L.erasor_hostcheck_lzf_decode(ps, len(stream), out.ctypes.data_as(ctypes.c_void_p), usize, keep_n, chunk, ctypes.byref(ntok), err, 512)
    return rc, out[:keep_n].tobytes(), ntok.value, err.value.decode()


def hc_lzf_serial(stream, usize):
    L = hostcheck()
    ks, ps = _ptr(stream)
    out = np.zeros(max(usize, 1), dtype=np.uint8)
    rc = L.erasor_hostcheck_lzf_serial(ps, len(stream), out.ctypes.data_as(ctypes.c_void_p), usize)
    return rc, out[:usize].tobytes()


def hc_lzf_compress(data):
    """the C++ greedy encoder (same output as lzf_compress)"""
    L = hostcheck()
    data = bytes(data)
    kd, pd = _ptr(data)
    cap = len(data) + len(data) // 32 + 16
    out = np.zeros(cap, dtype=np.uint8)
    n = ctypes.c_uint64(0)
    assert L.erasor_hostcheck_lzf_compress(pd, len(data), out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(n)) == 0
    return out[:n.value].tobytes()
