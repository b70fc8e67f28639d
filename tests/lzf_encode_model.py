"""Test-side restatement of the segmented LZF encoder behind erasor_pcd_format's binary_compressed mode (DESIGN.md section 12.3;
not part of the library), and ctypes access to its host build in liberasor_b200_hostcheck.so.

The rule, as lzf_encode.h states it:
- the input is cut into segments of SEG bytes (the last one may be shorter), each encoded on its own;
- cand(i) is the last earlier position of the segment whose three bytes have the same hash as bytes i..i+2 (every position with
  three bytes left counts, whatever the parse does); it counts when those three bytes are equal and i - cand(i) <= MAX_DIST.
  Here cand is found all at once: sort the positions by (hash, position), and each one's predecessor with the same hash is it;
- a match is extended to at most MAX_REF bytes and never past the segment's end;
- the parse is greedy from the segment's start (a match where one counts, else one literal), literal runs cut at 32; tokens are
  pcd_binary_model's lit_token / ref_token.
"""
import ctypes
import struct

import numpy as np

import pcd_binary_model as M

SEG = 16384
HASH_LOG = 13
MAX_REF = 264
MAX_DIST = 8192


def lzf_hash(b0, b1, b2):
    """the table key of three bytes (numpy arrays or ints)"""
    v = (np.asarray(b0, np.uint64) << 16) | (np.asarray(b1, np.uint64) << 8) | np.asarray(b2, np.uint64)
    return ((v * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - HASH_LOG)


def candidates(seg: bytes) -> np.ndarray:
    """cand(i) for every position of one segment with three bytes left, -1 where none counts"""
    a = np.frombuffer(seg, dtype=np.uint8)
    npos = max(len(a) - 2, 0)
    if not npos:
        return np.zeros(0, dtype=np.int64)
    h = lzf_hash(a[:npos], a[1:npos + 1], a[2:npos + 2])
    pos = np.arange(npos, dtype=np.int64)
    order = np.lexsort((pos, h))
    hs = h[order]
    same = hs[1:] == hs[:-1]
    prev = np.full(npos, -1, dtype=np.int64)
    prev[order[1:][same]] = order[:-1][same]
    c = np.maximum(prev, 0)
    ok = (prev >= 0) & (pos - prev <= MAX_DIST) & (a[c] == a[pos]) & (a[c + 1] == a[pos + 1]) & (a[c + 2] == a[pos + 2])
    return np.where(ok, prev, -1)


def _lits(b: bytes) -> bytes:
    return b"".join(M.lit_token(b[k:k + 32]) for k in range(0, len(b), 32))


def encode_segment(seg: bytes):
    """(token bytes, tokens) of one segment"""
    seg = bytes(seg)
    n = len(seg)
    cand = candidates(seg)
    starts = np.flatnonzero(cand >= 0)
    out, lit, tokens, k = bytearray(), 0, 0, 0
    while k < len(starts):
        q = int(starts[k])
        c = int(cand[q])
        most, ln = min(MAX_REF, n - q), 3
        while ln < most and seg[c + ln] == seg[q + ln]:
            ln += 1
        out += _lits(seg[lit:q])
        out += M.ref_token(ln, q - c)
        tokens += -(-(q - lit) // 32) + 1
        lit = q + ln
        k = int(np.searchsorted(starts, lit, side="left"))
    out += _lits(seg[lit:])
    tokens += -(-(n - lit) // 32)
    return bytes(out), tokens


def encode(data: bytes):
    """(stream, tokens, segments) of the whole input"""
    data = bytes(data)
    parts, tokens, segs = [], 0, 0
    for b in range(0, len(data), SEG):
        s, t = encode_segment(data[b:b + SEG])
        parts.append(s)
        tokens += t
        segs += 1
    return b"".join(parts), tokens, segs


def compress(data: bytes) -> bytes:
    """encode's stream alone (pcd_binary_model.write_pcd's compress=)"""
    return encode(data)[0]


def xyzi_records(xyzi):
    """float32 [n, 4] -> PointXYZI records with the very same bits (NaN payloads included)"""
    xyzi = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    return np.frombuffer(xyzi.tobytes(), dtype=M.record_dtype(M.XYZI)).copy()


def write_file(xyzi, mode: str, compress_fn=None) -> bytes:
    """the whole file erasor_pcd_format writes, through pcd_binary_model.write_pcd"""
    return M.write_pcd(M.XYZI, xyzi_records(xyzi), mode, compress=compress_fn or compress)


# ---- the host build -------------------------------------------------------------------------------------------------------
MODES = {"ascii": 0, "binary": 1, "binary_compressed": 2}


class FormatInfo(ctypes.Structure):
    """erasor_pcd_format_info_t"""
    _fields_ = [("data_mode", ctypes.c_uint32), ("segments", ctypes.c_uint32)] + \
               [(name, ctypes.c_uint64) for name in ("header_bytes", "uncompressed_size", "compressed_size", "lzf_tokens")]


_HC = None


def hostcheck():
    global _HC
    if _HC is None:
        L = M.hostcheck()
        vp, u64, sz = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_size_t
        L.erasor_hostcheck_lzf_encode.argtypes = [vp, u64, vp, u64, ctypes.POINTER(u64), ctypes.POINTER(u64), ctypes.POINTER(u64)]
        L.erasor_hostcheck_pcd_sizes_fit.argtypes = [u64, u64]
        L.erasor_hostcheck_pcd_format_file.argtypes = [vp, sz, ctypes.c_int, vp, sz, ctypes.POINTER(sz), ctypes.POINTER(FormatInfo)]
        _HC = L
    return _HC


def hc_encode(data: bytes):
    """(stream, tokens, segments) of the host build"""
    L = hostcheck()
    data = bytes(data)
    keep, p = M._ptr(data)
    cap = len(data) + len(data) // 16 + 64
    out = np.zeros(cap, dtype=np.uint8)
    clen, tok, seg = ctypes.c_uint64(0), ctypes.c_uint64(0), ctypes.c_uint64(0)
    assert L.erasor_hostcheck_lzf_encode(p, len(data), out.ctypes.data_as(ctypes.c_void_p), cap, ctypes.byref(clen), ctypes.byref(tok),
                                         ctypes.byref(seg)) == 0
    return out[:clen.value].tobytes(), tok.value, seg.value


def hc_sizes_fit(usize: int, csize: int) -> int:
    return hostcheck().erasor_hostcheck_pcd_sizes_fit(usize, csize)


def hc_format(xyzi, mode: str):
    """(rc, file bytes or None, info dict) of erasor_hostcheck_pcd_format_file"""
    L = hostcheck()
    c = np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4)
    src = c if len(c) else np.zeros((1, 4), np.float32)
    n, info = ctypes.c_size_t(0), FormatInfo()
    rc = L.erasor_hostcheck_pcd_format_file(src.ctypes.data_as(ctypes.c_void_p), len(c), MODES[mode], None, 0, ctypes.byref(n), ctypes.byref(info))
    data = None
    if rc == 0:
        out = np.zeros(max(n.value, 1), dtype=np.uint8)
        rc = L.erasor_hostcheck_pcd_format_file(src.ctypes.data_as(ctypes.c_void_p), len(c), MODES[mode], out.ctypes.data_as(ctypes.c_void_p),
                                                n.value, ctypes.byref(n), ctypes.byref(info))
        data = out[:n.value].tobytes()
    return rc, data, {name: int(getattr(info, name)) for name, _ in FormatInfo._fields_}


def soa(xyzi) -> bytes:
    """x[n] | y[n] | z[n] | intensity[n] of a float32 [n, 4] cloud"""
    return np.ascontiguousarray(np.ascontiguousarray(xyzi, dtype=np.float32).reshape(-1, 4).T).tobytes()


def stream_of(file: bytes) -> bytes:
    """the LZF stream of a binary_compressed file"""
    _, off = M.parse_header(file)
    csize, _ = struct.unpack_from("<II", file, off)
    return file[off + 8: off + 8 + csize]
