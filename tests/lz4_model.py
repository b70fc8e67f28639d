"""Test-side model of the LZ4 frame format as erasor_bag_index reads lz4 bag chunks (DESIGN.md section 12.2.1), written from the
public LZ4 frame and block format descriptions: XXH32, a block encoder whose parse the caller can dictate, a frame writer, a decoder,
and a writer of a bag's LZ4 twin.  A system liblz4, when ctypes can load it, cross-checks the model both ways.

lz4_twin(bag) rewrites a bag written by bag_model.write_bag (or any bag whose top-level records are those of rosbag) so that each
chunk's data is an LZ4 frame of the same bytes: the chunk record's compression becomes "lz4", its size stays the decoded length, and
the chunk positions in the chunk-info records and index_pos in the bag header are moved by the shrink.  The index data records'
offsets point into decoded data and stay valid.
"""
import ctypes
import ctypes.util
import struct

import numpy as np

import bag_model as M

MAGIC = 0x184D2204
P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
MASK = 0xFFFFFFFF


def _rotl(x, r): return ((x << r) | (x >> (32 - r))) & MASK


def xxh32(data, seed=0):
    data = bytes(data)
    n, i = len(data), 0
    if n >= 16:
        v = [(seed + P1 + P2) & MASK, (seed + P2) & MASK, seed & MASK, (seed - P1) & MASK]
        while i + 16 <= n:
            for k in range(4):
                v[k] = (_rotl((v[k] + struct.unpack_from("<I", data, i + 4 * k)[0] * P2) & MASK, 13) * P1) & MASK
            i += 16
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & MASK
    else:
        h = (seed + P5) & MASK
    h = (h + n) & MASK
    while i + 4 <= n:
        h = (_rotl((h + struct.unpack_from("<I", data, i)[0] * P3) & MASK, 17) * P4) & MASK
        i += 4
    while i < n:
        h = (_rotl((h + data[i] * P5) & MASK, 11) * P1) & MASK
        i += 1
    h ^= h >> 15
    h = (h * P2) & MASK
    h ^= h >> 13
    h = (h * P3) & MASK
    h ^= h >> 16
    return h


# ---- blocks ------------------------------------------------------------------------------------------------------------------
def _ext(v):
    out = b""
    while v >= 255:
        out += b"\xff"
        v -= 255
    return out + bytes([v])


def sequence(literals, off=0, mlen=0):
    """one sequence: the literals, then (off > 0) a match of mlen >= 4 bytes off back"""
    L = len(literals)
    tok = (min(L, 15) << 4) | (min(mlen - 4, 15) if off else 0)
    b = bytes([tok]) + (_ext(L - 15) if L >= 15 else b"") + bytes(literals)
    if off:
        b += struct.pack("<H", off) + (_ext(mlen - 4 - 15) if mlen - 4 >= 15 else b"")
    return b


def greedy_seqs(data):
    """a greedy parse [(lit, off, mlen)]: the last match starts 12 bytes or more before the end and the last 5 bytes are literals,
    as liblz4 requires; the final literals are implied"""
    n, seqs, last, i, anchor = len(data), [], {}, 0, 0
    while i + 12 < n + 0 and i < n - 12:
        key = data[i:i + 4]
        c = last.get(key)
        last[key] = i
        if c is not None and i - c <= 65535:
            m = 4
            while i + m < n - 5 and data[c + m] == data[i + m]:
                m += 1
            seqs.append((i - anchor, i - c, m))
            i += m
            anchor = i
        else:
            i += 1
    return seqs


def encode_block(data, seqs=None):
    """the block of data under the parse seqs [(literal count, offset, match length)] (greedy when None); the rest is the final
    literal run.  The parse is checked against data."""
    data = bytes(data)
    seqs = greedy_seqs(data) if seqs is None else seqs
    out, o = [], 0
    for lit, off, mlen in seqs:
        o += lit
        assert 1 <= off <= o and mlen >= 4
        for k in range(mlen):
            assert data[o + k] == data[o + k - off], "the parse does not reproduce the data"
        out.append(sequence(data[o - lit:o], off, mlen))
        o += mlen
    out.append(sequence(data[o:]))
    return b"".join(out)


def data_of_seqs(seqs, tail, rng):
    """the bytes a parse [(lit, off, mlen)] produces from random literals, then `tail` random literal bytes"""
    out = bytearray()
    for lit, off, mlen in seqs:
        out += rng.integers(0, 256, lit, dtype=np.uint8).tobytes()
        assert off <= len(out)
        for _ in range(mlen):
            out.append(out[-off])
    return bytes(out + rng.integers(0, 256, tail, dtype=np.uint8).tobytes())


# ---- frames ------------------------------------------------------------------------------------------------------------------
BLOCK_MAX = {4: 1 << 16, 5: 1 << 18, 6: 1 << 20, 7: 1 << 22}


def frame(blocks, bsid=4, block_sums=False, content_sum=True, content_size=None, flg=None, bd=None):
    """blocks: [(decoded bytes, how)] with how "lz" (greedy), "stored" or a parse for encode_block.  content_size: an int to write
    (None: none).  flg / bd override the descriptor bytes (for fences)."""
    f = 0x60 | (0x10 if block_sums else 0) | (0x04 if content_sum else 0) | (0x08 if content_size is not None else 0)
    f = f if flg is None else flg
    desc = bytes([f, (bsid << 4) if bd is None else bd]) + (struct.pack("<Q", content_size) if content_size is not None else b"")
    out = struct.pack("<I", MAGIC) + desc + bytes([(xxh32(desc) >> 8) & 0xFF])
    content = b""
    for data, how in blocks:
        content += data
        if how == "stored":
            body, size = data, len(data) | 0x80000000
        else:
            body = encode_block(data, None if how == "lz" else how)
            size = len(body)
            if how == "lz" and size >= len(data):                  # a greedy block that does not shrink is stored, as encoders do
                body, size = data, len(data) | 0x80000000
        out += struct.pack("<I", size) + body + (struct.pack("<I", xxh32(body)) if block_sums else b"")
    out += struct.pack("<I", 0)
    return out + (struct.pack("<I", xxh32(content)) if content_sum else b"")


def compress(data, bsid=4, block_sums=False, content_sum=True, stored=(), content_size=False):
    """data cut into block-max blocks, greedy; the blocks listed in stored are stored"""
    bm = BLOCK_MAX[bsid]
    parts = [data[a:a + bm] for a in range(0, len(data), bm)] or [b""]
    return frame([(p, "stored" if k in stored else "lz") for k, p in enumerate(parts) if p], bsid, block_sums, content_sum,
                 len(data) if content_size else None)


class Lz4Error(ValueError):
    pass


def decode_block(b, cap):
    out, i = bytearray(), 0
    while True:
        if i >= len(b):
            raise Lz4Error("the block ends inside a sequence")
        tok = b[i]
        i += 1
        L = tok >> 4
        if L == 15:
            while True:
                if i >= len(b):
                    raise Lz4Error("a length extension reads past the block")
                L += b[i]
                i += 1
                if b[i - 1] != 255:
                    break
        if L > len(b) - i:
            raise Lz4Error("a literal run reads past the block")
        out += b[i:i + L]
        i += L
        if i == len(b):
            break
        if len(b) - i < 2:
            raise Lz4Error("the block ends inside a sequence")
        off = b[i] | b[i + 1] << 8
        i += 2
        if off == 0 or off > len(out):
            raise Lz4Error("bad offset")
        M = tok & 15
        if M == 15:
            while True:
                if i >= len(b):
                    raise Lz4Error("a length extension reads past the block")
                M += b[i]
                i += 1
                if b[i - 1] != 255:
                    break
        for _ in range(M + 4):
            out.append(out[-off])
        if len(out) > cap:
            raise Lz4Error("output past the block max")
    if len(out) > cap:
        raise Lz4Error("output past the block max")
    return bytes(out)


def decode_frame(buf):
    buf = bytes(buf)
    if struct.unpack_from("<I", buf)[0] != MAGIC:
        raise Lz4Error("magic")
    flg, bd = buf[4], buf[5]
    p = 6 + (8 if flg & 0x08 else 0)
    if (xxh32(buf[4:p]) >> 8) & 0xFF != buf[p]:
        raise Lz4Error("header checksum")
    p += 1
    cap, out = BLOCK_MAX[(bd >> 4) & 7], b""
    while True:
        v = struct.unpack_from("<I", buf, p)[0]
        p += 4
        if v == 0:
            break
        n = v & 0x7FFFFFFF
        body = buf[p:p + n]
        p += n
        if flg & 0x10:
            if struct.unpack_from("<I", buf, p)[0] != xxh32(body):
                raise Lz4Error("block checksum")
            p += 4
        out += body if v >> 31 else decode_block(body, cap)
    if flg & 0x04:
        if struct.unpack_from("<I", buf, p)[0] != xxh32(out):
            raise Lz4Error("content checksum")
        p += 4
    if p != len(buf):
        raise Lz4Error("trailing bytes")
    return out


# ---- liblz4, when the system has it --------------------------------------------------------------------------------------------
class _FrameInfo(ctypes.Structure):
    _fields_ = [("blockSizeID", ctypes.c_int), ("blockMode", ctypes.c_int), ("contentChecksumFlag", ctypes.c_int), ("frameType", ctypes.c_int),
                ("contentSize", ctypes.c_ulonglong), ("dictID", ctypes.c_uint), ("blockChecksumFlag", ctypes.c_int)]


class _Prefs(ctypes.Structure):
    _fields_ = [("frameInfo", _FrameInfo), ("compressionLevel", ctypes.c_int), ("autoFlush", ctypes.c_uint), ("favorDecSpeed", ctypes.c_uint),
                ("reserved", ctypes.c_uint * 3)]


def liblz4():
    """the system liblz4 through ctypes, or None"""
    name = ctypes.util.find_library("lz4")
    if not name:
        return None
    try:
        L = ctypes.CDLL(name)
        L.LZ4F_compressFrameBound.restype = ctypes.c_size_t
        L.LZ4F_compressFrameBound.argtypes = [ctypes.c_size_t, ctypes.POINTER(_Prefs)]
        L.LZ4F_compressFrame.restype = ctypes.c_size_t
        L.LZ4F_compressFrame.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(_Prefs)]
        L.LZ4F_isError.argtypes = [ctypes.c_size_t]
        L.LZ4F_createDecompressionContext.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_uint]
        L.LZ4F_freeDecompressionContext.argtypes = [ctypes.c_void_p]
        L.LZ4F_decompress.restype = ctypes.c_size_t
        L.LZ4F_decompress.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t), ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t),
                                      ctypes.c_void_p]
        return L
    except (OSError, AttributeError):
        return None


def lib_compress(L, data, bsid=4, block_sums=False, content_sum=True):
    pr = _Prefs()
    pr.frameInfo.blockSizeID, pr.frameInfo.blockMode = bsid, 1
    pr.frameInfo.contentChecksumFlag, pr.frameInfo.blockChecksumFlag = int(content_sum), int(block_sums)
    cap = L.LZ4F_compressFrameBound(len(data), ctypes.byref(pr))
    out = ctypes.create_string_buffer(cap)
    n = L.LZ4F_compressFrame(out, cap, data, len(data), ctypes.byref(pr))
    assert not L.LZ4F_isError(n)
    return out.raw[:n]


def lib_decompress(L, buf, size):
    """liblz4's decode of the frame buf: (bytes, ok)"""
    ctx = ctypes.c_void_p()
    assert not L.LZ4F_isError(L.LZ4F_createDecompressionContext(ctypes.byref(ctx), 100))
    out = ctypes.create_string_buffer(size + 1)
    got, used, r = b"", 0, 1
    while r != 0 and not L.LZ4F_isError(r):                     # LZ4F_decompress may stop early; call until it reports the end
        dst, src = ctypes.c_size_t(size + 1), ctypes.c_size_t(len(buf) - used)
        r = L.LZ4F_decompress(ctx, out, ctypes.byref(dst), buf[used:], ctypes.byref(src), None)
        got += out.raw[:dst.value]
        used += src.value
        if not dst.value and not src.value:
            break
    L.LZ4F_freeDecompressionContext(ctx)
    return got, (not L.LZ4F_isError(r)) and r == 0 and used == len(buf)


# ---- the host build's greedy encoder, for inputs too large for Python ----------------------------------------------------------
def hc_frame(data, bsid=4, block_sums=False, content_sum=True):
    L = M.hostcheck()
    L.erasor_hostcheck_lz4_frame.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64,
                                             ctypes.POINTER(ctypes.c_uint64)]
    bm = BLOCK_MAX[bsid]
    cap = 15 + len(data) + (len(data) // bm + 1) * (8 + bm // 255 + 16)
    src = np.frombuffer(data, np.uint8) if len(data) else np.zeros(1, np.uint8)
    out = np.empty(cap, np.uint8)
    n = ctypes.c_uint64(0)
    assert L.erasor_hostcheck_lz4_frame(src.ctypes.data, len(data), bsid, int(block_sums), int(content_sum), out.ctypes.data, cap, ctypes.byref(n)) == 0
    return out[:n.value].tobytes()


class Lz4StatsC(ctypes.Structure):
    """erasor_bag_lz4_stats_t"""
    _fields_ = [(k, ctypes.c_uint64) for k in ("chunks", "decoded_chunks", "compressed_bytes", "decoded_bytes", "blocks", "stored_blocks",
                                               "block_checksums", "content_checksums")] + [("decode_ms", ctypes.c_double), ("checksum_ms", ctypes.c_double)]


def hc_stats():
    """erasor_bag_lz4_stats of the host build's last index, without the times"""
    st = Lz4StatsC()
    assert M.hostcheck().erasor_hostcheck_bag_lz4_stats(ctypes.byref(st)) == 0
    return {k: int(getattr(st, k)) for k, _ in Lz4StatsC._fields_ if not k.endswith("_ms")}


# ---- a bag's LZ4 twin --------------------------------------------------------------------------------------------------------
def top_records(data):
    """(pos, end, header fields {name: (value offset, bytes)}, data start, data length) of each top-level record"""
    out, a = [], 13
    mv = memoryview(data)
    while a < len(data):
        hl = struct.unpack_from("<I", data, a)[0]
        dl = struct.unpack_from("<I", data, a + 4 + hl)[0]
        out.append((a, a + 8 + hl + dl, M._fields(mv, a + 4, a + 4 + hl), a + 8 + hl, dl))
        a += 8 + hl + dl
    return out


def lz4_twin(data, frame_of=None, which=None):
    """the bag with each chunk (k-th chunk: when which(k)) stored as frame_of(chunk data) under compression lz4"""
    frame_of = frame_of or (lambda d: compress(d))
    out, moved, k = [data[:13]], {}, 0
    recs = top_records(data)
    shift = 0
    for pos, end, fs, d0, dl in recs:
        op = fs["op"][1][0]
        rec = data[pos:end]
        if op == 5 and (which is None or which(k)):
            body = data[d0:d0 + dl]
            rec = M.record([("op", M.u8(5)), ("compression", b"lz4"), ("size", M.u32(dl))], frame_of(body))
        if op == 5:
            moved[pos] = pos + shift
            k += 1
        out.append(rec)
        shift += len(rec) - (end - pos)
    b = bytearray(b"".join(out))
    # chunk positions in the chunk infos and index_pos in the bag header
    for pos, end, fs, d0, dl in top_records(bytes(b)):
        op = fs["op"][1][0]
        if op == 6:
            at = fs["chunk_pos"][0]
            struct.pack_into("<Q", b, at, moved[struct.unpack_from("<Q", b, at)[0]])
        elif op == 3:
            at = fs["index_pos"][0]
            old = struct.unpack_from("<Q", b, at)[0]
            struct.pack_into("<Q", b, at, old + shift)
    return bytes(b)
