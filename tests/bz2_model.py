"""bzip2 streams for the bz2 bag tests (DESIGN.md section 12.2.2): a bag's bz2 twin, a bit-level reader and splicer of the stream
fields (to build every fence from a valid stream), a small bzip2 encoder whose block split, code lengths and symbols the caller can
dictate (every stream it writes is first checked to decode with Python's bz2, which is libbz2), and the host build's bz2 stats."""
import bz2
import ctypes
import struct

import bag_model as M
from lz4_model import top_records

BLOCK_MAGIC, EOS_MAGIC = 0x314159265359, 0x177245385090


# ---- bits --------------------------------------------------------------------------------------------------------------------------
def to_bits(data):
    return "".join(f"{b:08b}" for b in data)


def from_bits(bits):
    bits += "0" * (-len(bits) % 8)
    return bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))


def crc32(data, crc=0xFFFFFFFF):
    for b in data:
        crc ^= b << 24
        for _ in range(8):
            crc = ((crc << 1) ^ 0x04C11DB7 if crc & 0x80000000 else crc << 1) & 0xFFFFFFFF
    return crc


def block_crc(data):
    return crc32(data) ^ 0xFFFFFFFF


def stream_crc(block_crcs):
    c = 0
    for b in block_crcs:
        c = (((c << 1) | (c >> 31)) & 0xFFFFFFFF) ^ b
    return c


# ---- a parse of a valid stream's fields (bit offsets in the stream), to edit them ---------------------------------------------------
def fields(stream):
    """[{start, crc, rand, orig, map, groups, nsel, sel, lens, syms, end}] per block (bit offsets) and the end-of-stream bit, by
    reading a valid stream"""
    s = to_bits(stream)
    pos, blocks = 32, []
    while int(s[pos:pos + 48], 2) == BLOCK_MAGIC:
        b = dict(start=pos, crc=pos + 48, rand=pos + 80, orig=pos + 81, map=pos + 105)
        p = pos + 105
        used = s[p:p + 16]
        p += 16
        n_in_use = 0
        for i in range(16):
            if used[i] == "1":
                n_in_use += s[p:p + 16].count("1")
                p += 16
        b["groups"] = p
        ng = int(s[p:p + 3], 2)
        b["nsel"] = p + 3
        nsel = int(s[p + 3:p + 18], 2)
        p += 18
        b["sel"] = p
        for _ in range(nsel):
            while s[p] == "1":
                p += 1
            p += 1
        b["lens"] = p
        tables = []
        for _ in range(ng):
            cur = int(s[p:p + 5], 2)
            p += 5
            lens = []
            for _ in range(n_in_use + 2):
                while s[p] == "1":
                    cur += 1 if s[p + 1] == "0" else -1
                    p += 2
                p += 1
                lens.append(cur)
            tables.append(lens)
        b["syms"] = p
        # walk the symbols with the tables to the end-of-block symbol
        sels, q, mtf = [], b["sel"], list(range(ng))
        for _ in range(nsel):
            j = 0
            while s[q] == "1":
                j += 1
                q += 1
            q += 1
            v = mtf.pop(j)
            mtf.insert(0, v)
            sels.append(v)
        codes = [canonical(t) for t in tables]
        k, eob = 0, n_in_use + 1
        while True:
            code = codes[sels[k // 50]]
            L = 1
            while s[p:p + L] not in code:
                L += 1
            sym = code[s[p:p + L]]
            p += L
            k += 1
            if sym == eob:
                break
        b["end"] = p
        b["ng"], b["nsel_v"], b["n_in_use"] = ng, nsel, n_in_use
        blocks.append(b)
        pos = p
    assert int(s[pos:pos + 48], 2) == EOS_MAGIC
    return blocks, pos


def canonical(lens):
    """bit string -> symbol of the canonical code of lens"""
    code, out = 0, {}
    for L in range(1, 21):
        for sym, ln in enumerate(lens):
            if ln == L:
                out[format(code, f"0{L}b")] = sym
                code += 1
        code <<= 1
    return out


def splice(stream, at, nbits, value_bits):
    """the stream with bits [at, at + nbits) replaced by the bit string value_bits"""
    s = to_bits(stream)
    return from_bits(s[:at] + value_bits + s[at + nbits:])


def set_field(stream, at, nbits, value):
    return splice(stream, at, nbits, format(value, f"0{nbits}b"))


def flip_bit(stream, bit):
    b = bytearray(stream)
    b[bit // 8] ^= 0x80 >> (bit % 8)
    return bytes(b)


# ---- a dictated encoder -----------------------------------------------------------------------------------------------------------
def rle1(data):
    out, i = bytearray(), 0
    while i < len(data):
        r = 1
        while r < 255 and i + r < len(data) and data[i + r] == data[i]:
            r += 1
        if r >= 4:
            out += bytes([data[i]]) * 4 + bytes([r - 4])
        else:
            out += data[i:i + r]
        i += r
    return bytes(out)


def bwt(x):
    n = len(x)
    if len(set(x)) == 1:
        return bytes(x), 0
    if len(set(x[:-1])) == 1 and x[-1] > x[0]:                      # a^N b: the rotations sort in start order
        return bytes([x[-1]]) + bytes(x[:-1]), 0
    rots = sorted(range(n), key=lambda i: x[i:] + x[:i])
    return bytes(x[(i - 1) % n] for i in rots), rots.index(0)


def mtf_symbols(last, used):
    """RUNA/RUNB and MTF symbols of the last column, then the end-of-block symbol"""
    mtf, syms, run = list(used), [], 0

    def flush():
        nonlocal run
        while run > 0:
            run -= 1
            syms.append(run & 1)
            run >>= 1
    for b in last:
        j = mtf.index(b)
        if j == 0:
            run += 1
            continue
        flush()
        mtf.insert(0, mtf.pop(j))
        syms.append(j + 1)
    flush()
    syms.append(len(used) + 1)
    return syms


def encode_block(rle_in, lens=None, ng=2, code_of=None):
    """the bits of one block (magic to the end-of-block symbol) of RLE1 output rle_in; its CRC field is the text "{crc}".  lens:
    the code lengths of every group (default: a complete code of two lengths); code_of: symbol -> bit string overriding the
    canonical code"""
    last, orig = bwt(rle_in)
    used = sorted(set(rle_in))
    return block_of_symbols(mtf_symbols(last, used), used, orig, lens, ng, code_of)


def block_of_symbols(syms, used, orig, lens=None, ng=2, code_of=None):
    """the bits of one block of the symbols syms (RUNA 0, RUNB 1, MTF k + 1, the end-of-block symbol last) over the bytes used"""
    alpha = len(used) + 2
    if lens is None:                                                 # a complete code: 2^k - alpha lengths k - 1, the rest k
        k = (alpha - 1).bit_length()
        lens = [k - 1] * ((1 << k) - alpha) + [k] * (2 * alpha - (1 << k))
    inv = {v: k for k, v in canonical(lens).items()}
    code_of = code_of or inv
    out = format(BLOCK_MAGIC, "048b") + "{crc}" + "0" + format(orig, "024b")
    groups16 = [i for i in range(16) if any(16 * i <= b < 16 * i + 16 for b in used)]
    out += "".join("1" if i in groups16 else "0" for i in range(16))
    for i in groups16:
        out += "".join("1" if 16 * i + j in used else "0" for j in range(16))
    nsel = (len(syms) + 49) // 50
    out += format(ng, "03b") + format(nsel, "015b") + "0" * nsel
    for _ in range(ng):
        cur = lens[0]
        out += format(cur, "05b")
        for L in lens:
            while cur < L:
                out += "10"
                cur += 1
            while cur > L:
                out += "11"
                cur -= 1
            out += "0"
    out += "".join(code_of[s] for s in syms)
    return out


def encode(data, level=9, split=None, parts=None, check=True, **kw):
    """a bzip2 stream of data: blocks of the RLE1 output cut at `split` (a list of RLE1 lengths; default one block), or of the
    RLE1 outputs `parts` as given, each encode_block(**kw); unless check is False, first checked to decode with Python's bz2"""
    if parts is None:
        r = rle1(data)
        cuts = split or [len(r)]
        parts, a = [], 0
        for c in cuts:
            parts.append(r[a:a + c])
            a += c
        assert a == len(r), "the split must cover the RLE1 output"
    bits, crcs = "", []
    for p in parts:
        raw = unrle1(p)
        crcs.append(block_crc(raw))
        bits += encode_block(p, **kw).replace("{crc}", format(crcs[-1], "032b"))
    bits += format(EOS_MAGIC, "048b") + format(stream_crc(crcs), "032b")
    out = b"BZh" + bytes([ord("0") + level]) + from_bits(bits)
    if check:
        assert bz2.decompress(out) == data
    return out


def stream_of_blocks(blocks, level=9):
    """a stream of block bits as block_of_symbols writes them, their CRCs 0 (for fences that fail before the CRC)"""
    bits = "".join(b.replace("{crc}", "0" * 32) for b in blocks) + format(EOS_MAGIC, "048b") + "0" * 32
    return b"BZh" + bytes([ord("0") + level]) + from_bits(bits)


def unrle1(p):
    out, i = bytearray(), 0
    while i < len(p):
        r = 1
        while r < 4 and i + r < len(p) and p[i + r] == p[i]:
            r += 1
        if r == 4:
            out += p[i:i + 4] + (bytes([p[i]]) * p[i + 4] if i + 4 < len(p) else b"")
            i += 5
        else:
            out += p[i:i + r]
            i += r
    return bytes(out)


# ---- a bag's bz2 twin -----------------------------------------------------------------------------------------------------------
def bz2_twin(data, stream_of=None, which=None, level=9):
    """the bag with each chunk (k-th chunk: when which(k)) stored as stream_of(chunk data) (default bz2.compress at level) under
    compression bz2"""
    stream_of = stream_of or (lambda d: bz2.compress(d, level))
    out, moved, k, shift = [data[:13]], {}, 0, 0
    for pos, end, fs, d0, dl in top_records(data):
        op = fs["op"][1][0]
        rec = data[pos:end]
        if op == 5 and (which is None or which(k)):
            rec = M.record([("op", M.u8(5)), ("compression", b"bz2"), ("size", M.u32(dl))], stream_of(data[d0:d0 + dl]))
        if op == 5:
            moved[pos] = pos + shift
            k += 1
        out.append(rec)
        shift += len(rec) - (end - pos)
    b = bytearray(b"".join(out))
    for pos, end, fs, d0, dl in top_records(bytes(b)):
        op = fs["op"][1][0]
        if op == 6:
            at = fs["chunk_pos"][0]
            struct.pack_into("<Q", b, at, moved[struct.unpack_from("<Q", b, at)[0]])
        elif op == 3:
            at = fs["index_pos"][0]
            struct.pack_into("<Q", b, at, struct.unpack_from("<Q", b, at)[0] + shift)
    return bytes(b)


# ---- the host build's stats --------------------------------------------------------------------------------------------------------
class Bz2StatsC(ctypes.Structure):
    """erasor_bag_bz2_stats_t"""
    _fields_ = [(k, ctypes.c_uint64) for k in ("chunks", "decoded_chunks", "compressed_bytes", "decoded_bytes", "blocks", "candidates")] + \
               [("streams_by_level", ctypes.c_uint64 * 9), ("scratch_bytes", ctypes.c_uint64)] + \
               [(k, ctypes.c_double) for k in ("scan_ms", "decode_ms", "bwt_ms", "rle_ms")]


def hc_stats():
    """erasor_bag_bz2_stats of the host build's last index, without the times and the scratch"""
    st = Bz2StatsC()
    assert M.hostcheck().erasor_hostcheck_bag_bz2_stats(ctypes.byref(st)) == 0
    out = {k: int(getattr(st, k)) for k, _ in Bz2StatsC._fields_ if not k.endswith("_ms") and k not in ("scratch_bytes", "streams_by_level")}
    out["streams_by_level"] = [int(v) for v in st.streams_by_level]
    return out


# ---- decoding a block of symbols, and a block magic planted inside a block's Huffman bits -------------------------------------------
def decode_symbols(syms, used, orig):
    """the RLE1 output of a block of symbols (the model of the device's decode and inverse BWT)"""
    mtf, last, run, N = list(used), [], 0, 1
    for s in syms[:-1]:
        if s <= 1:
            run += (s + 1) * N
            N *= 2
            continue
        last += [mtf[0]] * run
        run, N = 0, 1
        mtf.insert(0, mtf.pop(s - 1))
        last.append(mtf[0])
    last += [mtf[0]] * run
    n = len(last)
    cf, T = {}, [0] * n
    acc = 0
    for c in sorted(set(last)):
        cf[c] = acc
        acc += last.count(c)
    for i, c in enumerate(last):
        T[cf[c]] = i
        cf[c] += 1
    out, p = [], T[orig]
    for _ in range(n):
        out.append(last[p])
        p = T[p]
    return bytes(out)


def planted():
    """(block bits with the text "{crc}" for its CRC, its data): one block whose Huffman bits hold the block magic.  With codes 0
    (RUNA), 10 (RUNB) and 110 (MTF 1) every bit string ending in 0 and free of 111 is a symbol sequence, and the magic followed by
    a 0 is one; 111 ends the block."""
    used, lens = [0x41, 0x42], [1, 2, 3, 3]
    bits, syms = format(BLOCK_MAGIC, "048b") + "0", [2]
    i = 0
    while i < len(bits):
        for code, sym in (("0", 0), ("10", 1), ("110", 2)):
            if bits.startswith(code, i):
                syms.append(sym)
                i += len(code)
                break
        else:
            raise AssertionError("not a symbol sequence")
    syms += [2, 2, 3]
    for orig in range(64):
        r = decode_symbols(syms, used, orig)
        if orig < len(r) and not (len(r) >= 4 and len(set(r[-4:])) == 1):
            break
    return block_of_symbols(syms, used, orig, lens), unrle1(r)


def with_planted(d, level=9):
    """the stream of chunk data d, which holds planted()'s data: a block before it, the planted block, a block after it"""
    bits, P = planted()
    a = d.index(P)
    blocks = [(encode_block(rle1(d[:a])), d[:a]), (bits, P), (encode_block(rle1(d[a + len(P):])), d[a + len(P):])]
    out, crcs = "", []
    for b, raw in blocks:
        if not raw:
            continue
        crcs.append(block_crc(raw))
        out += b.replace("{crc}", format(crcs[-1], "032b"))
    stream = b"BZh" + bytes([ord("0") + level]) + from_bits(out + format(EOS_MAGIC, "048b") + format(stream_crc(crcs), "032b"))
    assert bz2.decompress(stream) == d and to_bits(stream).count(format(BLOCK_MAGIC, "048b")) == len(crcs) + 1
    return stream
