"""Writes tests/golden/node_tiny_lz4.bag: tests/golden/node_tiny.bag with both chunks stored as LZ4 frames, assembled with explicit
struct.pack calls and an encoder of its own, independently of tests/lz4_model.py, so that one misreading of the LZ4 frame format
cannot pass both the fixture and the model.  The frames are hand-built rather than taken from liblz4, so the file does not depend
on which liblz4 (if any) the generating machine has.

  chunk 1: three blocks of one frame (block max 64 KB, short non-final blocks): a compressed block, a stored block, a compressed
           block; block checksums; the content checksum
  chunk 2: one compressed block; the content size field; the content checksum
The encoder emits a match only for a run of one repeated byte (offset 1, length 4 or more); everything else is literals.  Every
other byte of the file is node_tiny.bag's, except the chunk records, the chunk-info chunk_pos fields and the bag header's
index_pos.  Run with python3 to rewrite the file.
"""
import os
import struct

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "node_tiny.bag")
PATH = os.path.join(HERE, "node_tiny_lz4.bag")


def xxh32(data, seed=0):
    p1, p2, p3, p4, p5, m = 0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F, 0x165667B1, 0xFFFFFFFF
    rot = lambda x, r: ((x << r) | (x >> (32 - r))) & m
    n, i = len(data), 0
    if n >= 16:
        acc = [(seed + p1 + p2) & m, (seed + p2) & m, seed, (seed - p1) & m]
        while n - i >= 16:
            for lane in range(4):
                (w,) = struct.unpack_from("<I", data, i + 4 * lane)
                acc[lane] = rot((acc[lane] + w * p2) & m, 13) * p1 & m
            i += 16
        h = (rot(acc[0], 1) + rot(acc[1], 7) + rot(acc[2], 12) + rot(acc[3], 18)) & m
    else:
        h = (seed + p5) & m
    h = (h + n) & m
    while n - i >= 4:
        (w,) = struct.unpack_from("<I", data, i)
        h = rot((h + w * p3) & m, 17) * p4 & m
        i += 4
    for b in data[i:]:
        h = rot((h + b * p5) & m, 11) * p1 & m
    h = ((h ^ (h >> 15)) * p2) & m
    h = ((h ^ (h >> 13)) * p3) & m
    return h ^ (h >> 16)


def length_bytes(v):
    """the extension bytes of a length field that overflowed its nibble by v"""
    return b"\xff" * (v // 255) + bytes([v % 255])


def token(lit, run):
    """literals lit, then (run > 0) a match of run bytes at offset 1"""
    t = (min(len(lit), 15) << 4) | (min(run - 4, 15) if run else 0)
    out = bytes([t]) + (length_bytes(len(lit) - 15) if len(lit) >= 15 else b"") + lit
    if run:
        out += struct.pack("<H", 1) + (length_bytes(run - 19) if run >= 19 else b"")
    return out


def encode(data):
    """a block: byte runs of 5 or more become (1 literal, offset-1 match); nothing within the last 12 bytes is matched"""
    out, start, i, n = b"", 0, 0, len(data)
    while i < n - 12:
        j = i + 1
        while j < n - 5 and data[j] == data[i]:
            j += 1
        if j - i >= 5:
            out += token(data[start:i + 1], j - i - 1)
            start = i = j
        else:
            i += 1
    return out + token(data[start:], 0)


def frame(parts, block_sums, content_size):
    """parts: (bytes, stored?) per block"""
    flg = 0x40 | 0x20 | 0x04 | (0x10 if block_sums else 0) | (0x08 if content_size else 0)
    content = b"".join(p for p, _ in parts)
    desc = bytes([flg, 0x40]) + (struct.pack("<Q", len(content)) if content_size else b"")
    out = struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32(desc) >> 8) & 0xFF])
    for p, stored in parts:
        body = p if stored else encode(p)
        out += struct.pack("<I", len(body) | (0x80000000 if stored else 0)) + body
        if block_sums:
            out += struct.pack("<I", xxh32(body))
    return out + struct.pack("<I", 0) + struct.pack("<I", xxh32(content))


def field(name, value):
    return struct.pack("<I", len(name) + 1 + len(value)) + name + b"=" + value


def build():
    src = open(SRC, "rb").read()
    out, pos, chunk_no, moved = [src[:13]], 13, 0, {}
    while pos < len(src):
        (hl,) = struct.unpack_from("<I", src, pos)
        (dl,) = struct.unpack_from("<I", src, pos + 4 + hl)
        end = pos + 8 + hl + dl
        rec = src[pos:end]
        if b"op=\x05" in src[pos + 4:pos + 4 + hl]:
            data = src[pos + 8 + hl:end]
            if chunk_no == 0:
                a, b = len(data) // 3, 2 * len(data) // 3
                f = frame([(data[:a], False), (data[a:b], True), (data[b:], False)], block_sums=True, content_size=False)
            else:
                f = frame([(data, False)], block_sums=False, content_size=True)
            h = field(b"op", b"\x05") + field(b"compression", b"lz4") + field(b"size", struct.pack("<I", len(data)))
            moved[pos] = sum(len(x) for x in out)
            rec = struct.pack("<I", len(h)) + h + struct.pack("<I", len(f)) + f
            chunk_no += 1
        out.append(rec)
        pos = end
    b = bytearray(b"".join(out))
    shift = len(b) - len(src)
    for old, new in moved.items():                                  # chunk_pos of the chunk infos
        i = b.index(b"chunk_pos=" + struct.pack("<Q", old)) + 10
        b[i:i + 8] = struct.pack("<Q", new)
    i = b.index(b"index_pos=") + 10                                 # the index section moved by the shrink
    b[i:i + 8] = struct.pack("<Q", struct.unpack_from("<Q", b, i)[0] + shift)
    return bytes(b)


if __name__ == "__main__":
    with open(PATH, "wb") as f:
        f.write(build())
    print(PATH)
