"""CPU model of the work K1's node-mode map path does on a bench.py workload: no GPU needed.
usage: k1_row_stats.py [config] [frames] [sm_count]

Restates the chunking (erasor_capi.cu choose_chunk: one wave of sm_count * 4 CTAs), the split of a chunk over K1's 8 warps,
the VoI cut and the polar bin (in float64, so a point within rounding of a bin edge may land in the neighbouring bin), and
counts per step: map rows scanned (32 points), dense VoI rows formed, the share of dense rows whose lanes all hold one key,
the distinct keys per dense row (the not-binned key included), and how the dense rows spread over the CTAs."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402
from erasor_b200 import synth  # noqa: E402

config = sys.argv[1] if len(sys.argv) > 1 else "seq05"
frames = int(sys.argv[2]) if len(sys.argv) > 2 else bench.FRAMES_PER_PASS
sm_count = int(sys.argv[3]) if len(sys.argv) > 3 else 132

p, map_world, poses, qs = bench.load_workload(config, 0, 1, frames)
R, S = p.num_rings, p.num_sectors
B = R * S
NW = 32 if 4 * ((B + 1) + 2 * B) + 8 * ((R + 2) & ~1) > 56 * 1024 else 8       # kernels.h k1_warps
n_map = len(map_world)
F = len(poses)


def choose_chunk(sizes, slots):
    total = sum(sizes)
    count = lambda ch: sum((n + ch - 1) // ch for n in sizes)
    cap = 65536
    ch = max(total // slots + 1, max(2048, 5 * B))
    ch = min((ch + 127) & ~127, cap)
    if count(cap) <= slots:
        while ch < cap and count(ch) > slots:
            ch = min(cap, (ch + max(128, ch // 64) + 127) & ~127)
    else:
        ch = cap
    return ch


slots = sm_count * (1 if NW == 32 else 4)
CH = choose_chunk([n_map] * F + [len(q) for q in qs], slots)
chunk_starts = np.arange(0, n_map, CH)
xyz = map_world[:, :3].astype(np.float64)

scanned_rows = 0
row_keys = []            # distinct keys per dense row
cta_rows = []            # dense rows per map CTA
for f in range(F):
    px, py = float(np.float32(poses[f, 0])), float(np.float32(poses[f, 1]))
    in_voi = (xyz[:, 0] - px) ** 2 + (xyz[:, 1] - py) ** 2 < p.max_range ** 2
    T = np.linalg.inv(synth.pose_matrix(poses[f]))
    body = xyz @ T[:3, :3].T + T[:3, 3]
    r = np.hypot(body[:, 0], body[:, 1])
    th = np.arctan2(body[:, 1], body[:, 0])
    th = np.where(th < 0, th + 2 * np.pi, th)
    ring = np.minimum((r / (p.max_range / R)).astype(np.int64), R - 1)
    sector = np.minimum((th / (2 * np.pi / S)).astype(np.int64), S - 1)
    ok = (body[:, 2] > p.min_h) & (body[:, 2] < p.max_h) & (r <= p.max_range)
    key = np.where(ok, sector * R + ring, B)
    for c0 in chunk_starts:
        ln = min(CH, n_map - c0)
        sub = (((ln + NW - 1) // NW) + 31) & ~31
        rows_here = 0
        for w in range(NW):
            w0, w1 = min(ln, w * sub), min(ln, w * sub + sub)
            scanned_rows += (w1 - w0 + 31) // 32
            k = key[c0 + w0:c0 + w1][in_voi[c0 + w0:c0 + w1]]
            for j in range(0, len(k), 32):
                row_keys.append(len(np.unique(k[j:j + 32])))
            rows_here += (len(k) + 31) // 32
        cta_rows.append(rows_here)

row_keys = np.array(row_keys)
cta_rows = np.array(cta_rows)
print(f"{config}: {F} nodes x {n_map} map points, {R}x{S} bins, chunk {CH} points, {len(chunk_starts)} map chunks per node, {NW} warps per CTA")
print(f"per step: {scanned_rows} map rows scanned, {len(row_keys)} dense rows "
      f"({len(row_keys) / max(scanned_rows, 1):.3f} per scanned row)")
print(f"uniform dense rows (one key): {int((row_keys == 1).sum())} ({(row_keys == 1).mean():.3f}); "
      f"mixed rows: mean {row_keys[row_keys > 1].mean():.2f} keys, median {np.median(row_keys[row_keys > 1]):.0f}, "
      f"90th percentile {np.percentile(row_keys[row_keys > 1], 90):.0f}, max {row_keys.max()}")
print(f"dense rows per map CTA: min {cta_rows.min()}  median {np.median(cta_rows):.0f}  max {cta_rows.max()}  "
      f"(max / mean {cta_rows.max() / cta_rows.mean():.2f})")
