"""Wall time of mapgen on the device: the stepwise composition (NaiveMapGenerator + device_producer: per node a partition, two
affines and a voxelisation through erasor_updater_mapgen_node, cloud_curr copied back, the map concatenated in numpy) against the
resident generator (capi.MapGen: one launch per node, the map on the device), alternating in one run, on two workloads:

  seq05   the bench's seq 05 twin: 161 nodes of ~115 k points (synth.Scene(seed=5), 64 beams x 1800), normal mode
  long    a large-scale twin of 1600 nodes (the same scene driven 10 times over, 32 beams x 900): parking fires at nodes 2, 502,
          1002 and 1502

Both paths must give bit-identical saved clouds.  Prints ms per node (accumulation, device work finished), the final save time
(both saved clouds on the host), kernel launches and host synchronisations per node, the card and its power limit.
    python scripts/mapgen_timing.py [--reps 2]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from erasor_b200 import capi, mapgen, synth  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def workload(name):
    sc = synth.Scene(seed=5, length=160.0, n_nodes=161, n_dynamic=12)
    if name == "seq05":
        return [(k, sc.pose7(k), sc.scan(k, n_beams=64, n_az=1800, seed_offset=17)) for k in range(161)], 0.2, False
    scans = [sc.scan(k, n_beams=32, n_az=900, seed_offset=17) for k in range(161)]
    nodes = []
    for k in range(1600):
        lap, j = divmod(k, 161)
        p = np.array(sc.pose7(j), dtype=np.float64)
        p[1] += 200.0 * lap                     # each lap on its own stretch of the map
        nodes.append((k, p, scans[j]))
    return nodes, 0.2, True


def run_stepwise(nodes, leaf, large):
    from erasor_b200 import params
    # what mapgen.device_producer() builds, with the updater object in reach for its launch count
    upd = capi.Updater(params.updater_preset("seq_05"), params.preset("seq_05"), np.zeros((1, 4), dtype=np.float32))
    gen = mapgen.NaiveMapGenerator(lambda c, lf: upd.voxelize(c, lf), leafsize=leaf, is_large_scale=large,
                                   node_producer=lambda o, c: upd.mapgen_node(o, c))
    l0 = upd.kernel_launch_count()
    t0 = time.perf_counter()
    for _, odom, cloud in nodes:
        gen.accum_point_cloud(odom, cloud)          # synchronous: cloud_curr is on the host when it returns
    t1 = time.perf_counter()
    orig, v = gen.save_naive_map()
    t2 = time.perf_counter()
    launches = upd.kernel_launch_count() - l0
    upd.close()
    # erasor_updater_mapgen_node synchronises three times per node: the partition's count, the voxel count, the copy back
    return dict(ms_node=1e3 * (t1 - t0) / len(nodes), save_ms=1e3 * (t2 - t1), launches_node=launches / len(nodes), syncs_node=3.0), (orig, v)


def run_resident(nodes, leaf, large):
    gen = capi.MapGen(leaf, large)
    t0 = time.perf_counter()
    for _, odom, cloud in nodes:
        gen.accum(odom, cloud)
    gen.synchronize()
    t1 = time.perf_counter()
    c = gen.counters()
    orig, v = gen.save_naive_map()
    t2 = time.perf_counter()
    gen.close()
    return dict(ms_node=1e3 * (t1 - t0) / len(nodes), save_ms=1e3 * (t2 - t1), launches_node=c["launches"] / len(nodes),
                syncs_node=(c["host_syncs"] - 1) / len(nodes), regrowths=c["regrowths"]), (orig, v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--workloads", default="seq05,long")
    a = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit {pl}")
    for w in a.workloads.split(","):
        nodes, leaf, large = workload(w)
        npts = sum(len(c) for _, _, c in nodes)
        print(f"[{w}] {len(nodes)} nodes, {npts / len(nodes):.0f} points per scan, leafsize {leaf}, large-scale {large}")
        ref = None
        for rep in range(a.reps):
            for label, fn in (("stepwise", run_stepwise), ("resident", run_resident)):
                r, out = fn(nodes, leaf, large)
                if ref is None:
                    ref = out
                for x, y in zip(out, ref):
                    assert x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"{w}: {label} differs"
                extra = f", {r['regrowths']} regrowths" if "regrowths" in r else ""
                print(f"  rep {rep} {label:9s}: {r['ms_node']:8.3f} ms/node, save {r['save_ms']:8.1f} ms, "
                      f"{r['launches_node']:.3f} launches/node, {r['syncs_node']:.3f} host syncs/node{extra}")
        print(f"  saved clouds bit-identical: original {len(ref[0])} points, voxelised {len(ref[1])} points")


if __name__ == "__main__":
    main()
