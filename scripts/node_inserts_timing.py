"""Cost and quality of node-mode inserts (DESIGN.md section 8.4) and of their re-test pass (section 8.4.1) on the bench's seq-05
twin (20 nodes, one resident map).

  check    first, for version 3 with and without skip_voxelize: every node's inserts and offsets of one 20-node call against the
           oracle model (tests/node_inserts_model.py), bit for bit
  timing   node-mode scans/s with inserts off, on (pass 1) and of the re-test pass (pass 2, erasor_process_nodes_retest over
           the re-test map of pass 1's 20 nodes), the same workload (device-resident queries, asynchronous submissions dealt
           round-robin over the lanes as bench.py does), one lane and four lanes; the arms alternate within every repetition and
           each arm has its own handles, so all replay captured graphs; and the re-test map's build time (erasor_map_create_retest)
  quality  NN-matched PR/RR (erasor_b200/evaluate.py, GT = the labelled initial map) of node mode's final map without inserts
           (map[keep], as bench.py scores it) and with them (map[keep] ++ every node's inserts), for the bench preset and the
           configs.3_seqs_00_01_02_07 presets, and of the re-test pass's final map (M2[keep2]: the kept map and every node's
           inserts under pass 2's mask), next to the sequential updater on the same twin (161 nodes, every 8th processed)
Prints one JSON object; the card's name and power limit are read in the same run.
  usage: python scripts/node_inserts_timing.py [--reps 7] [--steps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from erasor_b200 import capi, evaluate, params, synth  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def check(p, map_world, poses, qs, qo, dq):
    from oracle import oracle_py
    import node_inserts_model as NI
    oracle_py.build()
    ref, ref_off, _ = NI.node_inserts(oracle_py, p, map_world, poses, qs)
    m, h = capi.Map(map_world), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    h.process_nodes_ptr(poses, dq.data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE)
    ins, off = h.node_inserts()
    ok = bool(np.array_equal(off, ref_off) and np.array_equal(ins.view(np.uint32), ref.view(np.uint32)))
    h.close(); m.close()
    if not ok:
        raise SystemExit(f"inserts differ from the oracle model (version {p.version}, skip_voxelize {p.skip_voxelize})")
    return int(ref_off[-1])


def pass1_map(p, map_world, poses, qo, dq):
    """the resident map after pass 1 with inserts on (all nodes in one call), its store filled"""
    m, h = capi.Map(map_world), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    h.process_nodes_ptr(poses, dq.data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE)
    m.append_inserts(h)
    h.close()
    return m


def retest_build(p, map_world, poses, qo, dq, reps):
    """erasor_map_create_retest's wall time (synchronous: compaction, the kept-count read, the store copy) on pass 1's map"""
    m = pass1_map(p, map_world, poses, qo, dq)
    ms = []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        r = m.create_retest()
        ms.append(1e3 * (time.perf_counter() - t0))
        size = r.size
        r.close()
    out = {"median_ms": round(float(np.median(ms[1:])), 3), "all_ms": [round(x, 3) for x in ms[1:]], "map_points": int(m.size),
           "kept_points": int(np.count_nonzero(m.get_keep())), "retest_map_points": int(size)}
    m.close()
    return out


def timing(p, map_world, poses, qo, dq, lanes, reps, steps):
    import torch
    m = capi.Map(map_world)
    src = pass1_map(p, map_world, poses, qo, dq[0])
    r = src.create_retest()
    arms = {}
    for name, on in (("off", False), ("on", True), ("retest", False)):
        hs = [capi.Handle(p) for _ in range(lanes)]
        for h in hs:
            h.attach_map(r if name == "retest" else m)
            h.set_node_inserts(on)
        arms[name] = hs
    F = len(qo) - 1

    def run(name, n):
        hs = arms[name]
        for i in range(n):
            if name == "retest":                              # (refused while pending: wait first, as process_nodes does inside)
                hs[i % len(hs)].wait()
                hs[i % len(hs)].process_nodes_retest_ptr(poses, dq[i % len(dq)].data_ptr(), qo, 0, 0.0, 0, capi.PTR_DEVICE, asynchronous=True)
            else:
                hs[i % len(hs)].process_nodes_ptr(poses, dq[i % len(dq)].data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE, asynchronous=True)
        for h in hs:
            h.wait()

    for name in arms:
        run(name, 2 * lanes)                                   # warm: buffers, captured graphs
    out = {k: [] for k in arms}
    for _ in range(reps):
        for name in arms:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name, steps * lanes)
            torch.cuda.synchronize()
            out[name].append(steps * lanes * F / (time.perf_counter() - t0))
    for hs in arms.values():
        for h in hs:
            h.close()
    r.close(); src.close(); m.close()
    return {k: {"median_scans_per_s": round(float(np.median(v))), "all": [round(x) for x in v]} for k, v in out.items()}


def node_quality(p, map_world, poses, qo, dq):
    m, h = capi.Map(map_world), capi.Handle(p)
    h.attach_map(m)
    h.set_node_inserts(True)
    h.process_nodes_ptr(poses, dq.data_ptr(), qo, 0.0, 0, 0, capi.PTR_DEVICE)
    ins, _ = h.node_inserts()
    keep = m.get_keep().astype(bool)
    # the re-test pass over the same nodes: M2 = map[keep] ++ inserts, node j seeing the inserts of the nodes before it
    m.append_inserts(h)
    r = m.create_retest()
    h.set_node_inserts(False)
    h.attach_map(r)
    h.process_nodes_retest_ptr(poses, dq.data_ptr(), qo, 0, 0.0, 0, capi.PTR_DEVICE)
    M2 = np.empty((r.size, 4), dtype=np.float32)
    capi._memcpy_from_device(M2, r.points_ptr)
    keep2 = r.get_keep().astype(bool)
    h.close(); r.close(); m.close()
    q = {}
    for name, est in (("without_inserts", map_world[keep]), ("with_inserts", np.concatenate([map_world[keep], ins])),
                      ("with_inserts_retest", M2[keep2])):
        res = evaluate.evaluate(map_world, est)
        q[name] = {"PR": round(res["PR"], 3), "RR": round(res["RR"], 3), "F1": round(res["F1"], 4)}
    q["inserted_points"] = int(len(ins))
    q["retest_rejected_inserts"] = int(np.count_nonzero(~keep2[int(keep.sum()):]))
    q["retest_rejected_kept_points"] = int(np.count_nonzero(~keep2[:int(keep.sum())]))
    return q


def sequential_quality(ep, map_world):
    up = params.updater_preset("seq_05")
    scene = synth.Scene(seed=5, length=160.0, n_nodes=161, n_dynamic=12)
    processed = [k for k in range(161) if (k + 1) % up.removal_interval == 0]
    d = bench._cache("seq05_twin_seed5_scans_ri8.npz", lambda: {f"s_{k}": scene.scan(k, seed_offset=17) for k in processed})
    empty = np.zeros((0, 4), dtype=np.float32)
    u = capi.Updater(up, ep, map_world)
    for k in range(161):
        u.process_node(k, scene.pose7(k), d[f"s_{k}"] if k in processed else empty)
    final = u.cloud(u.MAP_ARRANGED)
    u.close()
    r = evaluate.evaluate(map_world, final)
    return {"PR": round(r["PR"], 3), "RR": round(r["RR"], 3), "F1": round(r["F1"], 4)}


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    p0, map_world, poses, qs = bench.load_workload("seq05", 0, 1, bench.FRAMES_PER_PASS)
    qo = np.cumsum([0] + [len(q) for q in qs]).astype(np.uint64)
    Q = np.ascontiguousarray(np.concatenate(qs), dtype=np.float32)
    dq = [torch.from_numpy(Q).cuda() for _ in range(8)]
    res = {"card": card(), "nodes_per_call": len(qs), "map_points": int(len(map_world)), "timing": {}, "checked_inserted_points": {}}
    for skip in (1, 0):
        p = p0.replace(version=3, skip_voxelize=skip)
        key = f"v3_skip_voxelize_{skip}"
        res["checked_inserted_points"][key] = check(p, map_world, poses, qs, qo, dq[0])
        res.setdefault("retest_map_build", {})[key] = retest_build(p, map_world, poses, qo, dq[0], a.reps)
        for lanes in (1, 4):
            res["timing"][f"{key}_lanes_{lanes}"] = timing(p, map_world, poses, qo, dq, lanes, a.reps, a.steps)
    res["quality"] = {"seq_05 (bench)": node_quality(p0, map_world, poses, qo, dq[0])}
    res["quality"]["seq_05 (bench)"]["sequential_updater"] = sequential_quality(params.preset("seq_05"), map_world)
    for name in ("seq_00", "seq_01", "seq_02", "seq_07"):
        ep = params.preset(name)
        res["quality"][name] = node_quality(ep.replace(skip_voxelize=1), map_world, poses, qo, dq[0])
        res["quality"][name]["sequential_updater"] = sequential_quality(ep, map_world)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
