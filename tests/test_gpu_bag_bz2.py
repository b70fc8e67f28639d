"""GPU: erasor/node bags with bz2 chunks (DESIGN.md section 12.2.2).  The bz2 twin of a bag must give the same index, node metadata
(except data_offset) and clouds as the uncompressed bag, bit for bit, and the device must give exactly what the host build
(liberasor_b200_hostcheck.so, the same functions run serially) gives; only chunks holding kept nodes are decoded; every fence gives
the host build's code and message and leaves the handle usable; an lz4-only bag is read as before; and the drivers and
pipeline.run_bag read a bz2 bag as they read its uncompressed twin."""
import os

import numpy as np
import pytest

import bag_model as M
import bz2_model as B
import lz4_model as Z
import test_bz2_bag_model as F
from erasor_b200 import capi, pipeline
from test_gpu_bag import bag_case, bits, pinned, rand_nodes, run, write_config, LIB  # noqa: F401
from test_gpu_bag_lz4 import check_twin

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def check(codec, plain, twin, sizes=(1, 20, None)):
    """check_twin (pageable and pinned files, host and device outputs, bag_load and bag_load_list), then the bz2 stats against the
    host build's"""
    check_twin(codec, plain, twin, sizes)
    st = codec.bag_bz2_stats()
    want = B.hc_stats()
    assert {k: st[k] for k in want} == want
    assert st["scratch_bytes"] > 0 and st["scan_ms"] > 0 and st["decode_ms"] > 0
    return st


def test_golden_fixture():
    import make_bag_bz2_golden as G
    data = open(G.PATH, "rb").read()
    rc, msg, hinfo, hnodes = M.hc_read(data)
    assert rc == 0, msg
    with capi.PcdCodec() as codec:
        for buf in (data, pinned(data)):
            assert codec.bag_index(buf) == hinfo
            xyzi, _ = codec.bag_load(device_out=True)
            assert np.array_equal(bits(xyzi), np.concatenate([n["cloud"] for n in hnodes]).view(np.uint32))
            st = codec.bag_bz2_stats()
            assert st["blocks"] >= 4 and st["streams_by_level"][0] == 1 and st["streams_by_level"][8] == 1


@pytest.mark.parametrize("level", range(1, 10))
def test_every_level(level):
    nodes = rand_nodes(10, 20000, seed=level, empty=(3,), nan=True)
    plain = M.write_bag(M.kitti2node_messages(nodes, layout="odd_step"), chunk_bytes=1 << 20)
    with capi.PcdCodec() as codec:
        st = check(codec, plain, B.bz2_twin(plain, level=level), sizes=(3, None))
        assert st["streams_by_level"][level - 1] == st["chunks"]


def test_planted_false_candidate():
    plain, twin, D = F.planted_bag()
    with capi.PcdCodec() as codec:
        st = check(codec, plain, twin, sizes=(None,))
        assert st["candidates"] > st["blocks"] == 3


def test_seq05_twin_with_a_large_cloud_and_a_mixed_lz4_bag():
    nodes = rand_nodes(161, 4000, seed=5, big=2_600_000)
    plain = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=768 * 1024)
    with capi.PcdCodec() as codec:
        st = check(codec, plain, B.bz2_twin(plain, level=9))
        assert st["blocks"] > st["decoded_chunks"] and st["decoded_bytes"] < len(plain)
        mixed = B.bz2_twin(Z.lz4_twin(plain, lambda d: Z.hc_frame(d, 6, True, True), which=lambda k: k % 2 == 0),
                           which=lambda k: k % 2 == 1, level=1)
        check(codec, plain, mixed, sizes=(7, None))
        assert codec.bag_lz4_stats()["decoded_chunks"] > 0


def test_only_chunks_with_kept_nodes_are_decoded():
    nodes = rand_nodes(9, 500, seed=2)
    plain = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=1)        # one message per chunk
    twin = B.bz2_twin(plain)
    with capi.PcdCodec() as codec:
        for keep_first, kept in ((False, range(5, 40, 4)), (True, range(1, 40, 4))):
            codec.bag_index(twin, keep_first=keep_first)
            st = codec.bag_bz2_stats()
            assert st["chunks"] == 40 and st["decoded_chunks"] == len(kept) == st["blocks"]


def test_lz4_only_bags_keep_their_stats():
    plain = M.write_bag(M.kitti2node_messages(rand_nodes(6, 3000, seed=4)), chunk_bytes=50000)
    twin = Z.lz4_twin(plain, lambda d: Z.hc_frame(d, 4, True, True))
    with capi.PcdCodec() as codec:
        codec.bag_index(twin)
        st = codec.bag_lz4_stats()
        assert M.hc_read(twin)[0] == 0 and {k: st[k] for k in Z.hc_stats()} == Z.hc_stats() and st["decode_ms"] > 0
        assert codec.bag_bz2_stats() == dict(codec.bag_bz2_stats(), chunks=0, decoded_chunks=0, blocks=0, candidates=0, scratch_bytes=0)


def test_fences_give_the_host_builds_code_and_message_and_leave_the_handle_usable():
    plain = F.base()
    twin = B.bz2_twin(plain)
    want = np.concatenate([w["cloud"] for w in M.read_bag(plain)])
    cases = {k: v[0] for k, v in F.fence_bags().items()}
    with capi.PcdCodec() as codec:
        for name, data in cases.items():
            rc, msg, _, _ = M.hc_read(data)
            assert rc != 0, name
            for buf in (data, pinned(data)):
                with pytest.raises(capi.ErasorError) as e:
                    codec.bag_index(buf)
                assert e.value.code == rc, (name, str(e.value), msg)
                assert str(e.value).endswith(msg), (name, str(e.value), msg)
                assert codec.bag_bz2_stats()["chunks"] == 0
            codec.bag_index(twin)
            xyzi, _ = codec.bag_load(device_out=True)
            assert np.array_equal(bits(xyzi), want.view(np.uint32)), name


# ---- drivers and the pipeline, end to end ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bz2_bag(bag_case):  # noqa: F811
    tmp, nodes, bag, initial = bag_case
    twin = tmp / "05_0_to_15_w_interval_1_node_bz2.bag"
    twin.write_bytes(B.bz2_twin(open(bag, "rb").read(), level=9))
    return tmp, bag, str(twin)


@pytest.mark.parametrize("frame_independent", [False, True])
def test_run_bag_equals_the_uncompressed_twin(bz2_bag, frame_independent):
    tmp, bag, twin = bz2_bag
    cfg = write_config(tmp, tmp / "map.pcd", tmp)
    want = pipeline.run_bag(bag, cfg, frame_independent=frame_independent)
    got = pipeline.run_bag(twin, cfg, frame_independent=frame_independent)
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], np.ndarray):
            assert want[k].dtype == got[k].dtype and np.array_equal(np.ascontiguousarray(got[k]).view(np.uint8), np.ascontiguousarray(want[k]).view(np.uint8)), k
        else:
            assert got[k] == want[k], k


def test_drivers_equal_the_uncompressed_twin(bz2_bag):
    tmp, bag, twin = bz2_bag
    out = {}
    for name, path in (("plain", bag), ("bz2", twin)):
        save = tmp / f"bz2_nodes_{name}"
        save.mkdir()
        run([os.path.join(LIB, "static_map_nodes_main"), write_config(tmp, tmp / "map.pcd", save), path, "0", "3"])
        out[name] = open(save / "05_result.pcd", "rb").read()
        mg = tmp / f"bz2_mapgen_{name}"
        mg.mkdir()
        run([os.path.join(LIB, "mapgen_main"), path, str(mg), "0.2"])
        out["mapgen_" + name] = [open(os.path.join(mg, p), "rb").read() for p in sorted(os.listdir(mg))]
        up = tmp / f"bz2_updater_{name}"
        up.mkdir()
        run([os.path.join(LIB, "offline_map_updater_main"), write_config(tmp, tmp / "map.pcd", up), path])
        out["updater_" + name] = open(up / "05_result.pcd", "rb").read()
    assert out["plain"] == out["bz2"]
    assert out["mapgen_plain"] == out["mapgen_bz2"] and out["mapgen_plain"]
    assert out["updater_plain"] == out["updater_bz2"]
