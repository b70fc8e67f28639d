"""GPU: erasor/node bags with lz4 chunks (DESIGN.md section 12.2.1).  The LZ4 twin of a bag (tests/lz4_model.py) must give the same
index, node metadata (except data_offset) and clouds as the uncompressed bag, bit for bit, and the device must give exactly what the
host build (liberasor_b200_hostcheck.so, the same functions run serially) gives; only chunks holding kept nodes cross PCIe; every
fence leaves the handle usable; and the drivers and pipeline.run_bag read an LZ4 bag as they read its uncompressed twin."""
import os

import numpy as np
import pytest

import bag_model as M
import lz4_model as Z
import test_lz4_bag_model as F
from erasor_b200 import capi, pipeline
from test_gpu_bag import bag_case, bits, pinned, rand_nodes, run, write_config, LIB  # noqa: F401
from test_gpu_bag import check_loads

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def strip(layouts):
    return [dict(c, data_offset=0) for c in layouts]


def check_twin(codec, plain, twin, sizes=(1, 20, None)):
    """the twin against the uncompressed bag and the host build, from pageable and pinned memory, into host and device outputs"""
    want = M.read_bag(plain)
    rc, msg, hinfo, hnodes = M.hc_read(twin)
    assert rc == 0, msg
    info0 = codec.bag_index(plain)
    for buf in (twin, pinned(twin)):
        info = codec.bag_index(buf)
        assert info == info0 == hinfo
        seq, stamp, odom, clouds = codec.bag_meta()
        assert clouds == [n["layout"] for n in hnodes]                 # data_offset too: offsets in the decoded chunks
        assert strip(clouds) == strip([w["layout"] for w in want])
        for size in sizes:
            count = len(want) if size is None else min(size, len(want))
            first = (len(want) - count) // 2
            for dev in (False, True):
                xyzi, off = codec.bag_load(first, count, device_out=dev)
                ref = np.concatenate([w["cloud"] for w in want[first:first + count]]) if count else np.zeros((0, 4), np.float32)
                assert np.array_equal(bits(xyzi), ref.view(np.uint32))
        sel = list(range(len(want) - 1, -1, -3))
        xyzi, _ = codec.bag_load(nodes=sel, device_out=True)
        assert np.array_equal(bits(xyzi), np.concatenate([want[i]["cloud"] for i in sel]).view(np.uint32))
        assert [int(s) for s in seq] == [w["seq"] for w in want] and [int(s) for s in stamp] == [w["stamp_ns"] for w in want]
        assert np.array_equal(odom.view(np.uint64), np.stack([w["odom"] for w in want]).view(np.uint64))
    return codec.bag_lz4_stats()


def test_golden_fixture():
    plain = open(os.path.join(HERE, "golden", "node_tiny.bag"), "rb").read()
    twin = open(os.path.join(HERE, "golden", "node_tiny_lz4.bag"), "rb").read()
    with capi.PcdCodec() as codec:
        st = check_twin(codec, plain, twin)
        assert st["decoded_chunks"] == 2 and st["stored_blocks"] >= 1 and st["block_checksums"] >= 2 and st["content_checksums"] == 2


@pytest.mark.parametrize("bsid", [4, 5, 6, 7])
def test_block_sizes(bsid):
    nodes = rand_nodes(12, 30000, seed=bsid, empty=(4,), nan=True)
    plain = M.write_bag(M.kitti2node_messages(nodes, layout="odd_step"), chunk_bytes=3 << 20)
    twin = Z.lz4_twin(plain, lambda d: Z.hc_frame(d, bsid, block_sums=bsid % 2 == 0, content_sum=True))
    with capi.PcdCodec() as codec:
        st = check_twin(codec, plain, twin)
        assert st["blocks"] >= st["decoded_chunks"] and st["content_checksums"] == st["decoded_chunks"]


def test_mixed_chunks_and_repetitive_data():
    """every other chunk lz4; clouds of repeated patterns, so matches of offset 1..64 K with long overlaps reach the decoder"""
    rng = np.random.default_rng(3)
    nodes = []
    for k in range(8):
        period = [1, 2, 31, 32, 33, 4096, 65535, 7][k]
        pat = rng.integers(0, 1 << 30, (period + 3) // 4 + 1, dtype=np.uint32).view(np.uint8)[:period]
        raw = np.resize(pat, 16 * 20000)
        nodes.append((k, np.r_[np.zeros(3), [0, 0, 0, 1.0]], raw.view(np.float32).reshape(-1, 4).copy()))
    plain = M.write_bag(M.kitti2node_messages(nodes, layout="packed", debug=False), chunk_bytes=200000)
    twin = Z.lz4_twin(plain, lambda d: Z.hc_frame(d, 5, True, True), which=lambda k: k % 2 == 0)
    with capi.PcdCodec() as codec:
        check_twin(codec, plain, twin, sizes=(3, None))


def test_seq05_twin_with_a_large_cloud():
    nodes = rand_nodes(161, 4000, seed=5, big=2_600_000)
    plain = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=768 * 1024)
    twin = Z.lz4_twin(plain, lambda d: Z.hc_frame(d, 7, False, True))
    with capi.PcdCodec() as codec:
        st = check_twin(codec, plain, twin)
        assert st["decoded_bytes"] < len(plain) and st["decode_ms"] > 0


def test_only_chunks_with_kept_nodes_are_uploaded():
    nodes = rand_nodes(9, 500, seed=2)
    plain = M.write_bag(M.kitti2node_messages(nodes), chunk_bytes=1)        # one message per chunk
    frames = {}

    def frame_of(d):
        frames[len(frames)] = Z.compress(d, 4, False, True)
        return frames[len(frames) - 1]
    twin = Z.lz4_twin(plain, frame_of)
    with capi.PcdCodec() as codec:
        for keep_first, kept in ((False, range(5, 40, 4)), (True, range(1, 40, 4))):
            codec.bag_index(twin, keep_first=keep_first)
            st = codec.bag_lz4_stats()
            assert st["chunks"] == 40 and st["decoded_chunks"] == len(kept)
            assert st["compressed_bytes"] == sum(len(frames[k]) for k in kept)


def fence_cases():
    """name -> bag, every fence of tests/test_lz4_bag_model.py: frame and block rules, index entries, chunks without blocks, bad
    nodes in lz4 chunks, and bz2"""
    out = {f"frame_{k}": Z.lz4_twin(F.base(), v[0]) for k, v in F.FRAME_FENCES.items()}
    out.update({f"index_{k}": v[0] for k, v in F.index_fence_bags().items()})
    out.update({f"empty_{k}": v[0] for k, v in F.empty_chunk_bags().items()})
    out.update({f"node_{k}": t for k, t in enumerate(F.bad_node_bags()[1])})
    out["bz2"] = M.write_bag(M.kitti2node_messages(rand_nodes(2, 10, 2)), compression="bz2")
    return out


def test_fences_give_the_host_builds_code_and_message_and_leave_the_handle_usable():
    plain = F.base()
    twin = Z.lz4_twin(plain)
    want = np.concatenate([w["cloud"] for w in M.read_bag(plain)])
    cases = fence_cases()
    assert len(cases) >= 37
    with capi.PcdCodec() as codec:
        for name, data in cases.items():
            rc, msg, _, _ = M.hc_read(data)
            assert rc != 0, name
            for buf in (data, pinned(data)):
                with pytest.raises(capi.ErasorError) as e:
                    codec.bag_index(buf)
                assert e.value.code == rc, (name, str(e.value), msg)
                assert str(e.value).endswith(msg), (name, str(e.value), msg)   # the device's message is the host build's
                assert codec.bag_lz4_stats()["chunks"] == 0
                with pytest.raises(capi.ErasorError):
                    codec.bag_load(0, 1)
            codec.bag_index(twin)
            xyzi, _ = codec.bag_load(device_out=True)
            assert np.array_equal(bits(xyzi), want.view(np.uint32)), name


# ---- drivers and the pipeline, end to end ----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lz4_bag(bag_case):  # noqa: F811
    tmp, nodes, bag, initial = bag_case
    twin = tmp / "05_0_to_15_w_interval_1_node_lz4.bag"
    twin.write_bytes(Z.lz4_twin(open(bag, "rb").read(), lambda d: Z.hc_frame(d, 6, True, True)))
    return tmp, bag, str(twin)


@pytest.mark.parametrize("frame_independent", [False, True])
def test_run_bag_equals_the_uncompressed_twin(lz4_bag, frame_independent):
    tmp, bag, twin = lz4_bag
    cfg = write_config(tmp, tmp / "map.pcd", tmp)
    want = pipeline.run_bag(bag, cfg, frame_independent=frame_independent)
    got = pipeline.run_bag(twin, cfg, frame_independent=frame_independent)
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], np.ndarray):
            assert want[k].dtype == got[k].dtype and np.array_equal(np.ascontiguousarray(got[k]).view(np.uint8), np.ascontiguousarray(want[k]).view(np.uint8)), k
        else:
            assert got[k] == want[k], k


def test_static_map_nodes_main_equals_the_uncompressed_twin(lz4_bag):
    tmp, bag, twin = lz4_bag
    out = {}
    for name, path in (("plain", bag), ("lz4", twin)):
        save = tmp / f"nodes_{name}"
        save.mkdir()
        run([os.path.join(LIB, "static_map_nodes_main"), write_config(tmp, tmp / "map.pcd", save), path, "0", "3"])
        out[name] = open(save / "05_result.pcd", "rb").read()
    assert out["plain"] == out["lz4"]
