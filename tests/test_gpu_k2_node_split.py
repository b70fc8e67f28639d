"""Node mode's scatter (K2) against the oracle on crafted map layouts that stress how it splits a chunk's VoI lists.

K1 leaves, per chunk, one dense VoI list per K1 warp (8 warps, or 32 for big bin tables): warp k's list sits at positions
[k * sub, k * sub + count_k) of the chunk.  K2 gives each of its 8 warps an even share of those lists taken in order, stages
the positions of the share's entries in flagged bins (kK2Stage = 512 per warp, device_types.h) and scatters from the stage;
a warp with more taken entries re-walks its share.  Each case lays out one chunk's map points (VoI points in chosen K1 ranges,
the rest far outside the VoI) so that:
- every VoI point lies in one K1 warp's range, the other lists empty;
- the lists have lengths that are not multiples of 32 (one of them empty);
- K2 warp 0's share is all flagged points and fills its stage exactly, or exceeds it by one;
and the flagged bins' points interleave in map order, so every flagged bin straddles several K2 shares.  The keep mask and
the per-node counters must equal the oracle's fetch_VoI + ERASOR bit for bit, through the 8-warp K1 form (seq_05) and the
32-warp one (40 x 360 bins).

These cases check results, not which path a warp took.  Any contiguous in-order split of the lists, and either side of the
staging switch, gives the same bytes by design, so a split that is consistent but uneven, or a switch that re-walks one entry
early, passes them.  What fails is a split or a stage that loses, repeats or reorders entries -- e.g. a switch that stages one
entry too many writes into the next warp's staging row in the stage_over case."""
import numpy as np
import pytest

import bin_cases as C
from erasor_b200 import params as P

pytestmark = pytest.mark.gpu

IDENTITY = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float64)
STAGE = 512          # kK2Stage
K2_WARPS = 8

# preset, K1 warps, K1 range per warp (points; a multiple of 32)
FORMS = {"k1_8_warps": ("seq_05", 8, 576), "k1_32_warps": ("synthetic_40x360", 32, 160)}


def _counts(k1w, sub, kind):
    """VoI points per K1 list, and how many of the first ones (in list order) are flagged-bin points."""
    if kind == "one_list":
        c = [0] * k1w
        c[k1w // 2 - 1] = 150 if k1w == 32 else 576
        return c, None
    if kind == "ragged":
        base = [37, 0, 101, 5, 250, 1, 77, 131]
        return [min(base[k % 8] + (k // 8) * 3, sub - 3) for k in range(k1w)], None
    if kind in ("stage_full", "stage_over"):
        per_share = STAGE + (kind == "stage_over")
        total = per_share * K2_WARPS
        c = [total // k1w + (k < total % k1w) for k in range(k1w)]
        return c, per_share              # K2 warp 0's share: all flagged
    raise ValueError(kind)


def _layout(p, k1w, sub, kind, seed):
    rng = np.random.default_rng(seed)
    counts, all_flagged_head = _counts(k1w, sub, kind)
    L = sum(counts)
    assert all(c <= sub for c in counts)
    # which VoI entries (list order = map order) are points of flagged bins: K2 warp 0's share entirely when staging is probed
    # (the later shares about a third, well under the stage), a random half otherwise
    is_f = rng.random(L) < (0.33 if all_flagged_head else 0.5)
    if all_flagged_head:
        is_f[:all_flagged_head] = True
    nF, nN = int(is_f.sum()), int((~is_f).sum())
    # flagged points: six tall bins with a flat query in each, shuffled together so each bin spans the whole list
    sizes = np.full(6, nF // 6)
    sizes[: nF % 6] += 1
    R = p.num_rings
    specs = [C.Bin(2 + 2 * i % (R - 4), 3 + 5 * i, int(n), "rough", 40) for i, n in enumerate(sizes)]
    fm, q = C.flagged_bins(p, specs, seed=seed)
    # other VoI points: two bins with no query points (never flagged)
    half = nN // 2
    nm, _ = C.flagged_bins(p, [C.Bin(R // 2, 1, half, "rough", 0), C.Bin(R // 2 + 1, 2, nN - half, "rough", 0)], seed=seed + 1)
    nm = rng.permutation(nm)
    voi = np.empty((L, 4), dtype=np.float32)
    voi[is_f], voi[~is_f] = fm, nm
    # the chunk: K1 warp k's range [k * sub, (k + 1) * sub), its first counts[k] points inside the VoI, the rest far outside
    n = k1w * sub
    far = np.stack([np.full(n, 3.0 * p.max_range), rng.uniform(-5, 5, n), np.zeros(n), np.full(n, 7.0)], 1).astype(np.float32)
    m = far.copy()
    at = 0
    for k, c in enumerate(counts):
        m[k * sub: k * sub + c] = voi[at: at + c]
        at += c
    return m, q, counts, is_f, len(specs)


@pytest.fixture(scope="module")
def capi():
    from erasor_b200 import capi as Cap
    return Cap


@pytest.mark.parametrize("form", sorted(FORMS))
@pytest.mark.parametrize("kind", ["one_list", "ragged", "stage_full", "stage_over"])
@pytest.mark.parametrize("version", [3, 2])
def test_node_scatter_split(capi, oracle_mod, form, kind, version):
    preset, k1w, sub = FORMS[form]
    p = P.preset(preset).replace(skip_voxelize=1, version=version)
    m, q, counts, is_f, n_flag_bins = _layout(p, k1w, sub, kind, seed=31 + k1w)
    L = sum(counts)
    shares = [(L * w) // K2_WARPS for w in range(K2_WARPS + 1)]
    taken = [int(is_f[shares[w]: shares[w + 1]].sum()) for w in range(K2_WARPS)]
    if kind == "stage_full":
        assert taken[0] == STAGE and max(taken[1:]) < STAGE
    elif kind == "stage_over":
        assert taken[0] == STAGE + 1 and max(taken[1:]) < STAGE
    elif kind == "one_list":
        assert sum(c > 0 for c in counts) == 1
    else:
        assert any(c % 32 for c in counts) and 0 in counts

    gm = capi.Map(m)
    h = capi.Handle(p)
    h.attach_map(gm)
    kg, fk = h.process_nodes(IDENTITY[None], q, np.array([0, len(q)], dtype=np.uint64), want_frame_keep=True)
    voi, idx = oracle_mod.fetch_voi(m, IDENTITY, p.max_range)
    assert len(voi) == L
    o = oracle_mod.Oracle(p)
    o.run(voi, q)
    assert len(o.planes()) == n_flag_bins, "every crafted tall bin is flagged"
    _, rej = o.cloud(o.MAP_REJECTED)
    ok = np.ones(len(m), dtype=np.uint8)
    ok[idx[rej]] = 0
    assert (ok == 0).any()
    assert np.array_equal(fk[0], ok) and np.array_equal(kg, ok)
    nv, nfl, nrj = h.node_stats()
    assert (nv[0], nfl[0], nrj[0]) == (L, n_flag_bins, int((ok == 0).sum()))
    h.attach_map(None)
    gm.close()
    h.close()
