"""GPU tier: LocalMapping's device kernels on the inputs tests/test_local_mapping_windows.py builds, against the oracle bit for bit.

- k_tri_match + k_tri_rotation (ORBmatcher::SearchForTriangulation): every constructed case with bCoarse and check_orientation in
  {0, 1}; stereo, monocular and mixed flags; nq = 0, 1, 63, 64, 65, 513 (the TRI_QPB and warp boundaries) and ~1 000 against
  N2 = 1, 2, a keyframe and 16 384 rows; one keyframe against 10 and 20 neighbours in sequence on one handle with N2 growing and
  shrinking between calls (match12 and nmatches).
- k_distinctive (MapPoint::ComputeDistinctiveDescriptors): every observation-list size in one call of over 100 000 map points; a
  65 535-observation point (accepted) and a 65 536-observation one (refused, the handle still works).
- k_normal_depth (MapPoint::UpdateNormalAndDepth): trajectories 10 m, 500 m and 2 km from the origin on pyramids of (1.2, 8),
  (1.5, 5) and (2.0, 3) levels, n_points on and off multiples of 128, points without observations keeping the caller's values."""
import time

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, ComputeDistinctiveDescriptors, UpdateNormalAndDepth
from orb_slam3_detailed_comments_b200._native import OrbError
from test_local_mapping_windows import (PYRAMIDS, TRI_CASES, distinctive_lists, filler_lists, keyframes, normal_depth_case, oracle, pair,
                                        tri_case)

pytestmark = pytest.mark.gpu

Q_FIELDS = ("kp1", "desc1", "node1", "stereo1")
K2_FIELDS = ("kp2", "desc2", "node2", "valid2", "stereo2")


@pytest.fixture(scope="module")
def ex():
    e = ORBextractor(1200, 1.2, 8, 20, 7, max_width=752, max_height=480, max_batch=1)
    c = tri_case("plain")
    assert (e.GetScaleFactors().view(np.uint32) == c["sf"].view(np.uint32)).all()
    assert (e.GetScaleSigmaSquares().view(np.uint32) == c["s2"].view(np.uint32)).all()
    yield e
    e.close()


def check(ex, c, coarse, check_ori, what=""):
    got, nm = ORBmatcher(0.6, check_ori).SearchForTriangulation(ex, *[c[k] for k in Q_FIELDS], *[c[k] for k in K2_FIELDS], c["F12"], c["ep"],
                                                               bCoarse=coarse)
    ref, rnm = oracle(c, coarse, check_ori)
    bad = np.nonzero(got != ref)[0]
    assert nm == rnm and len(bad) == 0, (what, coarse, check_ori, nm, rnm, [(int(q), int(got[q]), int(ref[q])) for q in bad[:8]])
    return rnm


def resized(c, nq=None, n2=None, rng=None):
    """The pair with its first nq queries, and keyframe 2 cut or tiled (positions nudged per copy) to n2 rows."""
    c = dict(c)
    if nq is not None:
        for k in Q_FIELDS:
            c[k] = c[k][:nq]
    if n2 is not None:
        reps = -(-n2 // len(c["kp2"]))
        for k in K2_FIELDS:
            c[k] = np.concatenate([c[k]] * reps)[:n2].copy()
        if reps > 1:
            shift = (np.arange(n2) // len(c["kp2"]) % 4).astype(np.float32) * np.float32(0.25)
            c["kp2"]["x"] = c["kp2"]["x"] + shift
    return c


@pytest.mark.parametrize("name", TRI_CASES)
def test_triangulation_cases(ex, name):
    c = tri_case(name)
    total = 0
    for coarse in (0, 1):
        for check_ori in (0, 1):
            total += check(ex, c, coarse, check_ori, name)
    assert total > 0 or name == "den0"


@pytest.mark.parametrize("kind", ["stereo", "mono", "mixed"])
@pytest.mark.parametrize("nq", [0, 1, 63, 64, 65, 8 * 64 + 1, None])
def test_triangulation_sizes(ex, kind, nq):
    base = tri_case("mixed") if kind == "mixed" else pair(*keyframes(kind, 2, 11 if kind == "stereo" else 21)[:2])
    assert nq is None or len(base["src"]) >= nq
    ref_full, _ = oracle(base, False, False)
    for n2 in (1, 2, None, 16384):
        c = resized(base, nq, n2)
        if n2 in (1, 2):        # keyframe 2 reduced to rows the queries really match
            rows = np.unique(ref_full[ref_full >= 0])[:n2]
            for k in K2_FIELDS:
                c[k] = base[k][rows].copy()
        for coarse, check_ori in ((0, 0), (0, 1), (1, 1)):
            check(ex, c, coarse, check_ori, (kind, nq, n2))


@pytest.mark.parametrize("n_neighbours", [10, 20])
def test_keyframe_against_its_neighbours_in_sequence(ex, n_neighbours):
    """LocalMapping's loop: one keyframe against each covisible neighbour on one handle, keyframe 2's size changing every call."""
    kfs = keyframes("stereo", n_neighbours + 1, 11)
    sizes = [1200, 40, 16384, 3, 900, 9000, 1, 5000, 16384, 200, 2, 12000, 700, 16000, 64, 8000, 1500, 33, 16384, 10]
    matched = 0
    for j in range(1, n_neighbours + 1):
        c = pair(kfs[0], kfs[j], only_stereo=j % 5 == 0)
        c = resized(c, None, sizes[j - 1])
        matched += check(ex, c, j % 3 == 0, j % 2, ("neighbour", j, sizes[j - 1]))
    assert matched > 100


def test_distinctive_descriptors_in_one_large_call(ex):
    sizes, kinds, lists = distinctive_lists()
    fill = filler_lists(100_000 - len(lists))
    lists = lists + fill
    lists.insert(5, np.zeros((0, 32), np.uint8))            # points without observations
    lists.append(np.zeros((0, 32), np.uint8))
    off = np.concatenate([[0], np.cumsum([len(d) for d in lists])]).astype(np.int32)
    got = ComputeDistinctiveDescriptors(ex, off, np.concatenate(lists))
    assert len(got) == len(lists) >= 100_000
    ref = np.array([po.distinctive_descriptor(d) for d in lists], np.int32)
    bad = np.nonzero(got != ref)[0]
    assert len(bad) == 0, [(int(i), len(lists[i]), int(got[i]), int(ref[i])) for i in bad[:8]]


def test_distinctive_descriptors_at_the_observation_limit(ex):
    rng = np.random.default_rng(7)
    row = rng.integers(0, 256, (1, 32), dtype=np.uint8)
    small = [rng.integers(0, 256, (n, 32), dtype=np.uint8) for n in (3, 40)]
    lists = [small[0], np.repeat(row, 65535, 0), small[1]]
    off = np.concatenate([[0], np.cumsum([len(d) for d in lists])]).astype(np.int32)
    t0 = time.perf_counter()
    got = ComputeDistinctiveDescriptors(ex, off, np.concatenate(lists))
    print(f"65 535-observation call: {time.perf_counter() - t0:.3f} s")
    assert list(got) == [po.distinctive_descriptor(small[0]), 0, po.distinctive_descriptor(small[1])]
    over = [small[0], np.repeat(row, 65536, 0)]
    off = np.concatenate([[0], np.cumsum([len(d) for d in over])]).astype(np.int32)
    with pytest.raises(OrbError, match=r"orb_status -5: map point with more than 65535 observations"):
        ComputeDistinctiveDescriptors(ex, off, np.concatenate(over))
    off = np.concatenate([[0], np.cumsum([len(d) for d in small])]).astype(np.int32)
    assert list(ComputeDistinctiveDescriptors(ex, off, np.concatenate(small))) == [po.distinctive_descriptor(d) for d in small]


@pytest.mark.parametrize("scale,levels", PYRAMIDS)
@pytest.mark.parametrize("distance", [10.0, 500.0, 2000.0])
def test_update_normal_and_depth_far_from_the_origin(scale, levels, distance):
    e = ORBextractor(1200, scale, levels, 20, 7, max_width=640, max_height=480, max_batch=1)
    try:
        sf = e.GetScaleFactors()
        for n_points in (1, 128, 256, 300, 1000):
            c = normal_depth_case(distance, scale, levels, n_points=n_points, seed=n_points, empty_every=17 if n_points > 1 else 2)
            nrm, mx, mn = UpdateNormalAndDepth(e, c["off"], c["centres"], c["pos"], c["refc"], c["lvl"], c["n0"], c["mx0"], c["mn0"])
            for i, n in enumerate(c["counts"]):
                if n == 0:
                    assert (nrm[i].view(np.uint32) == c["n0"][i].view(np.uint32)).all() and mx[i] == c["mx0"][i] and mn[i] == c["mn0"][i]
                    continue
                a, b = c["off"][i], c["off"][i + 1]
                rn, rmx, rmn = po.update_normal_and_depth(c["centres"][a:b], c["pos"][i], c["refc"][i], c["lvl"][i], sf)
                assert (nrm[i].view(np.uint32) == rn.view(np.uint32)).all(), (n_points, i, nrm[i], rn)
                assert np.float32(mx[i]).view(np.uint32) == np.float32(rmx).view(np.uint32), (n_points, i)
                assert np.float32(mn[i]).view(np.uint32) == np.float32(rmn).view(np.uint32), (n_points, i)
    finally:
        e.close()
