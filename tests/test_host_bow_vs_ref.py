"""CPU tier, build container only: host/ORBmatcher_bow_b200.cc -- the translation unit that replaces both ORBmatcher::SearchByBoW overloads --
against the REFERENCE's own functions (src/ORBmatcher.cc:259-493, 892-1043, compiled verbatim in oracle/_ref part 2); and
host/ORBmatcher_triangulation_b200.cc against SearchForTriangulation (:1045-1323) likewise (relative pose, epipole, fundamental matrix,
query / validity / stereo flags, the pair list).  The unit's searches
are answered by the CPU oracle (tests/host/bow_stub.cc) over the arrays it marshals, so what is compared is the marshaling: the
FeatureVector merge order of the keyframe's good map points, the vocabulary node of every target feature, which map point lands in
which slot of vpMapPointMatches / vpMatches12 (bad and missing points, features without a BoW node), and the return values."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
MINE = os.path.join(HERE, "host", "bow_cpu_mine")


def _build():
    if os.path.exists(os.path.join(po.REFERENCE_ROOT, "src", "ORBmatcher.cc")):
        subprocess.check_call(["bash", os.path.join(HERE, "host", "build_bow_cpu.sh")])
    return os.path.exists(MINE) and po.build_ref2() is not None


pytestmark = pytest.mark.skipif(not _build(), reason="tests/host/bow_cpu_mine / oracle/_ref part 2 not built and /root/reference absent")
_spec = importlib.util.spec_from_file_location("_m2", os.path.join(HERE, "test_oracle_vs_ref_matcher2.py"))
_m = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_m)
two_frames = _m.two_frames


@pytest.mark.parametrize("nnratio,check,seed", [(0.7, True, 1), (0.9, False, 2), (0.75, True, 3)])
def test_both_overloads_equal_the_reference_functions(tmp_path, two_frames, nnratio, check, seed):
    (k1, d1, u1, dep1), (k2, d2, u2, dep2), sf = two_frames
    rng = np.random.default_rng(seed)
    node1, node2 = _m.node_of(d1, 97), _m.node_of(d2, 97)
    node1[5::23] = -1; node2[::17] = -1                        # features without a BoW entry on both sides
    has1, has2 = dep1 > 0, rng.random(len(k2)) < 0.7
    bad1, bad2 = has1 & (rng.random(len(k1)) < 0.05), has2 & (rng.random(len(k2)) < 0.04)
    d = str(tmp_path)
    for name, a in dict(k1=k1, k2=k2).items():
        assert a.dtype.itemsize == 28
        np.ascontiguousarray(a).tofile(os.path.join(d, name + ".kp"))
    for name, a in dict(d1=d1, d2=d2, has1=has1, bad1=bad1, has2=has2, bad2=bad2).items():
        np.ascontiguousarray(a, np.uint8).tofile(os.path.join(d, name + ".u8"))
    node1.astype(np.int32).tofile(os.path.join(d, "node1.i32")); node2.astype(np.int32).tofile(os.path.join(d, "node2.i32"))
    only_stereo, coarse = seed == 2, seed == 3
    T1, T2 = _m._quat_pose(0.0, [0, 0, 0]), _m._quat_pose(0.4, [-0.03, -0.002, -0.01])
    ur1, ur2 = (u1, u2) if seed != 1 else (np.full(len(k1), -1, np.float32), np.full(len(k2), -1, np.float32))
    np.concatenate([np.float32([nnratio, 1.0 if check else 0.0, float(only_stereo), float(coarse)]), _m.CAM6[:4], np.float32(T1), np.float32(T2), np.float32([100 if seed != 2 else 30])]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
    _m.BOUNDS.astype(np.float32).tofile(os.path.join(d, "bounds.f32"))
    tri1, tri2 = rng.random(len(k1)) < 0.4, rng.random(len(k2)) < 0.3
    tri1.astype(np.uint8).tofile(os.path.join(d, "tri_has1.u8")); tri2.astype(np.uint8).tofile(os.path.join(d, "tri_has2.u8"))
    np.ascontiguousarray(ur1, np.float32).tofile(os.path.join(d, "ur1.f32")); np.ascontiguousarray(ur2, np.float32).tofile(os.path.join(d, "ur2.f32"))
    r = subprocess.run([MINE, d], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "bow_cpu ok" in r.stdout, (r.stdout[-1000:], r.stderr[-1000:])
    fa, fb = np.fromfile(os.path.join(d, "out_frame_match.i32"), np.int32), np.fromfile(os.path.join(d, "out_kf_match.i32"), np.int32)
    ra, rb = np.fromfile(os.path.join(d, "out_ret.i32"), np.int32)
    K1 = po.RefKeyFrame(k1, d1, u1, node1, has1, bad1, sf, sf * sf, _m.CAM6[:4])
    K2 = po.RefKeyFrame(k2, d2, u2, node2, has2, bad2, sf, sf * sf, _m.CAM6[:4])
    F = po.RefFrame(k2, d2, u2, _m.BOUNDS, sf, _m.CAM6)
    wa, na = po.ref2_search_bow(F, node2, K1, nnratio, check)           # per frame feature: the keyframe-1 feature whose map point it received
    wb, nb = po.ref2_search_bow_kf(K1, K2, nnratio, check)              # per keyframe-1 feature: the keyframe-2 feature
    assert ra == na and len(fa) == len(k2) and (fa == wa).all()
    assert rb == nb and len(fb) == len(k1) and (fb == wb).all()
    assert na > 40 and nb > 30
    # SearchForTriangulation: the keyframes carry poses, uRight and the camera; features that hold a map point are skipped on both sides
    # (bad or not), so the reference keyframes are built without the bad flags that only the BoW overloads read
    tri = np.fromfile(os.path.join(d, "out_tri_pairs.i32"), np.int32)
    rc, pairs = tri[-1], tri[:-1].reshape(-1, 2)
    K1t = po.RefKeyFrame(k1, d1, ur1, node1, tri1, None, sf, sf * sf, _m.CAM6[:4], T1)
    K2t = po.RefKeyFrame(k2, d2, ur2, node2, tri2, None, sf, sf * sf, _m.CAM6[:4], T2)
    wm, wn, _, _ = po.ref2_search_triangulation(K1t, K2t, only_stereo, coarse, check)
    want = np.stack([np.nonzero(wm >= 0)[0], wm[wm >= 0]], 1)
    assert rc == wn and pairs.shape == want.shape and (pairs == want).all()
    assert wn > (3 if not coarse else 40)
    # SearchForInitialization, the current frame once resident on the "device", once uploaded from its own arrays
    window = 100 if seed != 2 else 30
    F1i, F2i = po.RefFrame(k1, d1, None, _m.BOUNDS, sf, _m.CAM6), po.RefFrame(k2, d2, None, _m.BOUNDS, sf, _m.CAM6)
    prev0 = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    im, inn, iprev = po.ref2_search_initialization(F1i, F2i, prev0, window, nnratio, check)
    got = np.fromfile(os.path.join(d, "out_init.i32"), np.int32).reshape(2, len(k1) + 1)
    gprev = np.fromfile(os.path.join(d, "out_init_prev.f32"), np.float32).reshape(2, len(k1), 2)
    for p in range(2):
        assert got[p, -1] == inn and (got[p, :-1] == im).all() and (gprev[p] == iprev).all()
    assert inn > 50
