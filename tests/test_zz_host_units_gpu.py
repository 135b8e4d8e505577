"""GPU tier: the nine host translation units that tests/test_zz_host_boundary_gpu.py does not run -- both ORBmatcher::SearchByBoW
overloads, SearchForInitialization, SearchForTriangulation, Fuse(pKF, vpMapPoints), the relocalisation SearchByProjection, the Sim3
SearchByProjection overloads and Fuse(pKF, Scw), Frame::ComputeBoW, Optimizer::PoseOptimization and Optimizer::LocalInertialBA --
linked with the library and run through the reference's class declarations on the inputs their C++ callers build.
tests/host/host_units (tests/host/build_units.sh, built by __graft_entry__.build()) records every C ABI call a unit makes (-Wl,--wrap=), so
each case checks two independent things:
  (a) the device answer against the oracle on exactly the recorded inputs (the F12 / epipole the triangulation unit computed included);
  (b) the unit's own work, restated here from the recorded answer: which queries it sent in which order, and what it wrote back
      (FeatureVector merge order, which MapPoint* lands in which slot, vbPrevMatched, mvbOutlier, SetPose, mBowVec / mFeatVec, the Fuse
      mutations, the LocalInertialBA write-back)."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth
from orb_slam3_detailed_comments_b200.vocabulary import synthetic_vocabulary

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "host", "host_units")
W, H, NF = 640, 480, 1200
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11
CAM6 = np.array([FX, FY, CX, CY, BF, B], np.float32)
BOUNDS = np.array([0, W, 0, H], np.float32)
KP = po.KP_DTYPE
EXT = {np.dtype(np.float32): "f32", np.dtype(np.int32): "i32", np.dtype(np.uint8): "u8", np.dtype(np.float64): "f64"}


def node_of(d, m):
    return (((d[:, 0].astype(np.int32) >> 3) * 7 + (d[:, 5].astype(np.int32) >> 4) * 3 + (d[:, 17].astype(np.int32) >> 5)) % m).astype(np.int32)


def quat_pose(yaw_deg, t):
    a = np.deg2rad(yaw_deg) / 2
    return np.array([0, np.sin(a), 0, np.cos(a), *t], np.float32)


class Run:
    """One run of the driver in directory d: inputs written, outputs and recorded calls read back."""

    def __init__(self, d, unit, meta, arrays, w=W, h=H, nf=NF):
        self.d = d
        os.makedirs(d, exist_ok=True)
        m = dict(W=w, H=h, nfeatures=nf, fx=FX, fy=FY, cx=CX, cy=CY, bf=BF, b=B, minx=0, maxx=w, miny=0, maxy=h)
        m.update(meta)
        with open(os.path.join(d, "meta.txt"), "w") as f:
            for k, v in m.items():
                f.write(f"{k} {float(v)!r}\n")
        with open(os.path.join(d, "unit.txt"), "w") as f:
            f.write(unit)
        for name, a in arrays.items():
            a = np.ascontiguousarray(a)
            a.tofile(os.path.join(d, name if "." in name else f"{name}.{EXT[a.dtype]}"))
        assert os.path.exists(BIN), "tests/host/host_units is not built (run __graft_entry__.build())"
        r = subprocess.run([BIN, d], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0 and "host_units ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]

    def out(self, name, dt):
        return np.fromfile(os.path.join(self.d, name), dt)

    def has(self, tag, k):
        return os.path.exists(os.path.join(self.d, f"rec_{tag}{k}_status"))

    def rec(self, tag, k, field, dt):
        return np.fromfile(os.path.join(self.d, f"rec_{tag}{k}_{field}"), dt)

    def errors(self):
        with open(os.path.join(self.d, "out_errors.txt")) as f:
            return [l for l in f.read().splitlines() if l]


@pytest.fixture(scope="module")
def scene():
    """Two stereo frames of one scene (the second shifted by a few pixels, with noise) through the oracle: frame A plays the keyframe /
    reference frame, frame B is the image the driver extracts on the device (the current frame)."""
    rng = np.random.default_rng(9)
    l, r, _ = synth.stereo_pair(W, H, seed=510)
    out = []
    for k in range(2):
        if k == 1:
            noise = rng.integers(-3, 4, (H, W))
            l = np.clip(np.roll(l, (4, 1), (1, 0)).astype(int) + noise, 0, 255).astype(np.uint8)
            r = np.clip(np.roll(r, (4, 1), (1, 0)).astype(int) + noise, 0, 255).astype(np.uint8)
        eL, eR = po.OracleExtractor(NF, 1.2, 8, 20, 7), po.OracleExtractor(NF, 1.2, 8, 20, 7)
        _, kL, dL = eL(l, (0, 1000))
        _, kR, dR = eR(r)
        uR, dep, _ = po.stereo_matches(eL, eR, kL, dL, kR, dR, np.float32(BF), np.float32(B))
        out.append(dict(img=l, k=kL, d=dL, ur=uR, dep=dep))
    return dict(A=out[0], B=out[1], ex=eL)


def check_frame(run, S):
    """The frame the driver extracted is the oracle's frame B (the resident frame every device-side answer is checked against)."""
    k = run.out("out_frame_kps.bin", KP)
    assert len(k) == len(S["B"]["k"]) and (k.view(np.uint8) == S["B"]["k"].view(np.uint8)).all()
    assert (run.out("out_frame_desc.u8", np.uint8).reshape(-1, 32) == S["B"]["d"]).all()


def kf_arrays(tag, f, node, has, bad, ur=None, T=None):
    return {f"{tag}.kp": f["k"], f"{tag}_desc": f["d"], f"{tag}_node": node.astype(np.int32), f"{tag}_has": has.astype(np.uint8),
            f"{tag}_bad": bad.astype(np.uint8), f"{tag}_ur": (f["ur"] if ur is None else ur).astype(np.float32),
            f"{tag}_T": (quat_pose(0, [0, 0, 0]) if T is None else T).astype(np.float32)}


def featvec_queries(node, ok):
    """The FeatureVector walk: ascending node, ascending feature index inside a node, features that pass `ok`."""
    return np.array([i for n in sorted(set(node[node >= 0].tolist())) for i in np.nonzero(node == n)[0] if ok[i]], np.int64)


# ---------------------------------------------------------------------------------------------------------------------------------
# SearchByBoW(KF, F): the frame on the device
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nnratio,check,case", [(0.7, True, "plain"), (0.9, False, "plain"), (0.75, True, "no_good_point")])
def test_search_by_bow_frame(tmp_path, scene, nnratio, check, case):
    A, B = scene["A"], scene["B"]
    rng = np.random.default_rng(3)
    node1, fnode = node_of(A["d"], 97), node_of(B["d"], 97)
    node1[5::23] = -1; fnode[::17] = -1                      # features without a BoW node on both sides
    has = (A["dep"] > 0) | (rng.random(len(A["k"])) < 0.3)
    bad = has & (rng.random(len(A["k"])) < 0.05)             # bad and missing map points
    if case == "no_good_point":
        bad = has.copy()
    run = Run(str(tmp_path), "bow", dict(nnratio=nnratio, checkori=int(check)),
              dict(img=B["img"], frame_node=fnode, **kf_arrays("k1", A, node1, has, bad)))
    check_frame(run, scene)
    N = len(B["k"])
    out = run.out("out_bow.i32", np.int32)
    assert len(out) == N + 1                                  # vpMapPointMatches sized F.N
    q = featvec_queries(node1, has & ~bad)
    assert any("Nleft" in e for e in run.errors()) and not run.has("bow", 1)   # the fisheye frame was refused before any search
    if case == "no_good_point":
        assert out[N] == 0 and (out[:N] == -1).all() and not run.has("bow", 0)
        return
    # (b) the queries the unit sent, and what it wrote back from the answer
    assert (run.rec("bow", 0, "qnode", np.int32) == node1[q]).all()
    assert (run.rec("bow", 0, "qangle", np.float32).view(np.uint32) == A["k"]["angle"][q].view(np.uint32)).all()
    assert (run.rec("bow", 0, "qdesc", np.uint8).reshape(-1, 32) == A["d"][q]).all()
    assert (run.rec("bow", 0, "fnode", np.int32) == fnode).all()
    fm, nm = run.rec("bow", 0, "fm", np.int32), run.rec("bow", 0, "nm", np.int32)[0]
    assert out[N] == nm and (out[:N] == np.where(fm >= 0, q[np.clip(fm, 0, None)], -1)).all()
    # (a) the device answer against the oracle on the recorded inputs
    wfm, wnm = po.search_bow(B["k"], B["d"], run.rec("bow", 0, "fnode", np.int32), run.rec("bow", 0, "qnode", np.int32),
                             run.rec("bow", 0, "qangle", np.float32), run.rec("bow", 0, "qdesc", np.uint8).reshape(-1, 32), nnratio, check)
    assert nm == wnm and (fm == wfm).all() and wnm > 40


# ---------------------------------------------------------------------------------------------------------------------------------
# SearchByBoW(KF, KF) and SearchForTriangulation on the keyframe-search handle
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("other_scale,mono", [(None, False), (1.3, False), (None, True)])   # 1.3: an extractor with other level tables
def test_keyframe_searches(tmp_path, scene, other_scale, mono):
    A, B = scene["A"], scene["B"]
    rng = np.random.default_rng(4)
    n1, n2 = len(A["k"]), len(B["k"])
    node1, node2 = node_of(A["d"], 61), node_of(B["d"], 61)
    node1[7::19] = -1; node2[::13] = -1
    has1, has2 = rng.random(n1) < 0.7, rng.random(n2) < 0.7
    bad1, bad2 = has1 & (rng.random(n1) < 0.05), has2 & (rng.random(n2) < 0.05)
    ur1, ur2 = (np.full(n1, -1, np.float32), np.full(n2, -1, np.float32)) if mono else (A["ur"], B["ur"])
    # keyframe 2 sees the scene shifted by (4, 1) px; this relative pose puts that shift ~3 px off the epipolar lines, where the
    # level-scaled gate 3.84 * sigma2[octave] (ORBmatcher.cc:1210) accepts or rejects a match depending on the level tables
    T1, T2 = quat_pose(0.0, [0, 0, 0]), quat_pose(0.0, [-0.05, -0.0866, 0.01])
    tri1, tri2 = rng.random(n1) < 0.4, rng.random(n2) < 0.3
    arrays = dict(img=B["img"], **kf_arrays("k1", A, node1, has1, bad1, ur1, T1), **kf_arrays("k2", B, node2, has2, bad2, ur2, T2),
                  k1_trihas=tri1.astype(np.uint8), k2_trihas=tri2.astype(np.uint8))
    meta = dict(nnratio=0.75, checkori=1, use_other=int(other_scale is not None), other_scale=other_scale or 1.2, other_levels=8)
    if other_scale is None and not mono:                      # a host keyframe beyond 16 384 rows: refused, the handle still searches
        reps = 16385 // n2 + 1
        big = dict(k=np.tile(B["k"], reps)[:16385], d=np.tile(B["d"], (reps, 1))[:16385], ur=np.tile(B["ur"], reps)[:16385])
        arrays.update(kf_arrays("kb", big, np.tile(node2, reps)[:16385], np.ones(16385, bool), np.zeros(16385, bool)))
        meta["big_n"] = 16385
    run = Run(str(tmp_path), "bowkf", meta, arrays)
    err = run.errors()
    # no frame search yet and no handle named: both keyframe searches refuse, and the process carries on
    assert len(err) >= 2 and "no device workspace" in err[0] and "no device workspace" in err[1]
    handles = run.out("handles.u64", np.uint64)
    want_h = handles[1] if other_scale is not None else handles[0]
    ex = po.OracleExtractor(NF, other_scale or 1.2, 8, 20, 7)
    sf, s2 = ex.scale_factors, ex.level_sigma2
    # ---- SearchByBoW(KF, KF) ----
    assert run.rec("bowkf", 0, "handle", np.uint64)[0] == want_h
    q = featvec_queries(node1, has1 & ~bad1)
    assert (run.rec("bowkf", 0, "qnode", np.int32) == node1[q]).all()
    assert (run.rec("bowkf", 0, "desc1", np.uint8).reshape(-1, 32) == A["d"][q]).all()
    assert (run.rec("bowkf", 0, "valid2", np.uint8) == (has2 & ~bad2)).all() and (run.rec("bowkf", 0, "node2", np.int32) == node2).all()
    assert (run.rec("bowkf", 0, "kp2", KP).view(np.uint8) == B["k"].view(np.uint8)).all()
    m12, nm = run.rec("bowkf", 0, "m12", np.int32), run.rec("bowkf", 0, "nm", np.int32)[0]
    wm, wn = po.search_bow_kf(run.rec("bowkf", 0, "kp2", KP), run.rec("bowkf", 0, "desc2", np.uint8).reshape(-1, 32), run.rec("bowkf", 0, "node2", np.int32),
                              run.rec("bowkf", 0, "valid2", np.uint8), run.rec("bowkf", 0, "qnode", np.int32), run.rec("bowkf", 0, "qangle", np.float32),
                              run.rec("bowkf", 0, "desc1", np.uint8).reshape(-1, 32), 0.75, True)
    assert nm == wn and (m12 == wm).all() and wn > 30
    fb = run.out("out_bowkf.i32", np.int32)
    want = np.full(n1, -1, np.int32)
    want[q[m12 >= 0]] = m12[m12 >= 0]
    assert len(fb) == n1 + 1 and fb[n1] == nm and (fb[:n1] == want).all()
    # ---- SearchForTriangulation, bOnlyStereo x bCoarse ----
    tri = run.out("out_tri.i32", np.int32)
    pos = 0
    R1, R2 = quat_to_R(T1), quat_to_R(T2)
    k = 0                                                     # index of the recorded call: a combination without queries makes none
    tables_matter = False
    for combo in range(4):
        only_stereo, coarse = bool(combo & 1), bool(combo & 2)
        stereo1, stereo2 = ur1 >= 0, ur2 >= 0
        qt = featvec_queries(node1, ~tri1 & (stereo1 | (not only_stereo)))
        if len(qt) == 0:                                      # a monocular keyframe searched for stereo matches only: 0, no pairs
            assert mono and only_stereo and list(tri[pos:pos + 2]) == [0, 0]
            pos += 2
            continue
        assert run.rec("tri", k, "handle", np.uint64)[0] == want_h
        assert (run.rec("tri", k, "kp1", KP).view(np.uint8) == A["k"][qt].view(np.uint8)).all()
        assert (run.rec("tri", k, "node1", np.int32) == node1[qt]).all() and (run.rec("tri", k, "stereo1", np.uint8) == stereo1[qt]).all()
        assert (run.rec("tri", k, "valid2", np.uint8) == (~tri2 & (stereo2 | (not only_stereo)))).all()
        assert (run.rec("tri", k, "stereo2", np.uint8) == stereo2).all() and (run.rec("tri", k, "node2", np.int32) == node2).all()
        assert list(run.rec("tri", k, "flags", np.int32)) == [int(coarse), 1]
        F12, ep = run.rec("tri", k, "F12", np.float32).reshape(3, 3), run.rec("tri", k, "ep2", np.float32)
        wF, wep = fundamental(R1, T1[4:], R2, T2[4:])
        assert np.abs(F12 / np.abs(F12).max() - wF / np.abs(wF).max()).max() < 1e-4 and np.abs(ep - wep).max() < 1e-2 * max(1.0, np.abs(wep).max())
        m, n = run.rec("tri", k, "m12", np.int32), run.rec("tri", k, "nm", np.int32)[0]
        r = lambda f, t: run.rec("tri", k, f, t)
        wm, wn = po.search_triangulation(r("kp1", KP), r("desc1", np.uint8).reshape(-1, 32), r("node1", np.int32), r("stereo1", np.uint8), r("kp2", KP),
                                         r("desc2", np.uint8).reshape(-1, 32), r("node2", np.int32), r("valid2", np.uint8), r("stereo2", np.uint8),
                                         F12.ravel(), ep, sf, s2, coarse, True)
        assert n == wn and (m == wm).all()
        assert wn > (3 if not coarse else 40) or only_stereo
        if other_scale is not None:                           # the stubs' 1.2 / 8 tables would give another answer on these inputs
            e12 = po.OracleExtractor(NF, 1.2, 8, 20, 7)
            wm12, wn12 = po.search_triangulation(r("kp1", KP), r("desc1", np.uint8).reshape(-1, 32), r("node1", np.int32), r("stereo1", np.uint8),
                                                 r("kp2", KP), r("desc2", np.uint8).reshape(-1, 32), r("node2", np.int32), r("valid2", np.uint8),
                                                 r("stereo2", np.uint8), F12.ravel(), ep, e12.scale_factors, e12.level_sigma2, coarse, True)
            tables_matter |= wn12 != wn or bool((wm12 != wm).any())
        npairs = tri[pos]
        pairs = tri[pos + 1:pos + 1 + 2 * npairs].reshape(-1, 2)
        ret = tri[pos + 1 + 2 * npairs]
        pos += 2 + 2 * npairs
        sel = np.argsort(qt[m >= 0], kind="stable")
        want_pairs = np.stack([qt[m >= 0][sel], m[m >= 0][sel]], 1) if (m >= 0).any() else np.zeros((0, 2), np.int64)
        assert ret == n and pairs.shape == want_pairs.shape and (pairs == want_pairs).all()     # ascending idx1
        k += 1
    assert not os.path.exists(os.path.join(run.d, f"rec_tri{k}_status"))
    assert tables_matter or other_scale is None
    if "big_n" in meta:
        assert run.rec("bowkf", 1, "status", np.int32)[0] == -5 and any("feature rows" in e for e in err[2:]), err   # ORB_ERR_UNSUPPORTED
        assert run.out("out_after_refusal.i32", np.int32)[0] == nm


def quat_to_R(T7):
    x, y, z, w = (float(v) for v in T7[:4])
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def fundamental(R1, t1, R2, t2):
    """F12 = K^-T [t12]x R12 K^-1 and the epipole of camera 1 in image 2, in double (ORBmatcher.cc:1052-1073, Pinhole.cpp:191-194)."""
    t1, t2 = np.asarray(t1, np.float64), np.asarray(t2, np.float64)
    C1 = -R1.T @ t1
    C2 = R2 @ C1 + t2
    ep = np.array([FX * C2[0] / C2[2] + CX, FY * C2[1] / C2[2] + CY])
    R12 = R1 @ R2.T
    t12 = -R12 @ t2 + t1
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    K = np.array([[FX, 0, CX], [0, FY, CY], [0, 0, 1]])
    Ki = np.linalg.inv(K)
    return Ki.T @ tx @ R12 @ Ki, ep


# ---------------------------------------------------------------------------------------------------------------------------------
# SearchForInitialization: F2 resident, or uploaded because another frame is resident
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("uploaded,window,check", [(False, 100, True), (True, 100, True), (False, 10, False)])
def test_search_for_initialization(tmp_path, scene, uploaded, window, check):
    A, B = scene["A"], scene["B"]
    prev = np.stack([A["k"]["x"], A["k"]["y"]], 1).astype(np.float32)
    arrays = {"img": B["img"], "img2.u8": A["img"], "f1.kp": A["k"], "f1_desc": A["d"], "f1_prev": prev}
    run = Run(str(tmp_path), "init", dict(uploaded=int(uploaded), window=window, nnratio=0.9, checkori=int(check)), arrays)
    check_frame(run, scene)
    _check_init(run, A["k"], A["d"], prev, B["k"], B["d"], uploaded, window, 0.9, check)
    if uploaded:
        assert len(run.out("out_resident_kps.bin", KP)) != len(B["k"])    # the resident frame really differs in N


def _check_init(run, k1, d1, prev, k2, d2, uploaded, window, nnratio, check):
    n1 = len(k1)
    par = run.rec("init", 0, "par", np.float32)
    assert list(par) == [window, np.float32(nnratio), float(check), -1.0 if uploaded else 0.0, float(len(k2)) if uploaded else 0.0]
    assert (run.rec("init", 0, "kp1", KP).view(np.uint8) == k1.view(np.uint8)).all() and (run.rec("init", 0, "prev", np.float32).reshape(-1, 2) == prev).all()
    cam = run.rec("init", 0, "cam", np.float32)
    if uploaded:
        assert (run.rec("init", 0, "kp2", KP).view(np.uint8) == k2.view(np.uint8)).all() and (run.rec("init", 0, "desc2", np.uint8).reshape(-1, 32) == d2).all()
    m12, nm = run.rec("init", 0, "m12", np.int32), run.rec("init", 0, "nm", np.int32)[0]
    wm, wn = po.search_initialization(k1, d1, prev, k2, d2, cam[6:10], window, nnratio, check)
    assert nm == wn and (m12 == wm).all() and wn > 50
    out, pout = run.out("out_init.i32", np.int32), run.out("out_init_prev.f32", np.float32).reshape(-1, 2)
    assert len(out) == n1 + 1 and out[n1] == nm and (out[:n1] == m12).all()
    want = prev.copy()                                       # vbPrevMatched refreshed from the matches (:880-884)
    want[m12 >= 0, 0] = k2["x"][m12[m12 >= 0]]
    want[m12 >= 0, 1] = k2["y"][m12[m12 >= 0]]
    assert (pout.view(np.uint32) == want.view(np.uint32)).all()


def test_search_for_initialization_five_times_the_features(tmp_path):
    """ORB-SLAM3's monocular initialisation extractor (5x features) on a EuRoC-shaped 752x480 frame: F2 holds more rows than the
    shared-memory matcher takes, so the global-memory form runs behind the unit."""
    from test_zz_many_features_gpu import INIT_LAST_SHARED
    w, h, nf = 752, 480, 5000
    img = np.roll(synth.frame(w, h, 301, 1.0, 400), (2, 3), (0, 1))     # the scene of test_zz_many_features_gpu.py's EuRoC frames
    e = po.OracleExtractor(nf, 1.2, 8, 20, 7)
    _, k2, d2 = e(img, (0, 1000))
    assert len(k2) > INIT_LAST_SHARED
    rng = np.random.default_rng(8)
    sel = rng.choice(len(k2), 2500, replace=False)
    k1 = k2[sel].copy()
    k1["x"] += rng.normal(0, 1.0, len(sel)).astype(np.float32)
    k1["y"] += rng.normal(0, 1.0, len(sel)).astype(np.float32)
    d1 = d2[sel].copy()
    prev = np.stack([k1["x"], k1["y"]], 1).astype(np.float32)
    run = Run(str(tmp_path), "init", dict(uploaded=0, window=100, nnratio=0.9, checkori=1),
              {"img": img, "f1.kp": k1, "f1_desc": d1, "f1_prev": prev}, w=w, h=h, nf=nf)
    assert (run.out("out_frame_kps.bin", KP).view(np.uint8) == k2.view(np.uint8)).all()
    _check_init(run, k1, d1, prev, k2, d2, False, 100, 0.9, True)


# ---------------------------------------------------------------------------------------------------------------------------------
# the searches that project map points: relocalisation, Fuse(pKF, vpMapPoints), the Sim3 family
# ---------------------------------------------------------------------------------------------------------------------------------
def points_from(f, rng, sf, jitter=1.0, flip=0.02):
    """Map points at the stereo features of frame f (camera at the origin): world position, normal, raw distances, noisy descriptor."""
    idx = np.nonzero(f["dep"] > 0)[0]
    k = f["k"][idx]
    z = f["dep"][idx].astype(np.float64)
    x = (k["x"] + rng.normal(0, jitter, len(idx)) - CX) * z / FX
    y = (k["y"] + rng.normal(0, jitter, len(idx)) - CY) * z / FY
    xw = np.stack([x, y, z], 1).astype(np.float32)
    dist = np.linalg.norm(xw.astype(np.float64), axis=1)
    normal = (xw / dist[:, None]).astype(np.float32)
    maxd = (dist * sf[k["octave"]]).astype(np.float32)
    mind = (maxd / sf[-1]).astype(np.float32)
    qd = f["d"][idx].copy()
    fl = rng.random(qd.shape) < flip
    qd[fl] ^= (1 << rng.integers(0, 8, int(fl.sum()))).astype(np.uint8)
    return idx, dict(xw=xw, normal=normal, max=maxd, min=mind, desc=qd)


def q_arrays(P, bad, obs):
    return dict(q_xw=P["xw"], q_normal=P["normal"], q_max=P["max"], q_min=P["min"], q_desc=P["desc"], q_bad=bad.astype(np.uint8), q_obs=obs.astype(np.int32))


def unit_quat(q):
    """SE3f's quaternion normalisation (refshim/Eigen/Core Quaternion::normalize) in float: x y z w of the unit quaternion."""
    x, y, z, w = (np.float32(v) for v in q)
    n = np.sqrt(np.float32(np.float32(np.float32(x * x + y * y) + z * z) + w * w))
    return np.array([x / n, y / n, z / n, w / n], np.float32)


def check_kf_inputs(run, k, variant, th, hamming_max, check, cam10, P, src, Tcw7, Ow, normal=True, angle=None, tol=0.0):
    """(b) for orbm_search_keyframe: every input the unit sent is the caller's -- variant, th, the Hamming bound, the orientation flag, the
    camera and bounds, the pose, and per query (in the unit's query order `src`) the world position, the normal, the RAW
    mfMaxDistance / mfMinDistance, the descriptor and the keyframe feature's angle.  tol: the pose is a float Sophus product (0: exact)."""
    r = lambda f, t: run.rec("kf", k, f, t)
    assert list(r("par", np.float32)[:4]) == [variant, np.float32(th), np.float32(hamming_max), float(check)]
    assert (r("cam", np.float32).view(np.uint32) == np.asarray(cam10, np.float32).view(np.uint32)).all()
    T, O = r("Tcw", np.float32), r("Ow", np.float32)
    if np.dot(T[:4], Tcw7[:4]) < 0:
        T = np.concatenate([-T[:4], T[4:]])
    assert np.abs(T - Tcw7).max() <= tol and np.abs(O - Ow).max() <= max(tol, 1e-6), (T, Tcw7, O, Ow)
    for fld, key in (("xw", "xw"), ("maxd", "max"), ("mind", "min")):
        assert (r(fld, np.float32).view(np.uint32) == P[key][src].view(np.uint32).ravel()).all(), fld
    assert (r("qdesc", np.uint8).reshape(-1, 32) == P["desc"][src]).all()
    nr = r("normal", np.float32)
    assert (nr.view(np.uint32) == P["normal"][src].view(np.uint32).ravel()).all() if normal else nr.size == 0
    ang = r("angle", np.float32)
    assert (ang.view(np.uint32) == angle.view(np.uint32)).all() if angle is not None else ang.size == 0


def oracle_kf(run, k, variant, kps, desc, uright, sf, check=True):
    r = lambda f, t: run.rec("kf", k, f, t)
    isg = (1.0 / (sf * sf)).astype(np.float32)
    cam = r("cam", np.float32)
    par = r("par", np.float32)
    claimed = r("claimed", np.uint8)
    normal, angle = r("normal", np.float32), r("angle", np.float32)
    return po.search_keyframe(variant, kps, desc, uright, cam[6:10], sf, isg, po.logf(1.2), cam[:6], r("Tcw", np.float32), r("Ow", np.float32),
                              r("xw", np.float32).reshape(-1, 3), normal.reshape(-1, 3) if normal.size else None, r("maxd", np.float32), r("mind", np.float32),
                              r("qdesc", np.uint8).reshape(-1, 32), angle if angle.size else None, claimed if claimed.size else None, par[1], par[2], check)


@pytest.mark.parametrize("orbdist,check", [(64, True), (100, False), (100, True)])
def test_relocalisation_search(tmp_path, scene, orbdist, check):
    B = scene["B"]
    sf = scene["ex"].scale_factors
    rng = np.random.default_rng(orbdist + int(check))
    idx, P = points_from(B, rng, sf)
    n = len(idx)
    bad, already = rng.random(n) < 0.05, rng.random(n) < 0.1      # bad points; a non-empty sAlreadyFound
    slot = np.full(len(B["k"]), -1, np.int32)                       # the candidate keyframe: feature i holds point slot[i]
    keep = rng.random(n) < 0.8
    slot[idx[keep]] = np.nonzero(keep)[0]
    claimed = (rng.random(len(B["k"])) < 0.15).astype(np.uint8)     # frame features that already hold a map point
    T = quat_pose(0.1, [0.01, -0.005, 0.02])
    run = Run(str(tmp_path), "reloc", dict(frame_T=1, th=10, orbdist=orbdist, checkori=int(check)),
              {"img": B["img"], "frame_T": T, "r.kp": B["k"], "r_slot": slot, "r_already": already.astype(np.uint8), "frame_claimed": claimed,
               **q_arrays(P, bad, np.ones(n))})
    check_frame(run, scene)
    # (b) queries: the keyframe's good points not in sAlreadyFound, in feature order
    src = [int(slot[i]) for i in range(len(B["k"])) if slot[i] >= 0 and not bad[slot[i]] and not already[slot[i]]]
    qf = [i for i in range(len(B["k"])) if slot[i] >= 0 and not bad[slot[i]] and not already[slot[i]]]
    Tq = np.concatenate([unit_quat(T[:4]), T[4:]])
    Rq = quat_to_R(Tq)
    check_kf_inputs(run, 0, 3, 10, orbdist, check, [*CAM6, 0, W, 0, H], P, src, Tq, -Rq.T @ Tq[4:].astype(np.float64), normal=False,
                    angle=B["k"]["angle"][qf])
    assert (run.rec("kf", 0, "claimed", np.uint8) == claimed).all() and not os.path.exists(os.path.join(run.d, "rec_kf0_kp"))   # the frame on the device
    match, nm = run.rec("kf", 0, "match", np.int32), run.rec("kf", 0, "nm", np.int32)[0]
    out = run.out("out_reloc.i32", np.int32)
    want = np.where(claimed == 1, -2, -1).astype(np.int32)
    for qq, f in enumerate(match):
        if f >= 0:
            want[f] = src[qq]
    assert out[-1] == nm and (out[:-1] == want).all()
    # (a)
    wm, wn, _ = oracle_kf(run, 0, 3, B["k"], B["d"], None, sf, check)
    assert nm == wn and (match == wm).all() and wn > 50


def target_arrays(f, ur, slot, T=None):
    return {"t.kp": f["k"], "t_desc": f["d"], "t_ur": ur.astype(np.float32), "t_slot": slot.astype(np.int32),
            "t_T": (quat_pose(0, [0, 0, 0]) if T is None else T).astype(np.float32)}


@pytest.mark.parametrize("th,mono", [(3.0, False), (8.0, False), (3.0, True)])
def test_fuse(tmp_path, scene, th, mono):
    B = scene["B"]
    sf = scene["ex"].scale_factors
    rng = np.random.default_rng(int(th) + 10 * mono)
    idx, P = points_from(B, rng, sf, jitter=0.8)
    n = len(idx)
    N = len(B["k"])
    # objects 0..n-1: the points being fused; n..n+m-1: the keyframe's own points (features of another random subset)
    own = rng.choice(N, N // 4, replace=False)
    _, P2 = points_from(dict(B, dep=np.where(np.isin(np.arange(N), own), np.maximum(B["dep"], 3.0), -1)), rng, sf)
    allP = {k: np.concatenate([P[k], P2[k]]) for k in P}
    m = len(P2["xw"])
    bad = np.concatenate([rng.random(n) < 0.05, rng.random(m) < 0.05])
    obs = rng.integers(1, 6, n + m)
    slot = np.full(N, -1)
    slot[np.sort(own)[:m]] = n + np.arange(m)
    q_slot = np.concatenate([np.arange(n), [-1, -1], rng.choice(n, 20)]).astype(np.int32)   # NULL entries and repeated pointers
    in_kf = (rng.random(n + m) < 0.05) & (np.arange(n + m) < n)                            # points already in the keyframe
    ur = np.full(N, -1, np.float32) if mono else B["ur"]
    run = Run(str(tmp_path), "fuse", dict(th=th), {"img": B["img"], **target_arrays(B, ur, slot), **q_arrays(allP, bad, obs), "q_slot": q_slot,
                                                   "q_in_kf": in_kf.astype(np.uint8)})
    # (b) queries: vpMapPoints minus NULL, bad, IsInKeyFrame (own points observe the keyframe)
    in_kf_all = in_kf | (np.arange(n + m) >= n) & np.isin(np.arange(n + m), slot[slot >= 0])
    src = [int(j) for j in q_slot if j >= 0 and not bad[j] and not in_kf_all[j]]
    check_kf_inputs(run, 0, 0, th, 50, True, [*CAM6, 0, W, 0, H], allP, src, quat_pose(0, [0, 0, 0]), np.zeros(3))
    assert (run.rec("kf", 0, "uright", np.float32).view(np.uint32) == ur.view(np.uint32)).all()
    assert (run.rec("kf", 0, "kp", KP).view(np.uint8) == B["k"].view(np.uint8)).all() and (run.rec("kf", 0, "desc", np.uint8).reshape(-1, 32) == B["d"]).all()
    best, nm = run.rec("kf", 0, "match", np.int32), run.rec("kf", 0, "nm", np.int32)[0]
    # restated mutations in query order (:1508-1532)
    badnow, inkf, nobs, kslot, log, fused = bad.copy(), in_kf_all.copy(), obs + in_kf_all, slot.copy(), [], 0
    for qq, j in enumerate(src):
        b = best[qq]
        if b < 0:
            continue
        if badnow[j] or inkf[j]:
            continue
        o = kslot[b]
        if o >= 0:
            if not badnow[o]:
                if nobs[o] > nobs[j]:
                    log += [1, j, o, -1]; badnow[j] = True
                else:
                    log += [1, o, j, -1]; badnow[o] = True
        else:
            log += [3, j, -1, int(b)]; inkf[j] = True; nobs[j] += 1; kslot[b] = j
        fused += 1
    got = run.out("out_fuse_log.i32", np.int32)
    assert got[-1] == fused and list(got[:-1]) == log and fused > 30
    assert (run.out("out_fuse_kf.i32", np.int32) == kslot).all()
    # (a)
    wm, wn, _ = oracle_kf(run, 0, 0, B["k"], B["d"], ur, sf)
    assert nm == wn and (best == wm).all()


@pytest.mark.parametrize("scale", [1.0, 1.3])
def test_sim3_searches(tmp_path, scene, scale):
    B = scene["B"]
    sf = scene["ex"].scale_factors
    rng = np.random.default_rng(int(scale * 10))
    idx, P = points_from(B, rng, sf)
    n, N = len(idx), len(B["k"])
    q = quat_pose(2.0, [0, 0, 0])[:4].astype(np.float64)
    R = quat_to_R(q)
    t = np.array([0.05, -0.02, 0.1])
    # camera-frame points pc = R X + t / s  =>  X = R^T (pc - t / s)
    P["xw"] = ((P["xw"].astype(np.float64) - t / scale) @ R).astype(np.float32)
    P["normal"] = (P["normal"].astype(np.float64) @ R).astype(np.float32)
    bad = rng.random(n) < 0.05
    slot = np.full(N, -1)
    own = rng.choice(n, n // 10, replace=False)               # some points are already the keyframe's own (Fuse skips them)
    slot[idx[own]] = own
    matched = np.full(N, -1, np.int32)                        # vpMatched pre-filled: occupied slots, and points matched already
    matched[rng.random(N) < 0.1] = -2
    pre = rng.choice(n, 30, replace=False)
    free = np.nonzero(matched == -1)[0]
    matched[rng.choice(free, 30, replace=False)] = pre
    sp = np.array([*q, *t, scale, 10, 1.0], np.float32)
    run = Run(str(tmp_path), "sim3", {}, {"img": B["img"], **target_arrays(B, B["ur"], slot), **q_arrays(P, bad, np.ones(n)), "s_params": sp,
                                          "s_matched": matched})
    proj = run.out("out_sim3_proj.i32", np.int32)
    # both SearchByProjection overloads: the same queries, the same answer
    skip = set(matched[matched >= 0].tolist())
    src = [j for j in range(n) if not bad[j] and j not in skip]
    claimed = (matched != -1).astype(np.uint8)
    want = matched.copy()
    Tsim = np.concatenate([q, t / scale])                     # SE3f(Scw.rotationMatrix(), Scw.translation() / Scw.scale())
    Osim = -R.T @ (t / scale)
    cam10 = [*CAM6, 0, W, 0, H]
    for k in (0, 1):
        check_kf_inputs(run, k, 2, 10, 50 * 1.0, True, cam10, P, src, Tsim, Osim, tol=1e-6)
        assert (run.rec("kf", k, "claimed", np.uint8) == claimed).all()
        wm, wn, _ = oracle_kf(run, k, 2, B["k"], B["d"], B["ur"], sf)
        assert (run.rec("kf", k, "match", np.int32) == wm).all() and run.rec("kf", k, "nm", np.int32)[0] == wn
    best = run.rec("kf", 0, "match", np.int32)
    for qq, j in enumerate(src):
        if best[qq] >= 0:
            want[best[qq]] = j
    nm = run.rec("kf", 0, "nm", np.int32)[0]
    assert (proj[:N] == want).all() and proj[N] == nm and nm > 30
    assert (proj[N + 1:2 * N + 1] == want).all() and proj[2 * N + 1] == nm
    wkf = np.where((want != matched), want, -1)               # vpMatchedKF: the source keyframe of every newly matched point
    assert (proj[2 * N + 2:] == wkf).all()
    # Fuse(pKF, Scw, vpPoints, th, vpReplacePoint): the keyframe's own good points are skipped
    own_good = set(int(j) for j in own if not bad[j])
    fsrc = [j for j in range(n) if not bad[j] and j not in own_good]
    check_kf_inputs(run, 2, 1, 10, 50, True, cam10, P, fsrc, Tsim, Osim, tol=1e-6)
    assert run.rec("kf", 2, "claimed", np.uint8).size == 0
    fb, fnm = run.rec("kf", 2, "match", np.int32), run.rec("kf", 2, "nm", np.int32)[0]
    wm, wn, _ = oracle_kf(run, 2, 1, B["k"], B["d"], B["ur"], sf)
    assert (fb == wm).all() and fnm == wn
    repl, log, kslot, fused = np.full(n, -1), [], slot.copy(), 0
    for qq, j in enumerate(fsrc):
        b = fb[qq]
        if b < 0:
            continue
        if kslot[b] >= 0:
            if not bad[kslot[b]]:
                repl[j] = kslot[b]
        else:
            log += [3, j, -1, int(b)]; kslot[b] = j
        fused += 1
    got = run.out("out_sim3_fuse.i32", np.int32)
    assert (got[:n] == repl).all() and got[n] == fused and fused > 30
    assert list(run.out("out_sim3_fuse_log.i32", np.int32)) == log and (run.out("out_sim3_fuse_kf.i32", np.int32) == kslot).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# Frame::ComputeBoW
# ---------------------------------------------------------------------------------------------------------------------------------
def _real_subtree():
    z = np.load(os.path.join(ROOT, "tests", "golden", "orbvoc_subtree.npz"))
    voc = {k[4:]: z[k] for k in z.files if k.startswith("sub_")}
    voc["L"] = int(voc["L"])
    return voc


@pytest.mark.parametrize("which", ["synthetic", "real_subtree"])
def test_compute_bow(tmp_path, scene, which):
    A, B = scene["A"], scene["B"]
    voc = synthetic_vocabulary(k=10, L=4, seed=5) if which == "synthetic" else _real_subtree()
    arrays = {"img": B["img"], "img2.u8": A["img"], "child_offset": voc["child_offset"].astype(np.int32), "child_ids": voc["child_ids"].astype(np.int32),
              "node_word": voc["node_word"].astype(np.int32), "node_desc": voc["node_desc"].astype(np.uint8), "node_weight": voc["node_weight"].astype(np.float64)}
    run = Run(str(tmp_path), "voc", dict(L=voc["L"]), arrays)
    check_frame(run, scene)
    # one orbv_create per vocabulary object, with the tree as flattened by the unit; one transform per frame (the second ComputeBoW returns early)
    assert os.path.exists(os.path.join(run.d, "rec_vcreate0_L")) and not os.path.exists(os.path.join(run.d, "rec_vcreate1_L"))
    for f in ("child_offset", "child_ids", "node_word"):
        assert (run.rec("vcreate", 0, f, np.int32) == voc[f]).all()
    leaf = voc["child_offset"][1:] == voc["child_offset"][:-1]
    wt = np.where(leaf, voc["node_weight"], 0.0)
    wt[0] = 0.0
    assert (run.rec("vcreate", 0, "node_weight", np.float64).view(np.uint64) == wt.view(np.uint64)).all()
    assert (run.rec("vcreate", 0, "node_desc", np.uint8).reshape(-1, 32)[1:] == voc["node_desc"][1:]).all()
    assert run.has("vtransform", 1) and not run.has("vtransform", 2)
    oi, ow = run.out("out_voc.i32", np.int32), run.out("out_voc.f64", np.float64)
    pi = pw = 0
    for k, f in enumerate((B, A)):
        r = lambda fld, t: run.rec("vtransform", k, fld, t)
        assert list(r("par", np.int32)) == [4, 0]
        # (a) the device transform against the oracle
        w = po.bow_transform(voc, f["d"], 4)
        cnt = r("bow_count", np.int32)[0]
        assert (r("word", np.int32) == w["word"]).all() and (r("node", np.int32) == w["node"]).all()
        assert (r("weight", np.float64).view(np.uint64) == w["weight"].view(np.uint64)).all()
        assert cnt == len(w["bow_word"]) and (r("bow_word", np.int32) == w["bow_word"]).all()
        assert (r("bow_weight", np.float64).view(np.uint64) == w["bow_weight"].view(np.uint64)).all()
        # (b) mBowVec / mFeatVec from the recorded answer; the second call changed nothing
        assert oi[pi] == 0 and oi[pi + 1] == cnt
        assert (oi[pi + 2:pi + 2 + cnt] == r("bow_word", np.int32)).all() and (ow[pw:pw + cnt].view(np.uint64) == r("bow_weight", np.float64).view(np.uint64)).all()
        pi += 2 + cnt; pw += cnt
        node, weight = r("node", np.int32), r("weight", np.float64)
        fv = {}
        for i in range(len(node)):
            if weight[i] > 0:
                fv.setdefault(int(node[i]), []).append(i)
        want = [len(fv)]
        for nd in sorted(fv):
            want += [nd, len(fv[nd])] + fv[nd]
        assert list(oi[pi:pi + len(want)]) == want
        pi += len(want)
    assert pi == len(oi) and pw == len(ow)


# ---------------------------------------------------------------------------------------------------------------------------------
# Optimizer::PoseOptimization(Frame*)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mixed_40pct_outliers", "two_correspondences", "eight_edges"])
def test_pose_optimization(tmp_path, scene, case):
    B = scene["B"]
    ex = scene["ex"]
    rng = np.random.default_rng(21)
    N = len(B["k"])
    dep = np.where(B["dep"] > 0, B["dep"], rng.uniform(3, 20, N)).astype(np.float64)
    xw = np.stack([(B["k"]["x"] - CX) * dep / FX, (B["k"]["y"] - CY) * dep / FY, dep], 1).astype(np.float32)
    stereo = (B["dep"] > 0) & (rng.random(N) < 0.7)            # a mixed monocular / stereo frame
    ur = np.where(stereo, B["ur"], -1).astype(np.float32)
    has = np.zeros(N, bool)
    n_has = dict(mixed_40pct_outliers=int(0.6 * N), two_correspondences=2, eight_edges=8)[case]
    has[rng.choice(N, n_has, replace=False)] = True
    out_sel = has & (rng.random(N) < (0.4 if case == "mixed_40pct_outliers" else 0.0))
    xw[out_sel] += rng.normal(0, 0.5, (int(out_sel.sum()), 3)).astype(np.float32)
    T = quat_pose(0.3, [0.02, -0.01, 0.03])                   # the prior: off the true (identity) pose
    isg = ex.inv_level_sigma2
    run = Run(str(tmp_path), "pose", dict(frame_T=1), {"img": B["img"], "frame_T": T, "p_xw": xw, "p_ur": ur, "p_inv_sigma2": isg, "p_has": has.astype(np.uint8)})
    pose = run.out("out_pose.f32", np.float32)
    outl = run.out("out_outlier.u8", np.uint8)
    ret, sets = run.out("out_pose_ret.i32", np.int32)
    if case == "two_correspondences":                          # :292-293: 0, the pose untouched, the flags it owns cleared
        assert ret == 0 and sets == 0 and not run.has("pose", 0)
        assert (pose == T).all() and (outl == np.where(has, 0, 1)).all()
        return
    # (b) one edge per feature with a map point, in feature order
    f = np.nonzero(has)[0]
    assert (run.rec("pose", 0, "xw", np.float32).reshape(-1, 3) == xw[f]).all()
    obs = np.stack([B["k"]["x"][f], B["k"]["y"][f], np.where(ur[f] < 0, -1, ur[f])], 1).astype(np.float32)
    assert (run.rec("pose", 0, "obs", np.float32).reshape(-1, 3).view(np.uint32) == obs.view(np.uint32)).all()
    assert (run.rec("pose", 0, "inv_sigma2", np.float32) == isg[B["k"]["octave"][f]]).all()
    assert (run.rec("pose", 0, "pose", np.float32) == T).all()
    po_out, e_out = run.rec("pose", 0, "pose_out", np.float64), run.rec("pose", 0, "outlier", np.uint8)
    inl = run.rec("pose", 0, "inliers", np.int32)[0]
    want = np.ones(N, np.uint8)
    want[f] = e_out
    assert (outl == want).all() and ret == inl and sets == 1
    # SetPose(SE3<float>(q.cast<float>(), t.cast<float>())): the doubles narrowed, the quaternion normalised in float -- bit for bit
    want_pose = np.concatenate([unit_quat(po_out[:4].astype(np.float32)), po_out[4:].astype(np.float32)])
    assert (pose.view(np.uint32) == want_pose.view(np.uint32)).all(), (pose, want_pose)
    # (a) the bar of tests/test_poseopt_gpu.py::_check on the recorded problem
    st = run.rec("pose", 0, "stats", np.int32)
    g = dict(pose=po_out, outlier=e_out, inliers=inl, rounds=st[0], iterations=st[1], trials=st[2])
    fr = dict(pose=T, world_pos=xw[f], obs=obs, inv_sigma2=isg[B["k"]["octave"][f]])
    from test_poseopt_gpu import TOL, CAM5
    assert np.allclose(np.float32(CAM5), run.rec("pose", 0, "cam5", np.float32))
    r = po.pose_optimization(fr["pose"], fr["world_pos"], fr["obs"], fr["inv_sigma2"], np.float32(CAM5))
    assert g["rounds"] == r["rounds"] and abs(g["iterations"] - r["iterations"]) <= 2 and abs(g["trials"] - r["trials"]) <= 4
    assert np.abs(g["pose"] - r["pose"]).max() < TOL
    assert abs(g["inliers"] - r["inliers"]) <= 1 and int((g["outlier"] != r["outlier"]).sum()) <= 1
    if case == "mixed_40pct_outliers":
        assert e_out.sum() > 0.3 * len(f)


# ---------------------------------------------------------------------------------------------------------------------------------
# Optimizer::LocalInertialBA over the mock maps of tests/test_host_liba_vs_ref.py
# ---------------------------------------------------------------------------------------------------------------------------------
def _liba_cases():
    from test_host_liba_vs_ref import CASES
    return sorted(CASES)


@pytest.mark.parametrize("name", _liba_cases())
def test_local_inertial_ba(tmp_path, name):
    from test_host_liba_vs_ref import CASES, write_case
    from test_liba_gpu import check
    c = dict(CASES[name])
    Wn = synth.inertial_window(keep_pre=True, **c.pop("win"))
    n_opt = c.pop("n_opt")
    corrupt = c.pop("corrupt", 0.0)
    failed = c.pop("nan_point", False)
    if failed:
        Wn["point"][17, 1] = np.nan
    if corrupt:
        rng = np.random.default_rng(11)
        sel = rng.random(len(Wn["obs"])) < corrupt
        Wn["obs"][sel, :2] += rng.normal(0, 25, (int(sel.sum()), 2))
    d = str(tmp_path)
    arr = write_case(d, Wn, n_opt, **c)
    with open(os.path.join(d, "unit.txt"), "w") as f:
        f.write("liba")
    r = subprocess.run([BIN, d], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "host_units ok" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
    rd = lambda n, t: np.fromfile(os.path.join(d, n), t)
    rc = lambda f, t: rd(f"rec_liba0_{f}", t)
    assert not os.path.exists(os.path.join(d, "rec_liba1_status"))
    nK, nM, nE, nL = rc("sizes", np.int32)
    scal = rc("scal", np.float64)
    # (a) the device solve against the oracle on the recorded problem
    ref = po.liba(rc("state", np.float64).reshape(nK, 21), rc("fixed", np.uint8), rc("point", np.float64).reshape(nM, 3), rc("edge_kf", np.int32),
                  rc("edge_mp", np.int32), rc("obs", np.float64).reshape(nE, 3), rc("inv_sigma2", np.float64), rc("Tcb", np.float64), scal[1:6],
                  rc("links", np.uint8).view(po.LIBA_LINK), scal[6], int(scal[7]))
    st = rc("stats", np.float64)
    got = dict(state=rc("state_out", np.float64).reshape(nK, 21), point=rc("point_out", np.float64).reshape(nM, 3), iterations=int(st[0]), trials=int(st[1]),
               chi2=st[3])
    assert scal[6] == (1e-2 if c.get("large") else 1.0) and int(scal[7]) == (4 if c.get("large") else 10)
    if not failed:                                             # a NaN window: nothing to compare but the failure rule below
        check(got, ref)
    # (b) the links the unit built: EdgeInertial's information from the keyframe's preintegration (inverse of C's 9 x 9 block, symmetrised),
    # scaled by 1e-2 and made robust on the oldest link of the window (Optimizer.cc:2467-2479), robust on every link with bRecInit
    st0 = rc("state", np.float64).reshape(nK, 21)
    kmap = [int(np.argmin(np.abs(Wn["state"][:, 9:12] - st0[i, 9:12]).sum(1))) for i in range(nK)]     # problem keyframe -> map keyframe
    links = rc("links", np.uint8).view(po.LIBA_LINK)
    oldest = min(kmap[int(L["k2"])] for L in links)
    for L in links:
        k2 = kmap[int(L["k2"])]
        assert kmap[int(L["k1"])] == k2 - 1
        Ci = np.linalg.inv(np.asarray(Wn["pre"][k2 - 1]["C"], np.float32).astype(np.float64).reshape(15, 15)[:9, :9])
        want = (Ci + Ci.T) / 2 * (1e-2 if k2 == oldest else 1.0)
        assert np.abs(L["info"].reshape(9, 9) - want).max() <= 1e-4 * np.abs(want).max(), (k2, oldest)
        assert L["robust"] == int(k2 == oldest or bool(c.get("rec_init")))
    # the write-back from the recorded answer, per object: problem keyframe i is map keyframe kmap[i], problem point p is the map point
    # whose float position it was given (pmap[p])
    nKF, nMP = len(Wn["state"]), len(arr["point"])
    cnt = rd("out_counters.i32", np.int32)
    per_kf = cnt[5:].reshape(nKF, 6)
    pose = rd("out_pose.f32", np.float32).reshape(nKF, 7)
    vel, bias = rd("out_vel.f32", np.float32).reshape(nKF, 3), rd("out_bias.f32", np.float32).reshape(nKF, 6)
    pt, upd, alive = rd("out_point.f32", np.float32).reshape(-1, 3), rd("out_updates.i32", np.int32), rd("out_alive.i32", np.int32)
    pose_in = np.stack([np.concatenate([unit_quat(q[:4]), q[4:]]) for q in arr["kf_pose"]])    # mock_Tcw as the map holds it
    if failed:                                                 # "FAIL LOCAL-INERTIAL BA": nothing written or erased, the marks left set
        assert cnt[4] == 0 and upd.sum() == 0 and (per_kf[:, :3] == 0).all() and (alive == 3).all()
        assert (per_kf[1:n_opt + 1, 4] == 100 + n_opt).all()
        assert (pose.view(np.uint32) == pose_in.view(np.uint32)).all() and (pt.view(np.uint32) == arr["point"].view(np.uint32)).all()
        return
    assert cnt[4] == 1
    fixed = rc("fixed", np.uint8)
    N = int((fixed == 0).sum())
    assert (fixed[:N] == 0).all()                              # optimisable keyframes first
    Tcb = rc("Tcb", np.float64)
    Rcb, tcb = Tcb[:9].reshape(3, 3), Tcb[9:]
    free = {kmap[i]: i for i in range(N)}
    for k in range(nKF):
        if k not in free:                                      # fixed keyframes and keyframes outside the window: untouched
            assert per_kf[k, 0] == 0 and per_kf[k, 1] == 0 and per_kf[k, 2] == 0
            assert (pose[k].view(np.uint32) == pose_in[k].view(np.uint32)).all()
            assert (vel[k] == arr["kf_vel"][k]).all() and (bias[k] == arr["kf_bias"][k]).all()
            continue
        S, S0 = got["state"][free[k]], st0[free[k]]
        assert list(per_kf[k, :3]) == [1, 1, 1] and per_kf[k, 4] == 0 and per_kf[k, 5] == 0
        # SetPose: ImuCamPose::Update, Rcw = Rcb Rbw, tcw = Rcb tbw + tcb, cast to float (a vertex no step moved keeps the keyframe's pose)
        if (S[:12] != S0[:12]).any():
            Rbw = S[:9].reshape(3, 3).T
            Rcw, tcw = Rcb @ Rbw, Rcb @ (-(Rbw @ S[9:12])) + tcb
        else:
            Rcw, tcw = quat_to_R(pose_in[k]), pose_in[k, 4:].astype(np.float64)
        # the float quaternion Sophus takes from the float rotation matrix: held to float rounding (1e-6), far below what the wrong
        # keyframe's solution or a transposed rotation would give
        assert np.abs(quat_to_R(pose[k]) - Rcw).max() < 1e-6 and np.abs(pose[k, 4:] - tcw).max() < 1e-6, k
        assert (vel[k].view(np.uint32) == S[12:15].astype(np.float32).view(np.uint32)).all()                       # SetVelocity
        assert (bias[k].view(np.uint32) == S[[18, 19, 20, 15, 16, 17]].astype(np.float32).view(np.uint32)).all()   # SetNewBias(acc, gyro)
    key = {arr["point"][j].tobytes(): j for j in range(nMP)}
    p_in = rc("point", np.float64).reshape(nM, 3)
    pmap = np.array([key[p_in[p].astype(np.float32).tobytes()] for p in range(nM)])
    assert (upd[pmap] == 1).all() and upd.sum() == nM                                                      # UpdateNormalAndDepth once each
    assert (pt[pmap].view(np.uint32) == got["point"].astype(np.float32).view(np.uint32)).all()               # SetWorldPos
    others = np.setdiff1d(np.arange(nMP), pmap)
    assert (pt[others].view(np.uint32) == arr["point"][others].view(np.uint32)).all()
    # erasures (:2690-2726) from the recorded chi2 / depth flags: monocular edges against 5.991 (1.5x that for points closer than 10 m, or
    # behind the camera), stereo edges against 7.815; both links of an erased edge are gone, every other edge keeps both
    obs, chi2, dpos = rc("obs", np.float64).reshape(nE, 3), rc("edge_chi2", np.float64), rc("edge_depth_positive", np.uint8)
    ekf, emp = rc("edge_kf", np.int32), rc("edge_mp", np.int32)
    mono2, stereo2 = np.float32(5.991), np.float32(7.815)
    edge_of = {}
    for e in range(len(arr["edge_kf"])):
        edge_of.setdefault((int(arr["edge_kf"][e]), int(arr["edge_mp"][e])), []).append(e)
    want_alive = np.full(len(alive), 3, np.int32)
    for e in range(nE):
        mp = int(pmap[emp[e]])
        if obs[e, 2] < 0:
            close = arr["point_track_depth"][mp] < np.float32(10)
            erase = (chi2[e] > mono2 and not close) or (chi2[e] > np.float32(1.5) * mono2 and close) or not dpos[e]
        else:
            erase = chi2[e] > stereo2
        if erase:
            want_alive[edge_of[(kmap[int(ekf[e])], mp)]] = 0
    assert (alive == want_alive).all()
