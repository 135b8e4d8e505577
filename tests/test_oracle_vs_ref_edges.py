"""CPU tier, build container only: the oracle's reprojection edges against the reference's OWN.
oracle/_ref/liborb_ref7.so holds EdgeStereoSE3ProjectXYZ / EdgeStereoSE3ProjectXYZOnlyPose ::cam_project and ::linearizeOplus
(Thirdparty/g2o/g2o/types/types_six_dof_expmap.cpp), EdgeSE3ProjectXYZ / EdgeSE3ProjectXYZOnlyPose ::linearizeOplus
(src/OptimizableTypes.cpp) and Pinhole::projectJac / project (src/CameraModels/Pinhole.cpp), cut out of /root/reference at build time and
compiled verbatim.  Equality is on the bits of every Jacobian entry and residual: which expression goes where, its association, and the
float / double types of the stereo projection (`const float invz = 1.0f/z` is a double division rounded to float; the binary edge's
`bf*invz` is a float product, the pose-only edge's a double one).

The device kernels evaluate the stereo projection slightly differently (float(z) first, a float division, double products; csrc/lba.cu,
csrc/poseopt.cu) -- a deviation this pin found.  The oracle reproduces that arithmetic under set_stereo_form(1), which is what the GPU
tier compares the kernels with (tests/conftest.py), and the tests at the bottom bound the distance between the two forms on the GPU
tier's own problems: that distance is part of the device's distance from the reference and has to stay inside the 1e-4 bar."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth

pytestmark = pytest.mark.skipif(po.build_ref7() is None, reason="oracle/_ref part 7 not built and /root/reference absent")
CAM5 = np.array([435.2, 435.2, 320.0, 240.0, 47.9], np.float32)
HERE = os.path.dirname(os.path.abspath(__file__))


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _cases(seed, n, zlo, zhi):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        q = rng.normal(0, 1, 4)
        q /= np.linalg.norm(q)
        pose = np.concatenate([q, rng.normal(0, 0.5, 3)])
        x, y, z, w = q
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        pc = np.array([rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(zlo, zhi)])
        yield pose, R.T @ (pc - pose[4:]), rng


@pytest.mark.parametrize("zlo,zhi", [(0.3, 3.0), (2.0, 40.0), (40.0, 4000.0), (-5.0, -0.5)])
def test_binary_edges_bitwise(zlo, zhi):
    """LocalBundleAdjustment's edges: _jacobianOplusXi (point), _jacobianOplusXj (pose) and the error, monocular and stereo; also behind the
    camera, where the optimiser still evaluates them (isDepthPositive is asked afterwards)."""
    for pose, X, rng in _cases(1, 1500, zlo, zhi):
        for obs in (np.array([rng.uniform(0, 640), rng.uniform(0, 480), -1.0]), np.array([rng.uniform(0, 640), rng.uniform(0, 480), rng.uniform(0, 600)])):
            A, B, r = po.ref7_edge(pose, X, obs, CAM5, unary=False)
            A2, B2, r2 = po.edge(pose, X, obs, CAM5)
            assert (_bits(A) == _bits(A2)).all() and (_bits(B) == _bits(B2)).all() and (_bits(r) == _bits(r2)).all(), (pose, X, obs)


@pytest.mark.parametrize("zlo,zhi", [(0.3, 3.0), (2.0, 40.0), (40.0, 4000.0), (-5.0, -0.5)])
def test_pose_only_edges_bitwise(zlo, zhi):
    """PoseOptimization's edges: the stereo one is written with reciprocals (invz, invz_2), not the binary edge's quotients."""
    differs = 0
    for pose, X, rng in _cases(2, 1500, zlo, zhi):
        for obs in (np.array([rng.uniform(0, 640), rng.uniform(0, 480), -1.0]), np.array([rng.uniform(0, 640), rng.uniform(0, 480), rng.uniform(0, 600)])):
            _, B, r = po.ref7_edge(pose, X, obs, CAM5, unary=True)
            D, B2, r2 = po.pose_edge(pose, X, obs, CAM5)
            assert D == len(r) and (_bits(B) == _bits(B2)).all() and (_bits(r) == _bits(r2)).all(), (pose, X, obs)
            if D == 3:
                differs += int((_bits(B) != _bits(po.edge(pose, X, obs, CAM5)[1])).any())
    assert differs > 100          # the two stereo Jacobians are different roundings of the same derivative: the test can tell them apart


def test_device_form_is_the_round_1_oracle():
    """set_stereo_form(1) is the arithmetic the kernels were validated against on the GPU: it reproduces, bit for bit, the vectors the
    golden file held before the pin (kept under *_devform)."""
    G = np.load(os.path.join(HERE, "golden", "golden_v1.npz"))
    pr = {k[7:]: G[k] for k in G.files if k.startswith("lba_in_")}
    prev = po.set_stereo_form(1)
    try:
        r = po.lba(pr["pose"], pr["fixed"], pr["point"], pr["edge_kf"], pr["edge_mp"], pr["obs"], pr["inv_sigma2"], pr["cam5"], 0.0, 10)
    finally:
        po.set_stereo_form(prev)
    assert (_bits(r["pose"]) == _bits(G["lba_pose_devform"])).all() and (_bits(r["point"]) == _bits(G["lba_point_devform"])).all()
    assert prev == 0 and po.set_stereo_form(0) == 0
    G2 = np.load(os.path.join(HERE, "golden", "golden_v2.npz"))          # ... and the pose optimisation of golden_v2 likewise
    assert not (_bits(G2["po_pose"]) == _bits(G2["po_pose_devform"])).all()
    assert (G2["po_outlier"] == G2["po_outlier_devform"]).all() and (G2["po_stats"][:2] == G2["po_stats_devform"][:2]).all()
    assert np.abs(G2["po_pose"] - G2["po_pose_devform"]).max() < 2e-6


def _both_forms(fn):
    out = []
    for form in (0, 1):
        prev = po.set_stereo_form(form)
        try:
            out.append(fn())
        finally:
            po.set_stereo_form(prev)
    return out


@pytest.mark.parametrize("kw,lam", [(dict(seed=0), 0.0), (dict(seed=2), 100.0), (dict(n_kf=8, n_fixed=3, n_mp=400, seed=6, mono_frac=0.0, outlier_frac=0.1), 100.0),
                                    (dict(n_kf=32, n_fixed=2, n_mp=1500, seed=7), 0.0), (dict(n_kf=12, n_fixed=2, n_mp=900, seed=23), 100.0),
                                    (dict(n_kf=5, n_fixed=1, n_mp=200, seed=5, mono_frac=1.0, outlier_frac=0.0), 0.0)])
def test_device_stereo_form_bound_local_ba(kw, lam):
    """tests/test_lba_gpu.py's problems in both forms: same LM iterations, trials and outlier classification; keyframe poses within 1e-6;
    points within 1e-4 (the far two-view points move by tens of micrometres along the ray for a 6e-8 relative change of the disparity)."""
    pr = synth.lba_problem(**kw)
    a, b = _both_forms(lambda: po.lba(pr["pose"], pr["fixed"], pr["point"], pr["edge_kf"], pr["edge_mp"], pr["obs"], pr["inv_sigma2"], pr["cam5"], lam, 10))
    assert (a["iterations"], a["trials"]) == (b["iterations"], b["trials"])
    assert np.abs(a["pose"] - b["pose"]).max() < 1e-6 and np.abs(a["point"] - b["point"]).max() < 1e-4
    assert np.median(np.abs(a["point"] - b["point"]).max(1)) < 2e-6
    thr = np.where(pr["obs"][:, 2] < 0, 5.991, 7.815)
    assert ((a["edge_chi2"] > thr) == (b["edge_chi2"] > thr)).all() and (a["edge_depth_pos"] == b["edge_depth_pos"]).all()
    if kw.get("mono_frac") == 1.0:          # no stereo edge: the forms are the same arithmetic
        assert (_bits(a["pose"]) == _bits(b["pose"])).all() and (_bits(a["point"]) == _bits(b["point"])).all()


def test_device_stereo_form_bound_pose_optimization():
    """tests/test_poseopt_gpu.py's frames in both forms: same rounds, inliers and outlier flags, poses within 2e-6.  (The LM trial counts of
    converged rounds are rounding noise -- they differ by tens between the forms -- which is why the GPU tier bounds them loosely.)"""
    spec = importlib.util.spec_from_file_location("_tp", os.path.join(HERE, "test_poseopt_gpu.py"))
    tp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tp)
    frames = [tp.make_frame(s, n) for s, n in [(0, 600), (1, 1200), (2, 300), (3, 550), (4, 2000), (5, 64)]]
    frames += [tp.make_frame(6, 500, mono_frac=1.0), tp.make_frame(7, 500, mono_frac=0.0, outlier_frac=0.4), tp.make_frame(8, 400, motion=4.0),
               tp.make_frame(11, 9, outlier_frac=0.0), tp.make_frame(12, 100)]
    for f in frames:
        a, b = _both_forms(lambda: po.pose_optimization(f["pose"], f["world_pos"], f["obs"], f["inv_sigma2"], np.float32(tp.CAM5)))
        assert a["rounds"] == b["rounds"] and a["inliers"] == b["inliers"] and (a["outlier"] == b["outlier"]).all()
        assert np.abs(a["pose"] - b["pose"]).max() < 2e-6
