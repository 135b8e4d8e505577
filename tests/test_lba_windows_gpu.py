"""GPU tier: k_lba (csrc/lba.cu) against the oracle on the windows of tests/test_lba_windows.py -- covisibility windows of up to
160 free keyframes, points observed by up to 40 keyframes, the three window shapes the reference produces and synth.lba_problem
does not, every cluster size the launcher can pick -- and the determinism DESIGN.md §12 claims: the same problem gives the same
bits run after run and wherever it sits in a batch; only the cluster size may change the order of the sums.

The oracle runs here in the device's stereo form (conftest); its results are computed in this module, never taken from the CPU
tier, which runs the reference's form."""
import functools

import numpy as np
import pytest

from orb_slam3_detailed_comments_b200 import Optimizer, OrbError
from test_lba_gpu import _compare
from test_lba_windows import CASES, _R, oracle, window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def opt():
    o = Optimizer(0)
    yield o
    o.close()


@functools.lru_cache(maxsize=None)
def case(name):
    return window(**CASES[name])


@functools.lru_cache(maxsize=None)
def ref(name, lam):
    return oracle(case(name), lam)


def _compare_small_lambda(g, r, pr, drift=1.0):
    """test_lba_gpu._compare with its per-edge chi2 bar (1e-6 + 1e-5 |chi2|) split by what the edge's arithmetic allows.

    A stereo edge's chi2 is a step function of depth: the reference's edge (and both implementations) takes
    invz = float(1 / float(z)), so two solutions whose depths differ by far less than the bar allows still differ by a whole
    float32 step of invz where float(z) rounds differently.  On such edges the gap may also hold the change of float32 invz
    between the two depths (`jump`, per edge below); on an H100 the device used at most 0.55 of one such step beyond the bar on
    these windows, one-ulp changes of the oracle's inputs reach 0.56.  On every edge the bar holds, times `drift`: after nine
    accepted steps from lambda 100, lambda is near 2e-3 and the oracle's own result moves by up to 4.9x the bar when its points
    and free poses move by one ulp (measured per case, values in DRIFT; 1 at lambda 0).  All other bars of _compare apply
    unchanged."""
    stereo = pr["obs"][:, 2] >= 0
    Xr, Xg = _camera(pr, r), _camera(pr, g)
    zr, zg = np.float32(Xr[:, 2]), np.float32(Xg[:, 2])
    flip = stereo & (zr != zg)
    assert flip.mean() < 0.1                                                                    # measured: up to 6.7 % (160free)
    cam = np.asarray(pr["cam5"], np.float64)
    invz = 1.0 / Xr[:, 2]
    step = np.abs(1.0 / zr - 1.0 / zg) + 2.0 ** -23 * invz      # the two float depths' reciprocals, each rounded by half an ulp
    slope = np.sqrt((Xr[:, 0] * cam[0]) ** 2 + (Xr[:, 1] * cam[1]) ** 2 + (Xr[:, 0] * cam[0] - cam[4]) ** 2)   # |d residual / d invz|
    res = np.sqrt(np.maximum(r["edge_chi2"], 0) / pr["inv_sigma2"])
    jump = pr["inv_sigma2"] * (2 * res * slope * step + (slope * step) ** 2)
    bar = 1e-6 + 1e-5 * np.abs(r["edge_chi2"])
    d = np.abs(g["edge_chi2"] - r["edge_chi2"])
    assert (d[~flip] <= drift * bar[~flip]).all(), float((d[~flip] / bar[~flip]).max())
    assert (d[flip] <= drift * bar[flip] + jump[flip]).all(), float(((d - drift * bar) / jump)[flip].max())
    _compare(dict(g, edge_chi2=r["edge_chi2"]), r, pr)                       # the remaining bars ...
    thr = np.where(pr["obs"][:, 2] < 0, 5.991, 7.815)                        # ... with the outlier classification on the device's chi2
    clear = np.abs(r["edge_chi2"] - thr) > 1e-6 * thr
    assert ((g["edge_chi2"] > thr) == (r["edge_chi2"] > thr))[clear].all()


def _camera(pr, res):
    R = np.array([_R(q) for q in res["pose"][:, :4]])
    return np.einsum("eij,ej->ei", R[pr["edge_kf"]], res["point"][pr["edge_mp"]]) + res["pose"][pr["edge_kf"], 4:]


# The oracle's own drift at lambda 100 on edges whose float32 depth does not change, in units of the per-edge chi2 bar, when its
# points and free poses move by one ulp (64 draws on 40free_tail40: 1.88; 12 on the others; 4 per batch window), rounded up.  The device
# on an H100: 1.71, 1.18, 0.52, 0.94, 3.87, 0.54, 1.09 / 2.04 (batches of 3 / 34).
DRIFT = {"40free_tail40": 1.9, "100free": 2.6, "24free": 1.6, "25free": 1.6, "160free": 4.9, "edgeless_kf": 1.4, "batch": 3.8}


def _same_bits(a, b):
    for k in ("pose", "point", "edge_chi2", "edge_depth_pos"):
        assert a[k].tobytes() == b[k].tobytes(), k
    for k in ("iterations", "trials", "chi2", "chi2_init", "lambda_"):
        assert np.float64(a[k]).tobytes() == np.float64(b[k]).tobytes(), (k, a[k], b[k])


# ---- 1. real-sized windows: both LDL^T paths (<= 24 free keyframes in shared memory, global memory beyond) up to the 160 limit
@pytest.mark.parametrize("lam", [0.0, 100.0])
@pytest.mark.parametrize("name", ["40free_tail40", "100free", "24free", "25free", "160free"])
def test_window_matches_oracle(opt, name, lam):
    pr = case(name)
    g, r = opt.LocalBundleAdjustment(pr, lambda_init=lam), ref(name, lam)
    if lam == 0.0:
        _compare(g, r, pr)
    else:
        _compare_small_lambda(g, r, pr, DRIFT[name])


# ---- 2. one free keyframe beyond the limit is refused, before any device work, and leaves the handle usable
def test_161_free_keyframes_are_refused(opt):
    big = window(161, 4, 2500, seed=109, max_obs=20)
    assert (big["fixed"] == 0).sum() == 161
    with pytest.raises(OrbError, match=r"^orb_status -5: more than 160 free keyframes"):
        opt.LocalBundleAdjustment(big)
    with pytest.raises(OrbError, match=r"^orb_status -5:"):
        opt.LocalBundleAdjustmentBatch([case("edgeless_kf"), big])
    pr = case("24free")
    _compare(opt.LocalBundleAdjustment(pr, lambda_init=0.0), ref("24free", 0.0), pr)


# ---- 3. window shapes the reference produces: an edgeless free keyframe, fixed-only points, single-stereo-edge points
@pytest.mark.parametrize("lam", [0.0, 100.0])
@pytest.mark.parametrize("name", ["edgeless_kf", "fixed_only_points", "single_stereo_points"])
def test_reference_window_shapes(opt, name, lam):
    pr = case(name)
    g = opt.LocalBundleAdjustment(pr, lambda_init=lam)
    if lam == 100.0 and name == "edgeless_kf":
        _compare_small_lambda(g, ref(name, lam), pr, DRIFT[name])
    else:
        _compare(g, ref(name, lam), pr)
    if name == "edgeless_kf":
        # g2o leaves the vertex out; the device keeps it with a lambda * I block and a zero right-hand side, so the update is zero
        # and each accepted step only renormalises the quaternion
        k = pr["edgeless_kf"]
        q = pr["pose"][k, :4]
        assert (g["pose"][k, 4:] == pr["pose"][k, 4:]).all()
        assert np.abs(g["pose"][k, :4] - q / np.sqrt(q @ q)).max() <= 8 * np.finfo(np.float64).eps


# ---- 4. every cluster size on one problem (ORB_LBA_CLUSTER caps the launcher's choice; it is read at every call)
@pytest.mark.parametrize("cluster", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("name,lam", [("40free_tail40", 0.0), ("40free_tail40", 100.0), ("24free", 0.0)])
def test_every_cluster_size(opt, monkeypatch, name, lam, cluster):
    monkeypatch.setenv("ORB_LBA_CLUSTER", str(cluster))
    pr = case(name)
    g, r = opt.LocalBundleAdjustment(pr, lambda_init=lam), ref(name, lam)
    if lam == 0.0:
        _compare(g, r, pr)
    else:
        _compare_small_lambda(g, r, pr, DRIFT[name])


# ---- 5. batches whose size selects each branch of the launcher (lba.cu: 16 CTAs per problem for <= 2 problems, then 8 / 4 / 2 / 1
# while n * CTAs fits the SMs)
def _branches():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [(2, 16), (3, 8), (sms // 8 + 1, 4), (sms // 4 + 1, 2), (sms // 2 + 1, 1)]


@functools.lru_cache(maxsize=None)
def _small_windows(n):
    """n small varied windows (4-12 keyframes, one more where an edgeless one is added; 150-400 points observed by up to all of
    them; some with single-stereo-edge points); the largest batch also holds one window above 24 free keyframes."""
    rng = np.random.default_rng(n)
    prs = []
    for i in range(n):
        n_fixed = int(rng.integers(1, 4))
        n_free = int(rng.integers(max(1, 4 - n_fixed), 13 - n_fixed))
        prs.append(window(n_free, n_fixed, int(rng.integers(150, 401)), seed=10000 + 100 * n + i, p_tail=0.1,
                          edgeless_kf=(i % 5 == 3 and n_free >= 2), single_stereo_points=(20 if i % 7 == 5 else 0)))
    if n == _branches()[-1][0]:
        prs[n // 3] = window(26, 4, 900, seed=10000 + 100 * n + n, max_obs=30)
    return prs


@pytest.mark.parametrize("branch", range(5))
def test_batch_sizes_select_every_cluster_size(opt, monkeypatch, branch):
    monkeypatch.delenv("ORB_LBA_CLUSTER", raising=False)
    size, _ = _branches()[branch]
    prs = _small_windows(size)
    lam = 100.0 if branch % 2 else 0.0
    assert len(prs) == size and (branch < 4 or max((p["fixed"] == 0).sum() for p in prs) > 24)
    for pr, g in zip(prs, opt.LocalBundleAdjustmentBatch(prs, lambda_init=lam)):
        _compare_small_lambda(g, oracle(pr, lam), pr, DRIFT["batch"] if lam else 1.0)


# ---- 6. determinism and batch independence, bit for bit: a problem solved alone at cluster size c, solved again, and solved first,
# in the middle and last of a batch whose size makes the launcher choose c
@pytest.mark.parametrize("probe", ["24free", "25free"])
@pytest.mark.parametrize("branch", range(5))
def test_bits_do_not_depend_on_run_or_batch(opt, monkeypatch, branch, probe):
    size, cs = _branches()[branch]
    pr, lam = case(probe), 0.0
    monkeypatch.setenv("ORB_LBA_CLUSTER", str(cs))
    alone = opt.LocalBundleAdjustment(pr, lambda_init=lam)
    _same_bits(alone, opt.LocalBundleAdjustment(pr, lambda_init=lam))
    _compare(alone, ref(probe, lam), pr)
    monkeypatch.delenv("ORB_LBA_CLUSTER")
    others = _small_windows(size)
    for pos in sorted({0, size // 2, size - 1}):
        prs = list(others)
        prs[pos] = pr
        _same_bits(alone, opt.LocalBundleAdjustmentBatch(prs, lambda_init=lam)[pos])
