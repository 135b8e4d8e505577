"""CPU tier: local-BA windows shaped like the ones LocalMapping hands to Optimizer::LocalBundleAdjustment, and the oracle on them.

synth.lba_problem (bench.py's and the golden vectors' generator) gives every point 4-8 observations from keyframes at most 6 apart
and is kept bit-stable.  window() below covers what it does not: covisibility windows of up to 160 free keyframes, long
observation tails (a landmark tracked over tens of keyframes), fixed keyframes between the free ones, and three shapes the
reference produces:
  * a free keyframe without edges (its points were just culled; g2o leaves the vertex out of the optimisation),
  * points whose edges all go to fixed keyframes (the initial keyframe, which Optimizer.cc fixes, is in the window),
  * points with a single stereo edge (MapPoint::nObs counts a stereo observation twice, so MapPointCulling keeps them).
It never makes a point with a single monocular edge (nObs <= 2 is culled) or a window without free keyframes (the new keyframe
is never the initial one).  tests/test_lba_windows_gpu.py runs the device on the cases listed in CASES."""
import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200.synth import _quat_from_rotvec, _quat_mul, _quat_rot

FX, FY, CX, CY, BF, W, H = 435.2, 435.2, 320.0, 240.0, 47.9, 640, 480


def _R(q):
    return _quat_rot(q, np.eye(3)).T     # rows of R(q): _quat_rot(q, v) = v @ R.T


def _observe(Rs, ts, X):
    """Pixel (u, v, ur) and depth of world point X in every keyframe of Rs / ts."""
    pc = np.einsum("kij,j->ki", Rs, X) + ts
    z = pc[:, 2]
    zs = np.where(z > 0.5, z, 1.0)
    u, v = FX * pc[:, 0] / zs + CX, FY * pc[:, 1] / zs + CY
    ur = u - BF / zs
    vis = (z > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H) & (ur > 0)
    return u, v, ur, vis


def window(n_free, n_fixed, n_mp, seed, span=20, max_obs=40, p_tail=0.14, mono_frac=0.1, outlier_frac=0.03, edgeless_kf=False,
           fixed_only_points=0, single_stereo_points=0):
    """A local-BA window in synth.lba_problem's dict layout (Optimizer._pack and po.lba take it as is).

    n_free + n_fixed keyframes (+1 free keyframe when edgeless_kf) on a slow sideways / forward trajectory, so that a point stays
    in view over +-span keyframes; the fixed ones sit at random places along it.  Each of the n_mp points is anchored in one
    keyframe and tracked over the nearest keyframes that see it: 2 + a geometric(p_tail) number of observations, capped at
    max_obs (the cap bounds the tail, not the mean).  Edge noise, 10 % monocular edges, 3 % gross outliers and the pose / point
    perturbations follow synth.lba_problem.  Then, by flag: one free keyframe no point observes (its index in "edgeless_kf"),
    fixed_only_points points observed only by fixed keyframes ("fixed_only_mp"), single_stereo_points points with one stereo
    edge to a free keyframe ("single_stereo_mp").  Points and edges are in random order."""
    assert n_free >= 1, "the reference never runs local BA without a free keyframe"
    rng = np.random.default_rng(seed)
    n_kf = n_free + n_fixed + int(edgeless_kf)
    Tq, Tt = [], []
    for k in range(n_kf):
        q = _quat_from_rotvec(np.array([0.01 * np.sin(k / 7.0), np.deg2rad(4.0) * np.sin(k / 15.0), 0.0]))
        c = np.array([0.04 * k, 0.02 * np.sin(k / 5.0), 0.03 * k])      # camera centre in the world
        Tq.append(q)
        Tt.append(-_quat_rot(q, c))
    Tq, Tt = np.array(Tq), np.array(Tt)
    Rs = np.array([_R(q) for q in Tq])
    fixed = np.zeros(n_kf, np.uint8)
    fixed[rng.choice(n_kf, n_fixed, replace=False)] = 1
    edgeless = -1
    if edgeless_kf:
        edgeless = int(rng.choice(np.flatnonzero(fixed == 0)))
    usable = np.arange(n_kf) != edgeless
    scales = 1.2 ** np.arange(8)

    def make_point(anchors, allowed, nobs, stereo_only=False):
        """One point anchored in a random keyframe of `anchors`, seen by the nobs nearest `allowed` keyframes within +-span
        (fewer when fewer see it; None when that leaves a multi-edge point with fewer than two)."""
        k0 = int(rng.choice(anchors))
        z = rng.uniform(2.0, 15.0)
        u, v = rng.uniform(30, W - 30), rng.uniform(30, H - 30)
        X = _quat_rot(Tq[k0] * np.array([-1, -1, -1, 1]), np.array([(u - CX) * z / FX, (v - CY) * z / FY, z]) - Tt[k0])
        cand = np.flatnonzero(allowed & (np.abs(np.arange(n_kf) - k0) <= span))
        cand = cand[np.lexsort((rng.random(len(cand)), np.abs(cand - k0)))]     # nearest first, ties in random order
        uu, vv, ur, vis = _observe(Rs[cand], Tt[cand], X)
        seen = np.flatnonzero(vis)[:nobs]
        if len(seen) < min(nobs, 2):
            return None
        edges = []
        for i in sorted(seen):
            octave = int(rng.integers(0, 8))
            sig = scales[octave]
            n = rng.normal(0, sig, 3)
            if rng.random() < outlier_frac:
                n += rng.choice([-1, 1], 3) * 20.0
            mono = (not stereo_only) and rng.random() < mono_frac
            edges.append((int(cand[i]), np.float32(uu[i] + n[0]), np.float32(vv[i] + n[1]), -1.0 if mono else np.float32(ur[i] + n[2]),
                          np.float32(1.0 / np.float32(sig * sig))))
        return X, edges

    pts, edges_of, kinds = [], [], []
    free_kf = np.flatnonzero((fixed == 0) & usable)
    tries = 0
    while len(pts) < n_mp:
        tries += 1
        assert tries < 50 * n_mp, "trajectory too short for the requested points"
        nobs = min(max_obs, 1 + int(rng.geometric(p_tail)))
        r = make_point(np.flatnonzero(usable), usable, nobs)
        if r is not None:
            pts.append(r[0]); edges_of.append(r[1]); kinds.append(0)
    for kind, count, anchors, allowed in ((1, fixed_only_points, np.flatnonzero(fixed == 1), fixed == 1),
                                          (2, single_stereo_points, free_kf, (fixed == 0) & usable)):
        made = 0
        while made < count:
            tries += 1
            assert tries < 50 * (n_mp + fixed_only_points + single_stereo_points), "cannot place the requested points"
            nobs = 1 if kind == 2 else min(max_obs, 1 + int(rng.geometric(p_tail)))
            r = make_point(anchors, allowed, nobs, stereo_only=(kind == 2))
            if r is not None:
                pts.append(r[0]); edges_of.append(r[1]); kinds.append(kind); made += 1
    order = rng.permutation(len(pts))                  # points in random order: the injected ones are spread over the warps
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    ekf, emp, obs, inv_s2 = [], [], [], []
    for l, es in enumerate(edges_of):
        for (k, uu, vv, ur, w) in es:
            ekf.append(k); emp.append(int(rank[l])); obs.append([uu, vv, ur]); inv_s2.append(w)
    eperm = rng.permutation(len(ekf))
    pts_gt = np.array(pts)[order]
    kinds = np.array(kinds)[order]
    pose = np.zeros((n_kf, 7))
    for k in range(n_kf):
        q, t = Tq[k], Tt[k]
        if not fixed[k]:
            q = _quat_mul(_quat_from_rotvec(rng.normal(0, np.deg2rad(0.2), 3)), q)
            t = t + rng.normal(0, 0.01, 3)
        q = q / np.linalg.norm(q)
        if q[3] < 0:
            q = -q
        pose[k, :4], pose[k, 4:] = q, t
    point = (pts_gt + rng.normal(0, 0.02, pts_gt.shape)).astype(np.float32).astype(np.float64)
    return dict(pose=pose.astype(np.float32).astype(np.float64), fixed=fixed, point=point,
                edge_kf=np.array(ekf, np.int32)[eperm], edge_mp=np.array(emp, np.int32)[eperm], obs=np.array(obs, np.float64)[eperm],
                inv_sigma2=np.array(inv_s2, np.float64)[eperm],
                cam5=np.array([np.float32(FX), np.float32(FY), np.float32(CX), np.float32(CY), np.float32(BF)], np.float64),
                pose_gt=np.concatenate([Tq, Tt], 1), point_gt=pts_gt, edgeless_kf=edgeless,
                fixed_only_mp=np.flatnonzero(kinds == 1), single_stereo_mp=np.flatnonzero(kinds == 2))


# The windows the GPU tier runs (tests/test_lba_windows_gpu.py), by name: window() keyword arguments.
CASES = {
    "40free_tail40": dict(n_free=40, n_fixed=20, n_mp=3000, seed=101, max_obs=40),
    "100free": dict(n_free=100, n_fixed=30, n_mp=6000, seed=102, max_obs=30),
    "24free": dict(n_free=24, n_fixed=6, n_mp=2000, seed=103, max_obs=30),     # n = 144: the largest system factorised in shared memory
    "25free": dict(n_free=25, n_fixed=6, n_mp=2000, seed=104, max_obs=30),     # n = 150: the smallest one factorised in global memory
    "160free": dict(n_free=160, n_fixed=20, n_mp=8000, seed=105, max_obs=30),  # n = 960: the largest the library accepts
    "edgeless_kf": dict(n_free=12, n_fixed=4, n_mp=1000, seed=106, edgeless_kf=True),
    "fixed_only_points": dict(n_free=10, n_fixed=8, n_mp=1000, seed=107, fixed_only_points=150),
    "single_stereo_points": dict(n_free=10, n_fixed=3, n_mp=1000, seed=108, single_stereo_points=150),
}


def oracle(pr, lam, iters=10):
    return po.lba(pr["pose"], pr["fixed"], pr["point"], pr["edge_kf"], pr["edge_mp"], pr["obs"], pr["inv_sigma2"], pr["cam5"], lam, iters)


def _nobs(pr):
    return np.bincount(pr["edge_mp"], minlength=len(pr["point"]))


def test_observation_tail():
    pr = window(60, 20, 4000, seed=1, max_obs=40)
    nobs = _nobs(pr)
    assert nobs.min() >= 2 and nobs.max() == 40
    assert (nobs > 8).sum() > 800 and (nobs > 20).sum() > 50, np.bincount(nobs)
    assert len(pr["edge_kf"]) > 25000
    # a landmark has at most one edge per keyframe
    assert len(np.unique(pr["edge_mp"].astype(np.int64) * len(pr["pose"]) + pr["edge_kf"])) == len(pr["edge_kf"])
    # cases with a tighter cap reach it, and a window shorter than the cap is bounded by its keyframes
    assert _nobs(window(**CASES["24free"])).max() == 30
    assert _nobs(window(5, 2, 300, seed=3, max_obs=40)).max() == 7


@pytest.mark.parametrize("case", list(CASES))
def test_named_cases_have_long_tails(case):
    """Every GPU-tier window keeps points past one and two rounds of build_points' 8-lane loop (> 8, > 16 observations), and
    the windows that set max_obs reach it (40free_tail40: past four rounds, > 32)."""
    kw = CASES[case]
    nobs = _nobs(window(**kw))
    assert (nobs > 8).sum() >= 300
    if "max_obs" in kw:
        assert nobs.max() == kw["max_obs"] and (nobs > 16).sum() >= 150
    if kw.get("max_obs") == 40:
        assert (nobs > 32).sum() >= 10


def test_edges_are_noisy_projections_of_the_ground_truth():
    pr = window(30, 10, 2000, seed=2)
    R = np.array([_R(q) for q in pr["pose_gt"][:, :4]])
    pc = np.einsum("eij,ej->ei", R[pr["edge_kf"]], pr["point_gt"][pr["edge_mp"]]) + pr["pose_gt"][pr["edge_kf"], 4:]
    assert (pc[:, 2] > 0.5).all()
    u, v = FX * pc[:, 0] / pc[:, 2] + CX, FY * pc[:, 1] / pc[:, 2] + CY
    sig = 1.0 / np.sqrt(pr["inv_sigma2"])
    assert set(np.round(sig ** 2, 3)) <= set(np.round(np.float32(1.2) ** (2 * np.arange(8)), 3))
    mono = pr["obs"][:, 2] < 0
    assert 0.07 < mono.mean() < 0.13
    ru = np.abs(pr["obs"][:, 0] - u) / sig
    rr = np.abs(pr["obs"][~mono, 2] - (u - BF / pc[:, 2])[~mono]) / sig[~mono]
    assert np.median(ru) < 1.0 and (ru > 20 / sig - 5).mean() > 0.01
    outl = np.abs(pr["obs"][:, 1] - v) / sig > 6
    assert 0.015 < outl.mean() < 0.045           # 3 % gross outliers of 20 px (the ones at octave 7 hide in the noise)
    assert np.median(rr) < 1.0


def test_fixed_flags_and_edges_per_keyframe():
    pr = window(12, 5, 800, seed=4, edgeless_kf=True)
    n_kf = len(pr["pose"])
    assert n_kf == 18 and pr["fixed"].sum() == 5 and pr["fixed"].dtype == np.uint8
    k = pr["edgeless_kf"]
    assert 0 <= k < n_kf and pr["fixed"][k] == 0
    per_kf = np.bincount(pr["edge_kf"], minlength=n_kf)
    assert per_kf[k] == 0 and (np.delete(per_kf, k) > 0).all()
    assert per_kf.sum() == len(pr["edge_kf"])
    # fixed keyframes are spread along the trajectory, not only at its start
    assert np.flatnonzero(pr["fixed"]).max() > 5
    # fixed keyframes keep their ground-truth pose (rounded to float32 like the map); free ones are perturbed
    fx = pr["fixed"] == 1
    assert np.abs(pr["pose"][fx, 4:] - pr["pose_gt"][fx, 4:]).max() < 1e-6
    assert np.abs(pr["pose"][~fx, 4:] - pr["pose_gt"][~fx, 4:]).max() > 1e-3
    assert window(12, 5, 800, seed=4)["edgeless_kf"] == -1


def test_injected_points():
    pr = window(**CASES["fixed_only_points"])
    fo = pr["fixed_only_mp"]
    assert len(fo) == 150
    sel = np.isin(pr["edge_mp"], fo)
    assert (pr["fixed"][pr["edge_kf"][sel]] == 1).all()
    assert (_nobs(pr)[fo] >= 2).all()
    # (tracked points near fixed keyframes can end up fixed-only too)
    has_free = np.zeros(len(pr["point"]), bool)
    has_free[pr["edge_mp"][pr["fixed"][pr["edge_kf"]] == 0]] = True
    assert not has_free[fo].any() and (~has_free).sum() >= 150

    pr = window(**CASES["single_stereo_points"])
    ss = pr["single_stereo_mp"]
    nobs = _nobs(pr)
    assert len(ss) == 150 and (nobs[ss] == 1).all()
    assert (np.flatnonzero(nobs == 1) == np.sort(ss)).all()        # the only single-edge points, ...
    sel = np.isin(pr["edge_mp"], ss)
    assert (pr["obs"][sel, 2] >= 0).all()                          # ... stereo (never a single monocular edge) ...
    assert (pr["fixed"][pr["edge_kf"][sel]] == 0).all()            # ... to free keyframes
    assert len(window(6, 2, 300, seed=9)["single_stereo_mp"]) == 0


def test_no_single_monocular_edge_points():
    for kw in CASES.values():
        pr = window(**kw)
        nobs = _nobs(pr)
        single = np.flatnonzero(nobs == 1)
        sel = np.isin(pr["edge_mp"], single)
        assert (pr["obs"][sel, 2] >= 0).all()
        assert (pr["fixed"] == 0).any()


def test_window_is_deterministic():
    a, b = window(8, 2, 300, seed=11), window(8, 2, 300, seed=11)
    for k in ("pose", "fixed", "point", "edge_kf", "edge_mp", "obs", "inv_sigma2"):
        assert (a[k] == b[k]).all()


@pytest.mark.parametrize("lam", [0.0, 100.0])
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reduces_chi2(case, lam):
    pr = window(**CASES[case])
    r = oracle(pr, lam)
    assert r["iterations"] >= 1 and np.isfinite(r["chi2"])
    assert r["chi2"] < r["chi2_init"]
    assert (r["pose"][pr["fixed"] == 1] == pr["pose"][pr["fixed"] == 1]).all()


def test_oracle_leaves_an_edgeless_keyframe_at_its_normalised_pose():
    """g2o leaves a vertex without edges out of the optimisation; the oracle keeps it in the reduced system, where its block is
    lambda * I with a zero right-hand side, so its update is exactly zero and the exp-map product only renormalises the quaternion."""
    pr = window(**CASES["edgeless_kf"])
    k = pr["edgeless_kf"]
    for lam in (0.0, 100.0):
        r = oracle(pr, lam)
        q = pr["pose"][k, :4]
        assert (r["pose"][k, :4] == q / np.sqrt(q @ q)).all(), (r["pose"][k, :4], q / np.sqrt(q @ q))
        assert (r["pose"][k, 4:] == pr["pose"][k, 4:]).all()
