"""CPU tier: LocalInertialBA windows shaped like the ones host/Optimizer_liba_b200.cc hands to liba_solve, the oracle on them, and the
device algorithm (csrc/liba_core.cuh built for the host, tests/test_liba_emul.py) against the oracle on them.

synth.inertial_window (bench.py's and the golden vectors' generator) is kept bit-stable.  It puts the temporal chain first, fixes a
prefix of the keyframes, and lets every keyframe that can see a point observe it.  window() below builds what the host unit builds
from a map instead (Optimizer_liba_b200.cc:59-196, after Optimizer.cc:2217-2660):
  * the temporal window: n_free optimisable keyframes (10, or 25 with bLarge) and the fixed keyframe before them, joined by inertial
    links preintegrated from synthetic 200 Hz IMU samples (synth.preintegrate, optimizer.link_information); the oldest link is
    robust and its information is scaled by 1e-2;
  * n_cov other keyframes of the map near the window, without links.  Walking the window's points in order, each point fixes its
    first observer that is neither in the window nor fixed yet, until 200 keyframes are fixed (maxFixKF).  After that a point keeps
    only its edges to keyframes already in the problem, so the cap leaves some points with a single edge;
  * points anchored in the window and seen by 2 + geometric(p_tail) keyframes, capped at max_obs: tracked points by the anchor's
    neighbours in the chain, then by the keyframes nearest in space; a share (revisit_frac) by the anchor and older keyframes only;
  * the arrays in the unit's order: free keyframes newest first, then the temporal fixed one, then the covisible ones in the order
    they were fixed; points in (window keyframe, feature) order; edges grouped by point, each point's in observation-map order.
Flags add the other shapes the unit produces: the keyframe order shuffled; a free keyframe with inertial links and no reprojection
edge (its points were culled); a free keyframe without a link to its predecessor ("NOT INERTIAL LINK TO PREVIOUS FRAME"); points
with a single monocular or stereo edge; every link robust (bRecInit); and the early map, where the window reaches the map's first
keyframe, which has no predecessor, so that keyframe becomes the fixed one (:84-94) and its own points join the window.
tests/test_liba_windows_gpu.py runs the device on the cases listed in CASES."""
import functools

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth
from orb_slam3_detailed_comments_b200._native import LIBA_LINK
from orb_slam3_detailed_comments_b200.optimizer import link_information
from test_liba_emul import TOL, emul, run_emul  # noqa: F401  (emul: the fixture)

FX, FY, CX, CY, BF, W, H = 435.2, 435.2, 320.0, 240.0, 47.9, 640, 480
RCB, TCB = synth._expm([0.01, -0.02, 0.015]), np.array([0.05, -0.01, 0.02])
MAX_FIX_KF = 200                # maxFixKF (Optimizer_liba_b200.cc:96): fixed keyframes of a window, the one before it included
ROLE_FREE, ROLE_TEMPORAL, ROLE_COVISIBLE = 0, 1, 2


def _camera(state, X):
    """Camera coordinates of world points X [n][3] in keyframes state [m][21]: [m][n][3]."""
    Rwb, twb = state[:, :9].reshape(-1, 3, 3), state[:, 9:12]
    Xb = np.einsum("kji,knj->kni", Rwb, X[None] - twb[:, None])
    return Xb @ RCB.T + TCB


def window(n_free, n_cov, n_mp, seed, max_obs=60, p_tail=0.12, revisit_frac=0.3, mono_frac=0.3, noise=0.5, outlier_frac=0.03,
           early_map=False, shuffle=False, links_only_kf=False, unlinked_kf=False, single_mono_points=0, single_stereo_points=0,
           rec_init=False):
    """A LocalInertialBA window in the dict layout InertialOptimizer.LocalInertialBA and po.liba take (see the module docstring).

    Metadata next to the arrays: "role" per keyframe (ROLE_*), "links_only_kf" / "unlinked_kf" (keyframe index or -1),
    "single_mono_mp" / "single_stereo_mp" (the injected single-edge points), "dropped" (observations the 200-keyframe cap dropped)."""
    assert n_free >= 1 and not (early_map and n_free > 2)
    rng = np.random.default_rng(seed)
    G = np.array([0, 0, -float(np.float32(9.81))])
    # ---- the temporal chain, oldest first (chain[0]: the fixed keyframe), as synth.inertial_window integrates it
    n_chain, dt, n_s = n_free + 1, 0.25, 50
    R, p, v = synth._expm(rng.normal(0, 0.2, 3)), rng.normal(0, 1, 3), rng.normal(0, 0.3, 3)
    chain, pres = [], []
    for c in range(n_chain):
        chain.append(np.concatenate([R.reshape(-1), p, v, np.zeros(6)]))
        if c == n_chain - 1:
            break
        tt = np.linspace(0, 1, n_s)[:, None]
        gyr = rng.normal(0, 0.1, 3) * (1 - tt) + rng.normal(0, 0.1, 3) * tt
        acc = rng.normal(0, 0.3, 3) * (1 - tt) + rng.normal(0, 0.3, 3) * tt - R.T @ G
        pre = synth.preintegrate(acc, gyr, dt / n_s)
        pres.append(pre)
        dT = pre["dT"]
        p, v = p + v * dT + 0.5 * G * dT * dT + R @ pre["dP"].astype(np.float64), v + G * dT + R @ pre["dV"].astype(np.float64)
        R = R @ pre["dR"].astype(np.float64)
    # ---- the map: the chain, then n_cov keyframes near it (older ones: they come first in observation-map order)
    cov = []
    for _ in range(n_cov):
        s = chain[rng.integers(0, n_chain)].copy()
        s[:9] = (s[:9].reshape(3, 3) @ synth._expm(rng.normal(0, 0.05, 3))).reshape(-1)
        s[9:12] += rng.normal(0, 0.3, 3)
        cov.append(s)
    kfs = np.array(chain + cov)
    n_map = len(kfs)
    age = np.empty(n_map, np.int64)                      # creation order: the map's other keyframes (in random order), then the chain
    age[n_chain:] = rng.permutation(n_cov)
    age[:n_chain] = n_cov + np.arange(n_chain)
    window_kf = list(range(n_chain - 1, 0 if not early_map else -1, -1))   # vOpt before the early map's pop: newest first
    links_only = n_chain - 1 - n_free // 2 if links_only_kf else -1        # a free keyframe no point observes
    unlinked = n_chain - 1 - (n_free - 1) // 2 if unlinked_kf else -1     # a free keyframe whose link to its predecessor is missing
    observer = np.arange(n_map) != links_only

    # ---- points: anchored in a window keyframe, seen by the nearest keyframes that see it
    scales = np.float32(1.2) ** np.arange(8)
    anchors = [k for k in window_kf if k != links_only]
    single_anchors = [k for k in range(1, n_chain) if k != links_only]
    centre = kfs[:, 9:12]
    pts, obs_of = [], []               # obs_of[i]: list of (map keyframe, u, v, ur, inv_sigma2)

    def make_point(k0, nobs, kind):
        z = rng.uniform(3.0, 10.0)
        uv = rng.uniform([30, 30], [W - 30, H - 30])
        Xc = np.array([(uv[0] - CX) * z / FX, (uv[1] - CY) * z / FY, z])
        X = kfs[k0, :9].reshape(3, 3) @ (RCB.T @ (Xc - TCB)) + kfs[k0, 9:12]
        if kind:
            seen = np.array([k0])
        else:
            Xc = _camera(kfs, X[None])[:, 0]
            zs = np.where(Xc[:, 2] > 0.5, Xc[:, 2], 1.0)
            u, vv = FX * Xc[:, 0] / zs + CX, FY * Xc[:, 1] / zs + CY
            vis = observer & (Xc[:, 2] > 0.5) & (u > 0) & (u < W) & (vv > 0) & (vv < H)
            cand = np.flatnonzero(vis)
            if rng.random() < revisit_frac:     # seen again by the anchor: the other observers are older keyframes, in any order
                cand = cand[(cand == k0) | (cand >= n_chain)]
                d = (cand != k0).astype(float)
            else:                               # tracked: the anchor, the chain nearest in time, then the keyframes nearest in space
                d = np.where(cand < n_chain, np.abs(cand - k0), n_chain + np.linalg.norm(centre[cand] - centre[k0], axis=1))
            seen = cand[np.lexsort((rng.random(len(cand)), d))][:nobs]      # ties in random order
            if len(seen) < 2:
                return False
        Xc = _camera(kfs[seen], X[None])[:, 0]
        obs = []
        for k, xc in zip(seen, Xc):
            level = int(rng.integers(0, 8))
            u, vv = FX * xc[0] / xc[2] + CX, FY * xc[1] / xc[2] + CY
            ur = u - BF / xc[2]
            n = rng.normal(0, noise, 3)
            if rng.random() < outlier_frac:
                n += rng.choice([-1, 1], 3) * 20.0
            mono = kind == 1 or (kind == 0 and (rng.random() < mono_frac or ur <= 0))
            obs.append((int(k), u + n[0], vv + n[1], -1.0 if mono else ur + n[2], float(1.0 / scales[level] ** 2)))
        pts.append(X)
        obs_of.append(obs)
        return True

    kinds = []
    for kind, count in ((0, n_mp), (1, single_mono_points), (2, single_stereo_points)):
        made = tries = 0
        while made < count:
            tries += 1
            assert tries < 50 * count, "cannot place the requested points"
            k0 = int(rng.choice(anchors if kind == 0 else single_anchors))
            if make_point(k0, min(max_obs, 1 + int(rng.geometric(p_tail))), kind):
                kinds.append(kind)
                made += 1
    kinds = np.array(kinds)

    # ---- the host unit's window (Optimizer_liba_b200.cc:64-111)
    feat = [[] for _ in range(n_map)]                    # each keyframe's features with a map point, in random feature order
    for i, obs in enumerate(obs_of):
        for (k, *_rest) in obs:
            feat[k].append(i)
    order_pts, taken = [], np.zeros(len(pts), bool)
    for k in window_kf:
        for i in rng.permutation(feat[k]) if feat[k] else []:
            if not taken[i]:
                taken[i] = True
                order_pts.append(int(i))
    assert taken.all()
    free_kf = window_kf[:-1] if early_map else window_kf     # the early map's oldest keyframe has no predecessor: it is popped ...
    fixed_kf = [0]                                           # ... and fixed; otherwise the predecessor chain[0] is the fixed one
    marked = set(free_kf) | {0}
    for i in order_pts:
        if len(fixed_kf) >= MAX_FIX_KF:
            break
        for k in sorted((o[0] for o in obs_of[i]), key=lambda k: age[k]):
            if k not in marked:
                marked.add(k)
                fixed_kf.append(k)
                break
    kf_list = free_kf + fixed_kf
    index = {k: j for j, k in enumerate(kf_list)}
    nKF, N = len(kf_list), len(free_kf)
    ekf, emp, obs, inv_s2, dropped = [], [], [], [], 0
    for j, i in enumerate(order_pts):
        for (k, u, vv, ur, w) in sorted(obs_of[i], key=lambda o: age[o[0]]):
            if k not in index:
                dropped += 1
                continue
            ekf.append(index[k]); emp.append(j); obs.append([u, vv, ur]); inv_s2.append(w)
    # ---- inertial links (:145-166): free keyframe i -> its predecessor, the oldest robust and scaled, every one robust with bRecInit
    links = []
    for i, k in enumerate(free_kf):
        if k == unlinked:
            continue
        pre = pres[k - 1]
        lk = np.zeros((), LIBA_LINK)
        lk["k1"], lk["k2"], lk["robust"], lk["dt"] = index[k - 1], i, int(i == N - 1 or rec_init), pre["dT"]
        for name in ("dR", "dV", "dP", "JRg", "JVg", "JVa", "JPg", "JPa"):
            lk[name] = pre[name].reshape(-1)
        lk["bias"] = pre["bias"]
        info, ig, ia = link_information(pre["C"], oldest=(i == N - 1))
        lk["info"], lk["infoG"], lk["infoA"] = info.reshape(-1), ig.reshape(-1), ia.reshape(-1)
        links.append(lk)
    links = np.array(links, LIBA_LINK).reshape(-1)
    # ---- the estimates: free keyframes and points perturbed (synth.inertial_window's amounts), keyframe positions as float, like the map
    state = kfs[kf_list].copy()
    for j in range(N):
        Rk = state[j, :9].reshape(3, 3)
        state[j, 9:12] += Rk @ rng.normal(0, 0.02, 3)
        state[j, :9] = (Rk @ synth._expm(rng.normal(0, 0.005, 3))).reshape(-1)
        state[j, 12:15] += rng.normal(0, 0.03, 3)
        state[j, 15:18] += rng.normal(0, 1e-3, 3)
        state[j, 18:21] += rng.normal(0, 1e-2, 3)
    point = np.array(pts)[order_pts] + rng.normal(0, 0.03, (len(order_pts), 3))
    fixed = (np.arange(nKF) >= N).astype(np.uint8)
    role = np.where(np.arange(nKF) < N, ROLE_FREE, np.where(np.arange(nKF) == N, ROLE_TEMPORAL, ROLE_COVISIBLE))
    ekf = np.array(ekf, np.int32)
    kinds = kinds[order_pts]
    lo, ul = (index[links_only] if links_only >= 0 else -1), (index[unlinked] if unlinked >= 0 else -1)
    if shuffle:                                          # the same window with its keyframes in random order
        perm = rng.permutation(nKF)
        new = np.empty(nKF, np.int64)
        new[perm] = np.arange(nKF)
        state, fixed, role, ekf = state[perm], fixed[perm], role[perm], new[ekf].astype(np.int32)
        links["k1"], links["k2"] = new[links["k1"]], new[links["k2"]]
        lo, ul = (int(new[lo]) if lo >= 0 else -1), (int(new[ul]) if ul >= 0 else -1)
    return dict(state=state, fixed=fixed, point=point, edge_kf=ekf, edge_mp=np.array(emp, np.int32),
                obs=np.array(obs, np.float64).reshape(-1, 3), inv_sigma2=np.array(inv_s2, np.float64), links=links,
                Tcb=np.concatenate([RCB.reshape(-1), TCB]), cam5=[FX, FY, CX, CY, BF],
                role=role, links_only_kf=lo, unlinked_kf=ul, single_mono_mp=np.flatnonzero(kinds == 1),
                single_stereo_mp=np.flatnonzero(kinds == 2), dropped=dropped)


# The windows the GPU tier runs (tests/test_liba_windows_gpu.py), by name: window() keyword arguments.  More than 10 free keyframes
# means bLarge (maxOpt 25), which also sets lambda 1e-2 and 4 iterations (Optimizer.cc:2211-2216, 2347-2355): settings().
CASES = {
    "10free_200fixed": dict(n_free=10, n_cov=300, n_mp=1500, seed=201),
    "25free_200fixed": dict(n_free=25, n_cov=300, n_mp=2500, seed=202),
    "10free_40fixed": dict(n_free=10, n_cov=40, n_mp=1200, seed=203),
    "early_map_1free": dict(n_free=1, n_cov=2, n_mp=200, seed=204, early_map=True),
    "early_map_2free": dict(n_free=2, n_cov=4, n_mp=300, seed=205, early_map=True),
    "shuffled": dict(n_free=10, n_cov=60, n_mp=800, seed=206, shuffle=True),
    "links_only_kf": dict(n_free=10, n_cov=40, n_mp=800, seed=207, links_only_kf=True),
    "unlinked_kf": dict(n_free=10, n_cov=40, n_mp=800, seed=208, unlinked_kf=True),
    "single_mono_points": dict(n_free=10, n_cov=40, n_mp=800, seed=209, single_mono_points=120),
    "single_stereo_points": dict(n_free=10, n_cov=40, n_mp=800, seed=210, single_stereo_points=120),
    "rec_init": dict(n_free=10, n_cov=40, n_mp=800, seed=211, rec_init=True),
}


def settings(pr):
    """(lambda_init, iterations) of the reference for this window: bLarge when it has more than 10 free keyframes."""
    return (1e-2, 4) if (pr["fixed"] == 0).sum() > 10 else (1.0, 10)


@functools.lru_cache(maxsize=None)
def case(name):
    return window(**CASES[name])


def oracle(pr, lam, iters):
    return po.liba(pr["state"], pr["fixed"], pr["point"], pr["edge_kf"], pr["edge_mp"], pr["obs"], pr["inv_sigma2"], pr["Tcb"],
                   pr["cam5"], pr["links"].view(po.LIBA_LINK), lam, iters)


def compare(g, r, pr):
    """The device algorithm's result g against the oracle's r, on every output the host unit reads.

    Iterations and trials exact; chi2_init to 1e-9 relative; chi2, chi2_last and lambda to 1e-6; every edge's and link's chi2 to
    rtol 1e-6 / atol 1e-8; the depth flags identical; the outlier
    classification (5.991 and 1.5 x 5.991 for monocular edges, 7.815 for stereo ones, as float like the unit's constants) identical
    on every edge not within 1e-6 of its threshold; the failure rule 2 (float) chi2_init < (float) chi2_last identical; states and
    points to TOL.  Returns the measured gaps (the largest state / point difference and the largest edge gap in units of its bar)."""
    assert g["iterations"] == r["iterations"] and g["trials"] == r["trials"], (g["iterations"], r["iterations"], g["trials"], r["trials"])
    assert abs(g["chi2_init"] - r["chi2_init"]) <= 1e-9 * max(1.0, r["chi2_init"]), (g["chi2_init"], r["chi2_init"])
    for k in ("chi2", "chi2_last"):
        assert abs(g[k] - r[k]) <= 1e-6 * max(1.0, r[k]), (k, g[k], r[k])
    assert abs(g["lambda_"] - r["lambda_"]) <= 1e-6 * r["lambda_"], (g["lambda_"], r["lambda_"])
    bar = 1e-8 + 1e-6 * np.abs(r["edge_chi2"])
    gap = np.abs(g["edge_chi2"] - r["edge_chi2"]) / bar
    assert (gap <= 1).all(), ("edge_chi2", float(gap.max()), int((gap > 1).sum()))
    lgap = np.abs(g["link_chi2"] - r["link_chi2"]) / (1e-8 + 1e-6 * np.abs(r["link_chi2"]))
    assert (lgap <= 1).all(), ("link_chi2", float(lgap.max()))
    assert (g["edge_depth_pos"] == r["edge_depth_pos"]).all(), int((g["edge_depth_pos"] != r["edge_depth_pos"]).sum())
    mono = pr["obs"][:, 2] < 0
    for thr, sel in ((np.float32(5.991), mono), (np.float32(1.5) * np.float32(5.991), mono), (np.float32(7.815), ~mono)):
        thr = float(thr)
        clear = sel & (np.abs(r["edge_chi2"] - thr) > 1e-6 * thr)
        assert ((g["edge_chi2"] > thr) == (r["edge_chi2"] > thr))[clear].all(), thr
    fail = lambda x: 2 * np.float32(x["chi2_init"]) < np.float32(x["chi2_last"])
    assert fail(g) == fail(r)
    ds, dp = float(np.abs(g["state"] - r["state"]).max()), float(np.abs(g["point"] - r["point"]).max())
    assert ds < TOL and dp < TOL, (ds, dp)
    return dict(state=ds, point=dp, edge_bar=float(gap.max()), link_bar=float(lgap.max()))


def _nobs(pr):
    return np.bincount(pr["edge_mp"], minlength=len(pr["point"]))


@pytest.mark.parametrize("name", list(CASES))
def test_window_has_the_claimed_shape(name):
    kw, pr = CASES[name], case(name)
    nKF, N = len(pr["state"]), kw["n_free"]
    role, fixed, links = pr["role"], pr["fixed"], pr["links"]
    assert (fixed == (role != ROLE_FREE)).all() and (role == ROLE_FREE).sum() == N and (role == ROLE_TEMPORAL).sum() == 1
    # the keyframe order: free ones, the temporal fixed one, the covisible ones -- or, shuffled, free ones among the fixed ones
    if kw.get("shuffle"):
        assert (np.diff(fixed.astype(int)) != 0).sum() > 4
    else:
        assert (role == np.sort(role)).all()
    # the fixed count: 200 where the map offers more covisible observers than the cap allows, else every covisible keyframe
    n_fixed = int(fixed.sum())
    assert n_fixed == (MAX_FIX_KF if kw["n_cov"] >= MAX_FIX_KF else kw["n_cov"] + 1), n_fixed
    assert (pr["dropped"] > 0) == (kw["n_cov"] >= MAX_FIX_KF)
    # links: one per free keyframe to its predecessor (one fewer with unlinked_kf), none to a covisible keyframe, the oldest robust
    assert len(links) == N - int(kw.get("unlinked_kf", False))
    assert (role[links["k2"]] == ROLE_FREE).all() and (role[links["k1"]] != ROLE_COVISIBLE).all()
    assert (role[links["k1"]] == ROLE_TEMPORAL).sum() == 1
    assert (links["robust"] == 1).sum() == (len(links) if kw.get("rec_init") else 1)
    assert len({(int(a), int(b)) for a, b in zip(links["k1"], links["k2"])}) == len(links)
    per_kf = np.bincount(pr["edge_kf"], minlength=nKF)
    if kw.get("links_only_kf"):
        k = pr["links_only_kf"]
        assert role[k] == ROLE_FREE and per_kf[k] == 0 and ((links["k1"] == k) | (links["k2"] == k)).sum() == 2
        assert (np.delete(per_kf, k) > 0).all()
    else:
        assert (per_kf > 0).all()
    if kw.get("unlinked_kf"):
        k = pr["unlinked_kf"]
        assert role[k] == ROLE_FREE and (links["k2"] == k).sum() == 0 and (links["k1"] == k).sum() == 1
    # edges grouped by point, points in first-seen order, at most one edge per (keyframe, point)
    assert (np.diff(pr["edge_mp"]) >= 0).all() and (np.unique(pr["edge_mp"]) == np.arange(len(pr["point"]))).all()
    assert len(np.unique(pr["edge_mp"].astype(np.int64) * nKF + pr["edge_kf"])) == len(pr["edge_kf"])
    # the observation tail: past 16 and past 32 edges on the real-sized windows; the 200-keyframe cap leaves single-edge points
    nobs = _nobs(pr)
    if N >= 10:
        assert (nobs > 16).sum() >= 50 and (nobs > 32).sum() >= 5, np.bincount(nobs)
    # single-edge points: the injected ones (one monocular or stereo edge to a free keyframe), and below the cap no others
    sm, ss = pr["single_mono_mp"], pr["single_stereo_mp"]
    mono = np.zeros(len(nobs), bool)
    mono[pr["edge_mp"][pr["obs"][:, 2] < 0]] = True
    assert len(sm) == kw.get("single_mono_points", 0) and (nobs[sm] == 1).all() and mono[sm].all()
    assert len(ss) == kw.get("single_stereo_points", 0) and (nobs[ss] == 1).all() and not mono[ss].any()
    assert (fixed[pr["edge_kf"][np.isin(pr["edge_mp"], np.concatenate([sm, ss]))]] == 0).all()
    if kw["n_cov"] >= MAX_FIX_KF:
        assert (mono & (nobs == 1)).sum() >= 3 and (~mono & (nobs == 1)).sum() >= 3
    else:
        assert (nobs == 1).sum() == len(sm) + len(ss)
    if kw.get("early_map"):          # the fixed keyframe's own points joined the window: some see no free keyframe
        has_free = np.zeros(len(nobs), bool)
        has_free[pr["edge_mp"][fixed[pr["edge_kf"]] == 0]] = True
        assert (~has_free).sum() >= 5


def test_window_is_deterministic():
    a, b = window(3, 5, 100, seed=7, shuffle=True), window(3, 5, 100, seed=7, shuffle=True)
    for k in ("state", "fixed", "point", "edge_kf", "edge_mp", "obs", "inv_sigma2", "links"):
        assert a[k].tobytes() == b[k].tobytes()


def test_edges_are_noisy_projections():
    """Every edge sees its point in front of the camera at the perturbed estimate; about 3 % are gross outliers (the outlier pass
    has edges to erase) and about 30 % are monocular."""
    pr = case("10free_40fixed")
    Xc = np.einsum("eji,ej->ei", pr["state"][pr["edge_kf"], :9].reshape(-1, 3, 3),
                   pr["point"][pr["edge_mp"]] - pr["state"][pr["edge_kf"], 9:12]) @ RCB.T + TCB
    u = FX * Xc[:, 0] / Xc[:, 2] + CX
    r = np.abs(pr["obs"][:, 0] - u)
    assert (Xc[:, 2] > 0.5).all() and np.median(r) < 5.0 and 0.01 < (r > 15).mean() < 0.06
    mono = pr["obs"][:, 2] < 0
    assert 0.2 < mono.mean() < 0.4


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_reduces_chi2(name):
    pr = case(name)
    lam, iters = settings(pr)
    r = oracle(pr, lam, iters)
    assert r["iterations"] >= 1 and np.isfinite(r["chi2"]) and r["chi2"] < r["chi2_init"]
    assert (r["state"][pr["fixed"] == 1] == pr["state"][pr["fixed"] == 1]).all()


@pytest.mark.parametrize("name", list(CASES))
def test_device_algorithm_matches_oracle(emul, name):   # noqa: F811
    pr = case(name)
    lam, iters = settings(pr)
    compare(run_emul(emul, pr, lam, iters), oracle(pr, lam, iters), pr)
