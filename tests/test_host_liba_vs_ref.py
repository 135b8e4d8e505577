"""CPU tier, build container only: host/Optimizer_liba_b200.cc -- the translation unit that replaces Optimizer::LocalInertialBA -- next to
the REFERENCE's own function (src/Optimizer.cc:2203-2812), cut out at build time and compiled verbatim over graph stand-ins
(tests/host/liba_ref_graph.h).  Both walk the same mock map (keyframe chain through mPrevKF with IMU::Preintegrated members, map points,
observations) and both hand their problem to the oracle's orc_liba -- ours through liba_solve's arrays, the reference's through the
vertices and edges it created -- so what is compared is everything the function itself decides: the temporal window, which keyframe
before it is fixed, one further fixed observer per point, vertex states, which pairs get inertial links with which information scaling
and robust kernel, SetNewBias on the preintegrations, the reprojection edges and their order, lambda / iterations for bLarge, the
chi2 / bClose / depth tests, the failure rule, erasures, the poses / velocities / biases / points written back and the marks reset."""
import os
import subprocess

import numpy as np
import pytest

from oracle.pyoracle import REFERENCE_ROOT
from orb_slam3_detailed_comments_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
MINE, REF = os.path.join(HERE, "host", "liba_cpu_mine"), os.path.join(HERE, "host", "liba_cpu_ref")


def _build():
    if os.path.exists(os.path.join(REFERENCE_ROOT, "src", "Optimizer.cc")):
        subprocess.check_call(["bash", os.path.join(HERE, "host", "build_liba_cpu.sh")])
    return os.path.exists(MINE) and os.path.exists(REF)


pytestmark = pytest.mark.skipif(not _build(), reason="tests/host/liba_cpu_* not built and the reference (ORB_REFERENCE_ROOT) absent")


def _quat(R):
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0)
        q = np.array([(R[2, 1] - R[1, 2]) * 0.5 / s, (R[0, 2] - R[2, 0]) * 0.5 / s, (R[1, 0] - R[0, 1]) * 0.5 / s, 0.5 * s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q = np.zeros(4)
        q[i] = 0.5 * s
        q[3] = (R[k, j] - R[j, k]) * 0.5 / s
        q[j] = (R[j, i] + R[i, j]) * 0.5 / s
        q[k] = (R[k, i] + R[i, k]) * 0.5 / s
    return q / np.linalg.norm(q)


def write_case(d, W, n_opt, *, large=False, rec_init=False, keyframes_in_map=None, chain_has_prev=True, bad_points=0.0, bad_kf=(), seed=0):
    """The mock map behind window W (synth.inertial_window: index 0 = the keyframe before the window, 1 .. n_opt the chain oldest to newest,
    then other observers).  chain_has_prev False cuts the link 1 -> 0: the window's oldest keyframe has no predecessor."""
    rng = np.random.default_rng(seed)
    nKF, nMP = len(W["state"]), len(W["point"])
    Rcb, tcb = np.asarray(W["Tcb"][:9]).reshape(3, 3), np.asarray(W["Tcb"][9:])
    pose, flags, pre = np.zeros((nKF, 7), np.float32), np.zeros((nKF, 4), np.int32), np.zeros((nKF, 292), np.float32)
    for k in range(nKF):
        Rwb, twb = W["state"][k, :9].reshape(3, 3), W["state"][k, 9:12]
        Rcw = Rcb @ Rwb.T
        tcw = Rcb @ (-Rwb.T @ twb) + tcb
        pose[k] = np.concatenate([_quat(Rcw), tcw])
        is_chain = k <= n_opt
        flags[k] = [1 if is_chain else 0, -1, 1 if k in bad_kf else 0, 0]
        if 1 <= k <= n_opt and (k > 1 or chain_has_prev):
            flags[k, 1] = k - 1
            P = W["pre"][k - 1]
            pre[k] = np.concatenate([[P["dT"]], P["C"].reshape(-1), P["bias"]] + [P[n].reshape(-1) for n in ("dR", "dV", "dP", "JRg", "JVg", "JVa", "JPg", "JPa")])
            flags[k, 3] = 1
    if not chain_has_prev:
        flags[0, 0] = 0           # an unrelated observer now
    vel = W["state"][:, 12:15].astype(np.float32)
    bias = np.concatenate([W["state"][:, 18:21], W["state"][:, 15:18]], 1).astype(np.float32)     # bax bay baz bwx bwy bwz
    with open(os.path.join(d, "meta.txt"), "w") as f:
        cam = W["cam5"]
        for k, v in dict(fx=cam[0], fy=cam[1], cx=cam[2], cy=cam[3], bf=cam[4], b=0.11, nkf=nKF, nmp=nMP, ba_kf=n_opt, large=int(large), rec_init=int(rec_init),
                         keyframes_in_map=keyframes_in_map if keyframes_in_map is not None else n_opt + 2).items():
            f.write(f"{k} {v}\n")
    arrays = dict(kf_pose=pose, kf_vel=vel, kf_bias=bias, kf_flags=flags, kf_pre=pre, tcb=np.concatenate([_quat(Rcb), tcb]).astype(np.float32),
                  point=W["point"].astype(np.float32), point_track_depth=rng.uniform(2, 25, nMP).astype(np.float32),
                  point_bad=(rng.random(nMP) < bad_points).astype(np.uint8), edge_kf=W["edge_kf"].astype(np.int32), edge_mp=W["edge_mp"].astype(np.int32),
                  edge_obs=W["obs"].astype(np.float32), edge_inv_sigma2=W["inv_sigma2"].astype(np.float32))
    ext = {np.dtype(np.float32): "f32", np.dtype(np.int32): "i32", np.dtype(np.uint8): "u8"}
    for name, a in arrays.items():
        a.tofile(os.path.join(d, f"{name}.{ext[a.dtype]}"))
    return arrays


def run(binary, d):
    r = subprocess.run([binary, d], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "liba_cpu ok" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])
    rd = lambda n, t: np.fromfile(os.path.join(d, n), t)
    return dict(pose=rd("out_pose.f32", np.float32).reshape(-1, 7), vel=rd("out_vel.f32", np.float32).reshape(-1, 3), bias=rd("out_bias.f32", np.float32).reshape(-1, 6),
                pre_bu=rd("out_pre_bu.f32", np.float32).reshape(-1, 6), point=rd("out_point.f32", np.float32).reshape(-1, 3), counters=rd("out_counters.i32", np.int32),
                alive=rd("out_alive.i32", np.int32), updates=rd("out_updates.i32", np.int32), log=r.stdout)


CASES = {
    "window_of_ten": dict(win=dict(n_opt=10, n_cov_fixed=3, n_mp=900, seed=1), n_opt=10),
    "large": dict(win=dict(n_opt=12, n_cov_fixed=2, n_mp=800, seed=2), n_opt=12, large=True, keyframes_in_map=40),
    "rec_init": dict(win=dict(n_opt=6, n_cov_fixed=2, n_mp=500, seed=3), n_opt=6, rec_init=True),
    "short_map": dict(win=dict(n_opt=8, n_cov_fixed=2, n_mp=600, seed=4), n_opt=8, keyframes_in_map=7),          # Nd = 5: a shorter window, its predecessor fixed
    "no_predecessor": dict(win=dict(n_opt=5, n_cov_fixed=3, n_mp=500, seed=5), n_opt=5, chain_has_prev=False, keyframes_in_map=30),   # the oldest keyframe becomes the fixed one
    "bad_points_and_observers": dict(win=dict(n_opt=7, n_cov_fixed=4, n_mp=700, seed=6), n_opt=7, bad_points=0.1, bad_kf=(9,)),
    "outliers": dict(win=dict(n_opt=7, n_cov_fixed=3, n_mp=700, seed=7), n_opt=7, corrupt=0.08),
    "nan_fails": dict(win=dict(n_opt=5, n_cov_fixed=2, n_mp=300, seed=8), n_opt=5, nan_point=True),      # isnan(err): "FAIL LOCAL-INERTIAL BA", nothing written, marks left
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_unit_equals_the_reference_function(tmp_path, name):
    c = dict(CASES[name])
    W = synth.inertial_window(keep_pre=True, **c.pop("win"))
    n_opt = c.pop("n_opt")
    corrupt = c.pop("corrupt", 0.0)
    if c.pop("nan_point", False):
        W["point"][17, 1] = np.nan
        failed = True
    else:
        failed = False
    if corrupt:
        rng = np.random.default_rng(11)
        sel = rng.random(len(W["obs"])) < corrupt
        W["obs"][sel, :2] += rng.normal(0, 25, (int(sel.sum()), 2))
    dm, dr = str(tmp_path / "mine"), str(tmp_path / "ref")
    os.makedirs(dm), os.makedirs(dr)
    arrays = write_case(dm, W, n_opt, **c)
    write_case(dr, W, n_opt, **c)
    a, b = run(MINE, dm), run(REF, dr)
    for k in ("pose", "vel", "bias", "pre_bu", "point"):
        assert (a[k].view(np.uint32) == b[k].view(np.uint32)).all(), (name, k, np.abs(a[k] - b[k]).max())
    for k in ("counters", "alive", "updates"):
        assert (a[k] == b[k]).all(), (name, k)
    if failed:
        assert a["counters"][4] == 0 and a["updates"].sum() == 0 and (a["counters"][5:].reshape(len(W["state"]), 6)[:, :3] == 0).all()
        assert (a["counters"][5:].reshape(len(W["state"]), 6)[1:n_opt + 1, 4] == 100 + n_opt).all()       # mnBALocalForKF still holds the BA keyframe's id
        return
    # and the run did something: the window's keyframes were written once each, points updated, some observations erased where planted
    nKF = len(W["state"])
    per_kf = a["counters"][5:].reshape(nKF, 6)
    live = np.array([k not in c.get("bad_kf", ()) for k in range(nKF)])     # a bad observer is marked fixed but never listed, so its mark stays (:2326-2333, :2750)
    assert a["counters"][4] == 1 and per_kf[:, 0].sum() >= 3 and (per_kf[:, 4] == 0).all() and (per_kf[live, 5] == 0).all()
    assert a["updates"].sum() > 100
    if corrupt:
        assert (a["alive"] == 0).sum() > 10
    assert per_kf[n_opt, 0] == 1 and (per_kf[n_opt + 1:, 0] == 0).all() and per_kf[0, 0] == 0      # the BA keyframe written once; observers and the keyframe before the window never
