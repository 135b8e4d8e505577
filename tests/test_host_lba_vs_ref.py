"""CPU tier, build container only: host/Optimizer_lba_b200.cc against the REFERENCE's own Optimizer::LocalBundleAdjustment.
tests/host/build_lba_cpu.sh cuts the function out of /root/reference/src/Optimizer.cc (and g2o's Levenberg functions out of
Thirdparty/g2o) and compiles it verbatim over the skeleton map of host/refshim and graph stand-ins whose numerics are the oracle's
LbaEngine; the host translation unit is linked with lba_solve_bool answered by the oracle (orc_lba) instead of the GPU.  Both walk
the same mock map: window selection (covisible neighbours, bad keyframes, other observers as fixed cameras, the map's initial
keyframe), vertex / edge construction, the lambda of inertial maps, the stop flag's early exit, optimize(10), the chi2 / depth test
of every edge (monocular edges first), the erasures on both sides, the pose / point write-back and the counters.  Equality is exact
(float bits): identical flattening order means identical engine input."""
import os
import subprocess

import numpy as np
import pytest

from oracle.pyoracle import REFERENCE_ROOT
from orb_slam3_detailed_comments_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = REFERENCE_ROOT
T = os.path.join(ROOT, "tests", "host")
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(REF, "src", "Optimizer.cc")), reason="reference checkout not present")
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11


@pytest.fixture(scope="module")
def binaries():
    subprocess.check_call(["bash", os.path.join(T, "build_lba_cpu.sh")])
    return os.path.join(T, "lba_cpu_mine"), os.path.join(T, "lba_cpu_ref")


def _run(binary, d, meta):
    with open(os.path.join(d, "meta.txt"), "w") as f:
        for k, v in meta.items():
            f.write(f"{k} {v}\n")
    subprocess.check_call([binary, d], stdout=subprocess.DEVNULL)
    rd = lambda name, dt: np.fromfile(os.path.join(d, name), dt)
    return dict(pose=rd("out_lba_pose.f32", np.float32), point=rd("out_lba_point.f32", np.float32), counters=rd("out_lba_counters.i32", np.int32),
                alive=rd("out_lba_alive.i32", np.int32), updates=rd("out_lba_updates.i32", np.int32))


CASES = [  # name, n_kf, n_mp, seed, ba_kf, n_observers, init_in_window, inertial, stop, null_stop, outlier_frac, mono_frac
    ("plain", 12, 500, 31, 3, 3, False, False, False, False, 0.03, 0.1),
    ("init_kf_in_window", 12, 500, 32, 3, 3, True, False, False, False, 0.03, 0.1),
    ("inertial_lambda", 12, 500, 33, 3, 3, False, True, False, False, 0.03, 0.1),
    ("stop_flag", 12, 500, 34, 3, 3, False, False, True, False, 0.03, 0.1),
    ("null_stop_pointer", 10, 300, 35, 2, 2, False, False, False, True, 0.05, 0.3),
    ("many_outliers", 14, 600, 36, 4, 4, False, False, False, False, 0.25, 0.2),
    ("mono_only", 8, 250, 37, 2, 2, False, False, False, False, 0.05, 1.0),
    ("no_fixed_keyframe", 6, 200, 38, 0, 0, False, False, False, False, 0.03, 0.1),   # every observer is covisible: "LBA aborted"
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_host_unit_equals_the_reference_function(binaries, tmp_path, case):
    name, n_kf, n_mp, seed, ba_kf, n_obs, init_in, inertial, stop, null_stop, outl, mono = case
    mine, ref = binaries
    pr = synth.lba_problem(n_kf=n_kf, n_fixed=max(n_obs, 1), n_mp=n_mp, seed=seed, outlier_frac=outl, mono_frac=mono)
    nKF, nMP = len(pr["pose"]), len(pr["point"])
    rng = np.random.default_rng(seed)
    role = np.array([2] * n_obs + [0] + [1] * (nKF - n_obs - 1), np.int32)   # observers only, the BA keyframe, its covisible neighbours
    if nKF - n_obs - 1 > 2:
        role[nKF - 1] = 3                                                    # one covisible neighbour has been culled (isBad)
    badmp = (rng.random(nMP) < 0.03).astype(np.uint8)
    init_id = 100 + n_obs + 2 if init_in else 0
    arrays = [("lba_pose.f32", pr["pose"].astype(np.float32)), ("lba_role.i32", role), ("lba_point.f32", pr["point"].astype(np.float32)),
              ("lba_edge_kf.i32", pr["edge_kf"]), ("lba_edge_mp.i32", pr["edge_mp"]), ("lba_obs.f32", pr["obs"].astype(np.float32)),
              ("lba_inv_sigma2.f32", pr["inv_sigma2"].astype(np.float32)), ("lba_badmp.u8", badmp)]
    meta = dict(fx=FX, fy=FY, cx=CX, cy=CY, bf=BF, b=B, lba_nkf=nKF, lba_nmp=nMP, lba_init_kf_id=init_id, lba_inertial=int(inertial),
                lba_stop=int(stop), lba_null_stop=int(null_stop))
    outs = []
    for i, binary in enumerate((mine, ref)):
        d = str(tmp_path / f"run{i}")
        os.makedirs(d)
        for fn, a in arrays:
            np.ascontiguousarray(a).tofile(os.path.join(d, fn))
        outs.append(_run(binary, d, meta))
    a, b = outs
    assert (a["counters"] == b["counters"]).all(), (a["counters"], b["counters"])
    assert (a["alive"] == b["alive"]).all() and (a["updates"] == b["updates"]).all()
    assert (a["pose"].view(np.uint32) == b["pose"].view(np.uint32)).all()
    assert (a["point"].view(np.uint32) == b["point"].view(np.uint32)).all()
    moved = a["counters"][3] > 0                                                # IncreaseChangeIndex ran: the optimisation happened
    if name in ("stop_flag", "no_fixed_keyframe"):
        assert not moved and (a["alive"] == 3).all()
    else:
        assert moved and (a["alive"] != 3).any() and a["updates"].sum() > 0     # something was optimised and some edges were erased
