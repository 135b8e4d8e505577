"""CPU tier, build container only: host/Optimizer_pose_b200.cc -- the translation unit that replaces Optimizer::PoseOptimization(Frame*) --
against the REFERENCE's own function (src/Optimizer.cc:55-412, compiled verbatim in oracle/_ref part 5).  Both run over the oracle's
numerics (ours through orbo_pose_optimization's arrays, answered by orc_pose_optimization; the reference's through the edges it created),
so what is compared is what the function itself decides: which features become edges (mono / stereo), cleared and final mvbOutlier flags
for every feature, the pose handed to SetPose as float bits, the return value, the early exit below three correspondences."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
MINE = os.path.join(HERE, "host", "pose_cpu_mine")


def _build():
    if os.path.exists(os.path.join(po.REFERENCE_ROOT, "src", "Optimizer.cc")):
        subprocess.check_call(["bash", os.path.join(HERE, "host", "build_pose_cpu.sh")])
    return os.path.exists(MINE) and po.build_ref5() is not None


pytestmark = pytest.mark.skipif(not _build(), reason="tests/host/pose_cpu_mine / oracle/_ref part 5 not built and /root/reference absent")
_spec = importlib.util.spec_from_file_location("_g2o_pin", os.path.join(HERE, "test_oracle_vs_ref_g2o.py"))
_g = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_g)


@pytest.mark.parametrize("seed,N,mp_frac,mono_frac,outlier_frac,motion", [(1, 1200, 0.5, 0.3, 0.15, 1.0), (2, 600, 0.9, 0.0, 0.05, 0.5), (3, 800, 0.4, 1.0, 0.2, 1.0),
                                                                          (4, 60, 0.5, 0.2, 0.3, 2.0), (5, 30, 0.3, 0.5, 0.1, 1.0), (6, 12, 0.2, 0.5, 0.0, 1.0),
                                                                          (7, 1500, 0.6, 0.3, 0.45, 3.0), (8, 5, 0.2, 0.5, 0.0, 1.0)])
def test_host_unit_equals_the_reference_function(tmp_path, seed, N, mp_frac, mono_frac, outlier_frac, motion):
    f = _g._frame(seed, N, mp_frac, mono_frac, outlier_frac, motion)
    cam5 = np.array([_g.FX, _g.FY, _g.CX, _g.CY, _g.BF], np.float32)
    d = str(tmp_path)
    for name, a in dict(cam5=cam5, pose=f["pose"].astype(np.float32), world_pos=f["world_pos"].astype(np.float32), kp_xy=f["kp_xy"].astype(np.float32),
                        uright=f["uright"].astype(np.float32), inv_level_sigma2=f["isg"].astype(np.float32)).items():
        a.tofile(os.path.join(d, name + ".f32"))
    f["has_mp"].astype(np.uint8).tofile(os.path.join(d, "has_mp.u8"))
    f["octave"].astype(np.int32).tofile(os.path.join(d, "octave.i32"))
    r = subprocess.run([MINE, d], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "pose_cpu ok" in r.stdout, (r.stdout[-1000:], r.stderr[-1000:])
    pose = np.fromfile(os.path.join(d, "out_pose.f32"), np.float32)
    outl = np.fromfile(os.path.join(d, "out_outlier.u8"), np.uint8)
    ret, sets = np.fromfile(os.path.join(d, "out_ret.i32"), np.int32)
    want = po.ref5_pose_optimization(f["pose"], f["has_mp"], f["world_pos"], f["kp_xy"], f["octave"], f["uright"], f["isg"], cam5)
    n_mp = int(f["has_mp"].sum())
    assert ret == want["inliers"]
    has = f["has_mp"].astype(bool)
    assert (outl[has] == want["outlier"][has]).all()
    assert (outl[~has] == 1).all()                        # features without a map point are not touched (the driver presets every flag)
    if n_mp >= 3:
        # Sophus::SO3's constructor normalises the float quaternion it is given (host/refshim/sophus/se3.hpp does, like the real one; the
        # stand-in under oracle/_ref part 5 hands it through): apply the same float normalisation to the reference's result
        f32 = np.float32
        q = want["pose"][:4].astype(f32)
        n = np.sqrt(f32(f32(f32(q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]))
        expect = np.concatenate([(q / n).astype(f32), want["pose"][4:].astype(f32)])
        assert sets == 1 and (pose.view(np.uint32) == expect.view(np.uint32)).all()
    else:
        assert sets == 0 and ret == 0 and (outl[has] == 0).all()
