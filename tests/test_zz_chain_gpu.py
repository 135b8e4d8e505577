"""GPU tier: the chained per-frame data flow of orbr_submit (orbr_chain: motion-model search -> PoseOptimization -> outlier release ->
Sophus::SE3f -> Frame::isInFrustum of the local map -> SearchByProjection(F, local map points) -> PoseOptimization over every map
point of the frame; Tracking.cc:3389-3522, 4010-4062) against the CPU oracle, stage by stage.  Integer stages (matches, claims,
skips, levels, in-view flags) and every float32 value of isInFrustum must be identical; the two optimised poses agree with the fp64
oracle to 1e-4 like tests/test_poseopt_gpu.py (the device's own first pose is what the later oracle stages start from).  The walk is
tests/_tracking.py's; the monocular and RGB-D forms are in tests/test_zz_mono_step_gpu.py and tests/test_zz_rgbd_step_gpu.py."""
import numpy as np
import pytest

from _tracking import run_chained_flow
from orb_slam3_detailed_comments_b200 import ORBextractor, camera, synth, replay

pytestmark = pytest.mark.gpu
W, H, NF = 640, 480, 1200
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11


def test_chained_frame_flow_matches_the_oracle_stage_by_stage():
    P = 2
    imgs = np.stack([im for p in range(P) for im in synth.stereo_pair(W, H, seed=400 + p)[:2]])
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * P)
    ex.extract_batch(imgs)
    ex.stereo_batch(P, BF, B)
    _, _, off, kps, desc = ex.download(2 * P)
    uR, dep = ex.stereo_download(int(off[-1]))
    frames = []
    for p in range(P):              # the LastFrame and local-map points are the features with a stereo depth; frame p is image 2p
        a, b = int(off[2 * p]), int(off[2 * p + 1])
        st = np.nonzero(dep[a:b] > 0)[0]
        frames.append(dict(k=kps[a:b], d=desc[a:b], z=dep[a:b], ur=uR[a:b], last=st[::2], other=st[1::2], rows=(a, b)))
    step = replay.TrackingStep(ex, camera(FX, FY, CX, CY, BF, B, W, H), BF, B, 15.0, 3.0, 0.8, True)
    _, _, nm0, nm2, checked = run_chained_flow(ex, step, imgs, off, frames, np.float32([FX, FY, CX, CY, BF, B]),
                                               np.arange(0, 2 * P, 2, dtype=np.int32), 2 * P * 1400, 15.0, 3.0)
    assert nm0.min() > 80 and nm2.min() > 100, (nm0, nm2)
    assert checked["released"] >= 3 and checked["skipped"] > 100 and checked["in_view"] > 400 and checked["local"] > 300, checked
    ex.close()
