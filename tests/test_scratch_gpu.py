"""GPU tier: the per-call scratch buffers -- a captured call that would have to grow its buffer is refused and leaves the handle
working, and orbm_search_triangulation refuses a missing input array before it stages or launches anything."""
import ctypes as C

import numpy as np
import pytest
import torch

from orb_slam3_detailed_comments_b200 import ORBextractor, OrbError, PoseOptimizationDevice
from orb_slam3_detailed_comments_b200 import _native as N

pytestmark = pytest.mark.gpu
W, H = 640, 480
CAM5 = (435.2, 435.2, 320.0, 240.0, 47.9)
ARRAYS = ("kp1", "desc1", "node1", "stereo1", "kp2", "desc2", "node2", "valid2", "stereo2")


def _pose_problem(ne, seed=5):
    """One monocular frame of `ne` edges: points in front of the camera seen from a slightly moved pose."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, _ = CAM5
    z = rng.uniform(2, 12, ne)
    u, v = rng.uniform(30, W - 30, ne), rng.uniform(30, H - 30, ne)
    xw = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1).astype(np.float32)
    obs = np.stack([u + rng.normal(0, 0.5, ne), v + rng.normal(0, 0.5, ne), -np.ones(ne)], 1).astype(np.float32)
    return dict(eoff=np.array([0, ne], np.int32), pose=np.array([[0, 0, 0, 1, 0.01, -0.005, 0.02]], np.float32), xw=xw, obs=obs,
                w=np.ones(ne, np.float32))


def test_growth_inside_a_capture_is_refused_and_the_handle_keeps_working():
    dev = torch.device("cuda", 0)
    ne = 400
    p = {k: torch.from_numpy(a).to(dev) for k, a in _pose_problem(ne).items()}
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)   # no search has sized its scratch

    outs = lambda: (torch.zeros((1, 7), dtype=torch.float64, device=dev), torch.zeros(ne, dtype=torch.uint8, device=dev),
                    torch.zeros(1, dtype=torch.int32, device=dev))
    run = lambda w, out: PoseOptimizationDevice(ex, 1, p["eoff"], p["pose"], p["xw"], p["obs"], w, CAM5, *out)
    first, captured, again = outs(), outs(), outs()   # allocated outside the capture
    run(p["w"], first)
    torch.cuda.synchronize()
    # n_edges_max = inv_sigma2.numel() sizes the scratch: 2^21 edges need far more than the eager call allocated
    big_w = torch.ones(1 << 21, dtype=torch.float32, device=dev)
    with pytest.raises(OrbError, match="sized by one eager call"):
        ex.graph_capture(lambda: run(big_w, captured))
    run(p["w"], again)
    torch.cuda.synchronize()
    for a, b in zip(again, first):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    ex.close()


@pytest.mark.parametrize("missing", ARRAYS)
def test_triangulation_rejects_a_null_array(missing):
    rng = np.random.default_rng(1)
    nq, n2 = 8, 12
    kp1, kp2 = np.zeros(nq, N.KP_DTYPE), np.zeros(n2, N.KP_DTYPE)
    arrays = dict(kp1=kp1, desc1=rng.integers(0, 256, (nq, 32), dtype=np.uint8), node1=np.zeros(nq, np.int32), stereo1=np.zeros(nq, np.uint8),
                  kp2=kp2, desc2=rng.integers(0, 256, (n2, 32), dtype=np.uint8), node2=np.zeros(n2, np.int32), valid2=np.ones(n2, np.uint8),
                  stereo2=np.zeros(n2, np.uint8))
    arrays[missing] = None
    t = N.orbm_triangulation(nq, n2, *[N.ptr(arrays[k]) for k in ARRAYS], (C.c_float * 9)(*[0.0] * 9), (C.c_float * 2)(0.0, 0.0), 0, 1)
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    L = N.lib()
    m = np.full(nq, -7, np.int32)
    nm = C.c_int32(0)
    launches = L.orb_kernel_launches()
    with pytest.raises(OrbError, match="missing triangulation arrays"):
        N.check(L.orbm_search_triangulation(ex._h, C.byref(t), N.ptr(m), C.byref(nm)))
    assert L.orb_kernel_launches() == launches
    ex.close()
