"""GPU tier: the entry points with a host and a device form return identical arrays from both forms on one seeded scene, and a
call with no queries, points or edges returns zero counts from both forms even where an earlier call left non-zero counts."""
import ctypes as C

import numpy as np
import pytest
import torch

from orb_slam3_detailed_comments_b200 import (ORBextractor, ORBmatcher, ORBVocabulary, PoseOptimization, PoseOptimizationDevice, camera,
                                              isInFrustum, isInFrustumDevice, synth, synthetic_vocabulary)
from orb_slam3_detailed_comments_b200 import _native as N

pytestmark = pytest.mark.gpu

W, H = 640, 480
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11
CAM5 = (FX, FY, CX, CY, BF)
DEV = torch.device("cuda", 0)
FRUSTUM_KEYS = ("in_view", "proj_x", "proj_y", "proj_xr", "level", "view_cos", "depth")


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _d(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _node(desc):
    """A stand-in vocabulary node per descriptor: a hash of three bytes into 97 buckets."""
    d = np.asarray(desc, np.int64)
    return ((d[:, 0] * 7 + d[:, 5] * 13 + d[:, 17]) % 97).astype(np.int32)


@pytest.fixture(scope="module")
def scene():
    l, r, _ = synth.stereo_pair(W, H, seed=71)
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ex.extract_batch(np.stack([l, r]))
    ex.stereo_batch(1, BF, B)
    n, mono, off, kps, desc = ex.download(2)
    uR, dep = ex.stereo_download(int(off[-1]))
    rng = np.random.default_rng(3)
    a, b = int(off[0]), int(off[1])
    k, d = kps[a:b], desc[a:b].copy()
    flip = rng.random(d.shape) < 0.03                       # queries: the left image's own features, jittered and a few bits off
    d[flip] ^= np.uint8(1 << 3)
    x = (k["x"] + rng.normal(0, 1.0, len(k))).astype(np.float32)
    y = (k["y"] + rng.normal(0, 1.0, len(k))).astype(np.float32)
    z = np.where(dep[a:b] > 0, dep[a:b], rng.uniform(2, 10, len(k))).astype(np.float32)   # stereo depth where the pair has one
    yield dict(ex=ex, off=off, total=int(off[-1]), k=k, d=d, x=x, y=y, z=z, rows_desc=desc, cam=camera(FX, FY, CX, CY, BF, B, W, H))
    ex.close()


def _sync():
    torch.cuda.synchronize()


def test_local_points_host_and_device_agree(scene):
    ex, cam, k, d, x, y = scene["ex"], scene["cam"], scene["k"], scene["d"], scene["x"], scene["y"]
    m = ORBmatcher(0.8, True)
    nq = len(k)
    q = dict(px=x, py=y, pxr=(x - BF / scene["z"]).astype(np.float32), lv=k["octave"].astype(np.int32), vc=np.ones(nq, np.float32), desc=d)

    def host(qoff, sl):
        match = np.full(max(nq, 1), 123, np.int32)
        nm = np.full(1, 77, np.int32)
        return m.SearchByProjection(ex, cam, [0], qoff, q["px"][sl], q["py"][sl], q["pxr"][sl], q["lv"][sl], q["vc"][sl], q["desc"][sl],
                                    th=3.0, out=(match, nm))

    def device(qoff, sl, out):
        _sync()
        m.SearchByProjectionDevice(ex, cam, 1, _t(np.array([0], np.int32)), _t(np.asarray(qoff, np.int32)), _t(q["px"][sl]), _t(q["py"][sl]),
                                   _t(q["pxr"][sl]), _t(q["lv"][sl]), _t(q["vc"][sl]), _t(q["desc"][sl]), *out, th=3.0)
        _sync()
        return out[0].cpu().numpy()[: qoff[1]], out[1].cpu().numpy()

    out = (torch.full((nq,), 123, dtype=torch.int32, device=DEV), torch.full((1,), 77, dtype=torch.int32, device=DEV))
    hm, hn = host([0, nq], slice(None))
    dm, dn = device([0, nq], slice(None), out)
    assert hn[0] > 50 and (hm == dm).all() and (hn == dn).all()
    hm, hn = host([0, 0], slice(0, 0))
    dm, dn = device([0, 0], slice(0, 0), out)
    assert hn[0] == 0 and dn[0] == 0


def test_last_frame_host_and_device_agree(scene):
    ex, cam, k, d, total = scene["ex"], scene["cam"], scene["k"], scene["d"], scene["total"]
    m = ORBmatcher(0.9, True)
    nq = len(k)
    z = scene["z"]
    xw = np.stack([(scene["x"] - CX) * z / FX, (scene["y"] - CY) * z / FY, z], 1).astype(np.float32)
    Tcw = np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32)
    q = dict(xw=xw, oct=k["octave"].astype(np.int32), ang=k["angle"].astype(np.float32), desc=d, obs=np.ones(nq, np.uint8))

    def host(qoff, sl):
        out = (np.full(total, 123, np.int32), np.full(1, 77, np.int32))
        return m.SearchByProjectionLastFrame(ex, cam, [0], qoff, Tcw, [0], q["xw"][sl], q["oct"][sl], q["ang"][sl], q["desc"][sl], q["obs"][sl],
                                             7.0, total, out=out)

    def device(qoff, sl, out):
        _sync()
        m.SearchByProjectionLastFrameDevice(ex, cam, 1, _t(np.array([0], np.int32)), _t(np.asarray(qoff, np.int32)), _t(Tcw),
                                            _t(np.array([0], np.int32)), _t(q["xw"][sl]), _t(q["oct"][sl]), _t(q["ang"][sl]),
                                            _t(q["desc"][sl]), _t(q["obs"][sl]), 7.0, *out)
        _sync()
        return out[0].cpu().numpy(), out[1].cpu().numpy()

    out = (torch.full((total,), 123, dtype=torch.int32, device=DEV), torch.full((1,), 77, dtype=torch.int32, device=DEV))
    hm, hn = host([0, nq], slice(None))
    dm, dn = device([0, nq], slice(None), out)
    assert hn[0] > 50 and (hm == dm).all() and (hn == dn).all()
    hm, hn = host([0, 0], slice(0, 0))
    dm, dn = device([0, 0], slice(0, 0), out)
    assert hn[0] == 0 and dn[0] == 0 and (hm == -1).all() and (dm == -1).all()


def test_bow_host_and_device_agree(scene):
    ex, k, d, total = scene["ex"], scene["k"], scene["d"], scene["total"]
    L = N.lib()
    nq = len(k)
    feat_node = _node(scene["rows_desc"])
    qn, qa = _node(d), k["angle"].astype(np.float32)

    def call(on_device, qoff, sl, fm, nm):
        arrs = [np.array([0], np.int32), np.asarray(qoff, np.int32), qn[sl], qa[sl], d[sl], feat_node]
        if on_device:
            arrs = [_t(a) for a in arrs]
            _sync()
        p = _d if on_device else N.ptr
        q = N.orbm_bow_queries(1, int(on_device), *[p(a) for a in arrs])
        N.check(L.orbm_search_bow(ex._h, C.byref(q), 0.7, 1, p(fm), p(nm)))
        if on_device:
            _sync()
            return fm.cpu().numpy(), nm.cpu().numpy()
        return fm, nm

    dfm, dnm = torch.full((total,), 123, dtype=torch.int32, device=DEV), torch.full((1,), 77, dtype=torch.int32, device=DEV)
    hm, hn = call(False, [0, nq], slice(None), np.full(total, 123, np.int32), np.full(1, 77, np.int32))
    dm, dn = call(True, [0, nq], slice(None), dfm, dnm)
    assert hn[0] > 50 and (hm == dm).all() and (hn == dn).all()
    hm, hn = call(False, [0, 0], slice(0, 0), hm, hn)
    dm, dn = call(True, [0, 0], slice(0, 0), dfm, dnm)
    assert hn[0] == 0 and dn[0] == 0 and (hm == -1).all() and (dm == -1).all()


def _pose_frames(ne, seed):
    rng = np.random.default_rng(seed)
    z = rng.uniform(2, 12, ne)
    u, v = rng.uniform(30, W - 30, ne), rng.uniform(30, H - 30, ne)
    xw = np.stack([(u - CX) * z / FX, (v - CY) * z / FY, z], 1).astype(np.float32)
    obs = np.stack([u + rng.normal(0, 0.5, ne), v + rng.normal(0, 0.5, ne), np.where(rng.random(ne) < 0.5, u - BF / z, -1.0)], 1)
    obs[: ne // 10, :2] += 40.0                                       # a few outliers
    return dict(pose=np.array([0, 0, 0, 1, 0.01, -0.005, 0.02], np.float32), world_pos=xw, obs=obs.astype(np.float32),
                inv_sigma2=np.ones(ne, np.float32))


def test_pose_optimization_host_and_device_agree(scene):
    ex = scene["ex"]

    def device(f, out):
        ne = len(f["world_pos"])
        _sync()
        PoseOptimizationDevice(ex, 1, _t(np.array([0, ne], np.int32)), _t(f["pose"][None]), _t(f["world_pos"]), _t(f["obs"]),
                               _t(f["inv_sigma2"]), CAM5, *out)
        _sync()
        return [o.cpu().numpy() for o in out]

    f = _pose_frames(500, 9)
    out = (torch.zeros((1, 7), dtype=torch.float64, device=DEV), torch.zeros(500, dtype=torch.uint8, device=DEV),
           torch.full((1,), 77, dtype=torch.int32, device=DEV))
    h = PoseOptimization(ex, [f], CAM5)[0]
    pose, outl, inl = device(f, out)
    assert h["inliers"] > 400 and h["inliers"] == inl[0]
    assert h["pose"].tobytes() == pose[0].tobytes() and h["outlier"].tobytes() == outl.tobytes()
    empty = dict(pose=f["pose"], world_pos=np.zeros((0, 3), np.float32), obs=np.zeros((0, 3), np.float32), inv_sigma2=np.zeros(0, np.float32))
    h = PoseOptimization(ex, [empty], CAM5)[0]
    pose, _, inl = device(empty, out)
    assert h["inliers"] == 0 and inl[0] == 0 and h["pose"].tobytes() == pose[0].tobytes()


def test_is_in_frustum_host_and_device_agree(scene):
    ex, cam = scene["ex"], scene["cam"]
    rng = np.random.default_rng(13)
    n = 3000
    xw = np.stack([rng.uniform(-8, 8, n), rng.uniform(-6, 6, n), rng.uniform(-2, 15, n)], 1).astype(np.float32)
    nr = xw / np.linalg.norm(xw, axis=1, keepdims=True)
    dist = np.linalg.norm(xw, axis=1)
    a = dict(Rcw=np.eye(3, dtype=np.float32).reshape(1, 9), tcw=np.zeros((1, 3), np.float32), Ow=np.zeros((1, 3), np.float32), world_pos=xw,
             normal=nr.astype(np.float32), max_dist=(dist * 1.5).astype(np.float32), min_dist=(dist * 0.5).astype(np.float32))
    h = isInFrustum(ex, cam, [0, n], **a)
    out = {kk: torch.zeros(n, dtype=torch.uint8 if kk == "in_view" else (torch.int32 if kk == "level" else torch.float32), device=DEV)
           for kk in FRUSTUM_KEYS}
    dv = {kk: _t(v) for kk, v in a.items()}
    _sync()
    isInFrustumDevice(ex, cam, 1, _t(np.array([0, n], np.int32)), **dv, out=out)
    _sync()
    assert h["in_view"].sum() > 100
    for kk in FRUSTUM_KEYS:
        assert h[kk].tobytes() == out[kk].cpu().numpy().tobytes(), kk
    # no points: both forms succeed and write nothing
    before = {kk: v.clone() for kk, v in out.items()}
    empty = {kk: (v[:0] if kk not in ("Rcw", "tcw", "Ow") else v) for kk, v in a.items()}
    assert all(len(v) == 0 for v in isInFrustum(ex, cam, [0, 0], **empty).values())
    _sync()
    isInFrustumDevice(ex, cam, 1, _t(np.array([0, 0], np.int32)), **{kk: (v[:0] if kk not in ("Rcw", "tcw", "Ow") else v) for kk, v in dv.items()},
                      out=out)
    _sync()
    for kk in FRUSTUM_KEYS:
        assert torch.equal(out[kk], before[kk]), kk


def test_transform_host_and_device_agree(scene):
    voc = synthetic_vocabulary(k=10, L=3, seed=31)
    V = ORBVocabulary(voc["child_offset"], voc["child_ids"], voc["node_desc"], voc["node_word"], voc["node_weight"], voc["L"])
    L = N.lib()

    def device(ex, rows, nimg, out):
        _sync()
        N.check(L.orbv_transform(ex._h, V._v, 2, 1, *[_d(o) for o in out]))
        _sync()
        got = [o.cpu().numpy() for o in out]
        return dict(word=got[0][:rows], node=got[1][:rows], weight=got[2][:rows], cnt=got[3][:nimg], bw=got[4][:nimg], bv=got[5][:nimg])

    def outs(ex, rows):
        mf = ex.max_features_per_image()
        z = lambda shape, dt: torch.full(shape, 77, dtype=dt, device=DEV)
        return (z((max(rows, 1),), torch.int32), z((max(rows, 1),), torch.int32), z((max(rows, 1),), torch.float64), z((2,), torch.int32),
                z((2, mf), torch.int32), z((2, mf), torch.float64))

    ex, total = scene["ex"], scene["total"]
    out = outs(ex, total)
    h = V.transform(ex, total, 2, levelsup=2)
    g = device(ex, total, 2, out)
    assert total > 100 and len(h["bow_word"][0]) > 10
    for kk in ("word", "node", "weight"):
        assert h[kk].tobytes() == g[kk].tobytes(), kk
    for i in range(2):
        c = int(g["cnt"][i])
        assert c == len(h["bow_word"][i])
        assert h["bow_word"][i].tobytes() == g["bw"][i, :c].tobytes() and h["bow_weight"][i].tobytes() == g["bv"][i, :c].tobytes()
    # a batch without features: both forms return zero BowVector sizes over the counts the call above left
    blank = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    blank.extract_batch(np.zeros((2, H, W), np.uint8))
    assert int(blank.download(2)[2][-1]) == 0
    mf = blank.max_features_per_image()
    cnt = np.full(2, 77, np.int32)
    word, node, weight = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.float64)
    bw, bv = np.zeros((2, mf), np.int32), np.zeros((2, mf), np.float64)
    N.check(L.orbv_transform(blank._h, V._v, 2, 0, *[N.ptr(a) for a in (word, node, weight, cnt, bw, bv)]))
    assert (cnt == 0).all()
    out = outs(blank, 0)
    assert (device(blank, 0, 2, out)["cnt"] == 0).all()
    blank.close()
    V.close()
