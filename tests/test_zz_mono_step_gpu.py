"""GPU tier: the monocular replay step (orbr_step::monocular: one image per frame through ORBextractor::operator() with
vLappingArea = {0, 1000}, Frame.cc:380; no ComputeStereoMatches, so every search and PoseOptimization sees mvuRight = -1).

- on two handles kept in flight from one host thread it gives exactly what the blocking per-call C ABI gives, and the first frame
  of a batch equals the CPU oracle: keypoints, descriptors, monoIndex and both match arrays (752x480 EuRoC-shaped frames, and
  1241x376 KITTI-shaped ones, where the two fill directions of the lapping area interleave);
- the chained flow in monocular mode matches the oracle stage by stage;
- a CUDA-graph replay of the device-resident monocular step equals the eager calls;
- the step refuses oversized batches, out-of-range frame images and a nonzero direction, and the handle stays usable;
- a stereo step right after a monocular one on the same handle equals the same stereo step on a fresh handle, and the reverse."""
import numpy as np
import pytest
import torch

from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth, PoseOptimizationFrames, replay
from orb_slam3_detailed_comments_b200._native import KP_DTYPE, OrbError
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
NF = 1200
TH_LAST, TH_LOC = 15.0, 1.0          # Tracking.cc: TrackWithMotionModel th = 15 (not stereo), SearchLocalPoints th = 1
ORB_ERR_INVALID = -1
# (W, H, fx, fy, cx, cy, bf of the synthetic disparity field); the step itself ignores bf / b
GEOM = {"euroc_752x480": (752, 480, 458.654, 457.296, 367.215, 248.375, 50.49),
        "kitti_1241x376": (1241, 376, 718.856, 718.856, 607.1928, 185.2157, 386.14)}
f32 = np.float32


def _frames(W, H, seeds):
    """left images and disparity fields of synthetic rectified stereo pairs; the monocular frame is the left image"""
    pairs = [synth.stereo_pair(W, H, seed=s) for s in seeds]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs]), [p[2] for p in pairs]


def _depth(disp, k, bf):
    """ground-truth depth of each keypoint from the synthetic disparity field"""
    H, W = disp.shape
    x = np.clip(np.rint(k["x"]).astype(np.int64), 0, W - 1)
    y = np.clip(np.rint(k["y"]).astype(np.int64), 0, H - 1)
    return (f32(bf) / disp[y, x]).astype(f32)


def _queries(ex, imgs, disps, g, rng):
    """Query sets from the frames' own features back-projected at their ground-truth depth (host arrays); frame f = image f."""
    W, H, FX, FY, CX, CY, BFGT = g
    P = len(imgs)
    ex.extract_batch(imgs, lapping=(0, 1000))
    n, _, off, kps, desc = ex.download(P)
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    loc = dict(off=[0], px=[], py=[], pxr=[], lvl=[], vc=[], desc=[], xw=[])
    for p in range(P):
        a, b = int(off[p]), int(off[p + 1])
        k, d = kps[a:b], desc[a:b]
        z = _depth(disps[p], k, BFGT)
        sel = np.arange(0, len(k), 2)
        pts = np.stack([(k["x"][sel] - CX) * z[sel] / FX, (k["y"][sel] - CY) * z[sel] / FY, z[sel]], 1).astype(f32)
        last["xw"].append(pts); last["oct"].append(k["octave"][sel].astype(np.int32)); last["ang"].append(k["angle"][sel].astype(f32))
        last["desc"].append(d[sel]); last["obs"].append((rng.random(len(sel)) < 0.9).astype(np.uint8)); last["off"].append(last["off"][-1] + len(sel))
        m = len(k)
        x = (k["x"] + rng.normal(0, 1.0, m)).astype(f32); y = (k["y"] + rng.normal(0, 1.0, m)).astype(f32)
        loc["px"].append(x); loc["py"].append(y); loc["pxr"].append(x.copy()); loc["lvl"].append(k["octave"].astype(np.int32))
        loc["vc"].append(rng.uniform(0.999, 1, m).astype(f32)); loc["desc"].append(d)
        loc["xw"].append(np.stack([(k["x"] - CX) * z / FX, (k["y"] - CY) * z / FY, z], 1).astype(f32)); loc["off"].append(loc["off"][-1] + m)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    fimg = np.arange(P, dtype=np.int32)
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=np.tile(np.array([0, 0, 0, 1, 0.002, 0.001, 0], f32), (P, 1)),
              dir=np.zeros(P, np.int32), xw=cat(last["xw"], f32), oct=cat(last["oct"], np.int32), ang=cat(last["ang"], f32),
              desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(fimg=fimg, off=np.array(loc["off"], np.int32), px=cat(loc["px"], f32), py=cat(loc["py"], f32), pxr=cat(loc["pxr"], f32),
              lvl=cat(loc["lvl"], np.int32), vc=cat(loc["vc"], f32), desc=cat(loc["desc"], np.uint8), xw=cat(loc["xw"], f32))
    return hl, hc


def _outputs(nimg, P, rc, nloc):
    z = lambda shape, dt: np.zeros(shape, dt)
    return dict(kps=z(rc, KP_DTYPE), desc=z((rc, 32), np.uint8), ur=z(rc, f32), dep=z(rc, f32), n=z(nimg, np.int32),
                offsets=z(nimg + 1, np.int32), fm=z(rc, np.int32), nm1=z(P, np.int32), mt=z(max(nloc, 1), np.int32), nm2=z(P, np.int32),
                pose=z((2, P, 7), np.float64), inl=z((2, P), np.int32), eoff=z((2, P + 1), np.int32), efeat=z((2, rc), np.int32), outl=z((2, rc), np.uint8))


def _mk(W, H, max_batch):
    return ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=max_batch)


@pytest.mark.parametrize("geom", list(GEOM))
@pytest.mark.parametrize("with_po", [False, True])
def test_mono_step_equals_blocking_calls_and_the_oracle(geom, with_po):
    g = GEOM[geom]
    W, H, FX, FY, CX, CY, BFGT = g
    P = 4
    rng = np.random.default_rng(21)
    cam = camera(FX, FY, CX, CY, 0.0, 0.0, W, H)
    frames = [_frames(W, H, [1300 + 10 * s + p for p in range(P)]) for s in range(3)]
    batches = [f[0] for f in frames]
    ref = _mk(W, H, P)
    exs = [_mk(W, H, P) for _ in range(2)]
    m_last, m_loc = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
    qs = [_queries(ref, f[0], f[2], g, rng) for f in frames]
    rc = P * 1400
    steps = [replay.TrackingStep(e, cam, 0.0, 0.0, TH_LAST, TH_LOC, 0.8, True, monocular=True) for e in exs]
    outs = [_outputs(P, P, rc, max(int(q[1]["off"][-1]) for q in qs)) for _ in exs]

    def submit(i):
        hl, hc = qs[i]
        steps[i % 2].submit(batches[i], last=hl, local=hc, pose=hl["Tcw"] if with_po else None, local_world_pos=hc["xw"] if with_po else None)

    submit(0)
    for i in range(3):                       # one host thread, two handles in flight: submit i + 1 before collecting i
        if i + 1 < 3:
            submit(i + 1)
        o = outs[i % 2]
        o["ur"][:] = 7.0; o["dep"][:] = 7.0
        rows = steps[i % 2].collect(o)
        hl, hc = qs[i]
        # the blocking per-call ABI on a third handle
        ref.extract_batch(batches[i], lapping=(0, 1000))
        n, mono, off, kps, desc = ref.download(P)
        assert rows == int(off[-1]) and (o["n"] == n).all() and (o["offsets"] == off).all() and n.min() > 1000
        assert (o["kps"][:rows].view(np.uint8) == kps.view(np.uint8)).all() and (o["desc"][:rows] == desc).all()
        assert (o["ur"][:rows] == -1).all() and (o["dep"][:rows] == -1).all()
        fm, nm1 = m_last.SearchByProjectionLastFrame(ref, cam, hl["fimg"], hl["off"], hl["Tcw"], hl["dir"], hl["xw"], hl["oct"], hl["ang"], hl["desc"],
                                                     hl["obs"], TH_LAST, rows)
        assert (o["fm"][:rows] == fm).all() and (o["nm1"] == nm1).all() and nm1.min() > 50
        mt, nm2 = m_loc.SearchByProjection(ref, cam, hc["fimg"], hc["off"], hc["px"], hc["py"], hc["pxr"], hc["lvl"], hc["vc"], hc["desc"], th=TH_LOC)
        nq = int(hc["off"][-1])
        assert (o["mt"][:nq] == mt).all() and (o["nm2"] == nm2).all() and nm2.min() > 100
        if with_po:
            cam5 = [FX, FY, CX, CY, 0.0]
            pose1, outl1, inl1 = PoseOptimizationFrames(ref, hl["fimg"], hl["Tcw"], hl["xw"], cam5, feature_match=fm, total_rows=rows)
            pose2, outl2, inl2 = PoseOptimizationFrames(ref, hc["fimg"], hl["Tcw"], hc["xw"], cam5, query_offset=hc["off"], query_match=mt, total_rows=rows)
            for k, (pose, outl, inl) in enumerate([(pose1, outl1, inl1), (pose2, outl2, inl2)]):
                assert (o["pose"][k] == pose).all() and (o["inl"][k] == inl).all() and inl.min() > 30
                got = np.zeros(rows, np.uint8)
                for p in range(P):
                    e0, e1 = int(o["eoff"][k][p]), int(o["eoff"][k][p + 1])
                    got[int(off[p]) + o["efeat"][k][e0:e1]] = o["outl"][k][e0:e1]
                assert (got == outl).all()
    # the last batch's first frame against the CPU oracle: extraction with lapping (0, 1000), monoIndex, both searches with mvuRight = -1
    o, off = outs[0], outs[0]["offsets"]          # batch 2 ran on handle 0
    hl, hc = qs[2]
    a, b = int(off[0]), int(off[1])
    rmono, rk, rd = po.OracleExtractor(NF, 1.2, 8, 20, 7)(batches[2][0], (0, 1000))
    assert (o["kps"][a:b].view(np.uint8) == rk.view(np.uint8)).all() and (o["desc"][a:b] == rd).all()
    assert mono[0] == rmono and (rmono == 0) == (W <= 1000)
    if W > 1000:                                  # both fill directions present: features left of x = 1000 back-filled, the others in front
        assert 0 < rmono < len(rk) and (rk["x"][:rmono] > 1000).all() and (rk["x"][rmono:] <= 1000).all()
    sf = ref.GetScaleFactors()
    bounds = f32([0, W, 0, H])
    cam6 = f32([FX, FY, CX, CY, 0.0, 0.0])
    k, d, ur = o["kps"][a:b], o["desc"][a:b], np.full(b - a, -1, f32)
    l0, l1, c0, c1 = int(hl["off"][0]), int(hl["off"][1]), int(hc["off"][0]), int(hc["off"][1])
    wfm, wn1 = po.search_last(k, d, ur, bounds, sf, cam6, hl["Tcw"][0], 0, hl["xw"][l0:l1], hl["oct"][l0:l1], hl["ang"][l0:l1], hl["desc"][l0:l1],
                              hl["obs"][l0:l1], TH_LAST, True)
    got_fm = o["fm"][a:b].copy()
    got_fm[got_fm >= 0] -= l0
    assert (got_fm == wfm).all() and wn1 == o["nm1"][0]
    wmt, wn2 = po.search_local(k, d, ur, bounds, sf, hc["px"][c0:c1], hc["py"][c0:c1], hc["pxr"][c0:c1], hc["lvl"][c0:c1], hc["vc"][c0:c1],
                               hc["desc"][c0:c1], TH_LOC, 0.8)
    assert (o["mt"][c0:c1] == wmt).all() and wn2 == o["nm2"][0]
    for e in exs + [ref]:
        e.close()


def _se3f_from_pose(p7):
    """Optimizer.cc:406-410 + Sophus::SO3f normalisation + Frame::UpdatePoseMatrices, float32 operation by operation."""
    q = p7[:4].astype(f32)
    t = p7[4:].astype(f32)
    ln = f32(np.sqrt(f32(f32(f32(q[0] * q[0]) + f32(q[2] * q[2])) + f32(f32(q[1] * q[1]) + f32(q[3] * q[3])))))
    q = (q / ln).astype(f32)
    x, y, z, w = q
    t2x, t2y, t2z = f32(2) * x, f32(2) * y, f32(2) * z
    twx, twy, twz = f32(t2x * w), f32(t2y * w), f32(t2z * w)
    txx, txy, txz, tyy, tyz, tzz = f32(t2x * x), f32(t2y * x), f32(t2z * x), f32(t2y * y), f32(t2z * y), f32(t2z * z)
    R = np.array([f32(1) - f32(tyy + tzz), f32(txy - twz), f32(txz + twy), f32(txy + twz), f32(1) - f32(txx + tzz), f32(tyz - twx),
                  f32(txz - twy), f32(tyz + twx), f32(1) - f32(txx + tyy)], f32).reshape(3, 3)
    i = np.array([-x, -y, -z], f32)
    p = (t * f32(-1)).astype(f32)
    uv = np.array([f32(i[1] * p[2]) - f32(i[2] * p[1]), f32(i[2] * p[0]) - f32(i[0] * p[2]), f32(i[0] * p[1]) - f32(i[1] * p[0])], f32)
    u = (uv + uv).astype(f32)
    c = np.array([f32(i[1] * u[2]) - f32(i[2] * u[1]), f32(i[2] * u[0]) - f32(i[0] * u[2]), f32(i[0] * u[1]) - f32(i[1] * u[0])], f32)
    Ow = np.array([f32(f32(p[k] + f32(w * u[k])) + c[k]) for k in range(3)], f32)
    return np.concatenate([q, t]).astype(f32), R, t, Ow


def test_mono_chained_flow_matches_the_oracle_stage_by_stage():
    g = GEOM["euroc_752x480"]
    W, H, FX, FY, CX, CY, BFGT = g
    P = 2
    rng = np.random.default_rng(5)
    cam = camera(FX, FY, CX, CY, 0.0, 0.0, W, H)
    imgs, _, disps = _frames(W, H, [1400 + p for p in range(P)])
    ex = _mk(W, H, P)
    ex.extract_batch(imgs, lapping=(0, 1000))
    n, _, off, kps, desc = ex.download(P)
    sf = ex.GetScaleFactors()
    isg = ex.GetInverseScaleSigmaSquares()
    bounds = f32([0, W, 0, H])
    cam6 = f32([FX, FY, CX, CY, 0.0, 0.0])
    Tpred = np.tile(np.array([0.0005, -0.0008, 0.0003, 1, 0.004, -0.003, 0.002], f32), (P, 1))
    Tpred[:, :4] /= np.linalg.norm(Tpred[:, :4], axis=1)[:, None]
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    ch = dict(off=[0], xw=[], normal=[], max_dist=[], min_dist=[], desc=[], last_query=[])
    per = []
    for p in range(P):
        a, b = int(off[p]), int(off[p + 1])
        k, d = kps[a:b], desc[a:b]
        z = _depth(disps[p], k, BFGT)
        allf = np.arange(len(k))
        selL, selB = allf[::2], allf[1::2]
        pts = lambda s: np.stack([(k["x"][s] - CX) * z[s] / FX, (k["y"][s] - CY) * z[s] / FY, z[s]], 1).astype(f32)
        xwL = pts(selL)
        gross = rng.random(len(selL)) < 0.06                       # map points moved sideways by 8 px: still inside the search window, so the
        xwL[gross, 0] += (f32(8.0) * xwL[gross, 2] / f32(FX)).astype(f32)   # search matches them; the reprojection error makes them outliers
        last["xw"].append(xwL); last["oct"].append(k["octave"][selL].astype(np.int32)); last["ang"].append(k["angle"][selL].astype(f32))
        last["desc"].append(d[selL]); last["obs"].append((rng.random(len(selL)) < 0.9).astype(np.uint8)); last["off"].append(last["off"][-1] + len(selL))
        nC = 200                                                   # local map: the LastFrame points (shuffled), points of other features, out-of-view points
        xwB = pts(selB)
        xwC = np.stack([rng.uniform(-30, 30, nC), rng.uniform(-20, 20, nC), rng.uniform(-10, 40, nC)], 1).astype(f32)
        xw = np.concatenate([xwL, xwB, xwC])
        dsc = np.concatenate([d[selL], d[selB], rng.integers(0, 256, (nC, 32), dtype=np.uint8)])
        lq = np.concatenate([np.arange(len(selL)), np.full(len(selB) + nC, -1)]).astype(np.int32)
        octs = np.concatenate([k["octave"][selL], k["octave"][selB], rng.integers(0, 8, nC)])
        dist = np.linalg.norm(xw, axis=1).astype(f32)
        maxd = (dist * sf[octs] * rng.uniform(0.75, 1.3, len(xw))).astype(f32)
        nrm = xw / np.maximum(dist[:, None], 1e-6) + rng.normal(0, 0.35, xw.shape)
        nrm = (nrm / np.linalg.norm(nrm, axis=1)[:, None]).astype(f32)
        perm = rng.permutation(len(xw))
        ch["xw"].append(xw[perm]); ch["normal"].append(nrm[perm]); ch["max_dist"].append(maxd[perm]); ch["min_dist"].append((maxd / sf[7]).astype(f32)[perm])
        ch["desc"].append(dsc[perm]); ch["last_query"].append(lq[perm]); ch["off"].append(ch["off"][-1] + len(xw))
        per.append(dict(k=k, d=d))
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    hl = dict(fimg=np.arange(P, dtype=np.int32), off=np.array(last["off"], np.int32), Tcw=Tpred, dir=np.zeros(P, np.int32), xw=cat(last["xw"], f32),
              oct=cat(last["oct"], np.int32), ang=cat(last["ang"], f32), desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(off=np.array(ch["off"], np.int32), xw=cat(ch["xw"], f32), normal=cat(ch["normal"], f32), max_dist=cat(ch["max_dist"], f32),
              min_dist=cat(ch["min_dist"], f32), desc=cat(ch["desc"], np.uint8), last_query=cat(ch["last_query"], np.int32))
    npnt = int(hc["off"][-1])
    rc = P * 1400
    o = _outputs(P, P, rc, npnt)
    z_ = lambda shape, dt: np.zeros(shape, dt)
    o.update(c_in_view=z_(npnt, np.uint8), c_px=z_(npnt, f32), c_py=z_(npnt, f32), c_pxr=z_(npnt, f32), c_level=z_(npnt, np.int32),
             c_vc=z_(npnt, f32), c_pose=z_((P, 7), f32))
    step = replay.TrackingStep(ex, cam, 0.0, 0.0, TH_LAST, TH_LOC, 0.8, True, monocular=True)
    step.submit(imgs, last=hl, pose=Tpred, chain=hc)
    rows = step.collect(o)
    assert rows == int(off[-1]) and (o["offsets"] == off).all() and (o["ur"][:rows] == -1).all()
    logsf = f32(np.log(f32(1.2)))
    cam5 = f32([FX, FY, CX, CY, 0.0])
    checked = dict(released=0, skipped=0, in_view=0, local=0)
    for p in range(P):
        a, b = int(off[p]), int(off[p + 1])
        k, d = per[p]["k"], per[p]["d"]
        ur = np.full(len(k), -1, f32)
        l0, l1, c0, c1 = int(hl["off"][p]), int(hl["off"][p + 1]), int(hc["off"][p]), int(hc["off"][p + 1])
        xwL, obsL = hl["xw"][l0:l1], hl["obs"][l0:l1]
        # 1. the motion-model search (bMono: direction 0)
        fm0, nm0 = po.search_last(k, d, ur, bounds, sf, cam6, Tpred[p], 0, xwL, hl["oct"][l0:l1], hl["ang"][l0:l1], hl["desc"][l0:l1], obsL, TH_LAST, True)
        assert nm0 == o["nm1"][p] and nm0 > 80
        # 2. its PoseOptimization over monocular edges
        feat = np.nonzero(fm0 >= 0)[0]
        e0, e1 = int(o["eoff"][0][p]), int(o["eoff"][0][p + 1])
        assert (o["efeat"][0][e0:e1] == feat).all()
        obs3 = np.stack([k["x"][feat], k["y"][feat], ur[feat]], 1)
        want1 = po.pose_optimization(Tpred[p], xwL[fm0[feat]], obs3, isg[k["octave"][feat]], cam5)
        assert (o["outl"][0][e0:e1] == want1["outlier"]).all() and o["inl"][0][p] == want1["inliers"]
        assert np.abs(o["pose"][0][p] - want1["pose"]).max() < 1e-4
        # 3. outliers released; claims of the local-map search
        fm1 = fm0.copy()
        fm1[feat[want1["outlier"] != 0]] = -1
        got_fm = o["fm"][a:b].copy()
        got_fm[got_fm >= 0] -= l0
        assert (got_fm == fm1).all()
        checked["released"] += int((want1["outlier"] != 0).sum())
        claimed = ((fm1 >= 0) & (obsL[np.maximum(fm1, 0)] != 0)).astype(np.uint8)
        seen = np.zeros(l1 - l0, bool)
        seen[fm0[feat]] = True
        # 4. the Sophus::SE3f the frame holds, from the device's first pose
        posef, R, t, Ow = _se3f_from_pose(o["pose"][0][p])
        assert (o["c_pose"][p].view(np.uint32) == posef.view(np.uint32)).all()
        # 5. Frame::isInFrustum of the local map, minus the points the motion-model search already put into the frame
        fr = po.is_in_frustum(R, t, Ow, bounds, cam6, 8, logsf, hc["xw"][c0:c1], hc["normal"][c0:c1], hc["max_dist"][c0:c1], hc["min_dist"][c0:c1], 0.5)
        lq = hc["last_query"][c0:c1]
        skip = (lq >= 0) & seen[np.maximum(lq, 0)]
        vis = fr["in_view"].astype(bool) & ~skip
        assert (o["c_in_view"][c0:c1].astype(bool) == vis).all()
        for key, arr in (("proj_x", "c_px"), ("proj_y", "c_py"), ("proj_xr", "c_pxr"), ("view_cos", "c_vc")):
            assert (o[arr][c0:c1][vis].view(np.uint32) == fr[key][vis].view(np.uint32)).all(), key
        assert (o["c_level"][c0:c1][vis] == fr["level"][vis]).all()
        checked["skipped"] += int(skip.sum()); checked["in_view"] += int(vis.sum())
        # 6. SearchByProjection(F, local map points) against the claims
        vi = np.nonzero(vis)[0]
        mt_v, nm2 = po.search_local(k, d, ur, bounds, sf, fr["proj_x"][vi], fr["proj_y"][vi], fr["proj_xr"][vi], fr["level"][vi], fr["view_cos"][vi],
                                    hc["desc"][c0:c1][vi], TH_LOC, 0.8, claimed=claimed, trackdepth=fr["depth"][vi])
        want_mt = np.full(c1 - c0, -1, np.int32)
        want_mt[vi] = mt_v
        assert (o["mt"][c0:c1] == want_mt).all() and nm2 == o["nm2"][p] and nm2 > 100
        checked["local"] += int(nm2)
        # 7. PoseOptimization over every map point the frame holds: motion-model survivors + local-map matches (the latter win a feature)
        holder = fm1.copy()
        src2 = np.zeros(len(k), bool)
        for q_ in np.nonzero(want_mt >= 0)[0]:
            holder[want_mt[q_]] = q_
            src2[want_mt[q_]] = True
        feat2 = np.nonzero(holder >= 0)[0]
        e0, e1 = int(o["eoff"][1][p]), int(o["eoff"][1][p + 1])
        assert (o["efeat"][1][e0:e1] == feat2).all()
        xw2 = np.where(src2[feat2][:, None], hc["xw"][c0:c1][holder[feat2]], xwL[np.minimum(holder[feat2], len(xwL) - 1)])
        obs3 = np.stack([k["x"][feat2], k["y"][feat2], ur[feat2]], 1)
        want2 = po.pose_optimization(posef, xw2, obs3, isg[k["octave"][feat2]], cam5)
        assert (o["outl"][1][e0:e1] == want2["outlier"]).all() and o["inl"][1][p] == want2["inliers"]
        assert np.abs(o["pose"][1][p] - want2["pose"]).max() < 1e-4
    assert checked["released"] >= 3 and checked["skipped"] > 100 and checked["in_view"] > 400 and checked["local"] > 200, checked
    ex.close()


def test_mono_graph_replay_equals_eager_calls():
    """the device-resident monocular step as tools/mono_bench.py times it: extraction with lapping (0, 1000) and both device searches
    under orbm_set_device_query_bounds, captured once and replayed"""
    g = GEOM["euroc_752x480"]
    W, H, FX, FY, CX, CY, BFGT = g
    P = 4
    rng = np.random.default_rng(9)
    dev = torch.device("cuda", 0)
    cam = camera(FX, FY, CX, CY, 0.0, 0.0, W, H)
    imgsA, _, dispA = _frames(W, H, [1500 + p for p in range(P)])
    imgsB, _, _ = _frames(W, H, [1600 + p for p in range(P)])
    ex, ref = _mk(W, H, P), _mk(W, H, P)
    hl, hc = _queries(ref, imgsA, dispA, g, rng)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dl, dc = {k: T(v) for k, v in hl.items()}, {k: T(v) for k, v in hc.items()}
    nlast, nloc = int(hl["off"][-1]), int(hc["off"][-1])
    rows_cap = P * ex.max_features_per_image()
    m_last, m_loc = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
    out = lambda: (torch.full((rows_cap,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev),
                   torch.full((nloc,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev))

    def step(e, src, o):
        e.extract_batch_device(src.data_ptr(), P, W, H, lapping=(0, 1000))
        m_last.SearchByProjectionLastFrameDevice(e, cam, P, dl["fimg"], dl["off"], dl["Tcw"], dl["dir"], dl["xw"], dl["oct"], dl["ang"], dl["desc"],
                                                 dl["obs"], TH_LAST, o[0], o[1])
        m_loc.SearchByProjectionDevice(e, cam, P, dc["fimg"], dc["off"], dc["px"], dc["py"], dc["pxr"], dc["lvl"], dc["vc"], dc["desc"], o[2], o[3], th=TH_LOC)

    def results(e, o):
        torch.cuda.synchronize()
        n, mono, off, kps, desc = e.download(P)
        rows = int(off[-1])
        return [n.copy(), mono.copy(), kps.view(np.uint8).copy(), desc.copy(), o[0][:rows].cpu().numpy(), o[1].cpu().numpy(), o[2].cpu().numpy(),
                o[3].cpu().numpy()]

    d_in = T(imgsA)
    oA = out(); step(ref, d_in, oA); wantA = results(ref, oA)
    d_inB = T(imgsB)
    oB = out(); step(ref, d_inB, oB); wantB = results(ref, oB)
    assert wantA[5].min() > 50 and wantA[7].min() > 100 and (wantA[1] == 0).all()
    o = out()
    ex.set_device_query_bounds(max(nlast, nloc), int(max(np.diff(hl["off"]).max(), np.diff(hc["off"]).max())), rows_cap)
    step(ex, d_in, o)
    for a, b in zip(results(ex, o), wantA):
        assert a.shape == b.shape and (a == b).all()
    gr = ex.graph_capture(lambda: step(ex, d_in, o))
    assert ex.graph_kernels(gr) >= 10
    for src, want in [(imgsA, wantA), (imgsB, wantB), (imgsA, wantA)]:
        d_in.copy_(torch.from_numpy(src))
        for t in o:
            t.fill_(-7)
        ex.graph_launch(gr)
        for i, (a, b) in enumerate(zip(results(ex, o), want)):
            assert a.shape == b.shape and (a == b).all(), i
    ex.graph_destroy(gr)
    ex.close(); ref.close()


def _stereo_queries(hl, hc):
    """the monocular query sets on a stereo batch of the same left images: frame p is image 2p"""
    sl, sc = dict(hl), dict(hc)
    sl["fimg"] = sc["fimg"] = (2 * hl["fimg"]).astype(np.int32)
    return sl, sc


def _run(step, imgs, P, nimg, hl, hc, po_=True):
    o = _outputs(nimg, P, nimg * 1400, int(hc["off"][-1]))
    step.submit(imgs, last=hl, local=hc, pose=hl["Tcw"] if po_ else None, local_world_pos=hc["xw"] if po_ else None)
    rows = step.collect(o)
    return rows, o


def _same(a, b):
    rows_a, oa = a
    rows_b, ob = b
    assert rows_a == rows_b
    for key in oa:
        x, y = oa[key], ob[key]
        if key in ("kps", "desc", "ur", "dep", "fm"):
            x, y = x[:rows_a], y[:rows_a]
        assert (x.view(np.uint8) == y.view(np.uint8)).all(), key


def test_mono_step_refusals_leave_the_handle_usable():
    g = GEOM["euroc_752x480"]
    W, H, FX, FY, CX, CY, BFGT = g
    P = 2
    rng = np.random.default_rng(13)
    cam = camera(FX, FY, CX, CY, BFGT, BFGT / FX, W, H)
    left, right, disps = _frames(W, H, [1700 + p for p in range(2 * P + 1)])
    probe = _mk(W, H, 2 * P + 1)
    hl5, hc5 = _queries(probe, left, disps, g, rng)
    hl, hc = _queries(probe, left[:P], disps[:P], g, rng)
    probe.close()
    ex, fresh = _mk(W, H, 2 * P), _mk(W, H, 2 * P)
    mono = replay.TrackingStep(ex, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True, monocular=True)

    def refused(imgs, last, local):
        with pytest.raises(OrbError, match=f"orb_status {ORB_ERR_INVALID}:"):
            mono.submit(imgs, last=last, local=local)
    # 2 * P + 1 frames on a handle of max_batch 2 * P
    refused(left, hl5, hc5)
    # a frame image equal to n_frames
    bad = dict(hl); bad["fimg"] = np.array([0, P], np.int32)
    refused(left[:P], bad, hc)
    badc = dict(hc); badc["fimg"] = np.array([P, 0], np.int32)
    refused(left[:P], hl, badc)
    # a nonzero direction: bMono never searches forward or backward
    for dval in (1, 2):
        bad = dict(hl); bad["dir"] = np.array([0, dval], np.int32)
        refused(left[:P], bad, hc)
    # the same handle runs a correct monocular step, then a correct stereo step; each equals a fresh handle's
    got = _run(mono, left[:P], P, P, hl, hc)
    want = _run(replay.TrackingStep(fresh, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True, monocular=True), left[:P], P, P, hl, hc)
    _same(got, want)
    assert got[1]["nm1"].min() > 50 and (got[1]["ur"][:got[0]] == -1).all()
    stereo_imgs = np.ascontiguousarray(np.stack([im for p in range(P) for im in (left[p], right[p])]))
    sl, sc = _stereo_queries(hl, hc)
    got = _run(replay.TrackingStep(ex, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True), stereo_imgs, P, 2 * P, sl, sc)
    fresh2 = _mk(W, H, 2 * P)
    want = _run(replay.TrackingStep(fresh2, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True), stereo_imgs, P, 2 * P, sl, sc)
    _same(got, want)
    for e in (ex, fresh, fresh2):
        e.close()


@pytest.mark.parametrize("with_po", [False, True])
def test_no_state_leaks_between_mono_and_stereo_steps(with_po):
    g = GEOM["euroc_752x480"]
    W, H, FX, FY, CX, CY, BFGT = g
    P = 2
    rng = np.random.default_rng(17)
    cam = camera(FX, FY, CX, CY, BFGT, BFGT / FX, W, H)
    left, right, disps = _frames(W, H, [1800 + p for p in range(P)])
    stereo_imgs = np.ascontiguousarray(np.stack([im for p in range(P) for im in (left[p], right[p])]))
    probe = _mk(W, H, P)
    hl, hc = _queries(probe, left, disps, g, rng)
    probe.close()
    sl, sc = _stereo_queries(hl, hc)
    used, fresh_s, fresh_m = _mk(W, H, 2 * P), _mk(W, H, 2 * P), _mk(W, H, 2 * P)
    mk = lambda e, m: replay.TrackingStep(e, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True, monocular=m)
    # stereo right after monocular on one handle == stereo on a fresh handle
    _run(mk(used, True), left, P, P, hl, hc, with_po)
    got_s = _run(mk(used, False), stereo_imgs, P, 2 * P, sl, sc, with_po)
    want_s = _run(mk(fresh_s, False), stereo_imgs, P, 2 * P, sl, sc, with_po)
    _same(got_s, want_s)
    rows, o = got_s
    assert (o["ur"][:rows] > 0).sum() > 500           # the stereo step has real mvuRight values ...
    # ... and monocular right after that stereo step == monocular on a fresh handle (mvuRight -1, not the stereo step's values)
    got_m = _run(mk(used, True), left, P, P, hl, hc, with_po)
    want_m = _run(mk(fresh_m, True), left, P, P, hl, hc, with_po)
    _same(got_m, want_m)
    assert (got_m[1]["ur"][:got_m[0]] == -1).all() and (got_m[1]["dep"][:got_m[0]] == -1).all()
    for e in (used, fresh_s, fresh_m):
        e.close()
