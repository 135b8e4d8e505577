"""Checks of the replay tracking step (orbr_submit / orbr_collect, replay.TrackingStep) shared by its stereo, monocular and RGB-D tests:
the output arrays `collect` fills, the chained flow's query sets and its stage-by-stage walk against the oracle, the comparison with the
blocking per-call C ABI, and the identity of two steps' results."""
import numpy as np

from orb_slam3_detailed_comments_b200 import ORBmatcher, PoseOptimizationFrames
from orb_slam3_detailed_comments_b200._native import KP_DTYPE
from oracle import pyoracle as po

f32 = np.float32
TOL = 1e-4                     # the optimised poses against the fp64 oracle, as tests/test_poseopt_gpu.py


def step_outputs(nimg, n_frames, rows_cap, n_local, chain_points=0):
    """The host arrays TrackingStep.collect fills for a batch of nimg images and n_frames frames; the chained flow's per-point arrays
    and pose when chain_points > 0."""
    z = lambda shape, dt: np.zeros(shape, dt)
    o = dict(kps=z(rows_cap, KP_DTYPE), desc=z((rows_cap, 32), np.uint8), ur=z(rows_cap, f32), dep=z(rows_cap, f32), n=z(nimg, np.int32),
             offsets=z(nimg + 1, np.int32), fm=z(rows_cap, np.int32), nm1=z(n_frames, np.int32), mt=z(max(n_local, 1), np.int32),
             nm2=z(n_frames, np.int32), pose=z((2, n_frames, 7), np.float64), inl=z((2, n_frames), np.int32), eoff=z((2, n_frames + 1), np.int32),
             efeat=z((2, rows_cap), np.int32), outl=z((2, rows_cap), np.uint8))
    if chain_points:
        o.update(c_in_view=z(chain_points, np.uint8), c_px=z(chain_points, f32), c_py=z(chain_points, f32), c_pxr=z(chain_points, f32),
                 c_level=z(chain_points, np.int32), c_vc=z(chain_points, f32), c_pose=z((n_frames, 7), f32))
    return o


def run_step(step, imgs, hl, hc, with_po=True, depth=None):
    """One submit and collect of `step` (PoseOptimization after both searches with with_po); returns (rows, outputs)."""
    o = step_outputs(len(imgs), len(hl["fimg"]), len(imgs) * 1400, int(hc["off"][-1]))
    step.submit(imgs, last=hl, local=hc, pose=hl["Tcw"] if with_po else None, local_world_pos=hc["xw"] if with_po else None, depth=depth)
    return step.collect(o), o


def same_results(a, b, stereo=False):
    """Two steps' (rows, outputs) are identical byte for byte, row arrays up to `rows`.  A stereo step writes mvuRight / mvDepth of the
    left images' rows only (ComputeStereoMatches is per left keypoint), so its right images' rows of ur / dep are not compared."""
    rows_a, oa = a
    rows_b, ob = b
    assert rows_a == rows_b
    rows = np.arange(rows_a)
    if stereo:
        off = oa["offsets"]
        rows = np.concatenate([np.arange(off[2 * p], off[2 * p + 1]) for p in range(len(off) // 2)])
    for key in oa:
        x, y = oa[key], ob[key]
        if key in ("kps", "desc", "fm"):
            x, y = x[:rows_a], y[:rows_a]
        elif key in ("ur", "dep"):
            x, y = x[rows], y[rows]
        assert (x.view(np.uint8) == y.view(np.uint8)).all(), key


def check_against_per_call(o, rows, ref, cam, hl, hc, th_last, th_local, cam5, with_po):
    """A collected step `o` equals the blocking per-call ABI on `ref`, which holds the same batch extracted (and its stereo): both
    projection searches, then with_po PoseOptimizationFrames on each search's result arrays -- poses, inliers and the outlier flags of
    the step's edge tables regrouped per row.  Returns nm1, nm2 and the (2, n_frames) inliers of the two PoseOptimization calls (None
    without)."""
    fm, nm1 = ORBmatcher(0.9, True).SearchByProjectionLastFrame(ref, cam, hl["fimg"], hl["off"], hl["Tcw"], hl["dir"], hl["xw"], hl["oct"], hl["ang"],
                                                               hl["desc"], hl["obs"], th_last, rows)
    assert (o["fm"][:rows] == fm).all() and (o["nm1"] == nm1).all()
    mt, nm2 = ORBmatcher(0.8, True).SearchByProjection(ref, cam, hc["fimg"], hc["off"], hc["px"], hc["py"], hc["pxr"], hc["lvl"], hc["vc"], hc["desc"],
                                                       th=th_local)
    nq = int(hc["off"][-1])
    assert (o["mt"][:nq] == mt).all() and (o["nm2"] == nm2).all()
    if not with_po:
        return nm1, nm2, None
    per_call = [PoseOptimizationFrames(ref, hl["fimg"], hl["Tcw"], hl["xw"], cam5, feature_match=fm, total_rows=rows),
                PoseOptimizationFrames(ref, hc["fimg"], hl["Tcw"], hc["xw"], cam5, query_offset=hc["off"], query_match=mt, total_rows=rows)]
    for k, (pose, outl, inl) in enumerate(per_call):
        assert (o["pose"][k] == pose).all() and (o["inl"][k] == inl).all()
        got = np.zeros(rows, np.uint8)
        for p, img in enumerate(hl["fimg"]):
            e0, e1 = int(o["eoff"][k][p]), int(o["eoff"][k][p + 1])
            got[int(o["offsets"][img]) + o["efeat"][k][e0:e1]] = o["outl"][k][e0:e1]
        assert (got == outl).all()
    return nm1, nm2, np.stack([inl for _, _, inl in per_call])


def se3f_from_pose(p7):
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


def chain_queries(frames, rng, sf, cam6, Tpred, fimg, gross_px=None, n_far=200, far_box=((-30, 30), (-20, 20), (-10, 40)), world=None):
    """The query sets (hl, hc) of orbr_chain.  frames[p]: keypoints k, descriptors d, depth z of every feature, and two disjoint feature
    selections `last` and `other`.  The LastFrame map points are the `last` features back-projected at z; 6 % of them are gross errors,
    at half their depth (gross_px None: same pixel, so the search matches them and the stereo residual throws them out) or moved gross_px
    pixels sideways (inside the search window, then thrown out by the reprojection error).  The local map holds those points in a
    shuffled order, the `other` features' points and n_far random points in far_box (camera coordinates), mostly out of view.
    world[p] = (R, t) of the frame's Tcw maps camera coordinates to the world; without it the world is the camera."""
    fx, fy, cx, cy = cam6[:4]
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    ch = dict(off=[0], xw=[], normal=[], max_dist=[], min_dist=[], desc=[], last_query=[])
    for p, f in enumerate(frames):
        k, d, z, selL, selB = f["k"], f["d"], f["z"], f["last"], f["other"]
        if world is None:
            to_world, Oc = (lambda Xc: Xc.astype(f32)), np.zeros(3, f32)
        else:
            R, t = world[p]
            to_world, Oc = (lambda Xc: ((Xc - t) @ R).astype(f32)), (-R.T @ t).astype(f32)
        cpts = lambda s: np.stack([(k["x"][s] - cx) * z[s] / fx, (k["y"][s] - cy) * z[s] / fy, z[s]], 1).astype(f32)
        XcL = cpts(selL)
        gross = rng.random(len(selL)) < 0.06
        if gross_px is None:
            XcL[gross] *= f32(0.5)
        else:
            XcL[gross, 0] += (f32(gross_px) * XcL[gross, 2] / fx).astype(f32)
        xwL = to_world(XcL)
        last["xw"].append(xwL); last["oct"].append(k["octave"][selL].astype(np.int32)); last["ang"].append(k["angle"][selL].astype(f32))
        last["desc"].append(d[selL]); last["obs"].append((rng.random(len(selL)) < 0.9).astype(np.uint8)); last["off"].append(last["off"][-1] + len(selL))
        xwB = to_world(cpts(selB))
        xwC = to_world(np.stack([rng.uniform(lo, hi, n_far) for lo, hi in far_box], 1))
        xw = np.concatenate([xwL, xwB, xwC])
        dsc = np.concatenate([d[selL], d[selB], rng.integers(0, 256, (n_far, 32), dtype=np.uint8)])
        lq = np.concatenate([np.arange(len(selL)), np.full(len(selB) + n_far, -1)]).astype(np.int32)
        octs = np.concatenate([k["octave"][selL], k["octave"][selB], rng.integers(0, len(sf), n_far)])
        dist = np.linalg.norm(xw - Oc, axis=1).astype(f32)
        maxd = (dist * sf[octs] * rng.uniform(0.75, 1.3, len(xw))).astype(f32)
        nrm = (xw - Oc) / np.maximum(dist[:, None], 1e-6) + rng.normal(0, 0.35, xw.shape)     # MapPoint::mNormalVector: camera -> point
        nrm = (nrm / np.linalg.norm(nrm, axis=1)[:, None]).astype(f32)
        perm = rng.permutation(len(xw))
        ch["xw"].append(xw[perm]); ch["normal"].append(nrm[perm]); ch["max_dist"].append(maxd[perm])
        ch["min_dist"].append((maxd / sf[-1]).astype(f32)[perm]); ch["desc"].append(dsc[perm]); ch["last_query"].append(lq[perm])
        ch["off"].append(ch["off"][-1] + len(xw))
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=Tpred, dir=np.zeros(len(frames), np.int32), xw=cat(last["xw"], f32),
              oct=cat(last["oct"], np.int32), ang=cat(last["ang"], f32), desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(off=np.array(ch["off"], np.int32), xw=cat(ch["xw"], f32), normal=cat(ch["normal"], f32), max_dist=cat(ch["max_dist"], f32),
              min_dist=cat(ch["min_dist"], f32), desc=cat(ch["desc"], np.uint8), last_query=cat(ch["last_query"], np.int32))
    return hl, hc


def run_chained_flow(ex, step, imgs, off, frames, cam6, fimg, rows_cap, th_last, th_local, gross_px=None, depth=None):
    """One chained step of `frames` (check_chained_flow's form) on `ex`, predicted a few mm and 0.05 degrees off the identity, with
    chain_queries' map from seed 5, checked stage by stage; `off` is the batch's compact row offsets.  Returns rows, the collected
    outputs and check_chained_flow's counts."""
    P = len(frames)
    sf, isg = ex.GetScaleFactors(), ex.GetInverseScaleSigmaSquares()
    Tpred = np.tile(np.array([0.0005, -0.0008, 0.0003, 1, 0.004, -0.003, 0.002], f32), (P, 1))
    Tpred[:, :4] /= np.linalg.norm(Tpred[:, :4], axis=1)[:, None]
    hl, hc = chain_queries(frames, np.random.default_rng(5), sf, cam6, Tpred, fimg, gross_px=gross_px)
    npnt = int(hc["off"][-1])
    o = step_outputs(len(imgs), P, rows_cap, npnt, chain_points=npnt)
    step.submit(imgs, last=hl, pose=Tpred, chain=hc, depth=depth)
    rows = step.collect(o)
    assert rows == int(off[-1]) and (o["offsets"] == off).all()
    bounds = f32([0, imgs.shape[2], 0, imgs.shape[1]])
    return (rows, o) + check_chained_flow(o, hl, hc, frames, cam6, bounds, sf, isg, th_last, th_local)


def check_chained_flow(o, hl, hc, frames, cam6, bounds, sf, isg, th_last, th_local):
    """The collected chained flow (orbr_chain: motion-model search -> PoseOptimization -> outlier release -> Sophus::SE3f ->
    Frame::isInFrustum of the local map -> SearchByProjection(F, local map points) -> PoseOptimization over every map point of the frame;
    Tracking.cc:3389-3522, 4010-4062) against the CPU oracle, stage by stage.  Integer stages and every float32 value of isInFrustum
    are identical; the two optimised poses agree with the fp64 oracle to TOL (the device's own first pose is what the later oracle stages
    start from).  frames[p]: keypoints k, descriptors d, mvuRight ur and the compact rows (a, b) of the frame's image.  Returns each
    frame's motion-model and local-map match counts and the totals of released outliers, skipped and in-view local-map points, local-map
    matches and stereo edges of the first PoseOptimization."""
    logsf = f32(np.log(sf[1]))
    cam5 = cam6[:5]
    nm0s, nm2s = [], []
    checked = dict(released=0, skipped=0, in_view=0, local=0, stereo=0)
    for p, f in enumerate(frames):
        k, d, ur, (a, b) = f["k"], f["d"], f["ur"], f["rows"]
        l0, l1, c0, c1 = int(hl["off"][p]), int(hl["off"][p + 1]), int(hc["off"][p]), int(hc["off"][p + 1])
        xwL, obsL = hl["xw"][l0:l1], hl["obs"][l0:l1]
        # 1. the motion-model search
        fm0, nm0 = po.search_last(k, d, ur, bounds, sf, cam6, hl["Tcw"][p], 0, xwL, hl["oct"][l0:l1], hl["ang"][l0:l1], hl["desc"][l0:l1], obsL,
                                  th_last, True)
        assert nm0 == o["nm1"][p]
        # 2. its PoseOptimization: one edge per matched feature, in feature order
        feat = np.nonzero(fm0 >= 0)[0]
        e0, e1 = int(o["eoff"][0][p]), int(o["eoff"][0][p + 1])
        assert (o["efeat"][0][e0:e1] == feat).all()
        obs3 = np.stack([k["x"][feat], k["y"][feat], ur[feat]], 1)
        checked["stereo"] += int((ur[feat] > 0).sum())
        want1 = po.pose_optimization(hl["Tcw"][p], xwL[fm0[feat]], obs3, isg[k["octave"][feat]], cam5)
        assert (o["outl"][0][e0:e1] == want1["outlier"]).all() and o["inl"][0][p] == want1["inliers"]
        assert np.abs(o["pose"][0][p] - want1["pose"]).max() < TOL
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
        # 4. the pose the frame holds (Sophus::SE3f) and its matrices, from the device's first pose
        posef, R, t, Ow = se3f_from_pose(o["pose"][0][p])
        assert (o["c_pose"][p].view(np.uint32) == posef.view(np.uint32)).all()
        # 5. Frame::isInFrustum of the local map points, minus the ones the motion-model search already put into the frame
        fr = po.is_in_frustum(R, t, Ow, bounds, cam6, len(sf), logsf, hc["xw"][c0:c1], hc["normal"][c0:c1], hc["max_dist"][c0:c1],
                              hc["min_dist"][c0:c1], 0.5)
        lq = hc["last_query"][c0:c1]
        skip = (lq >= 0) & seen[np.maximum(lq, 0)]
        vis = fr["in_view"].astype(bool) & ~skip
        assert (o["c_in_view"][c0:c1].astype(bool) == vis).all()
        for key, arr in (("proj_x", "c_px"), ("proj_y", "c_py"), ("proj_xr", "c_pxr"), ("view_cos", "c_vc")):
            assert (o[arr][c0:c1][vis].view(np.uint32) == fr[key][vis].view(np.uint32)).all(), key
        assert (o["c_level"][c0:c1][vis] == fr["level"][vis]).all()
        checked["skipped"] += int(skip.sum()); checked["in_view"] += int(vis.sum())
        # 6. SearchByProjection(F, local map points): the in-view ones, in list order, against the claims
        vi = np.nonzero(vis)[0]
        mt_v, nm2 = po.search_local(k, d, ur, bounds, sf, fr["proj_x"][vi], fr["proj_y"][vi], fr["proj_xr"][vi], fr["level"][vi], fr["view_cos"][vi],
                                    hc["desc"][c0:c1][vi], th_local, 0.8, claimed=claimed, trackdepth=fr["depth"][vi])
        want_mt = np.full(c1 - c0, -1, np.int32)
        want_mt[vi] = mt_v
        assert (o["mt"][c0:c1] == want_mt).all() and nm2 == o["nm2"][p]
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
        assert np.abs(o["pose"][1][p] - want2["pose"]).max() < TOL
        nm0s.append(nm0); nm2s.append(nm2)
    return np.array(nm0s), np.array(nm2s), checked
