"""GPU tier: Optimizer::PoseOptimization and its correspondence walk at the sizes the device path produces, against the fp64 CPU
oracle and numpy.  test_poseopt_gpu.py covers a narrow band (at most 2 000 edges and 9 frames, identity start, EuRoC's camera, depths
of 2-12 m); this file covers:
  A. k_pose_opt through PoseOptimization: edge counts at the kernel's boundaries (the n < 3 return, the one-round rule below 10 edges,
     the 256-thread stride) up to the 16 000 edges of the largest frame a search produces; launches of 64 and 128 frames with empty and
     one- or two-edge frames between large ones; starting poses rotated by up to pi with camera centres 10 m, 500 m and 2 km from the
     origin; the EuRoC, KITTI and 4K cameras; near points, far stereo points below a pixel of disparity and far monocular points,
     with 0, 15 and 60 % outliers.
  B. k_pose_edges through PoseEdgesDevice, bit for bit against numpy: on handles of 12 276 and 12 277 rows (either side of the
     48 KB a launch gets without opting into more shared memory) and of 16 160 rows; feature_match only, query_match only and both
     (the chained form); stereo and monocular frames; an empty frame, a match on a frame's last row and query entries past the frame.
  C. The callers at 16 000 features on the 4K stereo batch: PoseOptimizationFrames in both forms, the replay step with
     PoseOptimization, the chained flow stage by stage from a rotated start pose; and a KITTI-shaped monocular batch of 10 000 features.
Bar (as test_poseopt_gpu.py): same rounds, LM iteration / trial counts within the oracle's spread, pose within 1e-4, at most one
outlier flag different (a chi2 on the threshold)."""
import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import (ORBextractor, ORBmatcher, PoseEdgesDevice, PoseOptimization, PoseOptimizationFrames, camera,
                                              replay, synth)
from _tracking import chain_queries, check_chained_flow, step_outputs
from test_poseopt_gpu import qR, quat
from test_zz_many_features_gpu import cam_for, kitti, scene4k16k, step_queries   # noqa: F401  (kitti, scene4k16k: module fixtures)

pytestmark = pytest.mark.gpu
TOL = 1e-4
EUROC = (435.2, 435.2, 320.0, 240.0, 47.9)
KITTI = (718.856, 718.856, 607.19, 185.22, 386.1448)
CAM4K = cam_for(3840, 2160)[:5]
CAMS = dict(euroc=EUROC, kitti=KITTI, cam4k=CAM4K)
CENTRES = (10.0, 500.0, 2000.0)
# k_pose_edges holds one int per row of the handle in dynamic shared memory next to 48 B of __shared__ arrays (ptxas -v, sm_90a):
# without opting in, a launch gets 48 KB in all, so 12 276 rows is the last capacity that fits and 12 277 the first that needs more
PE_STATIC = 48
LAST_DEFAULT_ROWS = (48 * 1024 - PE_STATIC) // 4
assert LAST_DEFAULT_ROWS == 12276


# ---- frames and the oracle bar ----------------------------------------------------------------------------------------------
def qmul(a, b):
    """Hamilton product of two x y z w quaternions: qR(qmul(a, b)) == qR(a) @ qR(b)."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def unit(v):
    return v / np.linalg.norm(v)


def start_and_true_pose(rng, centre, angle=None, motion=(0.03, 2.0)):
    """A float32 Tcw whose rotation turns by up to pi about a random axis and whose camera centre lies `centre` metres from the origin,
    and the true pose: a motion of up to motion[0] metres and motion[1] degrees away from it."""
    ang = rng.uniform(0, np.pi) if angle is None else angle
    q0 = quat(rng.normal(size=3), ang)
    t0 = -qR(q0) @ (unit(rng.normal(size=3)) * centre)
    pose0 = np.concatenate([q0, t0]).astype(np.float32)
    q0f, t0f = pose0[:4].astype(np.float64), pose0[4:].astype(np.float64)
    dq = quat(rng.normal(size=3), np.deg2rad(rng.uniform(0.3, 1.0) * motion[1]))
    R = qR(qmul(dq, q0f / np.linalg.norm(q0f)))
    t = qR(dq) @ t0f + unit(rng.normal(size=3)) * rng.uniform(0.3, 1.0) * motion[0]
    return pose0, R, t


def make_frame(seed, n, cam, centre=10.0, angle=None, motion=(0.03, 2.0), mono_frac=0.3, outlier_frac=0.15, depth="mid", noise=0.7):
    """n map points (float32 world coordinates) seen by a camera whose true pose is `motion` away from the pose handed to the optimiser.
    depth="mid": 2-12 m.  depth="extremes": a third near (0.3-1 m), a third far stereo (40-400 m: below one pixel of disparity on
    EuRoC's camera), a third far monocular.  inv_sigma2 of all 8 levels of a 1.2 pyramid."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, bf = cam
    pose0, R, t = start_and_true_pose(rng, centre, angle, motion)
    if depth == "mid":
        z = rng.uniform(2, 12, n)
        stereo = rng.random(n) >= mono_frac
    else:
        kind = rng.integers(0, 3, n)
        z = np.where(kind == 0, rng.uniform(0.3, 1.0, n), rng.uniform(40, 400, n))
        stereo = (kind == 1) | ((kind == 0) & (rng.random(n) >= mono_frac))
    stereo &= bf / z < 2 * cx - 1                     # the right-eye column inside the image
    d = np.where(stereo, bf / z, 0.0)
    u = d + rng.random(n) * (2 * cx - d)
    v = rng.uniform(0, 2 * cy, n)
    Xc = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)
    Xw = ((Xc - t) @ R).astype(np.float32)
    Xc = Xw.astype(np.float64) @ R.T + t              # where the float32 points really are
    u, v = fx * Xc[:, 0] / Xc[:, 2] + cx, fy * Xc[:, 1] / Xc[:, 2] + cy
    obs = np.stack([u, v, u - bf / Xc[:, 2]], 1) + rng.normal(0, noise, (n, 3))
    obs[:, 2] = np.where(stereo, np.maximum(obs[:, 2], 0.0), -1.0)
    bad = rng.random(n) < outlier_frac
    obs[bad, :2] += rng.normal(0, 30, (int(bad.sum()), 2))
    w = 1 / (1.2 ** rng.integers(0, 8, n)) ** 2
    return dict(pose=pose0, world_pos=Xw, obs=obs.astype(np.float32), inv_sigma2=w.astype(np.float32), depth=z, stereo=stereo)


def check(g, f, cam):
    """test_poseopt_gpu.py's bar for one frame of PoseOptimization (host form, with the LM counts).  Near convergence the gain ratio
    is rounding noise, so the counts are held to within a couple of steps of the oracle's -- or, where they are not, of the range the
    oracle's own counts span when the map points move by one ulp.  (Far from the origin an ulp of a map point is a real change of
    the problem -- 1.2e-4 m at 2 km -- so the perturbed poses are not held to the tolerance, only their rounds and counts are used.)
    Far from the origin the rounding of Xc = R Xw + t (|t| up to 2 km, |Xc| a few metres) is ~1e-12 of chi2, above the gain of a
    converged LM step: every trial after convergence is accepted or rejected on rounding noise, lambda climbs to 1e9-1e17 and the
    trial count of such a frame spans 20-67 across one-ulp moves of its points.  Where the oracle's own trial counts spread wider
    than the +-4 allowance, the count is held to what g2o's loop can produce (1-10 trials per iteration); the iteration count, the
    rounds, the pose and the outlier flags keep their bar."""
    c5 = np.float32(cam)
    r = po.pose_optimization(f["pose"], f["world_pos"], f["obs"], f["inv_sigma2"], c5)
    its, trials = [r["iterations"]], [r["trials"]]

    def within():
        if max(trials) - min(trials) > 8:
            trials_ok = g["iterations"] <= g["trials"] <= 10 * g["iterations"]
        else:
            trials_ok = min(trials) - 4 <= g["trials"] <= max(trials) + 4
        return min(its) - 2 <= g["iterations"] <= max(its) + 2 and trials_ok

    if not within():
        for k in range(16):
            step = np.random.default_rng(k).choice([-1, 0, 1], f["world_pos"].shape) * np.float32(2 ** -23)
            rk = po.pose_optimization(f["pose"], (f["world_pos"] * (1 + step)).astype(np.float32), f["obs"], f["inv_sigma2"], c5)
            assert rk["rounds"] == r["rounds"]
            its.append(rk["iterations"])
            trials.append(rk["trials"])
    n = len(f["world_pos"])
    assert r["rounds"] == (0 if n < 3 else 1 if n < 10 else 4), (n, r["rounds"])
    assert g["rounds"] == r["rounds"] and within(), (n, g["rounds"], g["iterations"], g["trials"], r["rounds"], its, trials)
    assert np.abs(g["pose"] - r["pose"]).max() < TOL, (n, np.abs(g["pose"] - r["pose"]).max())
    assert abs(g["inliers"] - r["inliers"]) <= 1 and int((g["outlier"] != r["outlier"]).sum()) <= 1, (n, g["inliers"], r["inliers"])
    if n < 3:      # Optimizer.cc:292-293: returns 0 and leaves the frame's pose as it was
        assert g["inliers"] == 0 and g["rounds"] == 0 and (g["pose"] == f["pose"].astype(np.float64)).all() and not g["outlier"].any()
    return r


def check_pose(pose, inliers, outlier, f, cam):
    """The bar for the callers that return no LM counts (PoseOptimizationFrames, the replay step)."""
    r = po.pose_optimization(f["pose"], f["world_pos"], f["obs"], f["inv_sigma2"], np.float32(cam))
    assert np.abs(pose - r["pose"]).max() < TOL, np.abs(pose - r["pose"]).max()
    assert abs(int(inliers) - r["inliers"]) <= 1 and int((outlier != r["outlier"]).sum()) <= 1, (int(inliers), r["inliers"])
    return r


@pytest.fixture(scope="module")
def ex():
    e = ORBextractor(1000, 1.2, 8, 20, 7, max_width=640, max_height=480, max_batch=2)
    yield e
    e.close()


# ---- A. k_pose_opt through PoseOptimization ------------------------------------------------------------------------------------
BOUNDARY_SIZES = [2, 3, 9, 10, 11, 255, 256, 257, 513, 4096, 16000]


def test_edge_counts_at_the_kernel_boundaries(ex):
    """The n < 3 return, the last one-round (9) and first four-round (10) sizes, the 256-thread stride and the 16 000 edges of the
    largest frame a search produces, in one launch, mixed stereo / monocular, rotated and far-from-origin start poses."""
    frames = [make_frame(100 + i, n, EUROC, centre=CENTRES[i % 3], mono_frac=0.3 + 0.4 * (i % 2)) for i, n in enumerate(BOUNDARY_SIZES)]
    got = PoseOptimization(ex, frames, EUROC)
    for g, f in zip(got, frames):
        check(g, f, EUROC)
    assert [g["rounds"] for g in got] == [0, 1, 1, 4, 4, 4, 4, 4, 4, 4, 4]
    assert got[-1]["inliers"] > 0.8 * 16000 * 0.85


def batch_sizes(nf, seed):
    """Edge counts of a launch of nf frames: 3-3 000, with empty, one- and two-edge frames first, last and between large ones."""
    rng = np.random.default_rng(seed)
    n = rng.integers(3, 3001, nf)
    n[8::8] = np.resize([0, 1, 2], len(n[8::8]))
    n[7::8] = rng.integers(2500, 3001, len(n[7::8]))
    n[9::8] = rng.integers(2500, 3001, len(n[9::8]))
    n[0], n[1], n[-1], n[-2] = 0, 3000, 1, 2999
    return n


@pytest.mark.parametrize("nf,cam", [(64, "cam4k"), (128, "kitti")])
def test_launch_of_many_frames(ex, nf, cam):
    """One launch of the bench's 64 frames and one of 128: every frame's eoff slice, and the frames the kernel leaves alone come back
    as the reference leaves them."""
    sizes = batch_sizes(nf, nf)
    frames = [make_frame(1000 * nf + i, int(n), CAMS[cam], centre=CENTRES[i % 3], motion=(0.1, 5.0) if i % 5 == 0 else (0.03, 2.0),
                         mono_frac=(0.0, 0.3, 1.0)[i % 3], outlier_frac=(0.0, 0.15, 0.6)[(i // 3) % 3], depth=("mid", "extremes")[(i // 2) % 2])
              for i, n in enumerate(sizes)]
    got = PoseOptimization(ex, frames, CAMS[cam])
    assert len(got) == nf
    for g, f in zip(got, frames):
        check(g, f, CAMS[cam])
    assert sum(g["rounds"] == 0 for g in got) >= 3 + nf // 16


@pytest.mark.parametrize("cam", sorted(CAMS))
def test_far_and_rotated_start_poses(ex, cam):
    """Camera centres 10 m, 500 m and 2 km from the world origin (world points in float32 there), rotations up to pi, true motions of a
    few cm / degrees and of 10 cm / 5 degrees."""
    frames = [make_frame(300 + 10 * i + j, 900, CAMS[cam], centre=c, angle=(None, 3.1)[j % 2], motion=((0.02, 1.0), (0.1, 5.0))[j])
              for i, c in enumerate(CENTRES) for j in range(2)]
    got = PoseOptimization(ex, frames, CAMS[cam])
    for g, f in zip(got, frames):
        r = check(g, f, CAMS[cam])
        assert r["inliers"] > 0.6 * 900


@pytest.mark.parametrize("cam", sorted(CAMS))
def test_depth_extremes_and_outlier_shares(ex, cam):
    """Near points (0.3-1 m), far stereo points (40-400 m) and far monocular points in one frame; 0, 15 and 60 % outliers."""
    fx, fy, cx, cy, bf = CAMS[cam]
    frames = [make_frame(400 + i, 1500, CAMS[cam], centre=500.0, outlier_frac=share, depth="extremes") for i, share in enumerate((0.0, 0.15, 0.6))]
    far_stereo = frames[0]["stereo"] & (frames[0]["depth"] > 40)
    assert far_stereo.sum() > 300
    if cam == "euroc":
        assert (bf / frames[0]["depth"][far_stereo] < 1).mean() > 0.8          # disparity below a pixel
    got = PoseOptimization(ex, frames, CAMS[cam])
    for g, f in zip(got, frames):
        check(g, f, CAMS[cam])


# ---- B. k_pose_edges through PoseEdgesDevice, against numpy ------------------------------------------------------------------
FORMS = ("feature_match", "query_match", "both")


def edge_sources(off, frames, kinds, form, rng):
    """Search outputs of the frames (feature_match rows / query_match entries) and, per frame, the edges the walk must produce:
    (features in feature order, their world positions).  A query_match entry overrides the feature_match row of its feature; entries
    of -1 and of features past the frame's end are ignored.  kinds: "normal", "empty" (no match at all), "last" (+ the last row)."""
    total = int(off[-1])
    use_fm, use_qm = form in ("feature_match", "both"), form in ("query_match", "both")
    fm, xw1, qoff, qm, xq, want = np.full(total, -1, np.int32), [], [0], [], [], []
    n1 = 0
    for img, kind in zip(frames, kinds):
        a, b = int(off[img]), int(off[img + 1])
        nk = b - a
        holder, pos = np.full(nk, -1), np.zeros((nk, 3), np.float32)
        if use_fm and kind != "empty":
            feats = np.nonzero(rng.random(nk) < 0.5)[0]
            if kind == "last":
                feats = np.union1d(feats, [nk - 1])
            ids = n1 + rng.permutation(len(feats))                  # the search's queries are not in feature order
            p1 = rng.normal(0, 100, (len(feats), 3)).astype(np.float32)
            fm[a + feats] = ids
            holder[feats] = ids
            pos[feats] = p1[ids - n1]
            xw1.append(p1)
            n1 += len(feats)
        if use_qm:
            feats = np.nonzero(rng.random(nk) < (0 if kind == "empty" else 0.4))[0]
            if kind == "last":
                feats = np.union1d(feats, [nk - 1])
            junk = np.array([-1, -1, nk, nk + 1, nk + 37, 1 << 20], np.int32)
            ent = rng.permutation(np.concatenate([feats, junk]).astype(np.int32))
            pq = rng.normal(0, 100, (len(ent), 3)).astype(np.float32)
            q0 = qoff[-1]
            ok = (ent >= 0) & (ent < nk)
            holder[ent[ok]] = q0 + np.nonzero(ok)[0]
            pos[ent[ok]] = pq[ok]
            qm.append(ent)
            xq.append(pq)
            qoff.append(q0 + len(ent))
        f = np.nonzero(holder >= 0)[0]
        want.append((f, pos[f]))
        if kind == "empty":
            assert len(f) == 0
        if kind == "last":
            assert f[-1] == nk - 1
    cat = lambda xs, w: np.concatenate(xs).reshape(-1, w).astype(np.float32) if xs else np.zeros((0, w), np.float32)
    src = {}
    if use_fm:
        src["feature_match"] = fm
        src["world_pos"] = cat(xw1, 3)
    if use_qm:
        src["query_offset"] = np.array(qoff, np.int32)
        src["query_match"] = np.concatenate(qm).astype(np.int32)
        src["query_world_pos" if use_fm else "world_pos"] = cat(xq, 3)
    return src, want


def run_edge_walk(e, off, kps, uR, frames, kinds, form, rng):
    """PoseEdgesDevice on the frames against the walk restated in numpy, bit for bit (uR None: a monocular batch)."""
    import torch
    dev = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    src, want = edge_sources(off, frames, kinds, form, rng)
    cap = max(sum(int(off[i + 1] - off[i]) for i in frames), 1)
    o_off = torch.full((len(frames) + 1,), -7, dtype=torch.int32, device=dev)
    o_feat = torch.zeros(cap, dtype=torch.int32, device=dev)
    o_xw = torch.zeros((cap, 3), dtype=torch.float32, device=dev)
    o_obs = torch.zeros((cap, 3), dtype=torch.float32, device=dev)
    o_w = torch.zeros(cap, dtype=torch.float32, device=dev)
    PoseEdgesDevice(e, len(frames), T(np.array(frames, np.int32)), T(src.pop("world_pos")), o_off, o_feat, o_xw, o_obs, o_w,
                    **{k: T(v) for k, v in src.items()})
    torch.cuda.synchronize()
    eo, feat, xw, obs, w = (t.cpu().numpy() for t in (o_off, o_feat, o_xw, o_obs, o_w))
    isg = e.GetInverseScaleSigmaSquares()
    assert eo[0] == 0 and eo[-1] == sum(len(f) for f, _ in want), (eo, [len(f) for f, _ in want])
    for p, (img, (f, pos)) in enumerate(zip(frames, want)):
        a = int(off[img])
        s = slice(int(eo[p]), int(eo[p + 1]))
        assert eo[p + 1] - eo[p] == len(f), (form, p, eo[p + 1] - eo[p], len(f))
        assert (feat[s] == f).all(), (form, p)
        assert (xw[s].view(np.uint32) == pos.view(np.uint32)).all(), (form, p)
        k = kps[a + f]
        ur = uR[a + f] if uR is not None else np.full(len(f), -1, np.float32)
        assert (obs[s].view(np.uint32) == np.stack([k["x"], k["y"], ur], 1).astype(np.float32).view(np.uint32)).all(), (form, p)
        assert (w[s] == isg[k["octave"]]).all(), (form, p)
    return want


@pytest.fixture(scope="module", params=[LAST_DEFAULT_ROWS - 160, LAST_DEFAULT_ROWS - 159], ids=["12276rows", "12277rows"])
def window_handle(request):
    """Handles either side of the 48 KB default launch window of k_pose_edges; the row capacity (not the image) sizes the launch, so
    the images are 640x480."""
    nf, W, H, P = request.param, 640, 480, 3
    e = ORBextractor(nf, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * P)
    assert e.max_features_per_image() == nf + 20 * 8
    imgs = np.stack([x for s in range(P) for x in synth.stereo_pair(W, H, seed=710 + s)[:2]])
    yield dict(ex=e, imgs=imgs, P=P, rows=nf + 160)
    e.close()


@pytest.mark.parametrize("form", FORMS)
def test_edge_walk_either_side_of_the_default_window(window_handle, form):
    Wh = window_handle
    e, imgs, P = Wh["ex"], Wh["imgs"], Wh["P"]
    assert Wh["rows"] in (LAST_DEFAULT_ROWS, LAST_DEFAULT_ROWS + 1)
    rng = np.random.default_rng(Wh["rows"] + len(form))
    e.extract_batch(imgs)
    e.stereo_batch(P, EUROC[4], 0.11)
    _, _, off, kps, _ = e.download(2 * P)
    uR, _ = e.stereo_download(int(off[-1]))
    assert (uR[off[0]:off[1]] >= 0).sum() > 200
    run_edge_walk(e, off, kps, uR, [2, 1, 4, 0], ["normal", "empty", "last", "normal"], form, rng)
    # a monocular batch on the same handle (no stereo run): obs[:, 2] = -1
    e.extract_batch(np.ascontiguousarray(imgs[0::2]))
    _, _, off, kps, _ = e.download(P)
    run_edge_walk(e, off, kps, None, [2, 1, 0], ["normal", "empty", "last"], form, rng)


@pytest.mark.parametrize("form", FORMS)
def test_edge_walk_16k(scene4k16k, form):
    """The 3840x2160 stereo batch at 16 000 features (16 160 rows per image, 64 640 B of shared memory per launch)."""
    S = scene4k16k
    want = run_edge_walk(S["ex"], S["off"], S["kps"], S["uR"], [2, 1, 0], ["normal", "empty", "last"], form, np.random.default_rng(61))
    assert min(len(want[0][0]), len(want[2][0])) > 3000


# ---- C. the callers at 16 000 features ---------------------------------------------------------------------------------------
def device_frame_problem(S, p, rng, cam, centre, angle, outlier_frac=0.1):
    """Map points for the features of frame p (left image of pair p, or image p of a monocular batch): back-projected from the
    device's keypoints at their stereo depth (at 5-60 m where there is none) through a true pose `centre` metres from the origin and
    rotated by `angle`, in float32, with `outlier_frac` of them moved by a tenth of their depth.  Returns (start pose, world positions of every
    feature of the frame)."""
    fx, fy, cx, cy = cam[:4]
    i = S["img_of"](p)
    a, b = int(S["off"][i]), int(S["off"][i + 1])
    k, dep = S["kps"][a:b], (S["dep"][a:b] if S.get("dep") is not None else np.zeros(b - a, np.float32))
    z = np.where(dep > 0, dep, rng.uniform(5, 60, b - a)).astype(np.float64)
    Xc = np.stack([(k["x"] - cx) * z / fx, (k["y"] - cy) * z / fy, z], 1)
    pose0, R, t = start_and_true_pose(rng, centre, angle, (0.005, 0.3))     # stereo depths of the 4K scene are 0.3-1 m
    Xw = (Xc - t) @ R + rng.normal(0, 0.0005, Xc.shape) * z[:, None]          # about a pixel of noise at any depth
    bad = rng.random(b - a) < outlier_frac
    Xw[bad] += rng.normal(0, 0.1, (int(bad.sum()), 3)) * z[bad, None]
    return pose0, Xw.astype(np.float32)


def pose_frames_case(S, cam, rng, centres, angles):
    """PoseOptimizationFrames on every listed frame of the batch in both forms, against the oracle, including mvbOutlier of every row."""
    e, off, kps, P = S["ex"], S["off"], S["kps"], S["P"]
    uR = S["uR"]
    total = int(off[-1])
    isg = e.GetInverseScaleSigmaSquares()
    fimg = np.array([S["img_of"](p) for p in range(P)], np.int32)
    probs = [device_frame_problem(S, p, rng, cam, centres[p], angles[p]) for p in range(P)]
    poses = np.stack([pr[0] for pr in probs])
    for form in ("feature_match", "query_match"):
        qoff, xw_all, fm, qm, feats_of = [0], [], np.full(total, -1, np.int32), [], []
        for p in range(P):
            a, b = rows = int(off[fimg[p]]), int(off[fimg[p] + 1])
            feats = np.nonzero(rng.random(b - a) < 0.7)[0]
            feats = np.union1d(feats, [b - a - 1])
            order = rng.permutation(feats)
            fm[a + order] = qoff[-1] + np.arange(len(order))
            qm.append(order.astype(np.int32))
            xw_all.append(probs[p][1][order])
            qoff.append(qoff[-1] + len(order))
            feats_of.append((rows, feats))
        xw_all = np.concatenate(xw_all)
        kw = dict(feature_match=fm) if form == "feature_match" else dict(query_offset=np.array(qoff, np.int32), query_match=np.concatenate(qm))
        hp, ho, hi = PoseOptimizationFrames(e, fimg, poses, xw_all, cam, total_rows=total, **kw)
        touched = np.zeros(total, bool)
        for p, ((a, b), feats) in enumerate(feats_of):
            k = kps[a + feats]
            f = dict(pose=poses[p], world_pos=probs[p][1][feats], obs=np.stack([k["x"], k["y"], uR[a + feats]], 1), inv_sigma2=isg[k["octave"]])
            r = check_pose(hp[p], hi[p], ho[a + feats], f, cam)
            assert r["inliers"] > 0.6 * len(feats), (form, p, r["inliers"], len(feats))
            touched[a:b] = True
            rest = np.ones(b - a, bool)
            rest[feats] = False
            assert not ho[a:b][rest].any()
        assert not ho[:total][~touched].any()                  # rows of images that are not listed frames stay as they were


def test_pose_optimization_frames_16k(scene4k16k):
    S = scene4k16k
    pose_frames_case(S, np.float32(S["cam6"][:5]), np.random.default_rng(67), centres=(500.0, 2000.0), angles=(2.0, 3.1))


def test_kitti_monocular_10k(kitti):
    """A KITTI-shaped monocular batch of 10 000 features (10 160 rows, inside the default window): the monocular edge walk in every
    form, and PoseOptimizationFrames from far, rotated start poses."""
    S = kitti
    assert S["ex"].max_features_per_image() == 10160
    assert (S["uR"] == -1).all()
    for form in FORMS:
        run_edge_walk(S["ex"], S["off"], S["kps"], None, [1, 0], ["normal", "last"], form, np.random.default_rng(71))
    cam = np.float32(list(S["cam6"][:4]) + [KITTI[4]])      # bf of KITTI's rig; every observation is monocular
    pose_frames_case(S, cam, np.random.default_rng(73), centres=(2000.0, 500.0), angles=(1.0, 2.5))


@pytest.fixture(scope="module")
def step16k(scene4k16k):
    """A second handle of the 4K scene's size for orbr_submit (the step extracts the batch again on its own handle)."""
    S = scene4k16k
    e = ORBextractor(16000, 1.2, 8, 20, 7, max_width=S["w"], max_height=S["h"], max_batch=2 * S["P"])
    yield e
    e.close()


def test_replay_step_with_pose_optimization_16k(scene4k16k, step16k):
    """orbr_submit with PoseOptimization after both searches on 16 000-feature frames: poses, inliers, edge tables and outlier flags equal
    the per-call path (each search, then PoseOptimizationFrames on its result arrays) and the oracle."""
    S = scene4k16k
    ex, P, cam6 = S["ex"], S["P"], S["cam6"]
    fx, fy, cx, cy, bf, b = cam6
    cam, cam5 = camera(*cam6, S["w"], S["h"]), np.float32(cam6[:5])
    isg = ex.GetInverseScaleSigmaSquares()
    hl, hc = step_queries(S, np.random.default_rng(79))
    rows, off, kps, uR = int(S["off"][-1]), S["off"], S["kps"], S["uR"]
    fm, nm1 = ORBmatcher(0.9, True).SearchByProjectionLastFrame(ex, cam, hl["fimg"], hl["off"], hl["Tcw"], hl["dir"], hl["xw"], hl["oct"], hl["ang"],
                                                               hl["desc"], hl["obs"], 15.0, rows)
    mt, nm2 = ORBmatcher(0.8, True).SearchByProjection(ex, cam, hc["fimg"], hc["off"], hc["px"], hc["py"], hc["pxr"], hc["lvl"], hc["vc"], hc["desc"],
                                                       th=3.0)
    assert nm1.min() > 200 and nm2.min() > 200
    assert (hc["off"] == hl["off"]).all()
    local_xw = hl["xw"]                                 # step_queries draws both query sets from the same points, in the same order
    per_call = [PoseOptimizationFrames(ex, hl["fimg"], hl["Tcw"], hl["xw"], cam5, feature_match=fm, total_rows=rows),
                PoseOptimizationFrames(ex, hc["fimg"], hl["Tcw"], local_xw, cam5, query_offset=hc["off"], query_match=mt, total_rows=rows)]
    o = step_outputs(2 * P, P, 2 * P * 16160, int(hc["off"][-1]))
    st = replay.TrackingStep(step16k, cam, bf, b, 15.0, 3.0, 0.8, True)
    st.submit(np.ascontiguousarray(S["imgs"]), last=hl, local=hc, pose=hl["Tcw"], local_world_pos=local_xw)
    assert st.collect(o) == rows and (o["offsets"] == off).all()
    assert (o["fm"][:rows] == fm).all() and (o["mt"] == mt).all()
    for s, (hp, ho, hi) in enumerate(per_call):
        assert (o["pose"][s] == hp).all() and (o["inl"][s] == hi).all(), s
        for p in range(P):
            a, e = int(off[2 * p]), int(off[2 * p + 1])
            if s == 0:
                holder = fm[a:e].copy()
                holder[holder >= 0] -= hl["off"][p]
            else:
                holder = np.full(e - a, -1)
                q = np.arange(hc["off"][p], hc["off"][p + 1])
                q = q[mt[q] >= 0]
                holder[mt[q]] = q - hc["off"][p]
            feats = np.nonzero(holder >= 0)[0]
            e0, e1 = int(o["eoff"][s][p]), int(o["eoff"][s][p + 1])
            assert (o["efeat"][s][e0:e1] == feats).all(), (s, p)
            assert (o["outl"][s][e0:e1] == ho[a + feats]).all() and ho[a:e].sum() == ho[a + feats].sum(), (s, p)
            k = kps[a + feats]
            f = dict(pose=hl["Tcw"][p], world_pos=hl["xw"][hl["off"][p]:][holder[feats]], obs=np.stack([k["x"], k["y"], uR[a + feats]], 1),
                     inv_sigma2=isg[k["octave"]])
            r = check_pose(o["pose"][s][p], o["inl"][s][p], o["outl"][s][e0:e1], f, cam5)
            assert r["inliers"] > 0.7 * len(feats), (s, p, r["inliers"], len(feats))


def test_chained_flow_16k(scene4k16k, step16k):
    """The chained flow (orbr_chain) on the 16 000-feature batch, stage by stage as test_zz_chain_gpu.py does at 640x480, from a start
    pose rotated by 40 degrees with the camera 50 m from the world origin.  The handle's 16 160 rows size both edge walks' launches."""
    S = scene4k16k
    P, W, H = S["P"], S["w"], S["h"]
    BF, B = S["cam6"][4:]
    CAM6, BOUNDS = np.float32(S["cam6"]), np.float32([0, W, 0, H])
    cam = camera(*S["cam6"], W, H)
    rng = np.random.default_rng(83)
    ex, off, kps, desc, dep, uR = S["ex"], S["off"], S["kps"], S["desc"], S["dep"], S["uR"]
    sf, isg = ex.GetScaleFactors(), ex.GetInverseScaleSigmaSquares()
    # the frames' true poses: 40 degrees about a random axis, camera centre 50 m out; the prediction is a few mm / 0.05 degrees off
    Ttrue, Tpred = [], np.zeros((P, 7), np.float32)
    for p in range(P):
        q = quat(rng.normal(size=3), np.deg2rad(40))
        R = qR(q)
        t = -R @ (unit(rng.normal(size=3)) * 50.0)
        Ttrue.append((R, t))
        dq = quat(rng.normal(size=3), np.deg2rad(0.05))
        qp = qmul(dq, q)
        Tpred[p] = np.concatenate([qp / np.linalg.norm(qp), qR(dq) @ t + rng.normal(0, 0.001, 3)]).astype(np.float32)
    Tpred[:, :4] /= np.linalg.norm(Tpred[:, :4], axis=1)[:, None]
    frames = []
    for p in range(P):
        a, b = int(off[2 * p]), int(off[2 * p + 1])
        st = np.nonzero(dep[a:b] > 0)[0]
        frames.append(dict(k=kps[a:b], d=desc[a:b], z=dep[a:b], ur=uR[a:b], last=st[::2], other=st[1::2], rows=(a, b)))
    # the map in world coordinates: gross errors 12 px to the side, 1 000 points around each camera, mostly out of view
    hl, hc = chain_queries(frames, rng, sf, CAM6, Tpred, np.arange(0, 2 * P, 2, dtype=np.int32), gross_px=12, n_far=1000,
                           far_box=((-60, 60), (-40, 40), (-10, 80)), world=Ttrue)
    npnt = int(hc["off"][-1])
    o = step_outputs(2 * P, P, 2 * P * 16160, npnt, chain_points=npnt)
    step = replay.TrackingStep(step16k, cam, BF, B, 15.0, 3.0, 0.8, True)
    step.submit(np.ascontiguousarray(S["imgs"]), last=hl, pose=Tpred, chain=hc)
    rows = step.collect(o)
    assert rows == int(off[-1]) and (o["offsets"] == off).all()
    assert (o["kps"][:rows].view(np.uint8) == kps.view(np.uint8)).all() and (o["ur"][:rows].view(np.uint32) == uR.view(np.uint32)).all()
    nm0, nm2, checked = check_chained_flow(o, hl, hc, frames, CAM6, BOUNDS, sf, isg, 15.0, 3.0)
    assert nm0.min() > 150 and nm2.min() > 100, (nm0, nm2)      # the scene's stereo rows are few (~600 per frame)
    assert checked["released"] >= 3 and checked["skipped"] > 300 and checked["in_view"] > 400 and checked["local"] > 200, checked
    # the optimised pose is the true one to within the noise of 16 000 matches
    for p in range(P):
        assert np.abs(o["pose"][1][p][4:] - Ttrue[p][1]).max() < 0.05, (p, o["pose"][1][p][4:], Ttrue[p][1])
