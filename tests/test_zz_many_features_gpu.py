"""GPU tier: frames and keyframes of up to 16 384 feature rows through the matchers, bit for bit against the oracle.  Frames whose
shared-memory form does not fit a CTA run the global-memory form (the *_xl kernels); which form ran is read from the
library's launch counter (the global form adds k_stage_frames_xl).  Covered: ORB-SLAM3's 5x-feature monocular initialisation on a
EuRoC-shaped frame (F2 on the device and as host arrays); KITTI-shaped 1241x376 monocular frames at 10 000 features (both per-frame
searches, with and without the isInFrustum mask, SearchByBoW(KF, F), relocalisation); a 3840x2160 stereo batch at 16 000 features
(both per-frame searches, SearchByBoW(KF, F), relocalisation, orbv_transform with its BowVector, the replay step and a captured graph);
host keyframes of 5 401, 10 000 and 16 384 features through every ORBM_KF_* variant, SearchByBoW(KF, KF) and SearchForTriangulation;
the switch points (the last size the shared-memory form takes and one row more); and the refusals."""
import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth
from orb_slam3_detailed_comments_b200 import _native as N

pytestmark = pytest.mark.gpu
SMEM_OPTIN = 232448                     # an H100's opt-in shared memory per block


def launches():
    return int(N.lib().orb_kernel_launches())


def init_rsm(n2):
    """k_proj_resolve's shared memory for SearchForInitialization on n2 rows (matcher.cu launch_proj)."""
    fsm = (n2 * 23 + 16 + 15) // 16 * 16
    return fsm + 1024 * 8 * 8 + 1024 * 4 + n2 * 9 + 1024 * 5 + 256


RESOLVE_STATIC = 256                    # k_proj_resolve's __shared__ arrays (rotation histogram, kept bins, match count)
INIT_LAST_SHARED = max(n for n in range(4000, 6000) if init_rsm(n) + RESOLVE_STATIC <= SMEM_OPTIN)


def noisy_f1(kL, dL, rng):
    """F1 = a frame's features plus noisy copies of a third of its level-0 ones (test_matcher_gpu.py)."""
    l0 = np.nonzero(kL["octave"] == 0)[0]
    dup = rng.choice(l0, len(l0) // 3, replace=False)
    kp1 = np.concatenate([kL[dup], kL])
    dd = dL[dup].copy()
    flips = rng.integers(0, 256, (len(dup), 3))
    for j in range(3):
        dd[np.arange(len(dup)), flips[:, j] // 8] ^= (1 << (flips[:, j] % 8)).astype(np.uint8)
    d1 = np.concatenate([dd, dL])
    return kp1, d1, np.stack([kp1["x"], kp1["y"]], 1).astype(np.float32)


@pytest.fixture(scope="module")
def euroc():
    """752x480 monocular frames through ORBextractor(5 * 1000, 1.2, 8, 20, 7): Tracking's initialisation extractor for EuRoC."""
    w, h, nf = 752, 480, 5000
    a = synth.frame(w, h, 301, 1.0, 400)
    b = np.roll(a, (2, 3), (0, 1))
    ref = po.OracleExtractor(nf, 1.2, 8, 20, 7)
    _, kL, dL = ref(a, (0, 1000))
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    ex.extract_batch(b[None], (0, 1000))
    _, _, off, k2, d2 = ex.download(1)
    yield dict(w=w, h=h, ex=ex, kL=kL, dL=dL, k2=k2, d2=d2)
    ex.close()


def test_euroc_monocular_initialization(euroc):
    E = euroc
    ex, w, h = E["ex"], E["w"], E["h"]
    cam = camera(458.0, 457.0, 367.0, 248.0, 0.0, 0.11, w, h)
    bounds = np.array([0, w, 0, h], np.float32)
    kp1, d1, prev = noisy_f1(E["kL"], E["dL"], np.random.default_rng(3))
    assert len(E["k2"]) > 4700
    for win, nnratio, check in [(100, 0.9, True), (30, 0.8, False)]:
        m = ORBmatcher(nnratio, check)
        n0 = launches()
        g_dev, n_dev = m.SearchForInitialization(ex, cam, kp1, d1, prev, win, target_image=0)
        assert launches() - n0 == 4       # k_frame_grid, k_stage_frames_xl, k_proj_candidates_xl, k_proj_resolve_xl
        g_host, n_host = m.SearchForInitialization(ex, cam, kp1, d1, prev, win, kp2=E["k2"], desc2=E["d2"])
        rm, rnm = po.search_initialization(kp1, d1, prev, E["k2"], E["d2"], bounds, win, nnratio, check)
        assert n_dev == rnm and (g_dev == rm).all(), (win, n_dev, rnm, int((g_dev != rm).sum()))
        assert n_host == rnm and (g_host == rm).all(), win
        assert rnm > 100, rnm


def test_initialization_switch_point(euroc):
    """Host F2 of the last size the shared-memory form takes and one row more: both match the oracle, the second one stages its
    frame once in global memory (one launch more)."""
    E = euroc
    ex, w, h = E["ex"], E["w"], E["h"]
    cam = camera(458.0, 457.0, 367.0, 248.0, 0.0, 0.11, w, h)
    bounds = np.array([0, w, 0, h], np.float32)
    kp1, d1, prev = noisy_f1(E["kL"], E["dL"], np.random.default_rng(5))
    k2, d2 = E["k2"], E["d2"]
    counts = []
    for n2 in (INIT_LAST_SHARED, INIT_LAST_SHARED + 1):
        assert len(k2) >= n2
        m = ORBmatcher(0.9, True)
        n0 = launches()
        g, n = m.SearchForInitialization(ex, cam, kp1, d1, prev, 100, kp2=k2[:n2], desc2=d2[:n2])
        counts.append(launches() - n0)
        rm, rnm = po.search_initialization(kp1, d1, prev, k2[:n2], d2[:n2], bounds, 100, 0.9, True)
        assert n == rnm and (g == rm).all(), n2
    assert counts == [3, 4], counts


def cam_for(w, h):
    s = w / 640.0
    return 435.2 * s, 435.2 * s, w / 2.0, h / 2.0, 47.9 * s, 0.11


@pytest.fixture(scope="module")
def scene4k16k():
    """A 3840x2160 stereo batch of two pairs at 16 000 features per eye (16 160 rows per image)."""
    w, h, P, nf = 3840, 2160, 2, 16000
    fx, fy, cx, cy, bf, b = cam_for(w, h)
    imgs = np.zeros((2 * P, h, w), np.uint8)
    for p in range(P):
        imgs[2 * p], imgs[2 * p + 1], _ = synth.stereo_pair(w, h, seed=500 + p, dmin=2.0, dmax=0.5 * fx)
    lasts = []
    for p in range(P):
        eL, eR = po.OracleExtractor(nf, 1.2, 8, 20, 7), po.OracleExtractor(nf, 1.2, 8, 20, 7)
        _, kL, dL = eL(imgs[2 * p])
        _, kR, dR = eR(imgs[2 * p + 1])
        lasts.append((kL, dL) + tuple(po.stereo_matches(eL, eR, kL, dL, kR, dR, np.float32(bf), np.float32(b))[:2]))
        imgs[2 * p] = np.roll(imgs[2 * p], (1, 3 + p), (0, 1))
        imgs[2 * p + 1] = np.roll(imgs[2 * p + 1], (1, 3 + p), (0, 1))
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=2 * P)
    ex.extract_batch(imgs)
    ex.stereo_batch(P, bf, b)
    _, _, off, kps, desc = ex.download(2 * P)
    uR, dep = ex.stereo_download(int(off[-1]))
    yield dict(w=w, h=h, P=P, ex=ex, imgs=imgs, cam6=(fx, fy, cx, cy, bf, b), lasts=lasts, off=off, kps=kps, desc=desc, uR=uR, dep=dep,
               img_of=lambda p: 2 * p)            # frame p = the left image of pair p
    ex.close()


def test_search_local_points_16k(scene4k16k):
    S = scene4k16k
    P, ex, off, (fx, fy, cx, cy, bf, b) = S["P"], S["ex"], S["off"], S["cam6"]
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(17)
    qoff, px, py, pxr, lv, vc, qd = [0], [], [], [], [], [], []
    claimed = np.zeros(int(off[-1]), np.uint8)
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        sel = np.concatenate([sel, rng.choice(sel, len(sel))])
        jit = rng.normal(0, 1.5, (len(sel), 2)).astype(np.float32)
        x = (kL["x"][sel] + 3 + p + jit[:, 0]).astype(np.float32)
        y = (kL["y"][sel] + 1 + jit[:, 1]).astype(np.float32)
        px.append(x); py.append(y)
        pxr.append((x - np.float32(bf) / ldep[sel]).astype(np.float32))
        lv.append(np.clip(kL["octave"][sel] + rng.integers(-1, 2, len(sel)), 0, 7).astype(np.int32))
        vc.append(rng.uniform(0.99, 1.0, len(sel)).astype(np.float32))
        qd.append(dL[sel])
        qoff.append(qoff[-1] + len(sel))
        claimed[off[2 * p]:off[2 * p + 1]] = rng.random(off[2 * p + 1] - off[2 * p]) < 0.15
    px, py, pxr, lv, vc, qd = map(np.concatenate, (px, py, pxr, lv, vc, qd))
    n0 = launches()
    match, nm = ORBmatcher(0.8, True).SearchByProjection(ex, camera(fx, fy, cx, cy, bf, b, S["w"], S["h"]), [2 * p for p in range(P)], qoff,
                                                         px, py, pxr, lv, vc, qd, th=3.0, feature_claimed=claimed)
    assert launches() - n0 == 5           # k_frame_grid, k_stage_frames_xl, candidates, parallel and sequential resolve
    for p in range(P):
        a, e = off[2 * p], off[2 * p + 1]
        s = slice(qoff[p], qoff[p + 1])
        rmatch, rnm = po.search_local(S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], bounds, ex.GetScaleFactors(), px[s], py[s], pxr[s],
                                      lv[s], vc[s], qd[s], 3.0, 0.8, claimed=claimed[a:e])
        assert rnm == nm[p] and (match[s] == rmatch).all(), p
        assert rnm > 200


def test_search_last_frame_16k(scene4k16k):
    S = scene4k16k
    P, ex, off, cam6 = S["P"], S["ex"], S["off"], S["cam6"]
    fx, fy, cx, cy, bf, b = cam6
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(19)
    qoff, xw, lo, la, qd, ob, Tcw, dirs = [0], [], [], [], [], [], [], []
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        z = ldep[sel]
        xw.append(np.stack([(kL["x"][sel] - cx) * z / fx, (kL["y"][sel] - cy) * z / fy, z], 1).astype(np.float32))
        zmid = float(np.median(z))
        Tcw.append(np.array([0, 0, 0, 1, (3 + p) * zmid / fx, zmid / fy, 0.0], np.float32))
        lo.append(kL["octave"][sel].astype(np.int32)); la.append(kL["angle"][sel].astype(np.float32))
        qd.append(dL[sel]); ob.append((rng.random(len(sel)) < 0.7).astype(np.uint8)); dirs.append(0)
        qoff.append(qoff[-1] + len(sel))
    xw, lo, la, qd, ob = map(np.concatenate, (xw, lo, la, qd, ob))
    fm, nm = ORBmatcher(0.9, True).SearchByProjectionLastFrame(ex, camera(*cam6, S["w"], S["h"]), [2 * p for p in range(P)], qoff,
                                                                np.stack(Tcw), dirs, xw, lo, la, qd, ob, 15.0, int(off[-1]))
    for p in range(P):
        a, e = off[2 * p], off[2 * p + 1]
        s = slice(qoff[p], qoff[p + 1])
        rfm, rnm = po.search_last(S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], bounds, ex.GetScaleFactors(), np.array(cam6, np.float32),
                                  Tcw[p], dirs[p], xw[s], lo[s], la[s], qd[s], ob[s], 15.0, True)
        got = fm[a:e].copy()
        got[got >= 0] -= qoff[p]
        assert rnm == nm[p] and (got == rfm).all(), p
        assert rnm > 200


def test_refusals_keep_the_handle_working(euroc):
    """A handle of 20 000 features (20 160 rows) and a host F2 of 16 385 features are refused with ORB_ERR_UNSUPPORTED before anything
    is launched; the handle then searches a normal host frame correctly."""
    E = euroc
    w, h = E["w"], E["h"]
    cam = camera(458.0, 457.0, 367.0, 248.0, 0.0, 0.11, w, h)
    bounds = np.array([0, w, 0, h], np.float32)
    kp1, d1, prev = noisy_f1(E["kL"], E["dL"], np.random.default_rng(7))
    big = ORBextractor(20000, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    big.extract_batch(synth.frame(w, h, 303, 1.0, 400)[None], (0, 1000))
    m = ORBmatcher(0.9, True)
    n0 = launches()
    with pytest.raises(N.OrbError, match="orb_status -5"):
        m.SearchForInitialization(big, cam, kp1, d1, prev, 100, target_image=0)
    rep = np.resize(E["k2"], 16385)
    with pytest.raises(N.OrbError, match="orb_status -5"):
        m.SearchForInitialization(big, cam, kp1, d1, prev, 100, kp2=rep, desc2=np.resize(E["d2"], (16385, 32)))
    assert launches() == n0
    g, n = m.SearchForInitialization(big, cam, kp1, d1, prev, 100, kp2=E["k2"], desc2=E["d2"])
    rm, rnm = po.search_initialization(kp1, d1, prev, E["k2"], E["d2"], bounds, 100, 0.9, True)
    assert n == rnm and (g == rm).all() and rnm > 100
    big.close()


def test_tall_stereo_pair_is_refused():
    """k_stereo_match_v1 needs 13 B per right-eye row plus 8 B per image row: 4096x4096 with 16 000 features does not fit a CTA."""
    w = h = 4096
    fx, fy, cx, cy, bf, b = cam_for(w, h)
    L, R, _ = synth.stereo_pair(w, h, seed=9, dmin=2.0, dmax=0.5 * fx)
    ex = ORBextractor(16000, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=2)
    ex.extract_batch(np.stack([L, R]))
    with pytest.raises(N.OrbError, match="orb_status -5"):
        ex.stereo_batch(1, bf, b)
    # the handle keeps working: a 4096x2048 pair (13 B x 16 160 + 8 B x 2048 rows fits) against the oracle
    h2 = 2048
    L2, R2 = np.ascontiguousarray(L[:h2]), np.ascontiguousarray(R[:h2])
    ex.extract_batch(np.stack([L2, R2]))
    ex.stereo_batch(1, bf, b)
    _, _, off, kps, desc = ex.download(2)
    uR, dep = ex.stereo_download(int(off[-1]))
    eL, eR = po.OracleExtractor(16000, 1.2, 8, 20, 7), po.OracleExtractor(16000, 1.2, 8, 20, 7)
    _, kL, dL = eL(L2)
    _, kR, dR = eR(R2)
    ruR, rdep, _ = po.stereo_matches(eL, eR, kL, dL, kR, dR, np.float32(bf), np.float32(b))
    a, e = int(off[0]), int(off[1])
    assert (kps[a:e].view(np.uint8) == kL.view(np.uint8)).all() and (desc[a:e] == dL).all()
    assert (uR[a:e].view(np.uint32) == ruR.view(np.uint32)).all() and (dep[a:e].view(np.uint32) == rdep.view(np.uint32)).all()
    assert (rdep > 0).sum() > 200
    ex.close()


# ---- every search on large frames and keyframes ------------------------------------------------------------------------------
def fsm(n):
    return (n * 23 + 16 + 15) // 16 * 16


def shared_form(n, mode, seq):
    """Does launch_proj (matcher.cu) take the shared-memory form for a frame of n rows?  Each resolve kernel holds 256 B of static
    __shared__ arrays next to its dynamic block."""
    csm = max(fsm(n), (n * 17 + 3073 * 2 + 32 + 15) // 16 * 16)
    psm = fsm(n) + 9 * n + (8192 + 512) * 4 + 64
    rsm = fsm(n) + 1024 * 8 * 8 + 1024 * 4 + n * (9 if mode == 4 else 5) + 1024 * 5 + 256
    return csm <= SMEM_OPTIN and (not seq or psm + RESOLVE_STATIC <= SMEM_OPTIN) and rsm + RESOLVE_STATIC <= SMEM_OPTIN


def last_shared(mode, seq):
    return max(n for n in range(3000, 12000) if shared_form(n, mode, seq))


def launches_for(n, mode):
    """Kernel launches of one search call: k_frame_grid (grid modes), the candidate scan, the parallel resolve (modes 0 / 1), the
    sequential resolve -- and k_stage_frames_xl in the global-memory form."""
    seq = mode in (0, 1)
    return (mode != 2) + 1 + seq + 1 + (0 if shared_form(n, mode, seq) else 1)


def quat_pose(yaw_deg, t):
    a = np.deg2rad(yaw_deg) / 2
    return np.array([0, np.sin(a), 0, np.cos(a), *t], np.float32)


def camera_center(T):
    x, y, z, w = T[:4].astype(np.float64)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return (-R.T @ T[4:].astype(np.float64)).astype(np.float32)


def sim3(q_unit, t, s):
    q = (np.asarray(q_unit, np.float64) * np.sqrt(s)).astype(np.float32)
    sc = np.float32(np.float32(q[0] * q[0] + q[1] * q[1]) + np.float32(q[2] * q[2] + q[3] * q[3]))
    return np.concatenate([q, np.asarray(t, np.float32), [sc]]).astype(np.float32)


def node_of(d, m=97):
    return ((d[:, 0].astype(np.int32) >> 3) * 7 + (d[:, 5].astype(np.int32) >> 4) * 3 + (d[:, 17].astype(np.int32) >> 5)) % m


def kf_queries(S, p, rng, sf, dup):
    """Map points seen by the last frame of pair p (world = that frame), with the MapPoint fields the keyframe searches read."""
    fx, fy, cx, cy = S["cam6"][:4]
    kL, dL, luR, ldep = S["lasts"][p]
    sel = np.nonzero(ldep > 0)[0]
    sel = np.concatenate([sel, rng.choice(sel, int(dup * len(sel)))])
    z = ldep[sel]
    pts = np.stack([(kL["x"][sel] - cx) * z / fx, (kL["y"][sel] - cy) * z / fy, z], 1).astype(np.float32)
    pts += rng.normal(0, 0.002, pts.shape).astype(np.float32)
    dist = np.linalg.norm(pts, axis=1).astype(np.float32)
    nrm = pts / dist[:, None] + rng.normal(0, 0.2, pts.shape).astype(np.float32)
    nrm = (nrm / np.linalg.norm(nrm, axis=1)[:, None]).astype(np.float32)
    maxd = (dist * sf[kL["octave"][sel]]).astype(np.float32)
    return dict(world_pos=pts, normal=nrm, max_dist=maxd, min_dist=(maxd / sf[7]).astype(np.float32), desc=dL[sel],
                angle=kL["angle"][sel].astype(np.float32))


def pose_of(S, p):
    fx, fy = S["cam6"][:2]
    ldep = S["lasts"][p][3]
    zmid = float(np.median(ldep[ldep > 0]))
    return quat_pose(0.0, [(3 + p) * zmid / fx, 1 * zmid / fy, 0.0])


@pytest.fixture(scope="module")
def kitti():
    """KITTI-shaped 1241x376 monocular frames at 10 000 features (10 160 rows): last = oracle features of frame A at a constant depth
    of 10 m, current = A shifted by (3 + p, 1) px on the device."""
    w, h, P, nf = 1241, 376, 2, 10000
    fx, fy, cx, cy = 718.856, 718.856, 607.19, 185.22
    imgs, lasts = np.zeros((P, h, w), np.uint8), []
    for p in range(P):
        a = synth.frame(w, h, 600 + p, 1.0, 300)
        _, kL, dL = po.OracleExtractor(nf, 1.2, 8, 20, 7)(a)
        lasts.append((kL, dL, np.full(len(kL), -1, np.float32), np.full(len(kL), 10.0, np.float32)))
        imgs[p] = np.roll(a, (1, 3 + p), (0, 1))
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=P)
    ex.extract_batch(imgs)
    _, _, off, kps, desc = ex.download(P)
    yield dict(w=w, h=h, P=P, ex=ex, cam6=(fx, fy, cx, cy, 0.0, 0.54), lasts=lasts, off=off, kps=kps, desc=desc,
               uR=np.full(int(off[-1]), -1, np.float32), img_of=lambda p: p)
    ex.close()


def scene(request, name):
    return request.getfixturevalue(name)


def rows_of(S, p):
    i = S["img_of"](p)
    return int(S["off"][i]), int(S["off"][i + 1])


@pytest.mark.parametrize("name", ["kitti", "scene4k16k"])
@pytest.mark.parametrize("masked", [False, True])
def test_search_local_points_large(request, name, masked):
    S = scene(request, name)
    P, ex, (fx, fy, cx, cy, bf, b) = S["P"], S["ex"], S["cam6"]
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(23)
    qoff, parts = [0], []
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        sel = np.concatenate([sel, rng.choice(sel, len(sel) // 2)])
        x = (kL["x"][sel] + 3 + p + rng.normal(0, 1.5, len(sel))).astype(np.float32)
        y = (kL["y"][sel] + 1 + rng.normal(0, 1.5, len(sel))).astype(np.float32)
        xr = (x - np.float32(bf) / ldep[sel]).astype(np.float32) if bf > 0 else np.full(len(sel), -1, np.float32)
        lv = np.clip(kL["octave"][sel] + rng.integers(-1, 2, len(sel)), 0, 7).astype(np.int32)
        parts.append((x, y, xr, lv, rng.uniform(0.99, 1.0, len(sel)).astype(np.float32), dL[sel], (rng.random(len(sel)) < 0.8).astype(np.uint8)))
        qoff.append(qoff[-1] + len(sel))
    px, py, pxr, lv, vc, qd, vis = (np.ascontiguousarray(np.concatenate([pt[i] for pt in parts])) for i in range(7))
    n0 = launches()
    match, nm = ORBmatcher(0.8, True).SearchByProjection(ex, camera(fx, fy, cx, cy, bf, b, S["w"], S["h"]), [S["img_of"](p) for p in range(P)],
                                                         qoff, px, py, pxr, lv, vc, qd, th=3.0, in_view=vis if masked else None)
    assert launches() - n0 == launches_for(10160 if name == "kitti" else 16160, 0)
    for p in range(P):
        a, e = rows_of(S, p)
        s = slice(qoff[p], qoff[p + 1])
        keep = vis[s].astype(bool) if masked else np.ones(qoff[p + 1] - qoff[p], bool)
        idx = np.nonzero(keep)[0] + qoff[p]
        rmatch, rnm = po.search_local(S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], bounds, ex.GetScaleFactors(), px[idx], py[idx], pxr[idx],
                                      lv[idx], vc[idx], qd[idx], 3.0, 0.8)
        assert rnm == nm[p] and (match[idx] == rmatch).all() and (match[s][~keep] == -1).all(), (name, p)
        assert rnm > 200


def test_search_last_frame_kitti(kitti):
    S = kitti
    P, ex, cam6 = S["P"], S["ex"], S["cam6"]
    fx, fy, cx, cy, bf, b = cam6
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(29)
    qoff, xw, lo, la, qd, ob, Tcw = [0], [], [], [], [], [], []
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        z = ldep
        xw.append(np.stack([(kL["x"] - cx) * z / fx, (kL["y"] - cy) * z / fy, z], 1).astype(np.float32))
        Tcw.append(pose_of(S, p))
        lo.append(kL["octave"].astype(np.int32)); la.append(kL["angle"].astype(np.float32)); qd.append(dL)
        ob.append((rng.random(len(kL)) < 0.7).astype(np.uint8))
        qoff.append(qoff[-1] + len(kL))
    xw, lo, la, qd, ob = map(np.concatenate, (xw, lo, la, qd, ob))
    n0 = launches()
    fm, nm = ORBmatcher(0.9, True).SearchByProjectionLastFrame(ex, camera(*cam6, S["w"], S["h"]), list(range(P)), qoff, np.stack(Tcw), [0] * P,
                                                                xw, lo, la, qd, ob, 15.0, int(S["off"][-1]))
    assert launches() - n0 == launches_for(10160, 1)
    for p in range(P):
        a, e = rows_of(S, p)
        s = slice(qoff[p], qoff[p + 1])
        rfm, rnm = po.search_last(S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], bounds, ex.GetScaleFactors(), np.array(cam6, np.float32),
                                  Tcw[p], 0, xw[s], lo[s], la[s], qd[s], ob[s], 15.0, True)
        got = fm[a:e].copy()
        got[got >= 0] -= qoff[p]
        assert rnm == nm[p] and (got == rfm).all(), p
        assert rnm > 200


@pytest.mark.parametrize("name", ["kitti", "scene4k16k"])
def test_search_bow_and_reloc_on_device_frames(request, name):
    """SearchByBoW(KF, F) (mode 2: the frame view without the grid, vocabulary nodes read from global memory) and the relocalisation
    search SearchByProjection(F, KF, set) on frames still on the device."""
    S = scene(request, name)
    P, ex, cam6 = S["P"], S["ex"], S["cam6"]
    rows = 10160 if name == "kitti" else 16160
    total = int(S["off"][-1])
    feat_node = node_of(S["desc"]).astype(np.int32)
    feat_node[::17] = -1
    qoff, qn, qa, qd = [0], [], [], []
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        nd = node_of(dL[sel])
        order = np.lexsort((sel, nd))
        sel, nd = sel[order], nd[order]
        qn.append(nd.astype(np.int32)); qa.append(kL["angle"][sel].astype(np.float32)); qd.append(dL[sel])
        qoff.append(qoff[-1] + len(sel))
    qn, qa, qd = map(np.concatenate, (qn, qa, qd))
    n0 = launches()
    fm, nm = ORBmatcher(0.7, True).SearchByBoW(ex, [S["img_of"](p) for p in range(P)], qoff, qn, qa, qd, feat_node, total)
    assert launches() - n0 == launches_for(rows, 2)
    for p in range(P):
        a, e = rows_of(S, p)
        s = slice(qoff[p], qoff[p + 1])
        rfm, rnm = po.search_bow(S["kps"][a:e], S["desc"][a:e], feat_node[a:e], qn[s], qa[s], qd[s], 0.7, True)
        got = fm[a:e].copy()
        got[got >= 0] -= qoff[p]
        assert rnm == nm[p] and (got == rfm).all(), p
        assert rnm > 20
    rng = np.random.default_rng(31)
    sf, isg, logsf = ex.GetScaleFactors(), ex.GetInverseScaleSigmaSquares(), po.logf(1.2)
    claimed_rows = (rng.random(total) < 0.1).astype(np.uint8)
    targets, queries = [], []
    for p in range(P):
        T = pose_of(S, p)
        targets.append(dict(Tcw=T, Ow=camera_center(T), claimed_rows=claimed_rows))
        queries.append(kf_queries(S, p, rng, sf, dup=0.5))
    n0 = launches()
    got, nm = ORBmatcher(0.9, True).SearchByProjectionReloc(ex, camera(*cam6, S["w"], S["h"]), targets, queries, 10.0, 100,
                                                            target_images=[S["img_of"](p) for p in range(P)])
    assert launches() - n0 == launches_for(rows, 3)
    for p in range(P):
        a, e = rows_of(S, p)
        t, q = targets[p], queries[p]
        rm, rnm, _ = po.search_keyframe(3, S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], np.array([0, S["w"], 0, S["h"]], np.float32), sf, isg,
                                        logsf, np.array(cam6, np.float32), t["Tcw"], t["Ow"], q["world_pos"], None, q["max_dist"], q["min_dist"],
                                        q["desc"], q["angle"], claimed_rows[a:e], 10.0, 100.0)
        assert rnm == nm[p] and (got[p] == rm).all(), p
        assert rnm > 50


def host_keyframe(S, n):
    """n rows of a host keyframe: the 4K frame's rows, repeated past its end (duplicates are features like any other)."""
    a, e = rows_of(S, 0)
    idx = np.resize(np.arange(a, e), n)
    return S["kps"][idx], S["desc"][idx], S["uR"][idx]


KF_SIZES = [5401, last_shared(3, False), last_shared(3, False) + 1, 10000, 16384]


@pytest.mark.parametrize("n", KF_SIZES)
def test_host_keyframes_every_variant(scene4k16k, n):
    """Fuse x2 (variants 0, 1), SearchByProjection(KF, Scw) (2), SearchByProjection(F, KF, set) (3) and SearchBySim3's one-way search
    in both directions (4) on host keyframes of n features; KF_SIZES holds the switch point of the keyframe searches."""
    S = scene4k16k
    ex, cam6 = S["ex"], S["cam6"]
    cam = camera(*cam6, S["w"], S["h"])
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    sf, isg, logsf = ex.GetScaleFactors(), ex.GetInverseScaleSigmaSquares(), po.logf(1.2)
    kp, de, ur = host_keyframe(S, n)
    T = pose_of(S, 0)
    for variant, th, thr in [(0, 3.0, 50.0), (1, 4.0, 50.0), (2, 6.0, 50.0), (3, 10.0, 100.0)]:
        rng = np.random.default_rng(100 + variant)
        cl = (rng.random(n) < 0.2).astype(np.uint8) if variant >= 2 else None
        q = kf_queries(S, 0, rng, sf, dup=1.0 if variant >= 2 else 0.3)
        n0 = launches()
        got, nm = ORBmatcher(0.9, True)._search_keyframe(ex, cam, variant, [dict(kp=kp, desc=de, uright=ur, claimed=cl, Tcw=T, Ow=camera_center(T))],
                                                         [q], th, thr)
        assert launches() - n0 == launches_for(n, 3), (variant, n)
        rm, rnm, _ = po.search_keyframe(variant, kp, de, ur, bounds, sf, isg, logsf, np.array(cam6, np.float32), T, camera_center(T),
                                        q["world_pos"], q["normal"], q["max_dist"], q["min_dist"], q["desc"], q["angle"], cl, th, thr)
        assert rnm == nm[0] and (got[0] == rm).all(), (variant, n, rnm, nm[0])
        assert rnm > (0 if variant == 0 else 20), (variant, rnm)   # Fuse's chi2 gate keeps few of these stereo rows
    # variant 4: KF1's points into KF2 through S21 and, as the second target, back through a Sim3 of another scale
    rng = np.random.default_rng(104)
    q = kf_queries(S, 0, rng, sf, dup=0.0)
    q4 = dict(world_pos=q["world_pos"], max_dist=q["max_dist"], min_dist=q["min_dist"], desc=q["desc"])
    T1, zero = np.array([0, 0, 0, 1, 0, 0, 0], np.float32), np.zeros(3, np.float32)
    Ss = [sim3(T[:4], T[4:], 1.0), sim3(T[:4], T[4:] * 1.01, 1.01)]
    got, nm = ORBmatcher(0.9, True)._search_keyframe(ex, cam, 4, [dict(kp=kp, desc=de, Tcw=T1, Ow=zero, Sim3=s8) for s8 in Ss], [q4, q4],
                                                     7.5, 100.0)
    for t, s8 in enumerate(Ss):
        rm, rnm, _ = po.search_keyframe(4, kp, de, None, bounds, sf, isg, logsf, np.array(cam6, np.float32), T1, zero, q4["world_pos"], None,
                                        q4["max_dist"], q4["min_dist"], q4["desc"], None, None, 7.5, 100.0, sim3=s8)
        assert rnm == nm[t] and (got[t] == rm).all(), (4, t, n)
        assert rnm > 20, (4, t, rnm)


@pytest.mark.parametrize("n", [5401, 10000, 16384])
def test_host_keyframes_bow_and_triangulation(scene4k16k, n):
    """SearchByBoW(KF, KF) and SearchForTriangulation with KF2 of n features (k_tri_match's shared memory is 14 B per KF2 row)."""
    S = scene4k16k
    ex = S["ex"]
    fx, fy, cx, cy, bf, b = S["cam6"]
    rng = np.random.default_rng(37)
    k2, d2, ur2 = host_keyframe(S, n)
    kL, dL, luR, ldep = S["lasts"][0]
    node2 = node_of(d2).astype(np.int32)
    node2[::19] = -1
    valid2 = (rng.random(n) < 0.7).astype(np.uint8)
    sel = np.nonzero(rng.random(len(kL)) < 0.75)[0]
    sel = np.concatenate([sel, sel[::5]])
    nd = node_of(dL[sel])
    order = np.lexsort((sel, nd))
    sel, nd = sel[order], nd[order]
    pair = dict(kp2=k2, desc2=d2, node2=node2, valid2=valid2, query_node=nd.astype(np.int32), query_angle=kL["angle"][sel].astype(np.float32),
                desc1=dL[sel])
    n0 = launches()
    got, nm = ORBmatcher(0.75, True).SearchByBoWKeyFrames(ex, [pair])
    assert launches() - n0 == launches_for(n, 2)
    rm, rnm = po.search_bow_kf(k2, d2, node2, valid2, pair["query_node"], pair["query_angle"], pair["desc1"], 0.75, True)
    assert rnm == nm[0] and (got[0] == rm).all() and rnm > 50, (n, rnm, nm[0])
    sel = np.nonzero(rng.random(len(kL)) < 0.6)[0]
    nd = node_of(dL[sel], 61)
    order = np.lexsort((sel, nd))
    sel, nd = sel[order], nd[order]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    t = np.array([0.03, 0.002, 0.01], np.float32)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]], np.float32)
    F12 = (np.linalg.inv(K.T).astype(np.float32) @ tx @ np.linalg.inv(K).astype(np.float32)).astype(np.float32)
    ep = np.array([cx - 10, cy - 4], np.float32)
    st1, st2 = (luR[sel] >= 0).astype(np.uint8), (ur2 >= 0).astype(np.uint8)
    n2 = node_of(d2, 61).astype(np.int32)
    got, nm = ORBmatcher(0.6, True).SearchForTriangulation(ex, kL[sel], dL[sel], nd, st1, k2, d2, n2, valid2, st2, F12, ep)
    ref, rnm = po.search_triangulation(kL[sel], dL[sel], nd, st1, k2, d2, n2, valid2, st2, F12, ep, ex.GetScaleFactors(), ex.GetScaleSigmaSquares(),
                                       False, True)
    assert rnm == nm and (got == ref).all(), (n, rnm, nm)


def test_bow_vector_16k(scene4k16k):
    """orbv_transform with its BowVector on the 16 000-feature batch: k_bow_vector sorts 8 B x 16 384 in shared memory."""
    from orb_slam3_detailed_comments_b200 import ORBVocabulary, synthetic_vocabulary
    S = scene4k16k
    voc = synthetic_vocabulary(k=10, L=4, seed=41)
    V = ORBVocabulary(voc["child_offset"], voc["child_ids"], voc["node_desc"], voc["node_word"], voc["node_weight"], voc["L"])
    off = S["off"]
    got = V.transform(S["ex"], int(off[-1]), 2 * S["P"], levelsup=4)
    for i in range(2 * S["P"]):
        a, b = int(off[i]), int(off[i + 1])
        r = po.bow_transform(voc, S["desc"][a:b], 4)
        assert (got["word"][a:b] == r["word"]).all() and (got["node"][a:b] == r["node"]).all()
        assert (got["weight"][a:b].view(np.uint64) == r["weight"].view(np.uint64)).all()
        assert (got["bow_word"][i] == r["bow_word"]).all() and (got["bow_weight"][i].view(np.uint64) == r["bow_weight"].view(np.uint64)).all()
    V.close()


def step_queries(S, rng):
    """Host query sets of both per-frame searches on the 4K batch (orbm_last_queries / orbm_local_queries field names)."""
    fx, fy, cx, cy, bf, b = S["cam6"]
    P = S["P"]
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    loc = dict(off=[0], px=[], py=[], pxr=[], lvl=[], vc=[], desc=[])
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        z = ldep[sel]
        last["xw"].append(np.stack([(kL["x"][sel] - cx) * z / fx, (kL["y"][sel] - cy) * z / fy, z], 1).astype(np.float32))
        last["oct"].append(kL["octave"][sel].astype(np.int32)); last["ang"].append(kL["angle"][sel].astype(np.float32)); last["desc"].append(dL[sel])
        last["obs"].append((rng.random(len(sel)) < 0.8).astype(np.uint8)); last["off"].append(last["off"][-1] + len(sel))
        x = (kL["x"][sel] + 3 + p + rng.normal(0, 1.5, len(sel))).astype(np.float32)
        y = (kL["y"][sel] + 1 + rng.normal(0, 1.5, len(sel))).astype(np.float32)
        loc["px"].append(x); loc["py"].append(y); loc["pxr"].append((x - np.float32(bf) / z).astype(np.float32))
        loc["lvl"].append(kL["octave"][sel].astype(np.int32)); loc["vc"].append(rng.uniform(0.99, 1, len(sel)).astype(np.float32))
        loc["desc"].append(dL[sel]); loc["off"].append(loc["off"][-1] + len(sel))
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    fimg = np.arange(0, 2 * P, 2, dtype=np.int32)
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=np.stack([pose_of(S, p) for p in range(P)]), dir=np.zeros(P, np.int32),
              xw=cat(last["xw"], np.float32), oct=cat(last["oct"], np.int32), ang=cat(last["ang"], np.float32), desc=cat(last["desc"], np.uint8),
              obs=cat(last["obs"], np.uint8))
    hc = dict(fimg=fimg, off=np.array(loc["off"], np.int32), px=cat(loc["px"], np.float32), py=cat(loc["py"], np.float32),
              pxr=cat(loc["pxr"], np.float32), lvl=cat(loc["lvl"], np.int32), vc=cat(loc["vc"], np.float32), desc=cat(loc["desc"], np.uint8))
    return hl, hc


def test_replay_step_and_graph_16k(scene4k16k):
    """The tracking step through orbr_submit / orbr_collect on a second 16 000-feature handle equals the per-call path; both searches
    captured in a CUDA graph (after one bounded eager call, which sizes the global form's frame blocks) replay to the same bits."""
    import torch
    from orb_slam3_detailed_comments_b200 import replay
    from orb_slam3_detailed_comments_b200._native import KP_DTYPE
    S = scene4k16k
    ex, P, cam6 = S["ex"], S["P"], S["cam6"]
    fx, fy, cx, cy, bf, b = cam6
    cam = camera(*cam6, S["w"], S["h"])
    hl, hc = step_queries(S, np.random.default_rng(43))
    rows = int(S["off"][-1])
    m_last, m_loc = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
    fm, nm1 = m_last.SearchByProjectionLastFrame(ex, cam, hl["fimg"], hl["off"], hl["Tcw"], hl["dir"], hl["xw"], hl["oct"], hl["ang"], hl["desc"],
                                                 hl["obs"], 15.0, rows)
    mt, nm2 = m_loc.SearchByProjection(ex, cam, hc["fimg"], hc["off"], hc["px"], hc["py"], hc["pxr"], hc["lvl"], hc["vc"], hc["desc"], th=3.0)
    assert nm1.min() > 200 and nm2.min() > 200
    # the replay step on its own handle
    rc, nq = 2 * P * 16160, int(hc["off"][-1])
    z = lambda shape, dt: np.zeros(shape, dt)
    out = dict(kps=z(rc, KP_DTYPE), desc=z((rc, 32), np.uint8), ur=z(rc, np.float32), dep=z(rc, np.float32), n=z(2 * P, np.int32),
               offsets=z(2 * P + 1, np.int32), fm=z(rc, np.int32), nm1=z(P, np.int32), mt=z(nq, np.int32), nm2=z(P, np.int32))
    ex2 = ORBextractor(16000, 1.2, 8, 20, 7, max_width=S["w"], max_height=S["h"], max_batch=2 * P)
    st = replay.TrackingStep(ex2, cam, bf, b, 15.0, 3.0, 0.8, True)
    st.submit(np.ascontiguousarray(S["imgs"]), last=hl, local=hc)
    assert st.collect(out) == rows and (out["offsets"] == S["off"]).all()
    assert (out["fm"][:rows] == fm).all() and (out["nm1"] == nm1).all() and (out["mt"] == mt).all() and (out["nm2"] == nm2).all()
    ex2.close()
    # a captured graph of both device-pointer searches
    dev = torch.device("cuda", 0)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dl, dc = {k: T(v) for k, v in hl.items()}, {k: T(v) for k, v in hc.items()}
    o = (torch.full((rows,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev),
         torch.full((nq,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev))

    def step():
        m_last.SearchByProjectionLastFrameDevice(ex, cam, P, dl["fimg"], dl["off"], dl["Tcw"], dl["dir"], dl["xw"], dl["oct"], dl["ang"],
                                                 dl["desc"], dl["obs"], 15.0, o[0], o[1])
        m_loc.SearchByProjectionDevice(ex, cam, P, dc["fimg"], dc["off"], dc["px"], dc["py"], dc["pxr"], dc["lvl"], dc["vc"], dc["desc"], o[2], o[3],
                                       th=3.0)

    ex.set_device_query_bounds(max(int(hl["off"][-1]), nq), max(np.diff(hl["off"]).max(), np.diff(hc["off"]).max()), rows)
    step()
    torch.cuda.synchronize()
    want = [t.cpu().numpy().copy() for t in o]
    assert (want[0] == fm).all() and (want[1] == nm1).all() and (want[2] == mt).all() and (want[3] == nm2).all()
    g = ex.graph_capture(step)
    assert ex.graph_kernels(g) == launches_for(16160, 0) + launches_for(16160, 1)
    for t in o:
        t.fill_(-7)
    ex.graph_launch(g)
    torch.cuda.synchronize()
    for t, w in zip(o, want):
        assert (t.cpu().numpy() == w).all()
    ex.graph_destroy(g)
    ex.set_device_query_bounds(0, 0, 0)


def test_per_frame_switch_point():
    """Device frames of the last row capacity the shared-memory form of SearchByProjection(F, local map) takes, and one row more:
    both match the oracle, the second one runs the global form (one launch more)."""
    w, h = 752, 480
    cam = camera(458.0, 457.0, 367.0, 248.0, 40.0, 0.11, w, h)
    bounds = np.array([0, w, 0, h], np.float32)
    img = synth.frame(w, h, 305, 1.0, 400)
    rng = np.random.default_rng(47)
    for rows in (last_shared(0, True), last_shared(0, True) + 1):
        ex = ORBextractor(rows - 160, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
        ex.extract_batch(img[None])
        _, _, off, k, d = ex.download(1)
        n = len(k)
        x = (k["x"] + rng.normal(0, 1.5, n)).astype(np.float32)
        y = (k["y"] + rng.normal(0, 1.5, n)).astype(np.float32)
        lv, vc = k["octave"].astype(np.int32), rng.uniform(0.99, 1, n).astype(np.float32)
        xr = np.full(n, -1, np.float32)
        n0 = launches()
        match, nm = ORBmatcher(0.8, True).SearchByProjection(ex, cam, [0], [0, n], x, y, xr, lv, vc, d, th=3.0)
        assert launches() - n0 == launches_for(rows, 0), rows
        rmatch, rnm = po.search_local(k, d, np.full(n, -1, np.float32), bounds, ex.GetScaleFactors(), x, y, xr, lv, vc, d, 3.0, 0.8)
        assert rnm == nm[0] and (match == rmatch).all() and rnm > 500, rows
        ex.close()
    assert shared_form(last_shared(0, True), 0, True) and not shared_form(last_shared(0, True) + 1, 0, True)


def test_every_search_refuses_an_oversized_handle(euroc):
    """A handle of 20 000 features (20 160 rows): every search on its frames, and orbv_transform's BowVector, are refused before
    anything is launched."""
    w, h = euroc["w"], euroc["h"]
    cam = camera(458.0, 457.0, 367.0, 248.0, 40.0, 0.11, w, h)
    big = ORBextractor(20000, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    big.extract_batch(synth.frame(w, h, 303, 1.0, 400)[None])
    _, _, off, k, d = big.download(1)
    n = len(k)
    m = ORBmatcher(0.9, True)
    f32 = lambda v: np.full(n, v, np.float32)
    calls = [
        lambda: m.SearchByProjection(big, cam, [0], [0, n], k["x"].copy(), k["y"].copy(), f32(-1), k["octave"].astype(np.int32), f32(1), d, th=3.0),
        lambda: m.SearchByProjectionLastFrame(big, cam, [0], [0, n], np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32), [0],
                                              np.ones((n, 3), np.float32), k["octave"].astype(np.int32), f32(0), d, np.ones(n, np.uint8), 15.0, n),
        lambda: m.SearchByBoW(big, [0], [0, n], np.zeros(n, np.int32), f32(0), d, np.zeros(n, np.int32), n),
        lambda: m.SearchByProjectionReloc(big, cam, [dict(Tcw=np.array([0, 0, 0, 1, 0, 0, 0], np.float32), Ow=np.zeros(3, np.float32))],
                                          [dict(world_pos=np.ones((n, 3), np.float32), max_dist=f32(10), min_dist=f32(1), desc=d, angle=f32(0))],
                                          10.0, 100, target_images=[0]),
    ]
    n0 = launches()
    for call in calls:
        with pytest.raises(N.OrbError, match="orb_status -5"):
            call()
    from orb_slam3_detailed_comments_b200 import ORBVocabulary, synthetic_vocabulary
    voc = synthetic_vocabulary(k=10, L=3, seed=7)
    V = ORBVocabulary(voc["child_offset"], voc["child_ids"], voc["node_desc"], voc["node_word"], voc["node_weight"], voc["L"])
    with pytest.raises(N.OrbError, match="orb_status -5"):
        V.transform(big, n, 1, levelsup=2)
    assert launches() == n0
    V.close()
    big.close()
