"""GPU tier: frames up to 4096 px a side (1080p, 2K stereo heads, 1440p, 4K UHD and DCI 4K) against the oracle, bit for bit: keypoint
records, descriptors and their order (batch and single image, stereo and monocular lapping areas), levels on the 64-bit quadtree form
(k_quadtree_v1_k64, regions over 2048 px) next to levels on the 32-bit one, mvuRight / mvDepth, the two per-frame SearchByProjection
overloads on a 4K stereo batch, a captured and replayed 4K step, the refusal above 4128 px, and the drop-in ORB_SLAM3::ORBextractor
growing its handle from its default size."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth
from orb_slam3_detailed_comments_b200 import _native as N

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1920, 1080), (2208, 1242), (2560, 1440), (3840, 2160), (4096, 2160)]


def cam_for(w, h):
    """The benchmark's 640x480 camera scaled to the image: fx grows with the width, so the disparity range is ~fx px at 4K."""
    s = w / 640.0
    return 435.2 * s, 435.2 * s, w / 2.0, h / 2.0, 47.9 * s, 0.11


def check_rows(kps, desc, rk, rd, what):
    assert len(kps) == len(rk), (what, len(kps), len(rk))
    assert (kps.view(np.uint8) == rk.view(np.uint8)).all() and (desc == rd).all(), what


@pytest.mark.parametrize("w,h", SIZES)
def test_batch_and_single_image_bit_exact(w, h):
    nf = 2000 if w < 3000 else 5000
    imgs = np.stack([synth.frame(w, h, 40 + i, 1.0 + i, 200) for i in range(2)] + [np.random.default_rng(w).integers(0, 256, (h, w), dtype=np.uint8)])
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=3)
    ref = po.OracleExtractor(nf, 1.2, 8, 20, 7)
    ex.extract_batch(imgs)
    n, mono, off, kps, desc = ex.download(3)
    for i in range(3):
        rmono, rk, rd = ref(imgs[i])
        assert mono[i] == rmono
        check_rows(kps[off[i]:off[i + 1]], desc[off[i]:off[i + 1]], rk, rd, (w, h, i))
    for lap in [(0, 0), (0, 1000)]:                        # stereo {0,0} and mono {0,1000} lapping areas, one image at a time
        mono1, k1, d1 = ex(imgs[0], lap)
        rmono, rk, rd = ref(imgs[0], lap)
        assert mono1 == rmono
        check_rows(k1, d1, rk, rd, (w, h, lap))
    ex.close()


def test_levels_on_both_quadtree_forms():
    """2208x1242: level 0 (region 2176 px) sorts 64-bit elements, levels 1-7 the 32-bit ones; every level's DistributeOctTree output
    against the oracle, on a corner-rich frame whose level-0 candidates overflow the shared-memory sort into the global scratch."""
    w, h = 2208, 1242
    img = np.random.default_rng(5).integers(0, 256, (h, w), dtype=np.uint8)
    ex = ORBextractor(2000, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=1)
    ref = po.OracleExtractor(2000, 1.2, 8, 20, 7)
    mono, kps, desc = ex(img)
    rmono, rk, rd = ref(img)
    assert (ex.level_size(0)[0] - 32 > 2048) and (ex.level_size(1)[0] - 32 <= 2048)
    assert len(ex.candidates(0, 0)) > 16384
    for l in range(8):
        k, rl = ex.level_keypoints(0, l), ref.level_kps(l)
        rl3 = np.stack([rl["x"], rl["y"], rl["response"]], 1).astype(np.int32)
        assert k.shape == rl3.shape and (k == rl3).all(), l
    assert mono == rmono
    check_rows(kps, desc, rk, rd, "2208x1242")
    ex.close()


def stereo_batch(w, h, P, seed):
    fx, fy, cx, cy, bf, b = cam_for(w, h)
    imgs = np.zeros((2 * P, h, w), np.uint8)
    for p in range(P):
        imgs[2 * p], imgs[2 * p + 1], _ = synth.stereo_pair(w, h, seed=seed + p, dmin=2.0, dmax=0.5 * fx)
    return imgs, (fx, fy, cx, cy, bf, b)


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)])
def test_stereo_bit_exact(w, h):
    P, nf = 2, 2000
    imgs, (fx, fy, cx, cy, bf, b) = stereo_batch(w, h, P, 70)
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=2 * P)
    ex.extract_batch(imgs)
    ex.stereo_batch(P, bf, b)
    _, _, off, kps, desc = ex.download(2 * P)
    uR, dep = ex.stereo_download(int(off[-1]))
    matched = 0
    for p in range(P):
        eL, eR = po.OracleExtractor(nf, 1.2, 8, 20, 7), po.OracleExtractor(nf, 1.2, 8, 20, 7)
        _, kL, dL = eL(imgs[2 * p])
        _, kR, dR = eR(imgs[2 * p + 1])
        ruR, rdep, _ = po.stereo_matches(eL, eR, kL, dL, kR, dR, np.float32(bf), np.float32(b))
        a, e = off[2 * p], off[2 * p + 1]
        assert (uR[a:e].view(np.uint32) == ruR.view(np.uint32)).all() and (dep[a:e].view(np.uint32) == rdep.view(np.uint32)).all(), p
        matched += int((rdep > 0).sum())
    assert matched > 200
    ex.close()


@pytest.fixture(scope="module")
def scene4k():
    w, h, P, nf = 3840, 2160, 2, 2000
    imgs, cam6 = stereo_batch(w, h, P, 90)
    fx, fy, cx, cy, bf, b = cam6
    lasts = []
    for p in range(P):                                      # the last frames: the same pairs before a shift of (3 + p, 1) px
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
    yield dict(w=w, h=h, P=P, ex=ex, imgs=imgs, cam6=cam6, lasts=lasts, off=off, kps=kps, desc=desc, uR=uR, dep=dep)
    ex.close()


def test_search_local_points_4k(scene4k):
    S = scene4k
    P, ex, off, (fx, fy, cx, cy, bf, b) = S["P"], S["ex"], S["off"], S["cam6"]
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(7)
    qoff, px, py, pxr, lv, vc, qd = [0], [], [], [], [], [], []
    claimed = np.zeros(int(off[-1]), np.uint8)
    for p in range(P):
        kL, dL, luR, ldep = S["lasts"][p]
        sel = np.nonzero(ldep > 0)[0]
        sel = np.concatenate([sel, rng.choice(sel, 3 * len(sel))])
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
    match, nm = ORBmatcher(0.8, True).SearchByProjection(ex, camera(fx, fy, cx, cy, bf, b, S["w"], S["h"]), [2 * p for p in range(P)], qoff,
                                                         px, py, pxr, lv, vc, qd, th=3.0, feature_claimed=claimed)
    for p in range(P):
        a, e = off[2 * p], off[2 * p + 1]
        s = slice(qoff[p], qoff[p + 1])
        rmatch, rnm = po.search_local(S["kps"][a:e], S["desc"][a:e], S["uR"][a:e], bounds, ex.GetScaleFactors(), px[s], py[s], pxr[s],
                                      lv[s], vc[s], qd[s], 3.0, 0.8, claimed=claimed[a:e])
        assert rnm == nm[p] and (match[s] == rmatch).all(), p
        assert rnm > 50


def test_search_last_frame_4k(scene4k):
    S = scene4k
    P, ex, off, cam6 = S["P"], S["ex"], S["off"], S["cam6"]
    fx, fy, cx, cy, bf, b = cam6
    bounds = np.array([0, S["w"], 0, S["h"]], np.float32)
    rng = np.random.default_rng(11)
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
        assert rnm > 50


def test_graph_replay_4k(scene4k):
    """The 4K extraction + stereo step captured once and replayed gives the eager step's bits."""
    import torch
    S = scene4k
    ex, P = S["ex"], S["P"]
    fx, fy, cx, cy, bf, b = S["cam6"]
    d_imgs = torch.from_numpy(S["imgs"]).cuda()
    torch.cuda.synchronize()

    def step():
        ex.extract_batch_device(d_imgs.data_ptr(), 2 * P, S["w"], S["h"])
        ex.stereo_batch(P, bf, b)

    step()
    g = ex.graph_capture(step)
    ex.graph_launch(g)
    _, _, off, kps, desc = ex.download(2 * P)
    uR, dep = ex.stereo_download(int(off[-1]))
    ex.graph_destroy(g)
    assert (off == S["off"]).all() and (kps.view(np.uint8) == S["kps"].view(np.uint8)).all() and (desc == S["desc"]).all()
    assert (uR.view(np.uint32) == S["uR"].view(np.uint32)).all() and (dep.view(np.uint32) == S["dep"].view(np.uint32)).all()


def test_refusal_above_4128_px_keeps_the_handle():
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=4096, max_height=2160, max_batch=1)
    with pytest.raises(N.OrbError, match="orb_status -5"):
        ex(np.zeros((2160, 4129), np.uint8))
    img = synth.frame(4096, 2160, 3)
    mono, kps, desc = ex(img)
    rmono, rk, rd = po.OracleExtractor(1200, 1.2, 8, 20, 7)(img)
    assert mono == rmono
    check_rows(kps, desc, rk, rd, "after refusal")
    ex.close()
    with pytest.raises(N.OrbError, match="orb_status -5"):      # a handle sized above the limit is refused at creation
        ORBextractor(1200, 1.2, 8, 20, 7, max_width=4129, max_height=2160, max_batch=1)


def test_qt_variant_0_refuses_regions_over_2048_px(monkeypatch):
    monkeypatch.setenv("ORB_QT_VARIANT", "0")
    with pytest.raises(N.OrbError, match="orb_status -5"):
        ORBextractor(1200, 1.2, 8, 20, 7, max_width=2208, max_height=1242, max_batch=1)
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=1920, max_height=1080, max_batch=1)     # 1080p stays on the 32-bit form
    img = synth.frame(1920, 1080, 8)
    mono, kps, desc = ex(img)
    rmono, rk, rd = po.OracleExtractor(1200, 1.2, 8, 20, 7)(img)
    check_rows(kps, desc, rk, rd, "variant 0 at 1080p")
    ex.close()


def test_drop_in_extractor_grows_from_its_default_size(tmp_path):
    """ORB_SLAM3::ORBextractor (host/ORBextractor_b200.cc) created at its default 1280x1024 extracts a 1080p and then a 4K stereo pair;
    Frame::ComputeStereoMatches (host/Frame_stereo_b200.cc) runs on each pair."""
    H_ = os.path.join(ROOT, "orb_slam3_detailed_comments_b200", "host")
    ref_root = os.environ.get("ORB_REFERENCE_ROOT", "/root/reference")
    decl = ["-I", os.path.join(ref_root, "include"), "-I", ref_root] if os.path.exists(os.path.join(ref_root, "include", "ORBmatcher.h")) \
        else ["-I", os.path.join(ROOT, "tests", "host", "refdecl")]
    exe = str(tmp_path / "extractor_grow")
    lib = os.path.dirname(N.LIB_PATH)
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-include", os.path.join(H_, "refshim", "ref_skeleton.h"), "-I", os.path.join(H_, "refshim")]
                          + decl + ["-I", os.path.join(ROOT, "include"), "-I", H_, os.path.join(ROOT, "tests", "host", "extractor_grow.cc"),
                                    os.path.join(H_, "ORBextractor_b200.cc"), os.path.join(H_, "Frame_stereo_b200.cc"), "-L", lib,
                                    "-lorbslam3_b200", "-Wl,-rpath," + lib, "-lpthread", "-o", exe])
    d = str(tmp_path)
    nf = 2000
    sizes = [(1920, 1080), (3840, 2160)]
    cams, pairs = [], []
    for k, (w, h) in enumerate(sizes):
        l, r, _ = synth.stereo_pair(w, h, seed=300 + k, dmin=2.0, dmax=0.5 * cam_for(w, h)[0])
        l.tofile(os.path.join(d, f"left{k}.u8")); r.tofile(os.path.join(d, f"right{k}.u8"))
        pairs.append((l, r)); cams.append(cam_for(w, h))
    fx, fy, cx, cy, bf, b = cams[-1]
    meta = dict(n=2, nfeatures=nf, fx=fx, fy=fy, cx=cx, cy=cy, bf=bf, b=b, W0=1920, H0=1080, W1=3840, H1=2160)
    # one camera for both frames: Frame's static intrinsics are set per frame from these
    with open(os.path.join(d, "meta.txt"), "w") as f:
        for k, v in meta.items():
            f.write(f"{k} {float(v)!r}\n")
    r = subprocess.run([exe, d], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for k, (l, rimg) in enumerate(pairs):
        eL, eR = po.OracleExtractor(nf, 1.2, 8, 20, 7), po.OracleExtractor(nf, 1.2, 8, 20, 7)
        monoL, kL, dL = eL(l)
        monoR, kR, dR = eR(rimg)
        kps = np.fromfile(os.path.join(d, f"out_kpsL{k}.bin"), po.KP_DTYPE)
        check_rows(kps, np.fromfile(os.path.join(d, f"out_descL{k}.bin"), np.uint8).reshape(-1, 32), kL, dL, ("drop-in", k))
        assert (np.fromfile(os.path.join(d, f"out_kpsR{k}.bin"), po.KP_DTYPE).view(np.uint8) == kR.view(np.uint8)).all()
        assert list(np.fromfile(os.path.join(d, f"out_mono{k}.i32"), np.int32)) == [monoL, monoR]
        uR, dep, _ = po.stereo_matches(eL, eR, kL, dL, kR, dR, np.float32(bf), np.float32(b))
        assert (np.fromfile(os.path.join(d, f"out_uright{k}.f32"), np.float32).view(np.uint32) == uR.view(np.uint32)).all(), k
        assert (np.fromfile(os.path.join(d, f"out_depth{k}.f32"), np.float32).view(np.uint32) == dep.view(np.uint32)).all(), k
        assert (dep > 0).sum() > 100
