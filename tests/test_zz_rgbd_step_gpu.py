"""GPU tier: RGB-D frames on the device -- orbm_stereo_rgbd_batch (Frame::ComputeStereoFromRGBD with Tracking::GrabImageRGBD's depth
conversion, k_stereo_rgbd) and the RGB-D replay step (orbr_step::depth_maps).

- per call, mvuRight / mvDepth equal the oracle in float bits on every row: u16 and f32 maps, host and device memory, odd strides;
- the RGB-D step on two handles kept in flight equals the blocking per-call sequence, and its first frames equal the oracle fed the same
  depth-derived mvuRight: keypoints, descriptors, uright / depth, both match arrays and both PoseOptimization results, at 640x480 (TUM
  fr3) and 1280x720 (D435i), forward and backward, RGB and grey input.  Some queries are rejected by the stereo gates only, so the
  answer differs from the oracle's with mvuRight = -1: the gates are live;
- the chained flow in RGB-D mode matches the oracle stage by stage;
- a CUDA-graph replay of the device-resident step equals the eager calls;
- every refusal leaves the handle usable; stereo, monocular and RGB-D steps alternating on one handle, with and without PoseOptimization,
  leak no state;
- orbx_pack_keyframe_device carries the depth-derived uright of an RGB-D frame."""
import numpy as np
import pytest
import torch

from _tracking import check_against_per_call, run_chained_flow, run_step, same_results, step_outputs
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth, replay
from orb_slam3_detailed_comments_b200._native import OrbError
from oracle import pyingest
from oracle import pyoracle as po
from oracle import pyrgbd

pytestmark = pytest.mark.gpu
f32 = np.float32
TH_LAST, TH_LOC = 15.0, 3.0             # Tracking.cc for an RGB-D sensor: motion model th = 15, SearchLocalPoints th = 3
FACTOR = f32(1.0 / 5000)                # Tracking::mDepthMapFactor of the TUM sequences (DepthMapFactor 5000)
ORB_ERR_INVALID, ORB_ERR_UNSUPPORTED = -1, -5
# (W, H, n_features, fx, fy, cx, cy, bf)
GEOM = {"tum_640x480": (640, 480, 1000, 535.4, 539.2, 320.1, 247.6, 40.0),
        "d435i_1280x720": (1280, 720, 2000, 908.0, 908.0, 640.0, 360.0, 45.4)}


def _frames(W, H, bf, seeds, rgb=False):
    """camera images (grey, or RGB whose grey conversion is near the grey image) and u16 depth maps from synthetic disparity fields:
    z = bf / disparity in raw units of 1/5000 m, clipped to the u16 range, with 3 % holes"""
    imgs, maps = [], []
    for s in seeds:
        left, _, disp = synth.stereo_pair(W, H, seed=s)
        rng = np.random.default_rng(s)
        raw = np.clip(np.rint(f32(bf) / disp / FACTOR), 0, 65535).astype(np.uint16)
        raw[rng.random(raw.shape) < 0.03] = 0
        maps.append(raw)
        if rgb:
            d = rng.integers(-3, 4, left.shape)
            left = np.stack([np.clip(left.astype(int) + d, 0, 255), left, np.clip(left.astype(int) - d, 0, 255)], -1).astype(np.uint8)
        imgs.append(left)
    return np.ascontiguousarray(np.stack(imgs)), np.ascontiguousarray(np.stack(maps))


def _grey(imgs):
    return np.stack([pyingest.ingest(im, "rgb") for im in imgs]) if imgs.ndim == 4 else imgs


def _mk(W, H, nf, max_batch):
    return ORBextractor(nf, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=max_batch)


def _queries(kps, desc, off, dep, g, rng, direction):
    """Query sets from each frame's own features at their depth-map depth (host arrays); frame f = image f.  A quarter of the local-map
    queries predict a right coordinate 12 px off and a quarter of the LastFrame points sit at 10x their depth along the same ray: the
    monocular tests pass them, the stereo gates of a feature with mvuRight > 0 reject most of them."""
    W, H, NF, FX, FY, CX, CY, BF = g
    P = len(off) - 1
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    loc = dict(off=[0], px=[], py=[], pxr=[], lvl=[], vc=[], desc=[], xw=[], td=[])
    for p in range(P):
        a, b = int(off[p]), int(off[p + 1])
        k, d, z = kps[a:b], desc[a:b], np.where(dep[a:b] > 0, dep[a:b], f32(3.0)).astype(f32)
        sel = np.arange(0, len(k), 2)
        zs = z[sel] * np.where(rng.random(len(sel)) < 0.25, f32(10.0), f32(1.0)).astype(f32)
        pts = np.stack([(k["x"][sel] - f32(CX)) * zs / f32(FX), (k["y"][sel] - f32(CY)) * zs / f32(FY), zs], 1).astype(f32)
        last["xw"].append(pts); last["oct"].append(k["octave"][sel].astype(np.int32)); last["ang"].append(k["angle"][sel].astype(f32))
        last["desc"].append(d[sel]); last["obs"].append((rng.random(len(sel)) < 0.9).astype(np.uint8)); last["off"].append(last["off"][-1] + len(sel))
        m = len(k)
        x = (k["x"] + rng.normal(0, 1.0, m)).astype(f32); y = (k["y"] + rng.normal(0, 1.0, m)).astype(f32)
        xr = (x - f32(BF) / z + np.where(rng.random(m) < 0.25, f32(12.0), f32(0.0))).astype(f32)
        loc["px"].append(x); loc["py"].append(y); loc["pxr"].append(xr); loc["lvl"].append(k["octave"].astype(np.int32))
        loc["vc"].append(rng.uniform(0.999, 1, m).astype(f32)); loc["desc"].append(d); loc["td"].append(z)
        loc["xw"].append(np.stack([(k["x"] - f32(CX)) * z / f32(FX), (k["y"] - f32(CY)) * z / f32(FY), z], 1).astype(f32)); loc["off"].append(loc["off"][-1] + m)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    fimg = np.arange(P, dtype=np.int32)
    tz = {0: 0.0, 1: -0.06, 2: 0.06}[direction]          # the camera moved along its axis by more than mb = bf / fx: bForward / bBackward
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=np.tile(np.array([0, 0, 0, 1, 0.002, 0.001, tz], f32), (P, 1)),
              dir=np.full(P, direction, np.int32), xw=cat(last["xw"], f32), oct=cat(last["oct"], np.int32), ang=cat(last["ang"], f32),
              desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(fimg=fimg, off=np.array(loc["off"], np.int32), px=cat(loc["px"], f32), py=cat(loc["py"], f32), pxr=cat(loc["pxr"], f32),
              lvl=cat(loc["lvl"], np.int32), vc=cat(loc["vc"], f32), desc=cat(loc["desc"], np.uint8), xw=cat(loc["xw"], f32), td=cat(loc["td"], f32))
    return hl, hc


def _per_call(ex, imgs, maps, bf):
    """the blocking per-call sequence of an RGB-D batch: extraction with lapping (0, 0), then orbm_stereo_rgbd_batch"""
    P = len(maps)
    ex.extract_batch(imgs, lapping=(0, 0))
    n, mono, off, kps, desc = ex.download(P)
    ex.stereo_rgbd_batch(maps, FACTOR, bf)
    uR, dep = ex.stereo_download(int(off[-1]))
    return n, off, kps, desc, uR.copy(), dep.copy()


def _bits(a, b):
    return a.shape == b.shape and (np.ascontiguousarray(a).view(np.uint32) == np.ascontiguousarray(b).view(np.uint32)).all()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["u16", "f32"])
@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("pad", [0, 3])
def test_per_call_matches_the_oracle(fmt, where, pad):
    W, H, NF, FX, FY, CX, CY, BF = GEOM["tum_640x480"]
    imgs, raw = _frames(W, H, BF, [2100, 2101, 2102])
    ex = _mk(W, H, NF, 3)
    ex.extract_batch(imgs, lapping=(0, 0))
    n, _, off, kps, _ = ex.download(3)
    # an f32 map is what GrabImageRGBD leaves: raw * factor, converted already, passed with factor 1
    maps, factor = (raw, FACTOR) if fmt == "u16" else ((raw.astype(f32) * FACTOR).astype(f32), f32(1.0))
    buf = np.zeros((3, H, W + pad), maps.dtype)                    # rows `pad` elements longer than a row: an odd byte stride
    buf[:, :, :W] = maps
    view = buf[:, :, :W]
    arg = view if where == "host" else torch.from_numpy(buf).cuda()[:, :, :W]
    ex.stereo_rgbd_batch(arg, factor, BF)
    uR, dep = ex.stereo_download(int(off[-1]))
    for p in range(3):
        a, b = int(off[p]), int(off[p + 1])
        wu, wd = pyrgbd.stereo_from_rgbd(kps[a:b], view[p], factor, BF)
        assert _bits(uR[a:b], wu) and _bits(dep[a:b], wd), p
        assert (wd > 0).sum() > 0.9 * (b - a) and (wd == -1).sum() > 5          # the holes stay -1
    ex.close()


# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", list(GEOM))
@pytest.mark.parametrize("direction", [1, 2])
@pytest.mark.parametrize("rgb", [False, True])
def test_rgbd_step_equals_blocking_calls_and_the_oracle(geom, direction, rgb):
    g = GEOM[geom]
    W, H, NF, FX, FY, CX, CY, BF = g
    P = 3
    rng = np.random.default_rng(31 + direction)
    cam = camera(FX, FY, CX, CY, BF, BF / FX, W, H)
    batches = [_frames(W, H, BF, [2200 + 10 * s + p for p in range(P)], rgb) for s in range(3)]
    ref = _mk(W, H, NF, P)
    exs = [_mk(W, H, NF, P) for _ in range(2)]
    qs = []
    for imgs, maps in batches:
        n, off, kps, desc, uR, dep = _per_call(ref, _grey(imgs), maps, BF)
        qs.append(_queries(kps, desc, off, dep, g, rng, direction))
    rc = P * ref.max_features_per_image()
    fmt = "rgb" if rgb else "gray"
    steps = [replay.TrackingStep(e, cam, BF, BF / FX, TH_LAST, TH_LOC, 0.8, True, image_format=fmt, rgbd=True, depth_factor=FACTOR) for e in exs]
    outs = [step_outputs(P, P, rc, max(int(q[1]["off"][-1]) for q in qs)) for _ in exs]

    def submit(i):
        hl, hc = qs[i]
        steps[i % 2].submit(batches[i][0], last=hl, local=hc, pose=hl["Tcw"], local_world_pos=hc["xw"], depth=batches[i][1])

    cam5 = [FX, FY, CX, CY, BF]
    submit(0)
    for i in range(3):                       # one host thread, two handles in flight: submit i + 1 before collecting i
        if i + 1 < 3:
            submit(i + 1)
        o = outs[i % 2]
        o["ur"][:] = 7.0; o["dep"][:] = 7.0
        rows = steps[i % 2].collect(o)
        hl, hc = qs[i]
        # the blocking per-call ABI on a third handle, fed the oracle's grey images
        n, off, kps, desc, uR, dep = _per_call(ref, _grey(batches[i][0]), batches[i][1], BF)
        assert rows == int(off[-1]) and (o["n"] == n).all() and (o["offsets"] == off).all() and n.min() > 0.8 * NF
        assert (o["kps"][:rows].view(np.uint8) == kps.view(np.uint8)).all() and (o["desc"][:rows] == desc).all()
        assert _bits(o["ur"][:rows], uR) and _bits(o["dep"][:rows], dep) and (dep > 0).sum() > 0.8 * rows
        nm1, nm2, inl = check_against_per_call(o, rows, ref, cam, hl, hc, TH_LAST, TH_LOC, cam5, True)
        assert nm1.min() > 50 and nm2.min() > 100 and inl.min() > 30
    # the first frame of the last batch against the CPU oracle, fed the same depth-derived mvuRight
    o, off = outs[0], outs[0]["offsets"]          # batch 2 ran on handle 0
    hl, hc = qs[2]
    imgs, maps = batches[2]
    a, b = int(off[0]), int(off[1])
    rmono, rk, rd = po.OracleExtractor(NF, 1.2, 8, 20, 7)(_grey(imgs)[0], (0, 0))
    assert (o["kps"][a:b].view(np.uint8) == rk.view(np.uint8)).all() and (o["desc"][a:b] == rd).all()
    wu, wd = pyrgbd.stereo_from_rgbd(rk, maps[0], FACTOR, BF)
    assert _bits(o["ur"][a:b], wu) and _bits(o["dep"][a:b], wd)
    sf = ref.GetScaleFactors()
    isg = ref.GetInverseScaleSigmaSquares()
    bounds = f32([0, W, 0, H])
    cam6 = f32([FX, FY, CX, CY, BF, BF / FX])
    l0, l1, c0, c1 = int(hl["off"][0]), int(hl["off"][1]), int(hc["off"][0]), int(hc["off"][1])
    lastq = (hl["xw"][l0:l1], hl["oct"][l0:l1], hl["ang"][l0:l1], hl["desc"][l0:l1], hl["obs"][l0:l1])
    wfm, wn1 = po.search_last(rk, rd, wu, bounds, sf, cam6, hl["Tcw"][0], direction, *lastq, TH_LAST, True)
    got_fm = o["fm"][a:b].copy()
    got_fm[got_fm >= 0] -= l0
    assert (got_fm == wfm).all() and wn1 == o["nm1"][0]
    locq = (hc["px"][c0:c1], hc["py"][c0:c1], hc["pxr"][c0:c1], hc["lvl"][c0:c1], hc["vc"][c0:c1], hc["desc"][c0:c1])
    wmt, wn2 = po.search_local(rk, rd, wu, bounds, sf, *locq, TH_LOC, 0.8)
    assert (o["mt"][c0:c1] == wmt).all() and wn2 == o["nm2"][0]
    # the stereo gates are live: without mvuRight both searches answer differently
    mono_u = np.full(b - a, -1, f32)
    mfm, _ = po.search_last(rk, rd, mono_u, bounds, sf, cam6, hl["Tcw"][0], direction, *lastq, TH_LAST, True)
    mmt, _ = po.search_local(rk, rd, mono_u, bounds, sf, *locq, TH_LOC, 0.8)
    assert (mfm != wfm).sum() > 10 and (mmt != wmt).sum() > 10
    # both PoseOptimization calls: stereo edges where mvuRight > 0
    holder = np.full(b - a, -1, np.int64)
    for q in np.nonzero(wmt >= 0)[0]:
        holder[wmt[q]] = q
    feat1, feat2 = np.nonzero(wfm >= 0)[0], np.nonzero(holder >= 0)[0]
    for k, (feat, xw) in enumerate([(feat1, lastq[0][wfm[feat1]]), (feat2, hc["xw"][c0:c1][holder[feat2]])]):
        e0, e1 = int(o["eoff"][k][0]), int(o["eoff"][k][1])
        assert (o["efeat"][k][e0:e1] == feat).all()
        obs3 = np.stack([rk["x"][feat], rk["y"][feat], wu[feat]], 1)
        want = po.pose_optimization(hl["Tcw"][0], xw, obs3, isg[rk["octave"][feat]], f32(cam5))
        assert (o["outl"][k][e0:e1] == want["outlier"]).all() and o["inl"][k][0] == want["inliers"]
        assert np.abs(o["pose"][k][0] - want["pose"]).max() < 1e-4
        assert (wu[feat] > 0).sum() > 50                                       # stereo edges took part
    for e in exs + [ref]:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------------
def test_rgbd_chained_flow_matches_the_oracle_stage_by_stage():
    W, H, NF, FX, FY, CX, CY, BF = GEOM["tum_640x480"]
    P = 2
    imgs, maps = _frames(W, H, BF, [2400 + p for p in range(P)])
    ex = _mk(W, H, NF, P)
    _, off, kps, desc, uR, dep = _per_call(ex, imgs, maps, BF)
    frames = []
    for p in range(P):              # every feature at its depth-map depth (3 m in the holes); mvuRight from the depth map
        a, b = int(off[p]), int(off[p + 1])
        k = kps[a:b]
        frames.append(dict(k=k, d=desc[a:b], z=np.where(dep[a:b] > 0, dep[a:b], f32(3.0)).astype(f32),
                           ur=pyrgbd.stereo_from_rgbd(k, maps[p], FACTOR, BF)[0], last=np.arange(0, b - a, 2), other=np.arange(1, b - a, 2),
                           rows=(a, b)))
    step = replay.TrackingStep(ex, camera(FX, FY, CX, CY, BF, BF / FX, W, H), BF, BF / FX, TH_LAST, TH_LOC, 0.8, True, rgbd=True,
                               depth_factor=FACTOR)
    rows, o, nm0, nm2, checked = run_chained_flow(ex, step, imgs, off, frames, f32([FX, FY, CX, CY, BF, BF / FX]), np.arange(P, dtype=np.int32),
                                                  P * ex.max_features_per_image(), TH_LAST, TH_LOC, gross_px=8.0, depth=maps)
    assert _bits(o["ur"][:rows], uR)
    assert nm0.min() > 80 and nm2.min() > 100, (nm0, nm2)
    assert checked["released"] >= 3 and checked["skipped"] > 100 and checked["in_view"] > 400 and checked["local"] > 200, checked
    assert checked["stereo"] > 100, checked          # stereo edges wherever the map has a depth
    ex.close()


# ---------------------------------------------------------------------------------------------------------------------------
def test_rgbd_graph_replay_equals_eager_calls():
    """the device-resident RGB-D step as tools/rgbd_bench.py times it: RGB images and u16 maps in device memory, the extraction,
    orbm_stereo_rgbd_batch and both device searches, captured once and replayed"""
    g = GEOM["tum_640x480"]
    W, H, NF, FX, FY, CX, CY, BF = g
    P = 4
    rng = np.random.default_rng(9)
    dev = torch.device("cuda", 0)
    cam = camera(FX, FY, CX, CY, BF, BF / FX, W, H)
    imgsA, mapsA = _frames(W, H, BF, [2500 + p for p in range(P)], rgb=True)
    imgsB, mapsB = _frames(W, H, BF, [2600 + p for p in range(P)], rgb=True)
    ex, ref = _mk(W, H, NF, P), _mk(W, H, NF, P)
    _, off, kps, desc, uR, dep = _per_call(ref, _grey(imgsA), mapsA, BF)
    hl, hc = _queries(kps, desc, off, dep, g, rng, 1)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    dl, dc = {k: T(v) for k, v in hl.items()}, {k: T(v) for k, v in hc.items()}
    nlast, nloc = int(hl["off"][-1]), int(hc["off"][-1])
    rows_cap = P * ex.max_features_per_image()
    m_last, m_loc = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
    out = lambda: (torch.full((rows_cap,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev),
                   torch.full((nloc,), -7, dtype=torch.int32, device=dev), torch.zeros(P, dtype=torch.int32, device=dev))

    def step(e, src, dmap, o):
        e.extract_batch_device(src.data_ptr(), P, W, H, lapping=(0, 0), image_format="rgb")
        e.stereo_rgbd_batch(dmap, FACTOR, BF)
        m_last.SearchByProjectionLastFrameDevice(e, cam, P, dl["fimg"], dl["off"], dl["Tcw"], dl["dir"], dl["xw"], dl["oct"], dl["ang"], dl["desc"],
                                                 dl["obs"], TH_LAST, o[0], o[1])
        m_loc.SearchByProjectionDevice(e, cam, P, dc["fimg"], dc["off"], dc["px"], dc["py"], dc["pxr"], dc["lvl"], dc["vc"], dc["desc"], o[2], o[3], th=TH_LOC)

    def results(e, o):
        torch.cuda.synchronize()
        n, mono, off, kps, desc = e.download(P)
        rows = int(off[-1])
        u, d = e.stereo_download(rows)
        return [n.copy(), kps.view(np.uint8).copy(), desc.copy(), u.view(np.uint32).copy(), d.view(np.uint32).copy(), o[0][:rows].cpu().numpy(),
                o[1].cpu().numpy(), o[2].cpu().numpy(), o[3].cpu().numpy()]

    d_in, d_map = T(imgsA), T(mapsA)
    oA = out(); step(ref, d_in, d_map, oA); wantA = results(ref, oA)
    d_inB, d_mapB = T(imgsB), T(mapsB)
    oB = out(); step(ref, d_inB, d_mapB, oB); wantB = results(ref, oB)
    assert wantA[6].min() > 50 and wantA[8].min() > 100
    o = out()
    ex.set_device_query_bounds(max(nlast, nloc), int(max(np.diff(hl["off"]).max(), np.diff(hc["off"]).max())), rows_cap)
    step(ex, d_in, d_map, o)
    for a, b in zip(results(ex, o), wantA):
        assert a.shape == b.shape and (a == b).all()
    gr = ex.graph_capture(lambda: step(ex, d_in, d_map, o))
    assert ex.graph_kernels(gr) >= 10
    for src, dm, want in [(imgsA, mapsA, wantA), (imgsB, mapsB, wantB), (imgsA, mapsA, wantA)]:
        d_in.copy_(torch.from_numpy(src))
        d_map.copy_(torch.from_numpy(dm))
        for t in o:
            t.fill_(-7)
        ex.graph_launch(gr)
        for i, (a, b) in enumerate(zip(results(ex, o), want)):
            assert a.shape == b.shape and (a == b).all(), i
    ex.graph_destroy(gr)
    ex.close(); ref.close()


# ---------------------------------------------------------------------------------------------------------------------------
def _setup(P, seed):
    g = GEOM["tum_640x480"]
    W, H, NF, FX, FY, CX, CY, BF = g
    rng = np.random.default_rng(seed)
    cam = camera(FX, FY, CX, CY, BF, BF / FX, W, H)
    pairs = [synth.stereo_pair(W, H, seed=seed + p) for p in range(P)]
    imgs, maps = _frames(W, H, BF, [seed + p for p in range(P)])
    stereo_imgs = np.ascontiguousarray(np.stack([im for p in pairs for im in (p[0], p[1])]))
    probe = _mk(W, H, NF, P)
    _, off, kps, desc, _, dep = _per_call(probe, imgs, maps, BF)
    probe.close()
    hl, hc = _queries(kps, desc, off, dep, g, rng, 1)
    mk = lambda e, kind: replay.TrackingStep(e, cam, BF, BF / FX, TH_LAST, TH_LOC, 0.8, True, monocular=kind == "mono", rgbd=kind == "rgbd",
                                             depth_factor=FACTOR)
    sl, sc = dict(hl), dict(hc)
    sl["fimg"] = sc["fimg"] = (2 * hl["fimg"]).astype(np.int32)           # the same query sets on a stereo batch: frame p is image 2p
    ml = dict(hl); ml["dir"] = np.zeros(P, np.int32)                       # monocular: bMono
    return g, imgs, maps, stereo_imgs, hl, hc, sl, sc, ml, mk


def test_rgbd_refusals_leave_the_handle_usable():
    P = 2
    g, imgs, maps, stereo_imgs, hl, hc, sl, sc, ml, mk = _setup(P, 2700)
    W, H, NF, FX, FY, CX, CY, BF = g
    ex, fresh = _mk(W, H, NF, 2 * P), _mk(W, H, NF, 2 * P)
    rgbd = mk(ex, "rgbd")

    def refused(code, fn):
        with pytest.raises(OrbError, match=f"orb_status {code}:"):
            fn()
    # monocular together with depth maps
    both = mk(ex, "mono"); both.rgbd = True
    refused(ORB_ERR_INVALID, lambda: both.submit(imgs, last=ml, local=hc, depth=maps))
    # a frame image equal to n_frames
    bad = dict(hl); bad["fimg"] = np.array([0, P], np.int32)
    refused(ORB_ERR_INVALID, lambda: rgbd.submit(imgs, last=bad, local=hc, depth=maps))
    # camera images that System::TrackRGBD would resize together with the depth map
    rs = replay.TrackingStep(ex, camera(FX, FY, CX, CY, BF, BF / FX, W // 2, H // 2), BF, BF / FX, rgbd=True, depth_factor=FACTOR, resize=(W // 2, H // 2))
    refused(ORB_ERR_UNSUPPORTED, lambda: rs.submit(imgs, last=hl, local=hc, depth=maps[:, :H // 2, :W // 2].copy()))
    # depth rows shorter than the image's
    refused(ORB_ERR_INVALID, lambda: rgbd.submit(imgs, last=hl, local=hc, depth=maps[:, :, :W - 1].copy()))
    # the per-call entry point: more maps than the last batch holds, an unknown format, short or misaligned strides, no map
    ex.extract_batch(imgs, lapping=(0, 0))
    L, h = ex._L, ex._h
    import ctypes as C
    dp = C.c_void_p(maps.ctypes.data)
    for args in [(P + 1, dp, 1, 2 * W, 2 * W * H), (P, dp, 3, 2 * W, 2 * W * H), (P, dp, 1, 2 * W - 2, 2 * W * H), (P, dp, 1, 2 * W + 1, 2 * W * H),
                 (P, dp, 1, 2 * W, 2 * W * H - 2), (P, dp, 2, 2 * W, 2 * W * H), (P, None, 1, 2 * W, 2 * W * H)]:
        assert L.orbm_stereo_rgbd_batch(h, args[0], args[1], args[2], args[3], args[4], float(FACTOR), 0, float(BF)) == ORB_ERR_INVALID, args
    # the same handle then runs a correct RGB-D step and a correct stereo step; each equals a fresh handle's
    got = run_step(rgbd, imgs, hl, hc, depth=maps)
    same_results(got, run_step(mk(fresh, "rgbd"), imgs, hl, hc, depth=maps))
    assert (got[1]["dep"][:got[0]] > 0).sum() > 1000 and got[1]["nm1"].min() > 50
    got = run_step(mk(ex, "stereo"), stereo_imgs, sl, sc)
    fresh2 = _mk(W, H, NF, 2 * P)
    same_results(got, run_step(mk(fresh2, "stereo"), stereo_imgs, sl, sc), stereo=True)
    for e in (ex, fresh, fresh2):
        e.close()


def test_no_state_leaks_between_stereo_monocular_and_rgbd_steps():
    P = 2
    g, imgs, maps, stereo_imgs, hl, hc, sl, sc, ml, mk = _setup(P, 2800)
    W, H, NF = g[:3]
    used = _mk(W, H, NF, 2 * P)
    for with_po in (False, True):
        runs = {"stereo": lambda e: run_step(mk(e, "stereo"), stereo_imgs, sl, sc, with_po),
                "mono": lambda e: run_step(mk(e, "mono"), imgs, ml, hc, with_po), "rgbd": lambda e: run_step(mk(e, "rgbd"), imgs, hl, hc, with_po, maps)}
        want = {}
        for kind in runs:
            f = _mk(W, H, NF, 2 * P)
            want[kind] = runs[kind](f)
            f.close()
        for kind in ["stereo", "rgbd", "mono", "rgbd", "stereo", "mono", "stereo"]:     # every ordered pair of the three sensors
            same_results(runs[kind](used), want[kind], stereo=kind == "stereo")
        rows, o = want["stereo"]
        assert (o["ur"][:rows] > 0).sum() > 500, with_po                                 # the stereo step has real mvuRight values
        rows, o = want["mono"]
        assert (o["ur"][:rows] == -1).all() and (o["dep"][:rows] == -1).all(), with_po   # monocular after RGB-D still reports -1
        rows, o = want["rgbd"]
        assert (o["ur"][:rows] > 0).sum() > 1000, with_po
    used.close()


def test_pack_keyframe_carries_the_depth_derived_uright():
    W, H, NF, FX, FY, CX, CY, BF = GEOM["tum_640x480"]
    imgs, maps = _frames(W, H, BF, [2900, 2901])
    ex = _mk(W, H, NF, 2)
    _, off, kps, desc, uR, dep = _per_call(ex, imgs, maps, BF)
    dev = torch.device("cuda", 0)
    pose = torch.tensor([0, 0, 0, 1, 0.1, 0.2, 0.3], dtype=torch.float32, device=dev)
    for img in (0, 1):
        block = torch.zeros(ex.keyframe_block_bytes(), dtype=torch.uint8, device=dev)
        ex.pack_keyframe_device(img, pose, block)
        torch.cuda.synchronize()
        kf = replay.unpack_keyframe(block)
        a, b = int(off[img]), int(off[img + 1])
        assert len(kf["uright"]) == b - a and _bits(kf["uright"], uR[a:b]) and (kf["uright"] > 0).sum() > 0.8 * (b - a)
        assert (kf["desc"] == desc[a:b]).all()
    ex.close()
