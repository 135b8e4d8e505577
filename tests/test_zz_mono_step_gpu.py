"""GPU tier: the monocular replay step (orbr_step::monocular: one image per frame through ORBextractor::operator() with
vLappingArea = {0, 1000}, Frame.cc:380; no ComputeStereoMatches, so every search and PoseOptimization sees mvuRight = -1).

- on two handles kept in flight from one host thread it gives exactly what the blocking per-call C ABI gives, and the first frame
  of a batch equals the CPU oracle: keypoints, descriptors, monoIndex and both match arrays (752x480 EuRoC-shaped frames, and
  1241x376 KITTI-shaped ones, where the two fill directions of the lapping area interleave);
- the chained flow in monocular mode matches the oracle stage by stage;
- a CUDA-graph replay of the device-resident monocular step equals the eager calls;
- the step refuses oversized batches, out-of-range frame images and a nonzero direction, and the handle stays usable.
Monocular steps next to stereo and RGB-D ones on one handle are in tests/test_zz_rgbd_step_gpu.py."""
import numpy as np
import pytest
import torch

from _tracking import check_against_per_call, run_chained_flow, run_step, same_results, step_outputs
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth, replay
from orb_slam3_detailed_comments_b200._native import OrbError
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
    qs = [_queries(ref, f[0], f[2], g, rng) for f in frames]
    steps = [replay.TrackingStep(e, cam, 0.0, 0.0, TH_LAST, TH_LOC, 0.8, True, monocular=True) for e in exs]
    outs = [step_outputs(P, P, P * 1400, max(int(q[1]["off"][-1]) for q in qs)) for _ in exs]

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
        nm1, nm2, inl = check_against_per_call(o, rows, ref, cam, hl, hc, TH_LAST, TH_LOC, [FX, FY, CX, CY, 0.0], with_po)
        assert nm1.min() > 50 and nm2.min() > 100 and (inl is None or inl.min() > 30)
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


def test_mono_chained_flow_matches_the_oracle_stage_by_stage():
    W, H, FX, FY, CX, CY, BFGT = GEOM["euroc_752x480"]
    P = 2
    imgs, _, disps = _frames(W, H, [1400 + p for p in range(P)])
    ex = _mk(W, H, P)
    ex.extract_batch(imgs, lapping=(0, 1000))
    _, _, off, kps, desc = ex.download(P)
    frames = []
    for p in range(P):              # every feature at the ground-truth depth of the disparity field; mvuRight = -1
        a, b = int(off[p]), int(off[p + 1])
        k = kps[a:b]
        frames.append(dict(k=k, d=desc[a:b], z=_depth(disps[p], k, BFGT), ur=np.full(b - a, -1, f32), last=np.arange(0, b - a, 2),
                           other=np.arange(1, b - a, 2), rows=(a, b)))
    step = replay.TrackingStep(ex, camera(FX, FY, CX, CY, 0.0, 0.0, W, H), 0.0, 0.0, TH_LAST, TH_LOC, 0.8, True, monocular=True)
    # gross errors 8 px to the side: inside the search window, so the search matches them; the reprojection error makes them outliers
    rows, o, nm0, nm2, checked = run_chained_flow(ex, step, imgs, off, frames, f32([FX, FY, CX, CY, 0.0, 0.0]), np.arange(P, dtype=np.int32),
                                                  P * 1400, TH_LAST, TH_LOC, gross_px=8.0)
    assert (o["ur"][:rows] == -1).all()
    assert nm0.min() > 80 and nm2.min() > 100, (nm0, nm2)
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
    got = run_step(mono, left[:P], hl, hc)
    want = run_step(replay.TrackingStep(fresh, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True, monocular=True), left[:P], hl, hc)
    same_results(got, want)
    assert got[1]["nm1"].min() > 50 and (got[1]["ur"][:got[0]] == -1).all()
    stereo_imgs = np.ascontiguousarray(np.stack([im for p in range(P) for im in (left[p], right[p])]))
    sl, sc = _stereo_queries(hl, hc)
    got = run_step(replay.TrackingStep(ex, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True), stereo_imgs, sl, sc)
    fresh2 = _mk(W, H, 2 * P)
    want = run_step(replay.TrackingStep(fresh2, cam, BFGT, BFGT / FX, TH_LAST, TH_LOC, 0.8, True), stereo_imgs, sl, sc)
    same_results(got, want, stereo=True)
    for e in (ex, fresh, fresh2):
        e.close()
