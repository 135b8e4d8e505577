"""GPU tier: camera images converted and resized on the device (k_ingest: System::Track*'s cv::resize, then Tracking::GrabImage*'s
cv::cvtColor to grey, into level 0 of the pyramid).

- for every orb_image_format, with and without a resize, stereo and monocular, the replay step fed with the camera images gives
  exactly what the grey step gives fed with the oracle's grey images: keypoints, descriptors, mvuRight / mvDepth, both match arrays
  and both PoseOptimization results;
- level 0 of each image is cv2's resize-then-cvtColor, byte for byte;
- a CUDA-graph replay of orbx_extract_batch_device_format equals the eager call, also on new images written into the same buffer;
- an unknown format, a short stride and a target larger than the handle are refused (ORB_ERR_INVALID) and the handle stays usable;
- grey and colour steps alternating on one handle give what each gives alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from _tracking import run_step, same_results
from orb_slam3_detailed_comments_b200 import ORBextractor, camera, synth, replay
from orb_slam3_detailed_comments_b200 import _native as N
from orb_slam3_detailed_comments_b200._native import OrbError
from oracle import pyingest

pytestmark = pytest.mark.gpu
NF = 1200
f32 = np.float32
FX, FY, BF, B = 435.2, 435.2, 47.9, 0.11
FORMATS = ["gray", "rgb", "bgr", "rgba", "bgra"]
W, H = 640, 480
SRC_RESIZED = (960, 600)          # a camera larger than the extracted image, non-integer ratios in both axes


def _camera_images(grey, fmt, seed):
    """colour images whose channels are noisy copies of `grey` (random alpha): textured in every channel"""
    cn = N.FORMAT_CHANNELS[N.IMAGE_FORMATS[fmt]]
    if cn == 1:
        return np.ascontiguousarray(grey)
    rng = np.random.default_rng(seed)
    ch = [np.clip(grey.astype(np.int16) + rng.integers(-24, 25, grey.shape), 0, 255) for _ in range(3)]
    if cn == 4:
        ch.append(rng.integers(0, 256, grey.shape))
    return np.ascontiguousarray(np.stack(ch, -1).astype(np.uint8))


def _stereo_frames(sw, sh, nf, seed):
    pairs = [synth.stereo_pair(sw, sh, seed=seed + p) for p in range(nf)]
    return np.stack([im for p in pairs for im in (p[0], p[1])])


def _oracle_grey(images, fmt, size):
    return np.stack([pyingest.ingest(im, fmt, size) for im in images])


def _queries(ex, grey, nimg, mono):
    """query sets from the frames' own features at a made-up depth: the searches match plenty, which is all equality needs"""
    ex.extract_batch(grey, lapping=(0, 1000) if mono else (0, 0))
    n, _, off, kps, desc = ex.download(nimg)
    rng = np.random.default_rng(3)
    nf = nimg if mono else nimg // 2
    step = 1 if mono else 2
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    loc = dict(off=[0], px=[], py=[], pxr=[], lvl=[], vc=[], desc=[], xw=[])
    for f in range(nf):
        a, b = int(off[step * f]), int(off[step * f + 1])
        k, d = kps[a:b], desc[a:b]
        z = rng.uniform(2.0, 8.0, len(k)).astype(f32)
        xw = np.stack([(k["x"] - W / 2) * z / FX, (k["y"] - H / 2) * z / FY, z], 1).astype(f32)
        sel = np.arange(0, len(k), 2)
        last["xw"].append(xw[sel]); last["oct"].append(k["octave"][sel]); last["ang"].append(k["angle"][sel]); last["desc"].append(d[sel])
        last["obs"].append(np.ones(len(sel), np.uint8)); last["off"].append(last["off"][-1] + len(sel))
        x = (k["x"] + rng.normal(0, 1.0, len(k))).astype(f32); y = (k["y"] + rng.normal(0, 1.0, len(k))).astype(f32)
        loc["px"].append(x); loc["py"].append(y); loc["pxr"].append(x - BF / z); loc["lvl"].append(k["octave"])
        loc["vc"].append(np.ones(len(k), f32)); loc["desc"].append(d); loc["xw"].append(xw); loc["off"].append(loc["off"][-1] + len(k))
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    fimg = (np.arange(nf) * step).astype(np.int32)
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=np.tile(np.array([0, 0, 0, 1, 0, 0, 0], f32), (nf, 1)),
              dir=np.zeros(nf, np.int32), xw=cat(last["xw"], f32), oct=cat(last["oct"], np.int32), ang=cat(last["ang"], f32),
              desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(fimg=fimg, off=np.array(loc["off"], np.int32), px=cat(loc["px"], f32), py=cat(loc["py"], f32), pxr=cat(loc["pxr"], f32),
              lvl=cat(loc["lvl"], np.int32), vc=cat(loc["vc"], f32), desc=cat(loc["desc"], np.uint8), xw=cat(loc["xw"], f32))
    return hl, hc


def _run(ex, images, fmt, resize, mono, q):
    st = replay.TrackingStep(ex, camera(FX, FY, W / 2, H / 2, BF, B, W, H), BF, B, 15.0, 3.0, 0.8, True, monocular=mono,
                             image_format=fmt, resize=resize)
    return run_step(st, images, *q)


def _assert_same(got, want, mono):
    same_results(got, want, stereo=not mono)
    rows, o = got
    assert rows > 0 and o["nm1"].min() > 50 and o["nm2"].min() > 50


@pytest.fixture(scope="module")
def handles():
    return {m: ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=4) for m in ("step", "ref")}


@pytest.mark.parametrize("mono", [False, True], ids=["stereo", "mono"])
@pytest.mark.parametrize("fmt,resized", [(f, r) for f in FORMATS for r in (False, True) if f != "gray" or r])   # grey, same size: the grey step itself
def test_camera_step_equals_grey_step_on_oracle_images(handles, fmt, resized, mono):
    sw, sh = SRC_RESIZED if resized else (W, H)
    grey_src = _stereo_frames(sw, sh, 2, seed=400 + sw)
    if mono:
        grey_src = grey_src[::2].copy()
    images = _camera_images(grey_src, fmt, seed=7)
    grey = _oracle_grey(images, fmt, (W, H))
    q = _queries(handles["ref"], grey, len(grey), mono)
    want = _run(handles["ref"], grey, "gray", None, mono, q)
    got = _run(handles["step"], images, fmt, (W, H) if resized else None, mono, q)
    _assert_same(got, want, mono)


@pytest.mark.parametrize("cn,rgb", [(1, False), (3, False), (3, True), (4, False), (4, True)])
@pytest.mark.parametrize("src", [(W, H), (1280, 720), (320, 240)], ids=["same_size", "down", "up"])
def test_level0_is_cv2(handles, cn, rgb, src):
    cv2 = pytest.importorskip("cv2")
    grey_src = synth.frame_batch(3, *src, seed=11)
    images = _camera_images(grey_src, {1: "gray", 3: "bgr", 4: "bgra"}[cn], seed=5)
    ex = handles["step"]
    n, _ = ex.extract_batch(images, rgb=rgb, resize=(W, H))
    assert n.min() > 1000
    code = {(3, False): cv2.COLOR_BGR2GRAY, (3, True): cv2.COLOR_RGB2GRAY, (4, False): cv2.COLOR_BGRA2GRAY, (4, True): cv2.COLOR_RGBA2GRAY}
    for b, im in enumerate(images):
        want = cv2.resize(im, (W, H), interpolation=cv2.INTER_LINEAR)
        if cn > 1:
            want = cv2.cvtColor(want, code[(cn, rgb)])
        assert (ex.image_pyramid(b, 0) == want).all(), b


def test_graph_replay_of_the_device_entry_equals_eager():
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    sw, sh = 1280, 720
    imgs = [_camera_images(synth.frame_batch(2, sw, sh, seed=s), "bgr", seed=s) for s in (21, 31)]
    d = torch.from_numpy(imgs[0]).cuda()
    torch.cuda.synchronize()
    call = lambda: ex.extract_batch_device(d.data_ptr(), 2, W, H, image_format="bgr", src_size=(sw, sh))
    call()
    eager = ex.download(2)
    g = ex.graph_capture(call)
    try:
        ex.graph_launch(g)
        got = ex.download(2)
        assert all((x.view(np.uint8) == y.view(np.uint8)).all() for x, y in zip(got, eager))
        d.copy_(torch.from_numpy(imgs[1]))
        torch.cuda.synchronize()
        ex.graph_launch(g)
        got = ex.download(2)
    finally:
        ex.graph_destroy(g)
    d.copy_(torch.from_numpy(imgs[1]))
    torch.cuda.synchronize()
    call()
    eager = ex.download(2)
    assert eager[2][-1] > 2000
    assert all((x.view(np.uint8) == y.view(np.uint8)).all() for x, y in zip(got, eager))


def test_refusals_leave_the_handle_usable(handles):
    ex = handles["step"]
    L = N.lib()
    grey = _stereo_frames(W, H, 1, seed=77)
    images = _camera_images(grey, "bgra", seed=1)
    d = torch.from_numpy(images).cuda()
    torch.cuda.synchronize()
    ex.extract_batch(images, resize=(W, H))
    before = ex.download(2)

    def dev(fmt, stride, w, h):
        return L.orbx_extract_batch_device_format(ex._h, C.c_void_p(d.data_ptr()), 2, w, h, stride, stride * H, 0, 0, fmt, W, H)

    assert dev(5, W * 4, W, H) == -1 and dev(-1, W * 4, W, H) == -1          # unknown format
    assert dev(4, W * 4 - 1, W, H) == -1                                     # a row shorter than width x channels
    assert dev(4, W * 4, W + 16, H) == -1                                    # larger than the handle
    cam = camera(FX, FY, W / 2, H / 2, BF, B, W, H)
    for fields in (dict(image_format=9), dict(image_format=2, src_stride=W * 3 - 1), dict(image_format=2, width=W, height=H + 2),
                   dict(image_format=2, width=W + 2)):
        st = N.orbr_step(n_frames=1, images=N.ptr(images), width=W, height=H, bf=BF, b=B, src_width=W, src_height=H)
        for k, v in fields.items():
            setattr(st, k, v)
        assert L.orbr_submit(ex._h, C.byref(cam), C.byref(st)) == -1, fields
    with pytest.raises(OrbError):
        ex.extract_batch_device(d.data_ptr(), 2, W, H, image_format="bgra", stride=W)
    ex.extract_batch(images, resize=(W, H))
    after = ex.download(2)
    assert all((x.view(np.uint8) == y.view(np.uint8)).all() for x, y in zip(after, before))
    q = _queries(handles["ref"], grey, 2, False)
    _assert_same(_run(ex, grey, "gray", None, False, q), _run(handles["ref"], grey, "gray", None, False, q), False)


def test_grey_and_colour_steps_alternate_without_leaking(handles):
    grey_a = _stereo_frames(W, H, 2, seed=610)
    grey_b = _stereo_frames(*SRC_RESIZED, 2, seed=620)
    colour_b = _camera_images(grey_b, "rgb", seed=2)
    oracle_b = _oracle_grey(colour_b, "rgb", (W, H))
    qa = _queries(handles["ref"], grey_a, 4, False)
    qb = _queries(handles["ref"], oracle_b, 4, False)
    want_a = _run(handles["ref"], grey_a, "gray", None, False, qa)
    want_b = _run(handles["ref"], oracle_b, "gray", None, False, qb)
    ex = handles["step"]
    for _ in range(2):
        _assert_same(_run(ex, grey_a, "gray", None, False, qa), want_a, False)
        _assert_same(_run(ex, colour_b, "rgb", (W, H), False, qb), want_b, False)
