"""GPU tier: one extractor handle reused across image sizes gives, at every size, what a fresh handle of that size gives and what the
oracle gives (its workspace is laid out once, for its largest image, and nothing in it grows); and the per-frame projection and BoW
searches, in both forms, and the replay step refuse a call whose queries lack a required array, after which the handle's next call
gives what a fresh handle gives."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor, camera, replay, synth
from orb_slam3_detailed_comments_b200 import _native as N
from orb_slam3_detailed_comments_b200._native import KP_DTYPE

pytestmark = pytest.mark.gpu
NF = 1200
W, H = 640, 480
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11
DEV = torch.device("cuda", 0)


def _extract(ex, imgs, bf):
    ex.extract_batch(imgs)
    ex.stereo_batch(1, bf, B)
    n, mono, off, kps, desc = ex.download(2)
    ur, dep = ex.stereo_download(int(off[-1]))
    left = slice(int(off[0]), int(off[1]))          # mvuRight / mvDepth exist for the left image's rows only
    return dict(n=n, mono=mono, off=off, kps=kps, desc=desc, ur=ur[left], dep=dep[left])


def test_one_handle_across_image_sizes():
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=1920, max_height=1080, max_batch=2)
    ref = po.OracleExtractor(NF, 1.2, 8, 20, 7)
    for i, (w, h) in enumerate([(640, 480), (1241, 376), (752, 480), (1920, 1080), (640, 480)]):
        imgs = np.stack(synth.stereo_pair(w, h, seed=300 + i)[:2])
        bf = BF * w / 640
        got = _extract(ex, imgs, bf)
        fresh = ORBextractor(NF, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=2)
        want = _extract(fresh, imgs, bf)
        fresh.close()
        for k in got:
            assert got[k].tobytes() == want[k].tobytes(), (w, h, k)
        assert (got["dep"] > 0).sum() > 100, (w, h)
        off = got["off"]
        for b in range(2):
            rmono, rk, rd = ref(imgs[b])
            a, e = int(off[b]), int(off[b + 1])
            assert got["mono"][b] == rmono and e - a == len(rk), (w, h, b)
            assert (got["kps"][a:e].view(np.uint8) == rk.view(np.uint8)).all() and (got["desc"][a:e] == rd).all(), (w, h, b)
    ex.close()


def _handle(imgs):
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ex.extract_batch(imgs)
    ex.stereo_batch(1, BF, B)
    return ex


@pytest.fixture(scope="module")
def scene():
    l, r, _ = synth.stereo_pair(W, H, seed=71)
    imgs = np.stack([l, r])
    ex = _handle(imgs)
    n, _, off, kps, desc = ex.download(2)
    _, dep = ex.stereo_download(int(off[-1]))
    rng = np.random.default_rng(5)
    a, b = int(off[0]), int(off[1])
    k, d = kps[a:b], desc[a:b].copy()
    nq = len(k)
    d[rng.random(d.shape) < 0.03] ^= np.uint8(1 << 3)
    x = (k["x"] + rng.normal(0, 1.0, nq)).astype(np.float32)
    y = (k["y"] + rng.normal(0, 1.0, nq)).astype(np.float32)
    z = np.where(dep[a:b] > 0, dep[a:b], rng.uniform(2, 10, nq)).astype(np.float32)
    xw = np.stack([(x - CX) * z / FX, (y - CY) * z / FY, z], 1).astype(np.float32)
    node = lambda dd: ((dd[:, 0].astype(np.int64) * 7 + dd[:, 5].astype(np.int64) * 13 + dd[:, 17]) % 97).astype(np.int32)
    fimg, qoff = np.array([0], np.int32), np.array([0, nq], np.int32)
    oct_, ang = k["octave"].astype(np.int32), k["angle"].astype(np.float32)
    queries = {
        "local": dict(frame_image=fimg, query_offset=qoff, proj_x=x, proj_y=y, proj_xr=(x - BF / z).astype(np.float32), level=oct_,
                      view_cos=np.ones(nq, np.float32), track_depth=z, desc=d, feature_claimed=None, in_view=np.ones(nq, np.uint8)),
        "last": dict(frame_image=fimg, query_offset=qoff, Tcw=np.array([[0, 0, 0, 1, 0, 0, 0]], np.float32), direction=np.zeros(1, np.int32),
                     world_pos=xw, last_octave=oct_, last_angle=ang, desc=d, obs_positive=np.ones(nq, np.uint8)),
        "bow": dict(frame_image=fimg, query_offset=qoff, query_node=node(d), query_angle=ang, desc=d, feature_node=node(desc)),
    }
    yield dict(ex=ex, imgs=imgs, total=int(off[-1]), nq=nq, queries=queries, cam=camera(FX, FY, CX, CY, BF, B, W, H))
    ex.close()


SEARCHES = {   # query struct, required query arrays, the call, output lengths
    "local": (N.orbm_local_queries, ("proj_x", "proj_y", "proj_xr", "level", "view_cos", "desc"),
              lambda L, h, cam, q, o: L.orbm_search_local_points(h, C.byref(cam), C.byref(q), 3.0, 0.8, 0, 0.0, *o), lambda s: (s["nq"], 1)),
    "last": (N.orbm_last_queries, ("world_pos", "last_octave", "last_angle", "desc"),
             lambda L, h, cam, q, o: L.orbm_search_last_frame(h, C.byref(cam), C.byref(q), 7.0, 1, *o), lambda s: (s["total"], 1)),
    "bow": (N.orbm_bow_queries, ("query_node", "query_angle", "desc"),
            lambda L, h, cam, q, o: L.orbm_search_bow(h, C.byref(q), 0.7, 1, *o), lambda s: (s["total"], 1)),
}


def _search(s, ex, kind, on_device, drop=None):
    """One search on `ex` with the scene's queries, `drop` passed as NULL: (status, match, nmatches)."""
    qtype, _, call, sizes = SEARCHES[kind]
    arrs = {f: (None if f == drop else s["queries"][kind][f]) for f, _ in qtype._fields_[2:]}
    if on_device:
        arrs = {f: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for f, a in arrs.items()}
        outs = [torch.full((n,), 123, dtype=torch.int32, device=DEV) for n in sizes(s)]
        p = lambda a: None if a is None else C.c_void_p(a.data_ptr())
        torch.cuda.synchronize()
    else:
        outs = [np.full(n, 123, np.int32) for n in sizes(s)]
        p = N.ptr
    q = qtype(1, int(on_device), *[p(arrs[f]) for f, _ in qtype._fields_[2:]])
    st = call(N.lib(), ex._h, s["cam"], q, [p(o) for o in outs])
    if on_device:
        torch.cuda.synchronize()
        outs = [o.cpu().numpy() for o in outs]
    return st, outs[0], outs[1]


@pytest.mark.parametrize("kind", ["local", "last", "bow"])
def test_search_refuses_missing_query_arrays(scene, kind):
    fresh = _handle(scene["imgs"])
    _, want_m, want_n = _search(scene, fresh, kind, False)
    fresh.close()
    assert want_n[0] > 50
    for on_device in (False, True):
        for drop in SEARCHES[kind][1]:
            st, m, n = _search(scene, scene["ex"], kind, on_device, drop)
            assert st == -1 and "missing query arrays" in N.lib().orb_last_error().decode(), (kind, on_device, drop, st)
            assert (m == 123).all() and n[0] == 123, (kind, on_device, drop)   # nothing was written
            st, m, n = _search(scene, scene["ex"], kind, on_device)
            assert st == 0 and (m == want_m).all() and (n == want_n).all(), (kind, on_device, drop)


def _step_queries(s):
    q = s["queries"]
    last = {k: q["last"][f] for k, f in (("fimg", "frame_image"), ("off", "query_offset"), ("Tcw", "Tcw"), ("dir", "direction"),
                                          ("xw", "world_pos"), ("oct", "last_octave"), ("ang", "last_angle"), ("desc", "desc"), ("obs", "obs_positive"))}
    local = {k: q["local"][f] for k, f in (("fimg", "frame_image"), ("off", "query_offset"), ("px", "proj_x"), ("py", "proj_y"), ("pxr", "proj_xr"),
                                           ("lvl", "level"), ("vc", "view_cos"), ("desc", "desc"))}
    return last, local


def _step(s, ex, last, local):
    step = replay.TrackingStep(ex, s["cam"], BF, B, 7.0, 3.0, 0.8, True)
    pose = last["Tcw"]
    xw = s["queries"]["last"]["world_pos"]
    step.submit(s["imgs"], last=last, local=local, pose=pose, local_world_pos=xw)
    rc, nq = 2800, s["nq"]
    z = lambda shape, dt: np.zeros(shape, dt)
    out = dict(kps=z(rc, KP_DTYPE), desc=z((rc, 32), np.uint8), ur=z(rc, np.float32), dep=z(rc, np.float32), n=z(2, np.int32), offsets=z(3, np.int32),
               fm=z(rc, np.int32), nm1=z(1, np.int32), mt=z(nq, np.int32), nm2=z(1, np.int32), pose=z((2, 1, 7), np.float64), inl=z((2, 1), np.int32),
               eoff=z((2, 2), np.int32), efeat=z((2, rc), np.int32), outl=z((2, rc), np.uint8))
    rows = step.collect(out)
    a, b = int(out["offsets"][0]), int(out["offsets"][1])
    out["ur"], out["dep"] = out["ur"][a:b], out["dep"][a:b]
    for k in ("kps", "desc", "fm"):
        out[k] = out[k][:rows]
    for k in ("efeat", "outl"):
        out[k] = np.concatenate([out[k][i][: int(out["eoff"][i][-1])] for i in range(2)])
    return out


def test_replay_step_refuses_missing_query_arrays(scene):
    last, local = _step_queries(scene)
    fresh = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    want = _step(scene, fresh, last, local)
    fresh.close()
    assert want["nm1"][0] > 50 and want["nm2"][0] > 50
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    missing = [("last", k) for k in ("xw", "oct", "ang", "desc")] + [("local", k) for k in ("px", "py", "pxr", "lvl", "vc", "desc")]
    for which, key in missing:
        ql = {k: (None if (which, k) == ("last", key) else v) for k, v in last.items()}
        qc = {k: (None if (which, k) == ("local", key) else v) for k, v in local.items()}
        step = replay.TrackingStep(ex, scene["cam"], BF, B, 7.0, 3.0, 0.8, True)
        with pytest.raises(N.OrbError, match=r"orb_status -1: missing query arrays"):
            step.submit(scene["imgs"], last=ql, local=qc)
        got = _step(scene, ex, last, local)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), (which, key, k)
    ex.close()
