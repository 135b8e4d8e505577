"""GPU tier: the native replay step (orbr_submit / orbr_collect: host buffers in, host buffers out, nothing blocking in between) gives
exactly what the blocking per-call C ABI gives -- extraction, ComputeStereoMatches, both projection searches and PoseOptimization after
each -- on two handles kept in flight from one host thread; and orbx_pack_keyframe_device writes the block replay.pack_keyframe builds
on the host."""
import numpy as np
import pytest
import torch

from _tracking import check_against_per_call, step_outputs
from orb_slam3_detailed_comments_b200 import ORBextractor, camera, synth, replay
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
W, H, NF = 640, 480, 1200
FX, FY, CX, CY, BF, B = 435.2, 435.2, 320.0, 240.0, 47.9, 0.11


def _queries(ex, imgs, P, rng):
    """Query sets built from the frames' own stereo points (the bench's shape), host arrays."""
    ex.extract_batch(imgs)
    ex.stereo_batch(P, BF, B)
    n, _, off, kps, desc = ex.download(2 * P)
    uR, dep = ex.stereo_download(int(off[-1]))
    last = dict(off=[0], xw=[], oct=[], ang=[], desc=[], obs=[])
    loc = dict(off=[0], px=[], py=[], pxr=[], lvl=[], vc=[], desc=[], xw=[])
    for p in range(P):
        a, b = int(off[2 * p]), int(off[2 * p + 1])
        k, d, z = kps[a:b], desc[a:b], dep[a:b]
        sel = np.nonzero(z > 0)[0][::2]
        pts = np.stack([(k["x"][sel] - CX) * z[sel] / FX, (k["y"][sel] - CY) * z[sel] / FY, z[sel]], 1).astype(np.float32)
        last["xw"].append(pts); last["oct"].append(k["octave"][sel].astype(np.int32)); last["ang"].append(k["angle"][sel].astype(np.float32))
        last["desc"].append(d[sel]); last["obs"].append((rng.random(len(sel)) < 0.9).astype(np.uint8)); last["off"].append(last["off"][-1] + len(sel))
        m = len(k)
        zz = np.where(z > 0, z, 5.0).astype(np.float32)
        x = (k["x"] + rng.normal(0, 1.5, m)).astype(np.float32); y = (k["y"] + rng.normal(0, 1.5, m)).astype(np.float32)
        loc["px"].append(x); loc["py"].append(y); loc["pxr"].append((x - np.float32(BF) / zz).astype(np.float32)); loc["lvl"].append(k["octave"].astype(np.int32))
        loc["vc"].append(rng.uniform(0.99, 1, m).astype(np.float32)); loc["desc"].append(d)
        loc["xw"].append(np.stack([(k["x"] - CX) * zz / FX, (k["y"] - CY) * zz / FY, zz], 1).astype(np.float32)); loc["off"].append(loc["off"][-1] + m)
    cat = lambda xs, dt: np.ascontiguousarray(np.concatenate(xs).astype(dt))
    fimg = np.arange(0, 2 * P, 2, dtype=np.int32)
    hl = dict(fimg=fimg, off=np.array(last["off"], np.int32), Tcw=np.tile(np.array([0, 0, 0, 1, 0.002, 0.001, 0], np.float32), (P, 1)),
              dir=np.zeros(P, np.int32), xw=cat(last["xw"], np.float32), oct=cat(last["oct"], np.int32), ang=cat(last["ang"], np.float32),
              desc=cat(last["desc"], np.uint8), obs=cat(last["obs"], np.uint8))
    hc = dict(fimg=fimg, off=np.array(loc["off"], np.int32), px=cat(loc["px"], np.float32), py=cat(loc["py"], np.float32), pxr=cat(loc["pxr"], np.float32),
              lvl=cat(loc["lvl"], np.int32), vc=cat(loc["vc"], np.float32), desc=cat(loc["desc"], np.uint8), xw=cat(loc["xw"], np.float32))
    return hl, hc


@pytest.mark.parametrize("with_po", [False, True])
def test_replay_step_equals_blocking_calls(with_po):
    P = 2
    rng = np.random.default_rng(11)
    cam = camera(FX, FY, CX, CY, BF, B, W, H)
    batches = [np.stack([im for p in range(P) for im in synth.stereo_pair(W, H, seed=900 + 10 * s + p)[:2]]) for s in range(3)]
    ref = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * P)
    exs = [ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2 * P) for _ in range(2)]
    qs = [_queries(ref, b, P, rng) for b in batches]
    steps = [replay.TrackingStep(e, cam, BF, B, 15.0, 3.0, 0.8, True) for e in exs]
    outs = [step_outputs(2 * P, P, 2 * P * 1400, max(int(q[1]["off"][-1]) for q in qs)) for _ in exs]

    def submit(i):
        hl, hc = qs[i]
        steps[i % 2].submit(batches[i], last=hl, local=hc, pose=hl["Tcw"] if with_po else None, local_world_pos=hc["xw"] if with_po else None)

    # one host thread, two handles in flight: submit i + 1 before collecting i
    submit(0)
    for i in range(3):
        if i + 1 < 3:
            submit(i + 1)
        o = outs[i % 2]
        rows = steps[i % 2].collect(o)
        hl, hc = qs[i]
        # the blocking per-call ABI on a third handle
        ref.extract_batch(batches[i])
        ref.stereo_batch(P, BF, B)
        n, _, off, kps, desc = ref.download(2 * P)
        assert rows == int(off[-1]) and (o["n"] == n).all() and (o["offsets"] == off).all()
        uR, dep = ref.stereo_download(rows)
        left = np.zeros(rows, bool)
        for p in range(P):
            left[int(off[2 * p]):int(off[2 * p + 1])] = True
        assert (o["kps"][:rows].view(np.uint8) == kps.view(np.uint8)).all() and (o["desc"][:rows] == desc).all()
        assert (o["ur"][:rows].view(np.uint32)[left] == uR.view(np.uint32)[left]).all() and (o["dep"][:rows].view(np.uint32)[left] == dep.view(np.uint32)[left]).all()
        nm1, nm2, inl = check_against_per_call(o, rows, ref, cam, hl, hc, 15.0, 3.0, [FX, FY, CX, CY, BF], with_po)
        assert nm1.min() > 50 and nm2.min() > 200 and (inl is None or inl.min() > 30)
    # first frame against the CPU oracle directly (extraction bytes)
    eo = po.OracleExtractor(NF, 1.2, 8, 20, 7)
    _, rk, rd = eo(batches[2][0])
    a, b = int(outs[0]["offsets"][0]), int(outs[0]["offsets"][1])
    assert (outs[0]["kps"][a:b].view(np.uint8) == rk.view(np.uint8)).all() and (outs[0]["desc"][a:b] == rd).all()
    # a second submit on a handle whose step has not been collected is refused
    submit(0)
    with pytest.raises(Exception):
        submit(0)
    steps[0].collect(outs[0])
    for e in exs + [ref]:
        e.close()


def test_pack_keyframe_device_matches_host_pack():
    P = 1
    imgs = np.stack(synth.stereo_pair(W, H, seed=77)[:2])
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ex.extract_batch(imgs)
    ex.stereo_batch(P, BF, B)
    n, _, off, kps, desc = ex.download(2)
    uR, _ = ex.stereo_download(int(off[-1]))
    dev = torch.device("cuda", 0)
    pose = np.array([0.1, 0.2, 0.3, 0.9, 1, 2, 3], np.float32)
    blk = torch.zeros((ex.keyframe_block_bytes() + 255) // 256 * 256, dtype=torch.uint8, device=dev)
    ex.pack_keyframe_device(0, torch.from_numpy(pose).to(dev), blk)
    torch.cuda.synchronize()
    a, b = int(off[0]), int(off[1])
    want = replay.pack_keyframe(pose, kps[a:b], uR[a:b], desc[a:b]).numpy()
    got = blk.cpu().numpy()
    assert (got[:len(want)] == want).all() and n[0] > 1000
    u = replay.unpack_keyframe(got)
    assert (u["desc"] == desc[a:b]).all() and (u["octave"] == kps["octave"][a:b]).all()
    ex.close()
