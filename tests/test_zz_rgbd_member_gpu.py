"""GPU tier: the drop-in Frame::ComputeStereoFromRGBD (orb_slam3_detailed_comments_b200/host/Frame_stereo_b200.cc) LINKED AND RUN
through the reference's own class declarations, as the RGB-D Frame constructor calls it, followed by the drop-in
ORBmatcher::SearchByProjection(F, vpMapPoints) on that frame.  mvuRight / mvDepth must carry the oracle's bits, and the search must
return the oracle's stereo-gated matches: the searches read mvuRight from the device, so without the member they would see -1 and
answer as for a monocular frame.  tests/host/rgbd_member is built by __graft_entry__.build() (tests/host/build_rgbd_member.sh)."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from oracle import pyrgbd
from orb_slam3_detailed_comments_b200 import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "host", "rgbd_member")
W, H, NF = 640, 480, 1000
FX, FY, CX, CY, BF = 535.4, 539.2, 320.1, 247.6, 40.0           # TUM fr3
FACTOR = np.float32(1.0 / 5000)
f32 = np.float32


def test_compute_stereo_from_rgbd_member_and_the_search_after_it(tmp_path):
    assert os.path.exists(BIN), "tests/host/rgbd_member is not built (run __graft_entry__.build())"
    d = str(tmp_path)
    img, _, disp = synth.stereo_pair(W, H, seed=77)
    rng = np.random.default_rng(77)
    raw = np.clip(np.rint(f32(BF) / disp / FACTOR), 0, 65535).astype(np.uint16)
    raw[rng.random(raw.shape) < 0.03] = 0
    depth = (raw.astype(f32) * FACTOR).astype(f32)                   # Tracking::GrabImageRGBD's convertTo(CV_32F, mDepthMapFactor)
    img.tofile(os.path.join(d, "grey.u8"))
    depth.tofile(os.path.join(d, "depth.f32"))
    ex = po.OracleExtractor(NF, 1.2, 8, 20, 7)
    _, kps, desc = ex(img, (0, 0))
    uR, dep = pyrgbd.stereo_from_rgbd(kps, depth, f32(1.0), BF)
    N = len(kps)
    # SearchByProjection(F, vpMapPoints, th = 3) queries: the frame's features at their depth; a quarter predict mTrackProjXR 12 px off
    z = np.where(dep > 0, dep, f32(3.0)).astype(f32)
    loc = dict(px=(kps["x"] + rng.normal(0, 1.0, N)).astype(f32), py=(kps["y"] + rng.normal(0, 1.0, N)).astype(f32))
    loc["pxr"] = (loc["px"] - f32(BF) / z + np.where(rng.random(N) < 0.25, f32(12.0), f32(0.0))).astype(f32)
    loc["level"] = kps["octave"].astype(np.int32)
    loc["vcos"] = rng.uniform(0.999, 1.0, N).astype(f32)
    loc["depth"] = z
    loc["desc"] = desc.copy()
    for k, v in loc.items():
        v.tofile(os.path.join(d, f"loc_{k}." + {"float32": "f32", "int32": "i32", "uint8": "u8"}[str(v.dtype)]))
    meta = dict(W=W, H=H, nfeatures=NF, fx=FX, fy=FY, cx=CX, cy=CY, bf=BF, loc_n=N, loc_th=3.0, loc_nnratio=0.8)
    with open(os.path.join(d, "meta.txt"), "w") as f:
        for k, v in meta.items():
            f.write(f"{k} {float(v)!r}\n")
    r = subprocess.run([BIN, d], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    out = lambda name, dt: np.fromfile(os.path.join(d, name), dt)
    assert (out("out_kps.bin", np.uint8) == kps.view(np.uint8).ravel()).all()
    got_u, got_d = out("out_uright.f32", f32), out("out_depth.f32", f32)
    assert (got_u.view(np.uint32) == uR.view(np.uint32)).all() and (got_d.view(np.uint32) == dep.view(np.uint32)).all()
    assert (dep > 0).sum() > 0.9 * N and (dep == -1).sum() > 5
    # the drop-in search after it: the oracle's stereo-gated matches, not the monocular ones
    bounds = f32([0, W, 0, H])
    sf = ex.scale_factors
    res = out("out_local.i32", np.int32)
    args = (bounds, sf, loc["px"], loc["py"], loc["pxr"], loc["level"], loc["vcos"], loc["desc"], 3.0, f32(0.8))

    def features(match):
        want = np.full(N, -1, np.int32)
        for q, f in enumerate(match):
            if f >= 0:
                want[f] = q
        return want
    stereo, nm = po.search_local(kps, desc, uR, *args, trackdepth=z)
    mono, _ = po.search_local(kps, desc, np.full(N, -1, f32), *args, trackdepth=z)
    assert res[N] == nm and nm > 300
    assert (res[:N] == features(stereo)).all()
    assert (features(mono) != features(stereo)).sum() > 50
