#!/usr/bin/env python
"""Milliseconds per call of the matcher searches on large frames, in the shared-memory and the global-memory form: just below and just
above each search's switch point (where launch_proj changes form) and at 5 000 / 10 000 / 16 000 features.  Prints one JSON line with
the card name and power limit.

  python tools/many_features_bench.py [--repeats 20] [--out FILE]

Each timing is the wall time of a whole C-ABI call with host arrays in and out (query upload, every kernel, result download, the call's
own stream synchronisation), median over the repeats after three warm-up calls.  Frames come from one 3840x2160 synthetic stereo pair:
the per-frame searches run on extractor handles sized to the row count (n_features = rows - 20 x 8 levels), the keyframe searches on
host keyframes of exactly that many rows.  Which form ran is read from the library's launch counter."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera, synth  # noqa: E402
from orb_slam3_detailed_comments_b200 import _native as N  # noqa: E402

W, H = 3840, 2160
S = W / 640.0
FX, FY, CX, CY, BF, B = 435.2 * S, 435.2 * S, W / 2.0, H / 2.0, 47.9 * S, 0.11
OPTIN, STATIC = 232448, 256


def fsm(n):
    return (n * 23 + 16 + 15) // 16 * 16


def shared_form(n, mode):
    """launch_proj's choice (matcher.cu) for a frame of n rows on an H100."""
    csm = max(fsm(n), (n * 17 + 3073 * 2 + 32 + 15) // 16 * 16)
    psm = fsm(n) + 9 * n + (8192 + 512) * 4 + 64
    rsm = fsm(n) + 1024 * 64 + 1024 * 4 + n * (9 if mode == 4 else 5) + 1024 * 5 + 256
    return csm <= OPTIN and (mode not in (0, 1) or psm + STATIC <= OPTIN) and rsm + STATIC <= OPTIN


def switch(mode):
    return max(n for n in range(3000, 12000) if shared_form(n, mode))


def timed(fn, repeats):
    for _ in range(3):
        fn()
    L = N.lib()
    n0 = int(L.orb_kernel_launches())
    fn()
    launches = int(L.orb_kernel_launches()) - n0
    ts = []
    for _ in range(repeats):
        t = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts)), launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(1)
    L_img, R_img, _ = synth.stereo_pair(W, H, seed=11, dmin=2.0, dmax=0.5 * FX)
    cur = np.roll(L_img, (1, 3), (0, 1))
    cam = camera(FX, FY, CX, CY, BF, B, W, H)
    results = {"gpu": gpu, "unit": "ms per call (host arrays in / out, median)", "searches": {}}

    def add(search, rows, form, ms, launches):
        results["searches"].setdefault(search, []).append(dict(rows=rows, form=form, ms=round(ms, 4), launches=launches))

    # per-frame searches: handles of `rows` row capacity, frame = the shifted left image, queries from the unshifted one
    sizes0 = sorted({switch(0), switch(0) + 1, 5000, 10000, 16000})
    ref_ex = ORBextractor(16000, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
    ref_ex.extract_batch(np.stack([L_img, R_img]))
    ref_ex.stereo_batch(1, BF, B)
    _, _, off, kps, desc = ref_ex.download(2)
    uR, dep = ref_ex.stereo_download(int(off[-1]))
    kL, dL, zL = kps[: off[1]], desc[: off[1]], dep[: off[1]]
    sel = np.nonzero(zL > 0)[0]
    z = zL[sel]
    xw = np.stack([(kL["x"][sel] - CX) * z / FX, (kL["y"][sel] - CY) * z / FY, z], 1).astype(np.float32)
    x = (kL["x"][sel] + 3 + rng.normal(0, 1.5, len(sel))).astype(np.float32)
    y = (kL["y"][sel] + 1 + rng.normal(0, 1.5, len(sel))).astype(np.float32)
    xr = (x - np.float32(BF) / z).astype(np.float32)
    lv, vc, qd = kL["octave"][sel].astype(np.int32), rng.uniform(0.99, 1, len(sel)).astype(np.float32), dL[sel]
    Tcw = np.array([[0, 0, 0, 1, 3 * float(np.median(z)) / FX, float(np.median(z)) / FY, 0]], np.float32)
    node = lambda d: ((d[:, 0].astype(np.int32) >> 3) * 7 + (d[:, 5].astype(np.int32) >> 4) * 3 + (d[:, 17].astype(np.int32) >> 5)) % 97
    for rows in sizes0:
        ex = ORBextractor(rows - 160, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=2)
        ex.extract_batch(np.stack([cur, np.roll(R_img, (1, 3), (0, 1))]))
        ex.stereo_batch(1, BF, B)
        _, _, off2, k2, d2 = ex.download(2)
        total = int(off2[-1])
        m0, m1 = ORBmatcher(0.8, True), ORBmatcher(0.9, True)
        n = len(sel)
        ms, nl = timed(lambda: m0.SearchByProjection(ex, cam, [0], [0, n], x, y, xr, lv, vc, qd, th=3.0), a.repeats)
        add("SearchByProjection(F, local map)", rows, "shared" if shared_form(rows, 0) else "global", ms, nl)
        ms, nl = timed(lambda: m1.SearchByProjectionLastFrame(ex, cam, [0], [0, n], Tcw, [0], xw, lv, kL["angle"][sel].astype(np.float32), qd,
                                                              np.ones(n, np.uint8), 15.0, total), a.repeats)
        add("SearchByProjection(cur, last)", rows, "shared" if shared_form(rows, 1) else "global", ms, nl)
        fnode = node(d2).astype(np.int32)
        qn = node(qd).astype(np.int32)
        order = np.lexsort((np.arange(n), qn))
        ms, nl = timed(lambda: ORBmatcher(0.7, True).SearchByBoW(ex, [0], [0, n], qn[order], kL["angle"][sel][order].astype(np.float32),
                                                                   qd[order], fnode, total), a.repeats)
        add("SearchByBoW(KF, F)", rows, "shared" if shared_form(rows, 2) else "global", ms, nl)
        ex.close()
    # host keyframes / host F2 of exactly `rows` features
    kpR, dR = kps[: off[1]], desc[: off[1]]
    ex = ref_ex
    sf = ex.GetScaleFactors()
    dist = np.linalg.norm(xw, axis=1).astype(np.float32)
    maxd = (dist * sf[lv]).astype(np.float32)
    q = dict(world_pos=xw, max_dist=maxd, min_dist=(maxd / sf[7]).astype(np.float32), desc=qd, angle=kL["angle"][sel].astype(np.float32))
    T = Tcw[0]
    for mode, name in [(3, "SearchByProjection(F, KF, set)"), (4, "SearchForInitialization")]:
        for rows in sorted({switch(mode), switch(mode) + 1, 5000, 10000, 16000}):
            idx = np.resize(np.arange(len(kpR)), rows)
            kk, dd = kpR[idx], dR[idx]
            if mode == 3:
                tgt = [dict(kp=kk, desc=dd, Tcw=T, Ow=np.zeros(3, np.float32))]
                fn = lambda: ORBmatcher(0.9, True).SearchByProjectionReloc(ex, cam, tgt, [q], 10.0, 100)
            else:
                prev = np.stack([kL["x"], kL["y"]], 1).astype(np.float32)
                fn = lambda: ORBmatcher(0.9, True).SearchForInitialization(ex, cam, kL, dL, prev, 100, kp2=kk, desc2=dd)
            ms, nl = timed(fn, a.repeats)
            add(name, rows, "shared" if shared_form(rows, mode) else "global", ms, nl)
    ref_ex.close()
    line = json.dumps(results)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
