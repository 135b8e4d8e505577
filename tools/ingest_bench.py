#!/usr/bin/env python
"""Colour and resized camera images on the device: config 3's workload (640x480 stereo, 1200 features, bench.py) fed with BGR images.
Prints one JSON line with the card's name, power limit and SM clock read in the same process.

  python tools/ingest_bench.py [--batch 64] [--handles 4] [--steps 20] [--repeats 3] [--out FILE]

  e2e_bgr_device     BGR host images through orbr_submit / orbr_collect (image_format = BGR: the step uploads the colour images and
                     converts them on the device, k_ingest), one host thread, the handles in flight
  e2e_bgr_host_cv2   the same frames converted on the host with cv2.cvtColor(COLOR_BGR2GRAY) into pinned grey buffers, then the grey
                     step: what a caller does without the device conversion
  e2e_grey           the grey step on the already grey frames (what bench.py's e2e leg runs)
  resize_1280x720    1280x720 BGR frames resized to 640x480 and converted, on the device vs cv2.resize + cv2.cvtColor on the host
  graph_replay       frames resident in HBM, each batch one CUDA-graph replay (bench.py's value leg) with BGR input through
                     orbx_extract_batch_device_format, next to the same replay with grey input
The e2e legs alternate over --repeats rounds and report every round: frames/s and the host CPU seconds per frame of this process
(time.process_time: every host thread, cv2's included).  The first batch of every leg is checked against the grey step on cv2's
grey images before anything is timed.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cv2  # noqa: E402

import bench  # noqa: E402
from mono_bench import card  # noqa: E402


def colour_pool(grey, seed):
    """BGR images whose channels are noisy copies of the grey frames (every channel textured)"""
    rng = np.random.default_rng(seed)
    noise = rng.integers(-24, 25, grey.shape[-2:] + (3,), dtype=np.int16)
    return np.clip(grey[..., None].astype(np.int16) + noise, 0, 255).astype(np.uint8)


class IngestWorkload(bench.Workload):
    """bench.py's config-3 workload with a pinned BGR pool beside the grey one; step_device reads BGR when `colour` is set"""

    def __init__(self, B, NH, pool_bytes):
        super().__init__(3, B, NH, 0, 0, pool_bytes=pool_bytes)
        torch = self.torch
        self.bgr_host = torch.from_numpy(colour_pool(self.host_pool.numpy(), 1)).pin_memory()
        self.bgr_dev = self.bgr_host.cuda()
        self.colour = False

    def step_device(self, i, with_po=False, k=None, pb=None):
        if not self.colour:
            return super().step_device(i, with_po, k, pb)
        e = self.exs[i % self.NH if k is None else k]
        pb = i % self.pool_batches if pb is None else pb
        grey_call = e.extract_batch_device      # the step with the BGR batch of the same pool slot in place of the grey one
        e.extract_batch_device = lambda ptr, n, w, h: grey_call(self.bgr_dev[pb].data_ptr(), n, w, h, image_format="bgr", src_size=(w, h))
        try:
            return super().step_device(i, with_po, k, pb)
        finally:
            del e.extract_batch_device


def e2e_round(wl, steps, prepare, count):
    """count batches, one host thread, the handles in flight; prepare(i) returns the host images of batch i.  Returns (frames/s, host
    CPU s per frame)."""
    NH, P = wl.NH, wl.pool_batches
    submit = lambda i: steps[i % NH].submit(prepare(i), last=wl.P_LAST[i % P], local=wl.P_LOC[i % P])
    outs = [{k: v for k, v in o.items() if k not in ("pose", "inl", "eoff", "efeat", "outl")} for o in wl.OUT]
    wl.torch.cuda.synchronize()
    t0, c0 = time.perf_counter(), time.process_time()
    for j in range(min(NH - 1, count)):
        submit(j)
    for i in range(count):
        if i + NH - 1 < count:
            submit(i + NH - 1)
        steps[i % NH].collect(outs[i % NH])
    dt, dc = time.perf_counter() - t0, time.process_time() - c0
    return wl.B * count / dt, dc / (wl.B * count)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=bench.CONFIGS[3]["B"])
    ap.add_argument("--handles", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--pool-bytes", type=float, default=140e6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from orb_slam3_detailed_comments_b200.replay import TrackingStep
    wl = IngestWorkload(a.batch, a.handles, a.pool_bytes)
    torch, W, H, NH = wl.torch, wl.W, wl.H, wl.NH
    _, _, _, _, BF, BL = wl.cam_t
    wl.e2e_setup()
    mk = lambda **kw: [TrackingStep(e, wl.cam, BF, BL, bench.TH_LAST, bench.TH_LOCAL, 0.8, True, **kw) for e in wl.exs]
    grey_steps, bgr_steps = wl.steps_e2e, mk(image_format="bgr")
    big = (1280, 720)
    big_pool = [np.stack([cv2.resize(im, big, interpolation=cv2.INTER_LINEAR) for im in b]) for b in wl.bgr_host.numpy()[:2]]
    big_pool = [torch.from_numpy(b).pin_memory().numpy() for b in big_pool]
    rs_steps = mk(image_format="bgr", resize=(W, H))
    staging = [torch.zeros((wl.nimg, H, W), dtype=torch.uint8).pin_memory().numpy() for _ in range(NH)]   # one grey buffer per handle in flight
    bgr = wl.bgr_host.numpy()

    def host_cvt(i):
        out = staging[i % NH]
        for k, im in enumerate(bgr[i % wl.pool_batches]):
            cv2.cvtColor(im, cv2.COLOR_BGR2GRAY, dst=out[k])
        return out

    def host_resize_cvt(i):
        out = staging[i % NH]
        for k, im in enumerate(big_pool[i % 2]):
            cv2.cvtColor(cv2.resize(im, (W, H), interpolation=cv2.INTER_LINEAR), cv2.COLOR_BGR2GRAY, dst=out[k])
        return out

    legs = {"e2e_bgr_device": (bgr_steps, lambda i: bgr[i % wl.pool_batches]), "e2e_bgr_host_cv2": (grey_steps, host_cvt),
            "e2e_grey": (grey_steps, lambda i: wl.host_pool[i % wl.pool_batches].numpy()),
            "resize_1280x720_device": (rs_steps, lambda i: big_pool[i % 2]), "resize_1280x720_host_cv2": (grey_steps, host_resize_cvt)}
    # parity before timing: every leg's first batch gives what the grey step gives on cv2's grey images of the same frames
    want = {}
    for name, (steps, prep) in legs.items():
        ref = host_resize_cvt(0).copy() if name.startswith("resize") else host_cvt(0).copy()
        key = "resize" if name.startswith("resize") else "plain"
        if key not in want:
            grey_steps[0].submit(ref, last=wl.P_LAST[0], local=wl.P_LOC[0])
            o = {k: v.copy() for k, v in wl.OUT[0].items()}
            rows = grey_steps[0].collect(o)
            want[key] = (rows, o)
        if name == "e2e_grey":
            continue
        steps[0].submit(prep(0), last=wl.P_LAST[0], local=wl.P_LOC[0])
        got = {k: v.copy() for k, v in wl.OUT[0].items()}
        rows = steps[0].collect(got)
        wr, wo = want[key]
        assert rows == wr and all((got[k][:rows] == wo[k][:rows]).all() for k in ("desc", "fm", "ur")) and (got["mt"] == wo["mt"]).all(), name
        assert (got["kps"][:rows].view(np.uint8) == wo["kps"][:rows].view(np.uint8)).all(), name
    for name, (steps, prep) in legs.items():    # warm-up: every handle, every pool slot
        e2e_round(wl, steps, prep, 2 * NH)
    res = {name: [] for name in legs}
    for _ in range(a.repeats):
        for name, (steps, prep) in legs.items():
            fps, cpu = e2e_round(wl, steps, prep, a.steps)
            res[name].append({"frames_per_s": round(fps, 1), "host_cpu_ms_per_frame": round(1e3 * cpu, 4)})
    # resident graph replay, BGR vs grey input, alternating
    graph = {"grey": [], "bgr": []}
    nb = a.steps * NH
    for colour in (False, True):               # warm-up: captures every (handle, pool slot) graph
        wl.colour = colour
        wl.graphs_saved = getattr(wl, "graphs_saved", {})
        wl.graphs = wl.graphs_saved.setdefault(colour, {})
        wl.timed_device_loop(0, math.lcm(NH, wl.pool_batches), False, lambda: torch.cuda.synchronize())
    for _ in range(a.repeats):
        for colour in (False, True):
            wl.colour = colour
            wl.graphs = wl.graphs_saved[colour]
            ms = wl.timed_device_loop(0, nb, False, lambda: torch.cuda.synchronize())
            graph["bgr" if colour else "grey"].append(round(wl.B * nb / ms * 1e3, 1))
    for colour in (False, True):
        wl.graphs = wl.graphs_saved[colour]
        wl.close()
    line = {"card": card(), "workload": "config 3: 640x480 stereo, 1200 features, SearchByProjection(cur, last) + (F, local map)",
            "batch_frames": wl.B, "handles": NH, "steps": a.steps, "unit": "stereo frames/s",
            "h2d_image_bytes_per_frame": {"grey": 2 * W * H, "bgr": 2 * W * H * 3, "bgr_1280x720": 2 * 1280 * 720 * 3},
            "e2e": res, "graph_replay_frames_per_s": graph}
    s = json.dumps(line)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
