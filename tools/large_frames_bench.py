"""Stereo extraction at 1920x1080 and 3840x2160: frames/s of the resident CUDA-graph replay (extraction of both eyes +
ComputeStereoMatches, images already in HBM) and of the host-to-host orbr_submit / orbr_collect path, the handle's per-stage
milliseconds, the quadtree stage split by kernel (k_quadtree_v1_k64 for the levels whose region exceeds 2048 px, k_quadtree_v1 for the
others; torch.profiler kernel times), and the handle's device allocation at the batch used and at max_batch 128.  Seeded synthetic
stereo pairs, 2000 features, 8 levels.  Prints the card's name, power limit and maximum SM clock (read-only nvidia-smi query).

    python tools/large_frames_bench.py [--reps 20] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam3_detailed_comments_b200 import ORBextractor, camera, synth  # noqa: E402
from orb_slam3_detailed_comments_b200.replay import TrackingStep  # noqa: E402

NF = 2000
RING = 32            # orbx_handle::kProfRing: last_timings() averages this many batches


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:
        return {"error": repr(e)}


def allocation(w, h, B):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    ex.close()
    return int(used)


def run_shape(w, h, B, reps):
    s = w / 640.0
    fx, fy, cx, cy, bf, b = 435.2 * s, 435.2 * s, w / 2.0, h / 2.0, 47.9 * s, 0.11
    P = B // 2
    imgs = np.zeros((B, h, w), np.uint8)
    for p in range(P):
        imgs[2 * p], imgs[2 * p + 1], _ = synth.stereo_pair(w, h, seed=500 + p, dmin=2.0, dmax=0.5 * fx)
    out = {"shape": f"{B} images ({P} stereo frames) of {w}x{h}", "device_bytes_at_batch": allocation(w, h, B),
           "device_bytes_at_max_batch_128": allocation(w, h, 128)}
    ex = ORBextractor(NF, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
    dev = torch.from_numpy(imgs).cuda()
    torch.cuda.synchronize()

    def step():
        ex.extract_batch_device(dev.data_ptr(), B, w, h)
        ex.stereo_batch(P, bf, b)

    # per-stage milliseconds (the handle's stage events over its ring of batches)
    ex.set_profiling(True)
    for _ in range(2 * RING):
        ex.extract_batch_device(dev.data_ptr(), B, w, h)
    out["stage_ms_per_batch"] = {k: round(v, 4) for k, v in ex.last_timings().items()}
    ex.set_profiling(False)
    # the quadtree stage by kernel
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ex.extract_batch_device(dev.data_ptr(), B, w, h)
        torch.cuda.synchronize()
    qt = {}
    for e in prof.key_averages():
        if "k_quadtree" in e.key:
            form = "k_quadtree_v1_k64 (64-bit form)" if "k_quadtree_v1_k64" in e.key else "k_quadtree_v1 (32-bit form)"
            qt[form] = qt.get(form, 0.0) + e.device_time_total / 1000.0 / reps
    out["quadtree_ms_per_batch_by_form"] = {k: round(v, 4) for k, v in qt.items()}
    # resident graph replay
    step()
    g = ex.graph_capture(step)
    for _ in range(3):
        ex.graph_launch(g)
    torch.cuda.synchronize()
    st = torch.cuda.ExternalStream(int(ex.cuda_stream()))
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(st)
    for _ in range(reps):
        ex.graph_launch(g)
    t1.record(st)
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    ex.graph_destroy(g)
    out["graph_replay_ms_per_batch"] = round(ms, 4)
    out["graph_replay_stereo_frames_per_s"] = round(P / (ms * 1e-3), 1)
    # host buffers in, host buffers out: orbr_submit / orbr_collect
    ts = TrackingStep(ex, camera(fx, fy, cx, cy, bf, b, w, h), bf, b)
    cap = ex.max_features_per_image() * B
    pin = torch.from_numpy(imgs).pin_memory().numpy()
    o = {"kps": np.zeros(cap, [("f", "u1", 28)]), "desc": np.zeros((cap, 32), np.uint8), "ur": np.zeros(cap, np.float32),
         "dep": np.zeros(cap, np.float32), "n": np.zeros(B, np.int32), "offsets": np.zeros(B + 1, np.int32)}
    for _ in range(2):
        ts.submit(pin)
        ts.collect(o)
    t = time.perf_counter()
    for _ in range(reps):
        ts.submit(pin)
        ts.collect(o)
    dt = (time.perf_counter() - t) / reps
    out["e2e_ms_per_batch"] = round(dt * 1e3, 3)
    out["e2e_stereo_frames_per_s"] = round(P / dt, 1)
    ex.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0),
           "shapes": [run_shape(1920, 1080, 32, a.reps), run_shape(3840, 2160, 8, a.reps)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
