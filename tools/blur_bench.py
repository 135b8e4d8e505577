"""Blur stage A/B: k_blur<true> (ORB_BLUR_VARIANT=1) against k_blur_mma (2, the default) in one process, on the benchmark's
geometry (128 images of 640x480 per batch, seeded synthetic frames) and on the config-5 shape (32 images of 1280x720).

Both handles extract the same device-resident batch; the blur stage time is the handle's own stage events (set_profiling /
last_timings()["blur"], averaged over its ring of the last 32 batches).  Rounds alternate between the variants.  Prints ms per
batch, the algorithmic bandwidth (every level read once and its blurred copy written once) against the data sheet's 3.35 TB/s,
the outputs' equality, and the card's name, power limit and maximum SM clock (read-only nvidia-smi query).

    python tools/blur_bench.py [--rounds 8] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from orb_slam3_detailed_comments_b200 import ORBextractor, synth  # noqa: E402

RING = 32            # orbx_handle::kProfRing: last_timings() averages this many batches
HBM_TBS = 3.35       # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the numbers are still worth printing without it
        return {"error": repr(e)}


def run_shape(w, h, B, nf, rounds):
    imgs = synth.frame_batch(B, w, h, seed=11)
    dev = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    ex = {}
    for v in ("1", "2"):
        os.environ["ORB_BLUR_VARIANT"] = v    # read by orbx_create
        ex[v] = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
        ex[v].set_profiling(True)
    os.environ.pop("ORB_BLUR_VARIANT")
    levels = [ex["2"].level_size(l) for l in range(ex["2"].nlevels)]
    nbytes = 2 * B * sum(lw * lh for lw, lh in levels)
    for v in ex:                                   # warm-up: module load, first launches, the whole profiling ring
        for _ in range(RING):
            ex[v].extract_batch_device(dev.data_ptr(), B, w, h)
    torch.cuda.synchronize()
    ms = {v: [] for v in ex}
    for _ in range(rounds):
        for v in ex:
            for _ in range(RING):
                ex[v].extract_batch_device(dev.data_ptr(), B, w, h)
            ms[v].append(ex[v].last_timings()["blur"])
    same = all((ex["1"].image_pyramid(b, l, blurred=True) == ex["2"].image_pyramid(b, l, blurred=True)).all()
               for b in (0, B - 1) for l in range(len(levels)))
    out = {"shape": f"{B}x{w}x{h}", "batches_per_variant": rounds * RING, "algorithmic_bytes_per_batch": nbytes,
           "blurred_levels_identical": bool(same)}
    for v, name in (("1", "k_blur<true>"), ("2", "k_blur_mma")):
        m = float(np.median(ms[v]))
        out[name] = {"ms_per_batch_median": m, "ms_per_round": [round(x, 4) for x in ms[v]], "GB_per_s": nbytes / (m * 1e-3) / 1e9,
                     "share_of_3.35TB_per_s": nbytes / (m * 1e-3) / (HBM_TBS * 1e12)}
    for e in ex.values():
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8, help="alternating rounds of 32 batches per variant")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0),
           "shapes": [run_shape(640, 480, 128, 1200, a.rounds), run_shape(1280, 720, 32, 2000, a.rounds)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
