"""CPU tier: the CPU arm of tools/rgbd_bench.py (640x480 RGB-D, 1000 features).  The oracle's RGB-D frame gives most features a depth
and finds matches in both searches, and the script's command line parses without a GPU."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import rgbd_bench  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def test_oracle_rgbd_frame_has_depths_and_matches():
    _, greys, maps = rgbd_bench.make_frames(2)
    for i in range(2):
        r = rgbd_bench.oracle_rgbd_frame(greys[i], maps[i], po.OracleExtractor(rgbd_bench.NFEAT, 1.2, 8, 20, 7))
        n = len(r["k"])
        assert n > 800 and (r["dep"] > 0).sum() > 0.9 * n and (r["ur"][r["dep"] < 0] == -1).all()
        assert r["nm1"] == int((r["fm"] >= 0).sum()) and r["nm1"] > 300
        assert r["nm2"] == int((r["mt"] >= 0).sum()) and r["nm2"] > 300


def test_cpu_baseline_runs():
    _, greys, maps = rgbd_bench.make_frames(4)
    res = rgbd_bench.cpu_baseline(greys, maps)
    assert res["value"] > 0 and res["frames"] == 4


def test_rgbd_bench_help_runs():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "rgbd_bench.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "--batch" in r.stdout
