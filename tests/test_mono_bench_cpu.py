"""CPU tier: the CPU arm of tools/mono_bench.py (config 2, monocular 752x480).  The oracle's monocular frame finds matches in both
searches; where oracle/_ref is built, the reference's own source gives the same match counts on the same frames (the arm reports the
faster of the two, so they must do the same work); and the script's command line parses without a GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import mono_bench  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

needs_reference = pytest.mark.skipif(not bench.reference_source_available(), reason="oracle/_ref is not built and the reference is absent")


def test_oracle_mono_frame_back_fills_and_matches():
    imgs, disps = mono_bench.make_frames(2)
    for i in range(2):
        r = mono_bench.oracle_mono_frame(imgs[i], disps[i], po.OracleExtractor(mono_bench.NFEAT, 1.2, 8, 20, 7))
        assert r["mono"] == 0 and len(r["k"]) > 1000              # 752 px < 1000: every keypoint is back-filled
        assert r["nm1"] == int((r["fm"] >= 0).sum()) and r["nm1"] > 300
        assert r["nm2"] == int((r["mt"] >= 0).sum()) and r["nm2"] > 300


@needs_reference
def test_reference_source_mono_frame_equals_the_oracle_frame():
    imgs, disps = mono_bench.make_frames(2)
    for i in range(2):
        o = mono_bench.oracle_mono_frame(imgs[i], disps[i], po.OracleExtractor(mono_bench.NFEAT, 1.2, 8, 20, 7))
        nm1, nm2 = mono_bench.reference_mono_frame(imgs[i], disps[i], po.RefExtractor(mono_bench.NFEAT, 1.2, 8, 20, 7))
        assert (nm1, nm2) == (o["nm1"], o["nm2"]) and nm1 + nm2 > 600


def test_mono_bench_help_runs():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "mono_bench.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "--batch" in r.stdout
