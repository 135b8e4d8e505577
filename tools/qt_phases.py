#!/usr/bin/env python3
"""Phase clocks of k_quadtree_v1 (level-0 CTAs and the other levels apart) from the -DQT_PROFILE build of the library:

    nvcc ... -DQT_PROFILE -o orb_slam3_detailed_comments_b200/lib/liborbslam3_b200_qtprof.so   (tools/qt_phases.py --build)
    ORB_LIB_PATH=.../liborbslam3_b200_qtprof.so python tools/qt_phases.py [--sigma 1.5 --nrect 60]
"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PROF = os.path.join(ROOT, "orb_slam3_detailed_comments_b200", "lib", "liborbslam3_b200_qtprof.so")

if "--build" in sys.argv:
    from orb_slam3_detailed_comments_b200 import _native as N
    srcs = [os.path.join(N._CSRC, s) for s in N.SOURCES]
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + N.NVCC_FLAGS + ["-DQT_PROFILE", "-o", PROF] + srcs)
    print("built", PROF)
    sys.exit(0)

os.environ.setdefault("ORB_LIB_PATH", PROF)
import numpy as np
import torch
from orb_slam3_detailed_comments_b200 import ORBextractor, synth, _native as N

sigma = float(sys.argv[sys.argv.index("--sigma") + 1]) if "--sigma" in sys.argv else 1.5
nrect = int(sys.argv[sys.argv.index("--nrect") + 1]) if "--nrect" in sys.argv else 60
W, H, NB = 640, 480, 128
imgs = np.stack([synth.frame(W, H, seed=100 + (i % 8), sigma=sigma, nrect=nrect) for i in range(NB)])
ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=NB)
d = torch.from_numpy(imgs).cuda()
L = N.lib()
L.orbx_debug_qt_profile.argtypes = [C.c_void_p, C.c_int]
for _ in range(3):
    ex.extract_batch_device(d.data_ptr(), NB, W, H)
torch.cuda.synchronize()
L.orbx_debug_qt_profile(None, 1)
REP = 10
for _ in range(REP):
    ex.extract_batch_device(d.data_ptr(), NB, W, H)
out = np.zeros(32, np.int64)
L.orbx_debug_qt_profile(out.ctypes.data_as(C.c_void_p), 0)
names = ["element+pad", "bitonic sort", "roots", "sweeps", "ordered: std::sort", "ordered: split/scan/K", "ordered: scatter", "best per leaf"]
mhz = 1965.0
for base, tag, nct in ((0, "level 0 (1024-thread CTAs)", NB), (16, "levels 1-7 (256-thread CTAs)", 7 * NB)):
    tot = out[base:base + 8].sum()
    print(f"{tag}: {tot / (REP * nct) / mhz:.1f} us per CTA (sigma {sigma}, nrect {nrect})")
    for k, nm in enumerate(names):
        v = out[base + k] / (REP * nct)
        print(f"   {nm:24s} {v / 1e3:8.1f} kcycles  {v / mhz:7.1f} us  {100 * out[base + k] / max(tot, 1):5.1f} %")
