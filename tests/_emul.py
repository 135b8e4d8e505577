"""Builds tests/host_emul/libemul.so: the kernels' per-element math and SPMD cores compiled for the HOST (g++), so the CPU test
tier can check device algorithms against the oracle without a GPU."""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))


def build_and_load():
    d = os.path.join(HERE, "host_emul")
    so = os.path.join(d, "libemul.so")
    csrc = os.path.join(HERE, "..", "orb_slam3_detailed_comments_b200", "csrc")
    srcs = [os.path.join(d, "emul.cpp"), os.path.join(csrc, "devmath.cuh"), os.path.join(csrc, "liba_core.cuh"),
            os.path.join(csrc, "liba_pack.h"), os.path.join(csrc, "lba_pack.h"), os.path.join(csrc, "pack.h"), os.path.join(csrc, "quadtree_core.cuh"), os.path.join(csrc, "quadtree_sort_par.cuh"),
            os.path.join(csrc, "stereo_core.cuh"), os.path.join(csrc, "resize_core.cuh"), os.path.join(HERE, "..", "include", "orbslam3_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so, srcs[0], "-lpthread"])
    return C.CDLL(so)
