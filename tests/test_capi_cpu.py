"""CPU tier: the C-ABI library builds for sm_90a, loads without a GPU, exports every symbol that
include/orbslam3_b200.h declares, and fails loudly (no CPU fallback) when asked to compute."""
import ctypes as C
import os
import re

import pytest

from orb_slam3_detailed_comments_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    N.build()
    return N.lib()


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "orbslam3_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    names = set(re.findall(r"\b((?:orb|orbx|orbm|orbo|orbf|orbv|orbp|orbr|lba|liba)_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_every_declared_symbol_is_exported(lib):
    names = _declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/orbslam3_b200.h but not exported"
    # and the Python binding table covers the header
    assert set(N.SIGNATURES) == set(names), set(names) ^ set(N.SIGNATURES)


def test_struct_layouts_match_the_header():
    assert N.KP_DTYPE.itemsize == 28            # cv::KeyPoint
    assert C.sizeof(N.orbx_config) == 36
    assert C.sizeof(N.orbm_camera) == 40
    assert N.LIBA_LINK.itemsize == 1080         # liba_link
    assert C.sizeof(N.liba_problem) == 16 + 8 * 8 + 12 * 8 + 6 * 8 + 8
    assert C.sizeof(N.liba_result) == 5 * 8 + 8 + 4 * 8


def test_no_device_means_loud_failure(lib):
    if lib.orb_device_count() > 0:
        pytest.skip("a GPU is present")
    h = C.c_void_p()
    cfg = N.orbx_config(1000, 1.2, 8, 20, 7, 640, 480, 1, 0)
    assert lib.orbx_create(C.byref(cfg), C.byref(h)) == -6          # ORB_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.orb_last_error()
    o = C.c_void_p()
    assert lib.lba_create(0, C.byref(o)) == -6
    assert lib.liba_create(0, C.byref(o)) == -6 and b"no CPU fallback" in lib.orb_last_error()


def test_bad_arguments_are_rejected_without_a_device(lib):
    h = C.c_void_p()
    assert lib.orbx_create(None, C.byref(h)) == -1
    bad = N.orbx_config(1000, 1.0, 8, 20, 7, 640, 480, 1, 0)       # scaleFactor must exceed 1
    assert lib.orbx_create(C.byref(bad), C.byref(h)) == -1
    assert lib.orbx_counts(None, None, None, None) == -1
    assert lib.liba_create(0, None) == -1 and lib.liba_solve(None, 1, None, None) == -1
    assert lib.liba_link_information(None, 0, None, None, None) == -1


def test_product_sources_never_touch_the_oracle():
    pkg = os.path.join(ROOT, "orb_slam3_detailed_comments_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "pyoracle" not in src and "liborb_oracle" not in src and "oracle/" not in src.replace("oracle/tools", ""), f


def test_ctypes_structs_have_the_size_the_header_gives_them(tmp_path):
    """Every struct that crosses the C ABI by pointer: sizeof in C (gcc on include/orbslam3_b200.h) == ctypes.sizeof of the binding."""
    import subprocess
    names = ["orbx_config", "orbm_camera", "orbm_local_queries", "orbm_last_queries", "orbm_bow_queries", "orbm_kf_queries", "orbo_pose_problems",
             "orbo_edge_source", "orbo_frame_matches", "orbf_frustum_points", "orbm_init_queries", "orbm_bow_kf_queries", "orbm_triangulation",
             "lba_problem", "lba_result", "liba_problem", "liba_result", "orbr_chain", "orbr_step", "orbr_results"]
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "orbslam3_b200.h"\nint main(void) {\n' +
                   "".join(f'    printf("{n} %zu\\n", sizeof({n}));\n' for n in names) + "    return 0;\n}\n")
    exe = tmp_path / "sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for n in names:
        assert int(got[n]) == C.sizeof(getattr(N, n)), (n, got[n], C.sizeof(getattr(N, n)))
