"""CPU tier: the machine code of liborbslam3_b200_match_xl.so -- the matcher searches in their global-memory form, for frames whose
shared-memory form does not fit a CTA -- is the machine code whose `pytest -m gpu` run was green on an H100
(tests/golden/match_xl_sass_fingerprint.json, taken with scripts/sass_fingerprint.py from that build).  Local memory: the staging,
grouped-candidate and parallel-resolve kernels use none; k_proj_candidates_xl and k_proj_resolve_xl keep the stored-candidate arrays of
their shared bodies (matcher_core.cuh) in a 256-byte stack frame, as their shared-memory twins k_proj_candidates / k_proj_resolve of
liborbslam3_b200.so do: pinned at exactly the GPU-validated counts of local loads and stores, next to the twins' own counts."""
import importlib.util
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# local-memory loads + stores (STL / LDL) of the GPU-validated builds
XL_CAND_LOCAL, XL_RESOLVE_LOCAL = 17, 17          # k_proj_candidates_xl, k_proj_resolve_xl
TWIN_CAND_LOCAL, TWIN_RESOLVE_LOCAL = 17, 19      # k_proj_candidates, k_proj_resolve (liborbslam3_b200.so)
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not available")


@pytest.fixture(scope="module")
def libs():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    return N.MATCH_XL_LIB_PATH, N.LIB_PATH


def local_ops(lib):
    """kernel name -> number of local-memory loads and stores in its SASS"""
    out, name = {}, None
    for line in subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = 0
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and name and m.group(1).startswith(("STL", "LDL")):
            out[name] += 1
    return out


def test_match_xl_library_is_the_gpu_validated_build(libs):
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "match_xl_sass_fingerprint.json")))
    now = mod.fingerprints(libs[0])
    assert sorted(now) == sorted(ref)
    for k, v in ref.items():
        assert list(now[k]) == list(v), f"{k}: machine code differs from the GPU-validated build"


def test_global_form_adds_no_local_memory(libs):
    xl, main = local_ops(libs[0]), local_ops(libs[1])
    for k, n in xl.items():
        if "k_stage_frames_xl" in k or "k_proj_candidates_grp_xl" in k or "k_proj_resolve_par_xl" in k:
            assert n == 0, k
    pinned = {"_ZN3orb20k_proj_candidates_xlENS_10ProjParamsENS_11GlobalFrameE": XL_CAND_LOCAL,
              "_ZN3orb17k_proj_resolve_xlENS_10ProjParamsENS_11GlobalFrameE": XL_RESOLVE_LOCAL}
    twins = {"_ZN3orb17k_proj_candidatesENS_10ProjParamsE": TWIN_CAND_LOCAL, "_ZN3orb14k_proj_resolveENS_10ProjParamsE": TWIN_RESOLVE_LOCAL}
    for k, n in list(pinned.items()) + list(twins.items()):
        assert (xl.get(k) if k in xl else main[k]) == n, (k, xl.get(k, main.get(k)), n)
