"""CPU tier: the machine code the library ships is the machine code whose `pytest -m gpu` run was green on an H100.
tests/golden/sass_fingerprints.json is taken (scripts/sass_fingerprint.py) from the sm_90a build that last passed the whole GPU tier
(every kernel has had a device run: UNPROVEN is empty).  An intentional kernel change must come with a GPU run and a
refreshed fingerprint file; an unintentional one (a shared header edit that changes another kernel's code) fails here first.
Next to the fingerprints, the properties a few kernels were built for are checked in their own SASS: both passes of the tensor-core
blur run as u8 IMMA, and the 64-bit quadtree, the camera-image and RGB-D depth stages and the matcher's global-memory form keep to their
GPU-validated local-memory use."""
import importlib.util
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNPROVEN = ()
# local-memory loads + stores (STL / LDL) of the GPU-validated builds
XL_CAND_LOCAL, XL_RESOLVE_LOCAL = 17, 17          # k_proj_candidates_xl, k_proj_resolve_xl
TWIN_CAND_LOCAL, TWIN_RESOLVE_LOCAL = 17, 19      # their shared-memory twins k_proj_candidates, k_proj_resolve
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not available")


@pytest.fixture(scope="module")
def lib():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    return N.LIB_PATH


@pytest.fixture(scope="module")
def ops(lib):
    """kernel name -> the opcodes of its SASS, in order"""
    out, name = {}, None
    for line in subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and name:
            out[name].append(m.group(1))
    return out


def local_ops(kernel_ops):
    return sum(op.startswith(("STL", "LDL")) for op in kernel_ops)


def test_every_kernel_is_the_gpu_validated_build(lib):
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    now = mod.fingerprints(lib)
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_fingerprints.json")))
    proven = {k: v for k, v in ref.items() if not any(u in k for u in UNPROVEN)}
    assert len(proven) >= 24
    for k, v in proven.items():
        assert k in now, f"{k} disappeared from the library"
        assert list(now[k]) == list(v), f"{k}: machine code differs from the GPU-validated build"
    extra = [k for k in now if k not in proven]
    assert all(any(u in k for u in UNPROVEN) for k in extra), extra


def test_both_passes_are_imma_and_nothing_spills(ops):
    k = ops["_ZN3orb10k_blur_mmaENS_11ExtractGeomENS_11BlurMmaPlanE"]
    assert sum(op.startswith("IMMA.16832.U8.U8") for op in k) >= 6          # one step: 2 pass-H + 4 pass-V
    assert local_ops(k) == 0


def test_k64_quadtree_uses_no_local_memory(ops):
    """k_quadtree_v1_k64's 64-bit sort network stays in registers"""
    k = ops["_ZN3orb17k_quadtree_v1_k64ILi512ELi1EEEvNS_11ExtractGeomEiiPKjPKiPjPcliiiS6_PiS8_"]
    assert any(op.startswith("BAR.SYNC") for op in k)
    assert local_ops(k) == 0


def test_k_ingest_uses_no_local_memory(ops):
    assert local_ops(ops["_ZN3orb8k_ingestEN6orbdev10IngestPlanE"]) == 0


def test_k_stereo_rgbd_uses_no_local_memory(ops):
    assert local_ops(ops["_ZN3orb13k_stereo_rgbdEN6orbdev8RgbdPlanE"]) == 0


def test_global_form_adds_no_local_memory(ops):
    """The staging, grouped-candidate and parallel-resolve kernels of the matcher's global-memory form use no local memory;
    k_proj_candidates_xl and k_proj_resolve_xl keep the stored-candidate arrays of their shared bodies (matcher_core.cuh) in a
    256-byte stack frame, as their shared-memory twins do: pinned at exactly the GPU-validated counts, next to the twins' own."""
    xl = [k for k in ops if "k_stage_frames_xl" in k or "k_proj_candidates_grp_xl" in k or "k_proj_resolve_par_xl" in k]
    assert len(xl) == 5, xl
    for k in xl:
        assert local_ops(ops[k]) == 0, k
    pinned = {"_ZN3orb20k_proj_candidates_xlENS_10ProjParamsENS_11GlobalFrameE": XL_CAND_LOCAL,
              "_ZN3orb17k_proj_resolve_xlENS_10ProjParamsENS_11GlobalFrameE": XL_RESOLVE_LOCAL,
              "_ZN3orb17k_proj_candidatesENS_10ProjParamsE": TWIN_CAND_LOCAL,
              "_ZN3orb14k_proj_resolveENS_10ProjParamsE": TWIN_RESOLVE_LOCAL}
    for k, n in pinned.items():
        assert local_ops(ops[k]) == n, (k, local_ops(ops[k]), n)
