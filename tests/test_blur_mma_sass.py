"""CPU tier: the machine code of liborbslam3_b200_blur.so -- k_blur_mma, the tensor-core blur, in its own library next to
liborbslam3_b200.so -- is the machine code whose `pytest -m gpu` run was green on an H100 (tests/golden/blur_mma_sass_fingerprint.json,
taken with scripts/sass_fingerprint.py from that build), the library holds that one kernel, both passes run as u8 IMMA, and nothing
spills to local memory.  tests/test_sass_fingerprint.py keeps doing the same for every kernel of the main library."""
import importlib.util
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not available")


@pytest.fixture(scope="module")
def blur_lib():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    return N.BLUR_LIB_PATH


def test_blur_library_is_the_gpu_validated_build(blur_lib):
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "blur_mma_sass_fingerprint.json")))
    now = mod.fingerprints(blur_lib)
    assert sorted(now) == sorted(ref)
    for k, v in ref.items():
        assert list(now[k]) == list(v), f"{k}: machine code differs from the GPU-validated build"


def test_both_passes_are_imma_and_nothing_spills(blur_lib):
    sass = subprocess.run(["cuobjdump", "-sass", blur_lib], capture_output=True, text=True, check=True).stdout
    ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", sass)
    assert sum(op.startswith("IMMA.16832.U8.U8") for op in ops) >= 6          # one step: 2 pass-H + 4 pass-V
    assert not any(op.startswith(("STL", "LDL")) for op in ops)
