"""CPU tier: the machine code of lib/liborbslam3_b200_ingest.so (k_ingest, csrc/ingest.cu) is the build whose GPU tier
(tests/test_zz_ingest_gpu.py) was green on an H100, as tests/test_sass_fingerprint.py holds the main library to its own golden file:
tests/golden/ingest_sass_fingerprint.json, taken with scripts/sass_fingerprint.py.  k_ingest also keeps out of local memory."""
import importlib.util
import json
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not available")


@pytest.fixture(scope="module")
def lib():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    return N.INGEST_LIB_PATH


def test_k_ingest_is_the_gpu_validated_build(lib):
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "ingest_sass_fingerprint.json")))
    assert {k: list(v) for k, v in mod.fingerprints(lib).items()} == ref


def test_k_ingest_uses_no_local_memory(lib):
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    assert "k_ingest" in sass and "STL" not in sass and "LDL" not in sass
