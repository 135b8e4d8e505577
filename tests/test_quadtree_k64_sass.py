"""CPU tier: the machine code of liborbslam3_b200_qt64.so -- k_quadtree_v1_k64, DistributeOctTree on the 64-bit, 12-depth element, in
its own library next to liborbslam3_b200.so -- is the machine code whose `pytest -m gpu` run was green on an H100
(tests/golden/quadtree_k64_sass_fingerprint.json, taken with scripts/sass_fingerprint.py from that build); the library holds that one
kernel, and its 64-bit sort network stays in registers: no local-memory load or store.  tests/test_sass_fingerprint.py keeps doing the
same for every kernel of the main library."""
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
def qt64_lib():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    return N.QT64_LIB_PATH


def test_qt64_library_is_the_gpu_validated_build(qt64_lib):
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "quadtree_k64_sass_fingerprint.json")))
    now = mod.fingerprints(qt64_lib)
    assert sorted(now) == sorted(ref)
    for k, v in ref.items():
        assert list(now[k]) == list(v), f"{k}: machine code differs from the GPU-validated build"


def test_k64_quadtree_uses_no_local_memory(qt64_lib):
    sass = subprocess.run(["cuobjdump", "-sass", qt64_lib], capture_output=True, text=True, check=True).stdout
    ops = re.findall(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", sass)
    assert any(op.startswith("BAR.SYNC") for op in ops)
    assert not any(op.startswith(("STL", "LDL")) for op in ops)
