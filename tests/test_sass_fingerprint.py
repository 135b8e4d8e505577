"""CPU tier: the machine code the library ships is the machine code whose `pytest -m gpu` run was green on an H100.
tests/golden/sass_fingerprints.json is taken (scripts/sass_fingerprint.py) from the sm_90a build that last passed the whole GPU tier
(every kernel has had a device run: UNPROVEN is empty).  An intentional kernel change must come with a GPU run and a
refreshed fingerprint file; an unintentional one (a shared header edit that changes another kernel's code) fails here first."""
import importlib.util
import json
import os
import shutil

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNPROVEN = ()


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not available")
def test_validated_kernels_are_bit_identical():
    spec = importlib.util.spec_from_file_location("sass_fingerprint", os.path.join(ROOT, "scripts", "sass_fingerprint.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    now = mod.fingerprints()
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_fingerprints.json")))
    proven = {k: v for k, v in ref.items() if not any(u in k for u in UNPROVEN)}
    assert len(proven) >= 24
    for k, v in proven.items():
        assert k in now, f"{k} disappeared from the library"
        assert list(now[k]) == list(v), f"{k}: machine code differs from the GPU-validated build"
    extra = [k for k in now if k not in proven]
    assert all(any(u in k for u in UNPROVEN) for k in extra), extra
