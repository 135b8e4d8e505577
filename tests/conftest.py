import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: exhaustive CPU checks (still part of the CPU tier)")


@pytest.fixture(autouse=True)
def _device_stereo_form(request):
    """The GPU tier compares the optimiser kernels with the oracle evaluating the stereo projection the way the kernels do
    (oracle/lba_oracle.cpp g_stereo_form = 1: float(z) before a float division, double products) -- the arithmetic they were validated with,
    to 1e-9 on chi2 and on equal LM iteration / trial counts.  The oracle's default form is the reference's, bit for bit
    (tests/test_oracle_vs_ref_edges.py), and the same file bounds the distance between the two forms on the GPU tier's own problems
    (poses < 1e-6, points < 1e-4, same iterations and outlier flags).  The CPU tier runs in the reference's form."""
    if request.node.get_closest_marker("gpu") is None:
        yield
        return
    from oracle import pyoracle as po
    prev = po.set_stereo_form(1)
    try:
        yield
    finally:
        po.set_stereo_form(prev)
