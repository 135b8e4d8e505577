"""GPU tier: k_liba (csrc/liba.cu) against the oracle on the windows of tests/test_liba_windows.py -- the reference's window sizes
(10 or 25 free keyframes, 200 fixed ones, points observed by up to 60 keyframes), its array order and the shapes host/
Optimizer_liba_b200.cc produces -- on every output the host unit reads (states, points, every edge's chi2 and depth flag, the
initial and last-trial chi2 of the failure rule), through every cluster size the launcher can pick, and the determinism DESIGN.md
§4.13 claims: the same window gives the same bits run after run and wherever it sits in a batch; only the cluster size may change
the order of the sums."""
import functools

import numpy as np
import pytest

from orb_slam3_detailed_comments_b200.optimizer import InertialOptimizer
from test_liba_windows import CASES, case, compare, oracle, settings, window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def opt():
    o = InertialOptimizer(0)
    yield o
    o.close()


@functools.lru_cache(maxsize=None)
def ref(name):
    pr = case(name)
    return oracle(pr, *settings(pr))


def _same_bits(a, b):
    for k in ("state", "point", "edge_chi2", "link_chi2", "edge_depth_pos"):
        assert a[k].tobytes() == b[k].tobytes(), k
    for k in ("iterations", "trials", "chi2", "chi2_init", "chi2_last", "lambda_"):
        assert np.float64(a[k]).tobytes() == np.float64(b[k]).tobytes(), (k, a[k], b[k])


# ---- 1. every window of the CPU tier: the reference's sizes, its array order and the shapes the host unit produces
@pytest.mark.parametrize("name", list(CASES))
def test_window_matches_oracle(opt, monkeypatch, name):
    monkeypatch.delenv("ORB_LIBA_CLUSTER", raising=False)
    pr = case(name)
    print(name, compare(opt.LocalInertialBA(pr, *settings(pr)), ref(name), pr))


# ---- 2. every cluster size on the reference's two window sizes (ORB_LIBA_CLUSTER caps the launcher's choice; read at every call)
@pytest.mark.parametrize("cluster", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("name", ["10free_200fixed", "25free_200fixed"])
def test_every_cluster_size(opt, monkeypatch, name, cluster):
    monkeypatch.setenv("ORB_LIBA_CLUSTER", str(cluster))
    pr = case(name)
    print(name, cluster, compare(opt.LocalInertialBA(pr, *settings(pr)), ref(name), pr))


# ---- 3. batches whose size selects each branch of the ladder (common.cuh cluster_size_for: 16 CTAs per window for <= 2 windows,
# then 8 / 4 / 2 while every cluster fits the SMs at once, then 1)
def _branches():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return [(2, 16), (3, 8), (sms // 8 + 1, 4), (sms // 4 + 1, 2), (sms // 2 + 1, 1)]


@functools.lru_cache(maxsize=None)
def _small_windows(n):
    """n small varied windows (1-6 free keyframes, 2-11 covisible ones, 80-250 points; the shapes of test_liba_windows.window by
    turns); the largest batch also holds the 10 + 200 window."""
    rng = np.random.default_rng(n)
    prs = []
    for i in range(n):
        n_free = int(rng.integers(1, 7))
        kw = dict(n_free=n_free, n_cov=int(rng.integers(2, 12)), n_mp=int(rng.integers(80, 251)), seed=20000 + 100 * n + i, max_obs=20)
        flag = ["shuffle", "links_only_kf", "unlinked_kf", "single_mono_points", "single_stereo_points", "rec_init", "early_map",
                None][i % 8]
        if flag in ("single_mono_points", "single_stereo_points"):
            kw[flag] = 10
        elif flag == "early_map":
            kw.update(n_free=min(n_free, 2), early_map=True)
        elif flag and (n_free >= 3 or flag in ("shuffle", "rec_init")):
            kw[flag] = True
        prs.append(window(**kw))
    if n == _branches()[-1][0]:
        prs[n // 3] = case("10free_200fixed")
    return prs


@pytest.mark.parametrize("branch", range(5))
def test_batch_sizes_select_every_cluster_size(opt, monkeypatch, branch):
    monkeypatch.delenv("ORB_LIBA_CLUSTER", raising=False)
    size, _ = _branches()[branch]
    prs = _small_windows(size)
    assert len(prs) == size
    worst = {}
    for i, (pr, g) in enumerate(zip(prs, opt.LocalInertialBABatch(prs, 1.0, 10))):
        for k, v in compare(g, oracle(pr, 1.0, 10), pr).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(size, worst)


# ---- 4. determinism and batch independence, bit for bit: a window solved alone at cluster size c, solved again, and solved first,
# in the middle and last of a batch whose size makes the launcher choose c
@pytest.mark.parametrize("branch", range(5))
def test_bits_do_not_depend_on_run_or_batch(opt, monkeypatch, branch):
    size, cs = _branches()[branch]
    name = "10free_40fixed"
    pr = case(name)
    lam, iters = settings(pr)
    monkeypatch.setenv("ORB_LIBA_CLUSTER", str(cs))
    alone = opt.LocalInertialBA(pr, lam, iters)
    _same_bits(alone, opt.LocalInertialBA(pr, lam, iters))
    compare(alone, ref(name), pr)
    monkeypatch.delenv("ORB_LIBA_CLUSTER")
    others = _small_windows(size)
    for pos in sorted({0, size // 2, size - 1}):
        prs = list(others)
        prs[pos] = pr
        _same_bits(alone, opt.LocalInertialBABatch(prs, lam, iters)[pos])
