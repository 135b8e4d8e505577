"""CPU tier: the kernel's sorted-path quadtree (csrc/quadtree_core.cuh compiled for the host) against the
oracle's std::list / std::sort restatement of DistributeOctTree, on real FAST candidates and on adversarial
point sets (ties in score, clusters, near-empty levels, two root nodes)."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emul():
    d = os.path.join(HERE, "host_emul")
    so = os.path.join(d, "libemul.so")
    csrc = os.path.join(HERE, "..", "orb_slam3_detailed_comments_b200", "csrc")
    srcs = [os.path.join(d, "emul.cpp"), os.path.join(csrc, "devmath.cuh"), os.path.join(csrc, "quadtree_core.cuh"),
            os.path.join(csrc, "quadtree_sort_par.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so, srcs[0], "-lpthread"])
    L = C.CDLL(so)
    for f in (L.emul_distribute, L.emul_distribute_v1):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_int] + [C.c_int] * 6 + [C.c_void_p, C.c_int]
    L.emul_bitonic.restype = None
    L.emul_bitonic.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.emul_sort_items.restype = None
    L.emul_sort_items.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return L


def cell_geom(w, h):
    width, height = np.float32(w - 32), np.float32(h - 32)
    nCols, nRows = int(width / np.float32(35)), int(height / np.float32(35))
    return int(math.ceil(width / nCols)), int(math.ceil(height / nRows)), nCols


def run(emul, c, W, H, N):
    """Both variants of the ordered phase's sort (one thread / spread over the CTA) must give the same list."""
    wC, hC, nC = cell_geom(W, H)
    c = np.ascontiguousarray(c, np.int32)
    outs = []
    for fn in (emul.emul_distribute, emul.emul_distribute_v1):
        out = np.zeros((N + 32, 3), np.int32)
        S = fn(c.ctypes.data, len(c), W - 32, H - 32, N, wC, hC, nC, out.ctypes.data, len(out))
        assert S >= 0, "workspace capacity (N + 20 nodes) exceeded"
        outs.append(out[:S])
    assert outs[0].shape == outs[1].shape and (outs[0] == outs[1]).all(), "variant 1 differs from variant 0"
    return outs[0]


@pytest.mark.parametrize("w,h,seed,sigma,nrect,nf", [(640, 480, 1, 1.5, 60, 1200), (640, 480, 2, 6.0, 10, 1200),
                                                      (752, 480, 3, 1.5, 60, 1200), (1280, 720, 5, 1.5, 60, 2000),
                                                      (640, 480, 6, 1.5, 60, 300), (640, 480, 7, 1.5, 60, 5000)])
def test_real_candidates(emul, w, h, seed, sigma, nrect, nf):
    ex = po.OracleExtractor(nf, 1.2, 8, 20, 7)
    ex(synth.frame(w, h, seed, sigma, nrect))
    for l in range(8):
        c = ex.level_cands(l)
        W, H = ex.level_size(l)
        N = int(ex.features_per_level[l])
        ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
        got = run(emul, c, W, H, N)
        assert len(got) == len(ref) and (got == c[ref]).all(), (seed, l)
        assert len(got) <= N + 3 or len(got) <= 16     # the capacity argument of quadtree_core.cuh


def _grid_order(pts, W, H):
    # candidates must arrive in the reference order: cell row, cell column, then row-major inside the cell
    wC, hC, nC = cell_geom(W, H)
    p64 = pts.astype(np.int64)
    key = ((p64[:, 1] - 3) // hC * nC + (p64[:, 0] - 3) // wC) * (1 << 24) + p64[:, 1] * 4096 + p64[:, 0]
    return pts[np.argsort(key, kind="stable")]


@pytest.mark.parametrize("case", range(12))
def test_adversarial_point_sets(emul, case):
    rng = np.random.default_rng(100 + case)
    W, H = [(640, 480), (752, 480), (309, 231), (1280, 720)][case % 4]
    rw, rh = W - 32, H - 32
    n = [5, 40, 300, 3000, 9000, 1][case % 6]
    if case % 3 == 0:      # uniform
        xy = np.stack([rng.integers(3, rw - 3, n), rng.integers(3, rh - 3, n)], 1)
    elif case % 3 == 1:    # a few tight clusters
        ctr = np.stack([rng.integers(20, rw - 20, 4), rng.integers(20, rh - 20, 4)], 1)
        xy = ctr[rng.integers(0, 4, n)] + rng.integers(-15, 16, (n, 2))
    else:                  # a line along the root boundary + a corner blob
        xy = np.concatenate([np.stack([np.full(n // 2, rw // 2), rng.integers(3, rh - 3, n // 2)], 1),
                             np.stack([rng.integers(3, 40, n - n // 2), rng.integers(3, 40, n - n // 2)], 1)])
    xy = np.clip(xy, 3, [rw - 4, rh - 4])
    xy = np.unique(xy, axis=0)                       # FAST keypoints are distinct pixels
    score = rng.integers(7, 12 if case % 2 else 200, len(xy))     # few distinct scores => many ties
    c = _grid_order(np.concatenate([xy, score[:, None]], 1).astype(np.int32), W, H)
    for N in [1, 7, 60, 261]:
        ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
        got = run(emul, c, W, H, N)
        assert len(got) == len(ref) and (got == c[ref]).all(), (case, N)


def _sort_three_ways(emul, items):
    items = np.ascontiguousarray(items, np.uint32)
    outs = []
    for which in (0, 1, 2):
        o = np.zeros(len(items), np.uint32)
        emul.emul_sort_items(items.ctypes.data, len(items), which, o.ctypes.data)
        outs.append(o)
    return outs


@pytest.mark.parametrize("n", [1, 2, 3, 15, 16, 17, 18, 33, 64, 100, 257, 300, 777, 2000])
def test_parallel_std_sort_is_libstdcxx_move_for_move(emul, n):
    """std::sort(vSizeAndPointerToNode, compareNodes): the payload order of tied keys is part of the result.  libstdc++ itself,
    the one-thread transcription and the CTA-parallel restructuring must agree on every payload -- on heavy ties, sorted and
    reversed inputs, organ pipes, few distinct keys, and the median-of-3 killer that drives introsort into its heap-sort fallback."""
    rng = np.random.default_rng(n)
    idx = np.arange(n, dtype=np.uint32)
    cases = []
    for kc, kx in [(3, 2), (10, 30), (1, 1), (1000, 600), (2, 50)]:
        cases.append(np.stack([rng.integers(2, 2 + kc, n), rng.integers(0, kx, n), idx], 1))
    asc = np.stack([idx // 3, idx % 2, idx], 1)
    cases += [asc, asc[::-1].copy(), np.stack([np.minimum(idx, n - 1 - idx), np.zeros(n, np.uint32), idx], 1)]
    if n >= 64:        # Musser's median-of-3 killer: quicksort degenerates, the depth limit is hit -> __partial_sort (heap sort)
        k = n // 2 * 2
        h = k // 2
        a = np.zeros(k, np.uint32)
        for i in range(h):
            a[i] = i + 1 if i % 2 == 0 else h + i + (1 if h % 2 else 0)
            a[h + i] = 2 * (i + 1)
        cases.append(np.stack([a, np.zeros(k, np.uint32), np.arange(k, dtype=np.uint32)], 1))
        cases.append(np.stack([a // 4, a % 3, np.arange(k, dtype=np.uint32)], 1))      # the same shape with ties
    for c in cases:
        c = c.copy()
        c[:, 2] = np.arange(len(c))
        ref, one, par = _sort_three_ways(emul, c)
        assert (one == ref).all() and (par == ref).all()
        key = c[ref, 0].astype(np.int64) * 65536 + c[ref, 1]
        assert (np.diff(key) >= 0).all()


# ---- the same source run by T host threads with a real barrier under ThreadSanitizer ---------------------------------------------
@pytest.fixture(scope="module")
def qt_mt():
    d = os.path.join(HERE, "host_emul")
    exe = os.path.join(d, "qt_mt_tsan")
    csrc = os.path.join(HERE, "..", "orb_slam3_detailed_comments_b200", "csrc")
    srcs = [os.path.join(d, "qt_mt.cpp"), os.path.join(csrc, "devmath.cuh"), os.path.join(csrc, "quadtree_core.cuh"),
            os.path.join(csrc, "quadtree_sort_par.cuh")]
    if not os.path.exists(exe) or any(os.path.getmtime(s) > os.path.getmtime(exe) for s in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-fsanitize=thread", "-ffp-contract=off", "-std=c++20", "-o", exe, srcs[0], "-lpthread"])
    return exe


def run_mt(exe, c, W, H, N, variant, threads, tmp_path):
    wC, hC, nC = cell_geom(W, H)
    c = np.ascontiguousarray(c, np.int32)
    fin, fout = tmp_path / "c.bin", tmp_path / "o.bin"
    fin.write_bytes(np.array([len(c), W - 32, H - 32, N, wC, hC, nC, variant], np.int32).tobytes() + c.tobytes())
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66")
    pr = subprocess.run([exe, str(fin), str(fout), str(threads)], env=env, capture_output=True, text=True, timeout=600)
    assert pr.returncode == 0, "ThreadSanitizer / driver failure (%d):\n%s" % (pr.returncode, pr.stderr[-4000:])
    o = np.frombuffer(fout.read_bytes(), np.int32)
    return o[1:].reshape(-1, 3)[:o[0]]


@pytest.mark.parametrize("variant,threads", [(0, 3), (0, 8), (1, 3), (1, 8), (1, 32), (1, 64)])     # variant 1 also runs 1024-thread CTAs
def test_threaded_quadtree_is_race_free_and_matches_oracle(qt_mt, tmp_path, variant, threads):
    """Real FAST candidates of a 640x480 frame, all 8 levels: T threads + a real barrier + ThreadSanitizer.  Variant 0 is the kernel
    that ran green on the GPU tier (so this also says the harness agrees with the device about where barriers are needed);
    variant 1 is the CTA-parallel ordered-phase sort."""
    ex = po.OracleExtractor(1200, 1.2, 8, 20, 7)
    ex(synth.frame(640, 480, 1))
    for l in range(8):
        c = ex.level_cands(l)
        W, H = ex.level_size(l)
        N = int(ex.features_per_level[l])
        ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
        got = run_mt(qt_mt, c, W, H, N, variant, threads, tmp_path)
        assert len(got) == len(ref) and (got == c[ref]).all(), (variant, threads, l)


@pytest.mark.parametrize("case", [1, 2, 4, 8])
def test_threaded_quadtree_on_adversarial_sets(qt_mt, tmp_path, case):
    rng = np.random.default_rng(300 + case)
    W, H = 640, 480
    n = 400 * case
    ctr = np.stack([rng.integers(20, W - 52, 5), rng.integers(20, H - 52, 5)], 1)
    xy = np.unique(np.clip(ctr[rng.integers(0, 5, n)] + rng.integers(-25, 26, (n, 2)), 3, [W - 36, H - 36]), axis=0)
    c = _grid_order(np.concatenate([xy, rng.integers(7, 10, len(xy))[:, None]], 1).astype(np.int32), W, H)
    for N in (60, 261):
        ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
        got = run_mt(qt_mt, c, W, H, N, 1, 6, tmp_path)
        assert len(got) == len(ref) and (got == c[ref]).all(), (case, N)


@pytest.mark.parametrize("npow", [2, 4, 8, 16, 32, 64, 512, 1024, 4096, 8192, 16384])
def test_multi_stage_bitonic_sorts(emul, npow):
    rng = np.random.default_rng(npow)
    for trial in range(3):
        a = rng.integers(0, 1 << 32, npow, dtype=np.uint64).astype(np.uint32)
        if trial == 1:
            a[rng.integers(0, npow, npow // 3 + 1)] = 0xffffffff        # padding sentinels as in the kernel
        if trial == 2:
            a = np.sort(a)[::-1].copy()
        b0, b1, b2 = a.copy(), a.copy(), a.copy()
        emul.emul_bitonic(b0.ctypes.data, npow, 0)
        emul.emul_bitonic(b1.ctypes.data, npow, 1)      # two stages per pass
        emul.emul_bitonic(b2.ctypes.data, npow, 2)      # three stages per pass (the one k_quadtree_v1 uses)
        assert (b0 == np.sort(a)).all() and (b1 == b0).all() and (b2 == b0).all()


def test_parallel_std_sort_fuzz(emul):
    """hypothesis: random lengths and key ranges (dense ties to distinct keys) -- libstdc++ std::sort, the one-thread transcription and
    the CTA-parallel form agree on the full payload order every time."""
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=150, deadline=None)
    @given(st.integers(0, 700), st.integers(1, 40), st.integers(1, 300), st.integers(0, 2 ** 31 - 1), st.booleans())
    def run(n, kc, kx, seed, presorted):
        rng = np.random.default_rng(seed)
        c = np.stack([rng.integers(2, 2 + kc, n), rng.integers(0, kx, n), np.arange(n)], 1).astype(np.uint32).reshape(n, 3)
        if presorted and n:
            c = c[np.lexsort((c[:, 1], c[:, 0]))]
            c[:, 2] = np.arange(n)
        if n == 0:
            return
        ref, one, par = _sort_three_ways(emul, c)
        assert (one == ref).all() and (par == ref).all()
    run()
