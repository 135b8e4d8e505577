"""CPU tier: DistributeOctTree's 64-bit, 12-depth sort element (csrc/quadtree_core.cuh QtForm<uint64_t>, the source of
k_quadtree_v1_k64) compiled for the host, against the oracle's DistributeOctTree: level-0 regions of 1080p to 4096x2160 frames, point sets
that force depth 12, and regions exactly 2048 and 2049 px wide.  The same source runs one-threaded, under ThreadSanitizer with T threads
and a real barrier, and with the barriers counted."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "orb_slam3_detailed_comments_b200", "csrc")
SRCS = [os.path.join(HERE, "host_emul", "qt_k64.cpp")] + [os.path.join(CSRC, f) for f in ("devmath.cuh", "quadtree_core.cuh", "quadtree_sort_par.cuh")]
BUILDS = {"seq": ["-O2"], "tsan": ["-O1", "-g", "-fsanitize=thread", "-DQT_EMUL_THREADS"], "count": ["-O2", "-DQT_HOST_COUNT_SYNCS"]}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("qt_k64")
    out = {}
    for name, flags in BUILDS.items():
        out[name] = str(d / ("qt_k64_" + name))
        subprocess.check_call(["g++"] + flags + ["-ffp-contract=off", "-std=c++20", "-o", out[name], SRCS[0], "-lpthread"])
    return out


def cell_geom(w, h):
    width, height = np.float32(w - 32), np.float32(h - 32)
    nCols, nRows = int(width / np.float32(35)), int(height / np.float32(35))
    return int(math.ceil(width / nCols)), int(math.ceil(height / nRows)), nCols


def run(exe, c, W, H, N, bits, variant=1, threads=1, tmp=None):
    wC, hC, nC = cell_geom(W, H)
    c = np.ascontiguousarray(c, np.int32)
    fin, fout = os.path.join(tmp, "c.bin"), os.path.join(tmp, "o.bin")
    with open(fin, "wb") as f:
        f.write(np.array([len(c), W - 32, H - 32, N, wC, hC, nC, variant], np.int32).tobytes() + c.tobytes())
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1 exitcode=66")
    pr = subprocess.run([exe, fin, fout, str(threads), str(bits)], env=env, capture_output=True, text=True, timeout=900)
    assert pr.returncode == 0, "driver / ThreadSanitizer failure (%d):\n%s" % (pr.returncode, pr.stderr[-4000:])
    o = np.fromfile(fout, np.int32)
    return o[1:].reshape(-1, 3)[:o[0]], pr.stdout


def level_cands(ex, l):
    """The oracle's FAST candidates of level l in the reference order (no cap on their number)."""
    cap = 1 << 22
    a = np.zeros((cap, 3), np.int32)
    n = po.lib().orc_level_cands(ex.h, l, a.ctypes.data_as(C.c_void_p), cap)
    assert n < cap
    return a[:n].copy()


def corner_rich(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def check(exe, c, W, H, N, tmp, forms=(64,), variants=(0, 1)):
    ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
    for bits in forms:
        for v in variants:
            got, _ = run(exe["seq"], c, W, H, N, bits, v, tmp=tmp)
            assert len(got) == len(ref) and (got == c[ref]).all(), (W, H, N, bits, v)
    return ref


@pytest.mark.parametrize("w,h", [(1920, 1080), (2208, 1242), (2560, 1440), (3840, 2160), (4096, 2160)])
@pytest.mark.parametrize("kind", ["textured", "corner-rich"])
def test_level0_regions_match_oracle(exe, tmp_path, w, h, kind):
    img = synth.frame(w, h, 11, 1.0, 400) if kind == "textured" else corner_rich(w, h, 12)
    for nf in (1200, 2000, 5000):
        ex = po.OracleExtractor(nf, 1.2, 8, 20, 7)
        ex(img)
        c = level_cands(ex, 0)
        assert ex.level_size(0) == (w, h)
        if kind == "corner-rich":
            assert len(c) > 32768 * (w * h) // (3840 * 2160)      # far beyond the shared-memory sort capacity at 4K
        # the 1080p region (1888 px) is within the 32-bit form: both forms must agree with the oracle there
        check(exe, c, w, h, int(ex.features_per_level[0]), str(tmp_path), forms=(32, 64) if w - 32 <= 2048 else (64,))


def _grid_order(pts, W, H):
    wC, hC, nC = cell_geom(W, H)
    p64 = pts.astype(np.int64)
    key = ((p64[:, 1] - 3) // hC * nC + (p64[:, 0] - 3) // wC) * (1 << 24) + p64[:, 1] * 4096 + p64[:, 0]
    return pts[np.argsort(key, kind="stable")]


def _cands(xy, W, H, rng, lo=7, hi=200):
    xy = np.unique(np.clip(np.asarray(xy), 3, [W - 36, H - 36]), axis=0)
    score = rng.integers(lo, hi, len(xy))
    return _grid_order(np.concatenate([xy, score[:, None]], 1).astype(np.int32), W, H)


def _depth12_sets(W, H, rng):
    rw, rh = W - 32, H - 32
    corners = [(3, 3), (rw - 5, 3), (3, rh - 5), (rw - 5, rh - 5)]
    pairs = np.array([p for (x, y) in corners for p in ((x, y), (x + 1, y))])                       # one pixel apart at every corner
    diag = np.array([p for (x, y) in corners for p in ((x, y), (x + 1, y + 1))])
    ctr = np.stack([rng.integers(40, rw - 40, 6), rng.integers(40, rh - 40, 6)], 1)
    clusters = ctr[rng.integers(0, 6, 6000)] + rng.integers(-6, 7, (6000, 2))                        # dense clusters
    mids = []                                                                                         # every box midpoint down to depth 6
    boxes = [(0, 0, rw, rh)]
    for _ in range(6):
        nb = []
        for (x0, y0, x1, y1) in boxes:
            mx, my = x0 + (x1 - x0 + 1) // 2, y0 + (y1 - y0 + 1) // 2
            mids += [(mx, my), (mx - 1, my - 1), (mx, my - 1), (mx - 1, my)]
            nb += [(x0, y0, mx, my), (mx, y0, x1, my), (x0, my, mx, y1), (mx, my, x1, y1)]
        boxes = nb
    return {"corner pairs": pairs, "corner diagonals": diag, "clusters": clusters, "box midpoints": np.array(mids),
            "all": np.concatenate([pairs, clusters, np.array(mids)])}


@pytest.mark.parametrize("w,h", [(3840, 2160), (4096, 2160), (4128, 2080)])
def test_adversarial_sets_forcing_depth_12(exe, tmp_path, w, h):
    rng = np.random.default_rng(w + h)
    for name, xy in _depth12_sets(w, h, rng).items():
        for lo, hi in ((7, 200), (7, 9)):                       # distinct scores, then heavy ties
            c = _cands(xy, w, h, rng, lo, hi)
            for N in (1, 7, 60, 261, 2000):
                check(exe, c, w, h, N, str(tmp_path))


@pytest.mark.parametrize("region", [2048, 2049])
def test_regions_at_the_form_boundary(exe, tmp_path, region):
    """A 2048 px region is the largest the 32-bit form resolves to single pixels; at 2049 px only the 64-bit form is exact."""
    w, h = region + 32, 1200
    rng = np.random.default_rng(region)
    sets = _depth12_sets(w, h, rng)
    img = corner_rich(w, h, region)
    ex = po.OracleExtractor(2000, 1.2, 8, 20, 7)
    ex(img)
    cases = [(level_cands(ex, 0), int(ex.features_per_level[0]))] + [(_cands(xy, w, h, rng), N) for xy in sets.values() for N in (7, 261)]
    for c, N in cases:
        check(exe, c, w, h, N, str(tmp_path), forms=(32, 64) if region == 2048 else (64,))


@pytest.mark.parametrize("threads", [3, 8, 32])
def test_threaded_k64_is_race_free_and_matches_oracle(exe, tmp_path, threads):
    """Level 0 of a 2560x1440 frame and a depth-12 point set at 4096x2160, by T threads with a real barrier under ThreadSanitizer."""
    ex = po.OracleExtractor(2000, 1.2, 8, 20, 7)
    ex(synth.frame(2560, 1440, 3, 1.5, 200))
    rng = np.random.default_rng(threads)
    cases = [(level_cands(ex, 0), 2560, 1440, int(ex.features_per_level[0])),
             (_cands(_depth12_sets(4096, 2160, rng)["all"], 4096, 2160, rng, 7, 10), 4096, 2160, 261)]
    for c, W, H, N in cases:
        ref = po.distribute(c, 16, W - 16, 16, H - 16, N)
        for v in (0, 1):
            got, _ = run(exe["tsan"], c, W, H, N, 64, v, threads, str(tmp_path))
            assert len(got) == len(ref) and (got == c[ref]).all(), (W, H, v, threads)


def test_barrier_count_equals_the_32_bit_form(exe, tmp_path):
    """Where both forms apply, the 64-bit one executes exactly the barriers of the 32-bit one (same algorithm, wider element): the
    extra depth only adds work to nodes that are still multi-point after 11 halvings, which a <= 2048 px region never has."""
    ex = po.OracleExtractor(1200, 1.2, 8, 20, 7)
    ex(synth.frame(1920, 1080, 1))
    for l in range(8):
        c = level_cands(ex, l)
        W, H = ex.level_size(l)
        N = int(ex.features_per_level[l])
        for v in (0, 1):
            (g32, s32), (g64, s64) = [run(exe["count"], c, W, H, N, bits, v, tmp=str(tmp_path)) for bits in (32, 64)]
            assert (g32 == g64).all() and s32 == s64 and int(s32.split()[0]) > 0, (l, v, s32, s64)
