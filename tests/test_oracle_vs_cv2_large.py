"""CPU tier: the oracle's pyramid, per-cell FAST candidates and 7x7 blur pinned against the real cv2 build at 1920x1080 and 3840x2160,
the sizes the extractor now supports up to 4128 px a side.  Skipped when cv2 is not importable."""
import math

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import pyoracle as po  # noqa: E402
from orb_slam3_detailed_comments_b200 import synth  # noqa: E402

cv2.setNumThreads(1)
SIZES = [(1920, 1080), (3840, 2160)]


@pytest.fixture(scope="module", params=SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def extracted(request):
    w, h = request.param
    img = synth.frame(w, h, seed=w, sigma=1.2, nrect=300)
    ex = po.OracleExtractor(2000, 1.2, 8, 20, 7)
    ex(img)
    return img, ex


def test_resize_chain_matches_cv2(extracted):
    img, ex = extracted
    prev = img
    for l in range(1, 8):
        lw, lh = ex.level_size(l)
        prev = cv2.resize(prev, (lw, lh), interpolation=cv2.INTER_LINEAR)
        assert (ex.level_pyramid(l) == prev).all(), l


def test_gaussian_blur_matches_cv2(extracted):
    img, ex = extracted
    for l in (0, 1, 4):
        lv = np.ascontiguousarray(ex.level_pyramid(l))
        assert (po.blur(lv) == cv2.GaussianBlur(lv, (7, 7), 2, 2, borderType=cv2.BORDER_REFLECT_101)).all(), l


def _cv2_cells(level, ini=20, mn=7):
    H, W = level.shape
    minB, maxBX, maxBY = 16, W - 16, H - 16
    width, height = np.float32(maxBX - minB), np.float32(maxBY - minB)
    nCols, nRows = int(width / np.float32(35)), int(height / np.float32(35))
    wCell, hCell = int(math.ceil(width / nCols)), int(math.ceil(height / nRows))
    f_ini, f_min = cv2.FastFeatureDetector_create(ini, True), cv2.FastFeatureDetector_create(mn, True)
    out = []
    for i in range(nRows):
        iniY = minB + i * hCell
        maxY = min(iniY + hCell + 6, maxBY)
        if iniY >= maxBY - 3:
            continue
        for j in range(nCols):
            iniX = minB + j * wCell
            maxX = min(iniX + wCell + 6, maxBX)
            if iniX >= maxBX - 6:
                continue
            cell = np.ascontiguousarray(level[iniY:maxY, iniX:maxX])
            k = f_ini.detect(cell) or f_min.detect(cell)
            out += [(int(p.pt[0]) + j * wCell, int(p.pt[1]) + i * hCell, int(p.response)) for p in k]
    return np.array(out, np.int32).reshape(-1, 3)


def test_per_cell_fast_matches_cv2(extracted):
    import ctypes as C
    img, ex = extracted
    for l in (0, 1, 3, 7):
        ref = _cv2_cells(ex.level_pyramid(l))
        cap = 1 << 22                                      # level 0 at 4K has more candidates than OracleExtractor.level_cands holds
        a = np.zeros((cap, 3), np.int32)
        n = po.lib().orc_level_cands(ex.h, l, a.ctypes.data_as(C.c_void_p), cap)
        assert n == len(ref) and (a[:n] == ref).all(), l
