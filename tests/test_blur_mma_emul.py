"""CPU tier: k_blur_mma (csrc/blur_mma.cuh) -- the GaussianBlur on the tensor cores -- replayed lane by lane in numpy int64.

The lanes' constant A fragments come from the header's own bm_fragments() compiled for the host.  Everything the kernel does with
them is restated here at fragment level: the reflected staging (unstaged shared memory is random, as on the device), the m16n8k32
u8 register layouts of A, B and the accumulators, the pass-H accumulators re-read as pass-V B fragments under the sigma permutation,
the hi/lo byte split, the rounding constant in the C operand, the byte-2 epilogue and the 16-byte stores inside the level.  The
result is compared with the oracle's cv::GaussianBlur model on every tile of the usual level geometries, so a wrong permutation,
fragment index or edge rule shows up without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
TAPS = np.array([18, 34, 48, 56, 48, 34, 18], np.int64)
LANE = np.arange(32)
G, T = LANE >> 2, LANE & 3


@pytest.fixture(scope="module")
def frag(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("blur_mma") / "libblur_mma_emul.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "host_emul", "blur_mma_emul.cpp")])
    L = C.CDLL(so)
    f = np.zeros(256, np.uint32)
    L.emul_blur_fragments(f.ctypes.data_as(C.c_void_p))
    geo = np.zeros(3, np.int32)
    L.emul_blur_tile(geo.ctypes.data_as(C.c_void_p))
    return f.reshape(8, 32), tuple(int(v) for v in geo)


def _perm(a, b, sel):
    """__byte_perm: result byte k = byte (sel >> 4k) & 7 of (b:a)."""
    v = (np.asarray(a, np.int64) & 0xFFFFFFFF) | ((np.asarray(b, np.int64) & 0xFFFFFFFF) << 32)
    r = np.zeros(np.broadcast(a, b).shape, np.int64)
    for k in range(4):
        r |= ((v >> (8 * ((sel >> (4 * k)) & 7))) & 0xFF) << (8 * k)
    return r


def _mma(a, b0, b1, c):
    """mma.sync.m16n8k32.row.col.s32.u8.u8.s32 from per-lane registers: a (..., 32, 4), b0 / b1 (..., 32) -> d (..., 32, 4)."""
    a = np.asarray(a, np.int64)
    A = np.zeros(a.shape[:-2] + (16, 32), np.int64)
    for r in range(4):
        for i in range(4):
            A[..., G + 8 * (r & 1), 16 * (r >> 1) + 4 * T + i] = (a[..., r] >> (8 * i)) & 0xFF
    B = np.zeros(np.asarray(b0).shape[:-1] + (32, 8), np.int64)
    for r, b in enumerate((b0, b1)):
        for i in range(4):
            B[..., 16 * r + 4 * T + i, G] = (np.asarray(b, np.int64) >> (8 * i)) & 0xFF
    D = A @ B + c
    return np.stack([D[..., G, 2 * T], D[..., G, 2 * T + 1], D[..., G + 8, 2 * T], D[..., G + 8, 2 * T + 1]], -1)


def _reflect(i, n):
    i = np.where(i < 0, -i, i)
    return np.where(i >= n, 2 * n - 2 - i, i)


def _k_blur_mma(img, frag, geo, rng):
    """The whole kernel on one level image: every tile and warp at once, the six 16-row steps in order."""
    TW, TH, SROW = geo
    h, w = img.shape
    nty, ntx = (h + TH - 1) // TH, (w + TW - 1) // TW
    ah, av = frag[:4].T.astype(np.int64), frag[4:].T.astype(np.int64)        # (32 lanes, 4 registers)
    # staging: rows Y0 - 3 .. min(Y0 + TH + 2, h + 2) of columns X0 - 8 .. X0 + SROW - 9 -- the 8-byte words inside the row, then
    # the reflected columns -3 .. -1 and the columns from the last whole word to w + 2; what is not staged holds garbage
    smem = rng.integers(0, 256, (nty, ntx, (TH + 8) * SROW + 16), dtype=np.uint8)
    for ty in range(nty):
        for tx in range(ntx):
            X0, Y0 = tx * TW, ty * TH
            ys = Y0 - 3 + np.arange(min(TH + 6, h - Y0 + 6))
            c = X0 - 8 + np.arange(SROW)
            word = c - c % 8
            staged = ((word >= 0) & (word + 8 <= w)) | ((c >= -3) & (c < 0)) | ((c >= w & ~7) & (c < w + 3))
            tile = smem[ty, tx, :(TH + 6) * SROW].reshape(TH + 6, SROW)
            tile[:len(ys), staged] = img[_reflect(ys, h)][:, _reflect(c[staged], w)]
    words = smem.view(np.uint32).astype(np.int64)                             # (nty, ntx, words)
    warp = np.arange(TW // 16)[:, None]
    base = G * (SROW // 4) + 4 * warp + 1 + T                                   # (8 warps, 32 lanes): word of window column 4t, row g
    sout = np.zeros((nty, ntx, TH, SROW), np.uint8)

    def pass_h(r0):
        row = words[..., base + r0 * (SROW // 4)]
        d = _mma(ah, row, words[..., base + r0 * (SROW // 4) + 4], 0)
        return _perm(d[..., 0], d[..., 1], 0x5140), _perm(d[..., 2], d[..., 3], 0x5140)

    def pass_v(a, b, c, s, col0):
        lo = _mma(av, _perm(a, b, 0x5410), c & 0xFFFF, 32768)
        hi = _mma(av, _perm(a, b, 0x7632), c >> 16, 0)
        o = lo + (hi << 8)
        assert (o < 1 << 24).all()
        cols = 16 * warp + col0 + 2 * T
        for k, (dr, dc) in enumerate([(0, 0), (0, 1), (8, 0), (8, 1)]):
            sout[:, :, 16 * s + G + dr, cols + dc] = (o[..., k] >> 16) & 0xFF

    a0, a1 = pass_h(0)
    for s in range(TH // 16):
        b0, b1 = pass_h(16 * s + 8)
        c0, c1 = pass_h(16 * s + 16)
        pass_v(a0, b0, c0, s, 0)
        pass_v(a1, b1, c1, s, 8)
        a0, a1 = c0, c1
    # stores: rows < h, 16-byte segments that start inside the level (blur_pitch = round_up(w, 16))
    pitch = (w + 15) // 16 * 16
    dst = np.full((h, pitch), 0xEE, np.uint8)
    for ty in range(nty):
        for tx in range(ntx):
            X0, Y0 = tx * TW, ty * TH
            rows = min(TH, h - Y0)
            seg = min(TW, pitch - X0)
            dst[Y0:Y0 + rows, X0:X0 + seg] = sout[ty, tx, :rows, :seg]
    return dst


def _levels(w, h, n=8, scale=1.2):
    out, s = [], np.float32(1.0)
    for _ in range(n):
        inv = np.float32(1.0) / s
        out.append((int(np.rint(np.float32(w) * inv)), int(np.rint(np.float32(h) * inv))))   # ORBextractor.cc:1691-1692
        s = np.float32(s * np.float32(scale))
    return out


def test_fragments_are_the_banded_taps(frag):
    f, _ = frag
    a = f.T.astype(np.int64)
    A = np.zeros((2, 16, 32), np.int64)
    for r in range(4):
        for i in range(4):
            A[0][G + 8 * (r & 1), 16 * (r >> 1) + 4 * T + i] = (a[:, r] >> (8 * i)) & 0xFF
            A[1][G + 8 * (r & 1), 16 * (r >> 1) + 4 * T + i] = (a[:, 4 + r] >> (8 * i)) & 0xFF
    kh = np.zeros((16, 32), np.int64)
    kv = np.zeros((16, 32), np.int64)
    for m in range(16):
        kh[m, m + 1:m + 8] = TAPS                     # output column m reads window columns m + 1 .. m + 7 (column x0 - 4 + c)
        kv[m, m:m + 7] = TAPS                         # output row m reads window rows m .. m + 6 (row y0 - 3 + y')
    sigma = np.array([(k & 16) + [2 * t, 2 * t + 1, 8 + 2 * t, 9 + 2 * t][i] for k in range(32) for t, i in [((k & 15) >> 2, k & 3)]])
    assert (A[0] == kh).all()
    assert (A[1] == kv[:, sigma]).all()
    assert sorted(sigma) == list(range(32))


@pytest.mark.parametrize("w,h", [(640, 480), (500, 377), (1280, 720)])
def test_every_level_of_the_usual_geometries_matches_the_oracle(frag, w, h):
    rng = np.random.default_rng(w * 7 + h)
    for lw, lh in _levels(w, h):
        img = rng.integers(0, 256, (lh, lw), dtype=np.uint8)
        got = _k_blur_mma(img, *frag, rng)
        assert (got[:, :lw] == po.blur(img)).all(), (lw, lh)


def _adversarial(w, h):
    yy, xx = np.mgrid[0:h, 0:w]
    spots = np.zeros((h, w), np.uint8)
    for y, x in [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (1, 2), (h // 2, w // 2), (h - 2, w - 3), (95, 127), (96, 128),
                 (3, w // 3), (h // 3, 2)]:
        spots[y, x] = 255
    return {"zeros": np.zeros((h, w), np.uint8), "full": np.full((h, w), 255, np.uint8),
            "checker": ((xx + yy) % 2 * 255).astype(np.uint8), "stripes": ((xx // 3 + yy // 5) % 2 * 255).astype(np.uint8),
            "spots": spots}


@pytest.mark.parametrize("w,h", [(640, 480), (500, 377), (1280, 720), (533, 400), (257, 193), (179, 134)])
def test_saturated_and_sparse_images_match_the_oracle(frag, w, h):
    rng = np.random.default_rng(3)
    for name, img in _adversarial(w, h).items():
        got = _k_blur_mma(img, *frag, rng)
        assert (got[:, :w] == po.blur(img)).all(), name
