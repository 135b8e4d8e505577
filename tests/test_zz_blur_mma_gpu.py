"""GPU tier: k_blur_mma, the default blur (ORB_BLUR_VARIANT=2), gives every blurred level byte for byte as the oracle's
cv::GaussianBlur model and as k_blur<true> (ORB_BLUR_VARIANT=1): random and saturated / sparse images in one batch, the 640x480,
500x377 and 1280x720 pyramids (every edge and corner tile of every level), and a level 0 aliased in a caller's device buffer
whose row pitch is a multiple of 8 but not of 16."""
import numpy as np
import pytest
import torch

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor

pytestmark = pytest.mark.gpu

GEOMETRIES = [(640, 480), (500, 377), (1280, 720)]


def _images(w, h, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    spots = np.zeros((h, w), np.uint8)
    for y, x in [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (1, 2), (h // 2, w // 2), (95, 127), (96, 128), (h - 2, w - 3)]:
        spots[y, x] = 255
    return np.stack([rng.integers(0, 256, (h, w), dtype=np.uint8), np.zeros((h, w), np.uint8), np.full((h, w), 255, np.uint8),
                     ((xx + yy) % 2 * 255).astype(np.uint8), spots, rng.integers(0, 256, (h, w), dtype=np.uint8)])


def _handle(monkeypatch, variant, w, h, B, nf=1000):
    monkeypatch.setenv("ORB_BLUR_VARIANT", variant)   # read by orbx_create
    ex = ORBextractor(nf, 1.2, 8, 20, 7, max_width=w, max_height=h, max_batch=B)
    monkeypatch.delenv("ORB_BLUR_VARIANT")
    return ex


@pytest.mark.parametrize("w,h", GEOMETRIES)
def test_blurred_levels_match_the_oracle_and_k_blur(monkeypatch, w, h):
    imgs = _images(w, h, w + h)
    B = len(imgs)
    new, old = _handle(monkeypatch, "2", w, h, B), _handle(monkeypatch, "1", w, h, B)
    new.extract_batch(imgs)
    old.extract_batch(imgs)
    for b in range(B):
        for l in range(new.nlevels):
            got = new.image_pyramid(b, l, blurred=True)
            assert (got == old.image_pyramid(b, l, blurred=True)).all(), (b, l)
            assert (got == po.blur(new.image_pyramid(b, l))).all(), (b, l)
    new.close()
    old.close()


@pytest.mark.parametrize("w,h,stride", [(500, 377, 504), (640, 480, 648)])
def test_aliased_level0_with_an_8_byte_pitch(monkeypatch, w, h, stride):
    imgs = _images(w, h, 7)[[0, 5, 3]]
    B = len(imgs)
    buf = np.zeros((B, h, stride), np.uint8)
    buf[:, :, :w] = imgs
    dev = torch.from_numpy(buf).cuda()
    assert dev.data_ptr() % 16 == 0 and stride % 8 == 0 and stride % 16 != 0
    ex = _handle(monkeypatch, "2", w, h, B, nf=1200)
    ex.extract_batch_device(dev.data_ptr(), B, w, h, stride, stride * h)
    torch.cuda.synchronize()
    n, mono, off, kps, desc = ex.download(B)
    ref = po.OracleExtractor(1200, 1.2, 8, 20, 7)
    for b in range(B):
        for l in range(ex.nlevels):
            assert (ex.image_pyramid(b, l, blurred=True) == po.blur(ex.image_pyramid(b, l))).all(), (b, l)
        rmono, rk, rd = ref(imgs[b])
        assert n[b] == len(rk) and mono[b] == rmono, b
        assert (kps[off[b]:off[b + 1]].view(np.uint8) == rk.view(np.uint8)).all(), b
        assert (desc[off[b]:off[b + 1]] == rd).all(), b
    ex.close()
