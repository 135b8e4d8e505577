"""CPU tier: the camera-image models that run before Frame::Frame -- Tracking::GrabImage*'s cv::cvtColor to grey and System::Track*'s
cv::resize(INTER_LINEAR), resize first -- in the oracle (oracle/ingest_oracle.cpp) against cv2, and k_ingest's per-thread body
(csrc/resize_core.cuh ig_pixels4) compiled for the host against both."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import pyingest  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CODES = {"rgb": cv2.COLOR_RGB2GRAY, "bgr": cv2.COLOR_BGR2GRAY, "rgba": cv2.COLOR_RGBA2GRAY, "bgra": cv2.COLOR_BGRA2GRAY}
# (source width, height) -> (width, height): the camera sizes of the benchmarks down to config 3's 640 x 480 and config 2's
# 640 x 400, an upscale (whose first and last rows take cv::resize's unclamped row fraction), non-integer ratios in each axis
# both ways, exactly 2 in both axes (cv::resize's INTER_AREA fast path) and no resize
CASES = [((1280, 720), (640, 480)), ((752, 480), (640, 400)), ((640, 480), (1280, 960)), ((1000, 700), (613, 457)),
         ((500, 300), (777, 451)), ((1280, 720), (640, 360)), ((333, 251), (333, 251))]


@pytest.fixture(scope="module")
def emul():
    d = os.path.join(HERE, "host_emul")
    so, src = os.path.join(d, "libingest_emul.so"), os.path.join(d, "ingest_emul.cpp")
    deps = [src, os.path.join(HERE, "..", "orb_slam3_detailed_comments_b200", "csrc", "resize_core.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    L = C.CDLL(so)
    L.emul_ingest.restype = None
    L.emul_ingest.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
    return L


def run_emul(L, img, fmt, size):
    sh, sw = img.shape[:2]
    dw, dh = size
    dpitch = (dw + 15) // 16 * 16
    out = np.full((dh, dpitch), 0xEE, np.uint8)
    L.emul_ingest(img.ctypes.data, pyingest.FORMATS[fmt], sw, sh, img.strides[0], out.ctypes.data, dw, dh, dpitch)
    assert (out[:, dw:(dw + 3) // 4 * 4] == 0).all()        # the last word of a row is zero past the width
    return out[:, :dw]


def every_colour(cn, seed):
    """all 2^24 colours as a 4096 x 4096 image (channel 0 = low byte), random alpha for 4 channels"""
    v = np.arange(1 << 24, dtype=np.uint32)
    ch = [(v & 255), (v >> 8) & 255, (v >> 16) & 255]
    if cn == 4:
        ch.append(np.random.default_rng(seed).integers(0, 256, 1 << 24, dtype=np.uint32))
    return np.stack(ch, 1).astype(np.uint8).reshape(4096, 4096, cn)


def camera_image(rng, sw, sh, cn, stride_pad):
    """a random sw x sh image of cn channels whose rows are sw * cn + stride_pad bytes apart"""
    buf = rng.integers(0, 256, (sh, sw * cn + stride_pad), dtype=np.uint8)
    img = buf[:, :sw * cn]
    return img.reshape(sh, sw, cn) if cn > 1 else img


@pytest.mark.parametrize("fmt", ["rgb", "bgr", "rgba", "bgra"])
def test_conversion_of_every_colour_matches_cv2(fmt, emul):
    img = every_colour(3 if len(fmt) == 3 else 4, seed=len(fmt))
    want = cv2.cvtColor(img, CODES[fmt])
    assert (pyingest.ingest(img, fmt) == want).all()
    assert (run_emul(emul, img, fmt, (4096, 4096)) == want).all()


@pytest.mark.parametrize("src,dst", CASES)
@pytest.mark.parametrize("fmt", ["gray", "rgb", "bgr", "rgba", "bgra"])
@pytest.mark.parametrize("stride_pad", [0, 7])
def test_resize_then_convert_matches_cv2(src, dst, fmt, stride_pad, emul):
    cn = pyingest.CHANNELS[pyingest.FORMATS[fmt]]
    img = camera_image(np.random.default_rng(sum(src) + sum(dst) + cn), *src, cn, stride_pad)
    want = cv2.resize(img, dst, interpolation=cv2.INTER_LINEAR)
    if fmt != "gray":
        want = cv2.cvtColor(want, CODES[fmt])
    assert (pyingest.ingest(img, fmt, dst) == want).all()
    assert (run_emul(emul, img, fmt, dst) == want).all()


def test_resize_first_is_not_convert_first():
    """The two orders give different bytes, so the order is observable: System::Track* resizes before GrabImage* converts."""
    img = camera_image(np.random.default_rng(5), 1280, 720, 3, 0)
    a = pyingest.ingest(img, "bgr", (640, 480))
    b = cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), (640, 480), interpolation=cv2.INTER_LINEAR)
    assert (a != b).sum() > 10000
