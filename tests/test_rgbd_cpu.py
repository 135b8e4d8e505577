"""CPU tier of the RGB-D depth stage: Tracking::GrabImageRGBD's depth conversion and Frame::ComputeStereoFromRGBD for a camera with zero
distortion.  k_stereo_rgbd's per-thread body (csrc/rgbd_core.cuh), compiled for the host, and the oracle (oracle/rgbd_oracle.cpp
orc_stereo_from_rgbd, which converts the whole map first as the reference does) both equal a numpy float32 restatement in float bits:
every u16 value at three factors, float maps with the special values, the edges of the factor rule for both formats, and the truncation
of fractional keypoint coordinates.  Also: the new entry point fails loudly without a device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from oracle import pyrgbd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
f32 = np.float32
BF = f32(40.0)                                 # TUM fr3's bf
FACTORS = [f32(1.0 / 5000), f32(1.0 / 1000), f32(1.0)]


@pytest.fixture(scope="module")
def emul():
    d = os.path.join(HERE, "host_emul")
    so, src = os.path.join(d, "librgbd_emul.so"), os.path.join(d, "rgbd_emul.cpp")
    csrc = os.path.join(ROOT, "orb_slam3_detailed_comments_b200", "csrc")
    deps = [src, os.path.join(csrc, "rgbd_core.cuh"), os.path.join(csrc, "devmath.cuh"), os.path.join(ROOT, "include", "orbslam3_b200.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in deps):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so, src])
    L = C.CDLL(so)
    L.emul_rgbd_scaled.restype = C.c_int
    L.emul_rgbd_scaled.argtypes = [C.c_int, C.c_float]
    L.emul_rgbd.restype = None
    L.emul_rgbd.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    return L


def scaled(dtype, factor):
    """GrabImageRGBD: fabs(mDepthMapFactor - 1.0f) > 1e-5 || type != CV_32F -- the float difference compared in double"""
    return dtype == np.uint16 or abs(float(f32(factor) - f32(1))) > 1e-5


def restate(x, y, depth, factor, bf=BF):
    d = depth[y.astype(np.int64), x.astype(np.int64)].astype(f32)
    if scaled(depth.dtype, factor):
        d = (d * f32(factor)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ok = d > 0
        return np.where(ok, (x - f32(bf) / d).astype(f32), f32(-1)), np.where(ok, d, f32(-1))


def run_emul(L, x, y, depth, factor, bf=BF):
    xy = np.ascontiguousarray(np.stack([x, y], 1).astype(f32))
    uR, dep = np.zeros(len(x), f32), np.zeros(len(x), f32)
    L.emul_rgbd(xy.ctypes.data, len(x), depth.ctypes.data, 1 if depth.dtype == np.uint16 else 2, depth.strides[0], float(factor), float(bf),
                uR.ctypes.data, dep.ctypes.data)
    return uR, dep


def run_oracle(x, y, depth, factor, bf=BF):
    kps = np.zeros(len(x), po.KP_DTYPE)
    kps["x"], kps["y"] = x, y
    return pyrgbd.stereo_from_rgbd(kps, depth, factor, bf)


def same(a, b):
    return all((p.view(np.uint32) == q.view(np.uint32)).all() for p, q in zip(a, b))


def padded(depth, pad):
    """the same map with rows `pad` elements longer than its width"""
    buf = np.zeros((depth.shape[0], depth.shape[1] + pad), depth.dtype)
    buf[:, :depth.shape[1]] = depth
    return buf[:, :depth.shape[1]]


def keypoints_on_every_pixel(H, W, rng):
    """one keypoint per pixel at a fractional position inside it: (int)x, (int)y must land on that pixel"""
    v, u = np.mgrid[0:H, 0:W]
    x = (u.ravel() + rng.uniform(0, 0.999, H * W)).astype(f32)
    y = (v.ravel() + rng.uniform(0, 0.999, H * W)).astype(f32)
    return x, y


@pytest.mark.parametrize("factor", FACTORS)
@pytest.mark.parametrize("pad", [0, 3])
def test_every_u16_value(emul, factor, pad):
    rng = np.random.default_rng(1)
    depth = padded(rng.permutation(np.arange(1 << 16, dtype=np.uint16)).reshape(256, 256), pad)
    x, y = keypoints_on_every_pixel(256, 256, rng)
    want = restate(x, y, depth, factor)
    assert same(run_emul(emul, x, y, depth, factor), want)
    assert same(run_oracle(x, y, depth, factor), want)
    assert (want[1] > 0).sum() == (1 << 16) - 1                       # only the zero holes stay -1


def special_map(rng, H=64, W=64):
    specials = np.array([0.0, -0.0, -1.0, -1e-30, np.nan, np.inf, -np.inf, 1e-45, 1e-40, 1.17e-38, 3e-39, 0.5, 1.0, 5.2, 1e30, 65535.0], f32)
    vals = np.concatenate([specials, rng.uniform(0, 10, H * W - len(specials)).astype(f32)])
    return rng.permutation(vals).reshape(H, W).astype(f32)


@pytest.mark.parametrize("factor", [f32(1.0), f32(1.0 / 5000), f32(2.0)])
@pytest.mark.parametrize("pad", [0, 5])
def test_float_maps_with_special_values(emul, factor, pad):
    rng = np.random.default_rng(2)
    depth = padded(special_map(rng), pad)
    x, y = keypoints_on_every_pixel(64, 64, rng)
    want = restate(x, y, depth, factor)
    assert same(run_emul(emul, x, y, depth, factor), want)
    assert same(run_oracle(x, y, depth, factor), want)
    d = want[1]
    assert np.isinf(d).any() and ((d > 0) & (d < 1.2e-38)).any()        # +inf and denormal depths pass the d > 0 test


def rule_edges():
    """the float32 factors on either side of |factor - 1| = 1e-5, above and below 1"""
    out = []
    for sign in (1, -1):
        f = f32(1 + sign * 1e-5)
        while abs(float(f - f32(1))) > 1e-5:
            f = np.nextafter(f, f32(1))
        while abs(float(np.nextafter(f, f32(sign * 2)) - f32(1))) <= 1e-5:
            f = np.nextafter(f, f32(sign * 2))
        out += [f, np.nextafter(f, f32(sign * 2))]                         # last one inside, first one outside
    return out


@pytest.mark.parametrize("dtype", [np.uint16, np.float32])
def test_factor_rule_edges(emul, dtype):
    edges = rule_edges()
    assert [scaled(np.float32, f) for f in edges] == [False, True, False, True]
    rng = np.random.default_rng(3)
    depth = (rng.integers(0, 60000, (32, 32)).astype(dtype) if dtype == np.uint16 else rng.uniform(0, 60000, (32, 32)).astype(f32))
    x, y = keypoints_on_every_pixel(32, 32, rng)
    for f in edges:
        assert emul.emul_rgbd_scaled(1 if dtype == np.uint16 else 2, float(f)) == scaled(dtype, f)
        want = restate(x, y, depth, f)
        assert same(run_emul(emul, x, y, depth, f), want)
        assert same(run_oracle(x, y, depth, f), want)
        if dtype == np.float32 and not scaled(dtype, f):                   # close to 1 but not 1: the map is used as it is
            assert (want[1][want[1] > 0] == depth[y.astype(int), x.astype(int)][want[1] > 0]).all()


def test_truncation_of_fractional_coordinates(emul):
    depth = np.arange(1, 17, dtype=np.uint16).reshape(4, 4) * 1000
    x = np.array([0.0, 0.999, 1.0, 1.5, 2.999, 3.25, 0.4999, 3.999], f32)
    y = np.array([0.0, 0.999, 1.0, 2.5, 2.0001, 3.999, 3.0, 0.75], f32)
    want = restate(x, y, depth, f32(1 / 5000))
    assert (want[1] == (depth[[0, 0, 1, 2, 2, 3, 3, 0], [0, 0, 1, 1, 2, 3, 0, 3]].astype(f32) * f32(1 / 5000)).astype(f32)).all()
    assert same(run_emul(emul, x, y, depth, f32(1 / 5000)), want)
    assert same(run_oracle(x, y, depth, f32(1 / 5000)), want)


def test_entry_point_without_a_device():
    from orb_slam3_detailed_comments_b200 import _native as N
    N.build()
    L = N.lib()
    if L.orb_device_count() > 0:
        pytest.skip("a GPU is present")
    depth = np.zeros((4, 4), np.uint16)
    assert L.orbm_stereo_rgbd_batch(None, 1, depth.ctypes.data, 1, 8, 32, 0.0002, 0, 40.0) == -6      # ORB_ERR_NO_DEVICE
    assert b"no CPU fallback" in L.orb_last_error()
