"""CPU tier: what LocalMapping::CreateNewMapPoints and the map-point updates hand the device's k_tri_match / k_tri_rotation,
k_distinctive and k_normal_depth, built the way the reference's callers build it, plus constructed cases at the decisions those
kernels make.  tests/test_zz_local_mapping_gpu.py holds the device to the oracle on all of them, bit for bit.

- `keyframes()`: a keyframe and its covisible neighbours on a slow trajectory -- oracle features of synth stereo pairs (640 x 480,
  1200 features) or monocular frames (752 x 480, 1200 features), map-point flags, the real vocabulary's FeatureVector nodes
  (tests/golden/orbvoc_subtree.npz at levelsup = 4).
- `pair()`: host/ORBmatcher_triangulation_b200.cc's inputs for one keyframe pair: R12 / t12, F12 = K1^-T [t12]x R12 K2^-1 and the
  epipole in float32, keyframe-1 queries in FeatureVector order (node, then feature index), valid2 / stereo2 from mvuRight.
- `tri_case()`: the pair plus constructed features -- equal-distance duplicates, the epipole radius and one ulp either side, dsqr
  between the float and the double value of 3.84 sigma^2, den == 0, one node for every query, node -1 queries, rotation histograms
  with tied bins, a bin at exactly 10 % of the maximum and rotations just below 360 degrees.
- `distinctive_lists()` / `normal_depth_case()`: observation lists of 1 ... 2 000 keyframes, and normal / depth inputs along
  trajectories 10 m, 500 m and 2 km from the origin on pyramids of (1.2, 8), (1.5, 5) and (2.0, 3) levels.

The tests below check that each case has the property it names, and the oracle against tests/pyref.py on the triangulation cases."""
import functools
import os

import numpy as np
import pytest

import pyref
from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32
KP = po.KP_DTYPE
# EuRoC-like stereo rig at 640 x 480 and the EuRoC cam0 intrinsics at 752 x 480
CAMS = {"stereo": dict(w=640, h=480, fx=435.2, fy=435.2, cx=320.0, cy=240.0, bf=47.9, b=0.11),
        "mono": dict(w=752, h=480, fx=458.654, fy=457.296, cx=367.215, cy=248.375)}
NFEAT = 1200
PYRAMIDS = [(1.2, 8), (1.5, 5), (2.0, 3)]
TRI_CASES = ["plain", "only_stereo", "mixed", "ties", "epipole", "dsqr", "den0", "one_node", "node_neg", "hist_ties", "hist_tenth"]
HIST_TIES = {1: 10, 4: 10, 8: 10, 11: 10}       # four bins at the maximum: strict '>' keeps the first three
HIST_TENTH = {2: 20, 5: 2, 9: 1, 12: 1}         # bin 5 is exactly 10 % of the maximum (kept), bins 9 / 12 below it; 12 from ~360 deg


@functools.lru_cache(None)
def vocabulary():
    z = np.load(os.path.join(HERE, "golden", "orbvoc_subtree.npz"))
    sub = {k[4:]: z[k] for k in z.files if k.startswith("sub_")}
    sub["L"] = int(sub["L"])
    return sub


def feature_nodes(desc, levelsup=4):
    """The real tree's node of every feature at `levelsup` (100 nodes at level 2).  The pruned copy keeps only the paths of 68
    descriptors, so most walks end on a pruned inner node of weight 0; the node above is what the full tree gives, so it is kept."""
    return po.bow_transform(vocabulary(), desc, levelsup)["node"].astype(np.int32)


def rot(axis, deg):
    a = np.deg2rad(deg)
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return (np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K).astype(f32)


def trajectory(n, start, step, yaw_step=0.3):
    """Tcw (R, t) of n keyframes whose centres start at `start` and advance by `step` metres, yawing slowly."""
    poses = []
    for k in range(n):
        R = rot([0, 1, 0], yaw_step * k) @ rot([1, 0, 0], 0.2 * np.sin(0.4 * k))
        C = (np.asarray(start, np.float64) + k * np.asarray(step, np.float64)).astype(f32)
        poses.append((R.astype(f32), (-(R @ C)).astype(f32)))
    return poses


@functools.lru_cache(None)
def _images(kind, n, seed):
    cam = CAMS[kind]
    if kind == "stereo":
        l, r, _ = synth.stereo_pair(cam["w"], cam["h"], seed=seed)
    else:
        l, r = synth.frame(cam["w"], cam["h"], seed=seed), None
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):                  # the neighbours see the same texture a few pixels further along, with sensor noise
        sh = (2 * k, k // 2)
        noise = rng.integers(-3, 4, l.shape)
        out.append(tuple(None if im is None else np.clip(np.roll(im, sh, (1, 0)).astype(int) + noise, 0, 255).astype(np.uint8)
                         for im in (l, r)))
    return out


@functools.lru_cache(None)
def keyframes(kind="stereo", n=3, seed=11, mp_frac=0.4, step=(0.05, 0.0, 0.01)):
    """Keyframe 0 and n - 1 covisible neighbours: dicts of kp, desc, uR (mvuRight), has_mp, node, R / t (Tcw), cam."""
    cam = CAMS[kind]
    rng = np.random.default_rng(seed + 1)
    poses = trajectory(n, (0.0, 0.0, 0.0), step)
    kfs = []
    for k, (l, r) in enumerate(_images(kind, n, seed)):
        eL = po.OracleExtractor(NFEAT, 1.2, 8, 20, 7)
        _, kp, desc = eL(l)
        if r is not None:
            eR = po.OracleExtractor(NFEAT, 1.2, 8, 20, 7)
            _, kR, dR = eR(r)
            uR, _, _ = po.stereo_matches(eL, eR, kp, desc, kR, dR, cam["bf"], cam["b"])
        else:
            uR = np.full(len(kp), -1, f32)
        node = feature_nodes(desc)
        node[rng.random(len(kp)) < 0.02] = -1         # features of stopped words enter no FeatureVector node
        kfs.append(dict(kp=kp, desc=desc, uR=np.asarray(uR, f32), has_mp=rng.random(len(kp)) < mp_frac, node=node,
                        R=poses[k][0], t=poses[k][1], cam=cam, sf=eL.scale_factors.astype(f32), s2=eL.level_sigma2.astype(f32)))
    return kfs


def geometry(kf1, kf2):
    """F12 (row-major) and the epipole of keyframe 1's centre in keyframe 2, in float32 like ORBmatcher_triangulation_b200.cc."""
    R1, t1, R2, t2 = kf1["R"], kf1["t"], kf2["R"], kf2["t"]
    Cw = (-(R1.T @ t1)).astype(f32)
    C2 = (R2 @ Cw + t2).astype(f32)
    c1, c2 = kf1["cam"], kf2["cam"]
    with np.errstate(invalid="ignore", divide="ignore"):
        ep = np.array([f32(f32(c2["fx"]) * C2[0]) / C2[2] + f32(c2["cx"]), f32(f32(c2["fy"]) * C2[1]) / C2[2] + f32(c2["cy"])], f32)
    R12 = (R1 @ R2.T).astype(f32)
    t12 = (R1 @ (-(R2.T @ t2)).astype(f32) + t1).astype(f32)
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]], f32)
    K = lambda c: np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1]], f32)
    F12 = (np.linalg.inv(K(c1).T).astype(f32) @ tx @ R12 @ np.linalg.inv(K(c2)).astype(f32)).astype(f32)
    return F12.reshape(-1), ep


def pair(kf1, kf2, only_stereo=False):
    """SearchForTriangulation's device inputs for one keyframe pair (dict; `src` = keyframe-1 feature index of each query)."""
    st1, st2 = kf1["uR"] >= 0, kf2["uR"] >= 0
    cand = np.nonzero((kf1["node"] >= 0) & ~kf1["has_mp"] & (st1 | (not only_stereo)))[0]
    src = cand[np.lexsort((cand, kf1["node"][cand]))]          # FeatureVector order: node, then feature index
    F12, ep = geometry(kf1, kf2)
    return dict(src=src, kp1=kf1["kp"][src], desc1=kf1["desc"][src], node1=kf1["node"][src], stereo1=st1[src].astype(np.uint8),
                kp2=kf2["kp"].copy(), desc2=kf2["desc"].copy(), node2=kf2["node"].copy(),
                valid2=(~kf2["has_mp"] & (st2 | (not only_stereo))).astype(np.uint8), stereo2=st2.astype(np.uint8),
                F12=F12, ep=ep, sf=kf2["sf"], s2=kf2["s2"], meta={})


def oracle(c, coarse, check_ori):
    return po.search_triangulation(c["kp1"], c["desc1"], c["node1"], c["stereo1"], c["kp2"], c["desc2"], c["node2"], c["valid2"],
                                   c["stereo2"], c["F12"], c["ep"], c["sf"], c["s2"], coarse, check_ori)


def epiline(c, x1, y1):
    """(a, b, c) of keypoint (x1, y1)'s epipolar line in image 2, in the kernels' float32 order."""
    F = np.asarray(c["F12"], f32)
    x1, y1 = f32(x1), f32(y1)
    return tuple(f32(f32(f32(x1 * F[j]) + f32(y1 * F[3 + j])) + F[6 + j]) for j in range(3))


def dsqr(c, q, x2, y2):
    a, b, cc = epiline(c, c["kp1"]["x"][q], c["kp1"]["y"][q])
    num = f32(f32(f32(a * f32(x2)) + f32(b * f32(y2))) + cc)
    den = f32(f32(a * a) + f32(b * b))
    return f32(f32(num * num) / den) if den != 0 else None, den


def epipole_value(c, x2, y2):
    ex, ey = f32(f32(c["ep"][0]) - f32(x2)), f32(f32(c["ep"][1]) - f32(y2))
    return f32(f32(ex * ex) + f32(ey * ey))


def on_line(c, x1, y1, x2):
    a, b, cc = (float(v) for v in epiline(c, x1, y1))
    return x2, -(a * x2 + cc) / b


def _kp(x, y, angle, octave):
    k = np.zeros(1, KP)
    k["x"], k["y"], k["angle"], k["octave"], k["size"], k["response"] = x, y, angle, octave, 31.0, 1.0
    return k


class _Builder:
    """Appends constructed queries and keyframe-2 features to a pair; `finish()` re-sorts the queries into FeatureVector order and
    spreads the new keyframe-2 rows over the whole array, so duplicates and gate points sit at scattered indices."""

    def __init__(self, c, rng):
        self.c, self.rng = c, rng
        self.q = {k: [c[k]] for k in ("kp1", "desc1", "node1", "stereo1", "src")}
        self.k2 = {k: [c[k]] for k in ("kp2", "desc2", "node2", "valid2", "stereo2")}
        self.n1, self.n2 = 1 << 20, len(c["kp2"])      # constructed keyframe-1 features follow the real ones
        self.tags = []          # (query src, [new keyframe-2 rows], label)

    def descriptor(self):
        """A fresh descriptor whose real vocabulary node is one of keyframe 2's, and that node."""
        d = self.rng.integers(0, 256, (1, 32), dtype=np.uint8)
        return d, int(feature_nodes(d)[0])

    def query(self, x, y, angle, desc, node, stereo):
        s = self.n1
        self.n1 += 1
        for k, v in (("kp1", _kp(x, y, angle, 0)), ("desc1", desc), ("node1", np.int32([node])), ("stereo1", np.uint8([stereo])),
                     ("src", np.array([s]))):
            self.q[k].append(v)
        return s

    def feature(self, x, y, angle, octave, desc, node, stereo, valid=1):
        i = self.n2
        self.n2 += 1
        for k, v in (("kp2", _kp(x, y, angle, octave)), ("desc2", desc), ("node2", np.int32([node])), ("valid2", np.uint8([valid])),
                     ("stereo2", np.uint8([stereo]))):
            self.k2[k].append(v)
        return i

    def finish(self, tags):
        c = dict(self.c)
        for k, v in self.q.items():
            c[k] = np.concatenate(v)
        order = np.lexsort((c["src"], c["node1"]))
        for k in self.q:
            c[k] = c[k][order]
        perm = self.rng.permutation(self.n2)           # new row perm[i] <- old row i
        inv = np.empty_like(perm)
        inv[perm] = np.arange(self.n2)
        for k, v in self.k2.items():
            a = np.concatenate(v)
            c[k] = a[inv]
        pos = {int(s): j for j, s in enumerate(c["src"])}
        c["meta"] = dict(tags=[(pos[s], [int(perm[i]) for i in rows], label) for s, rows, label in tags])
        return c


def _ties(b, c, rng, n=24):
    tags = []
    for j in range(n):
        d, node = b.descriptor()
        x1, y1 = rng.uniform(40, 600), rng.uniform(40, 440)
        ang = f32(rng.uniform(0, 360))
        s = b.query(x1, y1, ang, d, node, stereo=j % 2)
        dd = d.copy()
        for bit in rng.choice(256, j % 9, replace=False):       # distances 0 ... 8, equal for every duplicate
            dd[0, bit // 8] ^= np.uint8(1 << (bit % 8))
        rows = []
        for k in range(2 + j % 4):
            x2, y2 = on_line(c, x1, y1, rng.uniform(30, 600))
            rows.append(b.feature(x2, y2, ang, int(rng.integers(0, 8)), dd, node, stereo=1 - (k % 2) * (j % 2)))
        tags.append((s, rows, "tie"))
    return tags


def _epipole(b, c, rng):
    """Monocular pairs whose squared distance to the epipole is exactly 100 scale[oct], or one ulp below or above it."""
    tags = []
    ep = c["ep"].astype(np.float64)
    for oct_ in range(len(c["sf"])):
        T = f32(f32(100) * c["sf"][oct_])
        for want, label in ((T, "epi_on"), (np.nextafter(T, f32(0)), "epi_below"), (np.nextafter(T, f32(np.inf)), "epi_above")):
            for _ in range(50):
                d, node = b.descriptor()
                ang = rng.uniform(0, 2 * np.pi)
                x1, y1 = f32(ep[0] + 120 * np.cos(ang)), f32(ep[1] + 120 * np.sin(ang))    # its line runs through the epipole
                la, lb, _ = (float(v) for v in epiline(c, x1, y1))
                u = np.array([lb, -la]) / np.hypot(la, lb)
                p = ep + np.sqrt(float(T)) * u
                ulp = lambda v: np.spacing(f32(abs(v)))
                xs = f32(p[0]) + np.arange(-40, 41, dtype=np.float64)[:, None] * ulp(p[0])
                ys = f32(p[1]) + np.arange(-40, 41, dtype=np.float64)[None, :] * ulp(p[1])
                xs, ys = np.broadcast_arrays(xs.astype(f32), ys.astype(f32))
                ex, ey = f32(ep[0]) - xs, f32(ep[1]) - ys
                v = ex * ex + ey * ey
                hit = np.argwhere(v == want)
                if len(hit):
                    x2, y2 = xs[tuple(hit[0])], ys[tuple(hit[0])]
                    s = b.query(x1, y1, f32(10), d, node, stereo=0)
                    tags.append((s, [b.feature(x2, y2, f32(10), oct_, d, node, stereo=0)], label))
                    break
    return tags


def dsqr_targets(s2):
    """Per octave the float dsqr that the double comparison and a float one decide differently, and which way."""
    out = {}
    for o, s in enumerate(s2):
        thr_d = 3.84 * float(s)
        thr_f = min(f32(f32(3.84) * f32(s)), f32(thr_d))
        if float(thr_f) < thr_d:
            out[o] = (thr_f, True)                       # accepted in double, refused by `dsqr < float threshold`
        hi = max(f32(f32(3.84) * f32(s)), f32(thr_d))
        below = np.nextafter(hi, f32(0))
        if float(below) >= thr_d and o not in out:
            out[o] = (below, False)                      # refused in double, accepted in float
    return out


def _dsqr(b, c, rng):
    tags = []
    for oct_, (want, _) in dsqr_targets(c["s2"]).items():
        for _ in range(40):
            d, node = b.descriptor()
            x0, y0, X2 = rng.uniform(60, 580), rng.uniform(60, 420), rng.uniform(60, 580)
            k = np.arange(-24, 25, dtype=np.float64)
            x1 = (f32(x0) + k[:, None] * np.spacing(f32(x0))).astype(f32)
            y1 = (f32(y0) + k[None, :] * np.spacing(f32(y0))).astype(f32)
            x1, y1 = np.broadcast_arrays(x1, y1)
            F = np.asarray(c["F12"], f32)
            a = (x1 * F[0] + y1 * F[3]) + F[6]
            bb = (x1 * F[1] + y1 * F[4]) + F[7]
            cc = (x1 * F[2] + y1 * F[5]) + F[8]
            den = a * a + bb * bb
            y2 = f32(-(float(a.flat[0]) * X2 + float(cc.flat[0]) - np.sqrt(float(want) * float(den.flat[0]))) / float(bb.flat[0]))
            found = None
            for dx in range(-12, 13):
                x2 = f32(X2 + dx * np.spacing(f32(X2)))
                num = (a * x2 + bb * y2) + cc
                v = (num * num) / den
                hit = np.argwhere(v == want)
                if len(hit):
                    found = (x1[tuple(hit[0])], y1[tuple(hit[0])], x2)
                    break
            if found:
                s = b.query(found[0], found[1], f32(10), d, node, stereo=1)
                tags.append((s, [b.feature(found[2], y2, f32(10), oct_, d, node, stereo=1)], "dsqr"))
                break
    return tags


def rotation_pair(rng, b_):
    """Angles (a1, a2) whose rotation bin (factor 1/30) is b_; bin 12 from a rotation just below 360 degrees."""
    while True:
        a1 = f32(rng.uniform(0, 360))
        if b_ == 12:
            a2 = np.nextafter(a1, f32(np.inf)) if rng.random() < 0.5 else f32(a1 + f32(rng.uniform(1e-4, 5)))
        else:
            a2 = f32(a1 - f32(30 * b_ + rng.uniform(-14, 14)))
        if 0 <= a2 < 360 and pyref.rot_bin(a1, a2) == b_:
            return a1, a2


def _hist(b, c, rng, counts):
    tags = []
    for bin_, n in counts.items():
        for _ in range(n):
            d, node = b.descriptor()
            x1, y1 = rng.uniform(40, 600), rng.uniform(40, 440)
            a1, a2 = rotation_pair(rng, bin_)
            s = b.query(x1, y1, a1, d, node, stereo=1)
            x2, y2 = on_line(c, x1, y1, rng.uniform(30, 600))
            tags.append((s, [b.feature(x2, y2, a2, int(rng.integers(0, 8)), d, node, stereo=1)], f"bin{bin_}"))
    return tags


@functools.lru_cache(None)
def tri_case(name, seed=0):
    """One constructed triangulation case on keyframe 0 and neighbour 1 (see the module docstring)."""
    rng = np.random.default_rng(100 + seed)
    if name == "den0":          # a neighbour at the same centre: t12 == 0 exactly, F12 == 0, every line has den == 0, epipole 0/0
        kfs = keyframes("stereo", 2, 11)
        k2 = dict(kfs[1], t=np.zeros(3, f32))
        c = pair(dict(kfs[0], t=np.zeros(3, f32)), dict(k2, R=rot([0, 1, 0], 2.0) @ kfs[0]["R"]))
        c["meta"] = {}
        return c
    kind = "mono" if name == "epipole" else "stereo"
    step = (0.02, 0.01, 0.3) if name == "epipole" else (0.05, 0.0, 0.01)     # forward motion puts the epipole inside the image
    kfs = keyframes(kind, 2, 11 if kind == "stereo" else 21, step=step)
    c = pair(kfs[0], kfs[1], only_stereo=name == "only_stereo")
    if name in ("plain", "only_stereo"):
        return c
    if name == "mixed":                 # stereo flags of either side drawn at random, some monocular against monocular
        c["stereo1"] = (rng.random(len(c["src"])) < 0.5).astype(np.uint8)
        c["stereo2"] = (rng.random(len(c["kp2"])) < 0.5).astype(np.uint8)
        return c
    if name == "one_node":              # levelsup = L: DBoW2 leaves every feature at the root, so all queries share one node
        c["node1"][:] = 0
        c["node2"] = np.where(c["node2"] >= 0, 0, -1).astype(np.int32)
        return c
    if name == "node_neg":
        c["node1"][rng.random(len(c["node1"])) < 0.15] = -1
        return c
    b = _Builder(c, rng)
    if name.startswith("hist"):         # a neighbour whose features all hold map points: only the constructed pairs match
        b.k2["valid2"][0] = np.zeros_like(c["valid2"])
        tags = _hist(b, c, rng, HIST_TIES if name == "hist_ties" else HIST_TENTH)
    else:
        tags = {"ties": _ties, "epipole": _epipole, "dsqr": _dsqr}[name](b, c, rng)
    return b.finish(tags)


def candidates(c, q):
    """Every keyframe-2 feature of query q's node that passes the validity, Hamming, epipole and epipolar gates: [(dist, i2)]."""
    node = int(c["node1"][q])
    if node < 0:
        return []
    out = []
    for i2 in np.nonzero((c["node2"] == node) & (c["valid2"] != 0))[0]:
        dist = pyref.hamming(c["desc1"][q], c["desc2"][i2])
        if dist > 50:
            continue
        x2, y2 = c["kp2"]["x"][i2], c["kp2"]["y"][i2]
        oc = c["kp2"]["octave"][i2]
        if not c["stereo1"][q] and not c["stereo2"][i2] and epipole_value(c, x2, y2) < f32(f32(100) * c["sf"][oc]):
            continue
        v, den = dsqr(c, q, x2, y2)
        if v is None or not float(v) < 3.84 * float(c["s2"][oc]):
            continue
        out.append((dist, int(i2)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# map points


def _cluster(rng, n, flips=60):
    """n observations of one base descriptor, each with up to `flips` - 1 random bits toggled."""
    base = rng.integers(0, 256, 32, dtype=np.uint8)
    pos = rng.integers(0, 256, (n, flips))
    used = np.arange(flips)[None, :] < rng.integers(0, flips, n)[:, None]
    cnt = np.zeros((n, 256), np.int32)
    np.add.at(cnt, (np.repeat(np.arange(n), flips).reshape(n, flips)[used], pos[used]), 1)
    return base[None] ^ np.packbits(cnt % 2 == 1, axis=1, bitorder="little")


DISTINCTIVE_N = [1, 2, 3, 4, 5, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025,
                 1999, 2000]


@functools.lru_cache(None)
def distinctive_lists(seed=0):
    """Observation descriptors of map points seen by 1 ... 2 000 keyframes: every N of DISTINCTIVE_N (N = 0, 1, 31, 32, 33 mod 32,
    even and odd) as a noisy cluster, as all-identical rows, as a few exact duplicates of a handful of rows (tied medians), and as
    a cluster beside copies of one far row (where a median of rank N / 2 would choose another row).
    Returns (sizes, kinds, list of [N][32] arrays)."""
    rng = np.random.default_rng(300 + seed)
    sizes, kinds, lists = [], [], []
    for n in DISTINCTIVE_N:
        lists.append(_cluster(rng, n))
        kinds.append("cluster")
        lists.append(np.repeat(rng.integers(0, 256, (1, 32), dtype=np.uint8), n, 0))
        kinds.append("identical")
        heads = _cluster(rng, min(n, 1 + n % 5), flips=90)         # a few distinct rows, each repeated: equal medians
        lists.append(heads[rng.integers(0, len(heads), n)])
        kinds.append("duplicates")
        # a noisy cluster followed by (n + 1) // 2 copies of a row far from it: for even n the copies hold the median of rank
        # (n - 1) / 2 at 0, while at rank n / 2 a cluster row ties with them and, coming first, would win
        far = _cluster(rng, 1, flips=1)
        lists.append(np.concatenate([_cluster(rng, n // 2, flips=20), np.repeat(far, n - n // 2, 0)]))
        kinds.append("halves")
        sizes += [n] * 4
    return sizes, kinds, lists


def median_choice(d, rank):
    """The observation whose distance of the given rank to the others (itself included) is smallest, first minimum."""
    x = np.unpackbits(d, axis=1).astype(np.int32)
    dist = (x[:, None, :] != x[None, :, :]).sum(2) if len(d) <= 600 else np.stack([(x[i] != x).sum(1) for i in range(len(d))])
    med = np.sort(dist, 1)[:, rank]
    return int(np.argmin(med)), med


def filler_lists(n, seed=1):
    """n map points with 1 ... 12 observations (the bulk of a real map)."""
    rng = np.random.default_rng(400 + seed)
    return [_cluster(rng, int(k)) for k in rng.integers(1, 13, n)]


def normal_depth_case(distance, scale, levels, n_points=300, seed=0, empty_every=17):
    """Map points observed from keyframes on a trajectory `distance` metres from the origin: obs offsets, observer centres, positions,
    reference-keyframe centres and levels (every octave in turn), and caller values that points without observations must keep."""
    rng = np.random.default_rng(500 + seed + int(distance))
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    start = d * distance
    step = np.cross(d, [0.0, 0.0, 1.0])
    step = 0.25 * step / np.linalg.norm(step)
    centres = np.array([start + k * step + rng.normal(0, 0.02, 3) for k in range(200)], f32)
    counts = rng.integers(1, 61, n_points)
    counts[::empty_every] = 0
    counts[1::23] = 1
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    oc, pos, refc = [], np.zeros((n_points, 3), f32), np.zeros((n_points, 3), f32)
    for i, c in enumerate(counts):
        k0 = int(rng.integers(0, 200 - max(c, 1)))
        obs = centres[k0:k0 + c]
        oc.append(obs)
        anchor = centres[k0] if c == 0 else obs[len(obs) // 2]
        pos[i] = anchor + rng.normal(size=3) * rng.choice([2.0, 20.0, 300.0])
        refc[i] = obs[0] if c else anchor
    lvl = (np.arange(n_points) % levels).astype(np.int32)
    sf = (scale ** np.arange(levels)).astype(f32)
    sf = np.array([f32(1.0)] + [f32(f32(sf[l - 1]) * f32(scale)) for l in range(1, levels)], f32)     # ORBextractor's float chain
    n0 = rng.normal(size=(n_points, 3)).astype(f32)
    mx0, mn0 = rng.uniform(1, 2, n_points).astype(f32), rng.uniform(0, 1, n_points).astype(f32)
    return dict(off=off, centres=np.concatenate(oc).astype(f32), pos=pos, refc=refc, lvl=lvl, sf=sf, n0=n0, mx0=mx0, mn0=mn0, counts=counts)


def normal_depth_np(c, order="eigen"):
    """UpdateNormalAndDepth in float32 numpy, norm summed as Eigen does (x^2 + (y^2 + z^2)), as (x^2 + y^2) + z^2, or with fmaf."""
    def norm(v):
        x, y, z = v[..., 0], v[..., 1], v[..., 2]
        if order == "eigen":
            s = x * x + (y * y + z * z)
        elif order == "left":
            s = (x * x + y * y) + z * z
        else:       # fmaf(x, x, fmaf(y, y, z * z)): one rounding per fused step
            s = (x.astype(np.float64) * x + (y.astype(np.float64) * y + (z * z)).astype(f32)).astype(f32)
        return np.sqrt(s.astype(f32)).astype(f32)
    n = len(c["counts"])
    nrm, mx, mn = c["n0"].copy(), c["mx0"].copy(), c["mn0"].copy()
    for i in range(n):
        a, b = c["off"][i], c["off"][i + 1]
        if a == b:
            continue
        v = (c["pos"][i] - c["centres"][a:b]).astype(f32)
        u = (v / norm(v)[:, None]).astype(f32)
        acc = np.zeros(3, f32)
        for r in u:
            acc = (acc + r).astype(f32)
        dist = norm((c["pos"][i] - c["refc"][i]).astype(f32))
        mx[i] = f32(dist * c["sf"][c["lvl"][i]])
        mn[i] = f32(mx[i] / c["sf"][-1])
        nrm[i] = (acc / f32(b - a)).astype(f32)
    return nrm, mx, mn


# ---------------------------------------------------------------------------------------------------------------------------
# tests


def test_keyframes_have_the_callers_shape():
    for kind, n in (("stereo", 3), ("mono", 3)):
        kfs = keyframes(kind, n, 11 if kind == "stereo" else 21)
        cam = CAMS[kind]
        for kf in kfs:
            assert len(kf["kp"]) > 0.9 * NFEAT and (kf["kp"]["x"] < cam["w"]).all() and (kf["kp"]["y"] < cam["h"]).all()
            assert ((kf["uR"] >= 0).mean() > 0.3) == (kind == "stereo")
            assert (kf["node"] >= 0).mean() > 0.9 and len(np.unique(kf["node"][kf["node"] >= 0])) > 10      # many real nodes
        c = pair(kfs[0], kfs[1])
        assert (np.diff(c["node1"]) >= 0).all() and all((np.diff(c["src"][c["node1"] == n]) > 0).all() for n in np.unique(c["node1"]))
        assert not kfs[0]["has_mp"][c["src"]].any() and (c["valid2"] == ~kfs[1]["has_mp"]).all()
        assert np.isfinite(c["F12"]).all() and np.abs(c["F12"]).max() > 0
        # F12 is the fundamental matrix of the pair: x1^T F12 x2 == 0 for a world point seen by both
        X = np.array([0.3, -0.2, 4.0], f32)
        proj = lambda kf: np.array([*(kf["cam"]["fx"] * (kf["R"] @ X + kf["t"])[:2] / (kf["R"] @ X + kf["t"])[2]
                                      + np.array([kf["cam"]["cx"], kf["cam"]["cy"]])), 1.0])
        x1, x2 = proj(kfs[0]), proj(kfs[1])
        line = x1 @ c["F12"].reshape(3, 3).astype(np.float64)
        assert abs(line @ x2) / np.hypot(line[0], line[1]) < 0.01
        m, nm = oracle(c, False, True)
        assert nm > 30, nm                  # the neighbours share texture: many real matches
    assert ((pair(*keyframes("stereo", 3, 11)[:2], only_stereo=True)["stereo1"]) == 1).all()


def test_ties_exist_and_go_to_the_later_index():
    c = tri_case("ties")
    n = 0
    for q, rows, _ in c["meta"]["tags"]:
        cand = candidates(c, q)
        best = min(d for d, _ in cand)
        tied = sorted(i for d, i in cand if d == best)
        assert len(tied) >= 2 and set(rows) <= set(tied), (q, rows, cand)
        m, _ = oracle(c, False, False)
        assert m[q] == tied[-1]             # `dist > bestDist -> skip`: the last of equal distances
        n += 1
    assert n >= 20


def test_epipole_points_straddle_the_radius():
    c = tri_case("epipole")
    labels = {}
    for q, (i2,), label in c["meta"]["tags"]:
        assert c["stereo1"][q] == 0 and c["stereo2"][i2] == 0
        T = f32(f32(100) * c["sf"][c["kp2"]["octave"][i2]])
        v = epipole_value(c, c["kp2"]["x"][i2], c["kp2"]["y"][i2])
        assert v == {"epi_on": T, "epi_below": np.nextafter(T, f32(0)), "epi_above": np.nextafter(T, f32(np.inf))}[label]
        ds, _ = dsqr(c, q, c["kp2"]["x"][i2], c["kp2"]["y"][i2])
        assert float(ds) < 3.84 * float(c["s2"][0])                   # the epipolar gate passes: only the epipole gate decides
        m, _ = oracle(c, False, False)
        assert (m[q] == i2) == (label != "epi_below"), (label, m[q], i2)
        labels[label] = labels.get(label, 0) + 1
    assert min(labels.get(k, 0) for k in ("epi_on", "epi_below", "epi_above")) >= 6, labels      # most octaves have all three


def test_dsqr_lands_between_the_float_and_double_bound():
    c = tri_case("dsqr")
    targets = dsqr_targets(c["s2"])
    assert len(c["meta"]["tags"]) >= 4 and len(targets) >= 4
    for q, (i2,), _ in c["meta"]["tags"]:
        o = c["kp2"]["octave"][i2]
        v, _ = dsqr(c, q, c["kp2"]["x"][i2], c["kp2"]["y"][i2])
        in_double = float(v) < 3.84 * float(c["s2"][o])
        assert in_double == targets[o][1]
        assert in_double != (v < f32(f32(3.84) * c["s2"][o])) or in_double != (v < f32(3.84 * float(c["s2"][o])))
        m, _ = oracle(c, False, False)
        assert (m[q] == i2) == in_double


def test_den0_lines():
    c = tri_case("den0")
    assert (c["F12"] == 0).all() and np.isnan(c["ep"]).all()
    assert all(dsqr(c, q, 1.0, 1.0)[1] == 0 for q in range(0, len(c["src"]), 50))
    m, nm = oracle(c, False, False)
    assert nm == 0 and (m == -1).all()                # den == 0: only bCoarse accepts
    m, nm = oracle(c, True, False)
    assert nm > 30


def test_node_cases():
    c = tri_case("one_node")
    assert (c["node1"] == 0).all() and (c["node2"][c["node2"] >= 0] == 0).all()
    assert oracle(c, False, True)[1] > 30
    c = tri_case("node_neg")
    neg = c["node1"] < 0
    assert neg.sum() > 20
    m, nm = oracle(c, False, False)
    assert (m[neg] == -1).all() and nm > 30


def test_histogram_cases_have_the_intended_counts():
    for name, counts, keep in (("hist_ties", HIST_TIES, {1, 4, 8}), ("hist_tenth", HIST_TENTH, {2, 5})):
        c = tri_case(name)
        m, nm = oracle(c, False, False)
        got = {}
        near360 = 0
        for q, (i2,), label in c["meta"]["tags"]:
            assert m[q] == i2
            a1, a2 = c["kp1"]["angle"][q], c["kp2"]["angle"][i2]
            b_ = pyref.rot_bin(a1, a2)
            got[b_] = got.get(b_, 0) + 1
            r = f32(a1 - a2)
            near360 += bool(r < 0 and f32(r + f32(360)) >= f32(359.99))
        assert got == counts and nm == sum(counts.values())
        assert pyref.three_maxima([[0] * got.get(i, 0) for i in range(30)]) != (-1, -1, -1)
        kept = {i for i in pyref.three_maxima([[0] * got.get(i, 0) for i in range(30)]) if i >= 0}
        assert kept == keep
        m2, nm2 = oracle(c, False, True)
        assert nm2 == sum(counts[k] for k in keep)
        if name == "hist_tenth":
            assert near360 >= 1 and f32(0.1) * f32(20) == f32(2)       # 2 == 10 % of 20 exactly: kept, not refused


@pytest.mark.parametrize("name", TRI_CASES)
def test_oracle_matches_pyref_on_the_cases(name):
    c = tri_case(name)
    if name == "one_node":          # every query scans every feature: a slice keeps the pure-Python walk short
        c = dict(c, kp1=c["kp1"][:150], desc1=c["desc1"][:150], node1=c["node1"][:150], stereo1=c["stereo1"][:150])
    for coarse, check in ((False, False), (False, True), (True, True)):
        m, nm = oracle(c, coarse, check)
        rm, rnm = pyref.search_for_triangulation(c["kp1"], c["desc1"], c["node1"], c["stereo1"], c["kp2"], c["desc2"], c["node2"],
                                                 c["valid2"], c["stereo2"], c["F12"], c["ep"], c["sf"], c["s2"], coarse, check)
        assert nm == rnm and (m == rm).all(), (name, coarse, check)


def test_distinctive_lists_have_their_properties():
    sizes, kinds, lists = distinctive_lists()
    assert {n % 32 for n in sizes} >= {0, 1, 31} and any(n % 2 == 0 for n in sizes) and any(n % 2 for n in sizes) and max(sizes) == 2000
    ties = 0
    for n, kind, d in zip(sizes, kinds, lists):
        assert len(d) == n
        if kind == "identical":
            assert (d == d[0]).all() and po.distinctive_descriptor(d) == 0
            continue
        if n > 300:
            continue
        best, med = median_choice(d, int(0.5 * (n - 1)))
        assert best == po.distinctive_descriptor(d), (n, kind)
        ties += int((med == med.min()).sum() >= 2)
        differs = median_choice(d, n // 2)[0] != best
        assert differs or not (kind == "halves" and n % 2 == 0 and n >= 4), n     # rank N / 2 would choose another row
    assert ties >= 10, ties                                                         # tied medians


@pytest.mark.parametrize("distance", [10.0, 500.0, 2000.0])
def test_normal_depth_cases(distance):
    flipped = 0
    for scale, levels in PYRAMIDS:
        c = normal_depth_case(distance, scale, levels)
        assert (c["counts"] == 0).any() and c["counts"].max() >= 40 and set(c["lvl"]) == set(range(levels))
        far = np.linalg.norm(c["centres"], axis=1)
        assert (far > 0.8 * distance - 5).all() and (far < 1.2 * distance + 60).all()
        nrm, mx, mn = normal_depth_np(c)
        for i in range(0, len(c["counts"]), 7):
            if c["counts"][i] == 0:
                continue
            a, b = c["off"][i], c["off"][i + 1]
            rn, rmx, rmn = po.update_normal_and_depth(c["centres"][a:b], c["pos"][i], c["refc"][i], c["lvl"][i], c["sf"])
            assert (rn.view(np.uint32) == nrm[i].view(np.uint32)).all() and f32(rmx) == mx[i] and f32(rmn) == mn[i]
        for order in ("left", "fma"):
            o = normal_depth_np(c, order)
            flipped += int(not ((o[0].view(np.uint32) == nrm.view(np.uint32)).all() and (o[1] == mx).all()))
    assert flipped >= 2 * (distance >= 500.0)       # far out, another summation order changes some bits
