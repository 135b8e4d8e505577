"""CPU tier, build container only: host/Frame_bow_b200.cc -- the translation unit that replaces Frame::ComputeBoW -- over a mock ORBVocabulary
whose nodes are protected members like DBoW2's (read through a derived class, no header change), with orbv_create / orbv_transform answered
by the CPU oracle (tests/host/voc_stub.cc).  The oracle's transform is pinned against the reference's own DBoW2 on ORBvoc.txt
(tests/test_oracle_vs_ref_dbow.py); what is checked here is the unit's own work: the flattening (children order, word ids and weights of the
leaves, depth), one flattening per vocabulary object, mBowVec in ascending word order with the oracle's doubles, mFeatVec listing feature i
under its level-4 node iff its word's weight is > 0, and the early return when mBowVec is already filled."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import synthetic_vocabulary

HERE = os.path.dirname(os.path.abspath(__file__))
MINE = os.path.join(HERE, "host", "voc_cpu_mine")


def _build():
    if os.path.exists(os.path.join(po.REFERENCE_ROOT, "include", "ORBextractor.h")):
        subprocess.check_call(["bash", os.path.join(HERE, "host", "build_voc_cpu.sh")])
    return os.path.exists(MINE)


pytestmark = pytest.mark.skipif(not _build(), reason="tests/host/voc_cpu_mine not built and /root/reference absent")


@pytest.mark.parametrize("k,L,seed,stop", [(8, 3, 1, 0.05), (10, 5, 2, 0.02), (4, 6, 3, 0.2)])
def test_compute_bow_fills_the_containers_like_dbow2(tmp_path, k, L, seed, stop):
    voc = synthetic_vocabulary(k=k, L=L, seed=seed, stop_fraction=stop)
    rng = np.random.default_rng(seed)
    N = 700
    leaves = np.nonzero(np.asarray(voc["node_word"]) >= 0)[0]
    desc = np.asarray(voc["node_desc"], np.uint8).reshape(-1, 32)[rng.choice(leaves, N)].copy()       # near words, a few bits off
    flip = rng.integers(0, 256, (N, 6))
    for i in range(N):
        for b in flip[i]:
            desc[i, b // 8] ^= np.uint8(1 << (b % 8))
    d = str(tmp_path)
    for name, dt in (("child_offset", np.int32), ("child_ids", np.int32), ("node_word", np.int32)):
        np.ascontiguousarray(voc[name], dt).tofile(os.path.join(d, name + ".i32"))
    np.int32([voc["L"]]).tofile(os.path.join(d, "meta.i32"))
    np.ascontiguousarray(voc["node_desc"], np.uint8).tofile(os.path.join(d, "node_desc.u8"))
    np.ascontiguousarray(voc["node_weight"], np.float64).tofile(os.path.join(d, "node_weight.f64"))
    desc.tofile(os.path.join(d, "desc.u8"))
    r = subprocess.run([MINE, d], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "voc_cpu ok" in r.stdout, (r.returncode, r.stdout[-1000:], r.stderr[-1000:])
    oi, ow = np.fromfile(os.path.join(d, "out.i32"), np.int32).tolist(), np.fromfile(os.path.join(d, "out.f64"), np.float64)
    pos, wpos = 0, 0
    for n in (N, N // 2):
        want = po.bow_transform(voc, desc[:n], 4)
        nb = oi[pos]; pos += 1
        words = np.array(oi[pos:pos + nb]); pos += nb
        weights = ow[wpos:wpos + nb]; wpos += nb
        assert nb == len(want["bow_word"]) and (words == want["bow_word"]).all() and (np.diff(words) > 0).all()
        assert (weights.view(np.uint64) == want["bow_weight"].view(np.uint64)).all()
        nf = oi[pos]; pos += 1
        got = {}
        for _ in range(nf):
            node, cnt = oi[pos], oi[pos + 1]; pos += 2
            got[node] = oi[pos:pos + cnt]; pos += cnt
        exp = {}
        for i in range(n):
            if want["weight"][i] > 0:
                exp.setdefault(int(want["node"][i]), []).append(i)
        assert got == exp and list(got) == sorted(got)
        assert (want["weight"] == 0).any() or stop < 0.03          # stopped words occur: the weight > 0 rule is exercised
    assert oi[pos] == 1 and pos == len(oi) - 1                     # one orbv_create for two frames
