"""GPU tier (runs last): orbv_transform over a pruned copy of the REAL ORBvoc.txt tree (tests/golden/orbvoc_subtree.npz: real node
descriptors and idf weights, 2..10 children per node, leaves at several depths, zero-weight words, childless pruned branches)
against the CPU oracle, on the descriptors the extractor produced.  Added after round 1's last GPU run, so it sorts after the
suites that have been green on an H100; the kernel path is the one tests/test_bow_gpu.py covers on synthetic uniform trees."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200 import ORBextractor, ORBVocabulary, synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _voc():
    z = np.load(os.path.join(HERE, "golden", "orbvoc_subtree.npz"))
    voc = {k[4:]: z[k] for k in z.files if k.startswith("sub_")}
    voc["L"] = int(voc["L"])
    return z, voc


def test_compute_bow_of_a_frame_matches_the_full_vocabulary_golden():
    """Frame::ComputeBoW end to end: device extraction (320x240, 500 features: a case test_extractor_gpu.py holds bit-exact) of the fixture frame, device transform over the real tree's
    pruned copy, against the values the FULL ORBvoc.txt tree gives (tests/golden/make_golden_voc.py)."""
    z, voc = _voc()
    ex = ORBextractor(500, 1.2, 8, 20, 7, max_width=320, max_height=240, max_batch=1)
    ex.extract_batch(synth.frame(320, 240, 4, 3.0, 20)[None])
    n, mono, off, kps, desc = ex.download(1)
    assert desc.shape == z["frame_desc"].shape and (desc == z["frame_desc"]).all()
    V = ORBVocabulary(voc["child_offset"], voc["child_ids"], voc["node_desc"], voc["node_word"], voc["node_weight"], voc["L"])
    got = V.transform(ex, int(off[-1]), 1, levelsup=4)
    assert (got["word"] == z["frame_word"]).all() and (z["orig_id"][got["node"]] == z["frame_node"]).all()
    assert (got["weight"].view(np.uint64) == z["frame_weight"].view(np.uint64)).all()
    assert (got["bow_word"][0] == z["frame_bow_word"]).all()
    assert (got["bow_weight"][0].view(np.uint64) == z["frame_bow_weight"].view(np.uint64)).all()
    V.close()
    ex.close()


@pytest.mark.parametrize("levelsup", [4, 2])
def test_transform_on_the_pruned_real_vocabulary(levelsup):
    z, voc = _voc()
    W, H, nimg = 640, 480, 2
    imgs = np.stack([synth.frame(W, H, 70 + i) for i in range(nimg)])
    ex = ORBextractor(1200, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=nimg)
    ex.extract_batch(imgs)
    n, mono, off, kps, desc = ex.download(nimg)
    V = ORBVocabulary(voc["child_offset"], voc["child_ids"], voc["node_desc"], voc["node_word"], voc["node_weight"], voc["L"])
    got = V.transform(ex, int(off[-1]), nimg, levelsup=levelsup)
    for i in range(nimg):
        a, b = int(off[i]), int(off[i + 1])
        r = po.bow_transform(voc, desc[a:b], levelsup)
        assert (got["word"][a:b] == r["word"]).all() and (got["node"][a:b] == r["node"]).all()
        assert (got["weight"][a:b].view(np.uint64) == r["weight"].view(np.uint64)).all()
        assert len(got["bow_word"][i]) == len(r["bow_word"]) and (got["bow_word"][i] == r["bow_word"]).all()
        assert (got["bow_weight"][i].view(np.uint64) == r["bow_weight"].view(np.uint64)).all()
    V.close()
    ex.close()
