"""CPU tier: the BoW oracle (orc_bow_transform) pinned on the reference's own vocabulary fixture.
tests/golden/orbvoc_subtree.npz is a pruned copy of the REAL ORBvoc.txt tree (k = 10, L = 6; variable child counts, leaves at depths
4-6, zero-weight words) along the paths of 68 descriptors, with the expected outputs computed on the FULL tree by the independent numpy
restatement tests/pyref.bow_transform (tests/golden/make_golden_voc.py).  When /root/reference is present (this container, not the
GPU box) the whole 1 082 073-node vocabulary is also loaded and walked by both."""
import io
import os
import tarfile

import numpy as np
import pytest

import pyref
from oracle import pyoracle as po
from orb_slam3_detailed_comments_b200.vocabulary import load_orbvoc_text

HERE = os.path.dirname(os.path.abspath(__file__))
TAR = os.path.join(po.REFERENCE_ROOT, "Vocabulary", "ORBvoc.txt.tar.gz")


@pytest.fixture(scope="module")
def gold():
    z = np.load(os.path.join(HERE, "golden", "orbvoc_subtree.npz"))
    sub = {k[4:]: z[k] for k in z.files if k.startswith("sub_")}
    sub["L"] = int(sub["L"])
    return z, sub


def test_fixture_is_the_real_tree_shape(gold):
    z, sub = gold
    assert int(z["full_nodes"]) == 1082073 and int(z["full_words"]) == 971814 and sub["L"] == 6
    hist = z["full_children_hist"]
    assert hist[10] == 105763 and hist[2:10].sum() > 4000          # most inner nodes have 10 children, several thousand have 2..9
    nchild = np.diff(sub["child_offset"])
    assert set(np.unique(nchild[nchild > 0])) - {10} != set()      # the pruned paths cross nodes with fewer than 10 children
    assert (z["weight"] == 0).sum() >= 2                            # stopped (zero-weight) words are hit


def test_oracle_matches_golden_on_the_pruned_real_tree(gold):
    z, sub = gold
    r = po.bow_transform(sub, z["desc"], 4)
    assert (r["word"] == z["word"]).all()
    assert (z["orig_id"][r["node"]] == z["node"]).all()
    assert (r["weight"].view(np.uint64) == z["weight"].view(np.uint64)).all()
    assert (r["bow_word"] == z["bow_word"]).all()
    assert (r["bow_weight"].view(np.uint64) == z["bow_weight"].view(np.uint64)).all()
    assert len(r["bow_word"]) == len(set(z["word"][z["weight"] > 0].tolist()))        # stopped words do not enter the BowVector


def test_compute_bow_of_an_extracted_frame_on_the_real_vocabulary(gold):
    """Frame::ComputeBoW end to end: the oracle extractor's descriptors of the fixture frame, walked down the (pruned) real tree."""
    from orb_slam3_detailed_comments_b200 import synth
    z, sub = gold
    ex = po.OracleExtractor(500, 1.2, 8, 20, 7)
    _, _, d = ex(synth.frame(320, 240, 4, 3.0, 20))
    assert d.shape == z["frame_desc"].shape and (d == z["frame_desc"]).all()
    r = po.bow_transform(sub, d, 4)
    assert (r["word"] == z["frame_word"]).all() and (z["orig_id"][r["node"]] == z["frame_node"]).all()
    assert (r["weight"].view(np.uint64) == z["frame_weight"].view(np.uint64)).all()
    assert (r["bow_word"] == z["frame_bow_word"]).all()
    assert (r["bow_weight"].view(np.uint64) == z["frame_bow_weight"].view(np.uint64)).all()
    assert len(r["bow_word"]) > 150 and abs(r["bow_weight"].sum() - 1.0) < 1e-12
    assert len(set(z["frame_node"].tolist())) > 50                  # mFeatVec: features spread over many level-2 nodes


def test_numpy_restatement_agrees_on_the_pruned_tree(gold):
    z, sub = gold
    for levelsup in (4, 2, 7):
        a, b = pyref.bow_transform(sub, z["desc"], levelsup), po.bow_transform(sub, z["desc"], levelsup)
        assert (a["word"] == b["word"]).all() and (a["node"] == b["node"]).all() and (a["weight"] == b["weight"]).all()
        assert (a["bow_word"] == b["bow_word"]).all() and (a["bow_weight"].view(np.uint64) == b["bow_weight"].view(np.uint64)).all()


def test_text_loader_on_a_small_file():
    text = b"3 2  0 0\n" + b"".join(
        b"%d %d %s %g\n" % (p, leaf, b" ".join(b"%d" % ((7 * i + j) % 256) for j in range(32)) + b" ", w)
        for i, (p, leaf, w) in enumerate([(0, 0, 0), (0, 1, 1.5), (0, 0, 0), (1, 1, 2.25), (1, 1, 0), (3, 1, 3.0), (3, 1, 0.5)]))
    v = load_orbvoc_text(io.BytesIO(text))
    assert v["k"] == 3 and v["L"] == 2 and len(v["node_word"]) == 8
    assert v["child_offset"].tolist() == [0, 3, 5, 5, 7, 7, 7, 7, 7] and v["child_ids"].tolist() == [1, 2, 3, 4, 5, 6, 7]
    assert v["node_word"].tolist() == [-1, -1, 0, -1, 1, 2, 3, 4] and v["node_weight"][4] == 2.25 and v["node_desc"][2, 3] == (7 * 1 + 3)
    with pytest.raises(ValueError):
        load_orbvoc_text(io.BytesIO(b"10 6 1 0\n0 1 " + b"0 " * 32 + b"1\n"))


@pytest.mark.skipif(not os.path.exists(TAR), reason="the reference's vocabulary fixture is only present in the build container")
def test_full_vocabulary_oracle_vs_numpy(gold):
    z, sub = gold
    with tarfile.open(TAR, "r:gz") as tf:
        full = load_orbvoc_text(tf.extractfile("ORBvoc.txt"))
    assert len(full["node_word"]) == int(z["full_nodes"])
    rng = np.random.default_rng(5)
    leaves = np.nonzero(full["node_word"] >= 0)[0]
    extra = full["node_desc"][rng.choice(leaves, 300)].copy()
    for r in range(len(extra)):
        for b in rng.integers(0, 256, int(rng.integers(0, 80))):
            extra[r, b // 8] ^= np.uint8(1 << (b % 8))
    desc = np.concatenate([z["desc"], extra, rng.integers(0, 256, (32, 32), dtype=np.uint8)])
    a, b = pyref.bow_transform(full, desc, 4), po.bow_transform(full, desc, 4)
    assert (a["word"] == b["word"]).all() and (a["node"] == b["node"]).all() and (a["weight"] == b["weight"]).all()
    assert (a["bow_word"] == b["bow_word"]).all() and (a["bow_weight"].view(np.uint64) == b["bow_weight"].view(np.uint64)).all()
    n = len(z["desc"])                                   # and the committed golden vectors are what the full tree gives
    assert (b["word"][:n] == z["word"]).all() and (b["node"][:n] == z["node"]).all()
    f = po.bow_transform(full, z["frame_desc"], 4)
    assert (f["word"] == z["frame_word"]).all() and (f["node"] == z["frame_node"]).all() and (f["bow_word"] == z["frame_bow_word"]).all()
    assert (f["bow_weight"].view(np.uint64) == z["frame_bow_weight"].view(np.uint64)).all()
