"""Generates tests/golden/orbvoc_subtree.npz from the reference's own vocabulary fixture (Vocabulary/ORBvoc.txt.tar.gz,
k = 10, L = 6, 1 082 072 nodes): a pruned copy of the REAL tree -- every node 64 seeded descriptors visit on their way down plus
all the siblings they are compared with, so the walk over the pruned tree is the walk over the full tree -- and the expected
word / node / weight / BowVector computed on the FULL tree by the numpy restatement in tests/pyref.py.  The same for the ORB
descriptors of one synthetic frame (oracle extractor, 320x240, 500 features): Frame::ComputeBoW end to end on the real vocabulary.
Run here (the reference is not available on the GPU box):  python tests/golden/make_golden_voc.py"""
import os
import sys
import tarfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
import pyref  # noqa: E402
from orb_slam3_detailed_comments_b200.vocabulary import load_orbvoc_text  # noqa: E402
from oracle.pyoracle import REFERENCE_ROOT  # noqa: E402

TAR = os.path.join(REFERENCE_ROOT, "Vocabulary", "ORBvoc.txt.tar.gz")


def load_full():
    with tarfile.open(TAR, "r:gz") as tf:
        return load_orbvoc_text(tf.extractfile("ORBvoc.txt"))


def golden_descriptors(voc, n=64, seed=2024):
    """Leaf descriptors of the real vocabulary with 0..60 random bits flipped (realistic paths, incl. shallow leaves and
    zero-weight words), a few inner-node descriptors, and a few uniformly random rows."""
    rng = np.random.default_rng(seed)
    co = voc["child_offset"]
    leaves = np.nonzero(voc["node_word"] >= 0)[0]
    nchild = np.diff(co)
    parent = np.zeros(len(nchild), np.int64)
    parent[voc["child_ids"]] = np.repeat(np.arange(len(nchild)), nchild)
    depth = np.zeros(len(nchild), np.int64)
    for i in range(1, len(nchild)):
        depth[i] = depth[parent[i]] + 1
    shallow = leaves[depth[leaves] < voc["L"]]
    zero_w = leaves[voc["node_weight"][leaves] == 0]

    def lands_on(cands, want):          # descriptors of `cands` whose own walk ends on a node for which want(node) holds
        got = []
        for c in cands:
            fid = 0
            while co[fid] != co[fid + 1]:
                kids = voc["child_ids"][co[fid]:co[fid + 1]]
                fid = int(kids[int(np.argmin(pyref.POP[voc["node_desc"][kids] ^ voc["node_desc"][c][None, :]].sum(1)))])
            if want(fid):
                got.append(c)
            if len(got) == 8:
                break
        return np.array(got, np.int64)

    sh = lands_on(rng.permutation(shallow), lambda f: depth[f] < voc["L"])
    zw = lands_on(rng.permutation(zero_w)[:5000], lambda f: voc["node_weight"][f] == 0)
    few = lands_on(rng.permutation(leaves[nchild[parent[leaves]] < 10])[:400], lambda f: nchild[parent[f]] < 10)
    sh = np.concatenate([sh, few])          # (kept in one group: descriptors left unperturbed)
    print('self-landing shallow leaves + leaves under narrow parents', len(sh), 'zero-weight leaves', len(zw))
    assert len(sh) >= 4 and len(zw) >= 2
    picks = np.concatenate([rng.choice(leaves, n - 4 - len(sh) - len(zw)), sh, zw, rng.choice(np.nonzero(nchild > 0)[0][1:], 4)])
    out = voc["node_desc"][picks].copy()
    for r in range(n - 4 - len(sh) - len(zw)):
        for b in rng.integers(0, 256, int(rng.integers(0, 61))):
            out[r, b // 8] ^= np.uint8(1 << (b % 8))
    out = np.concatenate([out, rng.integers(0, 256, (4, 32), dtype=np.uint8)])
    return np.ascontiguousarray(out[rng.permutation(len(out))])


def prune(voc, desc):
    co, ch = voc["child_offset"], voc["child_ids"]
    keep, expanded = {0}, set()
    for d in desc:
        fid = 0
        while co[fid] != co[fid + 1]:
            kids = ch[co[fid]:co[fid + 1]]
            keep.update(int(k) for k in kids)
            expanded.add(fid)
            fid = int(kids[int(np.argmin(pyref.POP[voc["node_desc"][kids] ^ d[None, :]].sum(1)))])
    orig = np.array(sorted(keep), np.int64)                 # ascending original id keeps parent-before-child and sibling order
    new_of = {int(o): i for i, o in enumerate(orig)}
    child_offset, child_ids = [0], []
    for o in orig:
        if int(o) in expanded:
            child_ids += [new_of[int(k)] for k in ch[co[o]:co[o + 1]]]
        child_offset.append(len(child_ids))
    return dict(child_offset=np.array(child_offset, np.int32), child_ids=np.array(child_ids, np.int32), node_desc=voc["node_desc"][orig],
                node_word=voc["node_word"][orig], node_weight=voc["node_weight"][orig], L=voc["L"]), orig


FRAME = dict(w=320, h=240, seed=4, sigma=3.0, nrect=20, nfeatures=500)   # a case tests/test_extractor_gpu.py holds bit-exact on an H100


def frame_descriptors():
    from oracle import pyoracle as po
    from orb_slam3_detailed_comments_b200 import synth
    ex = po.OracleExtractor(FRAME["nfeatures"], 1.2, 8, 20, 7)
    _, _, d = ex(synth.frame(FRAME["w"], FRAME["h"], FRAME["seed"], FRAME["sigma"], FRAME["nrect"]))
    return d


if __name__ == "__main__":
    full = load_full()
    desc = golden_descriptors(full)
    ref = pyref.bow_transform(full, desc, 4)
    fdesc = frame_descriptors()
    fref = pyref.bow_transform(full, fdesc, 4)
    sub, orig = prune(full, np.concatenate([desc, fdesc]))
    nchild = np.diff(full["child_offset"])
    np.savez_compressed(os.path.join(HERE, "orbvoc_subtree.npz"), desc=desc, orig_id=orig.astype(np.int32),
                        full_nodes=np.int64(len(nchild)), full_words=np.int64((full["node_word"] >= 0).sum()),
                        full_children_hist=np.bincount(nchild, minlength=11),
                        word=ref["word"], node=ref["node"], weight=ref["weight"], bow_word=ref["bow_word"], bow_weight=ref["bow_weight"],
                        frame_desc=fdesc, frame_word=fref["word"], frame_node=fref["node"], frame_weight=fref["weight"],
                        frame_bow_word=fref["bow_word"], frame_bow_weight=fref["bow_weight"],
                        **{"sub_" + k: np.asarray(v) for k, v in sub.items()})
    print("nodes kept", len(orig), "of", len(nchild), "; words hit", len(set(ref["word"].tolist())), "; zero-weight features",
          int((ref["weight"] == 0).sum()), "; size", os.path.getsize(os.path.join(HERE, "orbvoc_subtree.npz")))
