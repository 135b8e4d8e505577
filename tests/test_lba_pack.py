"""CPU tier: csrc/lba_pack.h -- the index structures k_lba walks and the batch layout it reads -- against a numpy restatement, on
synth.lba_problem and on the named windows of test_lba_windows.py, and lba_prepare's two refusals.  The emulation harness runs
lba_prepare + lba_pack with one host blob as both the pinned mirror and the device block."""
import ctypes as C

import numpy as np
import pytest

from orb_slam3_detailed_comments_b200 import _native as N
from orb_slam3_detailed_comments_b200.optimizer import Optimizer
from orb_slam3_detailed_comments_b200.synth import lba_problem
from test_lba_windows import CASES, window

ICH, SMEM_N, PCH, ALIGN = 128, 144, 8, 256      # LBA_ICH, LBA_SMEM_N, LBA_PCH and the packer's alignment
ORB_ERR_INVALID, ORB_ERR_UNSUPPORTED = -1, -5


@pytest.fixture(scope="module")
def emul():
    from _emul import build_and_load
    L = build_and_load()
    L.emul_lba_fields.restype = C.c_char_p
    L.emul_lba_pack.restype = C.c_int
    L.emul_lba_pack.argtypes = [C.POINTER(N.lba_problem), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def pack(L, problems):
    """(status, blob, [in, desc, work] bytes, one dict of descriptor members per problem: blob offsets / -1, and the ints)"""
    keep = []
    P = (N.lba_problem * len(problems))(*[Optimizer._pack(pr, 0.0, 10, keep)[0] for pr in problems])
    names = L.emul_lba_fields().decode().split()
    sizes = np.zeros(3, np.int64)
    status = L.emul_lba_pack(P, len(problems), None, N.ptr(sizes), None)
    if status != 0:
        return status, None, None, None
    blob = np.zeros(int(sizes.sum()), np.uint8)
    fields = np.zeros((len(problems), len(names)), np.int64)
    assert L.emul_lba_pack(P, len(problems), N.ptr(blob), N.ptr(sizes), N.ptr(fields)) == 0
    return 0, blob, sizes, [dict(zip(names, map(int, f))) for f in fields]


def restate(pr):
    """The index structures of one problem, restated: edges by map point and by free pose (edge order inside each), the upper
    pose-block pairs that share a landmark plus every diagonal, their co-observation items in landmark order, and the tasks."""
    fixed, ekf, emp = np.asarray(pr["fixed"]), np.asarray(pr["edge_kf"]), np.asarray(pr["edge_mp"])
    n_mp, n_e = len(pr["point"]), len(ekf)
    pidx = np.where(fixed == 0, np.cumsum(fixed == 0) - 1, -1).astype(np.int32)
    n_p = int((fixed == 0).sum())
    cnt = np.bincount(emp, minlength=n_mp)
    mp_start = np.concatenate([[0], np.cumsum(cnt)])
    mp_edge = np.argsort(emp, kind="stable")
    pe = pidx[ekf]
    free = np.flatnonzero(pe >= 0)
    pose_edge = free[np.argsort(pe[free], kind="stable")]
    pose_start = np.concatenate([[0], np.cumsum(np.bincount(pe[free], minlength=n_p))])
    pose_slot = np.full(n_e, -1)
    pose_slot[pose_edge] = np.arange(len(pose_edge))
    # every ordered pair (a, b) of edges of one landmark, landmark by landmark, a then b in mp_edge order
    lm = np.repeat(np.arange(n_mp), cnt)                          # landmark of each position of mp_edge
    ii = np.repeat(np.arange(n_e), cnt[lm])
    jj = mp_start[lm][ii] + np.arange(len(ii)) - np.repeat(np.cumsum(cnt[lm]) - cnt[lm], cnt[lm])
    a, b, l = mp_edge[ii], mp_edge[jj], lm[ii]
    p1, p2 = pe[a], pe[b]
    ok = (p1 >= 0) & (p2 >= p1) & ((p2 != p1) | (a == b))
    key = p1[ok].astype(np.int64) * n_p + p2[ok]
    order = np.argsort(key, kind="stable")
    items = np.stack([a[ok], b[ok], np.zeros(ok.sum(), np.int64), l[ok]], 1)[order]
    blocks = np.union1d(key, np.arange(n_p) * (n_p + 1))
    pair_start = np.concatenate([[0], np.searchsorted(key[order], blocks, "right")])
    task_start, block_task = [0], [0]
    for s, e in zip(pair_start[:-1], pair_start[1:]):
        task_start += [min(k + ICH, e) for k in range(s, e, ICH)]
        block_task.append(len(task_start) - 1)
    return dict(nP=n_p, pidx=pidx, mpStart=mp_start, mpEdge=mp_edge, poseStart=pose_start, poseEdge=pose_edge, poseSlot=pose_slot,
                blockP1=blocks // max(n_p, 1), blockP2=blocks % max(n_p, 1), pairStart=pair_start, ptItem=items,
                taskStart=np.array(task_start), blockTask=np.array(block_task))


INPUTS = ("pose0", "point0", "pidx", "ekf", "emp", "obs", "invs2", "mpStart", "mpEdge", "poseStart", "poseEdge", "pairStart", "ptItem",
          "taskStart", "blockTask", "poseSlot", "blockP1", "blockP2")


def needed_bytes(d):
    """bytes k_lba reads or writes through each pointer of descriptor d"""
    kf, mp, e, p, n, fe, nb, nt = d["nKF"], d["nMP"], d["nE"], d["nP"], d["n"], d["nFreeEdges"], d["nPairBlocks"], d["nTasks"]
    return dict(pose0=56 * kf, point0=24 * mp, pidx=4 * kf, ekf=4 * e, emp=4 * e, obs=24 * e, invs2=8 * e, mpStart=4 * (mp + 1),
                mpEdge=4 * e, poseStart=4 * (p + 1), poseEdge=4 * fe, pairStart=4 * (nb + 1), ptItem=0, taskStart=4 * (nt + 1),
                blockTask=4 * (nb + 1), poseSlot=4 * e, blockP1=4 * nb, blockP2=4 * nb, pose=56 * kf, point=24 * mp, poseSave=56 * kf,
                pointSave=24 * mp, Hpl=144 * e, W=216 * fe, posePart=216 * p * PCH, HsBlocks=288 * nb, bs=8 * n, xp=8 * n, partials=8 * 16,
                flags=4 * 3, taskSum=288 * nt, BD=144 * e, Hll=72 * mp, bl=24 * mp, Dinv=72 * mp, db=24 * mp, Hpp=288 * p, bp=48 * p,
                xl=24 * mp, HsGlobal=8 * n * n if n > SMEM_N else 0, err=8 * e, depthPos=e, stats=8 * 20)


def check(L, problems):
    status, blob, sizes, descs = pack(L, problems)
    assert status == 0
    n_in, n_desc, n_work = map(int, sizes)
    assert n_in % ALIGN == 0 and n_desc % ALIGN == 0 and n_desc >= 8 * len(problems)
    spans = []
    for pr, d in zip(problems, descs):
        R = restate(pr)

        def ints(name, count, k=1):
            a = np.frombuffer(blob, np.int32, count * k, d[name])
            return a if k == 1 else a.reshape(-1, k)
        n_e, n_mp, n_kf = len(pr["edge_kf"]), len(pr["point"]), len(pr["pose"])
        assert (d["nKF"], d["nMP"], d["nE"], d["nP"], d["n"]) == (n_kf, n_mp, n_e, R["nP"], 6 * R["nP"])
        assert d["nFreeEdges"] == len(R["poseEdge"]) and d["nPairBlocks"] == len(R["blockP1"]) and d["nTasks"] == len(R["taskStart"]) - 1
        assert d["nItems"] == 0 and d["ptItemStart"] == -1 and d["Prod"] == -1      # k_lba reads none of them
        # inputs copied as given
        np.testing.assert_array_equal(np.frombuffer(blob, np.float64, 7 * n_kf, d["pose0"]), np.ravel(pr["pose"]))
        np.testing.assert_array_equal(np.frombuffer(blob, np.float64, 3 * n_mp, d["point0"]), np.ravel(pr["point"]))
        np.testing.assert_array_equal(np.frombuffer(blob, np.float64, 3 * n_e, d["obs"]), np.ravel(pr["obs"]))
        np.testing.assert_array_equal(np.frombuffer(blob, np.float64, n_e, d["invs2"]), pr["inv_sigma2"])
        np.testing.assert_array_equal(ints("ekf", n_e), pr["edge_kf"])
        np.testing.assert_array_equal(ints("emp", n_e), pr["edge_mp"])
        # index structures
        np.testing.assert_array_equal(ints("pidx", n_kf), R["pidx"])
        np.testing.assert_array_equal(ints("mpStart", n_mp + 1), R["mpStart"])
        np.testing.assert_array_equal(ints("mpEdge", n_e), R["mpEdge"])
        np.testing.assert_array_equal(ints("poseStart", R["nP"] + 1), R["poseStart"])
        np.testing.assert_array_equal(ints("poseEdge", d["nFreeEdges"]), R["poseEdge"])
        np.testing.assert_array_equal(ints("poseSlot", n_e), R["poseSlot"])
        slot = ints("poseSlot", n_e)
        np.testing.assert_array_equal(slot[ints("poseEdge", d["nFreeEdges"])], np.arange(d["nFreeEdges"]))
        np.testing.assert_array_equal(ints("blockP1", d["nPairBlocks"]), R["blockP1"])
        np.testing.assert_array_equal(ints("blockP2", d["nPairBlocks"]), R["blockP2"])
        pair_start = ints("pairStart", d["nPairBlocks"] + 1)
        np.testing.assert_array_equal(pair_start, R["pairStart"])
        np.testing.assert_array_equal(ints("ptItem", int(pair_start[-1]), 4), R["ptItem"])
        task_start, block_task = ints("taskStart", d["nTasks"] + 1), ints("blockTask", d["nPairBlocks"] + 1)
        np.testing.assert_array_equal(task_start, R["taskStart"])
        np.testing.assert_array_equal(block_task, R["blockTask"])
        assert (np.diff(task_start) <= ICH).all() and (np.diff(task_start) > 0).all()
        np.testing.assert_array_equal(task_start[block_task], pair_start)      # a task never crosses a pose-block pair
        need = needed_bytes(d)
        need["ptItem"] = 16 * int(pair_start[-1])
        for name, nbytes in need.items():
            lo, hi = (0, n_in) if name in INPUTS else (n_in + n_desc, n_in + n_desc + n_work)
            assert d[name] % ALIGN == 0 and lo <= d[name] and d[name] + nbytes <= hi, name
            spans.append((d[name], max(nbytes, 1), name))
    spans.sort()
    for (o1, n1, a), (o2, _, b) in zip(spans, spans[1:]):
        assert o1 + n1 <= o2, (a, b)


def test_synth_problem(emul):
    check(emul, [lba_problem(n_kf=20, n_fixed=2, n_mp=3000, seed=0)])


@pytest.mark.parametrize("case", list(CASES))
def test_named_windows(emul, case):
    check(emul, [window(**CASES[case])])


def test_batch(emul):
    """one layout for a batch: every problem's structures in place, no array of one overlapping another's"""
    check(emul, [lba_problem(n_kf=12, n_fixed=2, n_mp=800, seed=1), window(**CASES["edgeless_kf"]),
                 window(**CASES["fixed_only_points"]), lba_problem(n_kf=30, n_fixed=4, n_mp=500, seed=2)])


def test_refusals(emul):
    pr = lba_problem(n_kf=20, n_fixed=0, n_mp=300, seed=3)
    for n_kf, status in ((160, 0), (161, ORB_ERR_UNSUPPORTED)):      # free keyframes without edges still count
        big = dict(pr, pose=np.tile(pr["pose"][:1], (n_kf, 1)), fixed=np.zeros(n_kf, np.uint8))
        assert pack(emul, [big])[0] == status, n_kf
    for key, value in (("edge_kf", -1), ("edge_kf", 20), ("edge_mp", -1), ("edge_mp", 300)):
        bad = dict(pr)
        bad[key] = pr[key].copy()
        bad[key][7] = value
        assert pack(emul, [pr, bad])[0] == ORB_ERR_INVALID, (key, value)
