"""CPU tier, build container only: host/ORBmatcher_fuse_b200.cc -- the translation unit that replaces ORBmatcher::Fuse(pKF, vpMapPoints, th) --
against the REFERENCE's own function (src/ORBmatcher.cc:1325-1544, compiled verbatim in oracle/_ref part 2).  The unit's search is answered
by the CPU oracle (tests/host/fuse_stub.cc) over the arrays it marshals -- among them MapPoint's RAW mfMinDistance / mfMaxDistance, read
through a derived class because they are protected.  Compared: the feature every query is fused into (the reference's GetMapPoint(bestIdx)
calls, in order) and the return value; and, against a restatement of :1508-1532 over the mock map, which mutation follows: Replace in
the direction of the point with more observations, nothing when the keyframe's point is bad, AddObservation + AddMapPoint otherwise --
including queries that land on a feature an earlier query of the same call has just been added to."""
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
MINE = os.path.join(HERE, "host", "fuse_cpu_mine")


def _build():
    if os.path.exists(os.path.join(po.REFERENCE_ROOT, "src", "ORBmatcher.cc")):
        subprocess.check_call(["bash", os.path.join(HERE, "host", "build_fuse_cpu.sh")])
    return os.path.exists(MINE) and po.build_ref2() is not None


pytestmark = pytest.mark.skipif(not _build(), reason="tests/host/fuse_cpu_mine / oracle/_ref part 2 not built and /root/reference absent")
_spec = importlib.util.spec_from_file_location("_m2f", os.path.join(HERE, "test_oracle_vs_ref_matcher2.py"))
_m = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_m)
two_frames, kf_target = _m.two_frames, _m.kf_target


@pytest.mark.parametrize("th", [3.0, 8.0])
def test_fuse_equals_the_reference_function(tmp_path, two_frames, kf_target, th):
    (k1, d1, u1, dep1), (k2, d2, u2, dep2), sf = two_frames
    rng = np.random.default_rng(int(th))
    T, isg, F = kf_target["T"], kf_target["isg"], kf_target["F"]
    has_mp = rng.random(len(k2)) < 0.3
    K = po.RefKeyFrame(k2, d2, u2, None, has_mp, None, sf, sf * sf, _m.CAM6[:4], T)
    po.ref2_kf_set_geometry(K, F, isg, _m.BF)
    q = _m._queries(k1, d1, dep1, rng, sf, 0.3)
    nobj = len(q["desc"])
    in_kf = (rng.random(nobj) < 0.05).astype(np.uint8)
    rf, rn = po.ref2_fuse(K, q, th, in_kf)
    # the mock map: Observations() of both sides, a bad map point in the keyframe now and then, NULL entries in vpMapPoints
    qobs, kfobs = rng.integers(1, 6, nobj).astype(np.int32), rng.integers(0, 6, len(k2)).astype(np.int32)
    slot = np.arange(nobj, dtype=np.int32)
    slot = np.insert(slot, rng.integers(0, nobj, 20), -1).astype(np.int32)
    d = str(tmp_path)
    np.ascontiguousarray(k2).tofile(os.path.join(d, "kf.kp"))
    for name, a in dict(kf_desc=d2, kf_has_mp=has_mp, q_desc=q["desc"], q_bad=q["bad"], q_in_kf=in_kf).items():
        np.ascontiguousarray(a, np.uint8).tofile(os.path.join(d, name + ".u8"))
    for name, a in dict(kf_uright=u2, q_xw=q["world_pos"], q_normal=q["normal"], q_max=q["max_dist"], q_min=q["min_dist"]).items():
        np.ascontiguousarray(a, np.float32).tofile(os.path.join(d, name + ".f32"))
    for name, a in dict(kf_mp_obs=kfobs, q_obs=qobs, q_slot=slot).items():
        np.ascontiguousarray(a, np.int32).tofile(os.path.join(d, name + ".i32"))
    np.concatenate([_m.CAM6, _m.BOUNDS, np.float32(T), np.float32([th, kf_target["logsf"]])]).astype(np.float32).tofile(os.path.join(d, "params.f32"))
    # inputs of the relocalisation search (second half of the driver): keyframe 1 with its own map points as queries
    orb_dist, check = (100, True) if th < 5 else (64, False)
    has1 = dep1 > 0
    bad1 = has1 & (rng.random(len(k1)) < 0.04)
    pts1 = _m._unproject(k1, np.where(has1, dep1, 1.0))
    dist1 = np.linalg.norm(pts1, axis=1).astype(np.float32)
    maxd1 = (dist1 * sf[k1["octave"]]).astype(np.float32)
    mind1 = (maxd1 / sf[7]).astype(np.float32)
    already, claimed = (rng.random(len(k1)) < 0.1).astype(np.uint8), (rng.random(len(k2)) < 0.1).astype(np.uint8)
    np.ascontiguousarray(k1).tofile(os.path.join(d, "r_kf.kp"))
    for name, a in dict(r_has=has1, r_bad=bad1, r_already=already, r_claimed=claimed, r_desc=d1).items():
        np.ascontiguousarray(a, np.uint8).tofile(os.path.join(d, name + ".u8"))
    for name, a in dict(r_xw=pts1, r_max=maxd1, r_min=mind1, r_params=np.float32([10.0 if th < 5 else 3.0, orb_dist, float(check)])).items():
        np.ascontiguousarray(a, np.float32).tofile(os.path.join(d, name + ".f32"))
    # inputs of the two Sim3 searches (third part of the driver)
    sc = 1.03
    S = _m._sim3(T[:4], T[4:].astype(np.float64) * sc, sc)
    ratio = 1.0 if th < 5 else 0.8
    sclaimed = (rng.random(len(k2)) < 0.2).astype(np.uint8)
    np.concatenate([S, np.float32([th, ratio])]).astype(np.float32).tofile(os.path.join(d, "s_params.f32"))
    sclaimed.tofile(os.path.join(d, "s_claimed.u8"))
    r = subprocess.run([MINE, d], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "fuse_cpu ok" in r.stdout, (r.returncode, r.stdout[-1000:], r.stderr[-1000:])
    out = np.fromfile(os.path.join(d, "out_log.i32"), np.int32)
    ret, log = int(out[-1]), out[:-1].reshape(-1, 4).tolist()
    # expected mutations from the reference's best features, :1508-1532 over the mock's semantics (Replace marks the replaced point bad)
    holder = {int(i): dict(id=100000 + int(i), obs=int(kfobs[i]) + 1, bad=False) for i in np.nonzero(has_mp)[0]}
    want, fused = [], 0
    for j in range(nobj):
        if q["bad"][j] or in_kf[j] or rf[j] < 0:
            continue
        b, me = int(rf[j]), dict(id=j, obs=int(qobs[j]), bad=False)
        hb = holder.get(b)
        if hb is not None:
            if not hb["bad"]:
                if hb["obs"] > me["obs"]:
                    want.append([1, me["id"], hb["id"], -1])
                else:
                    want.append([1, hb["id"], me["id"], -1]); hb["bad"] = True
        else:
            want.append([3, j, -1, b]); me["obs"] += 1; holder[b] = me
        fused += 1
    assert ret == rn == fused and log == want
    assert rn > 100 and sum(1 for w in want if w[0] == 1) > 10 and sum(1 for w in want if w[0] == 3) > 50
    # the Sim3 searches against the reference's own functions (a fresh keyframe: no bad points, nothing fused yet)
    so = np.fromfile(os.path.join(d, "out_sim3.i32"), np.int32).tolist()
    N2 = len(k2)
    K3 = po.RefKeyFrame(k2, d2, u2, None, has_mp, None, sf, sf * sf, _m.CAM6[:4], T)
    po.ref2_kf_set_geometry(K3, F, isg, _m.BF)
    wm, wn, _, _ = po.ref2_search_kf_sim3(K3, S, q, sclaimed, int(th), ratio)
    matched, r3, kfs_overload_agrees = np.array(so[:N2]), so[N2], so[N2 + 1]
    so = so[:N2 + 1] + so[N2 + 2:]
    wm2, wn2, _, _ = po.ref2_search_kf_sim3(K3, S, q, sclaimed, int(th), ratio, with_kfs=True)        # the reference's vpPointsKFs overload: the same matches
    assert kfs_overload_agrees == 1 and wn2 == wn and (wm2 == wm).all()
    exp = np.where(sclaimed != 0, -2, -1)
    for j in np.nonzero(wm >= 0)[0]:
        exp[wm[j]] = j
    assert r3 == wn and (matched == exp).all() and wn > 100
    wf, wfn, _, _ = po.ref2_fuse_sim3(K3, S, q, th)
    repl, r4, nlog = np.array(so[N2 + 1:N2 + 1 + nobj]), so[N2 + 1 + nobj], so[N2 + 2 + nobj]
    flog = np.array(so[N2 + 3 + nobj:]).reshape(nlog, 4).tolist()
    holder = {int(i): 100000 + int(i) for i in np.nonzero(has_mp)[0]}
    erepl, elog = np.full(nobj, -1), []
    for j in range(nobj):
        if q["bad"][j] or wf[j] < 0:
            continue
        b = int(wf[j])
        if b in holder:
            erepl[j] = holder[b]
        else:
            elog.append([3, j, -1, b]); holder[b] = j
    assert r4 == wfn and (repl == erepl).all() and flog == elog and wfn > 100
    # relocalisation search against the reference's own function
    K1 = po.RefKeyFrame(k1, d1, u1, None, has1, bad1, sf, sf * sf, _m.CAM6[:4])
    po.ref2_kf_set_mappoints(K1, pts1, maxd1, mind1, d1)
    wfm, wn = po.ref2_search_frame_kf(F, T, K1, already, claimed, 10.0 if th < 5 else 3.0, orb_dist, check)
    got = np.fromfile(os.path.join(d, "out_reloc.i32"), np.int32)
    assert got[-1] == wn and (got[:-1] == wfm).all() and wn > 30
