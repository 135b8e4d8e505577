#!/usr/bin/env python
"""Config 2 of BASELINE.json: tracking-thread frames/s on a monocular EuRoC-shaped synthetic stream, 752x480, 1200 features per
frame, extractor + matchers.  Prints one JSON line with the card's name, power limit and SM clocks read in the same process.

  python tools/mono_bench.py [--batch 128] [--handles 4] [--steps 20] [--e2e-repeats 5] [--latency-frames 200] [--cpu-frames 64]
                             [--no-cpu-baseline] [--out FILE]

Per frame, what Tracking::GrabImageMonocular -> Frame::Frame(monocular) -> Track does for a rectified camera with zero distortion
(Frame::UndistortKeyPoints is then an identity copy): ORBextractor::operator() with vLappingArea = {0, 1000} (Frame.cc:380),
SearchByProjection(cur, last, th = 15, bMono) and SearchByProjection(F, local map points, th = 1) (Tracking.cc: TrackWithMotionModel,
SearchLocalPoints), mvuRight = -1 throughout.  Images are the left images of synth.stereo_pair(752, 480, seed); EuRoC cam0
intrinsics.  The map points are the frame's own features back-projected at the ground-truth depth of the synthetic disparity field;
the local map is bench.local_map_queries' mix of those points and as many unrelated ones.

  parity             the first frames through orbr_submit / orbr_collect against the CPU oracle before anything is timed (aborts on a
                     mismatch): keypoint records and descriptors with lapping (0, 1000), monoIndex, both match arrays
  value              frames resident in HBM, each batch of --batch frames one CUDA-graph replay of orbx_extract_batch_device and both
                     device searches under orbm_set_device_query_bounds, --handles streams in flight, CUDA events
  e2e                host buffers in and out through orbr_submit / orbr_collect (monocular), one host thread, the handles in flight,
                     --e2e-repeats repeats
  latency_b1         one frame per step, graph replay and end to end, p50 / p99
  stages             per-stage milliseconds of the extractor (orbx_last_timings) over a serial eager pass
  pose_optimization  the same step with PoseOptimization after each search
  cpu_baseline       the oracle's monocular frame and, where oracle/_ref is built, the reference's own source; one frame per thread
                     (the monocular Frame constructor extracts on the calling thread) and every host thread over independent frames;
                     the faster implementation is the value
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

W, H, NFEAT = 752, 480, 1200
FX, FY, CX, CY = 458.654, 457.296, 367.215, 248.375     # EuRoC cam0
BASELINE_M = 0.110078                                    # EuRoC stereo baseline: converts the synthetic disparity field to depth
BF_GT = FX * BASELINE_M
CAM6 = (FX, FY, CX, CY, 0.0, 0.0)                        # a monocular Frame: no mbf / mb (they are ignored by the monocular step)
TH_LAST, TH_LOCAL = 15.0, 1.0
LAP = (0, 1000)
POSE = np.array([0, 0, 0, 1, 0.002, 0.001, 0], np.float32)
METRIC = "tracking-thread frames/sec (752x480 monocular, 1200 feat)"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:
        return {"error": repr(e)}


def make_frames(n, base=8):
    """n monocular frames and their disparity fields: `base` generated left images + cheap deterministic variants (inverted, flipped,
    shifted), each with its disparity field transformed alike."""
    from orb_slam3_detailed_comments_b200 import synth
    gen = [synth.stereo_pair(W, H, seed=200 + i)[::2] for i in range(min(base, n))]
    imgs, disps = np.empty((n, H, W), np.uint8), np.empty((n, H, W), np.float32)
    for i in range(n):
        l, d = gen[i % len(gen)]
        k = i // len(gen)
        if k % 4 in (2, 3):
            l, d = l[::-1], d[::-1]
        if k % 2 == 1:
            l = 255 - l
        sh = (k // 4) * 7
        imgs[i], disps[i] = np.roll(l, sh, axis=0), np.roll(d, sh, axis=0)
    return imgs, disps


def depth_at(disp, k):
    """ground-truth depth of every keypoint: the synthetic disparity field at its pixel, through the EuRoC bf"""
    x = np.clip(np.rint(k["x"]).astype(np.int64), 0, W - 1)
    y = np.clip(np.rint(k["y"]).astype(np.int64), 0, H - 1)
    return (np.float32(BF_GT) / disp[y, x]).astype(np.float32)


def frame_queries(k, d, z, rng):
    """(last, local) query arrays of one frame: the LastFrame map points are every feature at its depth, the local map is
    bench.local_map_queries' set (pxr = x: a monocular frame has no right coordinate)."""
    xw = np.stack([(k["x"] - CX) * z / FX, (k["y"] - CY) * z / FY, z], 1).astype(np.float32)
    last = dict(xw=xw, oct=k["octave"].astype(np.int32), ang=k["angle"].astype(np.float32), desc=np.ascontiguousarray(d),
                obs=np.ones(len(k), np.uint8))
    x, y, xr, lvl, vc, dq, xwl = bench.local_map_queries(k, d, z, rng, CAM6, W, H)
    return last, dict(px=x, py=y, pxr=xr, lvl=lvl, vc=vc, desc=dq, xw=xwl)


# ------------------------------------------------------------------------------------------------------------------------------
# CPU arm: the monocular frame through the oracle, and through the reference's own source (oracle/_ref) when it is built
# ------------------------------------------------------------------------------------------------------------------------------
def oracle_mono_frame(img, disp, ex, seed=7, queries=None):
    """One monocular frame through the CPU oracle: extraction with lapping (0, 1000), then both projection searches with mvuRight = -1.
    queries = (last, local) of this frame (the GPU arm's own sets: parity) or None (built from the oracle's features).
    Returns dict(mono, k, d, fm, nm1, mt, nm2)."""
    from oracle import pyoracle as po
    mono, k, d = ex(img, LAP)
    ur = np.full(len(k), -1, np.float32)
    bounds = np.array([0, W, 0, H], np.float32)
    ql, qc = queries if queries is not None else frame_queries(k, d, depth_at(disp, k), np.random.default_rng(seed))
    fm, nm1 = po.search_last(k, d, ur, bounds, ex.scale_factors, np.float32(CAM6), POSE, 0, ql["xw"], ql["oct"], ql["ang"], ql["desc"], ql["obs"],
                             TH_LAST, True)
    mt, nm2 = po.search_local(k, d, ur, bounds, ex.scale_factors, qc["px"], qc["py"], qc["pxr"], qc["lvl"], qc["vc"], qc["desc"], TH_LOCAL, 0.8)
    return dict(mono=mono, k=k, d=d, fm=fm, nm1=nm1, mt=mt, nm2=nm2)


def reference_mono_frame(img, disp, ex, seed=7):
    """The same frame through the reference's own source as far as it compiles here: the unmodified ORBextractor.cc with
    vLappingArea = {0, 1000}, then SearchByProjection(cur, last, th, bMono = true) and SearchByProjection(F, local map points) cut out
    of the reference over skeleton classes.  Returns (matches of the last-frame search, matches of the local-map search)."""
    from oracle import pyoracle as po
    _, k, d = ex(img, LAP)
    ql, qc = frame_queries(k, d, depth_at(disp, k), np.random.default_rng(seed))
    F = po.RefFrame(k, d, np.full(len(k), -1, np.float32), np.array([0, W, 0, H], np.float32), ex.scale_factors, np.float32(CAM6), POSE)
    _, nm1, _ = F.search_last(POSE, POSE, ql["xw"], ql["oct"], ql["ang"], ql["desc"], ql["obs"], TH_LAST, True, mono=True)
    _, nm2 = F.search_local(qc["px"], qc["py"], qc["pxr"], qc["lvl"], qc["vc"], qc["desc"], TH_LOCAL, 0.8)
    return nm1, nm2


def cpu_frames(imgs, disps, threads, impl="oracle"):
    """len(imgs) monocular frames on `threads` host threads, one frame per thread at a time.  Returns (frames/s, seconds)."""
    from concurrent.futures import ThreadPoolExecutor
    from oracle import pyoracle as po
    mk = po.OracleExtractor if impl == "oracle" else po.RefExtractor
    run1 = oracle_mono_frame if impl == "oracle" else reference_mono_frame
    nthr = max(1, threads)
    exs = [mk(NFEAT, 1.2, 8, 20, 7) for _ in range(nthr)]
    chunks = [list(range(w, len(imgs), nthr)) for w in range(nthr)]
    t0 = time.perf_counter()
    if nthr == 1:
        for i in chunks[0]:
            run1(imgs[i], disps[i], exs[0])
    else:
        with ThreadPoolExecutor(nthr) as pool:
            list(pool.map(lambda w: [run1(imgs[i], disps[i], exs[w]) for i in chunks[w]], range(nthr)))
    dt = time.perf_counter() - t0
    return len(imgs) / dt, dt


def cpu_baseline(imgs, disps):
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    impls = ["oracle"] + (["reference"] if bench.reference_source_available() else [])
    res = {}
    for impl in impls:
        cpu_frames(imgs[:2], disps[:2], 1, impl)                                  # page-in
        one, s1 = cpu_frames(imgs[:max(4, len(imgs) // 8)], disps, 1, impl)
        allc, sa = cpu_frames(imgs, disps, cores, impl)
        res[impl] = {"one_thread_frames_per_s": one, "all_threads_frames_per_s": allc, "threads": cores, "seconds": s1 + sa}
    best = max(res, key=lambda i: res[i]["all_threads_frames_per_s"])
    return {"value": res[best]["all_threads_frames_per_s"], "value_one_thread": res[best]["one_thread_frames_per_s"], "unit": "frames/s",
            "kind": best, "threads": cores, "frames": len(imgs), "implementations": res,
            "note": "per frame: ORBextractor with vLappingArea (0, 1000), SearchByProjection(cur, last, th 15, bMono), "
                    "SearchByProjection(F, local map points, th 1); one frame per thread (the monocular Frame constructor extracts on the "
                    "calling thread); the faster implementation is the value.  oracle = the CPU restatement (oracle/); reference = the "
                    "reference's own ORBextractor.cc and ORBmatcher.cc members (oracle/_ref), when built"}


# ------------------------------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------------------------------
class MonoWorkload:
    """Handles, a pool of frames (> L2) resident in HBM and in pinned host memory, per-batch query sets, captured graphs."""

    def __init__(self, B, NH, pool_bytes=140e6):
        import torch
        from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera
        self.torch, self.B, self.NH = torch, B, NH
        self.dev = torch.device("cuda", 0)
        self.cam = camera(*CAM6, W, H)
        self.exs = [ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=B) for _ in range(NH)]
        self.ex = self.exs[0]
        self.streams = [torch.cuda.ExternalStream(e.cuda_stream(), device=self.dev) for e in self.exs]
        self.m_last, self.m_local = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
        self.pool_batches = max(2, int(np.ceil(pool_bytes / (B * W * H))))
        self.imgs, self.disps = make_frames(B * self.pool_batches)
        self.host_pool = torch.from_numpy(self.imgs.reshape(self.pool_batches, B, H, W)).pin_memory()
        self.dev_pool = self.host_pool.cuda()
        self.graphs = {}
        self._build_queries()

    def _build_queries(self):
        torch, ex, B = self.torch, self.ex, self.B
        rng = np.random.default_rng(1234)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
        self.H_LAST, self.H_LOC, self.D_LAST, self.D_LOC, self.P_LAST, self.P_LOC = [], [], [], [], [], []
        for pb in range(self.pool_batches):
            ex.extract_batch_device(self.dev_pool[pb].data_ptr(), B, W, H, lapping=LAP)
            _, _, off, kps, desc = ex.download(B)
            qs = []
            for p in range(B):
                a, b = int(off[p]), int(off[p + 1])
                qs.append(frame_queries(kps[a:b], desc[a:b], depth_at(self.disps[pb * B + p], kps[a:b]), rng))
            offs = lambda key, j: np.concatenate([[0], np.cumsum([len(q[j][key]) for q in qs])]).astype(np.int32)
            cat = lambda key, j, dt: np.ascontiguousarray(np.concatenate([q[j][key] for q in qs]).astype(dt))
            fimg = np.arange(B, dtype=np.int32)
            hl = dict(fimg=fimg, off=offs("oct", 0), Tcw=np.tile(POSE, (B, 1)), dir=np.zeros(B, np.int32), xw=cat("xw", 0, np.float32),
                      oct=cat("oct", 0, np.int32), ang=cat("ang", 0, np.float32), desc=cat("desc", 0, np.uint8), obs=cat("obs", 0, np.uint8))
            hc = dict(fimg=fimg, off=offs("lvl", 1), px=cat("px", 1, np.float32), py=cat("py", 1, np.float32), pxr=cat("pxr", 1, np.float32),
                      lvl=cat("lvl", 1, np.int32), vc=cat("vc", 1, np.float32), desc=cat("desc", 1, np.uint8), xw=cat("xw", 1, np.float32))
            self.H_LAST.append(hl); self.H_LOC.append(hc)
            self.D_LAST.append({k: T(v) for k, v in hl.items()}); self.D_LOC.append({k: T(v) for k, v in hc.items()})
            self.P_LAST.append({k: pin(v) for k, v in hl.items()}); self.P_LOC.append({k: pin(v) for k, v in hc.items()})
        dev, rc = self.dev, B * ex.max_features_per_image()
        self.rows_cap = rc
        self.max_loc = max(int(h["off"][-1]) for h in self.H_LOC)
        max_last = max(int(h["off"][-1]) for h in self.H_LAST)
        maxq = max(max(int(np.diff(h["off"]).max()) for h in hs) for hs in (self.H_LAST, self.H_LOC))
        self.nq_last = float(np.mean([int(h["off"][-1]) for h in self.H_LAST])) / B
        self.nq_loc = float(np.mean([int(h["off"][-1]) for h in self.H_LOC])) / B
        zi = lambda n, dt: torch.zeros(n, dtype=dt, device=dev)
        self.d_fm = [torch.full((rc,), -1, dtype=torch.int32, device=dev) for _ in range(self.NH)]
        self.d_nm = [zi(2 * B, torch.int32) for _ in range(self.NH)]
        self.d_match = [torch.full((max(self.max_loc, 1),), -1, dtype=torch.int32, device=dev) for _ in range(self.NH)]
        self.d_po = [dict(off=zi(B + 1, torch.int32), feat=zi(rc, torch.int32), xw=zi((rc, 3), torch.float32), obs=zi((rc, 3), torch.float32),
                          w=zi(rc, torch.float32), pose=zi((2, B, 7), torch.float64), out=zi(rc, torch.uint8), inl=zi((2, B), torch.int32))
                     for _ in range(self.NH)]
        for e in self.exs:
            e.set_device_query_bounds(max(max_last, self.max_loc, 1), max(maxq, 1), rc)

    def step_device(self, i, with_po=False, k=None, pb=None):
        from orb_slam3_detailed_comments_b200 import PoseEdgesDevice, PoseOptimizationDevice
        k = i % self.NH if k is None else k
        pb = i % self.pool_batches if pb is None else pb
        B, e, dl, dc, po_ = self.B, self.exs[k], self.D_LAST[pb], self.D_LOC[pb], self.d_po[k]
        cam5 = [FX, FY, CX, CY, 0.0]
        e.extract_batch_device(self.dev_pool[pb].data_ptr(), B, W, H, lapping=LAP)
        self.m_last.SearchByProjectionLastFrameDevice(e, self.cam, B, dl["fimg"], dl["off"], dl["Tcw"], dl["dir"], dl["xw"], dl["oct"], dl["ang"],
                                                      dl["desc"], dl["obs"], TH_LAST, self.d_fm[k], self.d_nm[k][:B])
        if with_po:
            PoseEdgesDevice(e, B, dl["fimg"], dl["xw"], po_["off"], po_["feat"], po_["xw"], po_["obs"], po_["w"], feature_match=self.d_fm[k])
            PoseOptimizationDevice(e, B, po_["off"], dl["Tcw"], po_["xw"], po_["obs"], po_["w"], cam5, po_["pose"][0], po_["out"], po_["inl"][0])
        self.m_local.SearchByProjectionDevice(e, self.cam, B, dc["fimg"], dc["off"], dc["px"], dc["py"], dc["pxr"], dc["lvl"], dc["vc"], dc["desc"],
                                              self.d_match[k], self.d_nm[k][B:], th=TH_LOCAL)
        if with_po:
            PoseEdgesDevice(e, B, dc["fimg"], dc["xw"], po_["off"], po_["feat"], po_["xw"], po_["obs"], po_["w"], query_offset=dc["off"],
                            query_match=self.d_match[k])
            PoseOptimizationDevice(e, B, po_["off"], dl["Tcw"], po_["xw"], po_["obs"], po_["w"], cam5, po_["pose"][1], po_["out"], po_["inl"][1])

    def launch(self, i, with_po=False):
        """batch i on handle i % NH as one CUDA-graph replay (captured on first use, after one eager run sized the scratch)"""
        k, pb = i % self.NH, i % self.pool_batches
        g = self.graphs.get((k, pb, with_po))
        if g is None:
            self.step_device(i, with_po)
            self.torch.cuda.synchronize()
            g = self.graphs[(k, pb, with_po)] = self.exs[k].graph_capture(lambda: self.step_device(i, with_po))
        self.exs[k].graph_launch(g)

    def timed_device_loop(self, first, count, with_po=False):
        torch, streams = self.torch, self.streams
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(streams[0])
        for st in streams[1:]:
            st.wait_event(e0)
        for i in range(count):
            self.launch(first + i, with_po)
        for st in streams[1:]:
            ev = torch.cuda.Event()
            ev.record(st)
            streams[0].wait_event(ev)
        e1.record(streams[0])
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    # ---- end to end: orbr_submit / orbr_collect (monocular), one host thread, NH handles in flight ----
    def e2e_setup(self):
        from orb_slam3_detailed_comments_b200.replay import TrackingStep
        from orb_slam3_detailed_comments_b200._native import KP_DTYPE
        torch, B, rc = self.torch, self.B, self.rows_cap
        pz = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory().numpy()
        self.steps_e2e = [TrackingStep(e, self.cam, 0.0, 0.0, TH_LAST, TH_LOCAL, 0.8, True, monocular=True) for e in self.exs]
        self.OUT = [dict(kps=torch.zeros(rc * 28, dtype=torch.uint8).pin_memory().numpy().view(KP_DTYPE), desc=pz((rc, 32), torch.uint8),
                         ur=pz(rc, torch.float32), dep=pz(rc, torch.float32), n=pz(B, torch.int32), offsets=pz(B + 1, torch.int32),
                         fm=pz(rc, torch.int32), nm1=pz(B, torch.int32), mt=pz(max(self.max_loc, 1), torch.int32), nm2=pz(B, torch.int32),
                         pose=pz((2, B, 7), torch.float64), inl=pz((2, B), torch.int32), eoff=pz((2, B + 1), torch.int32),
                         efeat=pz((2, rc), torch.int32), outl=pz((2, rc), torch.uint8)) for _ in range(self.NH)]

    def e2e_submit(self, i, with_po=False):
        k, pb = i % self.NH, i % self.pool_batches
        pl, pc = self.P_LAST[pb], self.P_LOC[pb]
        self.steps_e2e[k].submit(self.host_pool[pb].numpy(), last=pl, local=pc, pose=pl["Tcw"] if with_po else None,
                                 local_world_pos=pc["xw"] if with_po else None)

    def e2e_collect(self, i, with_po=False):
        o = self.OUT[i % self.NH]
        if not with_po:
            o = {kk: v for kk, v in o.items() if kk not in ("pose", "inl", "eoff", "efeat", "outl")}
        return self.steps_e2e[i % self.NH].collect(o)

    def e2e_loop(self, first, count, with_po=False):
        """count batches from one host thread: batch i + NH - 1 is submitted before batch i is collected.  Returns seconds."""
        NH = self.NH
        self.torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j in range(min(NH - 1, count)):
            self.e2e_submit(first + j, with_po)
        for i in range(count):
            if i + NH - 1 < count:
                self.e2e_submit(first + i + NH - 1, with_po)
            self.e2e_collect(first + i, with_po)
        return time.perf_counter() - t0

    def parity_check(self, n_frames=2):
        """frames 0 .. n_frames-1 of pool batch 0 through orbr_submit / orbr_collect against the CPU oracle on the same images and
        query sets: keypoint records, descriptors, monoIndex and both match arrays must be identical"""
        from oracle import pyoracle as po
        self.e2e_submit(0)
        rows = self.e2e_collect(0)
        _, mono, _ = self.exs[0].counts(self.B)
        o, hl, hc = self.OUT[0], self.H_LAST[0], self.H_LOC[0]
        off = o["offsets"]
        if not (o["ur"][:rows] == -1).all():
            raise SystemExit("PARITY FAILURE: mvuRight of a monocular frame is not -1 -- no number is reported")
        ex = po.OracleExtractor(NFEAT, 1.2, 8, 20, 7)
        checked = dict(frames=n_frames, keypoints=0, last_queries=0, local_queries=0)
        for p in range(n_frames):
            a, b = int(off[p]), int(off[p + 1])
            l0, l1, c0, c1 = int(hl["off"][p]), int(hl["off"][p + 1]), int(hc["off"][p]), int(hc["off"][p + 1])
            ql = {k: hl[k][l0:l1] for k in ("xw", "oct", "ang", "desc", "obs")}
            qc = {k: hc[k][c0:c1] for k in ("px", "py", "pxr", "lvl", "vc", "desc")}
            want = oracle_mono_frame(self.imgs[p], self.disps[p], ex, queries=(ql, qc))
            got_fm = o["fm"][a:b].copy()
            got_fm[got_fm >= 0] -= l0
            for name, g_, w_ in [("keypoints", o["kps"][a:b].view(np.uint8), want["k"].view(np.uint8)), ("descriptors", o["desc"][a:b], want["d"]),
                                 ("monoIndex", np.int32([mono[p]]), np.int32([want["mono"]])),
                                 ("SearchByProjection(cur,last)", got_fm, want["fm"]), ("SearchByProjection(F,local)", o["mt"][c0:c1], want["mt"])]:
                if g_.shape != w_.shape or not (g_ == w_).all():
                    raise SystemExit(f"PARITY FAILURE (frame {p}, {name}): the GPU path differs from the CPU oracle -- no number is reported")
            checked["keypoints"] += b - a
            checked["last_queries"] += l1 - l0
            checked["local_queries"] += c1 - c0
        return {"ok": True, "against": "CPU oracle (oracle/), same images and query sets, through orbr_submit / orbr_collect (monocular)", **checked,
                "compared": "keypoint records (28 B) and descriptors with lapping (0, 1000), monoIndex, both match arrays: identical; mvuRight all -1"}

    def close(self):
        for (k, _, _), g in self.graphs.items():
            self.exs[k].graph_destroy(g)
        self.graphs = {}
        for e in self.exs:
            e.close()


def latency_section(n_iter):
    """B = 1: one monocular frame per step, device-resident graph replay (CUDA events) and end to end (host clock)"""
    import torch
    w1 = MonoWorkload(1, 1, pool_bytes=8 * W * H)
    out = {}
    for with_po in (False, True):
        for i in range(2 * w1.pool_batches):
            w1.launch(i, with_po)
        torch.cuda.synchronize()
        ts = []
        for i in range(n_iter):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(w1.streams[0])
            w1.launch(i, with_po)
            e1.record(w1.streams[0])
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        out["with_pose_optimization" if with_po else "headline_step"] = {
            "graph_replay_device_resident": bench.percentile_ms(ts), "kernels_per_frame": w1.ex.graph_kernels(w1.graphs[(0, 0, with_po)])}
    w1.e2e_setup()
    for with_po in (False, True):
        for i in range(5):
            w1.e2e_submit(i, with_po); w1.e2e_collect(i, with_po)
        ts = []
        for i in range(n_iter):
            t0 = time.perf_counter()
            w1.e2e_submit(i, with_po)
            w1.e2e_collect(i, with_po)
            ts.append(1e3 * (time.perf_counter() - t0))
        out["with_pose_optimization" if with_po else "headline_step"]["e2e_host_buffers"] = bench.percentile_ms(ts)
    w1.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--batch", type=int, default=128, help="monocular frames per batch (default 128: the image count of config 3's 64 pairs)")
    ap.add_argument("--handles", type=int, default=4, help="extractor handles (CUDA streams) the batches are pipelined over")
    ap.add_argument("--steps", type=int, default=20, help="timed steps of 16 batches")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--e2e-repeats", type=int, default=5)
    ap.add_argument("--latency-frames", type=int, default=200)
    ap.add_argument("--cpu-frames", type=int, default=64)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/mono_bench.py needs a CUDA device (no CPU fallback)")
    from orb_slam3_detailed_comments_b200 import _native
    BPS = 16
    B, NH = args.batch, max(2, args.handles)
    wl = MonoWorkload(B, NH)
    wl.e2e_setup()
    parity = wl.parity_check(2)

    # value: frames resident in HBM, one graph replay per batch, NH streams
    sampler = bench.ClockSampler(0)
    sampler.start()
    nwarm = max(args.warmup, 1) * BPS
    for i in range(max(nwarm, NH * wl.pool_batches)):
        wl.launch(i)
    torch.cuda.synchronize()
    sampler.wait_first()
    launches0 = _native.lib().orb_kernel_launches()
    t_begin = time.time()
    ms = wl.timed_device_loop(nwarm, args.steps * BPS)
    t_end = time.time()
    clocks = sampler.stop(t_begin, t_end)
    launches = _native.lib().orb_kernel_launches() - launches0
    value = B * BPS * args.steps / (ms * 1e-3)
    nm = wl.d_nm[0].cpu().numpy()

    # stages: a serial eager pass on handle 0 with the extractor's stage events
    wl.ex.set_profiling(True)
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    nser = 16
    torch.cuda.synchronize()
    s0.record(wl.streams[0])
    for i in range(nser):
        wl.step_device(i, False, k=0, pb=i % wl.pool_batches)
    s1.record(wl.streams[0])
    torch.cuda.synchronize()
    serial = s0.elapsed_time(s1) / nser
    stage = wl.ex.last_timings()
    wl.ex.set_profiling(False)
    n, _, _ = wl.ex.counts(B)
    n_cand = float(np.mean([sum(len(wl.ex.candidates(b, l)) for l in range(8)) for b in range(2)]))
    level_px = [wl.ex.level_size(l)[0] * wl.ex.level_size(l)[1] for l in range(8)]
    ab = bench.algorithmic_bytes(float(n.mean()), n_cand, level_px)
    ext = {k: stage[k] for k in ("pyramid", "fast", "quadtree", "blur", "orient_desc")}
    stages = {"ms_per_batch": {**ext, "searches": max(serial - stage["total"], 0.0), "serial_step_total": serial},
              "gb_per_s": {k: ab[k] * B / (ext[k] * 1e-3) / 1e9 for k in ext if ext[k] > 0}, "algorithmic_bytes_per_image": ab,
              "keypoints_per_image": float(n.mean()), "fast_candidates_per_image": n_cand,
              "note": "serial eager pass on one stream after the timed region (orbx_last_timings); searches = serial step minus extraction"}

    # e2e: host buffers in and out, one host thread, NH handles in flight
    wl.e2e_loop(0, max(2 * NH, BPS))
    reps = [wl.e2e_loop(nwarm + r, args.steps * BPS) for r in range(max(1, args.e2e_repeats))]
    rates = [B * BPS * args.steps / t for t in reps]
    e2e = float(np.median(rates))

    # the same step with PoseOptimization after each search
    n_po = max(NH, (args.steps * BPS) // 4)
    for i in range(NH * wl.pool_batches):
        wl.launch(i, True)
    ms_po = wl.timed_device_loop(0, n_po, True)
    wl.e2e_loop(0, 2 * NH, True)
    dt_po = wl.e2e_loop(NH, n_po, True)
    po_sec = {"batches": n_po, "value_frames_per_s": B * n_po / (ms_po * 1e-3), "e2e_frames_per_s": B * n_po / dt_po,
              "inliers_after_motion_model": float(wl.OUT[(NH + n_po - 1) % NH]["inl"][0].mean()),
              "inliers_after_local_map": float(wl.OUT[(NH + n_po - 1) % NH]["inl"][1].mean())}
    latency = latency_section(args.latency_frames)
    cpu = None
    if not args.no_cpu_baseline:
        cpu = cpu_baseline(wl.imgs[:args.cpu_frames], wl.disps[:args.cpu_frames])
    line = {"metric": METRIC, "value": value, "unit": "frames/s", "higher_is_better": True, "card": card(),
            "torch_device": torch.cuda.get_device_name(0), "clocks": clocks,
            "config": {"workload": "config 2: monocular 752x480 (EuRoC cam0 intrinsics, rectified, zero distortion), 1200 features; per frame: "
                                   f"ORBextractor with vLappingArea (0, 1000), SearchByProjection(cur,last,th={TH_LAST:g},bMono), "
                                   f"SearchByProjection(F,local map points,th={TH_LOCAL:g})",
                       "frames_per_batch": B, "batches_per_step": BPS, "steps": args.steps, "handles": NH, "levels": 8, "scale_factor": 1.2,
                       "fast_thresholds": [20, 7]},
            "detail": {"timed_region_s": ms * 1e-3, "kernels_per_batch": wl.ex.graph_kernels(wl.graphs[(0, 0, False)]),
                       "gpu_launches": int(launches), "queries_per_frame": {"last_frame": wl.nq_last, "local_map": wl.nq_loc},
                       "matches_per_frame": {"last_frame": float(nm[:B].mean()), "local_map": float(nm[B:].mean())},
                       "l2": f"input pool of {wl.pool_batches} batches = {wl.pool_batches * B * W * H / 1e6:.0f} MB > 50 MB L2 (H100)"},
            "parity": parity,
            "e2e": {"value": e2e, "unit": "frames/s", "repeats_frames_per_s": rates, "spread": (max(rates) - min(rates)) / e2e,
                    "api": "orbr_submit / orbr_collect with monocular = 1 (pinned host buffers in and out), one host thread, median of the repeats"},
            "latency_b1": latency, "stages": stages, "pose_optimization": po_sec, "cpu_baseline": cpu}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")
    wl.close()


if __name__ == "__main__":
    main()
