#!/usr/bin/env python
"""RGB-D tracking-thread frames/s on a TUM-fr3-shaped synthetic stream: 640x480 RGB frames with 16-bit depth maps at
DepthMapFactor 5000, 1000 features per frame, extractor + depth stereo + matchers.  Prints one JSON line with the card's name, power
limit and SM clocks read in the same process.

  python tools/rgbd_bench.py [--batch 128] [--handles 4] [--steps 20] [--e2e-repeats 5] [--latency-frames 200] [--cpu-frames 64]
                             [--no-cpu-baseline] [--out FILE]

Per frame, what Tracking::GrabImageRGBD -> Frame::Frame(RGB-D) -> Track does for a camera with zero distortion: cvtColor(RGB2GRAY),
the depth map's convertTo(CV_32F, 1/5000), ORBextractor::operator() with vLappingArea = {0, 0}, Frame::ComputeStereoFromRGBD,
SearchByProjection(cur, last, th = 15) and SearchByProjection(F, local map points, th = 3), both with the stereo gates of every feature
that has a depth.  TUM fr3 intrinsics (fx 535.4, fy 539.2, cx 320.1, cy 247.6, bf 40).  Depth is bf / the disparity field of
synth.stereo_pair in raw units of 1/5000 m, clipped to the u16 range, with 3 % holes; the map points are the frame's own features at
that depth, the local map bench.local_map_queries' mix of those points and as many unrelated ones.

  parity             the first frames through orbr_submit / orbr_collect against the CPU oracle before anything is timed (aborts on a
                     mismatch): keypoints and descriptors with lapping (0, 0), mvuRight / mvDepth bits, both match arrays
  value              frames resident in HBM, each batch of --batch frames one CUDA-graph replay of orbx_extract_batch_device_format (RGB),
                     orbm_stereo_rgbd_batch (u16 maps, on_device) and both device searches, --handles streams in flight, CUDA events
  e2e                host buffers in and out through orbr_submit / orbr_collect (RGB-D), one host thread, the handles in flight: u16 maps
                     converted on the device, against float maps converted on the host first (numpy, as convertTo would) and sent as f32
  latency_b1         one frame per step, graph replay and end to end, p50 / p99
  pose_optimization  the same step with PoseOptimization after each search
  member_b1          the per-call path of the drop-in Frame::ComputeStereoFromRGBD at B = 1: one grey image extracted, one 640x480
                     float map up, mvuRight / mvDepth back
  cpu_baseline       the oracle's RGB-D frame, one frame per thread and every host thread over independent frames
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from mono_bench import card  # noqa: E402

W, H, NFEAT = 640, 480, 1000
FX, FY, CX, CY, BF = 535.4, 539.2, 320.1, 247.6, 40.0   # TUM fr3 (bf: the settings' baseline x fx, ORB-SLAM3's TUM3.yaml)
CAM6 = (FX, FY, CX, CY, BF, BF / FX)
FACTOR = np.float32(1.0 / 5000)                          # Tracking::mDepthMapFactor = 1 / DepthMapFactor
TH_LAST, TH_LOCAL = 15.0, 3.0
LAP = (0, 0)
POSE = np.array([0, 0, 0, 1, 0.002, 0.001, 0], np.float32)
METRIC = "tracking-thread frames/sec (640x480 RGB-D, 1000 feat)"


def make_frames(n, base=8):
    """n RGB frames and their u16 depth maps: `base` generated frames + cheap deterministic variants (flipped, shifted), each map
    transformed alike.  Returns (rgb (n, H, W, 3), grey (n, H, W) = the oracle's conversion of rgb, depth (n, H, W) u16)."""
    from oracle import pyingest
    from orb_slam3_detailed_comments_b200 import synth
    gen = []
    for i in range(min(base, n)):
        left, _, disp = synth.stereo_pair(W, H, seed=300 + i)
        rng = np.random.default_rng(300 + i)
        raw = np.clip(np.rint(np.float32(BF) / disp / FACTOR), 0, 65535).astype(np.uint16)
        raw[rng.random(raw.shape) < 0.03] = 0
        d = rng.integers(-3, 4, left.shape)
        rgb = np.stack([np.clip(left.astype(int) + d, 0, 255), left, np.clip(left.astype(int) - d, 0, 255)], -1).astype(np.uint8)
        gen.append((rgb, raw))
    rgbs, maps = np.empty((n, H, W, 3), np.uint8), np.empty((n, H, W), np.uint16)
    for i in range(n):
        c, m = gen[i % len(gen)]
        k = i // len(gen)
        if k % 2 == 1:
            c, m = c[::-1], m[::-1]
        sh = (k // 2) * 7
        rgbs[i], maps[i] = np.roll(c, sh, axis=0), np.roll(m, sh, axis=0)
    greys = np.stack([pyingest.ingest(c, "rgb") for c in rgbs])
    return rgbs, greys, maps


def frame_queries(k, d, dep, rng):
    """(last, local) query arrays of one frame: the LastFrame map points are every feature at its depth-map depth (5 m in a hole), the
    local map is bench.local_map_queries' set with the right coordinate predicted from that depth"""
    z = np.where(dep > 0, dep, np.float32(5.0)).astype(np.float32)
    xw = np.stack([(k["x"] - CX) * z / FX, (k["y"] - CY) * z / FY, z], 1).astype(np.float32)
    last = dict(xw=xw, oct=k["octave"].astype(np.int32), ang=k["angle"].astype(np.float32), desc=np.ascontiguousarray(d),
                obs=np.ones(len(k), np.uint8))
    x, y, xr, lvl, vc, dq, xwl = bench.local_map_queries(k, d, z, rng, CAM6, W, H)
    return last, dict(px=x, py=y, pxr=xr, lvl=lvl, vc=vc, desc=dq, xw=xwl)


# ------------------------------------------------------------------------------------------------------------------------------
# CPU arm: the RGB-D frame through the oracle
# ------------------------------------------------------------------------------------------------------------------------------
def oracle_rgbd_frame(grey, depth, ex, seed=7, queries=None):
    """One RGB-D frame through the CPU oracle: extraction with lapping (0, 0), the whole depth map converted and sampled
    (ComputeStereoFromRGBD), then both projection searches with that mvuRight.  queries = (last, local) of this frame (the GPU arm's own
    sets: parity) or None (built from the oracle's features).  Returns dict(k, d, ur, dep, fm, nm1, mt, nm2)."""
    from oracle import pyoracle as po, pyrgbd
    _, k, d = ex(grey, LAP)
    ur, dep = pyrgbd.stereo_from_rgbd(k, depth, FACTOR, BF)
    bounds = np.array([0, W, 0, H], np.float32)
    ql, qc = queries if queries is not None else frame_queries(k, d, dep, np.random.default_rng(seed))
    fm, nm1 = po.search_last(k, d, ur, bounds, ex.scale_factors, np.float32(CAM6), POSE, 0, ql["xw"], ql["oct"], ql["ang"], ql["desc"], ql["obs"],
                             TH_LAST, True)
    mt, nm2 = po.search_local(k, d, ur, bounds, ex.scale_factors, qc["px"], qc["py"], qc["pxr"], qc["lvl"], qc["vc"], qc["desc"], TH_LOCAL, 0.8)
    return dict(k=k, d=d, ur=ur, dep=dep, fm=fm, nm1=nm1, mt=mt, nm2=nm2)


def cpu_frames(greys, maps, threads):
    """len(greys) RGB-D frames through the oracle on `threads` host threads, one frame per thread at a time.  Returns (frames/s, s)."""
    from concurrent.futures import ThreadPoolExecutor
    from oracle import pyoracle as po
    nthr = max(1, threads)
    exs = [po.OracleExtractor(NFEAT, 1.2, 8, 20, 7) for _ in range(nthr)]
    chunks = [list(range(w, len(greys), nthr)) for w in range(nthr)]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(nthr) as pool:
        list(pool.map(lambda w: [oracle_rgbd_frame(greys[i], maps[i], exs[w]) for i in chunks[w]], range(nthr)))
    dt = time.perf_counter() - t0
    return len(greys) / dt, dt


def cpu_baseline(greys, maps):
    cores = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    cpu_frames(greys[:2], maps[:2], 1)                                             # page-in
    one, s1 = cpu_frames(greys[:max(4, len(greys) // 8)], maps, 1)
    allc, sa = cpu_frames(greys, maps, cores)
    return {"value": allc, "value_one_thread": one, "unit": "frames/s", "kind": "oracle", "threads": cores, "frames": len(greys),
            "seconds": s1 + sa, "note": "per frame: ORBextractor with vLappingArea (0, 0) on the grey image, the depth map converted with "
                                        "factor 1/5000 and sampled (ComputeStereoFromRGBD), SearchByProjection(cur, last, th 15), "
                                        "SearchByProjection(F, local map points, th 3); the CPU restatement (oracle/)"}


# ------------------------------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------------------------------
class RgbdWorkload:
    """Handles, a pool of RGB frames and u16 maps (> L2) resident in HBM and in pinned host memory, per-batch query sets, graphs."""

    def __init__(self, B, NH, pool_bytes=160e6):
        import torch
        from orb_slam3_detailed_comments_b200 import ORBextractor, ORBmatcher, camera
        self.torch, self.B, self.NH = torch, B, NH
        self.dev = torch.device("cuda", 0)
        self.cam = camera(*CAM6, W, H)
        self.exs = [ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=B) for _ in range(NH)]
        self.ex = self.exs[0]
        self.streams = [torch.cuda.ExternalStream(e.cuda_stream(), device=self.dev) for e in self.exs]
        self.m_last, self.m_local = ORBmatcher(0.9, True), ORBmatcher(0.8, True)
        self.pool_batches = max(2, int(np.ceil(pool_bytes / (B * W * H * 5))))
        self.rgbs, self.greys, self.maps = make_frames(B * self.pool_batches)
        self.host_rgb = torch.from_numpy(self.rgbs.reshape(self.pool_batches, B, H, W, 3)).pin_memory()
        self.host_map = torch.from_numpy(self.maps.reshape(self.pool_batches, B, H, W).view(np.int16)).pin_memory()
        self.dev_rgb, self.dev_map = self.host_rgb.cuda(), self.host_map.cuda().view(torch.uint16)
        self.graphs = {}
        self._build_queries()

    def _build_queries(self):
        torch, ex, B = self.torch, self.ex, self.B
        rng = np.random.default_rng(1234)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()
        self.H_LAST, self.H_LOC, self.D_LAST, self.D_LOC, self.P_LAST, self.P_LOC = [], [], [], [], [], []
        for pb in range(self.pool_batches):
            ex.extract_batch_device(self.dev_rgb[pb].data_ptr(), B, W, H, lapping=LAP, image_format="rgb")
            ex.stereo_rgbd_batch(self.dev_map[pb], FACTOR, BF)
            _, _, off, kps, desc = ex.download(B)
            _, dep = ex.stereo_download(int(off[-1]))
            qs = [frame_queries(kps[int(off[p]):int(off[p + 1])], desc[int(off[p]):int(off[p + 1])], dep[int(off[p]):int(off[p + 1])], rng)
                  for p in range(B)]
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
        cam5 = [FX, FY, CX, CY, BF]
        e.extract_batch_device(self.dev_rgb[pb].data_ptr(), B, W, H, lapping=LAP, image_format="rgb")
        e.stereo_rgbd_batch(self.dev_map[pb], FACTOR, BF)
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

    # ---- end to end: orbr_submit / orbr_collect (RGB-D), one host thread, NH handles in flight ----
    def e2e_setup(self):
        from orb_slam3_detailed_comments_b200.replay import TrackingStep
        from orb_slam3_detailed_comments_b200._native import KP_DTYPE
        torch, B, rc = self.torch, self.B, self.rows_cap
        pz = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory().numpy()
        mk = lambda e, factor: TrackingStep(e, self.cam, BF, BF / FX, TH_LAST, TH_LOCAL, 0.8, True, image_format="rgb", rgbd=True, depth_factor=factor)
        self.steps_e2e = {"u16": [mk(e, FACTOR) for e in self.exs], "f32": [mk(e, 1.0) for e in self.exs]}
        self.f32_maps = [pz((B, H, W), torch.float32) for _ in range(self.NH)]
        self.OUT = [dict(kps=torch.zeros(rc * 28, dtype=torch.uint8).pin_memory().numpy().view(KP_DTYPE), desc=pz((rc, 32), torch.uint8),
                         ur=pz(rc, torch.float32), dep=pz(rc, torch.float32), n=pz(B, torch.int32), offsets=pz(B + 1, torch.int32),
                         fm=pz(rc, torch.int32), nm1=pz(B, torch.int32), mt=pz(max(self.max_loc, 1), torch.int32), nm2=pz(B, torch.int32),
                         pose=pz((2, B, 7), torch.float64), inl=pz((2, B), torch.int32), eoff=pz((2, B + 1), torch.int32),
                         efeat=pz((2, rc), torch.int32), outl=pz((2, rc), torch.uint8)) for _ in range(self.NH)]

    def e2e_submit(self, i, with_po=False, maps="u16"):
        k, pb = i % self.NH, i % self.pool_batches
        pl, pc = self.P_LAST[pb], self.P_LOC[pb]
        raw = self.host_map[pb].numpy().view(np.uint16)
        if maps == "f32":                      # what a caller without the device conversion does: convertTo(CV_32F, factor) per map
            np.multiply(raw, FACTOR, out=self.f32_maps[k], dtype=np.float32)
            depth = self.f32_maps[k]
        else:
            depth = raw
        self.steps_e2e[maps][k].submit(self.host_rgb[pb].numpy(), last=pl, local=pc, pose=pl["Tcw"] if with_po else None,
                                       local_world_pos=pc["xw"] if with_po else None, depth=depth)

    def e2e_collect(self, i, with_po=False, maps="u16"):
        o = self.OUT[i % self.NH]
        if not with_po:
            o = {kk: v for kk, v in o.items() if kk not in ("pose", "inl", "eoff", "efeat", "outl")}
        return self.steps_e2e[maps][i % self.NH].collect(o)

    def e2e_loop(self, first, count, with_po=False, maps="u16"):
        """count batches from one host thread: batch i + NH - 1 is submitted before batch i is collected.  Returns seconds."""
        NH = self.NH
        self.torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j in range(min(NH - 1, count)):
            self.e2e_submit(first + j, with_po, maps)
        for i in range(count):
            if i + NH - 1 < count:
                self.e2e_submit(first + i + NH - 1, with_po, maps)
            self.e2e_collect(first + i, with_po, maps)
        return time.perf_counter() - t0

    def parity_check(self, n_frames=2):
        """frames 0 .. n_frames-1 of pool batch 0 through orbr_submit / orbr_collect, with u16 maps and with host-converted float maps,
        against the CPU oracle on the same images, maps and query sets"""
        from oracle import pyoracle as po
        ex = po.OracleExtractor(NFEAT, 1.2, 8, 20, 7)
        checked = dict(frames=n_frames, keypoints=0, last_queries=0, local_queries=0, depths=0)
        for maps in ("u16", "f32"):
            self.e2e_submit(0, maps=maps)
            self.e2e_collect(0, maps=maps)
            o, hl, hc = self.OUT[0], self.H_LAST[0], self.H_LOC[0]
            off = o["offsets"]
            for p in range(n_frames):
                a, b = int(off[p]), int(off[p + 1])
                l0, l1, c0, c1 = int(hl["off"][p]), int(hl["off"][p + 1]), int(hc["off"][p]), int(hc["off"][p + 1])
                ql = {k: hl[k][l0:l1] for k in ("xw", "oct", "ang", "desc", "obs")}
                qc = {k: hc[k][c0:c1] for k in ("px", "py", "pxr", "lvl", "vc", "desc")}
                want = oracle_rgbd_frame(self.greys[p], self.maps[p], ex, queries=(ql, qc))
                got_fm = o["fm"][a:b].copy()
                got_fm[got_fm >= 0] -= l0
                for name, g_, w_ in [("keypoints", o["kps"][a:b].view(np.uint8), want["k"].view(np.uint8)), ("descriptors", o["desc"][a:b], want["d"]),
                                     ("mvuRight", o["ur"][a:b].view(np.uint32), want["ur"].view(np.uint32)),
                                     ("mvDepth", o["dep"][a:b].view(np.uint32), want["dep"].view(np.uint32)),
                                     ("SearchByProjection(cur,last)", got_fm, want["fm"]), ("SearchByProjection(F,local)", o["mt"][c0:c1], want["mt"])]:
                    if g_.shape != w_.shape or not (g_ == w_).all():
                        raise SystemExit(f"PARITY FAILURE ({maps} maps, frame {p}, {name}): the GPU path differs from the CPU oracle -- no number is reported")
                checked["keypoints"] += b - a
                checked["depths"] += int((want["dep"] > 0).sum())
                checked["last_queries"] += l1 - l0
                checked["local_queries"] += c1 - c0
        return {"ok": True, "against": "CPU oracle (oracle/), same images, depth maps and query sets, through orbr_submit / orbr_collect (RGB-D), "
                                       "u16 maps and host-converted float maps", **checked,
                "compared": "keypoint records and descriptors with lapping (0, 0), mvuRight / mvDepth bits, both match arrays: identical"}

    def close(self):
        for (k, _, _), g in self.graphs.items():
            self.exs[k].graph_destroy(g)
        self.graphs = {}
        for e in self.exs:
            e.close()


def latency_section(n_iter):
    """B = 1: one RGB-D frame per step, device-resident graph replay (CUDA events) and end to end (host clock)"""
    import torch
    w1 = RgbdWorkload(1, 1, pool_bytes=8 * W * H * 5)
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


def member_section(n_iter):
    """The per-call path of the drop-in Frame::ComputeStereoFromRGBD at B = 1, as the member makes it after ORBextractor::operator():
    one 640x480 float map (what GrabImageRGBD converted) up with factor 1, k_stereo_rgbd, mvuRight / mvDepth back (host clock)"""
    from orb_slam3_detailed_comments_b200 import ORBextractor
    rgbs, greys, maps = make_frames(4)
    f32 = [np.ascontiguousarray((m.astype(np.float32) * FACTOR).astype(np.float32))[None] for m in maps]
    ex = ORBextractor(NFEAT, 1.2, 8, 20, 7, max_width=W, max_height=H, max_batch=1)
    ts_member, ts_frame = [], []
    for i in range(n_iter + 5):
        t0 = time.perf_counter()
        _, k, _ = ex(greys[i % 4], LAP)
        t1 = time.perf_counter()
        ex.stereo_rgbd_batch(f32[i % 4], 1.0, BF)
        ex.stereo_download(len(k))
        t2 = time.perf_counter()
        if i >= 5:
            ts_frame.append(1e3 * (t2 - t0)); ts_member.append(1e3 * (t2 - t1))
    ex.close()
    return {"compute_stereo_from_rgbd": bench.percentile_ms(ts_member), "extract_and_member": bench.percentile_ms(ts_frame),
            "map_bytes": W * H * 4, "note": "host clock; ORBextractor::operator() then the member's orbm_stereo_rgbd_batch (host f32 map, factor 1) "
                                           "and orbm_stereo_download, one frame at a time"}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--batch", type=int, default=128, help="RGB-D frames per batch")
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
        raise SystemExit("tools/rgbd_bench.py needs a CUDA device (no CPU fallback)")
    from orb_slam3_detailed_comments_b200 import _native
    BPS = 16
    B, NH = args.batch, max(2, args.handles)
    wl = RgbdWorkload(B, NH)
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

    # e2e: host buffers in and out, one host thread, NH handles in flight; u16 maps against float maps converted on the host first
    e2e = {}
    for maps in ("u16", "f32"):
        wl.e2e_loop(0, max(2 * NH, BPS), maps=maps)
        reps = [wl.e2e_loop(nwarm + r, args.steps * BPS, maps=maps) for r in range(max(1, args.e2e_repeats))]
        rates = [B * BPS * args.steps / t for t in reps]
        e2e[maps] = {"value": float(np.median(rates)), "repeats_frames_per_s": rates}

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
    kernels = wl.ex.graph_kernels(wl.graphs[(0, 0, False)])
    wl.close()
    latency = latency_section(args.latency_frames)
    member = member_section(args.latency_frames)
    cpu = None
    if not args.no_cpu_baseline:
        _, greys, maps = make_frames(args.cpu_frames)
        cpu = cpu_baseline(greys, maps)
    line = {"metric": METRIC, "value": value, "unit": "frames/s", "higher_is_better": True, "card": card(),
            "torch_device": torch.cuda.get_device_name(0), "clocks": clocks,
            "config": {"workload": "640x480 RGB-D (TUM fr3 intrinsics, zero distortion), RGB frames + u16 depth at factor 1/5000, 1000 features; per "
                                   "frame: cvtColor, ORBextractor with vLappingArea (0, 0), ComputeStereoFromRGBD, "
                                   f"SearchByProjection(cur,last,th={TH_LAST:g}), SearchByProjection(F,local map points,th={TH_LOCAL:g})",
                       "frames_per_batch": B, "batches_per_step": BPS, "steps": args.steps, "handles": NH, "levels": 8, "scale_factor": 1.2,
                       "fast_thresholds": [20, 7]},
            "detail": {"timed_region_s": ms * 1e-3, "kernels_per_batch": kernels, "gpu_launches": int(launches),
                       "matches_per_frame": {"last_frame": float(nm[:B].mean()), "local_map": float(nm[B:].mean())},
                       "l2": f"input pool of {wl.pool_batches} batches = {wl.pool_batches * B * W * H * 5 / 1e6:.0f} MB > 50 MB L2 (H100)"},
            "parity": parity,
            "e2e": {"value": e2e["u16"]["value"], "unit": "frames/s", "u16_maps_converted_on_device": e2e["u16"],
                    "f32_maps_converted_on_host": e2e["f32"],
                    "api": "orbr_submit / orbr_collect with depth_maps (pinned RGB images and maps in, pinned results out), one host thread, "
                           "median of the repeats; the f32 leg converts each batch's maps with numpy before submitting"},
            "latency_b1": latency, "pose_optimization": po_sec, "member_b1": member, "cpu_baseline": cpu}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
