"""Multi-GPU sequence replay plumbing (SURVEY.md §8e): one process per GPU, frames / sequences sharded across
ranks with NO data-path collective; the only exchange is the gather of new-keyframe / map-point state when
several replicas share one map (Atlas multi-session), done with torch.distributed (NCCL over NVLink on the
GPU box, gloo in the CPU tests).  Payloads are ~60 KB per keyframe: latency-bound, off the per-frame path."""
import numpy as np
import torch
import torch.distributed as dist

KF_FIELDS = (("pose", np.float32, 7), ("kp_xy", np.float32, 2), ("kp_octave", np.int32, 1), ("uright", np.float32, 1),
             ("desc", np.uint8, 32))


def shard_frames(n_frames, rank, world):
    """Independent-frame replay: frame i goes to rank i % world (extraction + stereo are stateless)."""
    return np.arange(rank, n_frames, world)


def shard_sequences(n_sequences, rank, world):
    """Batched sequence replay (config 5): whole sequences stay on one GPU (tracking is temporal)."""
    return [s for s in range(n_sequences) if s % world == rank]


def pack_keyframe(pose7, kps, uright, desc):
    """SoA block of one new keyframe -> one contiguous uint8 tensor: [n:int32][pose 7 f32][n x (x,y f32)][n x octave i32]
    [n x uright f32][n x 32 B descriptors]."""
    n = len(kps)
    parts = [np.array([n], np.int32).view(np.uint8), np.asarray(pose7, np.float32).view(np.uint8),
             np.stack([kps["x"], kps["y"]], 1).astype(np.float32).reshape(-1).view(np.uint8),
             kps["octave"].astype(np.int32).view(np.uint8), np.asarray(uright, np.float32).view(np.uint8),
             np.ascontiguousarray(desc, np.uint8).reshape(-1)]
    return torch.from_numpy(np.concatenate(parts))


def unpack_keyframe(buf):
    b = buf.cpu().numpy() if isinstance(buf, torch.Tensor) else buf
    n = int(b[:4].view(np.int32)[0])
    o = 4
    pose = b[o:o + 28].view(np.float32).copy(); o += 28
    xy = b[o:o + 8 * n].view(np.float32).reshape(n, 2).copy(); o += 8 * n
    octave = b[o:o + 4 * n].view(np.int32).copy(); o += 4 * n
    ur = b[o:o + 4 * n].view(np.float32).copy(); o += 4 * n
    desc = b[o:o + 32 * n].reshape(n, 32).copy()
    return dict(pose=pose, xy=xy, octave=octave, uright=ur, desc=desc)


def gather_keyframes(block, device=None, group=None):
    """All-gather one (possibly empty) keyframe block per rank.  Ragged sizes are handled with a size exchange and
    padding to the maximum.  Returns the list of per-rank blocks (uint8 tensors, empty where a rank had none)."""
    world = dist.get_world_size(group)
    dev = device or block.device
    block = block.to(dev)
    size = torch.tensor([block.numel()], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(size) for _ in range(world)]
    dist.all_gather(sizes, size, group=group)
    mx = int(max(int(s.item()) for s in sizes))
    if mx == 0:
        return [torch.zeros(0, dtype=torch.uint8) for _ in range(world)]
    pad = torch.zeros(mx, dtype=torch.uint8, device=dev)
    pad[:block.numel()] = block
    out = [torch.zeros_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return [o[:int(s.item())].cpu() for o, s in zip(out, sizes)]


def max_over_ranks(ms, device):
    """Timing rule of bench.py: device-measured milliseconds, maximum over ranks."""
    t = torch.tensor([ms], dtype=torch.float64, device=device)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


# ---- native replay step (include/orbslam3_b200.h: orbr_submit / orbr_collect) -----------------------------------------------
class TrackingStep:
    """The tracking-thread step of a batch of stereo or monocular frames on one extractor handle, host buffers in / host buffers
    out: `submit` queues the image upload, the extraction (both eyes, then ComputeStereoMatches; or with monocular=True one image
    per frame with vLappingArea = {0, 1000} and mvuRight = -1, Frame.cc:380), SearchByProjection(cur, last),
    SearchByProjection(F, local map points) and (optionally) PoseOptimization after each search, and returns at once;
    `collect` waits and copies the results into the caller's (ideally pinned) arrays.  Keep several handles in flight from
    one host thread: submit on handles k+1 .. k+H-1 before collecting handle k.  A monocular step takes direction 0 for every
    frame (bMono) and ignores bf / b.  image_format (a key of _native.IMAGE_FORMATS: gray, rgb, bgr, rgba, bgra) is the layout of
    the submitted images, converted to grey on the device as Tracking::GrabImage* does; resize=(width, height) resizes them first on
    the device, as System::Track* does for Settings::newImSize, and the results are in the coordinates of the resized images.
    With rgbd=True each frame is one camera image plus its depth map (submit's depth=), extracted with vLappingArea = {0, 0}; mvuRight /
    mvDepth come from the map as Frame::ComputeStereoFromRGBD computes them, depth_factor being Tracking::mDepthMapFactor; b is unused."""

    def __init__(self, extractor, cam, bf, b, th_last=15.0, th_local=3.0, nnratio_local=0.8, check_orientation=True, far_points=False,
                 th_far=50.0, monocular=False, image_format="gray", resize=None, rgbd=False, depth_factor=1.0):
        import ctypes as C
        from . import _native as N
        self._C, self._N, self._L = C, N, N.lib()
        self.ex, self.cam = extractor, cam
        self.args = (float(bf), float(b), float(th_last), 1 if check_orientation else 0, float(th_local), float(nnratio_local),
                     1 if far_points else 0, float(th_far))
        self.monocular = bool(monocular)
        self.rgbd, self.depth_factor = bool(rgbd), float(depth_factor)
        self.image_format, self.resize = N.IMAGE_FORMATS[image_format], resize
        self._keep = None

    def submit(self, images, last=None, local=None, pose=None, local_world_pos=None, chain=None, depth=None):
        """images: (2 * n_frames, H, W[, C]) uint8 host array, (n_frames, H, W[, C]) for a monocular or RGB-D step, C the channels of
        image_format; last / local: dicts of host arrays with the field names of
        orbm_last_queries / orbm_local_queries (fimg, off, Tcw, dir, xw, oct, ang, desc, obs / fimg, off, px, py, pxr, lvl, vc, desc
        [, td, in_view]); pose + local_world_pos switch PoseOptimization on.  chain: dict(off, xw, normal, max_dist, min_dist, desc,
        last_query[, cos_limit]) of the frames' local map points selects the chained flow (orbr_chain): needs last and pose, no local.
        depth: the (n_frames, H', W') uint16 or float32 host depth maps of an RGB-D step, of the extracted size, rows contiguous."""
        C, N = self._C, self._N
        cn = N.FORMAT_CHANNELS[self.image_format]
        assert images.dtype == np.uint8 and images.flags["C_CONTIGUOUS"] and images.shape[3:] == ((cn,) if cn > 1 else ())
        nimg, h, w = images.shape[:3]
        src = (0, 0, 0, 0, 0)                    # grey images of the extracted size
        if self.image_format or self.resize is not None:
            src = (self.image_format, w, h, w * cn, w * h * cn)
            w, h = self.resize or (w, h)
        nf = nimg if (self.monocular or self.rgbd) else nimg // 2
        dsrc = (None, 0, 0, 0, 0.0)
        if self.rgbd:
            assert depth is not None and depth.ndim == 3 and depth.strides[2] == depth.itemsize
            dsrc = (N.ptr(depth), N.DEPTH_FORMATS[depth.dtype], depth.strides[1], depth.strides[0], self.depth_factor)
        bf, b, thl, ori, thc, nnr, far, thfar = self.args
        ql = qc = None
        if last is not None:
            ql = N.orbm_last_queries(nf, 0, *[N.ptr(last[k]) if last.get(k) is not None else None
                                              for k in ("fimg", "off", "Tcw", "dir", "xw", "oct", "ang", "desc", "obs")])
        if local is not None:
            qc = N.orbm_local_queries(nf, 0, *[N.ptr(local[k]) if local.get(k) is not None else None
                                               for k in ("fimg", "off", "px", "py", "pxr", "lvl", "vc", "td", "desc", "claimed", "in_view")])
        po = pose is not None
        ch = None
        if chain is not None:
            ch = N.orbr_chain(*[N.ptr(chain[k]) for k in ("off", "xw", "normal", "max_dist", "min_dist", "desc", "last_query")],
                              float(chain.get("cos_limit", 0.5)))
        st = N.orbr_step(nf, N.ptr(images), w, h, w, w * h, bf, b, C.pointer(ql) if ql is not None else None, thl, ori,
                         C.pointer(qc) if qc is not None else None, thc, nnr, far, thfar, 1 if po else 0,
                         N.ptr(pose) if po else None, N.ptr(local_world_pos) if (po and local_world_pos is not None) else None,
                         C.pointer(ch) if ch is not None else None, 1 if self.monocular else 0, *src, *dsrc)
        self._keep = (images, last, local, pose, local_world_pos, ql, qc, chain, ch, depth)   # the arrays must outlive the asynchronous copies
        N.check(self._L.orbr_submit(self.ex._h, C.byref(self.cam), C.byref(st)))

    def collect(self, out):
        """out: dict of preallocated host arrays -- kps, desc, ur, dep (cap_rows rows), n, offsets (one entry per image, + 1), fm, nm1, mt, nm2 and, with
        PoseOptimization, pose (2, nf, 7) f64, inl (2, nf) i32, eoff (2, nf + 1) i32, efeat (2, cap) i32, outl (2, cap) u8; chained
        flow: c_in_view, c_px, c_py, c_pxr, c_level, c_vc (per local map point) and c_pose (nf, 7) f32.
        Missing keys are not copied back.  Returns the number of compact rows of the batch."""
        C, N = self._C, self._N
        g = lambda k: N.ptr(out[k]) if out.get(k) is not None else None
        two = lambda k: (C.c_void_p * 2)(*[C.c_void_p(out[k][i].ctypes.data) if out.get(k) is not None else None for i in range(2)])
        cap = min(len(out[k]) for k in ("kps", "desc", "ur", "dep", "fm") if out.get(k) is not None)
        if out.get("efeat") is not None:
            cap = min(cap, out["efeat"].shape[1])
        res = N.orbr_results(int(cap), g("kps"), g("desc"), g("ur"), g("dep"), g("n"), g("offsets"), g("fm"), g("nm1"), g("mt"), g("nm2"),
                             two("pose"), two("inl"), two("eoff"), two("efeat"), two("outl"),
                             g("c_in_view"), g("c_px"), g("c_py"), g("c_pxr"), g("c_level"), g("c_vc"), g("c_pose"))
        rows = C.c_int32(0)
        N.check(self._L.orbr_collect(self.ex._h, C.byref(res), C.byref(rows)))
        self._keep = None
        return rows.value
