"""ORBextractor -- host-side mirror of ORB_SLAM3::ORBextractor (reference include/ORBextractor.h:43-109)
on top of the C ABI.  Same constructor arguments, same getters, `__call__` = operator()."""
import ctypes as C

import numpy as np

from . import _native as N


class ORBextractor:
    """ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)  (ORBextractor.h:49-50).

    `extractor(image, lapping=(0, 0))` returns (monoIndex, keypoints, descriptors) exactly like
    `operator()(image, mask, keypoints, descriptors, vLappingArea)` (ORBextractor.cc:1557-1682); an empty
    image returns (-1, empty, empty).  `extract_batch` is the batched form used for sequence replay.
    """

    def __init__(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width=1280, max_height=720,
                 max_batch=1, device=0):
        self._L = N.lib()
        self._h = C.c_void_p()
        cfg = N.orbx_config(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_width, max_height,
                            max_batch, device)
        N.check(self._L.orbx_create(C.byref(cfg), C.byref(self._h)))
        self.nfeatures, self.scaleFactor, self.nlevels = nfeatures, scaleFactor, nlevels
        self.iniThFAST, self.minThFAST = iniThFAST, minThFAST
        self.max_batch, self.device = max_batch, device
        sc, isc, s2, is2 = (np.zeros(nlevels, np.float32) for _ in range(4))
        q, um = np.zeros(nlevels, np.int32), np.zeros(16, np.int32)
        N.check(self._L.orbx_get_tables(self._h, N.ptr(sc), N.ptr(isc), N.ptr(s2), N.ptr(is2), N.ptr(q), N.ptr(um)))
        self._sc, self._isc, self._s2, self._is2 = sc, isc, s2, is2
        self.mnFeaturesPerLevel, self.umax = q, um

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.orbx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # getters, ORBextractor.h:61-81
    def max_features_per_image(self):
        return int(self._L.orbx_max_features(self._h))

    def GetLevels(self):
        return self.nlevels

    def GetScaleFactor(self):
        return self.scaleFactor

    def GetScaleFactors(self):
        return self._sc.copy()

    def GetInverseScaleFactors(self):
        return self._isc.copy()

    def GetScaleSigmaSquares(self):
        return self._s2.copy()

    def GetInverseScaleSigmaSquares(self):
        return self._is2.copy()

    def __call__(self, image, lapping=(0, 0)):
        if image is None or image.size == 0:
            return -1, np.zeros(0, N.KP_DTYPE), np.zeros((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2, "CV_8UC1 expected (ORBextractor.cc:1567)"
        if image.strides[1] != 1:
            image = np.ascontiguousarray(image)
        h, w = image.shape
        cap = 4 * self.nfeatures + 16 * self.nlevels
        kps = np.zeros(cap, N.KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n, mono = C.c_int32(0), C.c_int32(0)
        N.check(self._L.orbx_extract(self._h, C.c_void_p(image.ctypes.data), w, h, image.strides[0], int(lapping[0]),
                                     int(lapping[1]), N.ptr(kps), N.ptr(desc), cap, C.byref(n), C.byref(mono)))
        return mono.value, kps[:n.value].copy(), desc[:n.value].copy()

    # ---- batched API ---------------------------------------------------------------------------
    def extract_batch(self, images, lapping=(0, 0), rgb=False, resize=None):
        """images: (B, H, W) grey or (B, H, W, 3 | 4) colour uint8 host array.  Returns (n[B], mono[B]); results stay on the device.
        Colour images are converted to grey as Tracking::GrabImage* does: BGR(A) channel order, RGB(A) with rgb=True (mbRGB).
        resize=(width, height) resizes every image first, as System::Track* does for Settings::newImSize; keypoints are in the
        coordinates of the resized image.  Colour or resized images go to the device as they are (a torch copy on the handle's
        device) and are converted there."""
        images = np.ascontiguousarray(images, np.uint8)
        b, h, w = images.shape[:3]
        n = np.zeros(b, np.int32)
        mono = np.zeros(b, np.int32)
        if images.ndim == 3 and resize is None:
            N.check(self._L.orbx_extract_batch(self._h, N.ptr(images), b, w, h, w, h * w, int(lapping[0]), int(lapping[1]),
                                               N.ptr(n), N.ptr(mono)))
            return n, mono
        import torch
        assert images.ndim == 3 or images.shape[3] in (3, 4), "(B, H, W), (B, H, W, 3) or (B, H, W, 4) expected"
        fmt = "gray" if images.ndim == 3 else ("rgb" if rgb else "bgr") + ("a" if images.shape[3] == 4 else "")
        d = torch.from_numpy(images).to(torch.device("cuda", self.device))
        torch.cuda.current_stream(d.device).synchronize()      # the copy is on torch's stream, the extraction on the handle's
        self.extract_batch_device(d.data_ptr(), b, *(resize or (w, h)), lapping=lapping, image_format=fmt, src_size=(w, h))
        N.check(self._L.orbx_counts(self._h, N.ptr(n), N.ptr(mono), None))
        return n, mono

    def extract_batch_async(self, images, lapping=(0, 0)):
        """Like extract_batch but returns immediately (H2D + kernels are queued on the handle's stream); `images` must
        stay alive (pinned memory makes the copy truly asynchronous).  Pair with counts()/download()."""
        assert images.dtype == np.uint8 and images.flags["C_CONTIGUOUS"]
        b, h, w = images.shape
        N.check(self._L.orbx_extract_batch(self._h, N.ptr(images), b, w, h, w, h * w, int(lapping[0]), int(lapping[1]),
                                           None, None))

    def extract_batch_device(self, dptr, batch, width, height, stride=None, image_stride=None, lapping=(0, 0), image_format="gray",
                             src_size=None):
        """Images already in device memory.  image_format (a key of _native.IMAGE_FORMATS) and src_size=(width, height) of the
        images at dptr select orbx_extract_batch_device_format: converted to grey and resized to width x height on the device;
        stride / image_stride then describe the source (default: tight rows of src_size)."""
        fmt = N.IMAGE_FORMATS[image_format]
        if fmt == 0 and src_size is None:
            stride = stride or width
            image_stride = image_stride or stride * height
            N.check(self._L.orbx_extract_batch_device(self._h, C.c_void_p(dptr), batch, width, height, stride, image_stride,
                                                      int(lapping[0]), int(lapping[1])))
            return
        sw, sh = src_size or (width, height)
        stride = stride or sw * N.FORMAT_CHANNELS[fmt]
        image_stride = image_stride or stride * sh
        N.check(self._L.orbx_extract_batch_device_format(self._h, C.c_void_p(dptr), batch, width, height, stride, image_stride,
                                                         int(lapping[0]), int(lapping[1]), fmt, sw, sh))

    def counts(self, batch):
        n, mono, off = np.zeros(batch, np.int32), np.zeros(batch, np.int32), np.zeros(batch + 1, np.int32)
        N.check(self._L.orbx_counts(self._h, N.ptr(n), N.ptr(mono), N.ptr(off)))
        return n, mono, off

    def download(self, batch, out=None):
        """Compact results of the last batch.  `out` = (kps, desc) preallocated host arrays (pinned memory makes the
        D2H a DMA instead of a staged copy); returns (n, mono, offsets, kps[:rows], desc[:rows])."""
        n, mono, off = self.counts(batch)
        rows = int(off[batch])
        if out is None:
            kps = np.zeros(max(rows, 1), N.KP_DTYPE)
            desc = np.zeros((max(rows, 1), 32), np.uint8)
        else:
            kps, desc = out
            assert len(kps) >= rows and len(desc) >= rows
        N.check(self._L.orbx_download(self._h, N.ptr(kps), N.ptr(desc), max(len(kps), 1)))
        return n, mono, off, kps[:rows], desc[:rows]

    # ---- stage outputs (parity tests; mvImagePyramid is a public member of the reference class) ---
    def level_size(self, level):
        w, h = C.c_int32(), C.c_int32()
        N.check(self._L.orbx_level_size(self._h, level, C.byref(w), C.byref(h)))
        return w.value, h.value

    def image_pyramid(self, b, level, blurred=False):
        w, h = self.level_size(level)
        out = np.zeros((h, w), np.uint8)
        N.check(self._L.orbx_download_level(self._h, b, level, 1 if blurred else 0, N.ptr(out), w))
        return out

    def candidates(self, b, level):
        cap = 1 << 18
        out = np.zeros((cap, 3), np.int32)
        n = C.c_int32()
        N.check(self._L.orbx_download_candidates(self._h, b, level, N.ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def level_keypoints(self, b, level):
        cap = 1 << 16
        out = np.zeros((cap, 3), np.int32)
        n = C.c_int32()
        N.check(self._L.orbx_download_level_keypoints(self._h, b, level, N.ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    # ---- Frame::ComputeStereoMatches (Frame.cc:1102-1358) --------------------------------------
    def stereo_batch(self, n_pairs, bf, b):
        """Stereo-match the last batch (left = image 2p, right = image 2p+1); results stay on the device."""
        N.check(self._L.orbm_stereo_batch(self._h, n_pairs, float(bf), float(b)))

    def stereo_download(self, rows, out=None):
        if out is None:
            uR = np.zeros(max(rows, 1), np.float32)
            dep = np.zeros(max(rows, 1), np.float32)
        else:
            uR, dep = out
        N.check(self._L.orbm_stereo_download(self._h, N.ptr(uR), N.ptr(dep), max(len(uR), 1)))
        return uR[:rows], dep[:rows]

    # ---- Frame::ComputeStereoFromRGBD ---------------------------------------------------------------------------------------
    def stereo_rgbd_batch(self, depth, depth_factor, bf):
        """mvuRight / mvDepth of the first len(depth) images of the last batch (RGB-D frames, extracted with lapping (0, 0)) from their
        depth maps: depth is an (n, H, W) uint16 or float32 host array or CUDA tensor of the extracted size, rows contiguous (any row or
        image stride); depth_factor is Tracking::mDepthMapFactor (1 / the settings' DepthMapFactor), applied as GrabImageRGBD applies it.
        Results stay on the device (stereo_download reads them)."""
        on_device = hasattr(depth, "data_ptr")
        if on_device:
            import torch
            dt = np.dtype({torch.uint16: np.uint16, torch.float32: np.float32}[depth.dtype])
            ptr, strides = depth.data_ptr(), tuple(s * dt.itemsize for s in depth.stride())
        else:
            dt, ptr, strides = depth.dtype, depth.ctypes.data, depth.strides
        assert depth.ndim == 3 and strides[2] == dt.itemsize, "(n, H, W) maps with contiguous rows expected"
        fmt = N.DEPTH_FORMATS[dt]
        N.check(self._L.orbm_stereo_rgbd_batch(self._h, depth.shape[0], C.c_void_p(ptr), fmt, strides[1], strides[0], float(depth_factor),
                                               1 if on_device else 0, float(bf)))

    def stereo_pair(self, right, n_left, bf, b):
        """mvuRight, mvDepth for image 0 of `self` (left eye) against image 0 of `right`."""
        uR = np.zeros(max(n_left, 1), np.float32)
        dep = np.zeros(max(n_left, 1), np.float32)
        N.check(self._L.orbm_stereo_pair(self._h, right._h, float(bf), float(b), N.ptr(uR), N.ptr(dep), max(n_left, 1)))
        return uR[:n_left], dep[:n_left]

    def cuda_stream(self):
        return self._L.orbx_cuda_stream(self._h)

    # ---- CUDA-graph replay (include/orbslam3_b200.h: orbx_graph_*) ----
    def set_device_query_bounds(self, total_queries, max_queries_per_frame, total_rows):
        """Bounds for the device-pointer searches: with them set they read nothing back and do not synchronise."""
        N.check(self._L.orbm_set_device_query_bounds(self._h, int(total_queries), int(max_queries_per_frame), int(total_rows)))

    def graph_capture(self, step):
        """Runs step() -- device-pointer entry points on this handle only -- under stream capture; returns an opaque graph.
        The same step must have run once eagerly before (it sizes the scratch buffers)."""
        N.check(self._L.orbx_graph_begin(self._h))
        try:
            step()
        finally:
            g = C.c_void_p()
            status = self._L.orbx_graph_end(self._h, C.byref(g))
        N.check(status)
        return g

    def graph_launch(self, g):
        N.check(self._L.orbx_graph_launch(self._h, g))

    def graph_kernels(self, g):
        return int(self._L.orbx_graph_kernels(g))

    def graph_destroy(self, g):
        self._L.orbx_graph_destroy(g)

    def keyframe_block_bytes(self):
        return int(self._L.orbx_keyframe_block_bytes(self._h))

    def pack_keyframe_device(self, image, d_pose7, d_block):
        """Keyframe state of one image of the last batch into a device block (CUDA torch tensors; replay.unpack_keyframe reads it)."""
        N.check(self._L.orbx_pack_keyframe_device(self._h, int(image), C.c_void_p(d_pose7.data_ptr()), C.c_void_p(d_block.data_ptr()),
                                                  d_block.numel() * d_block.element_size()))

    def set_profiling(self, on=True):
        N.check(self._L.orbx_set_profiling(self._h, 1 if on else 0))

    def last_timings(self):
        t = np.zeros(7, np.float32)
        N.check(self._L.orbx_last_timings(self._h, N.ptr(t)))
        return dict(zip(["total", "pyramid", "fast", "quadtree", "blur", "orient_desc", "h2d"], t.tolist()))
