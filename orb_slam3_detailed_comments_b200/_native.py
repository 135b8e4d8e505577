"""ctypes binding of liborbslam3_b200.so (the C ABI declared in include/orbslam3_b200.h).

There is no CPU fallback: importing this module without the built library, or creating a handle without
a CUDA device, raises.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG, "csrc")
LIB_PATH = os.environ.get("ORB_LIB_PATH") or os.path.join(_PKG, "lib", "liborbslam3_b200.so")   # ORB_LIB_PATH: an instrumented build (tools/qt_phases.py)
SOURCES = ["extractor.cu", "stereo.cu", "matcher.cu", "triangulation.cu", "lba.cu", "poseopt.cu", "bow.cu", "mappoint.cu", "liba.cu", "knn.cu", "replay.cu"]

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])


# orb_image_format of include/orbslam3_b200.h, and the channels of each
IMAGE_FORMATS = {"gray": 0, "rgb": 1, "bgr": 2, "rgba": 3, "bgra": 4}
FORMAT_CHANNELS = {0: 1, 1: 3, 2: 3, 3: 4, 4: 4}
# orb_depth_format of include/orbslam3_b200.h, by the numpy dtype of the map
DEPTH_FORMATS = {np.dtype(np.uint16): 1, np.dtype(np.float32): 2}


class OrbError(RuntimeError):
    pass


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a into lib/liborbslam3_b200.so (nvcc cross-compiles on CPU)."""
    deps = [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)] + [os.path.join(_PKG, "..", "include", "orbslam3_b200.h"),
                                                                   os.path.abspath(__file__)]   # the recipe itself
    if os.environ.get("ORB_LIB_PATH"):
        return LIB_PATH                       # an explicitly chosen build is never rebuilt
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(d) for d in deps):
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    subprocess.check_call([nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] +
                          [os.path.join(_CSRC, s) for s in SOURCES])
    return LIB_PATH


class orbx_config(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("scale_factor", C.c_float), ("n_levels", C.c_int32),
                ("ini_th_fast", C.c_int32), ("min_th_fast", C.c_int32), ("max_width", C.c_int32),
                ("max_height", C.c_int32), ("max_batch", C.c_int32), ("device", C.c_int32)]


class orbm_camera(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "bf", "b", "min_x", "max_x", "min_y", "max_y")]


class orbm_local_queries(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("on_device", C.c_int32)] + [
        (n, C.c_void_p) for n in ("frame_image", "query_offset", "proj_x", "proj_y", "proj_xr", "level", "view_cos",
                                  "track_depth", "desc", "feature_claimed", "in_view")]


class orbm_last_queries(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("on_device", C.c_int32)] + [
        (n, C.c_void_p) for n in ("frame_image", "query_offset", "Tcw", "direction", "world_pos", "last_octave",
                                  "last_angle", "desc", "obs_positive")]


class orbm_bow_queries(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("on_device", C.c_int32)] + [
        (n, C.c_void_p) for n in ("frame_image", "query_offset", "query_node", "query_angle", "desc", "feature_node")]


class orbm_kf_queries(C.Structure):
    _fields_ = [("n_targets", C.c_int32)] + [
        (n, C.c_void_p) for n in ("target_image", "feat_offset", "kp", "desc", "uright", "feat_claimed", "Tcw", "Ow",
                                  "Sim3", "query_offset", "world_pos", "normal", "max_dist", "min_dist", "desc_q", "angle")]


class orbo_pose_problems(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("on_device", C.c_int32), ("edge_offset", C.c_void_p), ("pose", C.c_void_p),
                ("world_pos", C.c_void_p), ("obs", C.c_void_p), ("inv_sigma2", C.c_void_p)] + [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "bf")] + [("n_edges_max", C.c_int32)]


class orbo_edge_source(C.Structure):
    _fields_ = [("n_frames", C.c_int32)] + [(n, C.c_void_p) for n in ("frame_image", "feature_match", "query_offset", "query_match", "world_pos", "query_world_pos")]


class orbo_frame_matches(C.Structure):
    _fields_ = [("n_frames", C.c_int32)] + [(n, C.c_void_p) for n in ("frame_image", "pose", "feature_match", "query_offset", "query_match", "world_pos")] + \
        [("n_queries", C.c_int32)] + [(n, C.c_float) for n in ("fx", "fy", "cx", "cy", "bf")]


class orbr_chain(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("point_offset", "world_pos", "normal", "max_dist", "min_dist", "desc", "last_query")] + [("viewing_cos_limit", C.c_float)]


class orbr_step(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("images", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32),
                ("image_stride_bytes", C.c_size_t), ("bf", C.c_float), ("b", C.c_float), ("last", C.POINTER(orbm_last_queries)),
                ("th_last", C.c_float), ("check_orientation_last", C.c_int32), ("local", C.POINTER(orbm_local_queries)),
                ("th_local", C.c_float), ("nnratio_local", C.c_float), ("far_points", C.c_int32), ("th_far", C.c_float),
                ("pose_optimization", C.c_int32), ("pose", C.c_void_p), ("local_world_pos", C.c_void_p), ("chain", C.POINTER(orbr_chain)),
                ("monocular", C.c_int32), ("image_format", C.c_int32), ("src_width", C.c_int32), ("src_height", C.c_int32),
                ("src_stride", C.c_int32), ("src_image_stride_bytes", C.c_size_t), ("depth_maps", C.c_void_p), ("depth_format", C.c_int32),
                ("depth_stride", C.c_int32), ("depth_image_stride_bytes", C.c_size_t), ("depth_factor", C.c_float)]


class orbr_results(C.Structure):
    _fields_ = [("cap_rows", C.c_int32)] + [(n, C.c_void_p) for n in ("keypoints", "descriptors", "uright", "depth", "n", "offsets",
                                                                     "last_feature_match", "last_nmatches", "local_match", "local_nmatches")] + \
        [(n, C.c_void_p * 2) for n in ("pose", "inliers", "edge_offset", "edge_feature", "edge_outlier")] + \
        [(n, C.c_void_p) for n in ("chain_in_view", "chain_proj_x", "chain_proj_y", "chain_proj_xr", "chain_level", "chain_view_cos", "chain_pose_f")]


class orbf_frustum_points(C.Structure):
    _fields_ = [("n_frames", C.c_int32), ("on_device", C.c_int32)] + [
        (n, C.c_void_p) for n in ("point_offset", "Rcw", "tcw", "Ow", "world_pos", "normal", "max_dist", "min_dist")] + [("n_points_max", C.c_int32)]


class orbm_init_queries(C.Structure):
    _fields_ = [("n1", C.c_int32), ("kp1", C.c_void_p), ("desc1", C.c_void_p), ("prev_matched", C.c_void_p), ("n2", C.c_int32),
                ("kp2", C.c_void_p), ("desc2", C.c_void_p), ("target_image", C.c_int32)]


class orbm_bow_kf_queries(C.Structure):
    _fields_ = [("n_pairs", C.c_int32)] + [
        (n, C.c_void_p) for n in ("feat_offset", "kp2", "desc2", "node2", "valid2", "query_offset", "query_node", "query_angle", "desc1")]


class orbm_triangulation(C.Structure):
    _fields_ = [("n_queries", C.c_int32), ("n2", C.c_int32)] + [
        (n, C.c_void_p) for n in ("kp1", "desc1", "node1", "stereo1", "kp2", "desc2", "node2", "valid2", "stereo2")] + [
        ("F12", C.c_float * 9), ("epipole2", C.c_float * 2), ("coarse", C.c_int32), ("check_orientation", C.c_int32)]


class lba_problem(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_mp", C.c_int32), ("n_edges", C.c_int32)] + [
        (n, C.c_void_p) for n in ("pose", "fixed", "point", "edge_kf", "edge_mp", "obs", "inv_sigma2")] + [
        (n, C.c_double) for n in ("fx", "fy", "cx", "cy", "bf", "lambda_init")] + [("max_iters", C.c_int32)]


class lba_result(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("pose", "point", "edge_chi2", "edge_depth_positive")] + [
        ("iterations", C.c_int32), ("trials", C.c_int32), ("lambda_", C.c_double), ("chi2", C.c_double),
        ("chi2_initial", C.c_double)]


# liba_link of include/orbslam3_b200.h (1080 bytes)
LIBA_LINK = np.dtype([("k1", "<i4"), ("k2", "<i4"), ("robust", "<i4"), ("pad", "<i4"), ("dt", "<f8"), ("dR", "<f4", 9), ("dV", "<f4", 3),
                      ("dP", "<f4", 3), ("JRg", "<f4", 9), ("JVg", "<f4", 9), ("JVa", "<f4", 9), ("JPg", "<f4", 9), ("JPa", "<f4", 9),
                      ("bias", "<f4", 6), ("info", "<f8", 81), ("infoG", "<f8", 9), ("infoA", "<f8", 9)])
assert LIBA_LINK.itemsize == 1080


class liba_problem(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_mp", C.c_int32), ("n_edges", C.c_int32), ("n_links", C.c_int32)] + [
        (n, C.c_void_p) for n in ("state", "fixed", "point", "edge_kf", "edge_mp", "obs", "inv_sigma2", "links")] + [
        ("Tcb", C.c_double * 12)] + [(n, C.c_double) for n in ("fx", "fy", "cx", "cy", "bf", "lambda_init")] + [("max_iters", C.c_int32)]


class liba_result(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("state", "point", "edge_chi2", "link_chi2", "edge_depth_positive")] + [
        ("iterations", C.c_int32), ("trials", C.c_int32), ("lambda_", C.c_double), ("chi2", C.c_double), ("chi2_initial", C.c_double),
        ("chi2_last_trial", C.c_double)]


_lib = None
_VP, _I, _F = C.c_void_p, C.c_int32, C.c_float
_IP = C.POINTER(C.c_int32)

# name -> (restype, argtypes); tests check that every symbol of include/orbslam3_b200.h is exported
SIGNATURES = {
    "orb_last_error": (C.c_char_p, []),
    "orb_device_count": (C.c_int, []),
    "orb_kernel_launches": (C.c_int64, []),
    "orbx_create": (_I, [C.POINTER(orbx_config), C.POINTER(_VP)]),
    "orbx_destroy": (None, [_VP]),
    "orbx_get_tables": (_I, [_VP] + [_VP] * 6),
    "orbx_extract": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _VP, _VP, _I, _IP, _IP]),
    "orbx_extract_batch": (_I, [_VP, _VP, _I, _I, _I, _I, C.c_size_t, _I, _I, _VP, _VP]),
    "orbx_extract_batch_device": (_I, [_VP, _VP, _I, _I, _I, _I, C.c_size_t, _I, _I]),
    "orbx_extract_batch_device_format": (_I, [_VP, _VP, _I, _I, _I, _I, C.c_size_t, _I, _I, _I, _I, _I]),
    "orbx_counts": (_I, [_VP, _VP, _VP, _VP]),
    "orbx_download": (_I, [_VP, _VP, _VP, _I]),
    "orbx_level_size": (_I, [_VP, _I, _IP, _IP]),
    "orbx_download_level": (_I, [_VP, _I, _I, _I, _VP, _I]),
    "orbx_download_pyramid": (_I, [_VP, _I, _I, _VP, _VP]),
    "orbx_graph_begin": (_I, [_VP]),
    "orbx_graph_end": (_I, [_VP, C.POINTER(C.c_void_p)]),
    "orbx_graph_launch": (_I, [_VP, _VP]),
    "orbx_graph_kernels": (_I, [_VP]),
    "orbx_graph_destroy": (None, [_VP]),
    "orbm_set_device_query_bounds": (_I, [_VP, _I, _I, _I]),
    "orbx_download_candidates": (_I, [_VP, _I, _I, _VP, _I, _IP]),
    "orbx_download_level_keypoints": (_I, [_VP, _I, _I, _VP, _I, _IP]),
    "orbx_set_profiling": (_I, [_VP, _I]),
    "orbx_last_timings": (_I, [_VP, _VP]),
    "orbx_cuda_stream": (_VP, [_VP]),
    "orbm_stereo_batch": (_I, [_VP, _I, _F, _F]),
    "orbm_stereo_download": (_I, [_VP, _VP, _VP, _I]),
    "orbm_stereo_pair": (_I, [_VP, _VP, _F, _F, _VP, _VP, _I]),
    "orbm_stereo_rgbd_batch": (_I, [_VP, _I, _VP, _I, _I, C.c_size_t, _F, _I, _F]),
    "orbm_search_local_points": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbm_local_queries), _F, _F, _I, _F, _VP, _VP]),
    "orbm_search_bow": (_I, [_VP, C.POINTER(orbm_bow_queries), _F, _I, _VP, _VP]),
    "orbm_search_initialization": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbm_init_queries), _I, C.c_float, _I, _VP, _VP]),
    "orbm_search_bow_keyframes": (_I, [_VP, C.POINTER(orbm_bow_kf_queries), C.c_float, _I, _VP, _VP]),
    "orbm_search_keyframe": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbm_kf_queries), _I, C.c_float, C.c_float, _I, _VP, _VP]),
    "orbm_search_triangulation": (_I, [_VP, C.POINTER(orbm_triangulation), _VP, _VP]),
    "orbo_pose_optimization": (_I, [_VP, C.POINTER(orbo_pose_problems), _VP, _VP, _VP, _VP]),
    "orbo_pose_edges": (_I, [_VP, C.POINTER(orbo_edge_source), _VP, _VP, _VP, _VP, _VP]),
    "orbo_pose_optimization_frames": (_I, [_VP, C.POINTER(orbo_frame_matches), _VP, _VP, _VP]),
    "orbf_is_in_frustum": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbf_frustum_points), C.c_float] + [_VP] * 7),
    "orbx_max_features": (_I, [_VP]),
    "orbv_create": (_I, [_I, _I, _I, _VP, _VP, _VP, _VP, _VP, C.POINTER(_VP)]),
    "orbv_destroy": (None, [_VP]),
    "orbv_transform": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "orbp_distinctive_descriptors": (_I, [_VP, _I, _VP, _VP, _VP]),
    "orbp_update_normal_and_depth": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    "lba_create": (_I, [_I, C.POINTER(_VP)]),
    "lba_destroy": (None, [_VP]),
    "lba_solve": (_I, [_VP, C.POINTER(lba_problem), C.POINTER(lba_result), _VP]),
    "lba_solve_bool": (_I, [_VP, C.POINTER(lba_problem), C.POINTER(lba_result), _VP]),
    "lba_solve_batch": (_I, [_VP, _I, C.POINTER(lba_problem), C.POINTER(lba_result), _VP]),
    "orbm_hamming_knn2": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "liba_create": (_I, [_I, C.POINTER(_VP)]),
    "liba_destroy": (None, [_VP]),
    "liba_solve": (_I, [_VP, _I, C.POINTER(liba_problem), C.POINTER(liba_result)]),
    "liba_link_information": (_I, [_VP, _I, _VP, _VP, _VP]),
    "orbx_keyframe_block_bytes": (C.c_size_t, [_VP]),
    "orbx_pack_keyframe_device": (_I, [_VP, _I, _VP, _VP, C.c_size_t]),
    "orbr_submit": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbr_step)]),
    "orbr_collect": (_I, [_VP, C.POINTER(orbr_results), _IP]),
    "orbm_search_last_frame": (_I, [_VP, C.POINTER(orbm_camera), C.POINTER(orbm_last_queries), _F, _I, _VP, _VP]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OrbError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status):
    if status != 0:
        raise OrbError(f"orb_status {status}: {lib().orb_last_error().decode(errors='replace')}")


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)
