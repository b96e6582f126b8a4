"""ctypes binding of librgbl_b200.so (the C ABI in include/rgbl_b200.h).

The library is the product: if it is missing or cannot create a CUDA context the callers fail
loudly — there is no Python/CPU fallback path in this package.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "librgbl_b200.so"
CSRC = _PKG / "csrc"

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])

RGBL_OK, RGBL_E_INVALID, RGBL_E_CUDA, RGBL_E_CAPACITY, RGBL_E_EMPTY, RGBL_E_UNSUPPORTED = 0, -1, -2, -3, -4, -5
DEPTH_NONE, DEPTH_NEAREST_NEIGHBOR_PIXEL, DEPTH_AVERAGE_FILTERING, DEPTH_INVERSE_DILATION = 0, 1, 2, 3


class OrbParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("ini_th_fast", C.c_int32), ("min_th_fast", C.c_int32)]


class DepthParams(C.Structure):
    _fields_ = [("method", C.c_int32), ("min_dist", C.c_float), ("max_dist", C.c_float), ("bf", C.c_float),
                ("inv_dilation_scale", C.c_float), ("ku", C.c_int32), ("kv", C.c_int32),
                ("mask", C.c_uint8 * 81), ("avg_kernel", C.c_int32), ("nn_search_radius", C.c_float)]


class FrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("keys_un", C.c_void_p), ("uright", C.c_void_p), ("desc", C.c_void_p),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("n_levels", C.c_int32), ("scale_factors", C.c_void_p),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("log_scale_factor", C.c_float)]


class KeyFrameViewC(C.Structure):
    _fields_ = [("n", C.c_int32), ("desc", C.c_void_p), ("keys", C.c_void_p), ("keys_un", C.c_void_p), ("uright", C.c_void_p),
                ("depth", C.c_void_p), ("has_mp", C.c_void_p), ("n_nodes", C.c_int32), ("node_ids", C.c_void_p),
                ("node_start", C.c_void_p), ("node_feat", C.c_void_p), ("Tcw", C.c_float * 7)]


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("max_batch", C.c_int32),
                ("max_points", C.c_int32), ("max_candidates", C.c_int32), ("orb", OrbParams)]


def build(force: bool = False) -> Path:
    """Compile librgbl_b200.so in-tree with nvcc for sm_90a (see csrc/Makefile)."""
    for target in ([], ["testing"]):          # the product library, then the test-only twin library (csrc/rgbl_testing.h)
        cmd = ["make", "-j4", "-C", str(CSRC)] + target + (["-B"] if force else [])
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("building librgbl_b200.so failed:\n" + r.stdout)
    return LIB_PATH


_lib = None

# name -> (restype, argtypes); every symbol include/rgbl_b200.h declares must be listed here
_vp, _i, _f = C.c_void_p, C.c_int, C.c_float
_ip = C.POINTER(C.c_int)
SYMBOLS = {
    "rgbl_create": (_i, [C.POINTER(Config), C.POINTER(_vp)]),
    "rgbl_destroy": (None, [_vp]),
    "rgbl_last_error": (C.c_char_p, [_vp]),
    "rgbl_abi_version": (_i, []),
    "rgbl_keypoint_capacity": (_i, [_vp]),
    "rgbl_orb_tables": (_i, [C.POINTER(OrbParams), _vp, _vp, _vp, _vp, _vp, _vp]),
    "rgbl_orb_extract": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _ip, _ip]),
    "rgbl_orb_extract_batch": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "rgbl_orb_get_pyramid": (_i, [_vp, _i, _i, _vp, _i, _ip, _ip]),
    "rgbl_orb_get_level": (_i, [_vp, _i, _i, _vp, _i, _ip, _ip]),
    "rgbl_orb_get_blurred_level": (_i, [_vp, _i, _i, _vp, _i]),
    "rgbl_orb_get_candidates": (_i, [_vp, _i, _i, _vp, _i, _ip]),
    "rgbl_depth_from_pcd": (_i, [_vp, _vp, _i, _vp, _i, _i, C.POINTER(DepthParams), _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "rgbl_depth_structuring_element": (_i, [C.c_char_p, _i, _i, _vp]),
    "rgbl_frame_rgbl_batch": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp, C.POINTER(DepthParams), _vp, _vp, _vp, _vp, _i, _vp]),
    "rgbl_search_by_projection_last": (_i, [_vp, C.POINTER(FrameViewC), _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _vp, _vp, _ip]),
    "rgbl_is_in_frustum": (_i, [_vp, C.POINTER(FrameViewC), _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rgbl_search_by_projection_local": (_i, [_vp, C.POINTER(FrameViewC), _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _f, _f, _i, _f, _vp, _vp, _ip]),
    "rgbl_stereo_matches": (_i, [_vp, _i, _i, _f, _f, _vp, _vp, _i]),
    "rgbl_search_by_bow": (_i, [_vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _f, _i, _vp, _ip]),
    "rgbl_search_by_projection_reloc": (_i, [_vp, C.POINTER(FrameViewC), _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i, _vp, _vp, _ip]),
    "rgbl_pose_optimize": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _vp, _vp, _ip]),
    "rgbl_resident_upload": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp]),
    "rgbl_resident_upload_kitti": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp]),
    "rgbl_resident_upload_kitti_png": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp]),
    "rgbl_decode_png_gray": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i]),
    "rgbl_resident_process": (_i, [_vp, _vp, C.POINTER(DepthParams), _vp]),
    "rgbl_resident_download": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "rgbl_fuse_search": (_i, [_vp, C.POINTER(FrameViewC), _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    "rgbl_distinctive_descriptors": (_i, [_vp, _i, _vp, _vp, _vp]),
    "rgbl_search_for_triangulation": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp,
                                           _i, _i, _i, _vp, _ip]),
    "rgbl_create_new_map_points": (_i, [_vp, C.POINTER(KeyFrameViewC), _i, C.POINTER(KeyFrameViewC), _vp, _vp, _f, _f, _f, _f, _f, _i, _vp, _vp, _f,
                                        _i, _i, _vp, _vp, _vp, _vp, _i, _vp]),
    "rgbl_local_bundle_adjustment": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _i, _vp, _vp, _vp, _ip]),
    "rgbl_global_bundle_adjustment": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp, _f, _f, _f, _f, _f, _i, _i, _vp, _vp, _vp, _ip]),
    "rgbl_vocabulary_create": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, C.POINTER(C.c_void_p)]),
    "rgbl_vocabulary_destroy": (None, [_vp]),
    "rgbl_compute_bow": (_i, [_vp, _vp, _i, _vp, _i, _vp, _vp, _ip, _vp, _vp, _vp, _ip]),
    "rgbl_resident_compute_bow": (_i, [_vp, _vp, _i, _i, _vp, _vp, _ip, _vp, _vp, _vp, _ip]),
    "rgbl_resident_track": (_i, [_vp, _vp, _f, _f, _f, _f, _f, _f, _i, _vp, _vp, _vp]),
    "rgbl_resident_track_begin": (_i, [_vp, _vp, _f, _f, _f, _f, _f, _f, _i]),
    "rgbl_resident_track_end": (_i, [_vp, _vp, _vp, _vp]),
    "rgbl_resident_track_begin2": (_i, [_vp, _vp]),
    "rgbl_depth_from_map": (_i, [_vp, _vp, _i, _i, _i, _f, _vp, _vp, _i, _vp, _vp]),
    "rgbl_resident_stage": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _vp, _vp]),
    "rgbl_track_sequence": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "rgbl_resident_upload_rgbd": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _i]),
    "rgbl_resident_upload_rgbd_png": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp]),
    "rgbl_decode_png_depth16": (_i, [_vp, _i, _vp, _vp, _vp, _i]),
    "rgbl_resident_process_rgbd": (_i, [_vp, _f, _f, _vp]),
    "rgbl_resident_stage_rgbd": (_i, [_vp, _i, _i, _vp, _i, _i, _i, _vp, _i]),
    "rgbl_track_sequence_rgbd": (_i, [_vp, _f, _f, _vp, _vp, _vp, _i]),
    "rgbl_resident_upload_stereo": (_i, [_vp, _i, _vp, _vp, _i, _i, _i]),
    "rgbl_resident_upload_stereo_png": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i]),
    "rgbl_resident_process_stereo": (_i, [_vp, _f, _f, _vp]),
    "rgbl_resident_stage_stereo": (_i, [_vp, _i, _i, _vp, _vp, _i, _i, _i]),
    "rgbl_track_sequence_stereo": (_i, [_vp, _f, _f, _vp, _vp, _vp]),
    "rgbl_set_stereo_rectification": (_i, [_vp, _vp, _vp, _vp, _vp, _i]),
    "rgbl_set_input_resize": (_i, [_vp, _i, _i]),
    "rgbl_set_input_channels": (_i, [_vp, _i, _i]),
    "rgbl_set_sequences": (_i, [_vp, _i, _vp]),
    "rgbl_sequence_lanes_resident": (_i, [_vp, _ip]),
    "rgbl_resident_track_end2": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "rgbl_set_camera_distortion": (_i, [_vp, _f, _f, _f, _f, _vp, _i, _vp]),
    "rgbl_resident_download_keys_un": (_i, [_vp, _vp, _i, _vp]),
    "rgbl_set_host_quadtree": (_i, [_vp, _i]),
    "rgbl_timer_mark": (_i, [_vp, _i]),
    "rgbl_timer_elapsed_ms": (_i, [_vp, C.POINTER(C.c_double)]),
    "rgbl_profile_enable": (_i, [_vp, _i]),
    "rgbl_profile_reset": (_i, [_vp]),
    "rgbl_profile_num_stages": (_i, []),
    "rgbl_profile_stage_name": (C.c_char_p, [_i]),
    "rgbl_profile_read": (_i, [_vp, _i, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "rgbl_profile_totals": (_i, [_vp, C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "rgbl_descriptor_distance": (_i, [_vp, _vp]),
}


# TEST INFRASTRUCTURE (csrc/rgbl_testing.h): host twins of device algorithms, exported by the separate librgbl_b200_testing.so only
TESTING_SYMBOLS = {
    "rgbl_quadtree_select": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _i]),
    "rgbl_quadtree_select_block_emulation": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _i]),
    "rgbl_std_sort_emulation": (_i, [_vp, _i, _vp]),
    "rgbl_std_sort_block_emulation": (_i, [_vp, _i, _i, _vp]),
    "rgbl_describe_staged_emulation": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "rgbl_fast_strips_emulation": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _i]),
    "rgbl_testing_reduced_solve": (_i, [_i, _vp, _vp, _i, _vp, _vp]),
    "rgbl_orb_tables": None,          # plus the product's host-only table helper (same source file), bound like the product's
}
TESTING_LIB_PATH = LIB_PATH.with_name("librgbl_b200_testing.so")
_testing_lib = None


def testing_lib() -> C.CDLL:
    global _testing_lib
    if _testing_lib is None:
        if not TESTING_LIB_PATH.exists():
            raise RuntimeError(f"{TESTING_LIB_PATH} is missing: run `make -C orb_slam3_rgbl_b200/csrc testing`")
        L = C.CDLL(str(TESTING_LIB_PATH))
        for name, sig in TESTING_SYMBOLS.items():
            res, args = sig if sig else SYMBOLS[name]
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _testing_lib = L
    return _testing_lib


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
        L = C.CDLL(str(LIB_PATH))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)          # AttributeError if the ABI lost a symbol
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class RgblError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rgbl error {code}: {msg}")
        self.code = code


def check(rc: int, ctx=None):
    if rc != 0:
        msg = lib().rgbl_last_error(ctx)
        raise RgblError(rc, msg.decode() if msg else "")
