"""ctypes / numpy mirror of include/okvis_b200.h (the C-ABI of libokvis_b200.so).

Only plumbing lives here: struct layouts, the library loader and argument marshalling.  The
product path is the CUDA library; if it is missing, loading fails loudly (no CPU fallback).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libokvis_b200.so")

OKB_OK = 0
OKB_ERR_INVALID_ARG, OKB_ERR_CUDA, OKB_ERR_UNSUPPORTED, OKB_ERR_CAPACITY, OKB_ERR_NO_DEVICE, OKB_ERR_NUMERIC = (
    -1, -2, -3, -4, -5, -6)
OKB_ERR_SHARD_TIMEOUT = -7
DIST_NONE, DIST_RADTAN, DIST_EQUIDISTANT, DIST_RADTAN8 = 0, 1, 2, 3
BLOCK_POSE, BLOCK_SPEED_BIAS, BLOCK_EXTRINSICS = 0, 1, 2
IMU_TERM_OUT = 931      # OKB_IMU_TERM_OUT: doubles per term of okb_debug_imu_terms (H30 | g30 | cost)
TERMINATION = {0: "NO_CONVERGENCE", 1: "FUNCTION_TOLERANCE", 2: "PARAMETER_TOLERANCE", 3: "GRADIENT_TOLERANCE",
               4: "MIN_RADIUS", 5: "TIME_LIMIT", 6: "FAILURE"}

c_double_p = C.POINTER(C.c_double)
c_u8_p = C.POINTER(C.c_uint8)


class Camera(C.Structure):
    _fields_ = [("model", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("_pad", C.c_int32),
                ("fu", C.c_double), ("fv", C.c_double), ("cu", C.c_double), ("cv", C.c_double),
                ("dist", C.c_double * 8)]


class ImuParams(C.Structure):
    _fields_ = [("a_max", C.c_double), ("g_max", C.c_double), ("sigma_g_c", C.c_double), ("sigma_a_c", C.c_double),
                ("sigma_bg", C.c_double), ("sigma_ba", C.c_double), ("sigma_gw_c", C.c_double),
                ("sigma_aw_c", C.c_double), ("tau", C.c_double), ("g", C.c_double), ("a0", C.c_double * 3),
                ("rate", C.c_int32), ("_pad", C.c_int32)]


class MargPrior(C.Structure):
    _fields_ = [("n", C.c_int32), ("n_blocks", C.c_int32), ("block_kind", C.POINTER(C.c_int32)),
                ("block_idx", C.POINTER(C.c_uint32)), ("x0", c_double_p), ("J", c_double_p), ("e0", c_double_p)]


class MargJob(C.Structure):
    _fields_ = [("n_blocks", C.c_int32), ("n_imu_terms", C.c_int32), ("n_sb_priors", C.c_int32), ("n_landmarks", C.c_int32),
                ("block_kind", C.POINTER(C.c_int32)), ("block_idx", C.POINTER(C.c_uint32)), ("block_prev", C.POINTER(C.c_int32)),
                ("block_marginalize", C.POINTER(C.c_uint8)), ("imu_terms", C.POINTER(C.c_uint32)),
                ("sb_priors", C.POINTER(C.c_uint32)), ("landmarks", C.POINTER(C.c_uint32))]


def make_marg_job(block_kind, block_idx, block_prev, block_marginalize, imu_terms=(), sb_priors=(), landmarks=()):
    """okb_marg_job over numpy arrays (kept alive on the returned object)."""
    a = [np.ascontiguousarray(block_kind, np.int32), np.ascontiguousarray(block_idx, np.uint32),
         np.ascontiguousarray(block_prev, np.int32), np.ascontiguousarray(block_marginalize, np.uint8),
         np.ascontiguousarray(imu_terms, np.uint32), np.ascontiguousarray(sb_priors, np.uint32),
         np.ascontiguousarray(landmarks, np.uint32)]
    j = MargJob()
    j.n_blocks, j.n_imu_terms, j.n_sb_priors, j.n_landmarks = len(a[0]), len(a[4]), len(a[5]), len(a[6])
    j.block_kind = a[0].ctypes.data_as(C.POINTER(C.c_int32))
    j.block_idx = a[1].ctypes.data_as(C.POINTER(C.c_uint32))
    j.block_prev = a[2].ctypes.data_as(C.POINTER(C.c_int32))
    j.block_marginalize = a[3].ctypes.data_as(C.POINTER(C.c_uint8))
    j.imu_terms = a[4].ctypes.data_as(C.POINTER(C.c_uint32))
    j.sb_priors = a[5].ctypes.data_as(C.POINTER(C.c_uint32))
    j.landmarks = a[6].ctypes.data_as(C.POINTER(C.c_uint32))
    j._keep = a
    return j


class MatchGate(C.Structure):
    _fields_ = [("mode", C.c_int32), ("_pad", C.c_int32), ("kp_b", c_double_p), ("kp_size_b", c_double_p), ("proj_into_b", c_double_p),
                ("proj_uncertainty", c_double_p), ("kp_a", c_double_p), ("kp_size_a", c_double_p), ("bearing_a", c_double_p),
                ("bearing_b", c_double_p), ("ray_sigma_a", c_double_p), ("ray_sigma_b", c_double_p), ("cam_a", Camera), ("cam_b", Camera),
                ("T_AB", C.c_double * 7)]


GATE_NONE, GATE_3D2D, GATE_2D2D = 0, 1, 2


def make_match_gate(mode, kp_b, kp_size_b, proj_into_b=None, proj_uncertainty=None, kp_a=None, kp_size_a=None, bearing_a=None,
                    bearing_b=None, ray_sigma_a=None, ray_sigma_b=None, cam_a=None, cam_b=None, T_AB=None):
    """okb_match_gate over numpy arrays (kept alive on the returned object)."""
    g = MatchGate()
    g.mode = mode
    keep = []
    for name, arr in (("kp_b", kp_b), ("kp_size_b", kp_size_b), ("proj_into_b", proj_into_b), ("proj_uncertainty", proj_uncertainty),
                      ("kp_a", kp_a), ("kp_size_a", kp_size_a), ("bearing_a", bearing_a), ("bearing_b", bearing_b),
                      ("ray_sigma_a", ray_sigma_a), ("ray_sigma_b", ray_sigma_b)):
        if arr is not None:
            a = np.ascontiguousarray(arr, np.float64)
            keep.append(a)
            setattr(g, name, a.ctypes.data_as(c_double_p))
    for name, cam in (("cam_a", cam_a), ("cam_b", cam_b)):
        if cam is not None:
            C.memmove(C.addressof(getattr(g, name)), np.array([cam], camera_dtype).ctypes.data, C.sizeof(Camera))
    if T_AB is not None:
        for k in range(7):
            g.T_AB[k] = float(T_AB[k])
    g._keep = keep
    return g


class ImageDesc(C.Structure):
    _fields_ = [("img", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32), ("_pad", C.c_int32),
                ("cam", Camera), ("R_CW", C.c_double * 9)]


class MatchJob(C.Structure):
    _fields_ = [("A", C.c_void_p), ("B", C.c_void_p), ("skipA", C.c_void_p), ("skipB", C.c_void_p), ("nA", C.c_int32),
                ("nB", C.c_int32), ("threshold", C.c_float), ("num_best", C.c_int32), ("use_ratio", C.c_int32), ("_pad", C.c_int32),
                ("gate", C.POINTER(MatchGate)), ("out_topk", C.c_void_p), ("out_pairs", C.c_void_p)]


class TrackRound(C.Structure):
    _fields_ = [("feat_slot_a", C.c_int32), ("cam_a", C.c_int32), ("cam_b", C.c_int32), ("_pad", C.c_int32)]


class TrackJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("pose_b", C.c_int32), ("sb_b", C.c_int32), ("feat_slot_b", C.c_int32),
                ("threshold", C.c_float), ("num_best", C.c_int32), ("n_rounds", C.c_int32), ("_pad", C.c_int32),
                ("rounds", C.POINTER(TrackRound)), ("assoc", C.c_void_p), ("assoc_cap", C.c_int32), ("n_assoc", C.POINTER(C.c_int32)),
                ("num_matches", C.POINTER(C.c_int32)), ("num_uncertain", C.POINTER(C.c_int32)), ("uninit", C.POINTER(C.c_uint32)),
                ("uninit_cap", C.c_int32), ("n_uninit", C.POINTER(C.c_int32))]


class StereoJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("pose", C.c_int32), ("feat_slot", C.c_int32), ("cam_a", C.c_int32), ("cam_b", C.c_int32),
                ("threshold", C.c_float), ("num_best", C.c_int32), ("_pad", C.c_int32), ("out", C.c_void_p), ("out_cap", C.c_int32),
                ("n_out", C.POINTER(C.c_int32))]


class Match2D2DJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("pose_a", C.c_int32), ("feat_slot_a", C.c_int32), ("cam_a", C.c_int32),
                ("pose_b", C.c_int32), ("feat_slot_b", C.c_int32), ("cam_b", C.c_int32), ("sb_current", C.c_int32),
                ("threshold", C.c_float), ("num_best", C.c_int32), ("out", C.c_void_p), ("out_cap", C.c_int32),
                ("n_out", C.POINTER(C.c_int32))]


class KeyframeCam(C.Structure):
    _fields_ = [("n_points", C.c_int32), ("n_matched", C.c_int32), ("hull_all", C.c_int32), ("hull_matched", C.c_int32),
                ("inside", C.c_int32), ("skipped", C.c_int32), ("area_all", C.c_double), ("area_matched", C.c_double),
                ("overlap", C.c_double), ("ratio", C.c_double)]


class KeyframeResult(C.Structure):
    _fields_ = [("overlap", C.c_double), ("ratio", C.c_double), ("need_keyframe", C.c_int32), ("_pad", C.c_int32)]


class KeyframeJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("feat_slot", C.c_int32), ("n_cams", C.c_int32), ("overlap_threshold", C.c_float),
                ("matching_ratio_threshold", C.c_float), ("_pad", C.c_int32), ("cams", C.POINTER(KeyframeCam)),
                ("out", C.POINTER(KeyframeResult))]


class RansacResult(C.Structure):
    _fields_ = [("ret", C.c_int32), ("n_correspondences", C.c_int32), ("n_inliers", C.c_int32), ("best", C.c_int32),
                ("n_outliers", C.c_int32), ("_pad", C.c_int32), ("T_WS", C.c_double * 7)]


class RansacJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("feat_slot", C.c_int32), ("n_cams", C.c_int32), ("max_iterations", C.c_int32),
                ("threshold", C.c_double), ("seed", C.c_uint64), ("hyp_inliers", C.POINTER(C.c_int32)),
                ("outliers", C.c_void_p), ("outlier_cap", C.c_int32), ("_pad", C.c_int32), ("out", C.POINTER(RansacResult))]


class Ransac2dCam(C.Structure):
    _fields_ = [("n_correspondences", C.c_int32), ("rot_inliers", C.c_int32), ("rel_inliers", C.c_int32),
                ("rot_best", C.c_int32), ("rel_best", C.c_int32), ("rotation_only", C.c_int32), ("applied", C.c_int32),
                ("n_outliers", C.c_int32), ("R_rot", C.c_double * 9), ("R_rel", C.c_double * 9), ("t_rel", C.c_double * 3)]


class Ransac2dResult(C.Structure):
    _fields_ = [("ret", C.c_int32), ("rotation_only", C.c_int32), ("pose_set", C.c_int32), ("n_outliers", C.c_int32),
                ("T_WS", C.c_double * 7)]


class Ransac2dJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("pose_b", C.c_int32), ("feat_slot_b", C.c_int32), ("pose_a", C.c_int32),
                ("feat_slot_a", C.c_int32), ("n_cams", C.c_int32), ("initialize_pose", C.c_int32),
                ("max_iterations", C.c_int32), ("threshold", C.c_double), ("seed", C.c_uint64),
                ("hyp_inliers", C.POINTER(C.c_int32)), ("cams", C.POINTER(Ransac2dCam)), ("outliers", C.c_void_p),
                ("outlier_cap", C.c_int32), ("_pad", C.c_int32), ("out", C.POINTER(Ransac2dResult))]


class DetectStoreJob(C.Structure):
    _fields_ = [("win", C.c_int32), ("feat_slot", C.c_int32), ("n_cams", C.c_int32), ("_pad", C.c_int32),
                ("images", C.POINTER(ImageDesc)), ("out_kp", C.c_void_p), ("out_desc", C.c_void_p), ("n_out", C.POINTER(C.c_int32))]


class PropagateJob(C.Structure):
    _fields_ = [("params", C.POINTER(ImuParams)), ("samples", C.c_void_p), ("n_samples", C.c_int32), ("_pad", C.c_int32),
                ("t0_ns", C.c_int64), ("t1_ns", C.c_int64), ("pose", c_double_p), ("speed_bias", c_double_p),
                ("covariance", c_double_p), ("jacobian", c_double_p), ("n_used", C.POINTER(C.c_int32))]


class WindowDesc(C.Structure):
    _fields_ = [("n_poses", C.c_int32), ("n_speed_bias", C.c_int32), ("n_extrinsics", C.c_int32),
                ("n_landmarks", C.c_int32), ("n_cameras", C.c_int32), ("n_obs", C.c_int32),
                ("n_imu_terms", C.c_int32), ("n_imu_samples", C.c_int32), ("n_pose_priors", C.c_int32),
                ("n_sb_priors", C.c_int32), ("n_relpose_terms", C.c_int32), ("_pad", C.c_int32),
                ("poses", C.c_void_p), ("speed_bias", C.c_void_p), ("extrinsics", C.c_void_p),
                ("extrinsics_fixed", C.c_void_p), ("landmarks", C.c_void_p), ("cameras", C.c_void_p),
                ("obs", C.c_void_p), ("imu_terms", C.c_void_p), ("imu_samples", C.c_void_p),
                ("imu_params", ImuParams), ("pose_priors", C.c_void_p), ("sb_priors", C.c_void_p),
                ("relpose_terms", C.c_void_p), ("marg", C.POINTER(MargPrior))]


class SolveOptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("min_iterations", C.c_int32), ("time_limit_s", C.c_double),
                ("use_cauchy_loss", C.c_int32), ("_pad", C.c_int32)]


class Summary(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32),
                ("num_successful_steps", C.c_int32), ("termination", C.c_int32), ("imu_redo_count", C.c_int32),
                ("final_radius", C.c_double), ("solve_time_s", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class DetectParams(C.Structure):
    _fields_ = [("uniformity_radius", C.c_double), ("absolute_threshold", C.c_double), ("max_keypoints", C.c_int32),
                ("desc_bytes", C.c_int32), ("rotation_invariance", C.c_int32), ("_pad", C.c_int32)]


# numpy dtypes with the C layout (checked against ctypes sizes in tests/test_abi.py)
camera_dtype = np.dtype([("model", "<i4"), ("width", "<i4"), ("height", "<i4"), ("_pad", "<i4"), ("fu", "<f8"),
                         ("fv", "<f8"), ("cu", "<f8"), ("cv", "<f8"), ("dist", "<f8", (8,))], align=True)
observation_dtype = np.dtype([("pose_idx", "<u4"), ("lm_idx", "<u4"), ("ext_idx", "<u4"), ("cam_idx", "<u4"),
                              ("z", "<f8", (2,)), ("sqrt_info", "<f8")], align=True)
imu_sample_dtype = np.dtype([("t_ns", "<i8"), ("gyro", "<f8", (3,)), ("acc", "<f8", (3,))], align=True)
imu_term_dtype = np.dtype([("pose0", "<u4"), ("sb0", "<u4"), ("pose1", "<u4"), ("sb1", "<u4"), ("t0_ns", "<i8"),
                           ("t1_ns", "<i8"), ("sample_offset", "<u4"), ("sample_count", "<u4")], align=True)
pose_prior_dtype = np.dtype([("pose_idx", "<u4"), ("_pad", "<u4"), ("meas", "<f8", (7,)),
                             ("sqrt_info", "<f8", (36,))], align=True)
sb_prior_dtype = np.dtype([("sb_idx", "<u4"), ("_pad", "<u4"), ("meas", "<f8", (9,)),
                           ("sqrt_info", "<f8", (81,))], align=True)
relpose_dtype = np.dtype([("ext0", "<u4"), ("ext1", "<u4"), ("sqrt_info", "<f8", (36,))], align=True)
keypoint_dtype = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                           ("octave", "<i4")], align=True)
pair_dtype = np.dtype([("index_a", "<i4"), ("distance", "<f4")], align=True)
stereo_match_dtype = np.dtype([("kp_a", "<i4"), ("kp_b", "<i4"), ("lm_slot_a", "<i4"), ("lm_slot_b", "<i4"),
                               ("can_be_initialized", "<i4"), ("_pad", "<i4"), ("hp_W", "<f8", (4,))], align=True)
ransac_outlier_dtype = np.dtype([("cam", "<i4"), ("kp", "<i4"), ("lm_slot", "<i4")], align=True)
ransac2d_outlier_dtype = np.dtype([("cam", "<i4"), ("kp_a", "<i4"), ("kp_b", "<i4"), ("lm_slot", "<i4")], align=True)
track_assoc_dtype = np.dtype([("round", "<i4"), ("cam_b", "<i4"), ("kp_b", "<i4"), ("lm_slot", "<i4"), ("uncertain", "<i4"),
                              ("_pad", "<i4")], align=True)


def ptr(a):
    """void* of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def dptr(a):
    if a is None:
        return None
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_double_p)


def make_camera(model, width, height, fu, fv, cu, cv, dist=()):
    cam = np.zeros(1, camera_dtype)[0]
    cam["model"], cam["width"], cam["height"] = model, width, height
    cam["fu"], cam["fv"], cam["cu"], cam["cv"] = fu, fv, cu, cv
    d = np.zeros(8)
    d[:len(dist)] = dist
    cam["dist"] = d
    return cam


def make_imu_params(a_max=176.0, g_max=7.8, sigma_g_c=12.0e-4, sigma_a_c=8.0e-3, sigma_bg=0.03, sigma_ba=0.1,
                    sigma_gw_c=4.0e-6, sigma_aw_c=4.0e-5, tau=3600.0, g=9.81007, a0=(0.0, 0.0, 0.0), rate=200):
    """Defaults = config/config_fpga_p2_euroc.yaml:35-46 of the reference."""
    p = ImuParams()
    p.a_max, p.g_max, p.sigma_g_c, p.sigma_a_c = a_max, g_max, sigma_g_c, sigma_a_c
    p.sigma_bg, p.sigma_ba, p.sigma_gw_c, p.sigma_aw_c = sigma_bg, sigma_ba, sigma_gw_c, sigma_aw_c
    p.tau, p.g, p.rate = tau, g, rate
    p.a0[0], p.a0[1], p.a0[2] = a0
    return p


def load_library(path=LIB_PATH):
    """Loads libokvis_b200.so; raises (never falls back) if it is missing."""
    if not os.path.exists(path):
        raise RuntimeError("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'`; "
                           "there is no CPU fallback for the product path" % path)
    lib = C.CDLL(path)
    lib.okb_last_error.restype = C.c_char_p
    lib.okb_last_error.argtypes = [C.c_void_p]
    lib.okb_kernel_launches.restype = C.c_int64
    lib.okb_kernel_launches.argtypes = [C.c_void_p]
    lib.okb_stream.restype = C.c_void_p
    lib.okb_stream.argtypes = [C.c_void_p]
    lib.okb_ctx_create.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.okb_ctx_destroy.argtypes = [C.c_void_p]
    lib.okb_ctx_destroy.restype = None
    slots_t = C.POINTER(C.c_int32)
    lib.okb_optimize_slots.argtypes = [C.c_void_p, C.c_int, slots_t, C.POINTER(SolveOptions), C.POINTER(Summary)]
    lib.okb_optimize_slots_async.argtypes = [C.c_void_p, C.c_int, slots_t, C.POINTER(SolveOptions)]
    lib.okb_optimize_slots_finish.argtypes = [C.c_void_p, C.c_int, slots_t, C.POINTER(Summary)]
    tab_t = C.POINTER(C.POINTER(C.c_double))
    lib.okb_window_download_slots.argtypes = [C.c_void_p, C.c_int, slots_t, tab_t, tab_t, tab_t, tab_t]
    return lib
