"""ctypes binding of libdnr_b200.so (include/dnr.h).  There is NO fallback: if the library is missing
or a call fails, this module raises."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libdnr_b200.so")

FLAG_ACTIVATED, FLAG_ANTIALIASED, FLAG_NORMALS, FLAG_ACCUMULATE, FLAG_EXACT_LISTS = 1, 2, 4, 8, 16
FLAG_HOST_CAMERA = 32
FLAG_PERSISTENT_WS = 256
LOSS_FUSED_BWD, LOSS_IMG_U8, LOSS_NORMAL_U8, LOSS_EDGE_FROM_IMAGE = 1, 2, 4, 8
REC_FLOATS, REC_FLOATS_N, GRAD_FLOATS = 12, 16, 16
DEPTH_LOSS_TYPES = {None: 0, "EdgeAwareLogL1": 1, "LogL1": 2, "L1": 3, "MSE": 4}

_f, _i, _p = C.c_float, C.c_int32, C.c_void_p


class DnrArgs(C.Structure):
    """Field-for-field mirror of `struct DnrArgs` in include/dnr.h (tests/test_abi.py checks the order)."""

    _fields_ = [
        ("n_gauss", _i), ("width", _i), ("height", _i), ("tile_size", _i), ("sh_degree", _i), ("sh_bases", _i),
        ("flags", C.c_uint32), ("list_shift", _i),
        ("near_plane", _f), ("far_plane", _f), ("eps2d", _f), ("radius_clip", _f),
        ("background", _f * 3), ("reserved1", _f),
        ("n_isects", C.c_int64),
        ("viewmat", _p), ("K", _p), ("c2w", _p),
        ("means", _p), ("quats", _p), ("scales", _p), ("opacities", _p), ("sh_dc", _p), ("sh_rest", _p),
        ("radii", _p), ("means2d", _p), ("depths", _p), ("conics", _p), ("opac_act", _p), ("compensations", _p),
        ("colors", _p), ("normals_world", _p), ("tiles_per_gauss", _p), ("depth_keys", _p), ("records", _p), ("cull_lim", _p),
        ("ws_scan", _p), ("ws_sort", _p), ("flatten_ids", _p), ("tile_offsets", _p), ("n_isects_dev", _p),
        ("out_rgb", _p), ("out_depth", _p), ("out_alpha", _p), ("out_normal", _p), ("out_surface_normal", _p),
        ("last_ids", _p), ("normal_norm", _p), ("clamp_mask", _p), ("depth_max", _p),
        ("v_rgb", _p), ("v_depth", _p), ("v_normal", _p), ("v_alpha", _p), ("grad_records", _p),
        ("v_means", _p), ("v_quats", _p), ("v_scales", _p), ("v_opacities", _p), ("v_sh_dc", _p), ("v_sh_rest", _p),
        ("v_means2d", _p), ("v_means2d_abs", _p),
        ("gt_depth", _p), ("gt_normal", _p), ("gt_rgb", _p), ("loss_partials", _p), ("v_loss", _p),
        ("depth_lambda", _f), ("depth_tolerance", _f), ("depth_loss_type", _i), ("use_normal_loss", _i),
        ("host_cam", _f * 32),
        ("reserved2", _p),
        ("loss_flags", C.c_uint32), ("reserved3", _i), ("gt_image", _p), ("v_l1", _p), ("touched", _p), ("stats", _p),
        ("v_viewmat", _p),
    ]


class DnrAgsLoss(C.Structure):
    """Mirror of struct DnrAgsLoss (include/dnr.h)."""

    _fields_ = [("width", _i), ("height", _i), ("depth_loss_type", _i), ("flags", C.c_uint32), ("depth_lambda", _f),
                ("depth_tolerance", _f), ("normal_lambda", _f), ("reserved", _i), ("pred_depth", _p), ("gt_depth", _p),
                ("confidence", _p), ("image", _p), ("surf_normal", _p), ("gt_normal", _p), ("pred_normal", _p),
                ("partials", _p), ("v_loss", _p), ("keep_mask", _p)]


AGS_CONF_GATE, AGS_ANGLE_MASK, AGS_NORMAL_U8, AGS_IMG_U8, AGS_CONF_RAW, AGS_CONF_U8, AGS_SIGNED_CHW = 1, 2, 4, 8, 16, 32, 64


class DnrAdamSeg(C.Structure):
    """Mirror of struct DnrAdamSeg (include/dnr.h)."""

    _fields_ = [("p", _p), ("g", _p), ("m", _p), ("v", _p), ("n", C.c_int64), ("lr", C.c_double), ("eps", C.c_double),
                ("bc1", C.c_double), ("bc2_sqrt", C.c_double), ("dense", C.c_int64)]


class DnrGradSeg(C.Structure):
    """Mirror of struct DnrGradSeg (include/dnr.h)."""

    _fields_ = [("g", _p), ("width", _i), ("dense", _i)]


PEER_MAX = 8


class DnrPeerReduce(C.Structure):
    """Mirror of struct DnrPeerReduce (include/dnr.h)."""

    _fields_ = [("world", _i), ("rank", _i), ("n_gauss", _i), ("reserved", _i), ("peer_flat", _p * PEER_MAX),
                ("peer_touched", _p * PEER_MAX), ("mask", _p)]


class DnrKnnGrid(C.Structure):
    """Mirror of struct DnrKnnGrid (include/dnr.h)."""

    _fields_ = [("lo", _f * 3), ("cell", _f), ("inv_cell", _f), ("dims", C.c_int32 * 3)]


class DnrTsdfGrid(C.Structure):
    """Mirror of struct DnrTsdfGrid (include/dnr.h)."""

    _fields_ = [("origin", _f * 3), ("voxel", _f), ("sdf_trunc", _f), ("dims", C.c_int32 * 3), ("voxels", _p)]


class DnrMcField(C.Structure):
    """Mirror of struct DnrMcField (include/dnr.h)."""

    _fields_ = [("values", _p), ("valid", _p), ("tsdf", _p), ("dims", C.c_int32 * 3), ("iso", _f), ("origin", _f * 3),
                ("spacing", _f)]


class DnrPoissonGrid(C.Structure):
    """Mirror of struct DnrPoissonGrid (include/dnr.h)."""

    _fields_ = [("origin", _f * 3), ("cell", _f), ("depth", _i), ("reserved", _i)]


class DnrGridDesc(C.Structure):
    """Mirror of struct DnrGridDesc (include/dnr.h)."""

    _fields_ = [("origin", _f * 3), ("cell", _f), ("dims", C.c_int32 * 3), ("channels", _i)]


POISSON_MIN_DEPTH, POISSON_MAX_DEPTH, POISSON_MAX_CYCLES = 4, 10, 100
ISO_POSE, ISO_MAX_DEPTH = 36, 10
_d = C.c_double


class DnrIsoFrames(C.Structure):
    """Mirror of struct DnrIsoFrames (include/dnr.h)."""

    _fields_ = [("depth", _p), ("normals", _p), ("poses", _p), ("n_frames", _i), ("width", _i), ("height", _i),
                ("cam_normals", _i), ("K", _d * 9), ("inv_K", _d * 9), ("depth_scale", _d), ("rel_delta", _d)]


class DnrIsoParams(C.Structure):
    """Mirror of struct DnrIsoParams (include/dnr.h)."""

    _fields_ = [("max_tsdf_rel", _d), ("max_tsdf_abs", _d), ("min_dot", _d), ("use_normals", _i), ("passes", _i)]


class DnrIsoGrid(C.Structure):
    """Mirror of struct DnrIsoGrid (include/dnr.h)."""

    _fields_ = [("origin", _d * 3), ("cell", _d), ("max_depth", _i), ("threshold", _i)]


DN_MAX_K, DN_OMNIDATA, DN_DSINE, DN_DEPTH_TO_NORMAL = 256, 0, 1, 2


class DnrDnPose(C.Structure):
    """Mirror of struct DnrDnPose (include/dnr.h)."""

    _fields_ = [("rinv", _d * 9), ("t", _d * 3)]


class DnrDnSearch(C.Structure):
    """Mirror of struct DnrDnSearch (include/dnr.h)."""

    _fields_ = [("lo", _d * 3), ("cell", _d), ("center", _d * 3), ("k", _i), ("orient", _i)]


POINTER_FIELDS = {n for n, t in DnrArgs._fields_ if t is _p}

_lib: Optional[C.CDLL] = None

# hand-written kernels launched per C-ABI call (cub's radix-sort / scan passes are counted separately)
KERNELS_PER_CALL = {
    "dnr_project_fwd": (1, 0), "dnr_bin_scan": (2, 8), "dnr_bin_sort": (3, 4), "dnr_raster_fwd": (1, 0),
    "dnr_finalize_fwd": (1, 0), "dnr_normal_from_depth": (1, 0), "dnr_raster_bwd": (1, 0), "dnr_project_bwd": (1, 0),
    "dnr_loss_fwd": (2, 0), "dnr_loss_bwd": (1, 0), "dnr_ags_loss_fwd": (2, 0), "dnr_ags_loss_bwd": (1, 0), "dnr_scale_loss_fwd": (1, 0), "dnr_scale_loss_bwd": (1, 0),
    "dnr_l1_fwd": (1, 0), "dnr_l1_bwd": (1, 0), "dnr_u8_to_f32": (1, 0),
    "dnr_ssim_fwd": (1, 0), "dnr_ssim_bwd": (1, 0), "dnr_ssim_fwd_ex": (1, 0), "dnr_ssim_bwd_ex": (1, 0), "dnr_photometric_fwd": (2, 0), "dnr_photometric_bwd": (1, 0), "dnr_adam_step": (1, 0), "dnr_adam_step_reduce": (2, 0),
    "dnr_grad_zero": (1, 0),
    "dnr_knn_build": (2, 1), "dnr_knn_query": (1, 0), "dnr_density": (1, 0), "dnr_ray_densities": (1, 0),
    "dnr_tsdf_integrate": (1, 0), "dnr_mc_count": (1, 6), "dnr_mc_emit": (2, 0),
    "dnr_grid_sample": (1, 0), "dnr_mesh_visibility": (1, 0),
    "dnr_rgb_metrics": (1, 0), "dnr_depth_metrics": (1, 0), "dnr_normal_metrics": (8, 0),
    "dnr_iso_samples": (2, 2), "dnr_iso_eval": (1, 0), "dnr_iso_corners": (3, 4),
    "dnr_dn_backproject": (1, 0), "dnr_dn_normals": (8, 5), "dnr_dn_consistency": (1, 0),
}
LAUNCHES = {"handwritten": 0, "cub": 0}
DEBUG_CAPTURE = os.environ.get("DNR_DEBUG_CAPTURE") == "1"


def capture_ok(where: str) -> None:
    """With DEBUG_CAPTURE set: raises, naming `where`, once an ongoing stream capture is no longer valid."""
    if not DEBUG_CAPTURE:
        return
    import torch

    try:  # raises cudaErrorStreamCaptureInvalidated once the capture is broken
        torch.cuda.is_current_stream_capturing()
    except Exception as exc:  # noqa: BLE001
        raise DnrError(f"stream capture invalidated by {where}: {exc}") from exc


class _Counting:
    """Thin proxy over the CDLL that counts kernel launches per call (bench.py's gpu_launches)."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        k = KERNELS_PER_CALL.get(name)
        if k is None:
            return fn

        def call(*args):
            LAUNCHES["handwritten"] += k[0]
            LAUNCHES["cub"] += k[1]
            rc = fn(*args)
            if DEBUG_CAPTURE:  # name the C-ABI call that invalidates an ongoing stream capture
                capture_ok(f"{name} (rc {rc})")
            return rc

        self.__dict__[name] = call
        return call


class DnrError(RuntimeError):
    pass


def load():
    """Loads the shared library, failing loudly when it has not been built (python -m dn_splatter_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DnrError(
            f"{LIB_PATH} is missing: build it with `python -m dn_splatter_b200.build` "
            "(nvcc, sm_90a). dn_splatter_b200 has no CPU or PyTorch fallback."
        )
    lib = C.CDLL(LIB_PATH)
    A = C.POINTER(DnrArgs)
    lib.dnr_version.restype = C.c_int
    lib.dnr_error_string.restype = C.c_char_p
    lib.dnr_error_string.argtypes = [C.c_int]
    for name in ("dnr_project_fwd", "dnr_bin_sort", "dnr_raster_fwd", "dnr_finalize_fwd", "dnr_normal_from_depth",
                 "dnr_raster_bwd", "dnr_project_bwd", "dnr_loss_fwd"):
        fn = getattr(lib, name)
        fn.restype = C.c_int
        fn.argtypes = [A, C.c_void_p]
    lib.dnr_bin_scan.restype = C.c_int
    lib.dnr_bin_scan.argtypes = [A, C.c_void_p, C.POINTER(C.c_int64)]
    lib.dnr_loss_bwd.restype = C.c_int
    lib.dnr_loss_bwd.argtypes = [A, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_ags_loss_fwd.restype = C.c_int
    lib.dnr_ags_loss_fwd.argtypes = [C.POINTER(DnrAgsLoss), C.c_void_p]
    lib.dnr_ags_loss_bwd.restype = C.c_int
    lib.dnr_ags_loss_bwd.argtypes = [C.POINTER(DnrAgsLoss), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_scale_loss_fwd.restype = C.c_int
    lib.dnr_scale_loss_fwd.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dnr_scale_loss_bwd.restype = C.c_int
    lib.dnr_scale_loss_bwd.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_l1_fwd.restype = C.c_int
    lib.dnr_l1_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
    lib.dnr_l1_bwd.restype = C.c_int
    lib.dnr_l1_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_u8_to_f32.restype = C.c_int
    lib.dnr_u8_to_f32.argtypes = [C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    lib.dnr_ssim_fwd.restype = C.c_int
    lib.dnr_ssim_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_ssim_fwd_ex.restype = C.c_int
    lib.dnr_ssim_fwd_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p]
    lib.dnr_ssim_bwd_ex.restype = C.c_int
    lib.dnr_ssim_bwd_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]
    lib.dnr_photometric_fwd.restype = C.c_int
    lib.dnr_photometric_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                        C.c_void_p, C.c_void_p]
    lib.dnr_photometric_bwd.restype = C.c_int
    lib.dnr_photometric_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_adam_step.restype = C.c_int
    lib.dnr_adam_step.argtypes = [C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_void_p]
    lib.dnr_adam_step_reduce.restype = C.c_int
    lib.dnr_adam_step_reduce.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
    lib.dnr_grad_zero.restype = C.c_int
    lib.dnr_grad_zero.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.dnr_knn_workspace_bytes.restype = C.c_int64
    lib.dnr_knn_workspace_bytes.argtypes = [C.c_int32, C.c_void_p]
    lib.dnr_knn_build.restype = C.c_int
    lib.dnr_knn_build.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.dnr_knn_query.restype = C.c_int
    lib.dnr_knn_query.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p, C.c_void_p]
    lib.dnr_density.restype = C.c_int
    lib.dnr_density.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_int32, C.c_float, C.c_void_p, C.c_void_p]
    lib.dnr_ray_densities.restype = C.c_int
    lib.dnr_ray_densities.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_tsdf_integrate.restype = C.c_int
    lib.dnr_tsdf_integrate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_float, C.c_void_p]
    lib.dnr_mc_count_workspace_bytes.restype = C.c_int64
    lib.dnr_mc_count_workspace_bytes.argtypes = [C.c_void_p]
    lib.dnr_mc_count.restype = C.c_int
    lib.dnr_mc_count.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.dnr_mc_emit_workspace_bytes.restype = C.c_int64
    lib.dnr_mc_emit_workspace_bytes.argtypes = [C.c_void_p]
    lib.dnr_mc_emit.restype = C.c_int
    lib.dnr_mc_emit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]
    lib.dnr_poisson_splat_workspace_bytes.restype = C.c_int64
    lib.dnr_poisson_splat_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
    lib.dnr_poisson_splat.restype = C.c_int
    lib.dnr_poisson_splat.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_poisson_solve_workspace_bytes.restype = C.c_int64
    lib.dnr_poisson_solve_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.dnr_poisson_solve.restype = C.c_int
    lib.dnr_poisson_solve.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int32, C.c_void_p, C.c_int64,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_grid_sample.restype = C.c_int
    lib.dnr_grid_sample.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.dnr_mesh_depth_workspace_bytes.restype = C.c_int64
    lib.dnr_mesh_depth_workspace_bytes.argtypes = [C.c_int64]
    lib.dnr_mesh_depth.restype = C.c_int
    lib.dnr_mesh_depth.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_float, C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.dnr_mesh_visibility.restype = C.c_int
    lib.dnr_mesh_visibility.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                        C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_rgb_metrics.restype = C.c_int
    lib.dnr_rgb_metrics.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                    C.c_void_p]
    lib.dnr_depth_metrics.restype = C.c_int
    lib.dnr_depth_metrics.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p]
    lib.dnr_normal_metrics_workspace_bytes.restype = C.c_int64
    lib.dnr_normal_metrics_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.dnr_normal_metrics.restype = C.c_int
    lib.dnr_normal_metrics.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                       C.c_void_p, C.c_void_p]
    lib.dnr_ssim_bwd.restype = C.c_int
    lib.dnr_ssim_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]
    lib.dnr_bin_scan_workspace_bytes.restype = C.c_size_t
    lib.dnr_bin_scan_workspace_bytes.argtypes = [C.c_int32]
    lib.dnr_bin_sort_workspace_bytes.restype = C.c_size_t
    lib.dnr_bin_sort_workspace_bytes.argtypes = [C.c_int32, C.c_int64, C.c_int32]
    lib.dnr_iso_samples_workspace_bytes.restype = C.c_int64
    lib.dnr_iso_samples_workspace_bytes.argtypes = [C.c_void_p, C.c_int32]
    lib.dnr_iso_samples.restype = C.c_int
    lib.dnr_iso_samples.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_iso_eval.restype = C.c_int
    lib.dnr_iso_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.dnr_iso_octree_workspace_bytes.restype = C.c_int64
    lib.dnr_iso_octree_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
    lib.dnr_iso_octree.restype = C.c_int
    lib.dnr_iso_octree.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.dnr_iso_corners_workspace_bytes.restype = C.c_int64
    lib.dnr_iso_corners_workspace_bytes.argtypes = [C.c_void_p, C.c_int64]
    lib.dnr_iso_corners.restype = C.c_int
    lib.dnr_iso_corners.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_iso_fill.restype = C.c_int
    lib.dnr_iso_fill.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_dn_backproject.restype = C.c_int
    lib.dnr_dn_backproject.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_dn_normals_workspace_bytes.restype = C.c_int64
    lib.dnr_dn_normals_workspace_bytes.argtypes = [C.c_int64]
    lib.dnr_dn_normals.restype = C.c_int
    lib.dnr_dn_normals.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dnr_dn_consistency.restype = C.c_int
    lib.dnr_dn_consistency.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_double, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    _lib = _Counting(lib)
    return _lib


EXPORTS = (
    "dnr_version", "dnr_error_string", "dnr_project_fwd", "dnr_bin_scan_workspace_bytes", "dnr_bin_scan",
    "dnr_bin_sort_workspace_bytes", "dnr_bin_sort", "dnr_raster_fwd", "dnr_finalize_fwd", "dnr_normal_from_depth",
    "dnr_raster_bwd", "dnr_project_bwd", "dnr_loss_fwd", "dnr_loss_bwd", "dnr_ags_loss_fwd", "dnr_ags_loss_bwd", "dnr_scale_loss_fwd", "dnr_scale_loss_bwd",
    "dnr_l1_fwd", "dnr_l1_bwd", "dnr_u8_to_f32", "dnr_ssim_fwd", "dnr_ssim_bwd", "dnr_ssim_fwd_ex", "dnr_ssim_bwd_ex", "dnr_photometric_fwd", "dnr_photometric_bwd", "dnr_adam_step", "dnr_adam_step_reduce", "dnr_grad_zero", "dnr_knn_workspace_bytes", "dnr_knn_build", "dnr_knn_query",
    "dnr_density", "dnr_ray_densities", "dnr_tsdf_integrate", "dnr_mc_count_workspace_bytes", "dnr_mc_count",
    "dnr_mc_emit_workspace_bytes", "dnr_mc_emit", "dnr_poisson_splat_workspace_bytes", "dnr_poisson_splat",
    "dnr_poisson_solve_workspace_bytes", "dnr_poisson_solve", "dnr_grid_sample", "dnr_mesh_depth_workspace_bytes",
    "dnr_mesh_depth", "dnr_mesh_visibility", "dnr_rgb_metrics", "dnr_depth_metrics", "dnr_normal_metrics_workspace_bytes",
    "dnr_normal_metrics", "dnr_iso_samples_workspace_bytes", "dnr_iso_samples", "dnr_iso_eval",
    "dnr_iso_octree_workspace_bytes", "dnr_iso_octree", "dnr_iso_corners_workspace_bytes", "dnr_iso_corners", "dnr_iso_fill",
    "dnr_dn_backproject", "dnr_dn_normals_workspace_bytes", "dnr_dn_normals", "dnr_dn_consistency",
)


def check(code: int, what: str) -> None:
    if code != 0:
        msg = load().dnr_error_string(code).decode()
        raise DnrError(f"{what} failed with code {code}: {msg}")


def stream() -> C.c_void_p:
    """The current CUDA stream, as the `void* stream` argument of a library call."""
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def need_cuda(*tensors) -> None:
    for t in tensors:
        if t.device.type != "cuda":
            raise DnrError("dn_splatter_b200 needs CUDA tensors (no CPU path)")


def workspace_bytes(query, *args) -> int:
    """What the `dnr_*_workspace_bytes` query asks for; raises with the library's error code when it returns one."""
    n = int(query(*args))
    if n < 0:
        check(n, query.__name__)
    return n


def workspace(query, *args, device):
    """(uint8 workspace on `device`, its size in bytes) for the `dnr_*_workspace_bytes` query.  At least one byte is
    allocated: a zero-byte tensor's data_ptr() is 0, which the library rejects as DNR_E_NULL."""
    import torch

    n = workspace_bytes(query, *args)
    return torch.empty(max(n, 1), dtype=torch.uint8, device=device), n
