"""Host-side mirror of the reference's operator boundary for the PatchMatch hot path.

`runcuda(gs)` here takes the same information the reference's `int runcuda(GlobalState &gs)`
(gipuma.h:2) takes — AlgorithmParameters, the per-view Camera_cu fields, the view selection subset and
the images — and produces the same outputs (`lines.norm4`: world normal + depth, `lines.c`: cost).  All
compute goes through the C-ABI of `libgipuma_b200.so` (include/gipuma_b200.h, hand-written sm_90a
CUDA); there is no CPU path: loading fails loudly when the library has not been built, and every call
fails loudly without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GIPUMA_B200_LIB", os.path.join(_HERE, "libgipuma_b200.so"))

GPM_RNG_REFERENCE, GPM_RNG_STATEFUL = 0, 1


class GpmParams(C.Structure):
    _fields_ = [("box_hsize", C.c_int), ("box_vsize", C.c_int),
                ("tau_color", C.c_float), ("tau_gradient", C.c_float),
                ("alpha", C.c_float), ("gamma", C.c_float),
                ("min_disparity", C.c_float), ("max_disparity", C.c_float),
                ("iterations", C.c_int), ("n_best", C.c_int), ("cost_comb", C.c_int),
                ("good_factor", C.c_float), ("depthMin", C.c_float), ("depthMax", C.c_float)]


class GpmCamera(C.Structure):
    _fields_ = [("K", C.c_float * 9), ("K_inv", C.c_float * 9), ("R", C.c_float * 9),
                ("M_inv", C.c_float * 9), ("R_orig_inv", C.c_float * 9),
                ("t", C.c_float * 3), ("C", C.c_float * 3), ("P_col34", C.c_float * 3),
                ("fx", C.c_float), ("fy", C.c_float), ("f", C.c_float), ("alpha", C.c_float),
                ("baseline", C.c_float)]


class GpmBatchDesc(C.Structure):
    _fields_ = [("n_images", C.c_int), ("width", C.c_int), ("height", C.c_int),
                ("images", C.POINTER(C.c_void_p)), ("pitch_bytes", C.c_size_t), ("P", C.POINTER(C.c_double)),
                ("cam_scale", C.c_double), ("params", GpmParams), ("min_angle", C.c_float), ("max_angle", C.c_float),
                ("max_views", C.c_int), ("ref_indices", C.POINTER(C.c_int)), ("n_refs", C.c_int),
                ("devices", C.POINTER(C.c_int)), ("n_devices", C.c_int), ("seed", C.c_ulonglong),
                ("out_dir", C.c_char_p), ("out_norm4", C.POINTER(C.c_float)), ("out_cost", C.POINTER(C.c_float))]


class GpmBatchStats(C.Structure):
    _fields_ = [("jobs_done", C.c_int), ("sweep_ms_total", C.c_double), ("per_job_sweep_ms", C.POINTER(C.c_float)),
                ("per_job_views", C.POINTER(C.c_int)), ("per_job_device", C.POINTER(C.c_int))]


class GpmGeoBatchDesc(C.Structure):
    _fields_ = [("batch", GpmBatchDesc), ("channels", C.c_int), ("geo_iterations", C.c_int), ("weight", C.c_float),
                ("max_err", C.c_float)]


class GpmGeoBatchStats(C.Structure):
    _fields_ = [("batch", GpmBatchStats), ("n_pass1", C.c_int), ("pass1_views", C.POINTER(C.c_int)),
                ("pass1_sweep_ms", C.POINTER(C.c_float)), ("ref_views", C.POINTER(C.c_int))]


class GpmJobOpts(C.Structure):
    _fields_ = [("photometric", C.c_int), ("ncc_min_std", C.c_float), ("propagation", C.c_int)]


class GpmViewSel(C.Structure):
    _fields_ = [("kind", C.c_int), ("tau_init", C.c_float), ("alpha", C.c_float), ("tau_bad", C.c_float),
                ("n_good", C.c_int), ("n_bad", C.c_int), ("beta", C.c_float), ("w_keep", C.c_float)]


class GpmPriorBuild(C.Structure):
    _fields_ = [("step", C.c_int), ("support_cost", C.c_float)]


class GpmPriorInfo(C.Structure):
    _fields_ = [("support", C.c_longlong), ("triangles", C.c_longlong), ("with_prior", C.c_longlong)]


class GpmPriorOpts(C.Structure):
    _fields_ = [("weight", C.c_float), ("depth_sigma", C.c_float), ("normal_sigma_deg", C.c_float), ("step", C.c_int),
                ("support_cost", C.c_float), ("iterations", C.c_int), ("info", C.POINTER(GpmPriorInfo))]


class GpmJbuParams(C.Structure):
    _fields_ = [("radius", C.c_int), ("sigma_space", C.c_float), ("sigma_range", C.c_float)]


class GpmMsBatchDesc(C.Structure):
    _fields_ = [("geo", GpmGeoBatchDesc), ("levels", C.c_int), ("jbu", GpmJbuParams)]


MS_MAX_LEVELS = 4


class GpmMsBatchStats(C.Structure):
    _fields_ = [("batch", GpmBatchStats), ("n_views", C.c_int), ("views", C.POINTER(C.c_int)),
                ("level_sweep_ms", C.c_double * MS_MAX_LEVELS), ("level_upsample_ms", C.c_double * MS_MAX_LEVELS)]


class GpmMsPriorOpts(C.Structure):
    _fields_ = [("photometric", C.POINTER(GpmPriorOpts)), ("geometric", C.POINTER(GpmPriorOpts)),
                ("level_build_ms", C.c_double * MS_MAX_LEVELS)]


class GpmMsRestoreOpts(C.Structure):
    _fields_ = [("photo_iterations", C.c_int), ("threshold", C.c_float), ("iterations", C.c_int),
                ("restored", C.POINTER(C.c_int))]


class GpmRefineOpts(C.Structure):
    _fields_ = [("kind", C.c_int), ("perturbation", C.c_float)]


class GpmFuseCamera(C.Structure):
    _fields_ = [("M_inv", C.c_float * 9), ("P", C.c_float * 12), ("f", C.c_float)]


class GpmFuseDesc(C.Structure):
    _fields_ = [("n_views", C.c_int), ("width", C.c_int), ("height", C.c_int), ("norm4", C.c_void_p), ("images", C.c_void_p),
                ("channels", C.c_int), ("on_device", C.c_int), ("P", C.POINTER(C.c_double)), ("cam_scale", C.c_double),
                ("depth_min", C.c_float), ("depth_max", C.c_float), ("disp_thresh", C.c_float), ("normal_thresh", C.c_float),
                ("num_consistent", C.c_int), ("device", C.c_int)]


class GpmFuseRule(C.Structure):
    _fields_ = [("kind", C.c_int), ("reproj_px", C.c_float), ("depth_rel", C.c_float)]


class GpmFuseResult(C.Structure):
    _fields_ = [("count", C.c_longlong), ("capacity", C.c_longlong), ("vertices", C.c_void_p), ("source", C.c_void_p),
                ("used", C.c_void_p), ("fuse_ms", C.c_float), ("upload_ms", C.c_float)]


class GpmNnDesc(C.Structure):
    _fields_ = [("n_query", C.c_longlong), ("n_data", C.c_longlong), ("query", C.c_void_p), ("data", C.c_void_p),
                ("on_device", C.c_int), ("device", C.c_int), ("max_dist", C.c_float)]


class GpmNnResult(C.Structure):
    _fields_ = [("dist", C.c_void_p), ("upload_ms", C.c_float), ("build_ms", C.c_float), ("query_ms", C.c_float),
                ("cell_size", C.c_float), ("n_cells", C.c_longlong)]


class GpmTsdfDesc(C.Structure):
    _fields_ = [("n_views", C.c_int), ("width", C.c_int), ("height", C.c_int), ("depth", C.c_void_p), ("on_device", C.c_int),
                ("P", C.POINTER(C.c_double)), ("cam_scale", C.c_double), ("depth_min", C.c_float), ("depth_max", C.c_float),
                ("origin", C.c_float * 3), ("voxel", C.c_float), ("dims", C.c_int * 3), ("trunc", C.c_float),
                ("device", C.c_int)]


class GpmTsdfResult(C.Structure):
    _fields_ = [("D", C.c_void_p), ("weight", C.c_void_p), ("upload_ms", C.c_float), ("integrate_ms", C.c_float)]


class GpmMeshDesc(C.Structure):
    _fields_ = [("D", C.c_void_p), ("weight", C.c_void_p), ("on_device", C.c_int), ("origin", C.c_float * 3),
                ("voxel", C.c_float), ("dims", C.c_int * 3), ("min_weight", C.c_int), ("device", C.c_int)]


class GpmMeshResult(C.Structure):
    _fields_ = [("n_vertices", C.c_longlong), ("n_faces", C.c_longlong), ("vertex_capacity", C.c_longlong),
                ("face_capacity", C.c_longlong), ("vertices", C.c_void_p), ("faces", C.c_void_p),
                ("upload_ms", C.c_float), ("extract_ms", C.c_float)]


# one vertex of the fused point cloud: the packed 27-byte record of storePlyFileBinary (displayUtils.h:84-142)
PLY_VERTEX = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                       ("red", "u1"), ("green", "u1"), ("blue", "u1")])


class GipumaError(RuntimeError):
    pass


_lib = None


def load_library():
    """dlopen libgipuma_b200.so and declare the C-ABI.  Raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise GipumaError("%s is missing: build it with `python -m gipuma_b200.build` "
                          "(no CPU fallback exists)" % LIB_PATH)
    L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    vp, fp = C.c_void_p, C.POINTER(C.c_float)
    L.gpm_last_error.restype = C.c_char_p
    L.gpm_version.restype = C.c_char_p
    L.gpm_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int, C.c_int]
    L.gpm_destroy.argtypes = [vp]
    L.gpm_destroy.restype = None
    L.gpm_set_params.argtypes = [vp, C.POINTER(GpmParams)]
    L.gpm_set_reference.argtypes = [vp, vp, C.c_size_t, C.c_int, C.POINTER(GpmCamera)]
    L.gpm_set_view.argtypes = [vp, C.c_int, vp, C.c_size_t, C.c_int, C.POINTER(GpmCamera)]
    L.gpm_set_reference_color.argtypes = L.gpm_set_reference.argtypes
    L.gpm_set_view_color.argtypes = L.gpm_set_view.argtypes
    L.gpm_set_num_views.argtypes = [vp, C.c_int]
    L.gpm_set_view_depth.argtypes = [vp, C.c_int, vp, C.c_size_t, C.c_int]
    L.gpm_set_geometric.argtypes = [vp, C.c_float, C.c_float]
    L.gpm_set_photometric.argtypes = [vp, C.c_int, C.c_float]
    L.gpm_set_propagation.argtypes = [vp, C.c_int]
    L.gpm_set_view_selection.argtypes = [vp, C.POINTER(GpmViewSel)]
    L.gpm_get_view_masks.argtypes = [vp, vp]
    L.gpm_set_rng.argtypes = [vp, C.c_ulonglong, C.c_int]
    L.gpm_set_state.argtypes = [vp, vp, vp, C.c_int]
    L.gpm_get_state.argtypes = [vp, vp, vp, C.c_int]
    L.gpm_init.argtypes = [vp]
    L.gpm_sweep.argtypes = [vp, C.c_int]
    L.gpm_phase.argtypes = [vp, C.c_int, C.c_int]
    L.gpm_finalize.argtypes = [vp]
    L.gpm_cost_eval.argtypes = [vp, vp, vp, C.c_int]
    L.gpm_run.argtypes = [vp, fp]
    L.gpm_get_stats.argtypes = [vp, C.POINTER(C.c_ulonglong)]
    L.gpm_reset_stats.argtypes = [vp]
    L.gpm_set_option.argtypes = [vp, C.c_char_p, C.c_int]
    L.gpm_stream.argtypes = [vp]
    L.gpm_prepare_cameras.argtypes = [C.POINTER(C.c_double), C.c_int, C.c_double, C.POINTER(GpmCamera)]
    L.gpm_select_views.argtypes = [C.POINTER(GpmCamera), C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int,
                                   C.POINTER(C.c_int), fp]
    L.gpm_write_dmb.argtypes = [C.c_char_p, fp, C.c_int, C.c_int, C.c_int]
    L.gpm_read_dmb.argtypes = [C.c_char_p, fp, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.gpm_write_result_dmb.argtypes = [C.c_char_p, C.c_char_p, fp, C.c_int, C.c_int]
    L.gpm_init_planes.argtypes = [vp]
    L.gpm_shard_num_stages.argtypes = [vp]
    L.gpm_shard_stage_floats.argtypes = [vp, C.c_int]
    L.gpm_shard_stage_floats.restype = C.c_longlong
    L.gpm_shard_stage.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp]
    L.gpm_shard_finish_init.argtypes = [vp, vp, C.c_int]
    L.gpm_shard_unique_id.argtypes = [vp]
    L.gpm_shard_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.gpm_shard_comm_attach.argtypes = [vp, vp, C.c_int, C.c_int]
    L.gpm_shard_run.argtypes = [vp, fp]
    L.gpm_measure_fetch_peak.argtypes = [vp, C.POINTER(C.c_double)]
    L.gpm_batch_run.argtypes = [C.POINTER(GpmBatchDesc), C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run.argtypes = [C.POINTER(GpmGeoBatchDesc), C.POINTER(GpmGeoBatchStats)]
    L.gpm_batch_run_photo.argtypes = [C.POINTER(GpmBatchDesc), C.c_int, C.c_float, C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run_photo.argtypes = [C.POINTER(GpmGeoBatchDesc), C.c_int, C.c_float, C.POINTER(GpmGeoBatchStats)]
    L.gpm_batch_run_opts.argtypes = [C.POINTER(GpmBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run_opts.argtypes = [C.POINTER(GpmGeoBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmGeoBatchStats)]
    L.gpm_batch_run_vsel.argtypes = [C.POINTER(GpmBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel), C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run_vsel.argtypes = [C.POINTER(GpmGeoBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                         C.POINTER(GpmGeoBatchStats)]
    L.gpm_set_planar_prior.argtypes = [vp, vp, C.c_size_t, C.c_int]
    L.gpm_get_planar_prior.argtypes = [vp, vp, C.c_int]
    L.gpm_build_planar_prior.argtypes = [vp, C.POINTER(GpmPriorBuild), C.POINTER(GpmPriorInfo)]
    L.gpm_set_prior.argtypes = [vp, C.c_float, C.c_float, C.c_float]
    L.gpm_offer_prior.argtypes = [vp]
    L.gpm_batch_run_prior.argtypes = [C.POINTER(GpmBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                      C.POINTER(GpmPriorOpts), C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run_prior.argtypes = [C.POINTER(GpmGeoBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                          C.POINTER(GpmPriorOpts), C.POINTER(GpmGeoBatchStats)]
    L.gpm_batch_last_error.restype = C.c_char_p
    L.gpm_stream.restype = vp
    L.gpm_downsample.argtypes = [C.c_int, vp, C.c_size_t, C.c_int, C.c_int, C.c_int, vp, C.c_int]
    L.gpm_upsample_planes.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(GpmJbuParams), vp, vp]
    L.gpm_ms_batch_run.argtypes = [C.POINTER(GpmMsBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                   C.POINTER(GpmMsBatchStats)]
    L.gpm_ms_batch_run_prior.argtypes = [C.POINTER(GpmMsBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                         C.POINTER(GpmMsPriorOpts), C.POINTER(GpmMsBatchStats)]
    L.gpm_ms_batch_run_restore.argtypes = [C.POINTER(GpmMsBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                           C.POINTER(GpmMsPriorOpts), C.POINTER(GpmMsRestoreOpts), C.POINTER(GpmMsBatchStats)]
    L.gpm_set_geo_mask.argtypes = [vp, vp, C.c_size_t, C.c_int]
    L.gpm_set_refinement.argtypes = [vp, C.c_int, C.c_float]
    L.gpm_batch_run_refine.argtypes = [C.POINTER(GpmBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                       C.POINTER(GpmPriorOpts), C.POINTER(GpmRefineOpts), C.POINTER(GpmBatchStats)]
    L.gpm_geo_batch_run_refine.argtypes = [C.POINTER(GpmGeoBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                           C.POINTER(GpmPriorOpts), C.POINTER(GpmRefineOpts), C.POINTER(GpmGeoBatchStats)]
    L.gpm_ms_batch_run_refine.argtypes = [C.POINTER(GpmMsBatchDesc), C.POINTER(GpmJobOpts), C.POINTER(GpmViewSel),
                                          C.POINTER(GpmMsPriorOpts), C.POINTER(GpmMsRestoreOpts), C.POINTER(GpmRefineOpts),
                                          C.POINTER(GpmMsBatchStats)]
    L.gpm_fuse_cameras.argtypes = [C.POINTER(C.c_double), C.c_int, C.c_double, C.POINTER(GpmFuseCamera)]
    L.gpm_fuse.argtypes = [C.POINTER(GpmFuseDesc), C.POINTER(GpmFuseResult)]
    L.gpm_fuse_with_rule.argtypes = [C.POINTER(GpmFuseDesc), C.POINTER(GpmFuseRule), C.POINTER(GpmFuseResult)]
    L.gpm_write_ply.argtypes = [C.c_char_p, vp, C.c_longlong]
    L.gpm_nearest_dist.argtypes = [C.POINTER(GpmNnDesc), C.POINTER(GpmNnResult)]
    L.gpm_tsdf_integrate.argtypes = [C.POINTER(GpmTsdfDesc), C.POINTER(GpmTsdfResult)]
    L.gpm_mesh_extract.argtypes = [C.POINTER(GpmMeshDesc), C.POINTER(GpmMeshResult)]
    L.gpm_write_ply_mesh.argtypes = [C.c_char_p, vp, C.c_longlong, vp, C.c_longlong]
    for name in ("gpm_create", "gpm_set_params", "gpm_set_reference", "gpm_set_view", "gpm_set_reference_color",
                 "gpm_set_view_color", "gpm_set_num_views", "gpm_set_view_depth", "gpm_set_geometric", "gpm_set_photometric",
                 "gpm_set_propagation", "gpm_set_view_selection", "gpm_get_view_masks", "gpm_set_rng", "gpm_set_state", "gpm_get_state", "gpm_init", "gpm_sweep", "gpm_phase",
                 "gpm_finalize", "gpm_cost_eval", "gpm_run", "gpm_get_stats", "gpm_reset_stats", "gpm_set_option",
                 "gpm_init_planes", "gpm_shard_num_stages", "gpm_shard_stage", "gpm_shard_finish_init", "gpm_shard_unique_id",
                 "gpm_shard_comm_init", "gpm_shard_comm_attach", "gpm_shard_run", "gpm_measure_fetch_peak", "gpm_batch_run",
                 "gpm_geo_batch_run", "gpm_batch_run_photo", "gpm_geo_batch_run_photo", "gpm_batch_run_opts", "gpm_geo_batch_run_opts",
                 "gpm_batch_run_vsel", "gpm_geo_batch_run_vsel", "gpm_set_planar_prior", "gpm_get_planar_prior",
                 "gpm_build_planar_prior", "gpm_set_prior", "gpm_offer_prior", "gpm_batch_run_prior",
                 "gpm_geo_batch_run_prior", "gpm_downsample", "gpm_upsample_planes", "gpm_ms_batch_run", "gpm_ms_batch_run_prior",
                 "gpm_ms_batch_run_restore", "gpm_set_geo_mask", "gpm_set_refinement", "gpm_batch_run_refine",
                 "gpm_geo_batch_run_refine", "gpm_ms_batch_run_refine",
                 "gpm_prepare_cameras", "gpm_select_views", "gpm_write_dmb", "gpm_read_dmb", "gpm_write_result_dmb",
                 "gpm_fuse_cameras", "gpm_fuse", "gpm_fuse_with_rule", "gpm_write_ply", "gpm_nearest_dist",
                 "gpm_tsdf_integrate", "gpm_mesh_extract", "gpm_write_ply_mesh"):
        getattr(L, name).restype = C.c_int
    _lib = L
    return L


def pack_params(p) -> GpmParams:
    return GpmParams(p.box_hsize, p.box_vsize, p.tau_color, p.tau_gradient, p.alpha, p.gamma,
                     p.min_disparity, p.max_disparity, p.iterations, p.n_best, p.cost_comb,
                     p.good_factor, p.depthMin, p.depthMax)


def pack_camera(c) -> GpmCamera:
    g = GpmCamera()
    g.K[:] = c.K.ravel().tolist()
    g.K_inv[:] = c.K_inv.ravel().tolist()
    g.R[:] = c.R.ravel().tolist()
    g.M_inv[:] = c.M_inv.ravel().tolist()
    g.R_orig_inv[:] = c.R_orig_inv.ravel().tolist()
    g.t[:] = c.t.ravel().tolist()
    g.C[:] = c.C.ravel().tolist()
    g.P_col34[:] = c.P[:, 3].ravel().tolist()
    g.fx, g.fy, g.f, g.alpha, g.baseline = c.fx, c.fy, c.f, c.alpha, c.baseline
    return g


def _ptr(a):
    """void* of a numpy array, a torch tensor (host or CUDA) or a raw integer address.  The C-ABI reads / writes float32
    row-major memory: anything else is refused here instead of being reinterpreted silently."""
    if a is None:
        return None, 0
    if isinstance(a, int):
        return C.c_void_p(a), 1
    if isinstance(a, np.ndarray):
        if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
            raise TypeError("numpy buffers must be C-contiguous float32 (got %s, contiguous=%s)" % (a.dtype, a.flags["C_CONTIGUOUS"]))
        return C.c_void_p(a.ctypes.data), 0
    if hasattr(a, "data_ptr"):
        import torch
        if a.dtype != torch.float32 or not a.is_contiguous():
            raise TypeError("torch buffers must be contiguous float32 (got %s)" % (a.dtype,))
        if a.is_cuda:
            torch.cuda.current_stream(a.device).synchronize()      # the context works on its own stream: the producer must be done
        return C.c_void_p(a.data_ptr()), 1 if a.is_cuda else 0
    raise TypeError("unsupported buffer type %r" % type(a))


def _image(a):
    """Images may come as any real numpy dtype: converted to contiguous float32 here (what main.cpp's loaders produce)."""
    if isinstance(a, np.ndarray) and (a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]):
        return np.ascontiguousarray(a, dtype=np.float32)
    return a


# Defaults of the geometric-consistency pass (DESIGN.md §14), chosen from the measurement in tools/geo_bench.py.
GEO_WEIGHT, GEO_MAX_ERR = 0.5, 3.0


def check_geometric(weight: float, max_err: float):
    """The argument rules of gpm_set_geometric, checked before any call into the library."""
    if not (np.isfinite(weight) and weight >= 0):
        raise ValueError("weight must be finite and >= 0 (got %r)" % (weight,))
    if not (np.isfinite(max_err) and max_err > 0):
        raise ValueError("max_err must be finite and > 0 (got %r)" % (max_err,))


# Photometric costs (DESIGN.md §15): "pm", the reference's, and "ncc".  NCC_MIN_STD is the default of the NCC cost's min_std,
# in grey levels, chosen from the measurement in tools/ncc_bench.py.
PHOTOMETRIC = {"pm": 0, "ncc": 1}
NCC_MIN_STD = 4.0


def check_photometric(kind: str, min_std: float) -> int:
    """The argument rules of gpm_set_photometric, checked before any call into the library; returns the C-ABI's kind."""
    if kind not in PHOTOMETRIC:
        raise ValueError("photometric cost must be one of %s (got %r)" % (sorted(PHOTOMETRIC), kind))
    if kind == "ncc" and not (np.isfinite(min_std) and min_std > 0):
        raise ValueError("min_std must be finite and > 0 (got %r)" % (min_std,))
    return PHOTOMETRIC[kind]


# Propagation (DESIGN.md §16): "fixed", the reference's 8 neighbours (the default), and "adaptive", ACMH's adaptive
# checkerboard sampling.
PROPAGATION = {"fixed": 0, "adaptive": 1}


def check_propagation(kind: str) -> int:
    """The argument rule of gpm_set_propagation, checked before any call into the library; returns the C-ABI's kind."""
    if kind not in PROPAGATION:
        raise ValueError("propagation must be one of %s (got %r)" % (sorted(PROPAGATION), kind))
    return PROPAGATION[kind]


# View selection (DESIGN.md §17): "off", each hypothesis scored by the combination rule of the parameters (the default), and
# "joint", ACMH's multi-hypothesis joint view selection, for the NCC cost on grey images.  JVS_DEFAULTS are ACMH's parameters.
VIEW_SELECTION = {"off": 0, "joint": 1}
JVS_DEFAULTS = {"tau_init": 0.8, "alpha": 90.0, "tau_bad": 1.2, "n_good": 3, "n_bad": 3, "beta": 0.3, "w_keep": 0.2}


def view_sel(kind: str = "off", **params) -> GpmViewSel:
    """gpm_view_sel of `kind` with JVS_DEFAULTS overridden by `params`, every argument checked before any call into the
    library by the rules of gpm_set_view_selection."""
    if kind not in VIEW_SELECTION:
        raise ValueError("view selection must be one of %s (got %r)" % (sorted(VIEW_SELECTION), kind))
    unknown = sorted(set(params) - set(JVS_DEFAULTS))
    if unknown:
        raise ValueError("unknown view-selection parameters %s (known: %s)" % (unknown, sorted(JVS_DEFAULTS)))
    p = dict(JVS_DEFAULTS, **params)
    if kind == "joint":
        for k in ("tau_init", "alpha", "tau_bad", "beta"):
            if not (isinstance(p[k], (int, float, np.floating, np.integer)) and np.isfinite(p[k]) and p[k] > 0):
                raise ValueError("%s must be finite and > 0 (got %r)" % (k, p[k]))
        if not (isinstance(p["w_keep"], (int, float, np.floating, np.integer)) and np.isfinite(p["w_keep"]) and p["w_keep"] >= 0):
            raise ValueError("w_keep must be finite and >= 0 (got %r)" % (p["w_keep"],))
        for k, hi in (("n_good", 8), ("n_bad", 9)):
            if int(p[k]) != p[k] or not 1 <= p[k] <= hi:
                raise ValueError("%s must be an integer in 1..%d (got %r)" % (k, hi, p[k]))
    return GpmViewSel(VIEW_SELECTION[kind], float(p["tau_init"]), float(p["alpha"]), float(p["tau_bad"]), int(p["n_good"]),
                      int(p["n_bad"]), float(p["beta"]), float(p["w_keep"]))


# Planar prior (DESIGN.md §18): ACMP's scales, sigma_d = (depthMax - depthMin) / 64 (None here: it depends on the scene)
# and sigma_n = 5 degrees; step and support_cost of the prior's construction.  The weight per photometric cost is the best of
# the grid measured with tools/acs_bench.py --prior (§18's table).
PRIOR_DEFAULTS = {"weight": {"pm": 2.0, "ncc": 0.1}, "depth_sigma": None, "normal_sigma_deg": 5.0, "step": 5, "support_cost": 0.5}


def check_prior(weight: float, depth_sigma: float, normal_sigma_deg: float):
    """The argument rules of gpm_set_prior, checked before any call into the library."""
    if not (isinstance(weight, (int, float, np.floating, np.integer)) and np.isfinite(weight) and weight >= 0):
        raise ValueError("weight must be finite and >= 0 (got %r)" % (weight,))
    if not (isinstance(depth_sigma, (int, float, np.floating, np.integer)) and np.isfinite(depth_sigma) and depth_sigma > 0):
        raise ValueError("depth_sigma must be finite and > 0 (got %r)" % (depth_sigma,))
    if not (isinstance(normal_sigma_deg, (int, float, np.floating, np.integer)) and 0 < normal_sigma_deg <= 90):
        raise ValueError("normal_sigma_deg must be in (0, 90] (got %r)" % (normal_sigma_deg,))


def check_prior_build(step: int, support_cost: float):
    """The argument rules of gpm_build_planar_prior, checked before any call into the library."""
    if int(step) != step or not 1 <= step <= 64:
        raise ValueError("step must be an integer in 1..64 (got %r)" % (step,))
    if support_cost != support_cost:
        raise ValueError("support_cost must not be NaN")


def check_modes(photometric: str, view_selection: str, channels: int = 1, planar_prior: Optional[dict] = None):
    """The mode rules the batch drivers refuse a combination by (include/gipuma_b200.h, mode compatibility), checked before
    any call into the library: "joint" view selection needs the NCC cost, and both need grey images (channels 1); a planar
    prior (a dict, see prior_opts) needs grey images and excludes joint view selection."""
    if view_selection == "joint" and photometric != "ncc":
        raise ValueError("view_selection='joint' is built for the NCC cost (photometric='ncc')")
    if photometric == "ncc" and channels == 4:
        raise ValueError("the NCC photometric cost supports grey images only")
    if planar_prior is not None and (channels == 4 or view_selection == "joint"):
        raise ValueError("the planar prior supports grey images without joint view selection")


def prior_opts(planar_prior: Optional[dict], params, n_jobs: int, photometric: str = "pm"):
    """gpm_prior_opts of the batch drivers' prior stage from `planar_prior` (None: no stage; a dict overriding
    PRIOR_DEFAULTS, plus "iterations", the sweeps with the prior, 2 by default), every argument checked before any call into
    the library.  depth_sigma None: (depthMax - depthMin) / 64 of `params`.  Returns (opts or None, the per-job info array)."""
    if planar_prior is None:
        return None, None
    unknown = sorted(set(planar_prior) - set(PRIOR_DEFAULTS) - {"iterations"})
    if unknown:
        raise ValueError("unknown planar-prior parameters %s (known: %s)" % (unknown, sorted(PRIOR_DEFAULTS) + ["iterations"]))
    p = dict(PRIOR_DEFAULTS, iterations=2)
    p.update(planar_prior)
    if isinstance(p["weight"], dict):
        p["weight"] = p["weight"][photometric]
    if p["depth_sigma"] is None:
        p["depth_sigma"] = (float(params.depthMax) - float(params.depthMin)) / 64.0 if params is not None else 1.0
    check_prior(p["weight"], p["depth_sigma"], p["normal_sigma_deg"])
    check_prior_build(p["step"], p["support_cost"])
    if int(p["iterations"]) != p["iterations"] or p["iterations"] < 0:
        raise ValueError("iterations must be an integer >= 0 (got %r)" % (p["iterations"],))
    info = (GpmPriorInfo * max(n_jobs, 1))()
    return GpmPriorOpts(float(p["weight"]), float(p["depth_sigma"]), float(p["normal_sigma_deg"]), int(p["step"]),
                        float(p["support_cost"]), int(p["iterations"]), info), info


def _prior_info(info, k):
    return [{"support": i.support, "triangles": i.triangles, "with_prior": i.with_prior} for i in info[:k]] if info else None


MAXCOST = 1000.0


def check_prior_bound(params, photometric: str, geo_weight: float, geo_max_err: float, prior_weight: float):
    """The planar prior's bound (DESIGN.md §18), in the library's float32 order, checked before any call into the library:
    the largest valid cost of `params` (PM: ns at the initialisation window times the largest dissimilarity; NCC: 2) plus
    geo_weight * geo_max_err plus the prior's weight must stay below MAXCOST."""
    f = np.float32
    if prior_weight <= 0:
        return
    nside = int(params.box_hsize) // 2 + 1
    top = f(2.0) if photometric == "ncc" else \
        f(nside * nside) * ((f(1.0) - f(params.alpha)) * f(params.tau_color) + f(params.alpha) * f(params.tau_gradient))
    if not (top + f(geo_weight) * f(geo_max_err)) + f(prior_weight) < f(MAXCOST):
        raise ValueError("with the prior's weight %r a valid cost could reach MAXCOST (largest cost %g, geometric term %g)" %
                         (prior_weight, top, f(geo_weight) * f(geo_max_err)))


# Joint bilateral upsampling of planes between pyramid levels (DESIGN.md §19): candidates within `radius` coarse pixels,
# a Gaussian spatial weight of sigma_space fine pixels and a Cauchy range weight of sigma_range grey levels.  MS_LEVELS and
# MS_GEO_ITERATIONS are multiscale_pass's default pyramid depth and sweeps per level.  These are the settings measured with
# tools/ms_bench.py (§19's table), not the result of a search.
JBU_DEFAULTS = {"radius": 2, "sigma_space": 2.0, "sigma_range": 10.0}
MS_LEVELS, MS_GEO_ITERATIONS = 3, 2
# multiscale_pass's geometric prior stage (DESIGN.md §20) picks support points by costs that include the geometric term:
# its default support_cost, the better of the two values measured with tools/ms_bench.py --prior.
MS_GEO_PRIOR_SUPPORT_COST = PRIOR_DEFAULTS["support_cost"]


# multiscale_pass's detail restorer (ACMM's, as the project's rule; DESIGN.md §21): detection threshold per photometric cost,
# in that cost's units; photo_iterations None: params.iterations; iterations: sweeps after the restore.  The thresholds are
# the best of the few measured with tools/ms_bench.py --restore (§21's table), not the result of a search.
RESTORE_DEFAULTS = {"threshold": {"pm": 0.5, "ncc": 0.05}, "photo_iterations": None, "iterations": 2}


def restore_opts(detail_restorer: Optional[dict], params, n_jobs: int, photometric: str = "pm"):
    """gpm_ms_restore_opts from `detail_restorer` (None: no restorer; a dict overriding RESTORE_DEFAULTS), every argument
    checked before any call into the library.  Returns (opts or None, the per-job restored-count array)."""
    if detail_restorer is None:
        return None, None
    unknown = sorted(set(detail_restorer) - set(RESTORE_DEFAULTS))
    if unknown:
        raise ValueError("unknown detail-restorer parameters %s (known: %s)" % (unknown, sorted(RESTORE_DEFAULTS)))
    r = dict(RESTORE_DEFAULTS)
    r.update(detail_restorer)
    if isinstance(r["threshold"], dict):
        if photometric not in r["threshold"]:
            raise ValueError("the threshold dict has no entry for photometric=%r (got %r)" % (photometric, r["threshold"]))
        r["threshold"] = r["threshold"][photometric]
    if r["photo_iterations"] is None:
        r["photo_iterations"] = int(params.iterations)
    t = r["threshold"]
    # the library receives the threshold as float32: it must be finite after that rounding
    t32 = np.float32(np.inf)
    if not isinstance(t, bool) and isinstance(t, (int, float, np.floating, np.integer)):
        with np.errstate(over="ignore"):
            try:
                t32 = np.float32(t)
            except OverflowError:
                pass
    if not np.isfinite(t32):
        raise ValueError("threshold must be a number that is finite in float32 (got %r)" % (t,))
    for k, lo in (("photo_iterations", 1), ("iterations", 0)):
        v = r[k]
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= 2 ** 31 - 1:
            raise ValueError("%s must be an integer in %d..%d (got %r)" % (k, lo, 2 ** 31 - 1, v))
    restored = (C.c_int * max(n_jobs, 1))()
    return GpmMsRestoreOpts(int(r["photo_iterations"]), float(t32), int(r["iterations"]), restored), restored


# Refinement (DESIGN.md §23): "gipuma", the reference's steps of shrinking random offsets (the default), and "acmh", ACMH's
# five hypotheses from random and perturbed depths and normals.  REFINE_DEFAULTS["perturbation"] is ACMH's published
# perturbation (0.02), not a value tuned on this project's scenes.
REFINEMENT = {"gipuma": 0, "acmh": 1}
REFINE_DEFAULTS = {"perturbation": 0.02}


def check_refinement(kind: str, perturbation: float):
    """The argument rules of gpm_set_refinement, checked before any call into the library: a known kind and a perturbation
    that is, as the float32 the library receives, finite and in (0, 1).  Returns (the C-ABI's kind, that float32)."""
    if not isinstance(kind, str) or kind not in REFINEMENT:
        raise ValueError("refinement must be one of %s (got %r)" % (sorted(REFINEMENT), kind))
    e = np.float32(np.nan)
    if not isinstance(perturbation, bool) and isinstance(perturbation, (int, float, np.floating, np.integer)):
        with np.errstate(over="ignore"):
            e = np.float32(perturbation)
    if not (np.isfinite(e) and 0 < e < 1):
        raise ValueError("perturbation must be a number in (0, 1) in float32 (got %r)" % (perturbation,))
    return REFINEMENT[kind], e


def refine_opts(refinement) -> Optional[GpmRefineOpts]:
    """gpm_refine_opts of the batch drivers from `refinement`: None (Gipuma's, the library's NULL), a kind ("gipuma" or
    "acmh") with REFINE_DEFAULTS, or a dict with "kind" and optionally "perturbation"; checked before any call into the
    library."""
    if refinement is None:
        return None
    if isinstance(refinement, str):
        refinement = {"kind": refinement}
    if not isinstance(refinement, dict):
        raise ValueError("refinement must be None, a kind or a dict (got %r)" % (refinement,))
    unknown = sorted(set(refinement) - {"kind", "perturbation"})
    if unknown or "kind" not in refinement:
        raise ValueError("refinement dict needs 'kind' and may have 'perturbation' (got %r)" % (sorted(refinement),))
    kind, e = check_refinement(refinement["kind"], refinement.get("perturbation", REFINE_DEFAULTS["perturbation"]))
    return GpmRefineOpts(kind, float(e))


def jbu_params(radius: int = JBU_DEFAULTS["radius"], sigma_space: float = JBU_DEFAULTS["sigma_space"],
               sigma_range: float = JBU_DEFAULTS["sigma_range"]) -> GpmJbuParams:
    """gpm_jbu_params, every argument checked before any call into the library by the rules of gpm_upsample_planes."""
    if isinstance(radius, bool) or int(radius) != radius or not 0 <= radius <= 4:
        raise ValueError("radius must be an integer in 0..4 (got %r)" % (radius,))
    for name, v in (("sigma_space", sigma_space), ("sigma_range", sigma_range)):
        if not (isinstance(v, (int, float, np.floating, np.integer)) and np.isfinite(v) and v > 0):
            raise ValueError("%s must be finite and > 0 (got %r)" % (name, v))
    return GpmJbuParams(int(radius), float(sigma_space), float(sigma_range))


def level_size(n: int, level: int) -> int:
    """Pixels along one side at pyramid level `level` of a side of n pixels: each level halves it, rounding up."""
    for _ in range(level):
        n = (n + 1) // 2
    return n


def downsample(img, device: int = 0):
    """One pyramid level on the GPU (gpm_downsample): [H, W] grey or [H, W, 4] RGBA float32, numpy or a CUDA tensor, to
    [(H + 1) // 2, (W + 1) // 2(, 4)] of the same kind.  Coarse pixel (xc, yc) is the separable [1, 2, 1] / 4 average
    around fine pixel (2 xc, 2 yc) with replicated borders, which is what K / 2 describes (DESIGN.md §19)."""
    shape = tuple(img.shape)
    if len(shape) not in (2, 3) or (len(shape) == 3 and shape[2] != 4):
        raise ValueError("images must be [H, W] or [H, W, 4]")
    if shape[0] < 1 or shape[1] < 1:
        raise ValueError("images must have at least one pixel")
    H, W = shape[:2]
    ch = 1 if len(shape) == 2 else 4
    out_shape = ((H + 1) // 2, (W + 1) // 2) + shape[2:]
    if isinstance(img, np.ndarray):
        img = np.ascontiguousarray(img, dtype=np.float32)
        out = np.empty(out_shape, np.float32)
    else:
        import torch
        out = torch.empty(out_shape, dtype=torch.float32, device=img.device)
        device = img.device.index if img.is_cuda else device
    src, dev = _ptr(img)
    dst, _ = _ptr(out)
    lib = load_library()
    if lib.gpm_downsample(int(device), src, 0, W, H, ch, dst, dev) != 0:
        raise GipumaError("gpm_downsample: %s" % lib.gpm_last_error().decode())
    return out


def pyramid(img, levels: int, device: int = 0):
    """[img, downsample(img), ...]: `levels` images, full size first."""
    if isinstance(levels, bool) or int(levels) != levels or levels < 1:
        raise ValueError("levels must be an integer >= 1 (got %r)" % (levels,))
    out = [img]
    for _ in range(int(levels) - 1):
        out.append(downsample(out[-1], device))
    return out


def job_opts(photometric: str = "pm", ncc_min_std: float = NCC_MIN_STD, propagation: str = "fixed") -> GpmJobOpts:
    """gpm_job_opts of the batch drivers, every argument checked before any call into the library."""
    kind = check_photometric(photometric, ncc_min_std)
    prop = check_propagation(propagation)
    return GpmJobOpts(kind, float(ncc_min_std) if photometric == "ncc" else 0.0, prop)


class Context:
    """One gpm_ctx: a reference view with its source views on one GPU."""

    def __init__(self, width: int, height: int, max_views: int, device: int = 0):
        self.lib = load_library()
        self.W, self.H, self.max_views, self.device = width, height, max_views, device
        h = C.c_void_p()
        self._check(self.lib.gpm_create(C.byref(h), device, width, height, max_views))
        self.h = h

    def _check(self, rc: int):
        if rc != 0:
            raise GipumaError("gipuma_b200 error %d: %s" % (rc, self.lib.gpm_last_error().decode()))

    def close(self):
        if getattr(self, "h", None):
            self.lib.gpm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- inputs ---------------------------------------------------------------------------------
    def set_params(self, params):
        p = pack_params(params)
        self._check(self.lib.gpm_set_params(self.h, C.byref(p)))

    @staticmethod
    def _is_color(img) -> bool:
        """[H, W, 4] float images take the reference's -color_processing (float4) path; [H, W] the gray one."""
        shape = getattr(img, "shape", ())
        return len(shape) == 3 and shape[-1] == 4

    def set_reference(self, img, cam, pitch_bytes: int = 0):
        img = _image(img)
        ptr, dev = _ptr(img)
        g = cam if isinstance(cam, GpmCamera) else pack_camera(cam)
        fn = self.lib.gpm_set_reference_color if self._is_color(img) else self.lib.gpm_set_reference
        self._check(fn(self.h, ptr, pitch_bytes, dev, C.byref(g)))

    def set_view(self, v: int, img, cam, pitch_bytes: int = 0):
        img = _image(img)
        ptr, dev = _ptr(img)
        g = cam if isinstance(cam, GpmCamera) else pack_camera(cam)
        fn = self.lib.gpm_set_view_color if self._is_color(img) else self.lib.gpm_set_view
        self._check(fn(self.h, v, ptr, pitch_bytes, dev, C.byref(g)))

    def set_num_views(self, n: int):
        self._check(self.lib.gpm_set_num_views(self.h, n))

    def set_view_depth(self, v: int, depth, pitch_bytes: int = 0):
        """Depth map [H, W] of source view v (numpy or torch, host or device), along that view's own optical axis as
        finalize() writes it (0 = no depth): what the geometric-consistency term reads (DESIGN.md §14)."""
        if not 0 <= v < self.max_views:
            raise ValueError("view index %d outside 0..%d" % (v, self.max_views - 1))
        if tuple(depth.shape) != (self.H, self.W):
            raise ValueError("depth map must be [%d, %d], got %s" % (self.H, self.W, tuple(depth.shape)))
        depth = _image(depth)
        ptr, dev = _ptr(depth)
        self._check(self.lib.gpm_set_view_depth(self.h, v, ptr, pitch_bytes, dev))

    def set_geometric(self, weight: float, max_err: float = GEO_MAX_ERR):
        """Geometric-consistency term of every view's cost: weight * min(reprojection error, max_err) (DESIGN.md §14);
        weight 0 turns it off."""
        check_geometric(weight, max_err)
        self._check(self.lib.gpm_set_geometric(self.h, float(weight), float(max_err)))

    def set_geo_mask(self, mask):
        """Per-pixel mask of the geometric term (DESIGN.md §21): [H, W] (numpy or torch, host or device; bool or uint8), nonzero
        where the term is off; None clears it.  While the term is on, a masked pixel's costs are exactly those with the term
        off.  Refused while the planar prior is on."""
        if mask is None:
            self._check(self.lib.gpm_set_geo_mask(self.h, None, 0, 0))
            return
        if tuple(mask.shape) != (self.H, self.W):
            raise ValueError("mask must be [%d, %d], got %s" % (self.H, self.W, tuple(mask.shape)))
        if isinstance(mask, np.ndarray):
            m = np.ascontiguousarray(mask != 0, dtype=np.uint8)
            self._check(self.lib.gpm_set_geo_mask(self.h, C.c_void_p(m.ctypes.data), 0, 0))
            return
        import torch
        m = (mask != 0).to(torch.uint8).contiguous()
        if m.is_cuda:
            torch.cuda.current_stream(m.device).synchronize()     # the context works on its own stream
        self._check(self.lib.gpm_set_geo_mask(self.h, C.c_void_p(m.data_ptr()), 0, 1 if m.is_cuda else 0))

    def set_photometric(self, kind: str = "pm", min_std: float = NCC_MIN_STD):
        """Photometric cost of every view (DESIGN.md §15): "pm", the reference's (the default), or "ncc", 1 - the
        support-weighted normalised cross-correlation, for grey images and the 8-neighbour sweep.  min_std (grey levels):
        a window whose weighted standard deviation is below it costs 2; ignored for "pm"."""
        k = check_photometric(kind, min_std)
        self._check(self.lib.gpm_set_photometric(self.h, k, float(min_std) if kind == "ncc" else 0.0))

    def set_propagation(self, kind: str = "fixed"):
        """Which plane each pixel is offered from each of its 8 directions (DESIGN.md §16): "fixed", the reference's
        neighbours at 1 and 5 px (the default), or "adaptive", the cheapest pixel of a larger region per direction (ACMH's
        adaptive checkerboard sampling).  8-neighbour sweep only; may be switched at any point of a run."""
        self._check(self.lib.gpm_set_propagation(self.h, check_propagation(kind)))

    def set_view_selection(self, kind: str = "off", **params):
        """Which source views score a pixel's hypotheses (DESIGN.md §17): "off", each hypothesis its own by the parameters'
        combination rule (the default), or "joint", ACMH's multi-hypothesis joint view selection, whose parameters
        (JVS_DEFAULTS) may be overridden by keyword.  "joint" needs the NCC cost (set_photometric("ncc")), grey images and
        the 8-neighbour sweep."""
        v = view_sel(kind, **params)
        self._check(self.lib.gpm_set_view_selection(self.h, C.byref(v)))

    def set_prior(self, weight: float, depth_sigma: float, normal_sigma_deg: float = PRIOR_DEFAULTS["normal_sigma_deg"]):
        """Planar prior term of every cost (DESIGN.md §18): weight * q / (1 + q) with q = (depth offset / depth_sigma)^2 +
        (1 - cos of the normal angle) / (1 - cos normal_sigma_deg), against the pixel's prior plane; weight 0 turns it
        off.  Needs a prior map (set_planar_prior or build_planar_prior), grey images and no joint view selection."""
        check_prior(weight, depth_sigma, normal_sigma_deg)
        self._check(self.lib.gpm_set_prior(self.h, float(weight), float(depth_sigma), float(normal_sigma_deg)))

    def set_planar_prior(self, planes):
        """Prior map [H, W, 4] (n.xyz, d per pixel; all-zero: no prior), numpy or torch, host or device."""
        if tuple(planes.shape) != (self.H, self.W, 4):
            raise ValueError("prior map must be [%d, %d, 4], got %s" % (self.H, self.W, tuple(planes.shape)))
        if isinstance(planes, np.ndarray):
            planes = np.ascontiguousarray(planes, dtype=np.float32)
        ptr, dev = _ptr(planes)
        self._check(self.lib.gpm_set_planar_prior(self.h, ptr, 0, dev))

    def planar_prior(self) -> np.ndarray:
        m = np.empty((self.H, self.W, 4), dtype=np.float32)
        self._check(self.lib.gpm_get_planar_prior(self.h, C.c_void_p(m.ctypes.data), 0))
        return m

    def build_planar_prior(self, step: int = PRIOR_DEFAULTS["step"], support_cost: float = PRIOR_DEFAULTS["support_cost"]) -> dict:
        """Prior map from the stored state: the cheapest pixel of each step x step cell whose cost < support_cost, the
        Delaunay triangulation of those pixels and each triangle's plane.  Returns the counts."""
        check_prior_build(step, support_cost)
        b, info = GpmPriorBuild(int(step), float(support_cost)), GpmPriorInfo()
        self._check(self.lib.gpm_build_planar_prior(self.h, C.byref(b), C.byref(info)))
        return {"support": info.support, "triangles": info.triangles, "with_prior": info.with_prior}

    def offer_prior(self):
        """Every pixel with a prior takes its prior plane where that plane costs strictly less than the stored one."""
        self._check(self.lib.gpm_offer_prior(self.h))

    def view_masks(self) -> np.ndarray:
        """[H, W] uint64: bit j set where the last joint-view-selection launch selected view j."""
        m = np.empty((self.H, self.W), dtype=np.uint64)
        self._check(self.lib.gpm_get_view_masks(self.h, C.c_void_p(m.ctypes.data)))
        return m

    def set_refinement(self, kind: str = "gipuma", perturbation: float = REFINE_DEFAULTS["perturbation"]):
        """How each pixel refines its plane (DESIGN.md §23): "gipuma", the reference's steps (the default), or "acmh", ACMH's
        five hypotheses (d_r, n), (d, n_r), (d_r, n_r), (d, n_t), (d_t, n) of random (r) and perturbed (t) depths and
        normals, perturbation in (0, 1).  Not with the fused sweep or the source-view shard."""
        k, e = check_refinement(kind, perturbation)
        self._check(self.lib.gpm_set_refinement(self.h, k, float(e)))

    def set_rng(self, seed: int, mode: int = GPM_RNG_REFERENCE):
        self._check(self.lib.gpm_set_rng(self.h, seed, mode))

    def set_option(self, name: str, value: int):
        self._check(self.lib.gpm_set_option(self.h, name.encode(), int(value)))

    def load_scene(self, scene, seed: int = 0xC0FFEE, rng_mode: int = GPM_RNG_REFERENCE, images=None):
        """Upload a gipuma_b200.scene.Scene (images may be overridden by a list of device tensors)."""
        imgs = scene.images if images is None else images
        self.set_params(scene.params)
        self.set_reference(np.ascontiguousarray(imgs[0]) if isinstance(imgs, np.ndarray) else imgs[0], scene.cameras[0])
        for v, idx in enumerate(scene.subset):
            im = np.ascontiguousarray(imgs[idx]) if isinstance(imgs, np.ndarray) else imgs[idx]
            self.set_view(v, im, scene.cameras[idx])
        self.set_num_views(len(scene.subset))
        self.set_rng(seed, rng_mode)

    # -- state ----------------------------------------------------------------------------------
    def set_state(self, norm4=None, cost=None):
        """Overwrite the raw planes [H,W,4] and/or costs [H,W] (numpy or torch, host or device)."""
        if isinstance(norm4, np.ndarray):
            norm4 = np.ascontiguousarray(norm4, dtype=np.float32)
        if isinstance(cost, np.ndarray):
            cost = np.ascontiguousarray(cost, dtype=np.float32)
        p4, d4 = _ptr(norm4)
        pc, dc = _ptr(cost)
        if norm4 is not None and cost is not None and d4 != dc:
            raise ValueError("norm4 and cost must both be host or both be device buffers")
        self._check(self.lib.gpm_set_state(self.h, p4, pc, max(d4, dc)))

    def get_state(self):
        n4 = np.empty((self.H, self.W, 4), dtype=np.float32)
        c = np.empty((self.H, self.W), dtype=np.float32)
        self._check(self.lib.gpm_get_state(self.h, C.c_void_p(n4.ctypes.data), C.c_void_p(c.ctypes.data), 0))
        return n4, c

    def get_state_into(self, norm4, cost):
        """Copy the state into caller buffers (numpy or torch, host or device)."""
        p4, d4 = _ptr(norm4)
        pc, dc = _ptr(cost)
        self._check(self.lib.gpm_get_state(self.h, p4, pc, max(d4, dc)))

    # -- compute --------------------------------------------------------------------------------
    def init(self):
        self._check(self.lib.gpm_init(self.h))

    def sweep(self, iterations: int):
        self._check(self.lib.gpm_sweep(self.h, iterations))

    def phase(self, colour: int, phase_mask: int):
        self._check(self.lib.gpm_phase(self.h, colour, phase_mask))

    def finalize(self):
        self._check(self.lib.gpm_finalize(self.h))

    def cost_eval(self, planes: np.ndarray) -> np.ndarray:
        pl = np.ascontiguousarray(planes, dtype=np.float32)
        out = np.empty((self.H, self.W), dtype=np.float32)
        self._check(self.lib.gpm_cost_eval(self.h, C.c_void_p(pl.ctypes.data), C.c_void_p(out.ctypes.data), 0))
        return out

    def upsample_planes(self, coarse, radius: int = JBU_DEFAULTS["radius"], sigma_space: float = JBU_DEFAULTS["sigma_space"],
                        sigma_range: float = JBU_DEFAULTS["sigma_range"]):
        """Joint bilateral upsampling (gpm_upsample_planes, DESIGN.md §19) of a coarse level's raw planes coarse
        [(H + 1) // 2, (W + 1) // 2, 4] (numpy, or a CUDA tensor) to this context's level, guided by its reference image,
        with its parameters' depth range and its reference camera.  Returns (planes [H, W, 4], depth [H, W]) of the input's
        kind; depth 0 where no coarse plane could be used.  The context's state is not touched."""
        jbu = jbu_params(radius, sigma_space, sigma_range)
        Hc, Wc = (self.H + 1) // 2, (self.W + 1) // 2
        if tuple(coarse.shape) != (Hc, Wc, 4):
            raise ValueError("coarse planes must be [%d, %d, 4] for a %dx%d context (got %s)" % (Hc, Wc, self.W, self.H, tuple(coarse.shape)))
        if isinstance(coarse, np.ndarray):
            coarse = np.ascontiguousarray(coarse, dtype=np.float32)
            planes, depth = np.empty((self.H, self.W, 4), np.float32), np.empty((self.H, self.W), np.float32)
        else:
            import torch
            planes = torch.empty((self.H, self.W, 4), dtype=torch.float32, device=coarse.device)
            depth = torch.empty((self.H, self.W), dtype=torch.float32, device=coarse.device)
        pc, dev = _ptr(coarse)
        self._check(self.lib.gpm_upsample_planes(self.h, pc, Wc, Hc, dev, C.byref(jbu), _ptr(planes)[0], _ptr(depth)[0]))
        return planes, depth

    def run(self) -> float:
        """init + params.iterations sweeps + finalize; returns the sweep time in ms (reference's timed span)."""
        ms = C.c_float(0)
        self._check(self.lib.gpm_run(self.h, C.byref(ms)))
        return float(ms.value)

    # -- source-view sharding (multi-GPU) -----------------------------------------------------------
    def init_planes(self):
        self._check(self.lib.gpm_init_planes(self.h))

    def shard_num_stages(self) -> int:
        n = self.lib.gpm_shard_num_stages(self.h)
        if n < 0:
            self._check(n)
        return n

    def shard_stage_floats(self, stage: int) -> int:
        n = self.lib.gpm_shard_stage_floats(self.h, stage)
        if n < 0:
            self._check(int(n))
        return int(n)

    def shard_stage(self, colour: int, stage: int, gathered_prev, world: int, xchg):
        """Accept of the previous stage (from `gathered_prev`, device tensor or None) + evaluation of `stage` into `xchg`."""
        gp = C.c_void_p(gathered_prev.data_ptr()) if gathered_prev is not None else None
        xp = C.c_void_p(xchg.data_ptr()) if xchg is not None else None
        self._check(self.lib.gpm_shard_stage(self.h, colour, stage, gp, world, xp))

    def shard_finish_init(self, gathered, world: int):
        self._check(self.lib.gpm_shard_finish_init(self.h, C.c_void_p(gathered.data_ptr()), world))

    def shard_comm_init(self, unique_id: Optional[bytes], rank: int, world: int):
        """ncclCommInitRank behind the C-ABI; `unique_id` = the 128 bytes of shard_unique_id() of the group's rank 0."""
        buf = C.create_string_buffer(unique_id, 128) if unique_id is not None else None
        self._check(self.lib.gpm_shard_comm_init(self.h, buf, rank, world))

    def shard_run(self) -> float:
        """runcuda() with sharded views (gpm_shard_run): returns the sweep time in ms."""
        ms = C.c_float(0)
        self._check(self.lib.gpm_shard_run(self.h, C.byref(ms)))
        return float(ms.value)

    def stats(self) -> dict:
        s = (C.c_ulonglong * 8)()
        self._check(self.lib.gpm_get_stats(self.h, s))
        return {"launches": s[0], "hypotheses": s[1], "skipped": s[2], "pruned": s[3],
                "pairs": s[4], "pairs_full": s[5], "collectives": s[6]}

    def measure_fetch_peak(self) -> float:
        """Texture-unit ceiling on this GPU, in 1e9 filtered R32F fetches per second (gpm_measure_fetch_peak)."""
        v = C.c_double(0)
        self._check(self.lib.gpm_measure_fetch_peak(self.h, C.byref(v)))
        return float(v.value)

    def reset_stats(self):
        self._check(self.lib.gpm_reset_stats(self.h))

    @property
    def stream(self) -> int:
        return int(self.lib.gpm_stream(self.h) or 0)


def shard_unique_id() -> bytes:
    """128-byte NCCL unique id for gpm_shard_comm_init (call on the shard group's rank 0, broadcast to the others)."""
    lib = load_library()
    buf = C.create_string_buffer(128)
    rc = lib.gpm_shard_unique_id(buf)
    if rc != 0:
        raise GipumaError("gpm_shard_unique_id: %s" % lib.gpm_last_error().decode())
    return buf.raw


class LineState:
    """Outputs in the reference's LineState layout (linestate.h:8-24)."""

    def __init__(self, norm4: np.ndarray, c: np.ndarray):
        self.norm4 = norm4          # [rows, cols, 4]: world normal xyz, depth (0 where cost == MAXCOST)
        self.c = c                  # [rows, cols]


def runcuda(scene, seed: int = 0xC0FFEE, rng_mode: int = GPM_RNG_REFERENCE, device: int = 0,
            options: Optional[dict] = None):
    """The reference's `runcuda(GlobalState&)` for a Scene: returns (LineState, sweep_ms, stats)."""
    with Context(scene.cols, scene.rows, max(1, len(scene.subset)), device) as ctx:
        for k, v in (options or {}).items():
            ctx.set_option(k, v)
        ctx.load_scene(scene, seed=seed, rng_mode=rng_mode)
        ms = ctx.run()
        n4, c = ctx.get_state()
        st = ctx.stats()
    return LineState(n4, c), ms, st


# ---- host-side rows of SURVEY.md §8f (no GPU needed) ---------------------------------------------------------------

def prepare_cameras(Ps, cam_scale: float = 1.0):
    """C++ restatement of getCameraParameters (cameraGeometryUtils.h:174-353): list of 3x4 projections -> GpmCamera[]."""
    lib = load_library()
    P = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float64) for p in Ps]).reshape(-1))
    out = (GpmCamera * len(Ps))()
    rc = lib.gpm_prepare_cameras(P.ctypes.data_as(C.POINTER(C.c_double)), len(Ps), float(cam_scale), out)
    if rc != 0:
        raise GipumaError("gpm_prepare_cameras failed: %d" % rc)
    return out


def select_views(cams, cols: int, rows: int, min_angle: float, max_angle: float, max_views: int):
    """Deterministic selectViews (main.cpp:430-499).  Returns (subset, (depth_min, depth_max))."""
    lib = load_library()
    sub = (C.c_int * max(1, len(cams)))()
    rng = (C.c_float * 2)()
    n = lib.gpm_select_views(cams, len(cams), cols, rows, min_angle, max_angle, max_views, sub, rng)
    if n < 0:
        raise GipumaError("gpm_select_views failed: %d" % n)
    return [sub[i] for i in range(n)], (rng[0], rng[1])


def _batch_desc(imgs, Ps, params, refs, devices, cam_scale, min_angle, max_angle, max_views, seed, out_dir, n4, cc):
    """gpm_batch_desc over contiguous float32 images [n, H, W(, 4)] and output arrays (or None).  Returns it with the arrays
    it points into, which must outlive the call."""
    n, H, W = imgs.shape[:3]
    ptrs = (C.c_void_p * n)(*[C.c_void_p(imgs[i].ctypes.data) for i in range(n)])
    P = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float64) for p in Ps]).reshape(-1))
    refs_a = (C.c_int * len(refs))(*[int(r) for r in refs])
    devs = (C.c_int * len(devices))(*[int(d) for d in devices])
    d = GpmBatchDesc()
    d.n_images, d.width, d.height = n, W, H
    d.images, d.pitch_bytes = ptrs, 0
    d.P, d.cam_scale = P.ctypes.data_as(C.POINTER(C.c_double)), float(cam_scale)
    d.params = pack_params(params)
    d.min_angle, d.max_angle, d.max_views = float(min_angle), float(max_angle), int(max_views)
    d.ref_indices, d.n_refs, d.devices, d.n_devices, d.seed = refs_a, len(refs), devs, len(devices), seed
    d.out_dir = out_dir.encode() if out_dir else None
    d.out_norm4 = n4.ctypes.data_as(C.POINTER(C.c_float)) if n4 is not None else None
    d.out_cost = cc.ctypes.data_as(C.POINTER(C.c_float)) if cc is not None else None
    return d, (imgs, ptrs, P, refs_a, devs, n4, cc)


def _job_stats(n_refs):
    """gpm_batch_stats with per-job arrays for n_refs jobs."""
    return GpmBatchStats(0, 0.0, (C.c_float * n_refs)(), (C.c_int * n_refs)(), (C.c_int * n_refs)())


def batch_run(images, Ps, params, refs, devices=(0,), cam_scale: float = 1.0, min_angle: float = 10.0, max_angle: float = 30.0,
              max_views: int = 9, seed: int = 0xC0FFEE, out_dir: Optional[str] = None, want_outputs: bool = True,
              photometric: str = "pm", ncc_min_std: float = NCC_MIN_STD, propagation: str = "fixed",
              view_selection: str = "off", jvs_params: Optional[dict] = None, planar_prior: Optional[dict] = None,
              refinement=None):
    """Reference-view batch in ONE process (gpm_batch_run_prior; gpm_batch_run_refine with a refinement): `images`
    [n, H, W] float32 (shared, page-locked once), `Ps` n 3x4 projections, `refs` the reference views to process, `devices` the CUDA ordinals to use (one worker thread each),
    `photometric` the cost, "pm" or "ncc" with min_std `ncc_min_std` (Context.set_photometric), `propagation` "fixed" or
    "adaptive" (Context.set_propagation), `view_selection` "off" or "joint" with `jvs_params` overriding JVS_DEFAULTS
    (Context.set_view_selection; "joint" needs photometric="ncc"), `planar_prior` None or a dict (prior_opts): a prior stage
    after the params.iterations sweeps of every job (DESIGN.md §18), whose counts come back per job in stats["prior"],
    `refinement` None (Gipuma's), "gipuma", "acmh" or a dict with "kind" and "perturbation" (refine_opts; DESIGN.md §23).
    Returns (norm4 [len(refs), H, W, 4] or None, cost or None, stats dict)."""
    opts = job_opts(photometric, ncc_min_std, propagation)
    ref_o = refine_opts(refinement)
    vsel = view_sel(view_selection, **(jvs_params or {}))
    check_modes(photometric, view_selection, 1, planar_prior)
    prior, pinfo = prior_opts(planar_prior, params, len(refs), photometric)
    lib = load_library()
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    n, H, W = imgs.shape
    n4 = np.empty((len(refs), H, W, 4), np.float32) if want_outputs else None
    cc = np.empty((len(refs), H, W), np.float32) if want_outputs else None
    d, _keep = _batch_desc(imgs, Ps, params, refs, devices, cam_scale, min_angle, max_angle, max_views, seed, out_dir, n4, cc)
    st = _job_stats(len(refs))
    args = (C.byref(d), C.byref(opts), C.byref(vsel), C.byref(prior) if prior else None)
    rc = lib.gpm_batch_run_refine(*args, C.byref(ref_o), C.byref(st)) if ref_o else lib.gpm_batch_run_prior(*args, C.byref(st))
    if rc != 0:
        raise GipumaError("gpm_batch_run failed (%d): %s" % (rc, lib.gpm_batch_last_error().decode()))
    k = len(refs)
    return n4, cc, {"jobs_done": st.jobs_done, "sweep_ms_total": st.sweep_ms_total, "sweep_ms": st.per_job_sweep_ms[:k],
                    "views": st.per_job_views[:k], "device": st.per_job_device[:k], "prior": _prior_info(pinfo, k)}


def geometric_pass(images, Ps, params, refs, geo_iterations: int = 2, weight: float = GEO_WEIGHT, max_err: float = GEO_MAX_ERR,
                   cam_scale: float = 1.0, min_angle: float = 10.0, max_angle: float = 30.0, max_views: int = 9,
                   seed: int = 0xC0FFEE, devices=(0,), out_dir: Optional[str] = None, photometric: str = "pm",
                   ncc_min_std: float = NCC_MIN_STD, propagation: str = "fixed", view_selection: str = "off",
                   jvs_params: Optional[dict] = None, planar_prior: Optional[dict] = None, refinement=None):
    """PatchMatch with a geometric-consistency second pass (DESIGN.md §14) for the reference views `refs`, run by the
    native two-pass batch driver (gpm_geo_batch_run) over the worker pool of `devices` (one worker thread and context each;
    a device may be listed more than once).

    Pass 1, for every reference view and every source view one of them selects: init, params.iterations photometric sweeps,
    finalize; the view setup is gpm_batch_run's.  Every worker finishes pass 1 before pass 2 starts.  Pass 2, per reference
    view: the selected source views' pass-1 depth maps are uploaded, the geometric term is turned on (weight, max_err), the
    pass-1 planes get their exact costs under the new cost (cost_eval), and geo_iterations sweeps and finalize follow.  So a
    run has params.iterations + geo_iterations iterations in all.  images: [n, H, W] grey or [n, H, W, 4] colour; the other
    arguments as batch_run; out_dir: None, or where <ref, 8 digits>/{disp,normals}.dmb of the pass-2 results are written;
    photometric / ncc_min_std: the photometric cost of both passes, as batch_run ("ncc": grey images only); propagation:
    the propagation mode of both passes, as batch_run; view_selection / jvs_params: the view selection of both passes, as
    batch_run (pass 2 starts over at t = 0); planar_prior: a prior stage in pass 1 only, as batch_run (info["prior"]: the
    counts per pass-1 view, in info["pass1_views"]' order); refinement: the refinement of both passes, as batch_run.
    Returns (norm4 [len(refs), H, W, 4], cost [len(refs), H, W], info) with norm4 as batch_run returns it, so fuse and
    evaluate_cloud take it unchanged; info: "pass1_views" (the views pass 1 ran, ascending), "pass1_sweep_s" (in that order)
    and "pass2_sweep_s" (per reference view): CUDA-event seconds of each view's sweep call on its context's stream;
    "views" (image indices of the source views each reference view selected), "device" (the device that ran its pass 2)."""
    check_geometric(weight, max_err)
    opts = job_opts(photometric, ncc_min_std, propagation)
    ref_o = refine_opts(refinement)
    if int(geo_iterations) != geo_iterations or geo_iterations < 0:
        raise ValueError("geo_iterations must be an integer >= 0")
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    if imgs.ndim not in (3, 4) or (imgs.ndim == 4 and imgs.shape[3] != 4):
        raise ValueError("images must be [n, H, W] or [n, H, W, 4]")
    vsel = view_sel(view_selection, **(jvs_params or {}))
    check_modes(photometric, view_selection, 4 if imgs.ndim == 4 else 1, planar_prior)
    n, H, W = imgs.shape[:3]
    prior, pinfo = prior_opts(planar_prior, params, n, photometric)
    if len(Ps) != n:
        raise ValueError("one projection matrix per image is needed (%d images, %d matrices)" % (n, len(Ps)))
    refs = [int(r) for r in refs]
    if not refs or any(r < 0 or r >= n for r in refs):
        raise ValueError("reference views must be image indices in 0..%d" % (n - 1))
    if not 1 <= max_views <= 64:
        raise ValueError("max_views must be 1..64")
    lib = load_library()
    k = len(refs)
    n4 = np.empty((k, H, W, 4), np.float32)
    cc = np.empty((k, H, W), np.float32)
    d, _keep = _batch_desc(imgs, Ps, params, refs, devices, cam_scale, min_angle, max_angle, max_views, seed, out_dir, n4, cc)
    g = GpmGeoBatchDesc(d, 1 if imgs.ndim == 3 else 4, int(geo_iterations), float(weight), float(max_err))
    p1_views, p1_ms = (C.c_int * n)(), (C.c_float * n)()
    ref_views = (C.c_int * (k * int(max_views)))()
    jobs = _job_stats(k)                                   # owns the per-job arrays st.batch points into
    st = GpmGeoBatchStats(jobs, 0, p1_views, p1_ms, ref_views)
    args = (C.byref(g), C.byref(opts), C.byref(vsel), C.byref(prior) if prior else None)
    rc = lib.gpm_geo_batch_run_refine(*args, C.byref(ref_o), C.byref(st)) if ref_o else lib.gpm_geo_batch_run_prior(*args, C.byref(st))
    if rc != 0:
        raise GipumaError("gpm_geo_batch_run failed (%d): %s" % (rc, lib.gpm_batch_last_error().decode()))
    m = st.n_pass1
    views = [[v for v in ref_views[j * max_views:(j + 1) * max_views] if v >= 0] for j in range(k)]
    info = {"pass1_views": p1_views[:m], "pass1_sweep_s": [t / 1e3 for t in p1_ms[:m]],
            "pass2_sweep_s": [t / 1e3 for t in st.batch.per_job_sweep_ms[:k]], "views": views,
            "device": st.batch.per_job_device[:k], "prior": _prior_info(pinfo, m)}
    return n4, cc, info


def multiscale_pass(images, Ps, params, refs, levels: int = MS_LEVELS, geo_iterations: int = MS_GEO_ITERATIONS,
                    weight: float = GEO_WEIGHT, max_err: float = GEO_MAX_ERR, jbu: Optional[dict] = None,
                    cam_scale: float = 1.0, min_angle: float = 10.0, max_angle: float = 30.0, max_views: int = 9,
                    seed: int = 0xC0FFEE, devices=(0,), out_dir: Optional[str] = None, photometric: str = "pm",
                    ncc_min_std: float = NCC_MIN_STD, propagation: str = "fixed", view_selection: str = "off",
                    jvs_params: Optional[dict] = None, planar_prior: Optional[dict] = None, geo_prior: Optional[dict] = None,
                    detail_restorer: Optional[dict] = None, refinement=None):
    """Coarse-to-fine multi-scale PatchMatch (ACMM; DESIGN.md §19) for the reference views `refs`, run by the native
    multi-level batch driver (gpm_ms_batch_run_restore) over the worker pool of `devices`.

    V, the views refined, is the transitive closure of the references' view selections; each view keeps its level-0
    selection and depth range at every level.  Level l has the images downsampled l times (downsample) and K / 2^l.  At the
    coarsest level every view of V runs init, params.iterations photometric sweeps and finalize, then geo_iterations sweeps
    with the geometric term against the other views' depth maps of that level.  Each finer level upsamples every view's
    planes (Context.upsample_planes with `jbu`, a dict overriding JBU_DEFAULTS) into planes and a depth map, and then
    refines (at level 0 only the references) with geo_iterations sweeps against those depth maps.  levels = 1 is
    geometric_pass over V.  The other arguments are geometric_pass's.
    The planar prior (ACMMP; DESIGN.md §20), each None (no stage) or a dict as batch_run's planar_prior (prior_opts):
    planar_prior runs a prior stage at the coarsest level after the photometric sweeps, so the coarsest geometric sweeps
    read depth maps made with it; geo_prior runs one at every level after the geo_iterations sweeps, with support points
    chosen by costs that include the geometric term (its support_cost defaults to MS_GEO_PRIOR_SUPPORT_COST, in those
    units).  Both need grey images and exclude joint view selection.
    detail_restorer (DESIGN.md §21), None (off) or a dict overriding RESTORE_DEFAULTS: at level 0 each reference also runs a
    photometric-only estimate (photo_iterations sweeps from init); after the geometric stage, pixels where the geometric
    stage's plane costs photometrically more than `threshold` above the estimate's take the estimate's plane and sweep
    without the geometric term (a per-pixel mask) for `iterations` more sweeps, while the rest keep it.
    refinement (DESIGN.md §23), as batch_run: the refinement of every sweep, at every level and in every stage.
    Returns (norm4 [len(refs), H, W, 4], cost [len(refs), H, W], info) with norm4 as batch_run returns it, so fuse and
    evaluate_cloud take it unchanged; info: "views" (V, ascending), "level_sweep_s" (CUDA-event sweep seconds summed over
    the views, per level, full size first, prior sweeps included), "level_upsample_s" (host seconds of the upsampling calls,
    per level), "sweep_s" (each reference's level-0 sweep seconds), "device" (the device that refined it at level 0);
    "prior": {"photometric": per image index, "geometric": per level, per image index} of the prior's counts (None for a
    stage not run; zeros where a view ran no stage), "level_build_ms" (host milliseconds of the prior builds, per level);
    "restored" (detail pixels per reference, None without the restorer)."""
    check_geometric(weight, max_err)
    opts = job_opts(photometric, ncc_min_std, propagation)
    ref_o = refine_opts(refinement)
    if isinstance(levels, bool) or int(levels) != levels or not 1 <= levels <= MS_MAX_LEVELS:
        raise ValueError("levels must be an integer in 1..%d (got %r)" % (MS_MAX_LEVELS, levels))
    if int(geo_iterations) != geo_iterations or geo_iterations < 0:
        raise ValueError("geo_iterations must be an integer >= 0")
    unknown = sorted(set(jbu or {}) - set(JBU_DEFAULTS))
    if unknown:
        raise ValueError("unknown JBU parameters %s (known: %s)" % (unknown, sorted(JBU_DEFAULTS)))
    jp = jbu_params(**dict(JBU_DEFAULTS, **(jbu or {})))
    imgs = np.ascontiguousarray(images, dtype=np.float32)
    if imgs.ndim not in (3, 4) or (imgs.ndim == 4 and imgs.shape[3] != 4):
        raise ValueError("images must be [n, H, W] or [n, H, W, 4]")
    vsel = view_sel(view_selection, **(jvs_params or {}))
    channels = 4 if imgs.ndim == 4 else 1
    check_modes(photometric, view_selection, channels)
    n, H, W = imgs.shape[:3]
    if min(level_size(W, levels - 1), level_size(H, levels - 1)) < 8:
        raise ValueError("the coarsest level of %d levels of %dx%d images is %dx%d, below 8x8" %
                         (levels, W, H, level_size(W, levels - 1), level_size(H, levels - 1)))
    stages = {}
    for name, spec, geo_w, level, n_info in (("photometric", planar_prior, 0.0, levels - 1, n),
                                              ("geometric", geo_prior, weight, 0, MS_MAX_LEVELS * n)):
        if spec is None:
            continue
        check_modes(photometric, view_selection, channels, spec)
        if name == "geometric":
            spec = dict({"support_cost": MS_GEO_PRIOR_SUPPORT_COST}, **spec)
        stages[name] = prior_opts(spec, params, n_info, photometric)
        check_prior_bound(params, photometric, geo_w, max_err, stages[name][0].weight)
        if max(level_size(W, level), level_size(H, level)) > 4097:
            raise ValueError("the %s prior stage builds the prior at level %d, %dx%d, wider or taller than 4097 pixels" %
                             (name, level, level_size(W, level), level_size(H, level)))
    if len(Ps) != n:
        raise ValueError("one projection matrix per image is needed (%d images, %d matrices)" % (n, len(Ps)))
    refs = [int(r) for r in refs]
    if not refs or any(r < 0 or r >= n for r in refs):
        raise ValueError("reference views must be image indices in 0..%d" % (n - 1))
    if not 1 <= max_views <= 64:
        raise ValueError("max_views must be 1..64")
    k = len(refs)
    ro, restored = restore_opts(detail_restorer, params, k, photometric)
    lib = load_library()
    n4 = np.empty((k, H, W, 4), np.float32)
    cc = np.empty((k, H, W), np.float32)
    d, _keep = _batch_desc(imgs, Ps, params, refs, devices, cam_scale, min_angle, max_angle, max_views, seed, out_dir, n4, cc)
    m = GpmMsBatchDesc(GpmGeoBatchDesc(d, 1 if imgs.ndim == 3 else 4, int(geo_iterations), float(weight), float(max_err)),
                       int(levels), jp)
    views = (C.c_int * n)()
    jobs = _job_stats(k)                                   # owns the per-job arrays st.batch points into
    st = GpmMsBatchStats(jobs, 0, views)
    po = GpmMsPriorOpts(*[C.pointer(stages[s][0]) if s in stages else None for s in ("photometric", "geometric")])
    args = (C.byref(m), C.byref(opts), C.byref(vsel), C.byref(po), C.byref(ro) if ro else None)
    rc = lib.gpm_ms_batch_run_refine(*args, C.byref(ref_o), C.byref(st)) if ref_o else lib.gpm_ms_batch_run_restore(*args, C.byref(st))
    if rc != 0:
        raise GipumaError("gpm_ms_batch_run failed (%d): %s" % (rc, lib.gpm_batch_last_error().decode()))
    info = {"views": views[:st.n_views], "level_sweep_s": [t / 1e3 for t in st.level_sweep_ms[:levels]],
            "level_upsample_s": [t / 1e3 for t in st.level_upsample_ms[:levels]],
            "sweep_s": [t / 1e3 for t in st.batch.per_job_sweep_ms[:k]], "device": st.batch.per_job_device[:k],
            "level_build_ms": list(po.level_build_ms[:levels]), "restored": restored[:k] if ro else None}
    pinfo = {s: stages[s][1] if s in stages else None for s in ("photometric", "geometric")}
    info["prior"] = {"photometric": _prior_info(pinfo["photometric"], n),
                     "geometric": [_prior_info(pinfo["geometric"][l * n:(l + 1) * n], n) for l in range(levels)]
                     if pinfo["geometric"] else None}
    return n4, cc, info


def write_dmb(path: str, data: np.ndarray):
    a = np.ascontiguousarray(data, dtype=np.float32)
    ch = 1 if a.ndim == 2 else a.shape[2]
    rc = load_library().gpm_write_dmb(path.encode(), a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0], a.shape[1], ch)
    if rc != 0:
        raise GipumaError("gpm_write_dmb failed")


def read_dmb(path: str) -> np.ndarray:
    lib = load_library()
    r, c, ch = C.c_int(), C.c_int(), C.c_int()
    if lib.gpm_read_dmb(path.encode(), None, 0, C.byref(r), C.byref(c), C.byref(ch)) != 0:
        raise GipumaError("gpm_read_dmb: cannot read %s" % path)
    out = np.empty((r.value, c.value, ch.value), dtype=np.float32)
    if lib.gpm_read_dmb(path.encode(), out.ctypes.data_as(C.POINTER(C.c_float)), out.size, C.byref(r), C.byref(c), C.byref(ch)) != 0:
        raise GipumaError("gpm_read_dmb: short file %s" % path)
    return out[..., 0] if ch.value == 1 else out


def write_result_dmb(depth_path: str, normal_path: str, norm4: np.ndarray):
    a = np.ascontiguousarray(norm4, dtype=np.float32)
    rc = load_library().gpm_write_result_dmb(depth_path.encode(), normal_path.encode(), a.ctypes.data_as(C.POINTER(C.c_float)),
                                             a.shape[0], a.shape[1])
    if rc != 0:
        raise GipumaError("gpm_write_result_dmb failed")


# ---- depth-map fusion (gpm_fuse; DESIGN.md §12, §22) -----------------------------------------------------------------

FUSE_RULES = {"disparity": 0, "reprojection": 1}                 # GPM_FUSE_DISPARITY, GPM_FUSE_REPROJECTION
# The reprojection rule's thresholds: 2 pixels of reprojection error in the reference view and 1 % of relative depth, the
# values COLMAP-style fusion is usually run with (measured against the disparity rule in DESIGN.md §22).
FUSE_REPROJ_DEFAULTS = {"reproj_px": 2.0, "depth_rel": 0.01}


def _fuse_rule(rule, reproj_px, depth_rel) -> GpmFuseRule:
    """The gpm_fuse_rule of fuse's arguments; ValueError for what gpm_fuse_with_rule would refuse."""
    if rule not in FUSE_RULES:
        raise ValueError("rule must be one of %s, not %r" % (sorted(FUSE_RULES), rule))
    if rule == "disparity":
        if reproj_px is not None or depth_rel is not None:
            raise ValueError("reproj_px and depth_rel apply to rule='reprojection' only")
        return GpmFuseRule(FUSE_RULES[rule], 0.0, 0.0)
    t = dict(FUSE_REPROJ_DEFAULTS)
    for k, v in (("reproj_px", reproj_px), ("depth_rel", depth_rel)):
        if v is not None:
            t[k] = v
        f = C.c_float(float(t[k])).value                            # the float the C-ABI receives
        if not (np.isfinite(f) and f > 0):
            raise ValueError("%s must be finite and > 0, not %r" % (k, t[k]))
    return GpmFuseRule(FUSE_RULES[rule], t["reproj_px"], t["depth_rel"])


def fuse_cameras(Ps, cam_scale: float = 1.0):
    """The fusion's per-view cameras (gpm_fuse_cameras): un-rebased world frame, K scaled by cam_scale."""
    lib = load_library()
    P = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float64) for p in Ps]).reshape(-1))
    out = (GpmFuseCamera * len(Ps))()
    if lib.gpm_fuse_cameras(P.ctypes.data_as(C.POINTER(C.c_double)), len(Ps), float(cam_scale), out) != 0:
        raise GipumaError("gpm_fuse_cameras: bad projection matrix or cam_scale")
    return out


def fuse(norm4, Ps, depth_min: float, depth_max: float, disp_thresh: float = 0.1, normal_thresh: float = 30.0,
         num_consistent: int = 3, images=None, cam_scale: float = 1.0, device: int = 0, rule: str = "disparity",
         reproj_px: float = None, depth_rel: float = None):
    """Fuse N views' world-frame outputs into one point cloud on the GPU (gpm_fuse_with_rule).

    norm4: [N, H, W, 4] float32 (world normal xyz + depth, 0 = invalid; what batch_run returns), numpy or torch (host or
    CUDA); Ps: the N 3x4 projection matrices of those views (as passed to batch_run); images: None, [N, H, W] grey or
    [N, H, W, 4] RGBA float in [0, 255], in the same memory as norm4.  The defaults of the thresholds are the reference's
    DTU script's (scripts/dtu_fast.sh:23-26).  rule: "disparity" (the default: |f_j 0.54 / z - f_j 0.54 / d_j| <
    disp_thresh, a threshold tied to DTU's scale) or "reprojection" (the scale-free rule of DESIGN.md §22: the target's
    point reprojects into the reference view within reproj_px pixels and depth_rel relative depth; disp_thresh is not read;
    None takes FUSE_REPROJ_DEFAULTS).  Returns (vertices: PLY_VERTEX array in (view, y, x) order, info dict with count,
    source [count, 2] int32 (view, y*W + x), used [N, H, W] uint8 masks, fuse_ms, upload_ms)."""
    fr = _fuse_rule(rule, reproj_px, depth_rel)
    lib = load_library()
    shape = tuple(norm4.shape)
    if len(shape) != 4 or shape[3] != 4 or len(Ps) != shape[0]:
        raise ValueError("norm4 must be [N, H, W, 4] with one projection matrix per view")
    n, H, W = shape[:3]
    p4, dev = _ptr(norm4)
    pi, devi, ch = None, dev, 0
    if images is not None:
        ishape = tuple(images.shape)
        if ishape[:3] != (n, H, W) or len(ishape) not in (3, 4) or (len(ishape) == 4 and ishape[3] != 4):
            raise ValueError("images must be [N, H, W] or [N, H, W, 4]")
        pi, devi = _ptr(images)
        ch = 1 if len(ishape) == 3 else 4
    if devi != dev:
        raise ValueError("norm4 and images must both be host or both be device buffers")
    depth = norm4[..., 3]
    lo, hi = float(np.float32(depth_min)), float(np.float32(depth_max))
    cap = int(((depth >= lo) & (depth <= hi)).sum())                       # bounds the vertex count
    verts = np.zeros(max(cap, 1), dtype=PLY_VERTEX)
    src = np.zeros((max(cap, 1), 2), dtype=np.int32)
    used = np.zeros((n, H, W), dtype=np.uint8)
    P = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float64) for p in Ps]).reshape(-1))
    d = GpmFuseDesc(n, W, H, p4, pi, ch, dev, P.ctypes.data_as(C.POINTER(C.c_double)), float(cam_scale), float(depth_min),
                    float(depth_max), float(disp_thresh), float(normal_thresh), int(num_consistent), int(device))
    r = GpmFuseResult(0, cap, verts.ctypes.data, src.ctypes.data, used.ctypes.data, 0.0, 0.0)
    if lib.gpm_fuse_with_rule(C.byref(d), C.byref(fr), C.byref(r)) != 0:
        raise GipumaError("gpm_fuse: %s" % lib.gpm_last_error().decode())
    k = int(r.count)
    return verts[:k], {"count": k, "source": src[:k], "used": used, "fuse_ms": float(r.fuse_ms), "upload_ms": float(r.upload_ms)}


def fuse_batch_dir(out_dir: str, refs, Ps, depth_min: float, depth_max: float, disp_thresh: float = 0.1,
                   normal_thresh: float = 30.0, num_consistent: int = 3, images=None, cam_scale: float = 1.0, device: int = 0,
                   rule: str = "disparity", reproj_px: float = None, depth_rel: float = None):
    """fuse() over what batch_run(out_dir=...) wrote: <out_dir>/<ref, 8 digits>/{disp,normals}.dmb for each of `refs`.
    Ps and images (None or [n_images, H, W(, 4)]) are the whole sets given to batch_run, indexed by image; the fused views
    are `refs`, in that order."""
    _fuse_rule(rule, reproj_px, depth_rel)
    maps = []
    for ref in refs:
        base = os.path.join(out_dir, "%08d" % int(ref))
        dep, nrm = read_dmb(os.path.join(base, "disp.dmb")), read_dmb(os.path.join(base, "normals.dmb"))
        if nrm.ndim != 3 or nrm.shape[2] != 3 or dep.shape != nrm.shape[:2]:
            raise GipumaError("%s: depth and normal maps do not match" % base)
        maps.append(np.concatenate([nrm, dep[..., None]], axis=2))
    imgs = None if images is None else np.ascontiguousarray(np.asarray(images)[list(refs)], dtype=np.float32)
    return fuse(np.ascontiguousarray(np.stack(maps), dtype=np.float32), [Ps[r] for r in refs], depth_min, depth_max,
                disp_thresh, normal_thresh, num_consistent, imgs, cam_scale, device, rule, reproj_px, depth_rel)


def write_ply(path: str, vertices):
    """Binary little-endian PLY with the header of storePlyFileBinary (gpm_write_ply)."""
    v = np.ascontiguousarray(vertices, dtype=PLY_VERTEX)
    if load_library().gpm_write_ply(path.encode(), v.ctypes.data if len(v) else None, len(v)) != 0:
        raise GipumaError("gpm_write_ply: cannot write %s" % path)


def read_ply(path: str) -> np.ndarray:
    """Vertices of a PLY written by write_ply (or by the reference's storePlyFileBinary) as a PLY_VERTEX array."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header\n")
    if not data.startswith(b"ply\n") or end < 0:
        raise GipumaError("%s: not a PLY file" % path)
    header = data[:end].decode("ascii").splitlines()
    props = [ln.split()[1:] for ln in header if ln.startswith("property")]
    want = [[t, nm] for nm, t in zip(PLY_VERTEX.names, ["float"] * 6 + ["uchar"] * 3)]
    if "format binary_little_endian 1.0" not in header or props != want:
        raise GipumaError("%s: not the x, y, z, nx, ny, nz, red, green, blue binary layout" % path)
    count = int(next(ln.split()[2] for ln in header if ln.startswith("element vertex")))
    body = data[end + len(b"end_header\n"):]
    if len(body) != count * PLY_VERTEX.itemsize:
        raise GipumaError("%s: %d bytes of vertex data for %d vertices" % (path, len(body), count))
    return np.frombuffer(body, dtype=PLY_VERTEX).copy()


# ---- point-cloud evaluation (gpm_nearest_dist; DESIGN.md §13) ----------------------------------------------------------

def _points(a, what):
    """(N, 3) float32 points: a numpy array, a torch tensor (host or CUDA), or a structured array with x, y, z fields
    (the vertices of fuse / read_ply).  Returns (array or tensor, is_device)."""
    if isinstance(a, np.ndarray) and a.dtype.names is not None:
        if not {"x", "y", "z"} <= set(a.dtype.names):
            raise ValueError("%s: a structured array needs x, y and z fields" % what)
        a = np.stack([a["x"], a["y"], a["z"]], axis=1).astype(np.float32)
    if len(tuple(a.shape)) != 2 or tuple(a.shape)[1] != 3:
        raise ValueError("%s must be an (N, 3) array of points, got shape %s" % (what, tuple(a.shape)))
    if isinstance(a, np.ndarray):
        if a.dtype != np.float32:
            raise TypeError("%s must be float32 (got %s)" % (what, a.dtype))
        return np.ascontiguousarray(a), False
    if hasattr(a, "is_cuda"):
        return a.contiguous(), bool(a.is_cuda)
    raise TypeError("%s: unsupported point type %r" % (what, type(a)))


def nearest_distance(query, data, max_dist: float):
    """Exact distance from every query point to its nearest data point, on the GPU (gpm_nearest_dist).

    query, data: (N, 3) float32 numpy arrays or torch tensors (both host or both CUDA), or structured vertex arrays as
    fuse / read_ply return.  Per query: the fp32 sqrt of min over the data of (dx*dx + dy*dy) + dz*dz, or +inf when that
    exceeds max_dist or the data are empty.  Returns (dist, info): dist float32 of length N, numpy for host inputs and a
    CUDA tensor on the inputs' device otherwise; info has upload_ms, build_ms, query_ms (CUDA events), cell_size, n_cells."""
    lib = load_library()
    q, qdev = _points(query, "query")
    b, bdev = _points(data, "data")
    if qdev != bdev:
        raise ValueError("query and data must both be host or both be CUDA buffers")
    device = 0
    if qdev:
        import torch
        if q.device != b.device:
            raise ValueError("query and data must be on the same device")
        device = q.device.index
        out = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
    else:
        out = np.empty(q.shape[0], dtype=np.float32)
    pq, _ = _ptr(q)
    pb, _ = _ptr(b)
    po, _ = _ptr(out)
    d = GpmNnDesc(int(q.shape[0]), int(b.shape[0]), pq, pb, int(qdev), int(device), float(max_dist))
    r = GpmNnResult(po, 0.0, 0.0, 0.0, 0.0, 0)
    if lib.gpm_nearest_dist(C.byref(d), C.byref(r)) != 0:
        raise GipumaError(lib.gpm_last_error().decode())
    return out, {"upload_ms": float(r.upload_ms), "build_ms": float(r.build_ms), "query_ms": float(r.query_ms),
                 "cell_size": float(r.cell_size), "n_cells": int(r.n_cells)}


def _sum_in_order(x):
    return float(np.cumsum(x)[-1]) if len(x) else 0.0


def cloud_scores(d_rec, d_gt, max_dist: float, taus=(0.5, 1.0, 2.0)) -> dict:
    """Accuracy, completeness and F-scores from the two directions' nearest distances (numpy, float64, sums in index order).

    d_rec: distance of every reconstructed point to the ground truth; d_gt: of every ground-truth point to the
    reconstruction (+inf beyond max_dist, as nearest_distance returns them).  As in the DTU protocol, distances >= max_dist
    are outliers: accuracy_mean / _median are taken over d_rec < max_dist, completeness_mean / _median over d_gt < max_dist,
    overall is their mean, and accuracy_outliers / completeness_outliers are the shares >= max_dist.  For each tau in taus:
    precision = share of d_rec < tau, recall = share of d_gt < tau, f_score = 2 P R / (P + R), 0 when P + R = 0 (lists in
    the order of taus).  A tau > max_dist is refused: such distances were capped.  Empty sets: means and medians over no
    distances are NaN, shares of an empty set are 0."""
    a = np.asarray(d_rec, dtype=np.float64).reshape(-1)
    g = np.asarray(d_gt, dtype=np.float64).reshape(-1)
    taus = [float(t) for t in taus]
    if not (np.isfinite(max_dist) and max_dist > 0):
        raise ValueError("max_dist must be finite and > 0")
    for t in taus:
        if not (t > 0 and t <= max_dist):
            raise ValueError("tau %g is outside (0, max_dist = %g]: distances beyond max_dist were capped" % (t, max_dist))

    def share(x, below):
        return float(np.count_nonzero(x < below)) / len(x) if len(x) else 0.0

    def mean_median(x):
        x = x[x < max_dist]
        return (_sum_in_order(x) / len(x), float(np.median(x))) if len(x) else (float("nan"), float("nan"))

    acc, acc_med = mean_median(a)
    comp, comp_med = mean_median(g)
    P = [share(a, t) for t in taus]
    R = [share(g, t) for t in taus]
    F = [2.0 * p * r / (p + r) if p + r > 0 else 0.0 for p, r in zip(P, R)]
    return {"accuracy_mean": acc, "accuracy_median": acc_med, "completeness_mean": comp, "completeness_median": comp_med,
            "overall": 0.5 * (acc + comp), "accuracy_outliers": 1.0 - share(a, max_dist) if len(a) else 0.0,
            "completeness_outliers": 1.0 - share(g, max_dist) if len(g) else 0.0,
            "taus": taus, "precision": P, "recall": R, "f_score": F, "n_rec": len(a), "n_gt": len(g)}


def evaluate_cloud(rec, gt, max_dist: float = 20.0, taus=(0.5, 1.0, 2.0)) -> dict:
    """Score a reconstructed cloud against ground truth: nearest_distance in both directions on the GPU, then cloud_scores.
    rec, gt: as nearest_distance takes them (for instance the vertices of fuse and scene.gt_points).  The result also holds
    the two directions' timings under "accuracy_timing" and "completeness_timing"."""
    d_rec, t_rec = nearest_distance(rec, gt, max_dist)
    d_gt, t_gt = nearest_distance(gt, rec, max_dist)
    host = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in (d_rec, d_gt)]
    out = cloud_scores(host[0], host[1], max_dist, taus)
    out["accuracy_timing"], out["completeness_timing"] = t_rec, t_gt
    return out


# ---- meshing (gpm_tsdf_integrate, gpm_mesh_extract; DESIGN.md §24) ------------------------------------------------------

# Truncation in voxels and minimum number of views per lattice point: measured with tools/mesh_bench.py on an H100 (DESIGN.md
# §24), the best mean F-score at 0.5 unit over the smooth scene's three PM runs at a voxel of 1 unit (the only part of the
# sweep measured so far).
MESH_DEFAULTS = {"trunc_voxels": 3.0, "min_weight": 3}
MESH_MAX_DIM = 2048                                               # GPM_MESH_MAX_DIM
GPM_FUSE_MAX_VIEWS = 256
_INT_MAX = 2 ** 31 - 1


def _f32(x) -> float:
    return C.c_float(float(x)).value                              # the float the C-ABI receives


def _check_box(origin, voxel, dims):
    """The box rules of gpm_tsdf_integrate and gpm_mesh_extract; returns (origin floats, voxel, (nx, ny, nz))."""
    o = [float(x) for x in origin]
    if len(o) != 3 or not all(np.isfinite(_f32(x)) for x in o):
        raise ValueError("origin must be 3 finite numbers")
    d = [int(x) for x in dims]
    if len(d) != 3 or not all(2 <= x <= MESH_MAX_DIM for x in d):
        raise ValueError("dims must be 3 integers in [2, %d], not %r" % (MESH_MAX_DIM, tuple(dims)))
    if d[0] * d[1] * d[2] > _INT_MAX:
        raise ValueError("dims %r: more than 2^31 - 1 voxels" % (tuple(d),))
    s = _f32(voxel)
    if not (np.isfinite(s) and s > 0):
        raise ValueError("voxel must be finite and > 0, not %r" % (voxel,))
    return o, float(voxel), tuple(d)


def _check_min_weight(min_weight) -> int:
    if int(min_weight) != min_weight or int(min_weight) < 1:
        raise ValueError("min_weight must be an integer >= 1, not %r" % (min_weight,))
    return int(min_weight)


def _tensor_device(a, device):
    """(is_device, device ordinal) of a buffer: a CUDA tensor's own device, which a given `device` must match."""
    if hasattr(a, "is_cuda") and a.is_cuda:
        if device is not None and int(device) != a.device.index:
            raise ValueError("device %d differs from the tensor's %s" % (device, a.device))
        return True, a.device.index
    return False, 0 if device is None else int(device)


def tsdf_integrate(depth, Ps, origin, voxel: float, dims, trunc: float, depth_min: float, depth_max: float,
                   cam_scale: float = 1.0, device: Optional[int] = None):
    """Integrate N depth maps into a truncated signed distance volume on the GPU (gpm_tsdf_integrate, DESIGN.md §24).

    depth: [N, H, W] float32 (the w of batch_run's norm4, or the disp.dmb files; 0 and depths outside [depth_min,
    depth_max] are invalid), numpy or torch (host or CUDA); Ps: the N 3x4 projection matrices of those views; origin: the
    box's corner; voxel: its edge; dims: (nx, ny, nz); trunc: the truncation in world units.  Returns (D, Wt, info): D
    float32 and Wt uint16 volumes [nz, ny, nx] (NaN where Wt = 0) in the inputs' kind of memory (numpy, or CUDA tensors
    on the input's device), info with upload_ms and integrate_ms (CUDA events)."""
    o, s, d = _check_box(origin, voxel, dims)
    t = _f32(trunc)
    if not (np.isfinite(t) and t > 0):
        raise ValueError("trunc must be finite and > 0, not %r" % (trunc,))
    lo, hi = _f32(depth_min), _f32(depth_max)
    if not (np.isfinite(lo) and np.isfinite(hi) and 0 <= lo < hi):
        raise ValueError("need finite 0 <= depth_min < depth_max")
    if not (cam_scale > 0):
        raise ValueError("cam_scale must be > 0")
    shape = tuple(depth.shape)
    if len(shape) != 3 or not 1 <= shape[0] <= GPM_FUSE_MAX_VIEWS or len(Ps) != shape[0]:
        raise ValueError("depth must be [N, H, W], 1 <= N <= %d, with one projection matrix per view" % GPM_FUSE_MAX_VIEWS)
    if isinstance(depth, np.ndarray) and (depth.dtype != np.float32 or not depth.flags["C_CONTIGUOUS"]):
        depth = np.ascontiguousarray(depth, dtype=np.float32)
    on_dev, dev = _tensor_device(depth, device)
    lib = load_library()
    n, H, W = shape
    pd, _ = _ptr(depth)
    if on_dev:
        import torch
        D = torch.empty((d[2], d[1], d[0]), dtype=torch.float32, device=depth.device)
        Wt = torch.empty((d[2], d[1], d[0]), dtype=torch.uint16, device=depth.device)
        pD, pW = D.data_ptr(), Wt.data_ptr()
    else:
        D = np.empty((d[2], d[1], d[0]), np.float32)
        Wt = np.empty((d[2], d[1], d[0]), np.uint16)
        pD, pW = D.ctypes.data, Wt.ctypes.data
    P = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.float64) for p in Ps]).reshape(-1))
    desc = GpmTsdfDesc(n, W, H, pd, int(on_dev), P.ctypes.data_as(C.POINTER(C.c_double)), float(cam_scale), float(depth_min),
                       float(depth_max), (C.c_float * 3)(*o), s, (C.c_int * 3)(*d), float(trunc), dev)
    r = GpmTsdfResult(pD, pW, 0.0, 0.0)
    if lib.gpm_tsdf_integrate(C.byref(desc), C.byref(r)) != 0:
        raise GipumaError(lib.gpm_last_error().decode())
    return D, Wt, {"upload_ms": float(r.upload_ms), "integrate_ms": float(r.integrate_ms)}


def extract_mesh(D, Wt, origin, voxel: float, min_weight: int, device: Optional[int] = None):
    """Marching tetrahedra on the lattice of voxel centres on the GPU (gpm_mesh_extract, DESIGN.md §24).

    D: float32 and Wt: uint16 volumes [nz, ny, nx], both numpy or both CUDA tensors (what tsdf_integrate returns); a
    point is valid when Wt >= min_weight and inside when D < 0.  Calls once to count and once to fill.  Returns
    (vertices [V, 3] float32, faces [F, 3] int32, counter-clockwise seen from outside, info with upload_ms and extract_ms
    of the filling call)."""
    shape = tuple(D.shape)
    if len(shape) != 3 or tuple(Wt.shape) != shape:
        raise ValueError("D and Wt must be [nz, ny, nx] volumes of one shape")
    o, s, d = _check_box(origin, voxel, shape[::-1])
    mw = _check_min_weight(min_weight)
    on_dev, dev = _tensor_device(D, device)
    if _tensor_device(Wt, None)[0] != on_dev:
        raise ValueError("D and Wt must both be host or both be CUDA buffers")
    if on_dev:
        import torch
        if D.dtype != torch.float32 or Wt.dtype != torch.uint16 or Wt.device != D.device:
            raise TypeError("D must be float32 and Wt uint16, on one device")
        # a non-contiguous view is copied on torch's stream; gpm_mesh_extract reads on its own stream, so the copy must be
        # finished before the call: copy first, then synchronise
        D, Wt = D.contiguous(), Wt.contiguous()
        torch.cuda.current_stream(D.device).synchronize()
        pD, pW = D.data_ptr(), Wt.data_ptr()
    else:
        if not isinstance(D, np.ndarray) or D.dtype != np.float32 or not isinstance(Wt, np.ndarray) or Wt.dtype != np.uint16:
            raise TypeError("D must be float32 and Wt uint16 numpy arrays (or CUDA tensors)")
        D, Wt = np.ascontiguousarray(D), np.ascontiguousarray(Wt)
        pD, pW = D.ctypes.data, Wt.ctypes.data
    lib = load_library()
    desc = GpmMeshDesc(pD, pW, int(on_dev), (C.c_float * 3)(*o), s, (C.c_int * 3)(*d), mw, dev)
    r = GpmMeshResult(0, 0, 0, 0, None, None, 0.0, 0.0)
    rc = lib.gpm_mesh_extract(C.byref(desc), C.byref(r))              # count
    if rc != 0 and not (rc == -1 and (r.n_vertices > 0 or r.n_faces > 0) and r.n_vertices <= _INT_MAX):
        raise GipumaError(lib.gpm_last_error().decode())
    verts = np.zeros((max(int(r.n_vertices), 1), 3), np.float32)
    faces = np.zeros((max(int(r.n_faces), 1), 3), np.int32)
    r = GpmMeshResult(0, 0, int(r.n_vertices), int(r.n_faces), verts.ctypes.data, faces.ctypes.data, 0.0, 0.0)
    if lib.gpm_mesh_extract(C.byref(desc), C.byref(r)) != 0:         # fill
        raise GipumaError(lib.gpm_last_error().decode())
    return verts[:r.n_vertices], faces[:r.n_faces], {"upload_ms": float(r.upload_ms), "extract_ms": float(r.extract_ms)}


def mesh(depth, Ps, origin, voxel: float, dims, depth_min: float, depth_max: float, trunc: Optional[float] = None,
         min_weight: Optional[int] = None, cam_scale: float = 1.0, device: Optional[int] = None):
    """tsdf_integrate then extract_mesh.  trunc (world units) defaults to MESH_DEFAULTS["trunc_voxels"] voxels and
    min_weight to MESH_DEFAULTS["min_weight"].  Returns (vertices, faces, info with both stages' times)."""
    trunc = MESH_DEFAULTS["trunc_voxels"] * float(voxel) if trunc is None else trunc
    min_weight = MESH_DEFAULTS["min_weight"] if min_weight is None else min_weight
    _check_min_weight(min_weight)
    D, Wt, i1 = tsdf_integrate(depth, Ps, origin, voxel, dims, trunc, depth_min, depth_max, cam_scale, device)
    v, f, i2 = extract_mesh(D, Wt, origin, voxel, min_weight)
    return v, f, {"upload_ms": i1["upload_ms"], "integrate_ms": i1["integrate_ms"], "extract_ms": i2["extract_ms"]}


def _mesh_arrays(vertices, faces):
    v = np.ascontiguousarray(vertices, dtype=np.float32)
    f = np.ascontiguousarray(faces, dtype=np.int32)
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
        raise ValueError("vertices must be [V, 3] and faces [F, 3]")
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("a face index is outside [0, %d)" % len(v))
    return v, f


def write_ply_mesh(path: str, vertices, faces):
    """Binary little-endian PLY: float x, y, z per vertex, `property list uchar int vertex_indices` per face."""
    v, f = _mesh_arrays(vertices, faces)
    if load_library().gpm_write_ply_mesh(path.encode(), v.ctypes.data if len(v) else None, len(v),
                                         f.ctypes.data if len(f) else None, len(f)) != 0:
        raise GipumaError("gpm_write_ply_mesh: cannot write %s" % path)


def read_ply_mesh(path: str):
    """(vertices [V, 3] float32, faces [F, 3] int32) of a PLY mesh in the layout write_ply_mesh writes."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header\n")
    if not data.startswith(b"ply\n") or end < 0:
        raise GipumaError("%s: not a PLY file" % path)
    header = data[:end].decode("ascii").splitlines()
    want = ["ply", "format binary_little_endian 1.0", None, "property float x", "property float y", "property float z",
            None, "property list uchar int vertex_indices"]
    if len(header) != len(want) or any(w is not None and h != w for h, w in zip(header, want)) or \
            not header[2].startswith("element vertex ") or not header[6].startswith("element face "):
        raise GipumaError("%s: not the x, y, z + vertex_indices binary layout" % path)
    nv, nf = int(header[2].split()[2]), int(header[6].split()[2])
    body = data[end + len(b"end_header\n"):]
    if len(body) != 12 * nv + 13 * nf:
        raise GipumaError("%s: %d bytes of data for %d vertices and %d faces" % (path, len(body), nv, nf))
    v = np.frombuffer(body, dtype="<f4", count=3 * nv).reshape(nv, 3).copy()
    rec = np.frombuffer(body, dtype=np.dtype([("n", "u1"), ("i", "<i4", 3)]), offset=12 * nv, count=nf)
    if (rec["n"] != 3).any():
        raise GipumaError("%s: a face is not a triangle" % path)
    return v, rec["i"].astype(np.int32)


def sample_mesh(vertices, faces, spacing: float) -> np.ndarray:
    """Points on a triangle mesh, deterministic, for scoring it with evaluate_cloud as DTU's surface track does: each face
    a, b, c with n = ceil(longest edge / spacing) (at least 1) gives the barycentric lattice points
    a + (i / n)(b - a) + (j / n)(c - a), i, j >= 0, i + j <= n, computed in float64.  Faces in order; within a face
    i-major.  Returns (M, 3) float32."""
    if not (np.isfinite(spacing) and spacing > 0):
        raise ValueError("spacing must be finite and > 0")
    v, f = _mesh_arrays(vertices, faces)
    if not len(f):
        return np.zeros((0, 3), np.float32)
    V = v.astype(np.float64)
    a, b, c = V[f[:, 0]], V[f[:, 1]], V[f[:, 2]]
    L = np.max(np.stack([np.linalg.norm(b - a, axis=1), np.linalg.norm(c - b, axis=1), np.linalg.norm(a - c, axis=1)]), axis=0)
    n = np.maximum(1, np.ceil(L / spacing)).astype(np.int64)
    per = (n + 1) * (n + 2) // 2
    start = np.concatenate([[0], np.cumsum(per)])
    out = np.empty((int(start[-1]), 3), np.float64)
    for m in np.unique(n):
        sel = np.nonzero(n == m)[0]
        i, j = np.array([(i, j) for i in range(m + 1) for j in range(m + 1 - i)], dtype=np.float64).T / m
        pts = a[sel, None, :] + i[None, :, None] * (b - a)[sel, None, :] + j[None, :, None] * (c - a)[sel, None, :]
        idx = start[sel][:, None] + np.arange(len(i))[None, :]
        out[idx.reshape(-1)] = pts.reshape(-1, 3)
    return out.astype(np.float32)
