"""ctypes binding of libnrw.so (include/nrw.h).  There is NO fallback: if the CUDA library is
missing or a call fails, an exception is raised."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NRW_LIB_PATH") or os.path.join(_HERE, "libnrw.so")     # NRW_LIB_PATH: A/B builds (tools/)

NRW_GEMM_TCGEN05 = 0
NRW_GEMM_SIMT = 1


class NrwError(RuntimeError):
    pass


class ParamInfo(C.Structure):
    _fields_ = [("name", C.c_char_p), ("rows", C.c_int), ("cols", C.c_int), ("offset", C.c_longlong),
                ("numel", C.c_longlong)]


class SamplerCfg(C.Structure):
    _fields_ = [("n_samples", C.c_int), ("n_importance", C.c_int), ("up_sample_steps", C.c_int),
                ("n_outside", C.c_int), ("s_val_base", C.c_int), ("boundary_samples", C.c_int),
                ("perturb", C.c_int)]


class RenderCfg(C.Structure):
    _fields_ = [("R", C.c_int), ("S", C.c_int), ("n_outside", C.c_int), ("cos_anneal_ratio", C.c_float),
                ("background_rgb", C.c_void_p), ("reserved0", C.c_int), ("trim_sphere", C.c_int)]


_IO_FIELDS = ["o", "d", "z_vals", "z_out", "sample_dist", "a_emb", "inv_s", "color", "color_sphere", "color_bg",
              "cdf", "gradients", "weights", "weights_sum", "inside_sphere", "depth", "normals", "gradient_error",
              "sv_sdf", "sv_rgb", "sv_bg_alpha", "sv_bg_rgb", "sv_z_feed", "sv_relax_sum"]


class RenderIO(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _IO_FIELDS]


_GRAD_FIELDS = ["g_color", "g_color_sphere", "g_color_bg", "g_cdf", "g_gradients", "g_weights", "g_weights_sum",
                "g_depth", "g_normals", "g_gradient_error", "grad_params", "grad_a_emb", "grad_inv_s"]


class RenderGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _GRAD_FIELDS]


class OctreeRef(C.Structure):
    _fields_ = [("octree", C.c_void_p), ("prefix", C.c_void_p), ("level", C.c_int), ("scene_origin", C.c_float * 3),
                ("scale", C.c_float)]


class RaygenCfg(C.Structure):
    _fields_ = [("height", C.c_int), ("width", C.c_int), ("img_downscale", C.c_int), ("fx", C.c_float), ("fy", C.c_float),
                ("cx", C.c_float), ("cy", C.c_float), ("c2w", C.c_float * 12), ("w2c_z", C.c_double * 4),
                ("image_id", C.c_int), ("with_label", C.c_int), ("sem_height", C.c_int), ("sem_width", C.c_int),
                ("use_voxel", C.c_int), ("near", C.c_float), ("far", C.c_float), ("voxel_size", C.c_float),
                ("sfm", OctreeRef), ("expanded", OctreeRef), ("depth_percent", C.c_double), ("seed", C.c_ulonglong)]


_lib = None


def lib():
    """Load libnrw.so once; raise loudly when it is absent (no CPU / eager fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise NrwError(f"{LIB_PATH} not found: build it with neuralrecon-w_b200/build.sh "
                       "(or __graft_entry__.build()); the nrw package has no non-CUDA path")
    L = C.CDLL(LIB_PATH)
    vp, ll, i32, f32 = C.c_void_p, C.c_longlong, C.c_int, C.c_float
    L.nrw_last_error.restype = C.c_char_p
    L.nrw_version.restype = i32
    L.nrw_param_count.restype = i32
    L.nrw_param_table.argtypes = [i32, i32, C.POINTER(ParamInfo)]
    L.nrw_param_total.restype = ll
    L.nrw_param_total.argtypes = [i32, i32]
    L.nrw_ctx_create.argtypes = [C.POINTER(vp), i32, i32, i32, i32]
    L.nrw_ctx_destroy.argtypes = [vp]
    L.nrw_ctx_set_backward_planes.argtypes = [vp, i32]
    L.nrw_ctx_set_backward_gate_planes.argtypes = [vp, i32]
    L.nrw_packed_bytes.restype = ll
    L.nrw_packed_bytes.argtypes = [vp]
    L.nrw_workspace_bytes.restype = ll
    L.nrw_workspace_bytes.argtypes = [vp, i32, i32, i32, i32, i32, i32]
    L.nrw_ctx_bind.argtypes = [vp, vp, ll, vp, ll, i32, i32, i32, i32, i32, i32, vp]
    L.nrw_pack_weights.argtypes = [vp, vp, vp]
    L.nrw_sdf_query.argtypes = [vp, vp, ll, vp, vp]
    L.nrw_neuconw_forward.argtypes = [vp, vp, vp, vp, ll, vp, vp, vp, vp]
    L.nrw_nerf_forward.argtypes = [vp, vp, vp, vp, ll, vp, vp, vp]
    L.nrw_sample.argtypes = [vp, C.POINTER(SamplerCfg), i32] + [vp] * 14
    L.nrw_samples_per_ray.argtypes = [C.POINTER(SamplerCfg), i32]
    L.nrw_upsample_round.argtypes = [i32, i32, i32, f32] + [vp] * 10
    L.nrw_boundary_samples.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp]
    L.nrw_render_forward.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(RenderIO), vp]
    L.nrw_render_backward.argtypes = [vp, C.POINTER(RenderCfg), C.POINTER(RenderIO), C.POINTER(RenderGrads), vp]
    L.nrw_composite_forward.argtypes = [C.POINTER(RenderCfg), C.POINTER(RenderIO)] + [vp] * 7
    L.nrw_composite_backward.argtypes = [C.POINTER(RenderCfg), C.POINTER(RenderIO), C.POINTER(RenderGrads)] + [vp] * 7
    L.nrw_octree_near_far.argtypes = [vp, vp, vp, i32, vp, vp, i32, C.POINTER(f32), f32, vp, vp, vp, vp, vp]
    L.nrw_octree_hits.argtypes = [vp, vp, vp, i32, vp, vp, i32, C.POINTER(f32), f32, vp, vp, vp, vp, vp]
    L.nrw_octree_build_scratch_bytes.restype = ll
    L.nrw_octree_build_scratch_bytes.argtypes = [i32, i32, i32]
    L.nrw_octree_build.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, i32, i32, vp, vp, vp]
    f64 = C.c_double
    L.nrw_grad_sumsq.argtypes = [vp, ll, vp, vp]
    L.nrw_adam_clip_step.argtypes = [vp, vp, vp, vp, ll, vp, f64, f64, f64, f64, f64, i32, vp]
    L.nrw_compact_scratch_bytes.restype = ll
    L.nrw_compact_scratch_bytes.argtypes = [ll]
    L.nrw_raycache_gather.argtypes = [vp, vp, ll, vp, i32, C.POINTER(i32), i32, vp, vp, vp, vp, vp, vp, vp]
    L.nrw_grid_points_dense.argtypes = [i32, C.POINTER(f32), C.POINTER(f32), ll, ll, vp, vp]
    L.nrw_grid_points_sparse.argtypes = [vp, ll, i32, f32, C.POINTER(f32), C.POINTER(f32), f32, ll, ll, vp, vp, vp]
    L.nrw_threshold_compact.argtypes = [vp, vp, ll, f32, vp, vp, vp, vp]
    L.nrw_mc_scratch_bytes.restype = ll
    L.nrw_mc_scratch_bytes.argtypes = [i32, i32, i32]
    L.nrw_mc_count.argtypes = [vp, i32, i32, i32, f32, vp, vp, vp, vp]
    L.nrw_mc_emit.argtypes = [vp, i32, i32, i32, f32, vp, vp, ll, ll, vp, vp, vp, vp]
    L.nrw_nn_index_bytes.restype = ll
    L.nrw_nn_index_bytes.argtypes = [ll]
    L.nrw_nn_build.argtypes = [vp, ll, vp, vp]
    L.nrw_nn_query_scratch_bytes.restype = ll
    L.nrw_nn_query_scratch_bytes.argtypes = [ll]
    L.nrw_nn_query.argtypes = [vp, ll, vp, ll, vp, vp, vp, vp]
    L.nrw_mesh_sample_scratch_bytes.restype = ll
    L.nrw_mesh_sample_scratch_bytes.argtypes = [ll]
    L.nrw_mesh_sample.argtypes = [vp, ll, vp, ll, ll, C.c_ulonglong, vp, vp, vp, vp, vp]
    L.nrw_raster_scratch_bytes.restype = ll
    L.nrw_raster_scratch_bytes.argtypes = [ll, ll, i32, i32]
    L.nrw_raster_depth.argtypes = [vp, ll, vp, ll, C.POINTER(f64), f64, f64, f64, f64, i32, i32, f64, f64, i32, vp, vp, vp, vp]
    L.nrw_reproject_scratch_bytes.restype = ll
    L.nrw_reproject_scratch_bytes.argtypes = [i32, i32]
    L.nrw_reproject_mark.argtypes = [vp, i32, i32, f64, f64, f64, f64, C.POINTER(f64), vp, ll, f64, vp, vp, vp, vp]
    L.nrw_raygen_capacity.restype = ll
    L.nrw_raygen_capacity.argtypes = [i32, i32, f64]
    L.nrw_raygen_scratch_bytes.restype = ll
    L.nrw_raygen_scratch_bytes.argtypes = [i32, i32, i32, ll, ll]
    L.nrw_raygen_image.argtypes = [C.POINTER(RaygenCfg), vp, vp, vp, vp, ll, vp, vp, ll, vp, vp, ll, vp, vp, vp, vp]
    L.nrw_depth_range_scratch_bytes.restype = ll
    L.nrw_depth_range_scratch_bytes.argtypes = [ll, i32]
    L.nrw_depth_range.argtypes = [vp, ll, vp, i32, f64, f64, vp, vp, vp, vp, vp]
    L.nrw_voxel_cast.argtypes = [vp, vp, C.POINTER(i32), i32, C.POINTER(f32), f32, C.POINTER(f64), f32, f32, f32, f32, i32, i32,
                                 vp, vp, vp, vp, vp]
    L.nrw_voxel_lookup.argtypes = [vp, vp, C.POINTER(i32), i32, vp, ll, vp, vp, vp]
    L.nrw_view_roi_count.argtypes = [vp, vp, i32, ll, C.POINTER(f32), f32, vp, vp]
    L.nrw_label_static_count.argtypes = [vp, ll, C.POINTER(i32), i32, vp, vp]
    L.nrw_gemm_test_scratch_bytes.restype = ll
    L.nrw_gemm_test_scratch_bytes.argtypes = [i32, i32, i32]
    L.nrw_gemm_test.argtypes = [i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, i32, vp, vp, vp]
    L.nrw_launch_count.restype = ll
    L.nrw_debug_gemm_profile.argtypes = [vp]
    L.nrw_gemm_timing.argtypes = [i32, C.POINTER(C.c_double)]
    _lib = L
    return L


EXPORTS = ["nrw_last_error", "nrw_version", "nrw_param_count", "nrw_param_table", "nrw_param_total",
           "nrw_ctx_create", "nrw_ctx_destroy", "nrw_packed_bytes", "nrw_workspace_bytes", "nrw_ctx_bind",
           "nrw_pack_weights", "nrw_sdf_query", "nrw_neuconw_forward", "nrw_nerf_forward", "nrw_sample",
           "nrw_samples_per_ray", "nrw_upsample_round", "nrw_render_forward", "nrw_render_backward",
           "nrw_composite_forward", "nrw_composite_backward", "nrw_octree_near_far", "nrw_octree_hits",
           "nrw_gemm_test_scratch_bytes", "nrw_gemm_test", "nrw_launch_count", "nrw_debug_gemm_profile",
           "nrw_gemm_timing", "nrw_ctx_set_backward_planes", "nrw_octree_build_scratch_bytes", "nrw_octree_build",
           "nrw_grad_sumsq", "nrw_adam_clip_step", "nrw_boundary_samples", "nrw_compact_scratch_bytes", "nrw_raycache_gather",
           "nrw_grid_points_dense", "nrw_grid_points_sparse", "nrw_threshold_compact", "nrw_ctx_set_backward_gate_planes",
           "nrw_mc_scratch_bytes", "nrw_mc_count", "nrw_mc_emit",
           "nrw_nn_index_bytes", "nrw_nn_build", "nrw_nn_query_scratch_bytes", "nrw_nn_query", "nrw_mesh_sample_scratch_bytes",
           "nrw_mesh_sample", "nrw_raster_scratch_bytes", "nrw_raster_depth", "nrw_reproject_scratch_bytes",
           "nrw_reproject_mark", "nrw_raygen_capacity", "nrw_raygen_scratch_bytes", "nrw_raygen_image",
           "nrw_depth_range_scratch_bytes", "nrw_depth_range", "nrw_voxel_cast", "nrw_voxel_lookup",
           "nrw_view_roi_count", "nrw_label_static_count"]


def check(status, what=""):
    if status != 0:
        msg = lib().nrw_last_error()
        raise NrwError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def param_table(n_vocab, n_a):
    L = lib()
    n = L.nrw_param_count()
    arr = (ParamInfo * n)()
    check(L.nrw_param_table(n_vocab, n_a, arr), "nrw_param_table")
    out = []
    for p in arr:
        if p.rows == 0 and p.cols == 0:
            shape = ()
        elif p.cols == 0:
            shape = (p.rows,)
        else:
            shape = (p.rows, p.cols)
        out.append((p.name.decode(), shape, int(p.offset), int(p.numel)))
    return out, int(L.nrw_param_total(n_vocab, n_a))
