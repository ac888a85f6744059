"""ctypes binding of ``libnphm_b200.so`` (C ABI declared in ``include/nphm_b200.h``).

PyTorch is used here only for device memory, streams and the caching allocator; the arithmetic of
the hot path happens inside the library.  There is NO fallback: if the library is missing or a call
fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import (POINTER, Structure, byref, c_char_p, c_double, c_float, c_int, c_longlong,
                    c_void_p)
from typing import Optional

import numpy as np
import torch

IMPL_AUTO, IMPL_SIMT, IMPL_TC, IMPL_TC_PRUNED = 0, 1, 2, 3
_IMPL_BY_NAME = {'auto': IMPL_AUTO, 'simt': IMPL_SIMT, 'tc': IMPL_TC, 'tc_pruned': IMPL_TC_PRUNED}

# NPHM_B200_LIB: developer override to load another build of the library (A/B runs of kernel variants); default = the in-tree build
_LIB_PATH = os.environ.get('NPHM_B200_LIB') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libnphm_b200.so')
_lib = None

# every symbol include/nphm_b200.h declares (tests check that the library exports all of them)
EXPORTED_SYMBOLS = (
    'nphm_last_error', 'nphm_abi_version', 'nphm_device_info',
    'nphm_ensemble_create', 'nphm_ensemble_destroy', 'nphm_ensemble_set_prune_threshold', 'nphm_ensemble_load_weights',
    'nphm_ensemble_query', 'nphm_ensemble_query_grid', 'nphm_ensemble_get_logits_host',
    'nphm_mlp_create', 'nphm_mlp_destroy', 'nphm_mlp_load_weights', 'nphm_mlp_query',
    'nphm_mlp_query_layers', 'nphm_mlp_jacobian', 'nphm_mlp_backward_inputs', 'nphm_mlp_inverse_jacobian', 'nphm_adam_step',
    'nphm_mc_workspace_bytes', 'nphm_mc_count', 'nphm_mc_emit', 'nphm_marching_cubes_host',
    'nphm_fit_workspace_bytes', 'nphm_fit_identity_step', 'nphm_fit_surface_grad', 'nphm_fit_apply_gradient',
    'nphm_fit_batch_workspace_bytes', 'nphm_fit_identity_step_batched', 'nphm_fit_surface_grad_batched',
    'nphm_fit_apply_gradient_batched',
    'nphm_fit_identity_step_quirk', 'nphm_fit_surface_grad_quirk', 'nphm_fit_identity_step_batched_quirk',
    'nphm_fit_surface_grad_batched_quirk', 'nphm_ensemble_backward_inputs_quirk',
    'nphm_ensemble_backward_inputs', 'nphm_ensemble_anchors',
    'nphm_broyden_workspace_bytes', 'nphm_mlp_broyden_search', 'nphm_broyden_compact_workspace_bytes',
    'nphm_mlp_broyden_search_compact', 'nphm_nearest_neighbors',
    'nphm_mlp_train_workspace_bytes', 'nphm_mlp_train_forward', 'nphm_mlp_train_backward',
    'nphm_mlp_sdfgrad_workspace_bytes', 'nphm_mlp_sdfgrad_forward', 'nphm_mlp_sdfgrad_backward',
    'nphm_mlp_fit_workspace_bytes', 'nphm_mlp_fit_surface_grad', 'nphm_mlp_fit_surface_grad_batched',
    'nphm_ensemble_sdfgrad_workspace_bytes', 'nphm_ensemble_sdfgrad_forward', 'nphm_ensemble_sdfgrad_backward',
    'nphm_render_workspace_bytes', 'nphm_render_depth_normals',
    'nphm_band_slab_workspace_bytes', 'nphm_band_slab_begin', 'nphm_band_slab_corners', 'nphm_band_slab_gather',
    'nphm_band_slab_scatter', 'nphm_band_slab_classify', 'nphm_band_slab_grow', 'nphm_band_slab_fill', 'nphm_band_slab_block_states',
    'nphm_band_slab_export', 'nphm_band_slab_import',
    'nphm_band_heads_workspace_bytes', 'nphm_band_heads_begin', 'nphm_band_heads_corners', 'nphm_band_heads_classify',
    'nphm_band_heads_grow', 'nphm_band_heads_gather', 'nphm_band_heads_scatter', 'nphm_band_heads_fill',
    'nphm_band_heads_block_states', 'nphm_mc_heads_workspace_bytes', 'nphm_mc_heads_count', 'nphm_mc_heads_emit',
    'nphm_band_sparse_workspace_bytes', 'nphm_band_sparse_pool_sizes', 'nphm_band_sparse_begin', 'nphm_band_sparse_corners',
    'nphm_band_sparse_classify', 'nphm_band_sparse_grow', 'nphm_band_sparse_gather', 'nphm_band_sparse_scatter',
    'nphm_band_sparse_fill', 'nphm_band_sparse_block_states', 'nphm_band_sparse_export', 'nphm_band_sparse_import',
    'nphm_band_sparse_volume', 'nphm_band_sparse_mc_workspace_bytes', 'nphm_band_sparse_mc_count', 'nphm_band_sparse_mc_emit',
    'nphm_band_sparse_heads_workspace_bytes', 'nphm_band_sparse_heads_begin', 'nphm_band_sparse_heads_corners',
    'nphm_band_sparse_heads_classify', 'nphm_band_sparse_heads_grow', 'nphm_band_sparse_heads_gather',
    'nphm_band_sparse_heads_scatter', 'nphm_band_sparse_heads_fill', 'nphm_band_sparse_heads_block_states',
    'nphm_band_sparse_heads_mc_workspace_bytes', 'nphm_band_sparse_heads_mc_count', 'nphm_band_sparse_heads_mc_emit',
    'nphm_face_cdf_workspace_bytes', 'nphm_face_cdf', 'nphm_sample_faces', 'nphm_vertex_normals_workspace_bytes',
    'nphm_vertex_normals', 'nphm_interpolate_barycentric', 'nphm_transfer_correspondences',
    'nphm_trace_workspace_bytes', 'nphm_trace_begin', 'nphm_trace_compact', 'nphm_trace_counts', 'nphm_trace_gather',
    'nphm_trace_advance', 'nphm_trace_points', 'nphm_trace_finish',
    'nphm_pose_apply', 'nphm_pose_grad', 'nphm_pose_adam',
    'nphm_register_prepare', 'nphm_register_search',
)


class NativeError(RuntimeError):
    pass


# kernels of this library launched per call (ncu launch lists under profiles/); bench.py counts its launches with these
MC_LAUNCHES = 3                      # classify rows, scan rows, emit rows


def dense_grid_tiles(res: int, first: int, count: int) -> int:
    """Tiles of a dense tensor-core query of grid points [first, first + count) of the res^3 grid, as
    tc_ensemble_launch lays them out: 8 x 4 x 4 blocks for whole 8-plane groups, 1 x 16 x 8 blocks otherwise, linear
    128-point tiles where blocks would add more than 3 % tiles."""
    rr = res * res
    tbx, tby, tbz = (8, 4, 4) if first % rr == 0 and count % (8 * rr) == 0 else (1, 16, 8)
    px0, px1 = first // rr, (first + count - 1) // rr
    blocked = ((px1 - px0 + tbx) // tbx) * (-(-res // tby)) * (-(-res // tbz))
    linear = -(-count // 128)
    return blocked if blocked * 100 <= linear * 103 else linear


def launches_per_grid_query(impl='auto', n_members=40, res=256, first=0, count=None) -> int:
    """Kernels of one grid query over points [first, first + count) (default: the whole grid) of the res^3 grid: grid
    axes, anchors and folded constants, then
      'simt': the ensemble kernel;
      'tc_pruned', and 'auto' / 'tc' with NPHM_ENS_ABSORB=0: records, layer-2 slabs, tile member masks, the ensemble
        kernel;
      'auto' / 'tc' (absorption on: member by member): records, layer-2 slabs, member bounds over the grid, tile member
        masks, member bounds per sub-box, and per chunk of at most 2^17 tiles (2^24 rows) a member pass and the ensemble
        kernel per member and the finalize."""
    if impl == 'simt':
        return 4
    if impl == 'tc_pruned' or os.environ.get('NPHM_ENS_ABSORB', '1')[:1] == '0':
        return 3 + 4
    count = res ** 3 - first if count is None else count
    chunks = -(-dense_grid_tiles(res, first, count) // (1 << 17))
    return 3 + 5 + chunks * (2 * n_members + 1)


class EnsembleConfig(Structure):
    _fields_ = [('n_loc', c_int), ('n_symm_pairs', c_int), ('lat_dim_glob', c_int), ('lat_dim_loc', c_int),
                ('hidden_dim', c_int), ('n_layers', c_int), ('pos_mlp_dim', c_int)]


class MlpConfig(Structure):
    _fields_ = [('lat_dim', c_int), ('hidden_dim', c_int), ('n_layers', c_int), ('out_dim', c_int)]


class McParams(Structure):
    _fields_ = [('nx', c_int), ('ny', c_int), ('nz', c_int), ('x_global0', c_int), ('ghost_lo', c_int),
                ('negate', c_int), ('iso', c_double)]


class BandPool(Structure):
    _fields_ = [('vals', c_void_p), ('marks', c_void_p), ('blocks', c_void_p), ('list', c_void_p), ('chunk_cnt', c_void_p),
                ('chunk_off', c_void_p), ('slots', c_longlong), ('marks_bytes', c_longlong), ('list_len', c_longlong),
                ('n_chunks', c_longlong)]


class TraceParams(Structure):
    _fields_ = [('n_heads', c_int), ('n_rays', c_longlong), ('box_min', c_double * 3), ('box_max', c_double * 3),
                ('scale', c_double), ('znear', c_double), ('zfar', c_double), ('step_factor', c_float), ('min_step', c_float),
                ('hit_eps', c_float), ('max_steps', c_int)]


class RegisterParams(Structure):
    _fields_ = [('res', c_int), ('mini', c_float * 3), ('h', c_float * 3), ('n_obs', c_int), ('n_use', c_int), ('n_hyp', c_int),
                ('n_iter', c_int), ('fit_scale', c_int), ('tau0', c_double), ('tau1', c_double), ('damping', c_double)]


class FitParams(Structure):
    _fields_ = [('lambda_surface', c_float), ('lambda_reg_global', c_float), ('lambda_reg_loc', c_float),
                ('lambda_reg_unobserved', c_float), ('lambda_symm_dist', c_float), ('clamp', c_float),
                ('lr', c_float), ('step', c_int)]


def stack_supported(n_hidden_layers: int, hidden: int, cond_dim: int, out_dim: int = 1) -> bool:
    """Configurations ``nphm_mlp_create`` / ``build_stack`` (csrc/api.cu) accept: 2 to 10 hidden layers, a condition of at
    least one column, ``hidden > cond_dim + 3`` and 1 to 8 outputs; anything else takes the composite PyTorch path."""
    return 2 <= n_hidden_layers <= 10 and cond_dim >= 1 and hidden > cond_dim + 3 and 1 <= out_dim <= 8


def hidden_width(module, n_lin: int) -> int:
    """Hidden width of a DeepSDF-style stack: the input width of its LAST linear layer (``lin0`` is narrowed to
    ``hidden - d_in`` when the skip connection sits at layer 1, i.e. for 2 or 3 hidden layers)."""
    return getattr(module, 'lin%d' % (n_lin - 1)).in_features


def impl_code(impl) -> int:
    if isinstance(impl, str):
        return _IMPL_BY_NAME[impl]
    return int(impl)


def default_impl() -> int:
    """Kernel selection for the drop-in modules; override with NPHM_B200_IMPL=auto|simt|tc."""
    return _IMPL_BY_NAME[os.environ.get('NPHM_B200_IMPL', 'auto')]


def lib() -> ctypes.CDLL:
    """Load the native library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise NativeError('%s is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                          '(or `make -C nphm_b200/csrc`). The fused CUDA path has no fallback.' % _LIB_PATH)
    L = ctypes.CDLL(_LIB_PATH)
    L.nphm_last_error.restype = c_char_p
    L.nphm_abi_version.restype = c_int
    L.nphm_device_info.argtypes = [POINTER(c_int)] * 3
    L.nphm_ensemble_create.argtypes = [POINTER(EnsembleConfig), POINTER(c_void_p)]
    L.nphm_ensemble_destroy.argtypes = [c_void_p]
    L.nphm_ensemble_destroy.restype = None
    L.nphm_ensemble_set_prune_threshold.argtypes = [c_void_p, c_float]
    L.nphm_ensemble_load_weights.argtypes = [c_void_p, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p),
                                             POINTER(c_void_p), c_void_p, c_void_p]
    L.nphm_ensemble_query.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_longlong, c_void_p,
                                      c_void_p, c_int, c_void_p]
    L.nphm_ensemble_query_grid.argtypes = [c_void_p, c_void_p, POINTER(c_double), POINTER(c_double), c_int,
                                           c_longlong, c_longlong, c_longlong, c_void_p, c_void_p, c_int, c_void_p]
    L.nphm_ensemble_get_logits_host.argtypes = [c_void_p, c_void_p, POINTER(c_double), POINTER(c_double), c_int,
                                                c_longlong, c_void_p, c_int]
    L.nphm_mlp_create.argtypes = [POINTER(MlpConfig), POINTER(c_void_p)]
    L.nphm_mlp_destroy.argtypes = [c_void_p]
    L.nphm_mlp_destroy.restype = None
    L.nphm_mlp_load_weights.argtypes = [c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_void_p]
    L.nphm_mlp_query.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_int, c_void_p]
    L.nphm_mlp_query_layers.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p]
    L.nphm_mlp_jacobian.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_mlp_backward_inputs.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_mc_workspace_bytes.argtypes = [POINTER(McParams)]
    L.nphm_mc_workspace_bytes.restype = c_longlong
    L.nphm_mc_count.argtypes = [c_void_p, POINTER(McParams), c_void_p, POINTER(c_longlong), POINTER(c_longlong),
                                c_void_p]
    L.nphm_mc_emit.argtypes = [c_void_p, POINTER(McParams), c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_marching_cubes_host.argtypes = [c_void_p, c_int, c_int, c_int, c_double, c_int, c_void_p, c_void_p,
                                           POINTER(c_longlong), POINTER(c_longlong)]
    L.nphm_fit_workspace_bytes.argtypes = [c_void_p, c_longlong]
    L.nphm_fit_workspace_bytes.restype = c_longlong
    L.nphm_fit_identity_step.argtypes = [c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p,
                                         POINTER(FitParams), c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_fit_surface_grad.argtypes = [c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_float, c_void_p, c_void_p,
                                        c_void_p, c_void_p, c_void_p]
    L.nphm_ensemble_anchors.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p]
    L.nphm_ensemble_backward_inputs.argtypes = [c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_void_p]
    L.nphm_fit_apply_gradient.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, POINTER(FitParams), c_void_p, c_void_p,
                                          c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.nphm_fit_batch_workspace_bytes.argtypes = [c_void_p, c_int, c_longlong]
    L.nphm_fit_batch_workspace_bytes.restype = c_longlong
    L.nphm_fit_identity_step_batched.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p,
                                                 POINTER(FitParams), c_int, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_fit_surface_grad_batched.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_float, c_void_p,
                                                c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_fit_apply_gradient_batched.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, POINTER(FitParams), c_void_p,
                                                  c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    L.nphm_fit_identity_step_quirk.argtypes = [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p,
                                               POINTER(FitParams), c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_fit_surface_grad_quirk.argtypes = [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_float, c_void_p,
                                              c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_ensemble_backward_inputs_quirk.argtypes = [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p,
                                                      c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_fit_identity_step_batched_quirk.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p,
                                                       c_void_p, c_void_p, POINTER(FitParams), c_int, c_void_p, c_void_p, c_void_p,
                                                       c_longlong, c_void_p]
    L.nphm_fit_surface_grad_batched_quirk.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_float,
                                                      c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_adam_step.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_float, c_int, c_void_p]
    L.nphm_mlp_inverse_jacobian.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_broyden_workspace_bytes.argtypes = [c_longlong]
    L.nphm_broyden_workspace_bytes.restype = c_longlong
    L.nphm_mlp_broyden_search.argtypes = [c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_int,
                                          c_float, c_float, c_float, c_void_p, c_void_p, POINTER(c_int), c_void_p,
                                          c_void_p]
    L.nphm_broyden_compact_workspace_bytes.argtypes = [c_int, c_longlong]
    L.nphm_broyden_compact_workspace_bytes.restype = c_longlong
    L.nphm_mlp_broyden_search_compact.argtypes = L.nphm_mlp_broyden_search.argtypes
    L.nphm_nearest_neighbors.argtypes = [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_mlp_train_workspace_bytes.argtypes = [c_void_p, c_int, c_longlong, c_int]
    L.nphm_mlp_train_workspace_bytes.restype = c_longlong
    L.nphm_mlp_train_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_longlong, c_void_p, c_void_p,
                                         c_void_p]
    L.nphm_mlp_train_backward.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_longlong, POINTER(c_void_p),
                                          POINTER(c_void_p), c_void_p, c_void_p, c_void_p]
    L.nphm_mlp_sdfgrad_workspace_bytes.argtypes = [c_void_p, c_int, c_longlong]
    L.nphm_mlp_sdfgrad_workspace_bytes.restype = c_longlong
    L.nphm_mlp_sdfgrad_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_mlp_sdfgrad_backward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_longlong, POINTER(c_void_p),
                                            POINTER(c_void_p), c_void_p, c_void_p, c_void_p]
    L.nphm_mlp_fit_workspace_bytes.argtypes = [c_void_p, c_int, c_longlong]
    L.nphm_mlp_fit_workspace_bytes.restype = c_longlong
    L.nphm_mlp_fit_surface_grad.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_float, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_mlp_fit_surface_grad_batched.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_float, c_void_p,
                                                    c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_ensemble_sdfgrad_workspace_bytes.argtypes = [c_void_p, c_int, c_longlong]
    L.nphm_ensemble_sdfgrad_workspace_bytes.restype = c_longlong
    L.nphm_ensemble_sdfgrad_forward.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p,
                                                c_void_p]
    L.nphm_ensemble_sdfgrad_backward.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_longlong,
                                                 POINTER(c_void_p), POINTER(c_void_p), c_void_p, c_void_p, c_void_p]
    L.nphm_render_workspace_bytes.argtypes = [c_int, c_int, c_int]
    L.nphm_render_workspace_bytes.restype = c_longlong
    L.nphm_render_depth_normals.argtypes = [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_int, c_double,
                                            c_double, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    slab = [c_int, c_int, c_int, c_int]                 # res, block, l0, l1: the x-slab every step works on
    L.nphm_band_slab_workspace_bytes.argtypes = slab
    L.nphm_band_slab_workspace_bytes.restype = c_longlong
    L.nphm_band_slab_begin.argtypes = slab + [c_longlong, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_slab_corners.argtypes = slab + [c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_slab_gather.argtypes = slab + [POINTER(c_double), POINTER(c_double), c_longlong, c_void_p, c_void_p, c_longlong,
                                              c_void_p]
    L.nphm_band_slab_scatter.argtypes = slab + [c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_slab_classify.argtypes = slab + [c_float, c_void_p, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_slab_grow.argtypes = slab + [c_void_p, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_slab_fill.argtypes = slab + [c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_slab_block_states.argtypes = slab + [c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_slab_export.argtypes = slab + [c_int, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_slab_import.argtypes = slab + [c_int, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    heads = [c_int, c_int, c_int]                      # res, block, n_heads: S bands of the whole grid
    L.nphm_band_heads_workspace_bytes.argtypes = heads
    L.nphm_band_heads_workspace_bytes.restype = c_longlong
    L.nphm_band_heads_begin.argtypes = heads + [c_longlong, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_heads_corners.argtypes = heads + [c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_heads_classify.argtypes = heads + [c_float, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_heads_grow.argtypes = heads + [c_void_p, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_heads_gather.argtypes = heads + [POINTER(c_double), POINTER(c_double), c_longlong, c_void_p, c_void_p, c_longlong,
                                                 c_void_p]
    L.nphm_band_heads_scatter.argtypes = heads + [c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_heads_fill.argtypes = heads + [c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_heads_block_states.argtypes = heads + [c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_mc_heads_workspace_bytes.argtypes = [POINTER(McParams), c_int]
    L.nphm_mc_heads_workspace_bytes.restype = c_longlong
    L.nphm_mc_heads_count.argtypes = [c_void_p, POINTER(McParams), c_int, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_mc_heads_emit.argtypes = [c_void_p, POINTER(McParams), c_int, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_band_sparse_workspace_bytes.argtypes = slab
    L.nphm_band_sparse_workspace_bytes.restype = c_longlong
    L.nphm_band_sparse_pool_sizes.argtypes = slab + [c_longlong, POINTER(c_longlong)]
    mem = [c_void_p, c_longlong, POINTER(BandPool)]     # workspace, its bytes, the brick pool
    listing = mem + [POINTER(c_longlong), c_void_p]
    L.nphm_band_sparse_begin.argtypes = slab + [c_longlong] + listing
    L.nphm_band_sparse_corners.argtypes = slab + listing
    L.nphm_band_sparse_classify.argtypes = slab + [c_float] + listing
    L.nphm_band_sparse_grow.argtypes = slab + listing
    L.nphm_band_sparse_gather.argtypes = slab + [POINTER(c_double), POINTER(c_double), c_longlong, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_scatter.argtypes = slab + [c_longlong, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_fill.argtypes = slab + mem + [c_void_p]
    L.nphm_band_sparse_block_states.argtypes = slab + mem + [c_void_p, c_void_p]
    L.nphm_band_sparse_export.argtypes = slab + [c_int] + mem + [c_void_p, c_void_p]
    L.nphm_band_sparse_import.argtypes = slab + [c_int, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_volume.argtypes = slab + [c_int, c_int, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_mc_workspace_bytes.argtypes = slab + [c_longlong]
    L.nphm_band_sparse_mc_workspace_bytes.restype = c_longlong
    L.nphm_band_sparse_mc_count.argtypes = slab + mem + [c_void_p, c_longlong, POINTER(c_longlong), POINTER(c_longlong), c_void_p]
    L.nphm_band_sparse_mc_emit.argtypes = slab + mem + [c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_band_sparse_heads_workspace_bytes.argtypes = heads
    L.nphm_band_sparse_heads_workspace_bytes.restype = c_longlong
    heads_listing = mem + [c_void_p, c_void_p]           # counts: 4 S long longs
    L.nphm_band_sparse_heads_begin.argtypes = heads + [c_longlong] + heads_listing
    L.nphm_band_sparse_heads_corners.argtypes = heads + heads_listing
    L.nphm_band_sparse_heads_classify.argtypes = heads + [c_float] + heads_listing
    L.nphm_band_sparse_heads_grow.argtypes = heads + heads_listing
    L.nphm_band_sparse_heads_gather.argtypes = heads + [POINTER(c_double), POINTER(c_double), c_longlong, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_heads_scatter.argtypes = heads + [c_longlong, c_void_p] + mem + [c_void_p]
    L.nphm_band_sparse_heads_fill.argtypes = heads + mem + [c_void_p]
    L.nphm_band_sparse_heads_block_states.argtypes = heads + mem + [c_void_p, c_void_p]
    L.nphm_band_sparse_heads_mc_workspace_bytes.argtypes = heads + [c_longlong]
    L.nphm_band_sparse_heads_mc_workspace_bytes.restype = c_longlong
    L.nphm_band_sparse_heads_mc_count.argtypes = heads + mem + [c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_band_sparse_heads_mc_emit.argtypes = heads + mem + [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_face_cdf_workspace_bytes.argtypes = [c_longlong]
    L.nphm_face_cdf_workspace_bytes.restype = c_longlong
    L.nphm_face_cdf.argtypes = [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, POINTER(c_double), c_void_p, c_longlong, c_void_p]
    L.nphm_sample_faces.argtypes = [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p]
    L.nphm_vertex_normals_workspace_bytes.argtypes = [c_longlong, c_longlong]
    L.nphm_vertex_normals_workspace_bytes.restype = c_longlong
    L.nphm_vertex_normals.argtypes = [c_void_p, c_longlong, c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_interpolate_barycentric.argtypes = [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p, c_longlong, c_void_p,
                                               c_void_p]
    L.nphm_transfer_correspondences.argtypes = [c_void_p, c_longlong, c_void_p, c_void_p, c_longlong, c_void_p, c_longlong, c_void_p,
                                                c_void_p, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    tp = [POINTER(TraceParams)]
    L.nphm_trace_workspace_bytes.argtypes = [c_int, c_longlong]
    L.nphm_trace_workspace_bytes.restype = c_longlong
    L.nphm_trace_begin.argtypes = tp + [c_void_p, c_void_p, c_int, c_int, c_int, c_longlong, c_void_p, c_longlong, c_void_p]
    L.nphm_trace_compact.argtypes = tp + [c_int, c_void_p, c_longlong, c_void_p]
    L.nphm_trace_counts.argtypes = tp + [c_void_p, c_longlong, POINTER(c_int), c_void_p]
    L.nphm_trace_gather.argtypes = tp + [c_longlong, c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_trace_advance.argtypes = tp + [c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_trace_points.argtypes = tp + [c_void_p, c_longlong, c_void_p, c_void_p]
    L.nphm_trace_finish.argtypes = tp + [c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p]
    L.nphm_pose_apply.argtypes = [c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_int, c_void_p, c_void_p]
    L.nphm_pose_grad.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_longlong, c_void_p, c_int, c_double, c_void_p,
                                 c_void_p]
    L.nphm_pose_adam.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_int, c_int,
                                 c_void_p]
    L.nphm_register_prepare.argtypes = [c_void_p, c_int, c_float, c_float, c_float, c_void_p, c_void_p]
    L.nphm_register_search.argtypes = [POINTER(RegisterParams), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    for name in EXPORTED_SYMBOLS:                      # fail at load time, not at first use, if a symbol is missing
        getattr(L, name)
    _lib = L
    return L


def check(rc: int, what: str = ''):
    if rc != 0:
        msg = lib().nphm_last_error()
        raise NativeError('%s failed (%d): %s' % (what or 'libnphm_b200 call', rc,
                                                   msg.decode() if msg else 'unknown error'))


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _ptr_array(tensors):
    arr = (c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def _workspace(nbytes: int, what: str, device) -> torch.Tensor:
    """A uint8 workspace of the size a ``*_workspace_bytes`` entry point returned (-1: raise its error)."""
    if nbytes < 0:
        check(-1, what)
    return torch.empty(nbytes, device=device, dtype=torch.uint8)


def constant_latent_rows(lat_rep: torch.Tensor) -> Optional[torch.Tensor]:
    """``B x N x D`` (or ``B x 1 x D``) latent -> ``B x D`` if it is the same for all points of a batch
    entry, else ``None``.  Broadcast views (stride 0) are recognised without reading the data; a
    materialised ``repeat`` costs one comparison pass."""
    if lat_rep.dim() == 2:
        return lat_rep.contiguous()
    if lat_rep.shape[1] == 1 or lat_rep.stride(1) == 0:
        return lat_rep[:, 0].contiguous()
    first = lat_rep[:, :1]
    if bool((lat_rep == first).all()):
        return first[:, 0].contiguous()
    return None


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(dtype=torch.float32).contiguous()


class _Versioned:
    """Tracks parameter identity/version so that packed weights are rebuilt after in-place updates,
    ``load_state_dict`` or ``.to(device)``."""

    def _signature(self, params):
        return tuple((p.data_ptr(), p._version, str(p.device)) for p in params)


class EnsembleEngine(_Versioned):
    """Native handle for one ``FastEnsembleDeepSDFMirrored`` (packed weights live on its device)."""

    def __init__(self, module):
        self._h = c_void_p()
        e = module.ensembled_deep_sdf
        n_lin = e.num_layers - 1
        cfg = EnsembleConfig(module.num_kps, module.num_symm_pairs, module.lat_dim_glob, module.lat_dim_loc,
                             hidden_width(e, n_lin), n_lin - 1, module.pos_mlp_dim)
        check(lib().nphm_ensemble_create(byref(cfg), byref(self._h)), 'nphm_ensemble_create')
        self.n_lin = n_lin
        self.n_loc = module.num_kps
        self.lat_dim = module.lat_dim
        self.lat_dim_glob, self.lat_dim_loc = module.lat_dim_glob, module.lat_dim_loc
        self._sig = None
        self.device = None

    def __del__(self):
        try:
            if self._h and _lib is not None:
                _lib.nphm_ensemble_destroy(self._h)
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_prune_threshold(self, tau: float):
        """tau of the opt-in pruned kernel (impl='tc_pruned')."""
        check(lib().nphm_ensemble_set_prune_threshold(self._h, float(tau)), 'nphm_ensemble_set_prune_threshold')

    def _params(self, module):
        e = module.ensembled_deep_sdf
        ps = []
        for i in range(self.n_lin):
            lin = getattr(e, 'lin%d' % i)
            ps += [lin.weight, lin.bias]
        for i in (0, 2, 4):
            ps += [module.mlp_pos[i].weight, module.mlp_pos[i].bias]
        return ps

    def refresh(self, module):
        ps = self._params(module)
        anc = module.anchors            # plain attribute (EnsembledDeepSDF.py:192): may be re-assigned after first use
        sig = self._signature(ps) + ((anc.data_ptr(), anc._version, str(anc.device)) if anc is not None else (None,))
        if sig == self._sig:
            return
        dev = ps[0].device
        if dev.type != 'cuda':
            raise NativeError('the fused ensemble needs the module on a CUDA device (got %s)' % dev)
        with torch.cuda.device(dev):
            tens = [_f32c(p) for p in ps]
            lw = tens[0:2 * self.n_lin:2]
            lb = tens[1:2 * self.n_lin:2]
            pw = tens[2 * self.n_lin::2]
            pb = tens[2 * self.n_lin + 1::2]
            mean = _f32c(module.mean_anchors(dev)).reshape(-1)
            check(lib().nphm_ensemble_load_weights(self._h, _ptr_array(lw), _ptr_array(lb), _ptr_array(pw),
                                                   _ptr_array(pb), mean.data_ptr(), _stream_ptr(dev)),
                  'nphm_ensemble_load_weights')
            # the library copies on the current stream; keep the temporaries alive until it is done
            torch.cuda.current_stream(dev).synchronize()
        self._sig = sig
        self.device = dev

    # ---------------------------------------------------------------- queries
    def query(self, xyz: torch.Tensor, latents: torch.Tensor, eval_quirk: bool, quirk_period: Optional[int] = None,
              impl: Optional[int] = None):
        """xyz B x N x 3, latents B x lat_dim -> (sdf B x N x 1, anchors B x n_loc x 3)."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        latents = _f32c(latents).to(dev)
        sdf = torch.empty(B, N, 1, device=dev, dtype=torch.float32)
        anchors = torch.empty(B, self.n_loc, 3, device=dev, dtype=torch.float32)
        period = 0 if not eval_quirk else (N if quirk_period is None else int(quirk_period))
        with torch.cuda.device(dev):
            check(lib().nphm_ensemble_query(self._h, xyz.data_ptr(), latents.data_ptr(), B, N, period,
                                            sdf.data_ptr(), anchors.data_ptr(),
                                            default_impl() if impl is None else impl_code(impl), _stream_ptr(dev)),
                  'nphm_ensemble_query')
        return sdf, anchors

    def anchors(self, latents: torch.Tensor) -> torch.Tensor:
        """latents B x lat_dim -> anchors B x n_loc x 3 (the anchor head only, ``nphm_ensemble_anchors``)."""
        lat = _f32c(latents).reshape(-1, self.lat_dim)
        dev = lat.device
        out = torch.empty(lat.shape[0], self.n_loc, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().nphm_ensemble_anchors(self._h, lat.data_ptr(), lat.shape[0], out.data_ptr(), _stream_ptr(dev)),
                  'nphm_ensemble_anchors')
        return out

    def backward_inputs(self, xyz: torch.Tensor, latent: torch.Tensor, grad_sdf: torch.Tensor, quirk_period: int = 0):
        """Vector-Jacobian product of the training-mode forward (``nphm_ensemble_backward_inputs``): xyz (N,3), latent
        (lat_dim,), grad_sdf (N,) -> (sdf (N,), d/d latent (lat_dim,), d/d xyz (N,3)) - what autograd gives for
        ``decoder(xyz, latent)[0].backward(grad_sdf)``, without building a graph.  ``quirk_period > 0``: the eval-mode forward
        (``nphm_ensemble_backward_inputs_quirk``), every member's output is 1 at the rows with ``i % p == p - 1``; ``p = N`` is
        one eval-mode decoder call."""
        dev = xyz.device
        pts = _f32c(xyz).reshape(-1, 3)
        lat = _f32c(latent).reshape(-1).to(dev)
        g = _f32c(grad_sdf).reshape(-1)
        n = pts.shape[0]
        sdf = torch.empty(n, device=dev, dtype=torch.float32)
        g_lat = torch.empty(self.lat_dim, device=dev, dtype=torch.float32)
        g_pts = torch.empty(n, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            if quirk_period:
                check(lib().nphm_ensemble_backward_inputs_quirk(self._h, pts.data_ptr(), n, int(quirk_period), lat.data_ptr(),
                                                                g.data_ptr(), sdf.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(),
                                                                None, _stream_ptr(dev)),
                      'nphm_ensemble_backward_inputs_quirk')
            else:
                check(lib().nphm_ensemble_backward_inputs(self._h, pts.data_ptr(), n, lat.data_ptr(), g.data_ptr(),
                                                          sdf.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), None,
                                                          _stream_ptr(dev)),
                      'nphm_ensemble_backward_inputs')
        return sdf, g_lat, g_pts

    # ---------------------------------------------------------------- training through grad_x sdf (second order)
    def sdfgrad_forward(self, xyz_local: torch.Tensor, cond: torch.Tensor):
        """Every member's SDF and its gradient in the member's own frame, keeping what the backward needs
        (nphm_ensemble_sdfgrad_forward): xyz_local members x B x N x 3 (mirror applied), cond members x B x (lat_dim_glob +
        lat_dim_loc) -> ``(s members x B x N, g members x B x N x 3, workspace)``."""
        K, B, N, _ = xyz_local.shape
        dev = xyz_local.device
        xyz_local = _f32c(xyz_local)
        cond = _f32c(cond).to(dev)
        s = torch.empty(K, B, N, device=dev, dtype=torch.float32)
        g = torch.empty(K, B, N, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            ws = _workspace(lib().nphm_ensemble_sdfgrad_workspace_bytes(self._h, B, N), 'nphm_ensemble_sdfgrad_workspace_bytes', dev)
            check(lib().nphm_ensemble_sdfgrad_forward(self._h, xyz_local.data_ptr(), cond.data_ptr(), B, N, s.data_ptr(),
                                                      g.data_ptr(), ws.data_ptr(), _stream_ptr(dev)), 'nphm_ensemble_sdfgrad_forward')
        return s, g, ws

    def sdfgrad_backward(self, ws: torch.Tensor, grad_s: torch.Tensor, grad_g: torch.Tensor, layer_shapes, weights: bool = True,
                         biases: bool = True, want_cond: bool = True, want_xyz: bool = True):
        """Backward of :meth:`sdfgrad_forward` (nphm_ensemble_sdfgrad_backward) for grad_s members x B x N and grad_g
        members x B x N x 3; ``layer_shapes``: the ``ensembled_deep_sdf.lin{l}.weight`` shapes.  Returns ``(weight grads |
        None, bias grads | None, d/d cond members x B x C | None, d/d xyz_local members x B x N x 3 | None)``."""
        K, B, N, _ = grad_g.shape
        dev = grad_g.device
        gs, gg = _f32c(grad_s), _f32c(grad_g)
        gw = [torch.empty(s, device=dev, dtype=torch.float32) for s in layer_shapes] if weights else None
        gb = [torch.empty(s[:2], device=dev, dtype=torch.float32) for s in layer_shapes] if biases else None
        C = self.lat_dim_glob + self.lat_dim_loc
        g_cond = torch.empty(K, B, C, device=dev, dtype=torch.float32) if want_cond else None
        g_xyz = torch.empty(K, B, N, 3, device=dev, dtype=torch.float32) if want_xyz else None
        with torch.cuda.device(dev):
            check(lib().nphm_ensemble_sdfgrad_backward(self._h, gs.data_ptr(), gg.data_ptr(), ws.data_ptr(), ws.numel(), B, N,
                                                       _ptr_array(gw) if gw else None, _ptr_array(gb) if gb else None,
                                                       _ptr(g_cond), _ptr(g_xyz), _stream_ptr(dev)),
                  'nphm_ensemble_sdfgrad_backward')
        return gw, gb, g_cond, g_xyz

    def query_grid(self, latent: torch.Tensor, mini, maxi, res: int, first: int, count: int, quirk_period: int,
                   impl: Optional[int] = None, out: Optional[torch.Tensor] = None):
        """One latent over grid points [first, first+count) of the res^3 grid -> (sdf (count,), anchors)."""
        dev = latent.device
        latent = _f32c(latent).reshape(-1)
        if out is None:
            out = torch.empty(count, device=dev, dtype=torch.float32)
        anchors = torch.empty(self.n_loc, 3, device=dev, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        with torch.cuda.device(dev):
            check(lib().nphm_ensemble_query_grid(self._h, latent.data_ptr(), gmin, gmax, int(res), int(first),
                                                 int(count), int(quirk_period), out.data_ptr(), anchors.data_ptr(),
                                                 default_impl() if impl is None else impl_code(impl),
                                                 _stream_ptr(dev)),
                  'nphm_ensemble_query_grid')
        return out, anchors


def _mlp_impl(impl) -> int:
    code = default_impl() if impl is None else impl_code(impl)
    return IMPL_AUTO if code == IMPL_TC_PRUNED else code


class MlpEngine(_Versioned):
    """Native handle for one ``DeepSDF`` stack (also the backbone of ``DeformationNetwork``)."""

    def __init__(self, module):
        self._h = c_void_p()
        self.n_lin = module.num_layers - 1
        hidden = hidden_width(module, self.n_lin)
        cfg = MlpConfig(module.lat_dim, hidden, self.n_lin - 1, module.out_dim_net)
        check(lib().nphm_mlp_create(byref(cfg), byref(self._h)), 'nphm_mlp_create')
        self.out_dim = module.out_dim_net
        # which kernel family AUTO picks (mirrors tc_mlp_supported in csrc/mlp_chain.cu): nphm_mlp_query sends the
        # forward-deformation backbone (condition 232 / 200 / 264: modes compress / expr_only / glob_only) to the tensor cores;
        # every other shape runs layer by layer on the generic wgmma linear layer (csrc/tc_linear.cu, any width - e.g. the NPM
        # baseline 515 -> 1024 x 8); the fp32 FFMA kernel is kept for impl='simt'
        self.fused_shape = (hidden == 512 and self.n_lin == 7 and module.lat_dim in (232, 200, 264) and module.out_dim_net == 3)
        self.simt_ok = hidden <= 880
        self.lat_dim = module.lat_dim
        self.layer_shapes = [tuple(getattr(module, 'lin%d' % i).weight.shape) for i in range(self.n_lin)]
        self._sig = None

    def __del__(self):
        try:
            if self._h and _lib is not None:
                _lib.nphm_mlp_destroy(self._h)
        except Exception:
            pass

    def refresh(self, module):
        ps = []
        for i in range(self.n_lin):
            lin = getattr(module, 'lin%d' % i)
            ps += [lin.weight, lin.bias]
        sig = self._signature(ps)
        if sig == self._sig:
            return
        dev = ps[0].device
        if dev.type != 'cuda':
            raise NativeError('the fused MLP needs the module on a CUDA device (got %s)' % dev)
        with torch.cuda.device(dev):
            tens = [_f32c(p) for p in ps]
            check(lib().nphm_mlp_load_weights(self._h, _ptr_array(tens[0::2]), _ptr_array(tens[1::2]),
                                              _stream_ptr(dev)), 'nphm_mlp_load_weights')
            torch.cuda.current_stream(dev).synchronize()
        self._sig = sig

    def query(self, xyz: torch.Tensor, cond: torch.Tensor, impl: Optional[int] = None) -> torch.Tensor:
        """xyz B x N x 3, cond B x lat_dim -> B x N x out_dim."""
        code = _mlp_impl(impl)
        if (code == IMPL_AUTO and not self.fused_shape) or (code == IMPL_SIMT and not self.simt_ok):
            return self.query_layers(xyz, cond)
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        out = torch.empty(B, N, self.out_dim, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_query(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, out.data_ptr(), code, _stream_ptr(dev)),
                  'nphm_mlp_query')
        return out

    def query_layers(self, xyz: torch.Tensor, cond: torch.Tensor) -> torch.Tensor:
        """Forward, layer by layer on the generic wgmma linear layer (any width): xyz B x N x 3, cond B x lat_dim."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        out = torch.empty(B, N, self.out_dim, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_query_layers(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, out.data_ptr(), _stream_ptr(dev)),
                  'nphm_mlp_query_layers')
        return out

    def jacobian(self, xyz: torch.Tensor, cond: torch.Tensor):
        """(out B x N x out_dim, J B x N x out_dim x 3 = d out / d xyz) in one forward-mode pass (nphm_mlp_jacobian)."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        out = torch.empty(B, N, self.out_dim, device=dev, dtype=torch.float32)
        J = torch.empty(B, N, self.out_dim, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_jacobian(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, out.data_ptr(), J.data_ptr(),
                                          _stream_ptr(dev)), 'nphm_mlp_jacobian')
        return out, J

    def inverse_jacobian(self, xyz: torch.Tensor, cond: torch.Tensor):
        """(out B x N x 3, (I + d out / d xyz)^-1  B x N x 3 x 3) - the reference's ``jac(...).inverse()`` in one native call."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        out = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        J = torch.empty(B, N, 3, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_inverse_jacobian(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, out.data_ptr(), J.data_ptr(),
                                                  _stream_ptr(dev)), 'nphm_mlp_inverse_jacobian')
        return out, J

    def backward_inputs(self, xyz: torch.Tensor, cond: torch.Tensor, grad_out: torch.Tensor, want_xyz: bool = False,
                        reuse_value_pass: bool = False):
        """Adjoint pass (nphm_mlp_backward_inputs): grad_out B x N x out_dim -> (d/d cond  B x lat_dim, d/d xyz B x N x 3 | None).
        ``reuse_value_pass``: the preceding ``jacobian`` / ``inverse_jacobian`` call was at the same (xyz, cond)."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        g = _f32c(grad_out)
        g_cond = torch.empty(B, cond.shape[-1], device=dev, dtype=torch.float32)
        g_xyz = torch.empty(B, N, 3, device=dev, dtype=torch.float32) if want_xyz else None
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_backward_inputs(self._h, None if reuse_value_pass else xyz.data_ptr(), cond.data_ptr(), B, N,
                                                 g.data_ptr(), g_cond.data_ptr(), _ptr(g_xyz), _stream_ptr(dev)),
                  'nphm_mlp_backward_inputs')
        return g_cond, g_xyz

    # ------------------------------------------------------------ training (first order)
    def _grad_buffers(self, B, N, dev, weights, biases, want_cond, want_xyz):
        """Outputs of a training backward: (weight grads | None, bias grads | None, d/d cond | None, d/d xyz | None)."""
        shapes = self.layer_shapes
        gw = [torch.empty(s, device=dev, dtype=torch.float32) for s in shapes] if weights else None
        gb = [torch.empty(s[0], device=dev, dtype=torch.float32) for s in shapes] if biases else None
        g_cond = torch.empty(B, self.lat_dim, device=dev, dtype=torch.float32) if want_cond else None
        g_xyz = torch.empty(B, N, 3, device=dev, dtype=torch.float32) if want_xyz else None
        return gw, gb, g_cond, g_xyz

    def train_forward(self, xyz: torch.Tensor, cond: torch.Tensor, noise: Optional[torch.Tensor] = None):
        """Value pass that keeps what the backward needs (nphm_mlp_train_forward): xyz B x N x 3, cond B x lat_dim, noise
        B x N x noise_dim (added to the leading condition columns of every point) or None.  Returns ``(out B x N x out_dim,
        workspace)``; the workspace (a uint8 CUDA tensor) belongs to the caller and goes to :meth:`train_backward` with the
        same ``noise_dim``."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        nd = 0 if noise is None else int(noise.shape[-1])
        noise = None if noise is None else _f32c(noise).reshape(B, N, nd)
        out = torch.empty(B, N, self.out_dim, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            ws = _workspace(lib().nphm_mlp_train_workspace_bytes(self._h, B, N, nd), 'nphm_mlp_train_workspace_bytes', dev)
            check(lib().nphm_mlp_train_forward(self._h, xyz.data_ptr(), cond.data_ptr(), _ptr(noise), nd, B, N, out.data_ptr(),
                                               ws.data_ptr(), _stream_ptr(dev)), 'nphm_mlp_train_forward')
        return out, ws

    def train_backward(self, ws: torch.Tensor, grad_out: torch.Tensor, noise_dim: int = 0, weights: bool = True,
                       biases: bool = True, want_cond: bool = True, want_xyz: bool = False):
        """Backward of :meth:`train_forward` (nphm_mlp_train_backward) for grad_out B x N x out_dim; ``noise_dim``: the width of
        the noise that forward took (0: none).  Returns
        ``(weight grads [lin{l}.weight shape] | None, bias grads | None, d/d cond B x lat_dim | None, d/d xyz B x N x 3 | None)``."""
        B, N, _ = grad_out.shape
        dev = grad_out.device
        g = _f32c(grad_out)
        gw, gb, g_cond, g_xyz = self._grad_buffers(B, N, dev, weights, biases, want_cond, want_xyz)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_train_backward(self._h, g.data_ptr(), ws.data_ptr(), ws.numel(), int(noise_dim), B, N,
                                                _ptr_array(gw) if gw else None, _ptr_array(gb) if gb else None,
                                                _ptr(g_cond), _ptr(g_xyz), _stream_ptr(dev)), 'nphm_mlp_train_backward')
        return gw, gb, g_cond, g_xyz

    # ------------------------------------------------------------ training through grad_x sdf (second order)
    def sdfgrad_forward(self, xyz: torch.Tensor, cond: torch.Tensor):
        """SDF and its spatial gradient, keeping what the backward needs (nphm_mlp_sdfgrad_forward): xyz B x N x 3, cond
        B x lat_dim -> ``(sdf B x N x 1, d sdf / d xyz B x N x 3, workspace)``; one-output stacks only."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        sdf = torch.empty(B, N, 1, device=dev, dtype=torch.float32)
        grad = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            ws = _workspace(lib().nphm_mlp_sdfgrad_workspace_bytes(self._h, B, N), 'nphm_mlp_sdfgrad_workspace_bytes', dev)
            check(lib().nphm_mlp_sdfgrad_forward(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, sdf.data_ptr(), grad.data_ptr(),
                                                 ws.data_ptr(), _stream_ptr(dev)), 'nphm_mlp_sdfgrad_forward')
        return sdf, grad, ws

    def sdfgrad_backward(self, ws: torch.Tensor, grad_sdf: torch.Tensor, grad_grad: torch.Tensor, weights: bool = True,
                         biases: bool = True, want_cond: bool = True, want_xyz: bool = False):
        """Backward of :meth:`sdfgrad_forward` (nphm_mlp_sdfgrad_backward) for grad_sdf B x N x 1 and grad_grad B x N x 3; the
        workspace's tail is its scratch (all of its per-point memory), the part the forward filled stays as it was.
        Returns ``(weight grads | None, bias grads | None, d/d cond B x lat_dim | None, d/d xyz B x N x 3 | None)``."""
        B, N, _ = grad_grad.shape
        dev = grad_grad.device
        gs, gg = _f32c(grad_sdf), _f32c(grad_grad)
        gw, gb, g_cond, g_xyz = self._grad_buffers(B, N, dev, weights, biases, want_cond, want_xyz)
        with torch.cuda.device(dev):
            check(lib().nphm_mlp_sdfgrad_backward(self._h, gs.data_ptr(), gg.data_ptr(), ws.data_ptr(), ws.numel(), B, N,
                                                  _ptr_array(gw) if gw else None, _ptr_array(gb) if gb else None,
                                                  _ptr(g_cond), _ptr(g_xyz), _stream_ptr(dev)), 'nphm_mlp_sdfgrad_backward')
        return gw, gb, g_cond, g_xyz

    # ------------------------------------------------------------ fitting (surface term of a one-output stack)
    def fit_workspace(self, n_queries: int, n_points: int, device) -> torch.Tensor:
        """A workspace for :meth:`fit_surface_grad` at ``n_queries x n_points`` (a uint8 CUDA tensor the caller may keep)."""
        return _workspace(lib().nphm_mlp_fit_workspace_bytes(self._h, int(n_queries), int(n_points)), 'nphm_mlp_fit_workspace_bytes',
                          device)

    def fit_surface_grad(self, xyz: torch.Tensor, cond: torch.Tensor, mask: Optional[torch.Tensor], clamp: float,
                         want_xyz: bool = True, workspace: Optional[torch.Tensor] = None, out=None):
        """Surface term of the fitters (nphm_mlp_fit_surface_grad): ``mean |s|`` over the points with ``mask != 0`` and
        ``|s| < clamp``, xyz B x N x 3, cond B x lat_dim, mask B x N (or None: all valid).  Returns
        ``(loss_terms (8,): [0] loss (NaN if nothing is kept), [5] kept count;  d loss / d cond  B x lat_dim;
        d loss / d xyz  B x N x 3 | None)``.  ``workspace`` / ``out`` (a tuple like the result) let a loop reuse its buffers."""
        B, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        m = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
        if out is None:
            out = (torch.zeros(8, device=dev, dtype=torch.float32), torch.empty(B, self.lat_dim, device=dev, dtype=torch.float32),
                   torch.empty(B, N, 3, device=dev, dtype=torch.float32) if want_xyz else None)
        terms, g_cond, g_xyz = out
        with torch.cuda.device(dev):
            ws = self.fit_workspace(B, N, dev) if workspace is None else workspace
            check(lib().nphm_mlp_fit_surface_grad(self._h, xyz.data_ptr(), cond.data_ptr(), B, N, _ptr(m), float(clamp),
                                                  terms.data_ptr(), g_cond.data_ptr(), _ptr(g_xyz), ws.data_ptr(), ws.numel(),
                                                  _stream_ptr(dev)), 'nphm_mlp_fit_surface_grad')
        return terms, g_cond, g_xyz

    def fit_surface_grad_batched(self, xyz: torch.Tensor, cond: torch.Tensor, mask: Optional[torch.Tensor], clamp: float,
                                 want_xyz: bool = True, workspace: Optional[torch.Tensor] = None, out=None):
        """:meth:`fit_surface_grad` per scan (nphm_mlp_fit_surface_grad_batched): xyz S x n x 3, cond S x lat_dim, mask S x n (or
        None: all valid); scan k's loss is the mean |s| over its own kept points.  Returns ``(loss_terms S x 8, d loss_k / d cond_k
        S x lat_dim, d loss_k / d xyz  S x n x 3 | None)``.  ``workspace``: one of :meth:`fit_workspace` at ``(S, n)``."""
        S, N, _ = xyz.shape
        dev = xyz.device
        xyz = _f32c(xyz)
        cond = _f32c(cond).to(dev)
        m = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
        if out is None:
            out = (torch.zeros(S, 8, device=dev, dtype=torch.float32), torch.empty(S, self.lat_dim, device=dev, dtype=torch.float32),
                   torch.empty(S, N, 3, device=dev, dtype=torch.float32) if want_xyz else None)
        terms, g_cond, g_xyz = out
        with torch.cuda.device(dev):
            ws = self.fit_workspace(S, N, dev) if workspace is None else workspace
            check(lib().nphm_mlp_fit_surface_grad_batched(self._h, xyz.data_ptr(), cond.data_ptr(), _ptr(m), S, N, float(clamp),
                                                          terms.data_ptr(), g_cond.data_ptr(), _ptr(g_xyz), ws.data_ptr(),
                                                          ws.numel(), _stream_ptr(dev)), 'nphm_mlp_fit_surface_grad_batched')
        return terms, g_cond, g_xyz

    def broyden_search(self, obs: torch.Tensor, cond: torch.Tensor, x_init: torch.Tensor, J_inv_init: torch.Tensor,
                       max_steps: int = 15, cvg_thresh: float = 1e-6, dvg_thresh: float = 0.2, eps: float = 1e-6,
                       early_exit: bool = True, compact: bool = False):
        """Roots of ``x + F(x; cond) - obs`` by the reference's Broyden iteration, entirely on the device.
        obs, x_init: B x N x 3, cond: B x lat_dim, J_inv_init: B x N x 3 x 3.  ``compact``: each step runs the network and
        the update on the still-live samples only (nphm_mlp_broyden_search_compact; bitwise the same result), for point sets
        large enough that the frozen samples dominate.
        Returns ``(x B x N x 3, diff B x N, valid B x N bool, steps taken)``."""
        B, N, _ = obs.shape
        dev = obs.device
        obs = _f32c(obs)
        cond = _f32c(cond).to(dev)
        x = _f32c(x_init).clone()
        jinv = _f32c(J_inv_init.reshape(B, N, 9))
        diff = torch.empty(B, N, device=dev, dtype=torch.float32)
        valid = torch.empty(B, N, device=dev, dtype=torch.uint8)
        steps = c_int(0)
        with torch.cuda.device(dev):
            if compact:
                nbytes, fn = lib().nphm_broyden_compact_workspace_bytes(B, N), 'nphm_mlp_broyden_search_compact'
            else:
                nbytes, fn = lib().nphm_broyden_workspace_bytes(B * N), 'nphm_mlp_broyden_search'
            ws = torch.empty(max(int(nbytes), 256), device=dev, dtype=torch.uint8)
            check(getattr(lib(), fn)(self._h, cond.data_ptr(), B, N, obs.data_ptr(), x.data_ptr(),
                                     jinv.data_ptr(), int(max_steps), float(cvg_thresh), float(dvg_thresh),
                                     float(eps), diff.data_ptr(), valid.data_ptr(),
                                     byref(steps) if early_exit else None,       # None: no host sync, all steps run
                                     ws.data_ptr(), _stream_ptr(dev)), fn)
        return x, diff, valid.bool(), steps.value


# ------------------------------------------------------------------------------------------ marching cubes
def marching_cubes_device(volume: torch.Tensor, iso: float = 0.0, negate: bool = False, x_global0: int = 0,
                          ghost_lo: bool = False, vert_id_base: Optional[int] = None):
    """GPU marching cubes on a CUDA float32 volume (nx, ny, nz).  Returns (verts (V,3) float64 CUDA in global
    index units, tris (T,3) int64 CUDA).  With ``vert_id_base=None`` ids start at 0; a sharded caller passes the
    number of vertices of all earlier slabs, see ``nphm_b200.distributed``."""
    assert volume.is_cuda and volume.dtype == torch.float32 and volume.dim() == 3
    vol = volume.contiguous()
    dev = vol.device
    p = McParams(vol.shape[0], vol.shape[1], vol.shape[2], int(x_global0), int(bool(ghost_lo)), int(bool(negate)),
                 float(iso))
    L = lib()
    ws_bytes = L.nphm_mc_workspace_bytes(byref(p))
    if ws_bytes < 0:
        check(-1, 'nphm_mc_workspace_bytes')
    ws = torch.empty(max(int(ws_bytes), 256), device=dev, dtype=torch.uint8)
    nv, nt = c_longlong(0), c_longlong(0)
    with torch.cuda.device(dev):
        check(L.nphm_mc_count(vol.data_ptr(), byref(p), ws.data_ptr(), byref(nv), byref(nt), _stream_ptr(dev)),
              'nphm_mc_count')
        verts = torch.empty(nv.value, 3, device=dev, dtype=torch.float64)
        tris = torch.empty(nt.value, 3, device=dev, dtype=torch.int64)
        if nv.value or nt.value:
            check(L.nphm_mc_emit(vol.data_ptr(), byref(p), ws.data_ptr(), int(vert_id_base or 0),
                                 verts.data_ptr(), tris.data_ptr(), _stream_ptr(dev)), 'nphm_mc_emit')
    return verts, tris


def marching_cubes_count(volume: torch.Tensor, iso=0.0, negate=False, x_global0=0, ghost_lo=False):
    """Pass 1 only: (n_verts, n_tris, params, workspace) for a slab; used by the sharded extraction."""
    vol = volume.contiguous()
    dev = vol.device
    p = McParams(vol.shape[0], vol.shape[1], vol.shape[2], int(x_global0), int(bool(ghost_lo)), int(bool(negate)),
                 float(iso))
    L = lib()
    ws = torch.empty(max(int(L.nphm_mc_workspace_bytes(byref(p))), 256), device=dev, dtype=torch.uint8)
    nv, nt = c_longlong(0), c_longlong(0)
    with torch.cuda.device(dev):
        check(L.nphm_mc_count(vol.data_ptr(), byref(p), ws.data_ptr(), byref(nv), byref(nt), _stream_ptr(dev)),
              'nphm_mc_count')
    return nv.value, nt.value, p, ws


def marching_cubes_emit(volume: torch.Tensor, p: McParams, ws: torch.Tensor, n_verts: int, n_tris: int,
                        vert_id_base: int):
    vol = volume.contiguous()
    dev = vol.device
    verts = torch.empty(n_verts, 3, device=dev, dtype=torch.float64)
    tris = torch.empty(n_tris, 3, device=dev, dtype=torch.int64)
    if n_verts or n_tris:
        with torch.cuda.device(dev):
            check(lib().nphm_mc_emit(vol.data_ptr(), byref(p), ws.data_ptr(), int(vert_id_base), verts.data_ptr(),
                                     tris.data_ptr(), _stream_ptr(dev)), 'nphm_mc_emit')
    return verts, tris


def marching_cubes_host(volume: np.ndarray, iso: float = 0.0, negate: bool = False):
    """== ``mcubes.marching_cubes`` on a host array through the host-buffer C entry point."""
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    nx, ny, nz = vol.shape
    nv, nt = c_longlong(0), c_longlong(0)
    L = lib()
    check(L.nphm_marching_cubes_host(vol.ctypes.data, nx, ny, nz, float(iso), int(negate), None, None,
                                     byref(nv), byref(nt)), 'nphm_marching_cubes_host')
    verts = np.empty((nv.value, 3), np.float64)
    tris = np.empty((nt.value, 3), np.int64)
    if nv.value or nt.value:
        check(L.nphm_marching_cubes_host(vol.ctypes.data, nx, ny, nz, float(iso), int(negate), verts.ctypes.data,
                                         tris.ctypes.data, byref(nv), byref(nt)), 'nphm_marching_cubes_host')
    return verts, tris.view(np.uint64)


# ------------------------------------------------------------------------------------------ evaluation metrics
def nearest_neighbors(src: torch.Tensor, tgt: torch.Tensor):
    """(dist (n_src,) float64, idx (n_src,) int64) of the nearest ``tgt`` point of every ``src`` point (CUDA float32 clouds)."""
    assert src.is_cuda and tgt.is_cuda and src.shape[-1] == 3 and tgt.shape[-1] == 3
    dev = src.device
    s, t = _f32c(src).reshape(-1, 3), _f32c(tgt).reshape(-1, 3)
    dist = torch.empty(s.shape[0], device=dev, dtype=torch.float64)
    idx = torch.empty(s.shape[0], device=dev, dtype=torch.int64)
    with torch.cuda.device(dev):
        check(lib().nphm_nearest_neighbors(s.data_ptr(), s.shape[0], t.data_ptr(), t.shape[0], dist.data_ptr(), idx.data_ptr(),
                                           _stream_ptr(dev)), 'nphm_nearest_neighbors')
    return dist, idx


# ------------------------------------------------------------------------------------------ rendering
def check_face_range(faces: torch.Tensor, n_verts: int):
    """Raise ``ValueError`` unless every face index lies in ``[0, n_verts)`` (the native mesh entry points assume it)."""
    if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= n_verts):
        raise ValueError('face indices must lie in [0, %d) (got [%d, %d])' % (n_verts, int(faces.min()), int(faces.max())))


def render_depth_normals(verts: torch.Tensor, faces: torch.Tensor, world_to_eye: torch.Tensor, intrinsics: torch.Tensor,
                         height: int, width: int, znear: float = 0.1, zfar: float = 2.0, want_tri: bool = False):
    """Rasterize one mesh into V views in one call (nphm_render_depth_normals).  verts (n, 3) and faces (m, 3) on a CUDA device,
    world_to_eye (V, 3, 4) and intrinsics (V, 4: fx fy cx cy).  Returns ``(depth (V, H, W) float32 eye depth, 0 = background;
    normals (V, H, W, 3) uint8; triangle index (V, H, W) int32, -1 = background | None)``.  Face indices outside
    ``[0, n_verts)`` raise ``ValueError`` before the call."""
    assert verts.is_cuda and verts.shape[-1] == 3 and faces.shape[-1] == 3
    dev = verts.device
    v = _f32c(verts).reshape(-1, 3)
    f = faces.detach().to(device=dev, dtype=torch.int64).reshape(-1, 3)
    check_face_range(f, v.shape[0])
    f = f.to(torch.int32).contiguous()
    w2e = world_to_eye.detach().to(device=dev, dtype=torch.float64).reshape(-1, 12).contiguous()
    intr = intrinsics.detach().to(device=dev, dtype=torch.float64).reshape(-1, 4).contiguous()
    V = w2e.shape[0]
    assert intr.shape[0] == V
    H, W = int(height), int(width)
    L = lib()
    n_pix = V * max(H, 0) * max(W, 0)
    depth = torch.empty(n_pix, device=dev, dtype=torch.float32)
    normals = torch.empty(n_pix * 3, device=dev, dtype=torch.uint8)
    tri = torch.empty(n_pix, device=dev, dtype=torch.int32) if want_tri else None
    with torch.cuda.device(dev):
        ws = _workspace(L.nphm_render_workspace_bytes(V, H, W), 'nphm_render_workspace_bytes', dev)
        check(L.nphm_render_depth_normals(v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], w2e.data_ptr(), intr.data_ptr(), V,
                                          float(znear), float(zfar), H, W, depth.data_ptr(), normals.data_ptr(), _ptr(tri),
                                          ws.data_ptr(), ws.numel(), _stream_ptr(dev)), 'nphm_render_depth_normals')
    return (depth.view(V, H, W), normals.view(V, H, W, 3), None if tri is None else tri.view(V, H, W))


# ------------------------------------------------------------------------------------------ sphere tracing
TRACE_LIVE, TRACE_BRACKET, TRACE_HIT, TRACE_MISS, TRACE_OUT_OF_STEPS, TRACE_INVALID = range(6)


class SdfTrace:
    """The ray state of one chunk of a sphere trace (csrc/sdf_trace.cu): ``n_rays`` consecutive pixels of the views for each of
    ``n_heads`` heads.  The field is evaluated by the caller between :meth:`gather` and :meth:`advance`; nothing but
    :meth:`counts` reads back from the device."""

    def __init__(self, n_heads: int, n_rays: int, mini, maxi, scale: float, znear: float, zfar: float, step_factor: float,
                 min_step: float, hit_eps: float, max_steps: int, device):
        self.p = TraceParams(int(n_heads), int(n_rays), (c_double * 3)(*[float(v) for v in mini]),
                             (c_double * 3)(*[float(v) for v in maxi]), float(scale), float(znear), float(zfar), float(step_factor),
                             float(min_step), float(hit_eps), int(max_steps))
        self.device = device
        self.ws = _workspace(lib().nphm_trace_workspace_bytes(int(n_heads), int(n_rays)), 'nphm_trace_workspace_bytes', device)

    def _call(self, fn, *args):
        with torch.cuda.device(self.device):
            check(getattr(lib(), fn)(byref(self.p), *args), fn)

    def _mem(self):
        return self.ws.data_ptr(), self.ws.numel()

    def begin(self, cam_to_world: torch.Tensor, intrinsics: torch.Tensor, height: int, width: int, first_pixel: int):
        """cam_to_world (V, 12) and intrinsics (V, 4) float64 CUDA tensors."""
        self._c2w, self._intr = cam_to_world, intrinsics                  # kept alive until the stream has read them
        self._call('nphm_trace_begin', cam_to_world.data_ptr(), intrinsics.data_ptr(), cam_to_world.shape[0], int(height), int(width),
                   int(first_pixel), *self._mem(), _stream_ptr(self.device))

    def compact(self, refine: bool):
        self._call('nphm_trace_compact', int(bool(refine)), *self._mem(), _stream_ptr(self.device))

    def counts(self):
        """The per-head counts of the last :meth:`compact` (one read-back)."""
        out = (c_int * self.p.n_heads)()
        self._call('nphm_trace_counts', *self._mem(), out, _stream_ptr(self.device))
        return list(out)

    def gather(self, n_cols: int, out: torch.Tensor) -> torch.Tensor:
        """out: (n_heads, >= n_cols, 3) float32; returns its (n_heads, n_cols, 3) view of the listed rays' sample points."""
        pts = out.reshape(-1)[:self.p.n_heads * n_cols * 3]
        self._call('nphm_trace_gather', int(n_cols), *self._mem(), pts.data_ptr(), _stream_ptr(self.device))
        return pts.view(self.p.n_heads, n_cols, 3)

    def advance(self, refine: bool, sdf: torch.Tensor, valid: Optional[torch.Tensor] = None):
        """sdf (n_heads, n_cols) float32 at the gathered points, valid the same shape (bool / uint8) or None."""
        n_cols = sdf.shape[1]
        sdf = _f32c(sdf)
        v = None if valid is None else valid.to(torch.uint8).contiguous()
        self._call('nphm_trace_advance', int(bool(refine)), int(n_cols), sdf.data_ptr(), _ptr(v), *self._mem(), _stream_ptr(self.device))
        self._keep = (sdf, v)

    def points(self) -> torch.Tensor:
        out = torch.empty(self.p.n_heads, self.p.n_rays, 3, device=self.device, dtype=torch.float32)
        self._call('nphm_trace_points', *self._mem(), out.data_ptr(), _stream_ptr(self.device))
        return out

    def finish(self, grad: torch.Tensor, jinv: Optional[torch.Tensor], valid: Optional[torch.Tensor], first_pixel: int,
               depth: torch.Tensor, normals: torch.Tensor, points: Optional[torch.Tensor], status: torch.Tensor, steps: torch.Tensor):
        """Write the chunk into the (S, n_pixels, ...) images."""
        g = _f32c(grad)
        j = None if jinv is None else _f32c(jinv)
        v = None if valid is None else valid.to(torch.uint8).contiguous()
        self._call('nphm_trace_finish', *self._mem(), g.data_ptr(), _ptr(j), _ptr(v), depth.shape[1], int(first_pixel), depth.data_ptr(),
                   normals.data_ptr(), _ptr(points), status.data_ptr(), steps.data_ptr(), _stream_ptr(self.device))


# ------------------------------------------------------------------------------------------ training supervision
def _mesh(verts, faces, device=None):
    """(n, 3) float64 vertices and (m, 3) int32 faces from arrays or tensors, on ``device`` (None: the vertices' CUDA device, else
    the current one); face indices outside ``[0, n)`` raise ``ValueError`` before anything reaches the device."""
    v = torch.as_tensor(verts).detach().reshape(-1, 3)
    f = torch.as_tensor(faces).detach().to(torch.int64).reshape(-1, 3)
    check_face_range(f, v.shape[0])
    if device is None:
        device = v.device if v.is_cuda else torch.device('cuda', torch.cuda.current_device())
    return v.to(device=device, dtype=torch.float64).contiguous(), f.to(device=device, dtype=torch.int32).contiguous()


def _f64c(t, dev) -> torch.Tensor:
    return torch.as_tensor(t).detach().to(device=dev, dtype=torch.float64).contiguous()


def face_cdf(verts, faces, device=None) -> torch.Tensor:
    """Inclusive prefix sum of the face areas (nphm_face_cdf), (m,) float64 on the device.  Raises ``NativeError`` when the total
    area is 0 or not finite, or the mesh has no faces."""
    v, f = _mesh(verts, faces, device)
    dev = v.device
    cdf = torch.empty(f.shape[0], device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        ws = _workspace(lib().nphm_face_cdf_workspace_bytes(f.shape[0]), 'nphm_face_cdf_workspace_bytes', dev)
        check(lib().nphm_face_cdf(v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], cdf.data_ptr(), None, ws.data_ptr(), ws.numel(),
                                  _stream_ptr(dev)), 'nphm_face_cdf')
    return cdf


def sample_faces(cdf: torch.Tensor, uniforms: torch.Tensor):
    """Area-weighted samples (nphm_sample_faces) from a face CDF and (n, 3) float64 uniforms on the same CUDA device:
    ``(face (n,) int64, barycentrics (n, 3) float64)``."""
    dev = cdf.device
    u = _f64c(uniforms, dev).reshape(-1, 3)
    n = u.shape[0]
    face = torch.empty(n, device=dev, dtype=torch.int64)
    bary = torch.empty(n, 3, device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        check(lib().nphm_sample_faces(cdf.data_ptr(), cdf.numel(), u.data_ptr(), n, face.data_ptr(), bary.data_ptr(), _stream_ptr(dev)),
              'nphm_sample_faces')
    return face, bary


def vertex_normals(verts, faces, device=None) -> torch.Tensor:
    """Area-weighted unit vertex normals (nphm_vertex_normals), (n, 3) float64 on the device; (0, 0, 0) where the sum is zero."""
    v, f = _mesh(verts, faces, device)
    dev = v.device
    out = torch.empty(v.shape[0], 3, device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        ws = _workspace(lib().nphm_vertex_normals_workspace_bytes(v.shape[0], f.shape[0]), 'nphm_vertex_normals_workspace_bytes', dev)
        check(lib().nphm_vertex_normals(v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], out.data_ptr(), ws.data_ptr(), ws.numel(),
                                        _stream_ptr(dev)), 'nphm_vertex_normals')
    return out


def interpolate_barycentric(faces, face_idx: torch.Tensor, bary: torch.Tensor, attr) -> torch.Tensor:
    """``sum_k bary[:, k] attr[faces[face_idx, k]]`` (nphm_interpolate_barycentric), (n, 3) float64 on the device of
    ``face_idx``; ``attr`` has one row per vertex.  Face indices outside ``[0, len(attr))`` raise ``ValueError``."""
    dev = face_idx.device
    a, f = _mesh(attr, faces, dev)
    idx = face_idx.detach().to(dtype=torch.int64).contiguous()
    check_face_range(idx, f.shape[0])
    b = _f64c(bary, dev).reshape(-1, 3)
    out = torch.empty(b.shape[0], 3, device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        check(lib().nphm_interpolate_barycentric(f.data_ptr(), f.shape[0], idx.data_ptr(), b.data_ptr(), b.shape[0], a.data_ptr(),
                                                 a.shape[0], out.data_ptr(), _stream_ptr(dev)), 'nphm_interpolate_barycentric')
    return out


def transfer_correspondences(src_verts, src_faces, dst_verts, dst_faces, face_idx: torch.Tensor, bary: torch.Tensor, offsets):
    """Carry samples on the source mesh to the target mesh with the same faces (nphm_transfer_correspondences): ``face_idx`` and
    ``bary`` as :func:`sample_faces` returns them, ``offsets`` (n,).  Returns ``(p_src + o n_src, p_dst + o n_dst, n_src, n_dst)``,
    each (n, 3) float64 on the device of ``face_idx``."""
    dev = face_idx.device
    sv, sf = _mesh(src_verts, src_faces, dev)
    dv, df = _mesh(dst_verts, dst_faces, dev)
    if sf.shape[0] != df.shape[0]:
        raise ValueError('source and target meshes must have the same faces (got %d and %d)' % (sf.shape[0], df.shape[0]))
    idx = face_idx.detach().to(dtype=torch.int64).contiguous()
    check_face_range(idx, sf.shape[0])
    b = _f64c(bary, dev).reshape(-1, 3)
    o = _f64c(offsets, dev).reshape(-1)
    n = b.shape[0]
    out = [torch.empty(n, 3, device=dev, dtype=torch.float64) for _ in range(4)]
    with torch.cuda.device(dev):
        check(lib().nphm_transfer_correspondences(sv.data_ptr(), sv.shape[0], sf.data_ptr(), dv.data_ptr(), dv.shape[0], df.data_ptr(),
                                                  sf.shape[0], idx.data_ptr(), b.data_ptr(), o.data_ptr(), n,
                                                  *[t.data_ptr() for t in out], _stream_ptr(dev)), 'nphm_transfer_correspondences')
    return tuple(out)


# ------------------------------------------------------------------------------------------ narrow-band extraction
class NarrowBand:
    """Band state of the x-slab of block layers ``[l0, l1)`` of a ``res^3`` grid in blocks of ``block^3`` cells
    (``nphm_band_slab_*``, DESIGN §4.13, §4.16) in a workspace this object owns; ``l1=None`` takes every block layer, so the
    default slab is the whole grid.  The slab holds the voxel planes ``[x0, x1]``, with a volume of :attr:`n_planes` planes from
    :attr:`first_plane` (``x0 - 1``, the ghost plane, when ``l0 > 0``).  The listing steps return the number of voxels they listed;
    :meth:`gather` / :meth:`scatter` move the listed voxels' coordinates out and their values into the volume, and :meth:`export` /
    :meth:`import_` merge a plane shared with a neighbour."""

    def __init__(self, res: int, block: int, device, l0: int = 0, l1: Optional[int] = None):
        self.res, self.block = int(res), int(block)
        self.device = torch.device(device)
        # max(): block 0 must reach the native argument check, which rejects it, rather than fail in this division
        self.blocks_per_axis = -(-(self.res - 1) // max(self.block, 1))
        self.l0 = int(l0)
        self.l1 = self.blocks_per_axis if l1 is None else int(l1)
        self._geo = (self.res, self.block, self.l0, self.l1)
        with torch.cuda.device(self.device):
            self.ws = _workspace(lib().nphm_band_slab_workspace_bytes(*self._geo), 'nphm_band_slab_workspace_bytes', self.device)
        self.active_blocks = 0
        self.x0 = self.l0 * self.block
        self.x1 = min(self.l1 * self.block, self.res - 1)
        self.ghost = self.l0 > 0
        self.first_plane = self.x0 - int(self.ghost)
        self.n_planes = self.x1 + 1 - self.first_plane
        self.plane_bytes = 5 * self.res * self.res          # res^2 float32 values, then res^2 evaluated flags

    def _call(self, step, *args):
        with torch.cuda.device(self.device):
            check(getattr(lib(), 'nphm_band_slab_' + step)(*self._geo, *args, _stream_ptr(self.device)), 'nphm_band_slab_' + step)

    def _call_listing(self, step, *before_ws):
        counts = (c_longlong * 2)()
        self._call(step, *before_ws, self.ws.data_ptr(), self.ws.numel(), counts)
        self.active_blocks = counts[1]
        return counts[0]

    def begin(self, quirk_period: int = 0) -> int:
        """Reset; with ``quirk_period > 0`` list the eval-mode quirk voxels and activate the blocks around them."""
        return self._call_listing('begin', int(quirk_period))

    def corners(self) -> int:
        return self._call_listing('corners')

    def classify(self, tau: float, vol: torch.Tensor) -> int:
        return self._call_listing('classify', float(tau), vol.data_ptr())

    def grow(self, vol: torch.Tensor) -> int:
        return self._call_listing('grow', vol.data_ptr())

    def gather(self, n: int, mini, maxi) -> torch.Tensor:
        """(n, 3) float32 coordinates of the first ``n`` listed voxels."""
        xyz = torch.empty(int(n), 3, device=self.device, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        self._call('gather', gmin, gmax, int(n), _ptr(xyz) if n else None, self.ws.data_ptr(), self.ws.numel())
        return xyz

    def scatter(self, values: torch.Tensor, vol: torch.Tensor):
        v = _f32c(values).reshape(-1)
        self._call('scatter', v.numel(), v.data_ptr() if v.numel() else None, vol.data_ptr(), self.ws.data_ptr(), self.ws.numel())

    def fill(self, vol: torch.Tensor):
        self._call('fill', vol.data_ptr(), self.ws.data_ptr(), self.ws.numel())

    def block_states(self) -> torch.Tensor:
        """(l1 - l0, blocks, blocks) bool: which blocks of the slab are active."""
        nb = self.blocks_per_axis
        out = torch.empty(self.l1 - self.l0, nb, nb, device=self.device, dtype=torch.uint8)
        self._call('block_states', self.ws.data_ptr(), self.ws.numel(), out.data_ptr())
        return out != 0

    def volume(self) -> torch.Tensor:
        """An uninitialised (n_planes, res, res) float32 slab volume on the band's device."""
        return torch.empty(self.n_planes, self.res, self.res, device=self.device, dtype=torch.float32)

    def export(self, plane: int, vol: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """uint8 buffer of :attr:`plane_bytes`: the values of global ``plane`` and which of its voxels this slab evaluated."""
        buf = torch.empty(self.plane_bytes, device=self.device, dtype=torch.uint8) if out is None else out
        self._call('export', int(plane), vol.data_ptr(), self.ws.data_ptr(), self.ws.numel(), buf.data_ptr())
        return buf

    def import_(self, plane: int, buf: torch.Tensor, vol: torch.Tensor):
        """Merge a neighbour's :meth:`export` of the shared ``plane`` (x0 or x1), or copy its filled plane x0 - 1 into the ghost
        plane."""
        if buf.device != self.device or buf.dtype != torch.uint8 or buf.numel() != self.plane_bytes:
            raise ValueError('NarrowBand.import_: need a uint8 buffer of %d bytes on %s' % (self.plane_bytes, self.device))
        self._call('import', int(plane), buf.data_ptr(), vol.data_ptr(), self.ws.data_ptr(), self.ws.numel())


def NarrowBandSlab(res: int, block: int, l0: int, l1: int, device) -> NarrowBand:
    """The :class:`NarrowBand` of the x-slab of block layers ``[l0, l1)``, in the argument order the callers of the multi-GPU band
    use."""
    return NarrowBand(res, block, device, l0, l1)


class NarrowBandHeads:
    """The band of :class:`NarrowBand` on the whole ``res^3`` grid for ``n_heads`` heads in lockstep (``nphm_band_heads_*``,
    DESIGN §4.18): S latent codes of one decoder, each step one launch sequence for all of them.  The listing steps return the S
    counts (read back with one copy; :attr:`readbacks` counts the synchronising calls), :meth:`gather` / :meth:`scatter` move
    ``S x n_pad`` head-major rows, and :meth:`marching_cubes` meshes the S filled volumes with one count read-back.  Every head's
    state evolves exactly as a :class:`NarrowBand` driven through the same steps."""

    def __init__(self, res: int, block: int, device, n_heads: int):
        self.res, self.block, self.n_heads = int(res), int(block), int(n_heads)
        self.device = torch.device(device)
        self.blocks_per_axis = -(-(self.res - 1) // max(self.block, 1))
        self._geo = (self.res, self.block, self.n_heads)
        with torch.cuda.device(self.device):
            self.ws = _workspace(lib().nphm_band_heads_workspace_bytes(*self._geo), 'nphm_band_heads_workspace_bytes', self.device)
        self.active_blocks = [0] * self.n_heads
        self.readbacks = 0                  # stream synchronisations of the listing steps and marching cubes so far
        self.mc_bytes = 0                   # marching-cubes workspace of the last mesh

    @staticmethod
    def device_bytes_per_head(res: int, block: int) -> int:
        """Device bytes one head holds: its band workspace, volume and marching-cubes scratch."""
        L = lib()
        band = L.nphm_band_heads_workspace_bytes(int(res), int(block), 2) - L.nphm_band_heads_workspace_bytes(int(res), int(block), 1)
        p = McParams(int(res), int(res), int(res), 0, 0, 1, 0.0)
        mc = L.nphm_mc_heads_workspace_bytes(byref(p), 2) - L.nphm_mc_heads_workspace_bytes(byref(p), 1)
        if band < 0 or mc < 0:
            check(-1, 'nphm_band_heads_workspace_bytes')
        return int(band + mc + 4 * int(res) ** 3)

    def _call(self, step, *args):
        with torch.cuda.device(self.device):
            check(getattr(lib(), 'nphm_band_heads_' + step)(*self._geo, *args, _stream_ptr(self.device)), 'nphm_band_heads_' + step)

    def _call_listing(self, step, *before_ws):
        counts = (c_longlong * (2 * self.n_heads))()
        self._call(step, *before_ws, self.ws.data_ptr(), self.ws.numel(), counts)
        self.readbacks += 1
        self.active_blocks = list(counts[1::2])
        return list(counts[0::2])

    def begin(self, quirk_period: int = 0):
        """Reset every head; with ``quirk_period > 0`` list the eval-mode quirk voxels (the same for every head)."""
        return self._call_listing('begin', int(quirk_period))

    def corners(self):
        return self._call_listing('corners')

    def classify(self, tau: float, vols: torch.Tensor):
        return self._call_listing('classify', float(tau), vols.data_ptr())

    def grow(self, vols: torch.Tensor):
        return self._call_listing('grow', vols.data_ptr())

    def gather(self, n_pad: int, mini, maxi) -> torch.Tensor:
        """(S, n_pad, 3) float32 coordinates: each head's listed voxels, then padding rows that repeat one of them."""
        xyz = torch.empty(self.n_heads, int(n_pad), 3, device=self.device, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        self._call('gather', gmin, gmax, int(n_pad), _ptr(xyz) if n_pad else None, self.ws.data_ptr(), self.ws.numel())
        return xyz

    def scatter(self, values: torch.Tensor, vols: torch.Tensor):
        """values (S, n_pad) in the layout of :meth:`gather`: each head's listed rows into its volume, the padding dropped."""
        v = _f32c(values).reshape(self.n_heads, -1)
        n_pad = v.shape[1]
        self._call('scatter', n_pad, v.data_ptr() if n_pad else None, vols.data_ptr(), self.ws.data_ptr(), self.ws.numel())

    def fill(self, vols: torch.Tensor):
        self._call('fill', vols.data_ptr(), self.ws.data_ptr(), self.ws.numel())

    def block_states(self) -> torch.Tensor:
        """(S, blocks, blocks, blocks) bool: which blocks of each head are active."""
        nb = self.blocks_per_axis
        out = torch.empty(self.n_heads, nb, nb, nb, device=self.device, dtype=torch.uint8)
        self._call('block_states', self.ws.data_ptr(), self.ws.numel(), out.data_ptr())
        return out != 0

    def volumes(self) -> torch.Tensor:
        """Uninitialised (S, res, res, res) float32 volumes on the band's device."""
        return torch.empty(self.n_heads, self.res, self.res, self.res, device=self.device, dtype=torch.float32)

    def marching_cubes(self, vols: torch.Tensor):
        """Marching cubes on ``-vols`` at 0 for every head (``nphm_mc_heads_count`` / ``_emit``): ``(verts (V, 3) float64, tris
        (T, 3) int64, counts)`` with the S meshes one after the other in index units, ids local to each head, and ``counts`` the
        S ``(n_verts, n_tris)``; head h's part is what :func:`marching_cubes_device` ``(vols[h], 0, negate=True)`` gives."""
        v = vols.contiguous()
        assert v.shape == (self.n_heads, self.res, self.res, self.res) and v.dtype == torch.float32 and v.device == self.device
        p = McParams(self.res, self.res, self.res, 0, 0, 1, 0.0)
        L = lib()
        with torch.cuda.device(self.device):
            ws = _workspace(L.nphm_mc_heads_workspace_bytes(byref(p), self.n_heads), 'nphm_mc_heads_workspace_bytes', self.device)
            self.mc_bytes = ws.numel()
            counts = (c_longlong * (2 * self.n_heads))()
            check(L.nphm_mc_heads_count(v.data_ptr(), byref(p), self.n_heads, ws.data_ptr(), ws.numel(), counts,
                                        _stream_ptr(self.device)), 'nphm_mc_heads_count')
            self.readbacks += 1
            pairs = [(counts[2 * h], counts[2 * h + 1]) for h in range(self.n_heads)]
            verts = torch.empty(sum(c[0] for c in pairs), 3, device=self.device, dtype=torch.float64)
            tris = torch.empty(sum(c[1] for c in pairs), 3, device=self.device, dtype=torch.int64)
            if verts.shape[0] or tris.shape[0]:
                check(L.nphm_mc_heads_emit(v.data_ptr(), byref(p), self.n_heads, ws.data_ptr(), ws.numel(), verts.data_ptr(),
                                           tris.data_ptr(), _stream_ptr(self.device)), 'nphm_mc_heads_emit')
        return verts, tris, pairs


NPHM_ERR_CAPACITY = -4


class SparseNarrowBand:
    """The band of :class:`NarrowBand` with block-sparse storage (``nphm_band_sparse_*``, DESIGN §4.17): per block a state byte and
    a brick slot, per block corner a value, and a brick of ``(block+1)^3`` voxels for each active block only, in a pool that grows
    between rounds.  Same steps and attributes as :class:`NarrowBand`; :meth:`volume` returns the band itself, the store every step
    and :func:`sparse_marching_cubes_count` take, and :meth:`dense_volume` materialises the filled slab volume (small grids)."""

    def __init__(self, res: int, block: int, device, l0: int = 0, l1: Optional[int] = None, slots: Optional[int] = None):
        self.res, self.block = int(res), int(block)
        self.device = torch.device(device)
        self.blocks_per_axis = -(-(self.res - 1) // max(self.block, 1))
        self.l0 = int(l0)
        self.l1 = self.blocks_per_axis if l1 is None else int(l1)
        self._geo = (self.res, self.block, self.l0, self.l1)
        with torch.cuda.device(self.device):
            self.ws = _workspace(lib().nphm_band_sparse_workspace_bytes(*self._geo), 'nphm_band_sparse_workspace_bytes', self.device)
        self.active_blocks = 0
        self.x0 = self.l0 * self.block
        self.x1 = min(self.l1 * self.block, self.res - 1)
        self.ghost = self.l0 > 0
        self.first_plane = self.x0 - int(self.ghost)
        self.n_planes = self.x1 + 1 - self.first_plane
        self.plane_bytes = 5 * self.res * self.res
        self.brick_voxels = (self.block + 1) ** 3
        self.n_blocks = (self.l1 - self.l0) * self.blocks_per_axis ** 2
        self.slots_used = 0
        self.mc_bytes = 0                 # marching-cubes workspace of the last mesh
        self.native_syncs = 0             # count read-backs (stream synchronisations) of the native calls so far
        # list entries slot (block+1)^3 + local are u32: the pool never holds more bricks than that allows
        self.max_slots = min(self.n_blocks, ((1 << 32) - 1) // self.brick_voxels)
        # a surface crosses about as many blocks per layer as a layer has rows; the pool grows when the band needs more
        self._pool_tensors = None
        self._set_pool(min(self.max_slots, max(64, 4 * (self.l1 - self.l0) * self.blocks_per_axis)) if slots is None else int(slots))

    def _set_pool(self, slots: int, keep: int = 0):
        sizes = (c_longlong * 3)()
        check(lib().nphm_band_sparse_pool_sizes(*self._geo, int(slots), sizes), 'nphm_band_sparse_pool_sizes')
        marks_bytes, list_len, n_chunks = sizes[0], sizes[1], sizes[2]
        V, dev = self.brick_voxels, self.device
        old = self._pool_tensors
        if old is not None:                # release the scratch of the old pool before allocating the new one
            old = old[:3]
            self._pool_tensors = None
        vals = torch.empty(slots * V, device=dev, dtype=torch.float32)
        marks = torch.zeros(marks_bytes, device=dev, dtype=torch.uint8)
        blocks = torch.empty(max(slots, 1), device=dev, dtype=torch.int32)
        if old is not None and keep:
            vals[:keep * V].copy_(old[0][:keep * V])
            marks[:keep * V].copy_(old[1][:keep * V])
            blocks[:keep].copy_(old[2][:keep])
        del old
        lst = torch.empty(max(list_len, 1), device=dev, dtype=torch.int32)
        cnt = torch.empty(n_chunks, device=dev, dtype=torch.int32)
        off = torch.empty(n_chunks, device=dev, dtype=torch.int32)
        self._pool_tensors = (vals, marks, blocks, lst, cnt, off)
        self.pool = BandPool(vals.data_ptr() if slots else blocks.data_ptr(), marks.data_ptr(), blocks.data_ptr(), lst.data_ptr(),
                             cnt.data_ptr(), off.data_ptr(), int(slots), marks_bytes, list_len, n_chunks)
        self.slots = int(slots)

    def device_bytes(self) -> int:
        """Bytes the band holds on the device: workspace (block states and slots, corners, shared planes) and brick pool."""
        return self.ws.numel() + sum(t.numel() * t.element_size() for t in self._pool_tensors)

    def _mem(self):
        return self.ws.data_ptr(), self.ws.numel(), byref(self.pool)

    def _call(self, step, *args):
        with torch.cuda.device(self.device):
            check(getattr(lib(), 'nphm_band_sparse_' + step)(*self._geo, *args, _stream_ptr(self.device)), 'nphm_band_sparse_' + step)

    def _call_listing(self, step, *before):
        fn = getattr(lib(), 'nphm_band_sparse_' + step)
        counts = (c_longlong * 4)()
        with torch.cuda.device(self.device):
            while True:
                rc = fn(*self._geo, *before, *self._mem(), counts, _stream_ptr(self.device))
                self.native_syncs += 1
                if rc != NPHM_ERR_CAPACITY or counts[3] <= self.slots or counts[3] > self.max_slots:
                    break
                # the step wrote nothing past the pool and left the band as it was: grow the pool, keep the bricks, repeat
                self._set_pool(min(self.max_slots, max(int(counts[3]), 2 * self.slots)), keep=int(counts[2]))
            if rc == NPHM_ERR_CAPACITY and counts[3] > self.max_slots:
                raise NativeError('nphm_band_sparse_%s: the band needs %d bricks of %d voxels; list entries are u32, so a pool holds at '
                                  'most %d' % (step, counts[3], self.brick_voxels, self.max_slots))
            check(rc, 'nphm_band_sparse_' + step)
        self.active_blocks = counts[1]
        self.slots_used = counts[2]
        return counts[0]

    def _own(self, vol):
        if vol is not self:
            raise ValueError('SparseNarrowBand: the volume of a sparse band is the band itself (volume())')

    def begin(self, quirk_period: int = 0) -> int:
        return self._call_listing('begin', int(quirk_period))

    def corners(self) -> int:
        return self._call_listing('corners')

    def classify(self, tau: float, vol) -> int:
        self._own(vol)
        return self._call_listing('classify', float(tau))

    def grow(self, vol) -> int:
        self._own(vol)
        return self._call_listing('grow')

    def gather(self, n: int, mini, maxi) -> torch.Tensor:
        xyz = torch.empty(int(n), 3, device=self.device, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        self._call('gather', gmin, gmax, int(n), _ptr(xyz) if n else None, *self._mem())
        return xyz

    def scatter(self, values: torch.Tensor, vol):
        self._own(vol)
        v = _f32c(values).reshape(-1)
        self._call('scatter', v.numel(), v.data_ptr() if v.numel() else None, *self._mem())

    def fill(self, vol):
        self._own(vol)
        self._call('fill', *self._mem())

    def block_states(self) -> torch.Tensor:
        nb = self.blocks_per_axis
        out = torch.empty(self.l1 - self.l0, nb, nb, device=self.device, dtype=torch.uint8)
        self._call('block_states', *self._mem(), out.data_ptr())
        return out != 0

    def volume(self):
        return self

    def planes(self, x_first: int, n_planes: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Filled planes ``[x_first, x_first + n_planes)`` of the slab (ghost plane included) as an (n, res, res) float32 tensor."""
        if out is None:
            out = torch.empty(int(n_planes), self.res, self.res, device=self.device, dtype=torch.float32)
        self._call('volume', int(x_first), int(n_planes), out.data_ptr(), *self._mem())
        return out

    def dense_volume(self) -> torch.Tensor:
        """The filled (n_planes, res, res) slab volume the dense band holds: res^3 floats for the whole grid (small grids only)."""
        return self.planes(self.first_plane, self.n_planes)

    def export(self, plane: int, vol, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        self._own(vol)
        buf = torch.empty(self.plane_bytes, device=self.device, dtype=torch.uint8) if out is None else out
        self._call('export', int(plane), *self._mem(), buf.data_ptr())
        return buf

    def import_(self, plane: int, buf: torch.Tensor, vol):
        self._own(vol)
        if buf.device != self.device or buf.dtype != torch.uint8 or buf.numel() != self.plane_bytes:
            raise ValueError('SparseNarrowBand.import_: need a uint8 buffer of %d bytes on %s' % (self.plane_bytes, self.device))
        self._call('import', int(plane), buf.data_ptr(), *self._mem())


def sparse_marching_cubes_count(band: SparseNarrowBand, iso=0.0, negate=False, x_global0=0, ghost_lo=False):
    """:func:`marching_cubes_count` of the filled slab volume of a sparse band (``nphm_band_sparse_mc_count``), reading only its
    bricks: ``(n_verts, n_tris, None, workspace)`` for :func:`sparse_marching_cubes_emit`.  The band's volume is ``-sdf`` at 0, as
    the narrow band extracts it: ``negate`` must be true and ``iso`` 0."""
    if x_global0 != band.first_plane or bool(ghost_lo) != band.ghost:
        raise ValueError('sparse_marching_cubes_count: the slab starts at plane %d (ghost plane: %s)' % (band.first_plane, band.ghost))
    if not negate or float(iso) != 0.0:
        raise ValueError('sparse_marching_cubes_count: the band extracts the 0 level set of -sdf (negate=True, iso=0)')
    with torch.cuda.device(band.device):
        ws = _workspace(lib().nphm_band_sparse_mc_workspace_bytes(*band._geo, band.slots), 'nphm_band_sparse_mc_workspace_bytes',
                        band.device)
        band.mc_bytes = ws.numel()
        nv, nt = c_longlong(0), c_longlong(0)
        band.native_syncs += 1
        check(lib().nphm_band_sparse_mc_count(*band._geo, *band._mem(), ws.data_ptr(), ws.numel(), byref(nv), byref(nt),
                                              _stream_ptr(band.device)), 'nphm_band_sparse_mc_count')
    return nv.value, nt.value, None, ws


def sparse_marching_cubes_emit(band: SparseNarrowBand, params, ws, n_verts: int, n_tris: int, vert_id_base: int):
    """:func:`marching_cubes_emit` for :func:`sparse_marching_cubes_count`: (verts, tris) with the ids the whole volume gives."""
    dev = band.device
    verts = torch.empty(n_verts, 3, device=dev, dtype=torch.float64)
    tris = torch.empty(n_tris, 3, device=dev, dtype=torch.int64)
    if n_verts or n_tris:
        with torch.cuda.device(dev):
            check(lib().nphm_band_sparse_mc_emit(*band._geo, *band._mem(), ws.data_ptr(), ws.numel(), int(vert_id_base), verts.data_ptr(),
                                                 tris.data_ptr(), _stream_ptr(dev)), 'nphm_band_sparse_mc_emit')
    return verts, tris


class SparseNarrowBandHeads:
    """The band of :class:`SparseNarrowBand` on the whole ``res^3`` grid for ``n_heads`` heads in lockstep
    (``nphm_band_sparse_heads_*``, DESIGN §4.21), with the interface of :class:`NarrowBandHeads`: each listing step is one launch
    sequence and one count read-back for all heads (:attr:`readbacks` counts the synchronising calls), :meth:`gather` /
    :meth:`scatter` move ``S x n_pad`` head-major rows, and :meth:`marching_cubes` meshes every head with one count read-back.
    Each head keeps a frame (block states and slots, corners) and a brick pool; the S pools are of one size, in one allocation per
    buffer, and grow together: when a step finds a pool short, no head changes, every pool grows (keeping the used bricks) and the
    step repeats.  :meth:`volumes` returns the band itself, the store every step takes.  Every head's state and mesh are those of a
    :class:`SparseNarrowBand` of the whole grid driven through the same steps."""

    def __init__(self, res: int, block: int, device, n_heads: int, slots: Optional[int] = None):
        self.res, self.block, self.n_heads = int(res), int(block), int(n_heads)
        self.device = torch.device(device)
        self.blocks_per_axis = -(-(self.res - 1) // max(self.block, 1))
        self._geo = (self.res, self.block, self.n_heads)
        self._slab = (self.res, self.block, 0, self.blocks_per_axis)
        with torch.cuda.device(self.device):
            self.ws = _workspace(lib().nphm_band_sparse_heads_workspace_bytes(*self._geo), 'nphm_band_sparse_heads_workspace_bytes',
                                 self.device)
        self.brick_voxels = (self.block + 1) ** 3
        self.n_blocks = self.blocks_per_axis ** 3
        self.active_blocks = [0] * self.n_heads
        self.slots_used = [0] * self.n_heads
        self.readbacks = 0                # stream synchronisations of the listing steps and marching cubes so far
        self.mc_bytes = 0                 # marching-cubes workspace of the last mesh
        # list entries slot (block+1)^3 + local are u32 within each head's pool
        self.max_slots = min(self.n_blocks, ((1 << 32) - 1) // self.brick_voxels)
        self._pool_tensors = None
        self._set_pool(self.default_slots(self.res, self.block) if slots is None else int(slots))

    @staticmethod
    def default_slots(res: int, block: int) -> int:
        """Bricks each head's pool starts with, as :class:`SparseNarrowBand` (a surface crosses about as many blocks per layer as a
        layer has rows); the pools grow when the band needs more."""
        nb = -(-(int(res) - 1) // max(int(block), 1))
        return min(nb ** 3, ((1 << 32) - 1) // (int(block) + 1) ** 3, max(64, 4 * nb * nb))

    @staticmethod
    def device_bytes_per_head(res: int, block: int, slots: Optional[int] = None) -> int:
        """Device bytes one head holds at the start: its frame (block states and slots, corner values and marks), its brick pool of
        ``slots`` bricks (default :meth:`default_slots`) with the list and compaction scratch, and its marching-cubes workspace."""
        L = lib()
        res, block = int(res), int(block)
        slots = SparseNarrowBandHeads.default_slots(res, block) if slots is None else int(slots)
        frame = L.nphm_band_sparse_heads_workspace_bytes(res, block, 2) - L.nphm_band_sparse_heads_workspace_bytes(res, block, 1)
        mc = L.nphm_band_sparse_heads_mc_workspace_bytes(res, block, 2, slots) - L.nphm_band_sparse_heads_mc_workspace_bytes(res, block, 1, slots)
        nb = -(-(res - 1) // max(block, 1))
        sizes = (c_longlong * 3)()
        if frame < 0 or mc < 0 or L.nphm_band_sparse_pool_sizes(res, block, 0, nb, slots, sizes) != 0:
            check(-1, 'nphm_band_sparse_heads_workspace_bytes')
        pool = slots * (block + 1) ** 3 * 4 + sizes[0] + 4 * max(slots, 1) + 4 * max(sizes[1], 1) + 8 * sizes[2]
        return int(frame + pool + mc)

    def _set_pool(self, slots: int, keep: int = 0):
        sizes = (c_longlong * 3)()
        check(lib().nphm_band_sparse_pool_sizes(*self._slab, int(slots), sizes), 'nphm_band_sparse_pool_sizes')
        marks_bytes, list_len, n_chunks = sizes[0], sizes[1], sizes[2]
        S, V, dev = self.n_heads, self.brick_voxels, self.device
        old = self._pool_tensors
        if old is not None:                # release the scratch of the old pools before allocating the new ones
            old = old[:3]
            self._pool_tensors = None
        vals = torch.empty(S, slots * V, device=dev, dtype=torch.float32)
        marks = torch.zeros(S, marks_bytes, device=dev, dtype=torch.uint8)
        blocks = torch.empty(S, max(slots, 1), device=dev, dtype=torch.int32)
        if old is not None and keep:       # every head's used bricks, at the same place in its new pool
            vals[:, :keep * V].copy_(old[0][:, :keep * V])
            marks[:, :keep * V].copy_(old[1][:, :keep * V])
            blocks[:, :keep].copy_(old[2][:, :keep])
        del old
        lst = torch.empty(S, max(list_len, 1), device=dev, dtype=torch.int32)
        cnt = torch.empty(S, n_chunks, device=dev, dtype=torch.int32)
        off = torch.empty(S, n_chunks, device=dev, dtype=torch.int32)
        self._pool_tensors = (vals, marks, blocks, lst, cnt, off)
        # the native side steps from one head's pool to the next by these sizes: the rows above
        self.pool = BandPool(vals.data_ptr() if slots else blocks.data_ptr(), marks.data_ptr(), blocks.data_ptr(), lst.data_ptr(),
                             cnt.data_ptr(), off.data_ptr(), int(slots), marks_bytes, max(list_len, 1), n_chunks)
        self.slots = int(slots)

    def device_bytes(self) -> int:
        """Bytes the band holds on the device: the workspace (record and every head's frame) and the S brick pools."""
        return self.ws.numel() + sum(t.numel() * t.element_size() for t in self._pool_tensors)

    def _mem(self):
        return self.ws.data_ptr(), self.ws.numel(), byref(self.pool)

    def _call(self, step, *args):
        with torch.cuda.device(self.device):
            check(getattr(lib(), 'nphm_band_sparse_heads_' + step)(*self._geo, *args, _stream_ptr(self.device)),
                  'nphm_band_sparse_heads_' + step)

    def _call_listing(self, step, *before):
        fn = getattr(lib(), 'nphm_band_sparse_heads_' + step)
        S = self.n_heads
        counts = (c_longlong * (4 * S))()
        with torch.cuda.device(self.device):
            while True:
                rc = fn(*self._geo, *before, *self._mem(), counts, _stream_ptr(self.device))
                self.readbacks += 1
                need = max(counts[4 * h + 3] for h in range(S))
                if rc != NPHM_ERR_CAPACITY or need <= self.slots or need > self.max_slots:
                    break
                # no head changed and nothing was listed: grow every pool, keep the used bricks, repeat the same step
                self._set_pool(min(self.max_slots, max(int(need), 2 * self.slots)), keep=max(counts[4 * h + 2] for h in range(S)))
            if rc == NPHM_ERR_CAPACITY and need > self.max_slots:
                raise NativeError('nphm_band_sparse_heads_%s: a head needs %d bricks of %d voxels; list entries are u32, so a pool '
                                  'holds at most %d' % (step, need, self.brick_voxels, self.max_slots))
            check(rc, 'nphm_band_sparse_heads_' + step)
        self.active_blocks = [counts[4 * h + 1] for h in range(S)]
        self.slots_used = [counts[4 * h + 2] for h in range(S)]
        return [counts[4 * h] for h in range(S)]

    def _own(self, vols):
        if vols is not self:
            raise ValueError('SparseNarrowBandHeads: the volumes of a sparse band are the band itself (volumes())')

    def begin(self, quirk_period: int = 0):
        """Reset every head; with ``quirk_period > 0`` list the eval-mode quirk voxels (the same for every head)."""
        return self._call_listing('begin', int(quirk_period))

    def corners(self):
        return self._call_listing('corners')

    def classify(self, tau: float, vols):
        self._own(vols)
        return self._call_listing('classify', float(tau))

    def grow(self, vols):
        self._own(vols)
        return self._call_listing('grow')

    def gather(self, n_pad: int, mini, maxi) -> torch.Tensor:
        """(S, n_pad, 3) float32 coordinates: each head's listed voxels, then padding rows that repeat one of them."""
        xyz = torch.empty(self.n_heads, int(n_pad), 3, device=self.device, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        self._call('gather', gmin, gmax, int(n_pad), _ptr(xyz) if n_pad else None, *self._mem())
        return xyz

    def scatter(self, values: torch.Tensor, vols):
        """values (S, n_pad) in the layout of :meth:`gather`: each head's listed rows into its bricks, the padding dropped."""
        self._own(vols)
        v = _f32c(values).reshape(self.n_heads, -1)
        n_pad = v.shape[1]
        self._call('scatter', n_pad, v.data_ptr() if n_pad else None, *self._mem())

    def fill(self, vols):
        self._own(vols)
        self._call('fill', *self._mem())

    def block_states(self) -> torch.Tensor:
        """(S, blocks, blocks, blocks) bool: which blocks of each head are active."""
        nb = self.blocks_per_axis
        out = torch.empty(self.n_heads, nb, nb, nb, device=self.device, dtype=torch.uint8)
        self._call('block_states', *self._mem(), out.data_ptr())
        return out != 0

    def volumes(self):
        return self

    def marching_cubes(self, vols):
        """Marching cubes on every head's bricks (``nphm_band_sparse_heads_mc_count`` / ``_emit``): ``(verts (V, 3) float64, tris
        (T, 3) int64, counts)`` as :meth:`NarrowBandHeads.marching_cubes` gives them, head h's part what
        :func:`sparse_marching_cubes_count` / :func:`sparse_marching_cubes_emit` give for that head alone."""
        self._own(vols)
        L = lib()
        with torch.cuda.device(self.device):
            ws = _workspace(L.nphm_band_sparse_heads_mc_workspace_bytes(*self._geo, self.slots), 'nphm_band_sparse_heads_mc_workspace_bytes',
                            self.device)
            self.mc_bytes = ws.numel()
            counts = (c_longlong * (2 * self.n_heads))()
            check(L.nphm_band_sparse_heads_mc_count(*self._geo, *self._mem(), ws.data_ptr(), ws.numel(), counts,
                                                    _stream_ptr(self.device)), 'nphm_band_sparse_heads_mc_count')
            self.readbacks += 1
            pairs = [(counts[2 * h], counts[2 * h + 1]) for h in range(self.n_heads)]
            verts = torch.empty(sum(c[0] for c in pairs), 3, device=self.device, dtype=torch.float64)
            tris = torch.empty(sum(c[1] for c in pairs), 3, device=self.device, dtype=torch.int64)
            if verts.shape[0] or tris.shape[0]:
                check(L.nphm_band_sparse_heads_mc_emit(*self._geo, *self._mem(), ws.data_ptr(), ws.numel(), verts.data_ptr(),
                                                       tris.data_ptr(), _stream_ptr(self.device)), 'nphm_band_sparse_heads_mc_emit')
        return verts, tris, pairs
