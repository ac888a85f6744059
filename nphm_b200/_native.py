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
    'nphm_broyden_workspace_bytes', 'nphm_mlp_broyden_search', 'nphm_nearest_neighbors',
    'nphm_mlp_train_workspace_bytes', 'nphm_mlp_train_forward', 'nphm_mlp_train_backward',
    'nphm_mlp_sdfgrad_workspace_bytes', 'nphm_mlp_sdfgrad_forward', 'nphm_mlp_sdfgrad_backward',
    'nphm_mlp_fit_workspace_bytes', 'nphm_mlp_fit_surface_grad', 'nphm_mlp_fit_surface_grad_batched',
    'nphm_ensemble_sdfgrad_workspace_bytes', 'nphm_ensemble_sdfgrad_forward', 'nphm_ensemble_sdfgrad_backward',
    'nphm_render_workspace_bytes', 'nphm_render_depth_normals',
    'nphm_band_workspace_bytes', 'nphm_band_begin', 'nphm_band_corners', 'nphm_band_gather', 'nphm_band_scatter',
    'nphm_band_classify', 'nphm_band_grow', 'nphm_band_fill', 'nphm_band_block_states',
)


class NativeError(RuntimeError):
    pass


# kernels of this library launched per call (ncu launch lists under profiles/); bench.py counts its launches with these
MC_LAUNCHES = 3                      # classify rows, scan rows, emit rows


def launches_per_grid_query(impl='auto') -> int:
    """grid axes, anchors, folded constants, [tensor-core records, tile member masks], ensemble kernel."""
    return 4 + (2 if impl in ('auto', 'tc', 'tc_pruned') else 0)


class EnsembleConfig(Structure):
    _fields_ = [('n_loc', c_int), ('n_symm_pairs', c_int), ('lat_dim_glob', c_int), ('lat_dim_loc', c_int),
                ('hidden_dim', c_int), ('n_layers', c_int), ('pos_mlp_dim', c_int)]


class MlpConfig(Structure):
    _fields_ = [('lat_dim', c_int), ('hidden_dim', c_int), ('n_layers', c_int), ('out_dim', c_int)]


class McParams(Structure):
    _fields_ = [('nx', c_int), ('ny', c_int), ('nz', c_int), ('x_global0', c_int), ('ghost_lo', c_int),
                ('negate', c_int), ('iso', c_double)]


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
    L.nphm_band_workspace_bytes.argtypes = [c_int, c_int]
    L.nphm_band_workspace_bytes.restype = c_longlong
    L.nphm_band_begin.argtypes = [c_int, c_int, c_longlong, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_corners.argtypes = [c_int, c_int, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_gather.argtypes = [c_int, c_int, POINTER(c_double), POINTER(c_double), c_longlong, c_void_p, c_void_p, c_longlong,
                                   c_void_p]
    L.nphm_band_scatter.argtypes = [c_int, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_classify.argtypes = [c_int, c_int, c_float, c_void_p, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_grow.argtypes = [c_int, c_int, c_void_p, c_void_p, c_longlong, POINTER(c_longlong), c_void_p]
    L.nphm_band_fill.argtypes = [c_int, c_int, c_void_p, c_void_p, c_longlong, c_void_p]
    L.nphm_band_block_states.argtypes = [c_int, c_int, c_void_p, c_longlong, c_void_p, c_void_p]
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
        # forward-deformation backbone to the tensor cores; every other shape runs layer by layer on the generic wgmma linear layer
        # (csrc/tc_linear.cu, any width - e.g. the NPM baseline 515 -> 1024 x 8); the fp32 FFMA kernel is kept for impl='simt'
        self.fused_shape = (hidden == 512 and self.n_lin == 7 and module.lat_dim == 232 and module.out_dim_net == 3)
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
                       early_exit: bool = True):
        """Roots of ``x + F(x; cond) - obs`` by the reference's Broyden iteration, entirely on the device.
        obs, x_init: B x N x 3, cond: B x lat_dim, J_inv_init: B x N x 3 x 3.
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
            ws = torch.empty(max(int(lib().nphm_broyden_workspace_bytes(B * N)), 256), device=dev, dtype=torch.uint8)
            check(lib().nphm_mlp_broyden_search(self._h, cond.data_ptr(), B, N, obs.data_ptr(), x.data_ptr(),
                                                jinv.data_ptr(), int(max_steps), float(cvg_thresh), float(dvg_thresh),
                                                float(eps), diff.data_ptr(), valid.data_ptr(),
                                                byref(steps) if early_exit else None,       # None: no host sync, all steps run
                                                ws.data_ptr(), _stream_ptr(dev)), 'nphm_mlp_broyden_search')
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
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError('face indices must lie in [0, %d) (got [%d, %d])' % (v.shape[0], int(f.min()), int(f.max())))
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


# ------------------------------------------------------------------------------------------ narrow-band extraction
class NarrowBand:
    """Band state of one ``res^3`` grid in blocks of ``block^3`` cells (``nphm_band_*``, DESIGN §4.13) in a workspace this object
    owns.  The listing steps return the number of voxels they listed; :meth:`gather` / :meth:`scatter` move the listed voxels'
    coordinates out and their values into a ``res^3`` float32 CUDA volume."""

    def __init__(self, res: int, block: int, device):
        self.res, self.block = int(res), int(block)
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            self.ws = _workspace(lib().nphm_band_workspace_bytes(self.res, self.block), 'nphm_band_workspace_bytes', self.device)
        self.blocks_per_axis = -(-(self.res - 1) // self.block)
        self.active_blocks = 0

    def _call_listing(self, name, *before_ws):
        counts = (c_longlong * 2)()
        with torch.cuda.device(self.device):
            check(getattr(lib(), name)(self.res, self.block, *before_ws, self.ws.data_ptr(), self.ws.numel(), counts,
                                       _stream_ptr(self.device)), name)
        self.active_blocks = counts[1]
        return counts[0]

    def begin(self, quirk_period: int = 0) -> int:
        """Reset; with ``quirk_period > 0`` list the eval-mode quirk voxels and activate the blocks around them."""
        return self._call_listing('nphm_band_begin', int(quirk_period))

    def corners(self) -> int:
        return self._call_listing('nphm_band_corners')

    def classify(self, tau: float, vol: torch.Tensor) -> int:
        return self._call_listing('nphm_band_classify', float(tau), vol.data_ptr())

    def grow(self, vol: torch.Tensor) -> int:
        return self._call_listing('nphm_band_grow', vol.data_ptr())

    def gather(self, n: int, mini, maxi) -> torch.Tensor:
        """(n, 3) float32 coordinates of the first ``n`` listed voxels."""
        xyz = torch.empty(int(n), 3, device=self.device, dtype=torch.float32)
        gmin = (c_double * 3)(*[float(v) for v in mini])
        gmax = (c_double * 3)(*[float(v) for v in maxi])
        with torch.cuda.device(self.device):
            check(lib().nphm_band_gather(self.res, self.block, gmin, gmax, int(n), _ptr(xyz) if n else None, self.ws.data_ptr(),
                                         self.ws.numel(), _stream_ptr(self.device)), 'nphm_band_gather')
        return xyz

    def scatter(self, values: torch.Tensor, vol: torch.Tensor):
        v = _f32c(values).reshape(-1)
        with torch.cuda.device(self.device):
            check(lib().nphm_band_scatter(self.res, self.block, v.numel(), v.data_ptr() if v.numel() else None, vol.data_ptr(),
                                          self.ws.data_ptr(), self.ws.numel(), _stream_ptr(self.device)), 'nphm_band_scatter')

    def fill(self, vol: torch.Tensor):
        with torch.cuda.device(self.device):
            check(lib().nphm_band_fill(self.res, self.block, vol.data_ptr(), self.ws.data_ptr(), self.ws.numel(),
                                       _stream_ptr(self.device)), 'nphm_band_fill')

    def block_states(self) -> torch.Tensor:
        """(blocks, blocks, blocks) bool: which blocks are active."""
        nb = self.blocks_per_axis
        out = torch.empty(nb, nb, nb, device=self.device, dtype=torch.uint8)
        with torch.cuda.device(self.device):
            check(lib().nphm_band_block_states(self.res, self.block, self.ws.data_ptr(), self.ws.numel(), out.data_ptr(),
                                               _stream_ptr(self.device)), 'nphm_band_block_states')
        return out != 0
