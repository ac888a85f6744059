"""Drop-in mirror of the reference module ``NPHM.models.fitting``.

  * ``inference_identity_space``                 src/NPHM/models/fitting.py:180-285
  * ``inference_iterative_root_finding_joint``   src/NPHM/models/fitting.py:14-177

``inference_identity_space`` runs on the fused fitting kernels (``nphm_fit_identity_step``: forward, clamped |sdf|
loss, analytic latent gradient and Adam in five launches, no autograd graph) when the decoder is a
``FastEnsembleDeepSDFMirrored`` on a CUDA device; otherwise it falls back to autograd through the composite modules,
written here independently but following the same loop.  With a ``DeepSDF`` decoder (the NPM baseline of
scripts/configs/fitting_npm.yaml) on CUDA both fitters run natively as well (:class:`NpmIdentityFitter`,
:class:`NpmJointFitter`).  Host-side behaviour kept from the reference: the
point sampling draws from torch's global CPU generator in the same order (``torch.randint`` at :214,:219), the
``lambdas`` dict is mutated by the schedule (:199-206), Adam runs with lr 0.01*lr_scale halved by the schedule, and the
returned anchors are those of the LAST iteration's pre-update latent (:211).
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List

import torch
from torch import optim

from .. import _native
from .EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
from .iterative_root_finding import search, nabla          # noqa: F401  (same names as the reference imports)
from .diff_operators import gradient, jac                    # noqa: F401

NUM_OBSERVATIONS_PER_BATCH = 5
NUM_POINTS_PER_OBSERVATION = 1000


def _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr):
    """Eye-balled schedule of the reference (:199-206 / :40-52): divides lr and lambdas at fixed iterations."""
    key = int(j / step_scale)
    if key in schedule_cfg.get('lr', {}):
        lr = lr / schedule_cfg['lr'][key]
    for cfg_key, lam_key in (('symm_dist', 'symm_dist'), ('reg_glob', 'reg_global'), ('reg_loc', 'reg_loc'),
                             ('reg_expr', 'reg_expr')):
        if cfg_key in schedule_cfg and key in schedule_cfg[cfg_key] and (lam_key in lambdas or cfg_key != 'reg_expr'):
            lambdas[lam_key] /= schedule_cfg[cfg_key][key]
    return lr


def _clamp_for_iteration(j, step_scale):
    """Sequential strict filters l<0.1, (j>250) l<0.05, (j>500) l<0.0075 collapse to one threshold (:239-246)."""
    clamp = 0.1
    if j > int(250 * step_scale):
        clamp = 0.05
    if j > int(500 * step_scale):
        clamp = 0.0075
    return clamp


def _sample_indices(sizes, generator=None):
    """The draws of one iteration's sampling (:214-222): which observations, and which points of each.  ``generator=None``:
    torch's global CPU generator, as in the reference."""
    sampled_observations_idx = torch.randint(0, len(sizes), [NUM_OBSERVATIONS_PER_BATCH], generator=generator)
    subsample_idx = []
    for i in range(NUM_OBSERVATIONS_PER_BATCH):
        n = sizes[int(sampled_observations_idx[i])]
        subsample_idx.append(torch.randint(0, n, [min(NUM_POINTS_PER_OBSERVATION, n)], generator=generator))
    return sampled_observations_idx, subsample_idx


def _sample_observations(all_obs, generator=None):
    """Reference sampling order on the global CPU generator (:214-222), or on ``generator``."""
    sampled_observations_idx, subsample_idx = _sample_indices([o.shape[0] for o in all_obs], generator)
    sampled_points = []
    for i in range(NUM_OBSERVATIONS_PER_BATCH):
        obs = all_obs[sampled_observations_idx[i]]
        sampled_points.append(obs[subsample_idx[i].to(obs.device), :])
    return torch.stack(sampled_points, dim=0), sampled_observations_idx


def _current_anchors(decoder, lat_rep_shape, device):
    """Anchors of the current identity code, with graph.  The reference evaluates the whole decoder on a dummy point for
    this (fitting.py:57, :218); the drop-in ensemble exposes the anchor head directly (same values, ~50 launches less)."""
    if isinstance(decoder, FastEnsembleDeepSDFMirrored):
        return decoder.predict_anchors(lat_rep_shape)
    return decoder(torch.zeros([1, 1, 3], device=device), lat_rep_shape, None)[1]


def _fused_identity(decoder, grad_points: bool = False) -> bool:
    """Whether the fused fitting kernels take this decoder on CUDA (see :func:`fused_fit_config`)."""
    return (isinstance(decoder, FastEnsembleDeepSDFMirrored) and next(decoder.parameters()).is_cuda
            and fused_fit_config(decoder, grad_points))


# The FFMA fitting step (csrc/fit.cu fit_step_impl) keeps 3 + H + (N1 + 3) + 3 H + 8 + 8 * 16 = 139 + 4 H - C rows of 64 fp32
# points (N1 = H - C - 3, C = lat_dim_glob + lat_dim_loc) in at most 227 KiB of shared memory.
FFMA_FIT_MAX_ROWS = 227 * 1024 // (64 * 4)


def ffma_fit_rows(hidden: int, cond: int) -> int:
    return 139 + 4 * hidden - cond


def fused_fit_config(decoder, grad_points: bool = False) -> bool:
    """Whether the fused fitting kernels take an ensemble of this configuration, in its current mode: exactly what the C
    entry points accept.  They need 4 hidden layers.  The tensor-core configuration (:func:`_tc_ensemble`) serves every entry
    point.  Any other width runs the FFMA step, which serves only the single-scan training-mode step without point gradients
    (``nphm_fit_identity_step``) and only within its shared memory (:data:`FFMA_FIT_MAX_ROWS`).  So the eval-mode quirk (the
    reference's forward overwrites every member's output at the last point of each decoder call, EnsembledDeepSDF.py:260-261)
    and ``grad_points`` (the joint fitter's surface term, ``nphm_ensemble_backward_inputs``) need the tensor-core
    configuration; anything the kernels do not take goes to the autograd path.  The reference runs its fitters in training
    mode (scripts/fitting/fitting_pointclouds.py:268 calls ``decoder_shape.train()`` first)."""
    if decoder.ensembled_deep_sdf.num_layers != 6:
        return False
    if _tc_ensemble(decoder):
        return True
    hidden = _native.hidden_width(decoder.ensembled_deep_sdf, 5)
    return (decoder.training and not grad_points
            and ffma_fit_rows(hidden, decoder.lat_dim_glob + decoder.lat_dim_loc) <= FFMA_FIT_MAX_ROWS)


def _quirk_period(decoder, points_per_call: int) -> int:
    """The quirk period of the fused calls: 0 in training mode, else the points of one reference decoder call."""
    return 0 if decoder.training else int(points_per_call)


class IdentityFitter:
    """Stateful wrapper around ``nphm_fit_identity_step``: latent + Adam moments live on the device."""

    def __init__(self, decoder: FastEnsembleDeepSDFMirrored, device):
        self.decoder = decoder
        self.device = device
        self.engine = decoder.engine()
        self.latent = torch.zeros(decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latent)
        self.v = torch.zeros_like(self.latent)
        self.loss_terms = torch.zeros(8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latent)
        self.t = 0

    def step(self, points: torch.Tensor, lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True):
        """One iteration on ``points`` (rows x n x 3: the reference's one decoder call on its sampled rows).  In eval mode the
        last point of every row carries the quirk (``nphm_fit_identity_step_quirk`` with period n)."""
        pts = points.reshape(-1, 3).to(dtype=torch.float32).contiguous()
        period = _quirk_period(self.decoder, points.shape[-2] if points.dim() > 1 else 1)
        if apply_update:
            self.t += 1
        fp = _native.FitParams(float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0)),
                               float(lambdas.get('reg_loc', 0.0)), float(lambdas.get('reg_unobserved', 0.0)),
                               float(lambdas.get('symm_dist', 0.0)), float(clamp), float(lr), max(self.t, 1))
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with torch.cuda.device(self.device):
            if period:
                _native.check(_native.lib().nphm_fit_identity_step_quirk(
                    self.engine.handle, pts.data_ptr(), pts.shape[0], period, self.latent.data_ptr(), self.m.data_ptr(),
                    self.v.data_ptr(), ctypes.byref(fp), int(apply_update), self.loss_terms.data_ptr(), self.grad.data_ptr(),
                    None, stream), 'nphm_fit_identity_step_quirk')
            else:
                _native.check(_native.lib().nphm_fit_identity_step(
                    self.engine.handle, pts.data_ptr(), pts.shape[0], self.latent.data_ptr(), self.m.data_ptr(),
                    self.v.data_ptr(), ctypes.byref(fp), int(apply_update), self.loss_terms.data_ptr(),
                    self.grad.data_ptr(), None, stream),
                    'nphm_fit_identity_step')


class _FusedSurfaceLoss(torch.autograd.Function):
    """``sdf = decoder(xc, z_id); sdf[valid].abs()[< clamp].mean()`` of the joint fitter (reference fitting.py:114-125) as
    one native call (`nphm_fit_surface_grad`): tensor-core forward, analytic backward w.r.t. the identity code (member
    inputs, anchors, blend weights) and w.r.t. the query points.  Autograd continues from the point gradient into the
    implicit-differentiation correction and the deformation network.  In eval mode the last point of every row of ``xc``
    (rows x n x 3, one decoder call in the reference) carries the quirk (``nphm_fit_surface_grad_quirk``, period n)."""

    @staticmethod
    def forward(ctx, xc, lat_rep_shape, valid, clamp, decoder):
        dev = xc.device
        pts = xc.detach().reshape(-1, 3).to(torch.float32).contiguous()
        lat = lat_rep_shape.detach().reshape(-1).to(torch.float32).contiguous()
        mask = valid.reshape(-1).to(torch.uint8).contiguous()
        eng = decoder.engine()
        terms = torch.empty(8, device=dev, dtype=torch.float32)
        g_lat = torch.empty_like(lat)
        g_pts = torch.empty_like(pts)
        period = _quirk_period(decoder, xc.shape[-2])
        _surface_grad(eng, pts, period, lat, mask, clamp, terms, g_lat, g_pts, torch.cuda.current_stream(dev).cuda_stream)
        ctx.save_for_backward(g_lat, g_pts)
        ctx.shapes = (xc.shape, lat_rep_shape.shape)
        return terms[0].clone()

    @staticmethod
    def backward(ctx, grad_out):
        g_lat, g_pts = ctx.saved_tensors
        return grad_out * g_pts.reshape(ctx.shapes[0]), grad_out * g_lat.reshape(ctx.shapes[1]), None, None, None


def _surface_grad(eng, pts, period, lat, mask, clamp, terms, g_lat, g_pts, stream):
    """``nphm_fit_surface_grad`` on ``pts`` (n x 3), or its eval-mode form with quirk period ``period`` > 0."""
    lib = _native.lib()
    with torch.cuda.device(pts.device):
        if period:
            _native.check(lib.nphm_fit_surface_grad_quirk(eng.handle, pts.data_ptr(), pts.shape[0], period, lat.data_ptr(),
                                                          mask.data_ptr(), float(clamp), terms.data_ptr(), g_lat.data_ptr(),
                                                          g_pts.data_ptr(), None, stream), 'nphm_fit_surface_grad_quirk')
        else:
            _native.check(lib.nphm_fit_surface_grad(eng.handle, pts.data_ptr(), pts.shape[0], lat.data_ptr(), mask.data_ptr(),
                                                    float(clamp), terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), None,
                                                    stream), 'nphm_fit_surface_grad')


def inference_identity_space(decoder,
                             all_obs: List[torch.Tensor],
                             lambdas,
                             n_steps,
                             schedule_cfg: Dict,
                             step_scale=1,
                             lr_scale=1):
    """Fit the identity code to point-cloud observations.  Returns ``(lat_rep_shape (1,1,D), anchors (1,K,3))``; a
    ``DeepSDF`` decoder has no anchors (``None``), as in the reference."""
    device = all_obs[0].device
    lr = 0.01 * lr_scale
    if device.type == 'cuda' and _native_npm_decoder(decoder, 1):
        fitter = NpmIdentityFitter(decoder, device)
        for j in range(int(n_steps * step_scale)):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs, _ = _sample_observations(all_obs)
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr)
        return fitter.latent.reshape(1, 1, -1).clone().requires_grad_(True), None
    if _fused_identity(decoder) and device.type == 'cuda':
        fitter = IdentityFitter(decoder, device)
        z_prev = fitter.latent.clone()
        for j in range(int(n_steps * step_scale)):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs, _ = _sample_observations(all_obs)
            z_prev.copy_(fitter.latent)
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr)
        with torch.no_grad():
            _, anchors = fitter.engine.query(torch.zeros(1, 1, 3, device=device), z_prev.reshape(1, -1), eval_quirk=False)
        lat_rep_shape = fitter.latent.reshape(1, 1, -1).clone().requires_grad_(True)
        return lat_rep_shape, anchors
    return _inference_identity_space_autograd(decoder, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)


def _inference_identity_space_autograd(decoder, all_obs, lambdas, n_steps, schedule_cfg, step_scale=1, lr_scale=1):
    """The composite path of :func:`inference_identity_space`: autograd through the modules (any decoder, CPU or GPU)."""
    device = all_obs[0].device
    lr = 0.01 * lr_scale
    lat_dim = decoder.lat_dim
    lat_rep_shape = torch.zeros([1, 1, lat_dim], device=device, requires_grad=True)
    opt = optim.Adam(params=[lat_rep_shape], lr=lr)
    anchors = None
    for j in range(int(n_steps * step_scale)):
        new_lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        if new_lr != lr:
            lr = new_lr
            for group in opt.param_groups:
                group['lr'] = lr
        opt.zero_grad()
        anchors = _current_anchors(decoder, lat_rep_shape, device)
        obs, _ = _sample_observations(all_obs)
        nb = obs.shape[0]
        if hasattr(decoder, 'lat_dim_loc'):
            sdf, _ = decoder(obs, lat_rep_shape.repeat(nb, 1, 1), None)
        else:
            sdf, _ = decoder(obs, lat_rep_shape.repeat(nb, obs.shape[1], 1), None)
        l = sdf.abs()
        l = l[l < _clamp_for_iteration(j, step_scale)]
        loss_dict = {'surface': l.mean()}
        loss_dict.update(_latent_regularisers(decoder, lat_rep_shape))
        loss = 0
        for k in lambdas.keys():
            loss = loss + loss_dict[k] * lambdas[k]
        loss.backward()
        opt.step()
    return lat_rep_shape, anchors


def _latent_regularisers(decoder, lat_rep_shape):
    """reg_loc / reg_global / reg_unobserved / symm_dist of the reference (:252-272)."""
    out = {}
    if hasattr(decoder, 'lat_dim_glob'):
        g, lc = decoder.lat_dim_glob, decoder.lat_dim_loc
        out['reg_loc'] = (torch.norm(lat_rep_shape[..., g:], dim=-1) ** 2).mean()
        out['reg_global'] = (torch.norm(lat_rep_shape[..., :g], dim=-1) ** 2).mean()
        ru = 0
        for idx in (30, 31, 39):
            ru = ru + torch.norm(lat_rep_shape[..., g + idx * lc:g + (idx + 1) * lc], dim=-1).square().mean()
        out['reg_unobserved'] = ru
        n_pairs = decoder.num_symm_pairs
        loc = lat_rep_shape[:, :, g:g + 2 * n_pairs * lc].view(lat_rep_shape.shape[0], n_pairs * 2, lc)
        out['symm_dist'] = torch.norm(loc[:, ::2, :] - loc[:, 1::2, :], dim=-1).mean()
    else:
        out['symm_dist'] = 0
        out['reg_unobserved'] = 0
        out['reg_loc'] = 0
        out['reg_global'] = (torch.norm(lat_rep_shape, dim=-1) ** 2).mean()
    return out


def _native_joint(decoder, decoder_expr, device) -> bool:
    """The autograd-free joint fitter applies to the shipped configuration: a fused identity ensemble (see
    :func:`_fused_identity`) and a 'compress' DeformationNetwork in eval mode on the same CUDA device."""
    from .deepSDF import DeformationNetwork
    if device.type != 'cuda' or not _fused_identity(decoder, grad_points=True) or not isinstance(decoder_expr, DeformationNetwork):
        return False
    if decoder_expr.training or decoder_expr.mode != 'compress':
        return False
    bb = decoder_expr.defDeepSDF
    return next(bb.parameters()).is_cuda and bb.num_freq_bands is None and bb.beta == 100 and bb.out_dim_net == 3


class JointFitter:
    """One iteration of ``inference_iterative_root_finding_joint`` (reference fitting.py:38-175) WITHOUT an autograd graph.

    The reference builds xc = p - J^-1 (F_ex(p; theta) + p - stopgrad(.)) so that value(xc) = p and d xc / d theta =
    -J^-1 dF_ex/d theta (:99-106), then calls loss.backward() (:167).  Written out:
        g_x   = d surface / d xc                                   nphm_fit_surface_grad (with d surface / d z_id)
        u     = -J^-T g_x            per point, J = I + dF_ex/dx    nphm_mlp_inverse_jacobian (forward-mode, tensor cores)
        g_c   = sum_n (dF_ex/d cond)^T u_n   per sampled scan       nphm_mlp_backward_inputs (adjoint pass, tensor cores)
        cond  = [compressor([z_id | anchors]) (32) | z_ex (200)]    -> z_ex rows, and through the compressor to z_id and the
                                                                      anchors (mlp_pos backward inside nphm_fit_apply_gradient)
    followed by the regularisers and the two Adam updates (nphm_fit_apply_gradient, nphm_adam_step)."""

    def __init__(self, decoder, decoder_expr, num_observations: int, device):
        self.dec, self.dfn, self.device = decoder, decoder_expr, device
        self.eng = decoder.engine()
        self.mlp = decoder_expr.defDeepSDF.engine()
        E = decoder_expr.lat_dim_expr
        self.z_id = torch.zeros(decoder.lat_dim, device=device)
        self.m_id, self.v_id = torch.zeros_like(self.z_id), torch.zeros_like(self.z_id)
        self.z_ex = torch.zeros(num_observations, E, device=device)
        self.m_ex, self.v_ex = torch.zeros_like(self.z_ex), torch.zeros_like(self.z_ex)
        self.terms = torch.zeros(8, device=device)
        self.loss_terms = torch.zeros(8, device=device)
        self.t = 0
        self.anchors = None
        # Broyden early exit (the reference leaves its loop when nobody is active) costs a host sync every third step; without it
        # an iteration is a pure launch sequence.  Default: on for small batches is not worth a sync - off.
        self.early_exit = bool(int(os.environ.get('NPHM_BROYDEN_EARLY_EXIT', '0')))

    def step(self, obs, obs_idx, lambdas, clamp, lr, apply_update: bool = True):
        """One iteration; with ``apply_update=False`` nothing is modified and ``(d loss / d z_id, d loss / d z_ex)`` - the
        tensors the reference hands to its two ``Adam.step()`` calls - are returned."""
        nat, dev = _native, self.device
        nb, n_point, _ = obs.shape
        E, D = self.z_ex.shape[1], self.z_id.shape[0]
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.no_grad(), torch.cuda.device(dev):
            anchors = self.eng.anchors(self.z_id[None])                                  # 1 x K x 3, pre-update code (:59)
            self.anchors = anchors
            # condition of the deformation backbone (deepSDF.py:218-219): compressor([z_id | anchors]) (32) | z_ex (E)
            lin = self.dfn.compressor[0] if isinstance(self.dfn.compressor, torch.nn.Sequential) else self.dfn.compressor
            Wc, bc = lin.weight, lin.bias
            first = torch.cat([self.z_id, anchors.reshape(-1)])
            c32 = (Wc * first[None, :]).sum(1) + bc
            cond = torch.cat([c32[None, :].expand(nb, -1), self.z_ex[obs_idx]], dim=1).contiguous()
            # correspondence search (iterative_root_finding.py:91-168): J0^-1 at the observed points, Broyden on the device
            obs = obs.to(torch.float32).contiguous()
            _, j0_inv = self.mlp.inverse_jacobian(obs, cond)
            p, _, valid, _ = self.mlp.broyden_search(obs, cond, obs, j0_inv, max_steps=15, cvg_thresh=1e-6, dvg_thresh=0.2,
                                                     early_exit=self.early_exit)
            # implicit differentiation of the root (:99-106): J^-1 at the root
            _, j_inv = self.mlp.inverse_jacobian(p, cond)
            # surface term (:111-136): value + d/d z_id + d/d xc
            pts = p.reshape(-1, 3)
            mask = valid.reshape(-1).to(torch.uint8).contiguous()
            g_lat = torch.empty(D, device=dev)
            g_pts = torch.empty_like(pts)
            _surface_grad(self.eng, pts, _quirk_period(self.dec, n_point), self.z_id, mask, clamp, self.terms, g_lat, g_pts,
                          stream)
            u = -(j_inv * g_pts.reshape(nb, n_point, 3, 1)).sum(-2)                       # -J^-T g_x
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)     # nb x (32 + E); same points as j_inv
            g_first = (Wc * g_cond[:, :32].sum(0)[:, None]).sum(0)                       # compressor^T -> [z_id | anchors]
            g_zid = (g_lat + g_first[:D]).contiguous()
            g_anchors = g_first[D:].contiguous()
            stats = torch.stack([self.terms[5], self.terms[0] * self.terms[5]]).nan_to_num_(0.0).contiguous()
            # expression codes: surface route + reg_expr = mean_b ||z_ex[idx_b]||^2 (:137), dense Adam over all rows (:169)
            lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, obs_idx, lam_s * g_cond[:, 32:] + (2.0 * lam_e / nb) * self.z_ex[obs_idx])
            fp = nat.FitParams(lam_s, float(lambdas.get('reg_global', 0.0)), float(lambdas.get('reg_loc', 0.0)),
                               float(lambdas.get('reg_unobserved', 0.0)), float(lambdas.get('symm_dist', 0.0)), float(clamp),
                               float(lr), max(self.t, 1))
            g_total = None if apply_update else torch.empty(D, device=dev)
            nat.check(nat.lib().nphm_fit_apply_gradient(self.eng.handle, self.z_id.data_ptr(), self.m_id.data_ptr(),
                                                        self.v_id.data_ptr(), ctypes.byref(fp), g_zid.data_ptr(), stats.data_ptr(),
                                                        g_anchors.data_ptr(), int(apply_update), self.loss_terms.data_ptr(),
                                                        None if apply_update else g_total.data_ptr(), stream),
                      'nphm_fit_apply_gradient')
            if not apply_update:
                return g_total, g_zex
            nat.check(nat.lib().nphm_adam_step(self.z_ex.data_ptr(), g_zex.data_ptr(), self.m_ex.data_ptr(), self.v_ex.data_ptr(),
                                               self.z_ex.numel(), float(lr), self.t, stream), 'nphm_adam_step')
            return None


# ------------------------------------------------------------------------------------------ NPM baseline (DeepSDF decoders)
NPM_EXPR_DIM = 200          # the reference's expression code width when decoder_expr has no lat_dim_expr (fitting.py:26-29)


def _native_npm_decoder(decoder, out_dim: int) -> bool:
    """A ``DeepSDF`` the native fitters take: CUDA fp32, Softplus(100), no positional encoding, ``out_dim`` outputs and a
    stack the native builder accepts (the condition of ``DeepSDF.native_grad_supported``)."""
    from .deepSDF import DeepSDF
    if not isinstance(decoder, DeepSDF) or decoder.out_dim_net != out_dim:
        return False
    p = next(decoder.parameters())
    n_lin = decoder.num_layers - 1
    return (p.is_cuda and p.dtype == torch.float32 and decoder.num_freq_bands is None and decoder.beta == 100
            and _native.stack_supported(n_lin - 1, _native.hidden_width(decoder, n_lin), decoder.lat_dim))


def _native_npm_joint(decoder, decoder_expr, device) -> bool:
    """The NPM baseline of fitting_npm.yaml: a one-output ``DeepSDF`` identity decoder and a 3-output ``DeepSDF`` expression
    decoder conditioned on ``[z_id | z_ex]``, both on ``device``."""
    if device.type != 'cuda' or not (_native_npm_decoder(decoder, 1) and _native_npm_decoder(decoder_expr, 3)):
        return False
    if hasattr(decoder_expr, 'lat_dim_expr') or decoder_expr.lat_dim != decoder.lat_dim + NPM_EXPR_DIM:
        return False
    return next(decoder.parameters()).device == device and next(decoder_expr.parameters()).device == device


class NpmIdentityFitter:
    """``inference_identity_space`` for a one-output ``DeepSDF`` (reference fitting.py:180-285) without an autograd graph.
    Per iteration: the surface term with its code gradient (``nphm_mlp_fit_surface_grad``, all sampled points as one query
    with condition ``z``), ``reg_global = ||z||^2`` (gradient ``2 z``; the reference sets reg_loc, reg_unobserved and
    symm_dist to 0 for a DeepSDF), and Adam (``nphm_adam_step``)."""

    def __init__(self, decoder, device):
        self.device = device
        self.engine = decoder.engine()
        self.latent = torch.zeros(decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latent)
        self.v = torch.zeros_like(self.latent)
        self.loss_terms = torch.zeros(8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latent)
        self.t = 0
        self._ws = None

    def step(self, points: torch.Tensor, lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True):
        """One iteration on ``points`` (B x N x 3); with ``apply_update=False`` only ``grad`` and ``loss_terms`` are set."""
        pts = points.reshape(1, -1, 3).to(dtype=torch.float32).contiguous()
        if apply_update:
            self.t += 1
        lam_s, lam_g = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(self.device):
            if self._ws is None or self._ws[0] != pts.shape[1]:
                self._ws = (pts.shape[1], self.engine.fit_workspace(1, pts.shape[1], self.device))
            terms, g_cond, _ = self.engine.fit_surface_grad(pts, self.latent[None], None, clamp, want_xyz=False,
                                                            workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            torch.add(lam_s * g_cond[0], self.latent, alpha=2.0 * lam_g, out=self.grad)
            if apply_update:
                _native.check(_native.lib().nphm_adam_step(self.latent.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(),
                                                           self.v.data_ptr(), self.latent.numel(), float(lr), self.t,
                                                           torch.cuda.current_stream(self.device).cuda_stream), 'nphm_adam_step')


class NpmJointFitter:
    """One iteration of ``inference_iterative_root_finding_joint`` (reference fitting.py:38-175) for the NPM baseline
    (``DeepSDF`` identity and expression decoders) without an autograd graph.  The chain of :class:`JointFitter` without the
    compressor, anchors or mlp_pos:
        cond_b = [z_id | z_ex[idx_b]]
        J0^-1 at the observations, Broyden on the device (sync-free), J^-1 at the roots     nphm_mlp_inverse_jacobian / _broyden_search
        d surface / d z_id, g_x = d surface / d xc  (mask = valid)                          nphm_mlp_fit_surface_grad
        u = -J^-T g_x,  g_cond = sum_n (dF/d cond)^T u_n                                      nphm_mlp_backward_inputs (value pass reused)
        z_id += g_cond[:, :D] summed over the scans,  z_ex[idx_b] += g_cond[b, D:] + reg_expr,  two Adam steps.
    u is of order 1e-4; the adjoint pass, which works on fp16 hi | lo operands, scales each query's upstream into their range
    itself."""

    def __init__(self, decoder, decoder_expr, num_observations: int, device):
        self.device = device
        self.eng = decoder.engine()
        self.mlp = decoder_expr.engine()
        D = decoder.lat_dim
        self.z_id = torch.zeros(D, device=device)
        self.m_id, self.v_id = torch.zeros_like(self.z_id), torch.zeros_like(self.z_id)
        self.z_ex = torch.zeros(num_observations, decoder_expr.lat_dim - D, device=device)
        self.m_ex, self.v_ex = torch.zeros_like(self.z_ex), torch.zeros_like(self.z_ex)
        self.loss_terms = torch.zeros(8, device=device)
        self.t = 0
        self.anchors = None                     # a DeepSDF has no anchors
        self.early_exit = bool(int(os.environ.get('NPHM_BROYDEN_EARLY_EXIT', '0')))
        self._ws = None

    def step(self, obs, obs_idx, lambdas, clamp, lr, apply_update: bool = True):
        """One iteration; with ``apply_update=False`` nothing is modified and ``(d loss / d z_id, d loss / d z_ex)`` - the
        tensors the reference hands to its two ``Adam.step()`` calls - are returned."""
        nat, dev = _native, self.device
        nb, n_point, _ = obs.shape
        D = self.z_id.shape[0]
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
        lam_g = float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(dev):
            cond = torch.cat([self.z_id[None].expand(nb, D), self.z_ex[obs_idx]], dim=1).contiguous()
            obs = obs.to(torch.float32).contiguous()
            _, j0_inv = self.mlp.inverse_jacobian(obs, cond)
            p, _, valid, _ = self.mlp.broyden_search(obs, cond, obs, j0_inv, max_steps=15, cvg_thresh=1e-6, dvg_thresh=0.2,
                                                     early_exit=self.early_exit)
            _, j_inv = self.mlp.inverse_jacobian(p, cond)
            if self._ws is None or self._ws[0] != nb * n_point:
                self._ws = (nb * n_point, self.eng.fit_workspace(1, nb * n_point, dev))
            terms, g_lat, g_pts = self.eng.fit_surface_grad(p.reshape(1, -1, 3), self.z_id[None], valid, clamp,
                                                            workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            u = -(j_inv * g_pts.reshape(nb, n_point, 3, 1)).sum(-2)                     # -J^-T g_x
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)
            g_zid = lam_s * (g_lat[0] + g_cond[:, :D].sum(0)) + (2.0 * lam_g) * self.z_id
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, obs_idx, lam_s * g_cond[:, D:] + (2.0 * lam_e / nb) * self.z_ex[obs_idx])
            if not apply_update:
                return g_zid, g_zex
            for z, g, m, v in ((self.z_id, g_zid, self.m_id, self.v_id), (self.z_ex, g_zex, self.m_ex, self.v_ex)):
                nat.check(nat.lib().nphm_adam_step(z.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), z.numel(), float(lr),
                                                   self.t, stream), 'nphm_adam_step')
            return None


def inference_iterative_root_finding_joint(decoder,
                                           decoder_expr,
                                           all_obs: List[torch.Tensor],
                                           lambdas,
                                           n_steps,
                                           schedule_cfg: Dict,
                                           step_scale=1,
                                           lr_scale=1):
    """Joint identity + expression fitting with Broyden correspondences (reference :14-177).

    Shipped configuration (fused ensemble + 'compress' DeformationNetwork on CUDA): no autograd graph at all, see
    :class:`JointFitter`; the same for the NPM baseline (``DeepSDF`` decoders on CUDA), see :class:`NpmJointFitter`.
    ``NPHM_JOINT_AUTOGRAD=1`` keeps both on the composite path.  Anything else: the correspondence search runs on the device (`nphm_mlp_broyden_search`), the
    surface term comes from `nphm_fit_surface_grad`, the deformation network's part of the chain stays on autograd.  Returns
    ``(lat_rep (n_obs,1,E), lat_rep_shape (1,1,D), anchors)``."""
    device = all_obs[0].device
    num_observations = len(all_obs)
    if not os.environ.get('NPHM_JOINT_AUTOGRAD'):
        fitter = None
        if _native_joint(decoder, decoder_expr, device):
            fitter = JointFitter(decoder, decoder_expr, num_observations, device)
        elif _native_npm_joint(decoder, decoder_expr, device):
            fitter = NpmJointFitter(decoder, decoder_expr, num_observations, device)
        if fitter is not None:
            lr = 0.01 * lr_scale
            for j in range(int(n_steps * step_scale)):
                lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
                obs, obs_idx = _sample_observations(all_obs)
                fitter.step(obs, obs_idx.long().to(device), lambdas, _clamp_for_iteration(j, step_scale), lr)
            lat_rep = fitter.z_ex.reshape(num_observations, 1, -1).clone().requires_grad_(True)
            lat_rep_shape = fitter.z_id.reshape(1, 1, -1).clone().requires_grad_(True)
            return lat_rep, lat_rep_shape, fitter.anchors
    return _inference_joint_autograd(decoder, decoder_expr, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)


def _inference_joint_autograd(decoder, decoder_expr, all_obs, lambdas, n_steps, schedule_cfg, step_scale=1, lr_scale=1):
    """The composite path of :func:`inference_iterative_root_finding_joint`: the correspondence search on the device where
    the search supports the decoder, everything else on autograd through the modules."""
    device = all_obs[0].device
    num_observations = len(all_obs)
    lat_expr_dim = decoder_expr.lat_dim_expr if hasattr(decoder_expr, 'lat_dim_expr') else 200
    lat_rep = torch.zeros([num_observations, 1, lat_expr_dim], device=device, requires_grad=True)
    lat_rep_shape = torch.zeros([1, 1, decoder.lat_dim], device=device, requires_grad=True)
    lr = 0.01 * lr_scale
    opt = optim.Adam(params=[lat_rep_shape], lr=lr)
    opt_expr = optim.Adam(params=[lat_rep], lr=lr)
    anchors = None
    for j in range(int(n_steps * step_scale)):
        new_lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        if new_lr != lr:
            lr = new_lr
            for o in (opt, opt_expr):
                for group in o.param_groups:
                    group['lr'] = lr
        opt.zero_grad()
        opt_expr.zero_grad()
        anchors = _current_anchors(decoder, lat_rep_shape, device)
        obs, obs_idx = _sample_observations(all_obs)
        obs_idx = obs_idx.long().to(device)
        nb, n_point, _ = obs.shape
        glob_cond = torch.cat([lat_rep_shape.repeat(nb, 1, 1), lat_rep[obs_idx, :, :]], dim=-1)
        has_local = hasattr(decoder, 'lat_dim_loc')
        search_anchors = anchors.clone().unsqueeze(1).repeat(nb, n_point, 1, 1) if has_local else None
        p_corresp, search_result = search(obs, glob_cond.repeat(1, n_point, 1), decoder_expr, search_anchors,
                                          multi_corresp=False)
        p_corresp = p_corresp.detach()
        _anchors = anchors.clone().unsqueeze(1).repeat(nb, n_point, 1, 1) if anchors is not None else None
        # implicit differentiation of the root: value(xc) = p, d xc = -J^-1 d F_ex
        preds_posed, _ = decoder_expr(p_corresp, glob_cond.repeat(1, n_point, 1), _anchors)
        preds_posed = preds_posed + p_corresp
        grad_inv = jac(decoder_expr, p_corresp, glob_cond.repeat(1, n_point, 1), _anchors).inverse()
        correction = preds_posed - preds_posed.detach()
        correction = torch.einsum('bnij,bnj->bni', -grad_inv.detach(), correction)
        xc = p_corresp + correction
        if has_local and _fused_identity(decoder, grad_points=True) and xc.is_cuda:
            surface = _FusedSurfaceLoss.apply(xc, lat_rep_shape, search_result['valid_ids'],
                                              _clamp_for_iteration(j, step_scale), decoder)
        else:
            if has_local:
                sdf, _ = decoder(xc, lat_rep_shape.repeat(nb, 1, 1), None)
            else:
                sdf, _ = decoder(xc, lat_rep_shape.repeat(nb, n_point, 1), None)
            sdf = sdf[search_result['valid_ids'], :]
            l = sdf.abs()
            l = l[l < _clamp_for_iteration(j, step_scale)]
            surface = l.mean()
        loss_dict = {'surface': surface,
                     'reg_expr': (torch.norm(lat_rep[obs_idx, :, :], dim=-1) ** 2).mean()}
        loss_dict.update(_latent_regularisers(decoder, lat_rep_shape))
        loss = 0
        for k in lambdas.keys():
            loss = loss + loss_dict[k] * lambdas[k]
        loss.backward()
        opt.step()
        opt_expr.step()
    return lat_rep, lat_rep_shape, anchors


# ------------------------------------------------------------------------------------------ many scans in one launch sequence
def _sampling_plan(scans, n_iters: int):
    """One generator per scan that replays, for that scan, the draws the sequential fits would take from the global CPU
    generator: scan k's fit starts where scan k-1's ended.  The global generator is walked forward over every scan's
    ``n_iters`` iterations (indices only, nothing is gathered), so afterwards it is where the sequential calls leave it."""
    gens = []
    for all_obs in scans:
        g = torch.Generator()
        g.set_state(torch.get_rng_state())
        gens.append(g)
        sizes = [o.shape[0] for o in all_obs]
        for _ in range(n_iters):
            _sample_indices(sizes)
    return gens


def _pad_scans(points: List[torch.Tensor]):
    """Per-scan point sets (n_k x 3) -> (S x n x 3, S x n mask bytes or None).  Missing rows repeat the scan's first point
    (finite through every kernel) and are masked out of the loss."""
    n = max(p.shape[0] for p in points)
    if all(p.shape[0] == n for p in points):
        return torch.stack(points).contiguous(), None
    padded, masks = [], []
    for p in points:
        extra = n - p.shape[0]
        padded.append(torch.cat([p, p[:1].expand(extra, 3)]) if extra else p)
        m = torch.ones(n, dtype=torch.uint8, device=p.device)
        m[p.shape[0]:] = 0
        masks.append(m)
    return torch.stack(padded).contiguous(), torch.stack(masks).contiguous()


def _sequential(fit_one, scans, lambdas, *args):
    """The batched functions' contract, run one scan after another: every call gets a fresh copy of ``lambdas`` and the
    caller's dict ends as one call leaves it."""
    start, out = dict(lambdas), []
    for all_obs in scans:
        lam = dict(start)
        out.append(fit_one(all_obs, lam, *args))
        lambdas.update(lam)
    return out


TC_MAX_MEMBERS = 64         # the tensor-core kernels keep member sets in 64-bit masks (csrc tc_ensemble.cuh kMaxMembers)


def _tc_ensemble(decoder) -> bool:
    """The tensor-core configuration (csrc tc_ensemble_supported): 4 hidden layers of width 200, a condition of 96
    (lat_dim_glob + lat_dim_loc) and at most 64 members (n_loc + 1).  The scan-batched kernels, the eval-mode quirk and the
    point gradients need it."""
    e = decoder.ensembled_deep_sdf
    return (e.num_layers == 6 and _native.hidden_width(e, e.num_layers - 1) == 200
            and decoder.lat_dim_glob + decoder.lat_dim_loc == 96 and decoder.num_kps + 1 <= TC_MAX_MEMBERS)


class _QuirkPeriods:
    """The per-scan quirk periods of the batched eval-mode calls as an int32 device tensor, uploaded when they change."""

    def __init__(self):
        self._key, self._dev = None, None

    def __call__(self, periods: List[int], device) -> torch.Tensor:
        key = tuple(int(p) for p in periods)
        if key != self._key:
            self._key, self._dev = key, torch.tensor(key, dtype=torch.int32).to(device)
        return self._dev


class BatchedIdentityFitter:
    """:class:`IdentityFitter` for S scans at once (``nphm_fit_identity_step_batched``): latents and Adam moments S x D on the
    device, one launch sequence per iteration for all scans.  In eval mode (``nphm_fit_identity_step_batched_quirk``) scan
    k's period is the points per row of its sample, so each scan gets the quirk rows of its own single-scan call."""

    def __init__(self, decoder: FastEnsembleDeepSDFMirrored, n_scans: int, device):
        self.decoder = decoder
        self._periods = _QuirkPeriods()
        self.device = device
        self.engine = decoder.engine()
        self.latents = torch.zeros(n_scans, decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latents)
        self.v = torch.zeros_like(self.latents)
        self.loss_terms = torch.zeros(n_scans, 8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latents)
        self.t = 0
        self._ws = None

    def step(self, points: List[torch.Tensor], lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True):
        """One iteration; ``points[k]`` are scan k's sampled points (any shape ending in 3, lengths may differ)."""
        pts, mask = _pad_scans([p.reshape(-1, 3).to(dtype=torch.float32) for p in points])
        S, n = pts.shape[0], pts.shape[1]
        eval_mode = not self.decoder.training
        if apply_update:
            self.t += 1
        fp = _native.FitParams(float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0)),
                               float(lambdas.get('reg_loc', 0.0)), float(lambdas.get('reg_unobserved', 0.0)),
                               float(lambdas.get('symm_dist', 0.0)), float(clamp), float(lr), max(self.t, 1))
        lib = _native.lib()
        with torch.cuda.device(self.device):
            if self._ws is None or self._ws[0] != (S, n):
                self._ws = ((S, n), _native._workspace(lib.nphm_fit_batch_workspace_bytes(self.engine.handle, S, n),
                                                       'nphm_fit_batch_workspace_bytes', self.device))
            ws = self._ws[1]
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if eval_mode:
                periods = self._periods([p.shape[-2] if p.dim() > 1 else 1 for p in points], self.device)
                _native.check(lib.nphm_fit_identity_step_batched_quirk(
                    self.engine.handle, pts.data_ptr(), _native._ptr(mask), S, n, periods.data_ptr(), self.latents.data_ptr(),
                    self.m.data_ptr(), self.v.data_ptr(), ctypes.byref(fp), int(apply_update), self.loss_terms.data_ptr(),
                    self.grad.data_ptr(), ws.data_ptr(), ws.numel(), stream), 'nphm_fit_identity_step_batched_quirk')
            else:
                _native.check(lib.nphm_fit_identity_step_batched(
                    self.engine.handle, pts.data_ptr(), _native._ptr(mask), S, n, self.latents.data_ptr(), self.m.data_ptr(),
                    self.v.data_ptr(), ctypes.byref(fp), int(apply_update), self.loss_terms.data_ptr(), self.grad.data_ptr(),
                    ws.data_ptr(), ws.numel(), stream),
                    'nphm_fit_identity_step_batched')


def _scans_device(scans):
    devs = {o.device for all_obs in scans for o in all_obs}
    return devs.pop() if len(devs) == 1 else None


def inference_identity_space_batched(decoder,
                                     scans: List[List[torch.Tensor]],
                                     lambdas,
                                     n_steps,
                                     schedule_cfg: Dict,
                                     step_scale=1,
                                     lr_scale=1):
    """:func:`inference_identity_space` for several scans (``scans[k]``: the observations of scan k) at once.  Returns
    ``[(lat_rep_shape, anchors)]`` in scan order - what the single-scan function gives when called on each scan in turn, each
    call with a fresh copy of ``lambdas``; the global CPU generator and ``lambdas`` end as those calls leave them.  Runs all
    scans in one launch sequence per iteration for the fused ensemble on CUDA (:class:`BatchedIdentityFitter`, training or eval
    mode, see :func:`_fused_identity`)
    and for the NPM baseline's ``DeepSDF`` on CUDA (:class:`BatchedNpmIdentityFitter`); any other configuration calls the
    single-scan function scan by scan."""
    if not scans:
        return []
    device = _scans_device(scans)
    npm = device is not None and device.type == 'cuda' and _native_npm_decoder(decoder, 1)
    if not npm and (device is None or device.type != 'cuda' or not (_fused_identity(decoder) and _tc_ensemble(decoder))):
        return _sequential(lambda obs, lam: inference_identity_space(decoder, obs, lam, n_steps, schedule_cfg, step_scale,
                                                                     lr_scale), scans, lambdas)
    n_iters = int(n_steps * step_scale)
    gens = _sampling_plan(scans, n_iters)
    lr = 0.01 * lr_scale
    if npm:
        fitter = BatchedNpmIdentityFitter(decoder, len(scans), device)
        for j in range(n_iters):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs = [_sample_observations(all_obs, g)[0] for all_obs, g in zip(scans, gens)]
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr)
        return [(fitter.latents[k].reshape(1, 1, -1).clone().requires_grad_(True), None) for k in range(len(scans))]
    fitter = BatchedIdentityFitter(decoder, len(scans), device)
    z_prev = fitter.latents.clone()
    for j in range(n_iters):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        obs = [_sample_observations(all_obs, g)[0] for all_obs, g in zip(scans, gens)]
        z_prev.copy_(fitter.latents)
        fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr)
    out = []
    with torch.no_grad():
        for k in range(len(scans)):
            _, anchors = fitter.engine.query(torch.zeros(1, 1, 3, device=device), z_prev[k].reshape(1, -1), eval_quirk=False)
            out.append((fitter.latents[k].reshape(1, 1, -1).clone().requires_grad_(True), anchors))
    return out


def _pad_rows(obs: List[torch.Tensor], n_point: int, front: bool = False):
    """Subjects' samples (``obs[k]``: rows x n_k x 3) -> (all rows padded to n_point points, S rows n_point float32; the
    kept-point mask S x rows x n_point, or None when nothing is padded).  The padding repeats the row's first point, behind
    the row or, with ``front``, in front of it (then every row ends with its own last point)."""
    nb = obs[0].shape[0]
    keep = None
    if any(o.shape[1] != n_point for o in obs):
        keep = torch.ones(len(obs), nb, n_point, dtype=torch.bool, device=obs[0].device)
        for k, o in enumerate(obs):
            if front:
                keep[k, :, :n_point - o.shape[1]] = False
            else:
                keep[k, :, o.shape[1]:] = False

    def padded(o):
        if o.shape[1] == n_point:
            return o
        pad = o[:, :1].expand(nb, n_point - o.shape[1], 3)
        return torch.cat([pad, o] if front else [o, pad], dim=1)
    return torch.cat([padded(o) for o in obs]).to(torch.float32).contiguous(), keep


class BatchedJointFitter:
    """:class:`JointFitter` for S subjects at once.  Per iteration, for the 5 sampled observations of every subject:
        anchors of the S identity codes (nphm_ensemble_anchors), condition rows [compressor([z_id | anchors])[subject] | z_ex[row]]
        J0^-1, Broyden and J^-1 on all 5 S rows (per-row conditions; shorter subjects padded, the padding masked)
        nphm_fit_surface_grad_batched: per-subject surface term, d/d z_id and d/d point
        u = -J^-T g_x, one adjoint pass, the compressor adjoint summed per subject
        nphm_fit_apply_gradient_batched (regularisers, mlp_pos backward, Adam per subject)
        one nphm_adam_step over the expression codes of all subjects (element-wise, shared step and lr: the same as per subject).
    The expression codes are one (sum n_obs) x E tensor; subject k's rows start at ``offsets[k]``.  In eval mode a shorter
    subject's rows are padded in front instead of behind, so that every row ends with its subject's last sampled point - the
    quirk row of that subject's single-subject call - and one period, n_point, serves all subjects
    (``nphm_fit_surface_grad_batched_quirk``)."""

    def __init__(self, decoder, decoder_expr, num_observations: List[int], device):
        self.dec, self.dfn, self.device = decoder, decoder_expr, device
        self.eng = decoder.engine()
        self.mlp = decoder_expr.defDeepSDF.engine()
        E, S = decoder_expr.lat_dim_expr, len(num_observations)
        self.num_observations = list(num_observations)
        self.offsets = [sum(self.num_observations[:k]) for k in range(S)]
        self.z_id = torch.zeros(S, decoder.lat_dim, device=device)
        self.m_id, self.v_id = torch.zeros_like(self.z_id), torch.zeros_like(self.z_id)
        self.z_ex = torch.zeros(sum(self.num_observations), E, device=device)
        self.m_ex, self.v_ex = torch.zeros_like(self.z_ex), torch.zeros_like(self.z_ex)
        self.loss_terms = torch.zeros(S, 8, device=device)
        self.t = 0
        self.anchors = None
        self.early_exit = bool(int(os.environ.get('NPHM_BROYDEN_EARLY_EXIT', '0')))
        self._ws = None

    def step(self, obs: List[torch.Tensor], obs_idx: List[torch.Tensor], lambdas, clamp, lr, apply_update: bool = True):
        """One iteration; ``obs[k]`` (5 x n_k x 3) and ``obs_idx[k]`` (5, on the device) are subject k's sample.  With
        ``apply_update=False`` nothing is modified and ``(d loss / d z_id (S x D), [d loss / d z_ex of subject k])`` is returned."""
        nat, dev = _native, self.device
        S, D = self.z_id.shape
        nb = obs[0].shape[0]
        n_point = max(o.shape[1] for o in obs)
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        lib = nat.lib()
        with torch.no_grad(), torch.cuda.device(dev):
            anchors = self.eng.anchors(self.z_id)                                        # S x K x 3, pre-update codes
            self.anchors = anchors
            lin = self.dfn.compressor[0] if isinstance(self.dfn.compressor, torch.nn.Sequential) else self.dfn.compressor
            Wc, bc = lin.weight, lin.bias
            first = torch.cat([self.z_id, anchors.reshape(S, -1)], dim=1)
            c32 = (Wc[None] * first[:, None, :]).sum(2) + bc                             # S x 32
            rows = torch.cat([idx + off for idx, off in zip(obs_idx, self.offsets)])    # rows of z_ex, 5 S
            cond = torch.cat([c32.repeat_interleave(nb, dim=0), self.z_ex[rows]], dim=1).contiguous()
            # every subject padded to n_point points per observation (the padding repeats a point and is masked below); in eval
            # mode in front of the row, so that its last point stays last
            front = not self.dec.training
            obs_all, keep = _pad_rows(obs, n_point, front)                                # 5 S x n_point x 3
            _, j0_inv = self.mlp.inverse_jacobian(obs_all, cond)
            p, _, valid, _ = self.mlp.broyden_search(obs_all, cond, obs_all, j0_inv, max_steps=15, cvg_thresh=1e-6,
                                                     dvg_thresh=0.2, early_exit=self.early_exit)
            _, j_inv = self.mlp.inverse_jacobian(p, cond)
            n = nb * n_point
            pts = p.reshape(S, n, 3).contiguous()
            valid = valid.reshape(S, nb, n_point)
            mask = (valid if keep is None else valid & keep).reshape(S, n).to(torch.uint8).contiguous()
            if self._ws is None or self._ws[0] != (S, n):
                self._ws = ((S, n), nat._workspace(lib.nphm_fit_batch_workspace_bytes(self.eng.handle, S, n),
                                                   'nphm_fit_batch_workspace_bytes', dev))
            ws = self._ws[1]
            terms = torch.empty(S, 8, device=dev)
            g_lat = torch.empty(S, D, device=dev)
            g_pts = torch.empty_like(pts)
            if front:
                periods = torch.full((S,), n_point, dtype=torch.int32, device=dev)
                nat.check(lib.nphm_fit_surface_grad_batched_quirk(self.eng.handle, pts.data_ptr(), mask.data_ptr(), S, n,
                                                                  periods.data_ptr(), self.z_id.data_ptr(), float(clamp),
                                                                  terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(),
                                                                  ws.data_ptr(), ws.numel(), stream),
                          'nphm_fit_surface_grad_batched_quirk')
            else:
                nat.check(lib.nphm_fit_surface_grad_batched(self.eng.handle, pts.data_ptr(), mask.data_ptr(), S, n,
                                                            self.z_id.data_ptr(), float(clamp), terms.data_ptr(),
                                                            g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                          'nphm_fit_surface_grad_batched')
            u = -(j_inv * g_pts.reshape(S * nb, n_point, 3, 1)).sum(-2)                  # -J^-T g_x
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)     # 5 S x (32 + E)
            g_c32 = g_cond[:, :32].reshape(S, nb, 32).sum(1)
            g_first = (Wc[None] * g_c32[:, :, None]).sum(1)                              # compressor^T, S x (D + 3 K)
            g_zid = (g_lat + g_first[:, :D]).contiguous()
            g_anchors = g_first[:, D:].contiguous()
            stats = torch.stack([terms[:, 5], terms[:, 0] * terms[:, 5]], dim=1).nan_to_num_(0.0).contiguous()
            lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, rows, lam_s * g_cond[:, 32:] + (2.0 * lam_e / nb) * self.z_ex[rows])
            fp = nat.FitParams(lam_s, float(lambdas.get('reg_global', 0.0)), float(lambdas.get('reg_loc', 0.0)),
                               float(lambdas.get('reg_unobserved', 0.0)), float(lambdas.get('symm_dist', 0.0)), float(clamp),
                               float(lr), max(self.t, 1))
            g_total = None if apply_update else torch.empty(S, D, device=dev)
            nat.check(lib.nphm_fit_apply_gradient_batched(self.eng.handle, S, self.z_id.data_ptr(), self.m_id.data_ptr(),
                                                          self.v_id.data_ptr(), ctypes.byref(fp), g_zid.data_ptr(),
                                                          stats.data_ptr(), g_anchors.data_ptr(), int(apply_update),
                                                          self.loss_terms.data_ptr(), nat._ptr(g_total), stream),
                      'nphm_fit_apply_gradient_batched')
            if not apply_update:
                return g_total, [g_zex[o:o + c] for o, c in zip(self.offsets, self.num_observations)]
            nat.check(lib.nphm_adam_step(self.z_ex.data_ptr(), g_zex.data_ptr(), self.m_ex.data_ptr(), self.v_ex.data_ptr(),
                                         self.z_ex.numel(), float(lr), self.t, stream), 'nphm_adam_step')
            return None


class BatchedNpmIdentityFitter:
    """:class:`NpmIdentityFitter` for S scans at once: latents, Adam moments and ``grad`` S x D, ``loss_terms`` S x 8.  Per
    iteration one surface call over all scans (``nphm_mlp_fit_surface_grad_batched``, scan k = query k with condition z_k and
    its own loss), ``grad = lambda_s g_cond + 2 lambda_g z`` and one ``nphm_adam_step`` over the S D elements (Adam is
    element-wise and the scans share the step and lr)."""

    def __init__(self, decoder, n_scans: int, device):
        self.device = device
        self.engine = decoder.engine()
        self.latents = torch.zeros(n_scans, decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latents)
        self.v = torch.zeros_like(self.latents)
        self.loss_terms = torch.zeros(n_scans, 8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latents)
        self.t = 0
        self._ws = None

    def step(self, points: List[torch.Tensor], lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True):
        """One iteration; ``points[k]`` are scan k's sampled points (any shape ending in 3, lengths may differ)."""
        pts, mask = _pad_scans([p.reshape(-1, 3).to(dtype=torch.float32) for p in points])
        S, n = pts.shape[0], pts.shape[1]
        if apply_update:
            self.t += 1
        lam_s, lam_g = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(self.device):
            if self._ws is None or self._ws[0] != (S, n):
                self._ws = ((S, n), self.engine.fit_workspace(S, n, self.device))
            terms, g_cond, _ = self.engine.fit_surface_grad_batched(pts, self.latents, mask, clamp, want_xyz=False,
                                                                    workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            torch.add(lam_s * g_cond, self.latents, alpha=2.0 * lam_g, out=self.grad)
            if apply_update:
                _native.check(_native.lib().nphm_adam_step(self.latents.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(),
                                                           self.v.data_ptr(), self.latents.numel(), float(lr), self.t,
                                                           torch.cuda.current_stream(self.device).cuda_stream), 'nphm_adam_step')


class BatchedNpmJointFitter:
    """:class:`NpmJointFitter` for S subjects at once, with the padding and row bookkeeping of :class:`BatchedJointFitter`.  Per
    iteration, for the 5 sampled observations of every subject:
        condition rows [z_id[subject] | z_ex[row]]; J0^-1, sync-free Broyden and J^-1 on all 5 S rows
        nphm_mlp_fit_surface_grad_batched (mask = valid and not padding): per-subject surface term, d/d z_id and d/d point
        u = -J^-T g_x; one adjoint pass with the value pass reused (it scales every row's upstream on its own, so each subject's
        rows get what its single-subject call gives them)
        z_id: g_cond[:, :D] summed per subject; z_ex rows: g_cond[:, D:] + reg_expr; two nphm_adam_step calls.
    The expression codes are one (sum n_obs) x 200 tensor; subject k's rows start at ``offsets[k]``.  Memory grows linearly with
    S: the Jacobian, Broyden and adjoint buffers of 5 S n_point rows through the expression stack, about 1.4 GB per subject of
    5 x 1000 points (22.7 GB peak at S = 16, tools/bench_fit_batched.py --decoder npm), so an 80 GB card holds about 50
    subjects per batch; the caller chooses S, nothing is split."""

    def __init__(self, decoder, decoder_expr, num_observations: List[int], device):
        self.device = device
        self.eng = decoder.engine()
        self.mlp = decoder_expr.engine()
        D, S = decoder.lat_dim, len(num_observations)
        self.num_observations = list(num_observations)
        self.offsets = [sum(self.num_observations[:k]) for k in range(S)]
        self.z_id = torch.zeros(S, D, device=device)
        self.m_id, self.v_id = torch.zeros_like(self.z_id), torch.zeros_like(self.z_id)
        self.z_ex = torch.zeros(sum(self.num_observations), decoder_expr.lat_dim - D, device=device)
        self.m_ex, self.v_ex = torch.zeros_like(self.z_ex), torch.zeros_like(self.z_ex)
        self.loss_terms = torch.zeros(S, 8, device=device)
        self.t = 0
        self.anchors = None                     # a DeepSDF has no anchors
        self.early_exit = bool(int(os.environ.get('NPHM_BROYDEN_EARLY_EXIT', '0')))
        self._ws = None

    def step(self, obs: List[torch.Tensor], obs_idx: List[torch.Tensor], lambdas, clamp, lr, apply_update: bool = True):
        """One iteration; ``obs[k]`` (5 x n_k x 3) and ``obs_idx[k]`` (5, on the device) are subject k's sample.  With
        ``apply_update=False`` nothing is modified and ``(d loss / d z_id (S x D), [d loss / d z_ex of subject k])`` is returned."""
        nat, dev = _native, self.device
        S, D = self.z_id.shape
        nb = obs[0].shape[0]
        n_point = max(o.shape[1] for o in obs)
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
        lam_g = float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(dev):
            rows = torch.cat([idx + off for idx, off in zip(obs_idx, self.offsets)])    # rows of z_ex, 5 S
            cond = torch.cat([self.z_id.repeat_interleave(nb, dim=0), self.z_ex[rows]], dim=1).contiguous()
            keep = None
            if any(o.shape[1] != n_point for o in obs):
                keep = torch.ones(S, nb, n_point, dtype=torch.bool, device=dev)
                for k, o in enumerate(obs):
                    keep[k, :, o.shape[1]:] = False
            obs_all = torch.cat([o if o.shape[1] == n_point else torch.cat([o, o[:, :1].expand(nb, n_point - o.shape[1], 3)], dim=1)
                                 for o in obs]).to(torch.float32).contiguous()                 # 5 S x n_point x 3
            _, j0_inv = self.mlp.inverse_jacobian(obs_all, cond)
            p, _, valid, _ = self.mlp.broyden_search(obs_all, cond, obs_all, j0_inv, max_steps=15, cvg_thresh=1e-6,
                                                     dvg_thresh=0.2, early_exit=self.early_exit)
            _, j_inv = self.mlp.inverse_jacobian(p, cond)
            n = nb * n_point
            valid = valid.reshape(S, nb, n_point)
            mask = (valid if keep is None else valid & keep).reshape(S, n)
            if self._ws is None or self._ws[0] != (S, n):
                self._ws = ((S, n), self.eng.fit_workspace(S, n, dev))
            terms, g_lat, g_pts = self.eng.fit_surface_grad_batched(p.reshape(S, n, 3), self.z_id, mask, clamp,
                                                                    workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            u = -(j_inv * g_pts.reshape(S * nb, n_point, 3, 1)).sum(-2)                  # -J^-T g_x
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)
            g_zid = lam_s * (g_lat + g_cond[:, :D].reshape(S, nb, D).sum(1)) + (2.0 * lam_g) * self.z_id
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, rows, lam_s * g_cond[:, D:] + (2.0 * lam_e / nb) * self.z_ex[rows])
            if not apply_update:
                return g_zid, [g_zex[o:o + c] for o, c in zip(self.offsets, self.num_observations)]
            for z, g, m, v in ((self.z_id, g_zid, self.m_id, self.v_id), (self.z_ex, g_zex, self.m_ex, self.v_ex)):
                nat.check(nat.lib().nphm_adam_step(z.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), z.numel(), float(lr),
                                                   self.t, stream), 'nphm_adam_step')
            return None


def inference_iterative_root_finding_joint_batched(decoder,
                                                   decoder_expr,
                                                   subjects: List[List[torch.Tensor]],
                                                   lambdas,
                                                   n_steps,
                                                   schedule_cfg: Dict,
                                                   step_scale=1,
                                                   lr_scale=1):
    """:func:`inference_iterative_root_finding_joint` for several subjects (``subjects[k]``: the observations of subject k) at
    once.  Returns ``[(lat_rep (n_obs,1,E), lat_rep_shape (1,1,D), anchors)]`` in subject order, under the contract of
    :func:`inference_identity_space_batched`.  The shipped configuration (see :func:`_native_joint`) runs all subjects in one
    launch sequence per iteration (:class:`BatchedJointFitter`), and so does the NPM baseline (see :func:`_native_npm_joint`,
    :class:`BatchedNpmJointFitter`); anything else - CPU, other decoders or deformation modes, ``NPHM_JOINT_AUTOGRAD=1`` -
    calls the single-subject function subject by subject.  Memory grows linearly with the number of subjects; all subjects
    must fit on the device at once (nothing is split into smaller batches)."""
    if not subjects:
        return []
    device = _scans_device(subjects)
    batched = None
    if device is not None and not os.environ.get('NPHM_JOINT_AUTOGRAD'):
        if _native_npm_joint(decoder, decoder_expr, device):
            batched = BatchedNpmJointFitter
        elif _native_joint(decoder, decoder_expr, device) and _tc_ensemble(decoder):
            batched = BatchedJointFitter
    if batched is None:
        return _sequential(lambda obs, lam: inference_iterative_root_finding_joint(decoder, decoder_expr, obs, lam, n_steps,
                                                                                   schedule_cfg, step_scale, lr_scale),
                           subjects, lambdas)
    n_iters = int(n_steps * step_scale)
    gens = _sampling_plan(subjects, n_iters)
    fitter = batched(decoder, decoder_expr, [len(s) for s in subjects], device)
    lr = 0.01 * lr_scale
    for j in range(n_iters):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        sample = [_sample_observations(all_obs, g) for all_obs, g in zip(subjects, gens)]
        fitter.step([o for o, _ in sample], [i.long().to(device) for _, i in sample], lambdas,
                    _clamp_for_iteration(j, step_scale), lr)
    out = []
    for k, (off, cnt) in enumerate(zip(fitter.offsets, fitter.num_observations)):
        lat_rep = fitter.z_ex[off:off + cnt].reshape(cnt, 1, -1).clone().requires_grad_(True)
        lat_rep_shape = fitter.z_id[k].reshape(1, 1, -1).clone().requires_grad_(True)
        out.append((lat_rep, lat_rep_shape, None if fitter.anchors is None else fitter.anchors[k:k + 1].clone()))
    return out
