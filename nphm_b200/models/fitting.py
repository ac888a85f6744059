"""Drop-in mirror of the reference module ``NPHM.models.fitting``.

  * ``inference_identity_space``                 src/NPHM/models/fitting.py:180-285
  * ``inference_iterative_root_finding_joint``   src/NPHM/models/fitting.py:14-177
  * ``inference_expression_space``               the same joint loop with the identity code given and held fixed

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
from .pose import ObservationPoses, check_poses, compose_f64  # noqa: F401  (ObservationPoses is public here)
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


def _pose_step(fitter, q, g_q, rows, lam_s, lr, apply_update):
    """The pose's part of a posed step: ``poses.grad`` from ``g_q = d surface / d q`` at the sampled points ``q`` (rows x n x 3,
    row r from observation ``rows[r]``), then, with ``apply_update``, Adam at the fitter's step count with the pose rates
    scaled by lr / (the lr of the fitter's first step)."""
    if fitter.pose_lr0 is None:
        fitter.pose_lr0 = lr
    fitter.poses.gradient(q, g_q, rows, lam_s)
    if apply_update:
        fitter.poses.update(lr / fitter.pose_lr0, fitter.t)


class IdentityFitter:
    """Stateful wrapper around ``nphm_fit_identity_step``: latent + Adam moments live on the device.  With ``poses`` (an
    :class:`ObservationPoses` of the scan's observations) a step moves the sampled rows into the model frame first and fits
    the poses too; the fused step has no point gradient, so it then runs as ``nphm_fit_surface_grad`` with the point gradient
    and ``nphm_fit_apply_gradient`` (the joint fitter's route, the same math), which needs the tensor-core configuration."""

    def __init__(self, decoder: FastEnsembleDeepSDFMirrored, device, poses: ObservationPoses = None):
        self.decoder = decoder
        self.poses, self.pose_lr0, self._ones = poses, None, None
        self.device = device
        self.engine = decoder.engine()
        self.latent = torch.zeros(decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latent)
        self.v = torch.zeros_like(self.latent)
        self.loss_terms = torch.zeros(8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latent)
        self.t = 0

    def step(self, points: torch.Tensor, lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True,
             obs_idx: torch.Tensor = None):
        """One iteration on ``points`` (rows x n x 3: the reference's one decoder call on its sampled rows).  In eval mode the
        last point of every row carries the quirk (``nphm_fit_identity_step_quirk`` with period n).  With poses, ``obs_idx``
        (rows, on the device) gives each row's observation."""
        pts = points.reshape(-1, 3).to(dtype=torch.float32).contiguous()
        period = _quirk_period(self.decoder, points.shape[-2] if points.dim() > 1 else 1)
        if apply_update:
            self.t += 1
        fp = _native.FitParams(float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0)),
                               float(lambdas.get('reg_loc', 0.0)), float(lambdas.get('reg_unobserved', 0.0)),
                               float(lambdas.get('symm_dist', 0.0)), float(clamp), float(lr), max(self.t, 1))
        stream = torch.cuda.current_stream(self.device).cuda_stream
        with torch.cuda.device(self.device):
            if self.poses is not None:
                q = self.poses.apply(points, obs_idx)
                pts = q.reshape(-1, 3)
                if self._ones is None or self._ones.shape[0] != pts.shape[0]:
                    self._ones = torch.ones(pts.shape[0], dtype=torch.uint8, device=self.device)
                terms, g_pts = torch.empty(8, device=self.device), torch.empty_like(pts)
                g_lat = torch.empty_like(self.latent)
                _surface_grad(self.engine, pts, period, self.latent, self._ones, clamp, terms, g_lat, g_pts, stream)
                stats = torch.stack([terms[5], terms[0] * terms[5]]).nan_to_num_(0.0).contiguous()
                _native.check(_native.lib().nphm_fit_apply_gradient(
                    self.engine.handle, self.latent.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), ctypes.byref(fp),
                    g_lat.data_ptr(), stats.data_ptr(), None, int(apply_update), self.loss_terms.data_ptr(), self.grad.data_ptr(),
                    stream), 'nphm_fit_apply_gradient')
                _pose_step(self, q, g_pts.reshape(q.shape), obs_idx, float(lambdas.get('surface', 0.0)), lr, apply_update)
            elif period:
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
    """``nphm_fit_surface_grad`` on ``pts`` (n x 3), or its eval-mode form with quirk period ``period`` > 0.  ``g_lat=None``:
    no identity-code gradient (the kernels skip that work)."""
    lib = _native.lib()
    with torch.cuda.device(pts.device):
        if period:
            _native.check(lib.nphm_fit_surface_grad_quirk(eng.handle, pts.data_ptr(), pts.shape[0], period, lat.data_ptr(),
                                                          mask.data_ptr(), float(clamp), terms.data_ptr(), _native._ptr(g_lat),
                                                          g_pts.data_ptr(), None, stream), 'nphm_fit_surface_grad_quirk')
        else:
            _native.check(lib.nphm_fit_surface_grad(eng.handle, pts.data_ptr(), pts.shape[0], lat.data_ptr(), mask.data_ptr(),
                                                    float(clamp), terms.data_ptr(), _native._ptr(g_lat), g_pts.data_ptr(), None,
                                                    stream), 'nphm_fit_surface_grad')


def inference_identity_space(decoder,
                             all_obs: List[torch.Tensor],
                             lambdas,
                             n_steps,
                             schedule_cfg: Dict,
                             step_scale=1,
                             lr_scale=1,
                             poses: ObservationPoses = None):
    """Fit the identity code to point-cloud observations.  Returns ``(lat_rep_shape (1,1,D), anchors (1,K,3))``; a
    ``DeepSDF`` decoder has no anchors (``None``), as in the reference.  ``poses`` (an :class:`ObservationPoses` of
    ``len(all_obs)`` observations on their device): the observations are in their own frames and their similarity transforms
    to the model frame are fitted with the code, in place (DESIGN.md §4.24)."""
    device = all_obs[0].device
    check_poses(poses, len(all_obs), device)
    lr = 0.01 * lr_scale
    if device.type == 'cuda' and _native_npm_decoder(decoder, 1):
        fitter = NpmIdentityFitter(decoder, device, poses)
        for j in range(int(n_steps * step_scale)):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs, idx = _sample_observations(all_obs)
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr, obs_idx=_pose_rows(poses, idx, device))
        return fitter.latent.reshape(1, 1, -1).clone().requires_grad_(True), None
    if _fused_identity(decoder, grad_points=poses is not None) and device.type == 'cuda':
        fitter = IdentityFitter(decoder, device, poses)
        z_prev = fitter.latent.clone()
        for j in range(int(n_steps * step_scale)):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs, idx = _sample_observations(all_obs)
            z_prev.copy_(fitter.latent)
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr, obs_idx=_pose_rows(poses, idx, device))
        with torch.no_grad():
            _, anchors = fitter.engine.query(torch.zeros(1, 1, 3, device=device), z_prev.reshape(1, -1), eval_quirk=False)
        lat_rep_shape = fitter.latent.reshape(1, 1, -1).clone().requires_grad_(True)
        return lat_rep_shape, anchors
    return _inference_identity_space_autograd(decoder, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale, poses)


def _pose_rows(poses, idx, device):
    """The sampled rows' observation indices on the device for a posed fit (None without poses: no upload)."""
    return None if poses is None else idx.to(device=device, dtype=torch.int32)


class _TangentPoses:
    """The autograd fallback's pose: a zero tangent leaf per observation composed with the current pose (``compose_f64``);
    after ``backward`` its gradient is the pose gradient, and the update is the float64 Adam and retraction of the kernels."""

    def __init__(self, poses: ObservationPoses):
        self.poses, self.lr0, self.xi = poses, None, None

    def __call__(self, obs, idx):
        self.xi = torch.zeros(self.poses.n, 7, dtype=torch.float64, device=self.poses.device, requires_grad=True)
        return compose_f64(self.poses.table, obs, idx, self.xi)

    def step(self, lr, step):
        if self.lr0 is None:
            self.lr0 = lr
        self.poses.grad.copy_(self.xi.grad)
        self.poses.update(lr / self.lr0, step, native=False)


def _inference_identity_space_autograd(decoder, all_obs, lambdas, n_steps, schedule_cfg, step_scale=1, lr_scale=1,
                                       poses=None):
    """The composite path of :func:`inference_identity_space`: autograd through the modules (any decoder, CPU or GPU)."""
    device = all_obs[0].device
    lr = 0.01 * lr_scale
    lat_dim = decoder.lat_dim
    lat_rep_shape = torch.zeros([1, 1, lat_dim], device=device, requires_grad=True)
    opt = optim.Adam(params=[lat_rep_shape], lr=lr)
    tangent = None if poses is None else _TangentPoses(poses)
    anchors = None
    for j in range(int(n_steps * step_scale)):
        new_lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        if new_lr != lr:
            lr = new_lr
            for group in opt.param_groups:
                group['lr'] = lr
        opt.zero_grad()
        anchors = _current_anchors(decoder, lat_rep_shape, device)
        obs, idx = _sample_observations(all_obs)
        if tangent is not None:
            obs = tangent(obs, idx)
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
        if tangent is not None:
            tangent.step(lr, j + 1)
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


NATIVE_JOINT_MODES = ('compress', 'glob_only', 'expr_only')


def _native_joint(decoder, decoder_expr, device) -> bool:
    """The autograd-free joint fitter applies to a fused identity ensemble (see :func:`_fused_identity`) and a
    DeformationNetwork in eval mode on the same CUDA device whose condition is constant per query (modes compress, glob_only,
    expr_only; :class:`_IdentityRoute`).  glob_only also needs the identity code's global part to be as wide as the
    deformation network's ``lat_dim_glob_shape``."""
    from .deepSDF import DeformationNetwork
    if device.type != 'cuda' or not _fused_identity(decoder, grad_points=True) or not isinstance(decoder_expr, DeformationNetwork):
        return False
    if decoder_expr.training or decoder_expr.mode not in NATIVE_JOINT_MODES:
        return False
    if decoder_expr.mode == 'glob_only' and decoder_expr.lat_dim_glob_shape != decoder.lat_dim_glob:
        return False
    bb = decoder_expr.defDeepSDF
    return next(bb.parameters()).is_cuda and bb.num_freq_bands is None and bb.beta == 100 and bb.out_dim_net == 3


class _IdentityRoute:
    """How the identity code enters the deformation network's condition rows ``[prefix | z_ex]`` (deepSDF.py:203-224), and how
    the prefix columns of the adjoint pass's condition gradient go back to the identity code:

        mode       prefix (width P)                         d/d prefix goes to
        compress   compressor([z_id | anchors])  (32)       through the compressor to z_id and the anchors
        glob_only  z_id[:lat_dim_glob_shape]     (64)       summed over a subject's rows, added to d/d z_id[:P]
        expr_only  nothing                       (0)        nowhere

    ``z_ex`` takes the columns P: in every mode.  Only compress has an anchor term; the others hand the identity update a zero
    anchor gradient.  Shapes follow the fitter: one subject (``z_id`` D, anchors 1 x K x 3, rows nb x P) or S subjects
    (``z_id`` S x D, anchors S x K x 3, rows S nb x P); the compress arithmetic is the fitters' own, in their order."""

    def __init__(self, decoder_expr):
        self.mode = decoder_expr.mode
        if self.mode == 'compress':
            lin = decoder_expr.compressor[0] if isinstance(decoder_expr.compressor, torch.nn.Sequential) else decoder_expr.compressor
            self.Wc, self.bc = lin.weight, lin.bias
            self.width = self.Wc.shape[0]
        else:
            self.width = decoder_expr.lat_dim_glob_shape if self.mode == 'glob_only' else 0
        self._zero_anchors = None

    def prefix(self, z_id, anchors):
        """The condition prefix of each subject: P, or S x P."""
        if self.mode != 'compress':
            return z_id[..., :self.width]
        if z_id.dim() == 1:
            first = torch.cat([z_id, anchors.reshape(-1)])
            return (self.Wc * first[None, :]).sum(1) + self.bc
        first = torch.cat([z_id, anchors.reshape(z_id.shape[0], -1)], dim=1)
        return (self.Wc[None] * first[:, None, :]).sum(2) + self.bc

    def identity_gradients(self, g_lat, g_rows, anchors):
        """``(d/d z_id, d/d anchors)`` of the identity update: the surface term's ``g_lat`` (D or S x D) plus the prefix columns
        ``g_rows`` of the condition gradient (nb x P or S nb x P), and the anchor gradient (3 K or S x 3 K) it passes on."""
        D = g_lat.shape[-1]
        if self.mode == 'compress':
            if g_lat.dim() == 1:
                g_first = (self.Wc * g_rows.sum(0)[:, None]).sum(0)                    # compressor^T -> [z_id | anchors]
            else:
                g_c32 = g_rows.reshape(g_lat.shape[0], -1, self.width).sum(1)
                g_first = (self.Wc[None] * g_c32[:, :, None]).sum(1)                   # compressor^T, S x (D + 3 K)
            return (g_lat + g_first[..., :D]).contiguous(), g_first[..., D:].contiguous()
        if self._zero_anchors is None or self._zero_anchors.shape[:-1] != g_lat.shape[:-1]:
            self._zero_anchors = g_lat.new_zeros(*g_lat.shape[:-1], anchors[0].numel())
        if self.width == 0:
            return g_lat, self._zero_anchors
        g_zid = g_lat.clone()
        g_zid[..., :self.width] += g_rows.reshape(*g_lat.shape[:-1], -1, self.width).sum(-2)
        return g_zid, self._zero_anchors


def _adam_expressions(fitter, g_zex, lr, stream):
    """The update of a fixed-identity step: Adam on the expression codes alone."""
    _native.check(_native.lib().nphm_adam_step(fitter.z_ex.data_ptr(), g_zex.data_ptr(), fitter.m_ex.data_ptr(),
                                               fitter.v_ex.data_ptr(), fitter.z_ex.numel(), float(lr), fitter.t, stream),
                  'nphm_adam_step')
    return None


class JointFitter:
    """One iteration of ``inference_iterative_root_finding_joint`` (reference fitting.py:38-175) WITHOUT an autograd graph.

    The reference builds xc = p - J^-1 (F_ex(p; theta) + p - stopgrad(.)) so that value(xc) = p and d xc / d theta =
    -J^-1 dF_ex/d theta (:99-106), then calls loss.backward() (:167).  Written out:
        g_x   = d surface / d xc                                   nphm_fit_surface_grad (with d surface / d z_id)
        u     = -J^-T g_x            per point, J = I + dF_ex/dx    nphm_mlp_inverse_jacobian (forward-mode, tensor cores)
        g_c   = sum_n (dF_ex/d cond)^T u_n   per sampled scan       nphm_mlp_backward_inputs (adjoint pass, tensor cores)
        cond  = [prefix (P) | z_ex (E)]                             -> z_ex rows, and the prefix columns to z_id and the anchors
    followed by the regularisers and the two Adam updates (nphm_fit_apply_gradient, nphm_adam_step).  The prefix depends on
    the deformation mode (:class:`_IdentityRoute`): compress [compressor([z_id | anchors]) (32), whose gradient reaches the
    anchors through mlp_pos inside nphm_fit_apply_gradient], glob_only [z_id[:64]] or expr_only [nothing].

    ``fixed_identity=True`` holds ``z_id`` (set by the caller before the first step) fixed: the anchors and the condition prefix
    are computed once, the surface term runs without the identity-code gradient, and a step is the z_ex route alone
    (-J^-T g_x, adjoint pass, reg_expr, Adam).  ``loss_terms`` are then the surface call's (unweighted)."""

    def __init__(self, decoder, decoder_expr, num_observations: int, device, fixed_identity: bool = False,
                 poses: ObservationPoses = None):
        self.dec, self.dfn, self.device = decoder, decoder_expr, device
        self.fixed_identity = fixed_identity
        self.poses, self.pose_lr0 = poses, None
        self.route, self._prefix = _IdentityRoute(decoder_expr), None
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
        tensors the reference hands to its two ``Adam.step()`` calls - are returned (``d loss / d z_id`` is None with a fixed
        identity)."""
        nat, dev = _native, self.device
        nb, n_point, _ = obs.shape
        E, D = self.z_ex.shape[1], self.z_id.shape[0]
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.no_grad(), torch.cuda.device(dev):
            # condition of the deformation backbone (deepSDF.py:203-224): the identity prefix (P) | z_ex (E)
            if self._prefix is None or not self.fixed_identity:
                self.anchors = self.eng.anchors(self.z_id[None])                         # 1 x K x 3, pre-update code (:59)
                self._prefix = self.route.prefix(self.z_id, self.anchors)
            P = self.route.width
            cond = torch.cat([self._prefix[None, :].expand(nb, -1), self.z_ex[obs_idx]], dim=1).contiguous()
            # correspondence search (iterative_root_finding.py:91-168): J0^-1 at the observed points, Broyden on the device
            obs = obs.to(torch.float32).contiguous()
            if self.poses is not None:                                                   # q: the Broyden target and start
                obs = self.poses.apply(obs, obs_idx)
            _, j0_inv = self.mlp.inverse_jacobian(obs, cond)
            p, _, valid, _ = self.mlp.broyden_search(obs, cond, obs, j0_inv, max_steps=15, cvg_thresh=1e-6, dvg_thresh=0.2,
                                                     early_exit=self.early_exit)
            # implicit differentiation of the root (:99-106): J^-1 at the root
            _, j_inv = self.mlp.inverse_jacobian(p, cond)
            # surface term (:111-136): value + d/d z_id + d/d xc
            pts = p.reshape(-1, 3)
            mask = valid.reshape(-1).to(torch.uint8).contiguous()
            g_lat = None if self.fixed_identity else torch.empty(D, device=dev)
            g_pts = torch.empty_like(pts)
            _surface_grad(self.eng, pts, _quirk_period(self.dec, n_point), self.z_id, mask, clamp, self.terms, g_lat, g_pts,
                          stream)
            u = -(j_inv * g_pts.reshape(nb, n_point, 3, 1)).sum(-2)                       # -J^-T g_x
            if self.poses is not None:                                                   # d surface / d q = J^-T g_x = -u
                _pose_step(self, obs, u, obs_idx, -float(lambdas.get('surface', 0.0)), lr, apply_update)
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)     # nb x (P + E); same points as j_inv
            # expression codes: surface route + reg_expr = mean_b ||z_ex[idx_b]||^2 (:137), dense Adam over all rows (:169)
            lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, obs_idx, lam_s * g_cond[:, P:] + (2.0 * lam_e / nb) * self.z_ex[obs_idx])
            if self.fixed_identity:
                self.loss_terms.copy_(self.terms)
                return _adam_expressions(self, g_zex, lr, stream) if apply_update else (None, g_zex)
            g_zid, g_anchors = self.route.identity_gradients(g_lat, g_cond[:, :P], self.anchors)
            stats = torch.stack([self.terms[5], self.terms[0] * self.terms[5]]).nan_to_num_(0.0).contiguous()
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
    symm_dist to 0 for a DeepSDF), and Adam (``nphm_adam_step``).  With ``poses`` the sampled rows are moved into the model
    frame first and the surface call also returns the point gradient, from which the poses are fitted."""

    def __init__(self, decoder, device, poses: ObservationPoses = None):
        self.device = device
        self.poses, self.pose_lr0 = poses, None
        self.engine = decoder.engine()
        self.latent = torch.zeros(decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latent)
        self.v = torch.zeros_like(self.latent)
        self.loss_terms = torch.zeros(8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latent)
        self.t = 0
        self._ws = None

    def step(self, points: torch.Tensor, lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True,
             obs_idx: torch.Tensor = None):
        """One iteration on ``points`` (B x N x 3); with ``apply_update=False`` only ``grad`` and ``loss_terms`` (and the poses'
        ``grad``) are set.  With poses, ``obs_idx`` (B, on the device) gives each row's observation."""
        if apply_update:
            self.t += 1
        lam_s, lam_g = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(self.device):
            q = None if self.poses is None else self.poses.apply(points, obs_idx)
            pts = (points if q is None else q).reshape(1, -1, 3).to(dtype=torch.float32).contiguous()
            if self._ws is None or self._ws[0] != pts.shape[1]:
                self._ws = (pts.shape[1], self.engine.fit_workspace(1, pts.shape[1], self.device))
            terms, g_cond, g_xyz = self.engine.fit_surface_grad(pts, self.latent[None], None, clamp, want_xyz=q is not None,
                                                                workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            if q is not None:
                _pose_step(self, q, g_xyz.reshape(q.shape), obs_idx, lam_s, lr, apply_update)
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
    itself.  ``fixed_identity=True``: ``z_id`` (set by the caller) is held fixed, a step updates the expression codes alone (see
    :class:`JointFitter`)."""

    def __init__(self, decoder, decoder_expr, num_observations: int, device, fixed_identity: bool = False,
                 poses: ObservationPoses = None):
        self.device = device
        self.fixed_identity = fixed_identity
        self.poses, self.pose_lr0 = poses, None
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
            if self.poses is not None:                                                   # q: the Broyden target and start
                obs = self.poses.apply(obs, obs_idx)
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
            if self.poses is not None:                                                   # d surface / d q = J^-T g_x = -u
                _pose_step(self, obs, u, obs_idx, -lam_s, lr, apply_update)
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, obs_idx, lam_s * g_cond[:, D:] + (2.0 * lam_e / nb) * self.z_ex[obs_idx])
            if self.fixed_identity:
                return _adam_expressions(self, g_zex, lr, stream) if apply_update else (None, g_zex)
            g_zid = lam_s * (g_lat[0] + g_cond[:, :D].sum(0)) + (2.0 * lam_g) * self.z_id
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
                                           lr_scale=1,
                                           poses: ObservationPoses = None):
    """Joint identity + expression fitting with Broyden correspondences (reference :14-177).  ``poses``: the observations'
    similarity transforms to the model frame, fitted with the codes as in :func:`inference_identity_space`.

    Fused ensemble + eval-mode DeformationNetwork in mode compress (the shipped configuration), glob_only or expr_only on
    CUDA: no autograd graph at all, see :class:`JointFitter`; the same for the NPM baseline (``DeepSDF`` decoders on CUDA), see :class:`NpmJointFitter`.
    ``NPHM_JOINT_AUTOGRAD=1`` keeps both on the composite path.  Anything else: the correspondence search runs on the device (`nphm_mlp_broyden_search`), the
    surface term comes from `nphm_fit_surface_grad`, the deformation network's part of the chain stays on autograd.  Returns
    ``(lat_rep (n_obs,1,E), lat_rep_shape (1,1,D), anchors)``."""
    device = all_obs[0].device
    num_observations = len(all_obs)
    check_poses(poses, num_observations, device)
    if not os.environ.get('NPHM_JOINT_AUTOGRAD'):
        fitter = None
        if _native_joint(decoder, decoder_expr, device):
            fitter = JointFitter(decoder, decoder_expr, num_observations, device, poses=poses)
        elif _native_npm_joint(decoder, decoder_expr, device):
            fitter = NpmJointFitter(decoder, decoder_expr, num_observations, device, poses=poses)
        if fitter is not None:
            _run_joint(fitter, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)
            lat_rep = fitter.z_ex.reshape(num_observations, 1, -1).clone().requires_grad_(True)
            lat_rep_shape = fitter.z_id.reshape(1, 1, -1).clone().requires_grad_(True)
            return lat_rep, lat_rep_shape, fitter.anchors
    return _inference_joint_autograd(decoder, decoder_expr, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale,
                                     poses=poses)


def _run_joint(fitter, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale):
    """The reference loop (:38-175) around one native joint or fixed-identity fitter."""
    device = fitter.device
    lr = 0.01 * lr_scale
    for j in range(int(n_steps * step_scale)):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        obs, obs_idx = _sample_observations(all_obs)
        fitter.step(obs, obs_idx.long().to(device), lambdas, _clamp_for_iteration(j, step_scale), lr)


def _inference_joint_autograd(decoder, decoder_expr, all_obs, lambdas, n_steps, schedule_cfg, step_scale=1, lr_scale=1,
                              lat_rep_shape=None, lat_rep_init=None, poses=None):
    """The composite path of :func:`inference_iterative_root_finding_joint`: the correspondence search on the device where
    the search supports the decoder, everything else on autograd through the modules.  A given ``lat_rep_shape`` is held
    fixed (the path of :func:`inference_expression_space`): no identity optimizer, the anchors computed once, and ``z_ex``
    starts at ``lat_rep_init`` when one is given."""
    device = all_obs[0].device
    num_observations = len(all_obs)
    lat_expr_dim = decoder_expr.lat_dim_expr if hasattr(decoder_expr, 'lat_dim_expr') else 200
    lat_rep = torch.zeros([num_observations, 1, lat_expr_dim], device=device)
    if lat_rep_init is not None:
        lat_rep.copy_(lat_rep_init.detach().reshape(lat_rep.shape))
    lat_rep.requires_grad_(True)
    fixed = lat_rep_shape is not None
    if fixed:
        lat_rep_shape = lat_rep_shape.detach().reshape(1, 1, decoder.lat_dim).to(device=device, dtype=torch.float32).clone()
    else:
        lat_rep_shape = torch.zeros([1, 1, decoder.lat_dim], device=device, requires_grad=True)
    lr = 0.01 * lr_scale
    opt_expr = optim.Adam(params=[lat_rep], lr=lr)
    opts = [opt_expr] if fixed else [optim.Adam(params=[lat_rep_shape], lr=lr), opt_expr]
    anchors = None
    tangent = None if poses is None else _TangentPoses(poses)
    if fixed:
        with torch.no_grad():
            anchors = _current_anchors(decoder, lat_rep_shape, device)
    for j in range(int(n_steps * step_scale)):
        new_lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        if new_lr != lr:
            lr = new_lr
            for o in opts:
                for group in o.param_groups:
                    group['lr'] = lr
        for o in opts:
            o.zero_grad()
        if not fixed:
            anchors = _current_anchors(decoder, lat_rep_shape, device)
        obs, obs_idx = _sample_observations(all_obs)
        obs_idx = obs_idx.long().to(device)
        q = None
        if tangent is not None:                     # q: the Broyden target, d xc / d q = J^-1
            q = tangent(obs, obs_idx)
            obs = q.detach()
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
        if q is not None:
            correction = correction + torch.einsum('bnij,bnj->bni', grad_inv.detach(), q - q.detach())
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
        for o in opts:                      # the identity's optimizer first, as in the reference (:168-169)
            o.step()
        if tangent is not None:
            tangent.step(lr, j + 1)
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


def _batch_poses(poses, scans, device):
    """Checks one :class:`ObservationPoses` per scan (or ``poses=None``)."""
    if poses is None:
        return
    if len(poses) != len(scans):
        raise ValueError('%d poses for %d scans' % (len(poses), len(scans)))
    for p, all_obs in zip(poses, scans):
        check_poses(p, len(all_obs), device if device is not None else all_obs[0].device)


def _fit_posed(fit, scans, gens, lambdas, poses):
    """``fit(scans, gens, lambdas, shared)`` with the scans' poses in one shared table, written back afterwards."""
    if poses is None:
        return fit(scans, gens, lambdas)
    shared = ObservationPoses.concat(poses)
    out = fit(scans, gens, lambdas, shared)
    shared.scatter(poses)
    return out


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


def _posed_scans(poses, points: List[torch.Tensor], rows: torch.Tensor):
    """A posed batched identity step's points: the scans' sampled rows (``points[k]``: nb x n_k x 3) padded to one row block
    (S nb x n_point x 3, row r from observation ``rows[r]`` of the shared table) and moved into the model frame in one launch;
    returns that block and each scan's rows of it (nb x n_k x 3), the points the unposed step takes."""
    nb, n_point = points[0].shape[0], max(p.shape[1] for p in points)
    q, _ = _pad_rows(points, n_point)
    q = poses.apply(q, rows)
    return q, [q[k * nb:(k + 1) * nb, :p.shape[1]] for k, p in enumerate(points)]


def _rows_of_scans(g_pts: torch.Tensor, q: torch.Tensor, points: List[torch.Tensor]) -> torch.Tensor:
    """The per-scan point gradients of a batched surface call (S x n x 3, scan k's nb n_k points first) laid out as the row
    block ``q`` of :func:`_posed_scans`; the padding gets 0."""
    nb, n_point = points[0].shape[0], q.shape[1]
    if all(p.shape[1] == n_point for p in points):
        return g_pts.reshape(q.shape)
    out = torch.zeros_like(q)
    for k, p in enumerate(points):
        out[k * nb:(k + 1) * nb, :p.shape[1]] = g_pts[k, :nb * p.shape[1]].reshape(nb, p.shape[1], 3)
    return out


class BatchedIdentityFitter:
    """:class:`IdentityFitter` for S scans at once (``nphm_fit_identity_step_batched``): latents and Adam moments S x D on the
    device, one launch sequence per iteration for all scans.  In eval mode (``nphm_fit_identity_step_batched_quirk``) scan
    k's period is the points per row of its sample, so each scan gets the quirk rows of its own single-scan call.  With
    ``poses`` (one :class:`ObservationPoses` over all scans' observations, scan k's first at the sum of the earlier scans'
    counts) the step runs as :class:`IdentityFitter`'s posed step does: ``nphm_fit_surface_grad_batched`` with the point
    gradients, then ``nphm_fit_apply_gradient_batched``."""

    def __init__(self, decoder: FastEnsembleDeepSDFMirrored, n_scans: int, device, poses: ObservationPoses = None):
        self.decoder = decoder
        self.poses, self.pose_lr0 = poses, None
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

    def step(self, points: List[torch.Tensor], lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True,
             obs_idx: torch.Tensor = None):
        """One iteration; ``points[k]`` are scan k's sampled points (any shape ending in 3, lengths may differ).  With poses
        ``points[k]`` are scan k's sampled rows (nb x n_k x 3) and ``obs_idx`` (S nb, on the device) the rows' observations in
        the shared table."""
        scan_pts = points
        if self.poses is not None:
            q, scan_pts = _posed_scans(self.poses, points, obs_idx)
        pts, mask = _pad_scans([p.reshape(-1, 3).to(dtype=torch.float32) for p in scan_pts])
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
            if self.poses is not None:
                periods = self._periods([p.shape[-2] for p in points], self.device) if eval_mode else None
                terms, g_lat, g_pts = torch.empty(S, 8, device=self.device), torch.empty_like(self.latents), torch.empty_like(pts)
                if eval_mode:
                    _native.check(lib.nphm_fit_surface_grad_batched_quirk(
                        self.engine.handle, pts.data_ptr(), _native._ptr(mask), S, n, periods.data_ptr(), self.latents.data_ptr(),
                        float(clamp), terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                        'nphm_fit_surface_grad_batched_quirk')
                else:
                    _native.check(lib.nphm_fit_surface_grad_batched(
                        self.engine.handle, pts.data_ptr(), _native._ptr(mask), S, n, self.latents.data_ptr(), float(clamp),
                        terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                        'nphm_fit_surface_grad_batched')
                stats = torch.stack([terms[:, 5], terms[:, 0] * terms[:, 5]], dim=1).nan_to_num_(0.0).contiguous()
                _native.check(lib.nphm_fit_apply_gradient_batched(
                    self.engine.handle, S, self.latents.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), ctypes.byref(fp),
                    g_lat.data_ptr(), stats.data_ptr(), None, int(apply_update), self.loss_terms.data_ptr(), self.grad.data_ptr(),
                    stream), 'nphm_fit_apply_gradient_batched')
                _pose_step(self, q, _rows_of_scans(g_pts, q, points), obs_idx, float(lambdas.get('surface', 0.0)), lr,
                           apply_update)
            elif eval_mode:
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
                                     lr_scale=1,
                                     poses: List[ObservationPoses] = None):
    """:func:`inference_identity_space` for several scans (``scans[k]``: the observations of scan k) at once.  Returns
    ``[(lat_rep_shape, anchors)]`` in scan order - what the single-scan function gives when called on each scan in turn, each
    call with a fresh copy of ``lambdas``; the global CPU generator and ``lambdas`` end as those calls leave them.  Runs all
    scans in one launch sequence per iteration for the fused ensemble on CUDA (:class:`BatchedIdentityFitter`, training or eval
    mode, see :func:`_fused_identity`)
    and for the NPM baseline's ``DeepSDF`` on CUDA (:class:`BatchedNpmIdentityFitter`); any other configuration calls the
    single-scan function scan by scan.  ``poses``: one :class:`ObservationPoses` per scan, fitted in place as the single-scan
    function fits its ``poses``; all must share rates, ``fit_scale`` and ``fit`` (they update as one table)."""
    if not scans:
        return []
    _batch_poses(poses, scans, _scans_device(scans))
    fit = _identity_batch_fit(decoder, scans, n_steps, schedule_cfg, step_scale, lr_scale, posed=poses is not None)
    if fit is None:
        return _sequential(lambda e, lam: inference_identity_space(decoder, e[0], lam, n_steps, schedule_cfg, step_scale,
                                                                   lr_scale, poses=e[1]),
                           list(zip(scans, poses or [None] * len(scans))), lambdas)
    return _fit_posed(fit, scans, _sampling_plan(scans, int(n_steps * step_scale)), lambdas, poses)


def _identity_batch_fit(decoder, scans, n_steps, schedule_cfg, step_scale, lr_scale, posed: bool = False):
    """``fit(scans, gens, lambdas[, poses])``: the scan-batched identity fit with scan k drawing from ``gens[k]``, when a
    batched fitter takes this decoder on the scans' device; None when the scans are fitted one by one."""
    device = _scans_device(scans)
    npm = device is not None and device.type == 'cuda' and _native_npm_decoder(decoder, 1)
    if not npm and (device is None or device.type != 'cuda' or not (_fused_identity(decoder, posed) and _tc_ensemble(decoder))):
        return None
    return lambda chunk, gens, lambdas, poses=None: _fit_identity_batch(decoder, chunk, gens, lambdas, n_steps, schedule_cfg,
                                                                        step_scale, lr_scale, device, npm, poses)


def _sample_batch(scans, gens, offsets, device):
    """One iteration's samples of every scan, and (with poses, ``offsets`` not None) the rows' observations in the shared
    table on the device."""
    sample = [_sample_observations(all_obs, g) for all_obs, g in zip(scans, gens)]
    rows = None
    if offsets is not None:
        rows = torch.cat([i + o for (_, i), o in zip(sample, offsets)]).to(device=device, dtype=torch.int32)
    return [o for o, _ in sample], rows


def _fit_identity_batch(decoder, scans, gens, lambdas, n_steps, schedule_cfg, step_scale, lr_scale, device, npm, poses=None):
    n_iters = int(n_steps * step_scale)
    lr = 0.01 * lr_scale
    offsets = None if poses is None else [sum(len(s) for s in scans[:k]) for k in range(len(scans))]
    if npm:
        fitter = BatchedNpmIdentityFitter(decoder, len(scans), device, poses)
        for j in range(n_iters):
            lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
            obs, rows = _sample_batch(scans, gens, offsets, device)
            fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr, obs_idx=rows)
        return [(fitter.latents[k].reshape(1, 1, -1).clone().requires_grad_(True), None) for k in range(len(scans))]
    fitter = BatchedIdentityFitter(decoder, len(scans), device, poses)
    z_prev = fitter.latents.clone()
    for j in range(n_iters):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        obs, rows = _sample_batch(scans, gens, offsets, device)
        z_prev.copy_(fitter.latents)
        fitter.step(obs, lambdas, _clamp_for_iteration(j, step_scale), lr, obs_idx=rows)
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
        anchors of the S identity codes (nphm_ensemble_anchors), condition rows [prefix(z_id, anchors)[subject] | z_ex[row]]
        J0^-1, Broyden and J^-1 on all 5 S rows (per-row conditions; shorter subjects padded, the padding masked)
        nphm_fit_surface_grad_batched: per-subject surface term, d/d z_id and d/d point
        u = -J^-T g_x, one adjoint pass, the prefix columns routed to each subject's identity code (:class:`_IdentityRoute`)
        nphm_fit_apply_gradient_batched (regularisers, mlp_pos backward, Adam per subject)
        one nphm_adam_step over the expression codes of all subjects (element-wise, shared step and lr: the same as per subject).
    The expression codes are one (sum n_obs) x E tensor; subject k's rows start at ``offsets[k]``.  In eval mode a shorter
    subject's rows are padded in front instead of behind, so that every row ends with its subject's last sampled point - the
    quirk row of that subject's single-subject call - and one period, n_point, serves all subjects
    (``nphm_fit_surface_grad_batched_quirk``).  ``fixed_identity=True``: the S identity codes (set by the caller) are held
    fixed, as in :class:`JointFitter`."""

    def __init__(self, decoder, decoder_expr, num_observations: List[int], device, fixed_identity: bool = False,
                 poses: ObservationPoses = None):
        self.dec, self.dfn, self.device = decoder, decoder_expr, device
        self.fixed_identity = fixed_identity
        self.poses, self.pose_lr0 = poses, None
        self.route, self._prefix = _IdentityRoute(decoder_expr), None
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
        ``apply_update=False`` nothing is modified and ``(d loss / d z_id (S x D), [d loss / d z_ex of subject k])`` is returned
        (``d loss / d z_id`` is None with fixed identities)."""
        nat, dev = _native, self.device
        S, D = self.z_id.shape
        nb = obs[0].shape[0]
        n_point = max(o.shape[1] for o in obs)
        if apply_update:
            self.t += 1
        stream = torch.cuda.current_stream(dev).cuda_stream
        lib = nat.lib()
        with torch.no_grad(), torch.cuda.device(dev):
            if self._prefix is None or not self.fixed_identity:
                self.anchors = self.eng.anchors(self.z_id)                               # S x K x 3, pre-update codes
                self._prefix = self.route.prefix(self.z_id, self.anchors)                # S x P
            P = self.route.width
            rows = torch.cat([idx + off for idx, off in zip(obs_idx, self.offsets)])    # rows of z_ex, 5 S
            cond = torch.cat([self._prefix.repeat_interleave(nb, dim=0), self.z_ex[rows]], dim=1).contiguous()
            # every subject padded to n_point points per observation (the padding repeats a point and is masked below); in eval
            # mode in front of the row, so that its last point stays last
            front = not self.dec.training
            obs_all, keep = _pad_rows(obs, n_point, front)                                # 5 S x n_point x 3
            if self.poses is not None:                                                   # q: the Broyden target and start
                obs_all = self.poses.apply(obs_all, rows)
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
            g_lat = None if self.fixed_identity else torch.empty(S, D, device=dev)
            g_pts = torch.empty_like(pts)
            if front:
                periods = torch.full((S,), n_point, dtype=torch.int32, device=dev)
                nat.check(lib.nphm_fit_surface_grad_batched_quirk(self.eng.handle, pts.data_ptr(), mask.data_ptr(), S, n,
                                                                  periods.data_ptr(), self.z_id.data_ptr(), float(clamp),
                                                                  terms.data_ptr(), nat._ptr(g_lat), g_pts.data_ptr(),
                                                                  ws.data_ptr(), ws.numel(), stream),
                          'nphm_fit_surface_grad_batched_quirk')
            else:
                nat.check(lib.nphm_fit_surface_grad_batched(self.eng.handle, pts.data_ptr(), mask.data_ptr(), S, n,
                                                            self.z_id.data_ptr(), float(clamp), terms.data_ptr(),
                                                            nat._ptr(g_lat), g_pts.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                          'nphm_fit_surface_grad_batched')
            u = -(j_inv * g_pts.reshape(S * nb, n_point, 3, 1)).sum(-2)                  # -J^-T g_x
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)     # 5 S x (P + E)
            lam_s, lam_e = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_expr', 0.0))
            if self.poses is not None:                                                   # d surface / d q = J^-T g_x = -u
                _pose_step(self, obs_all, u, rows, -lam_s, lr, apply_update)
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, rows, lam_s * g_cond[:, P:] + (2.0 * lam_e / nb) * self.z_ex[rows])
            if self.fixed_identity:
                self.loss_terms.copy_(terms)
                if not apply_update:
                    return None, [g_zex[o:o + c] for o, c in zip(self.offsets, self.num_observations)]
                return _adam_expressions(self, g_zex, lr, stream)
            g_zid, g_anchors = self.route.identity_gradients(g_lat, g_cond[:, :P], self.anchors)
            stats = torch.stack([terms[:, 5], terms[:, 0] * terms[:, 5]], dim=1).nan_to_num_(0.0).contiguous()
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
    element-wise and the scans share the step and lr).  With ``poses`` (over all scans' observations, as for
    :class:`BatchedIdentityFitter`) the surface call also returns the point gradients, from which the poses are fitted."""

    def __init__(self, decoder, n_scans: int, device, poses: ObservationPoses = None):
        self.device = device
        self.poses, self.pose_lr0 = poses, None
        self.engine = decoder.engine()
        self.latents = torch.zeros(n_scans, decoder.lat_dim, device=device, dtype=torch.float32)
        self.m = torch.zeros_like(self.latents)
        self.v = torch.zeros_like(self.latents)
        self.loss_terms = torch.zeros(n_scans, 8, device=device, dtype=torch.float32)
        self.grad = torch.zeros_like(self.latents)
        self.t = 0
        self._ws = None

    def step(self, points: List[torch.Tensor], lambdas: Dict[str, float], clamp: float, lr: float, apply_update: bool = True,
             obs_idx: torch.Tensor = None):
        """One iteration; ``points[k]`` are scan k's sampled points (any shape ending in 3, lengths may differ); with poses as
        in :meth:`BatchedIdentityFitter.step`."""
        if apply_update:
            self.t += 1
        lam_s, lam_g = float(lambdas.get('surface', 0.0)), float(lambdas.get('reg_global', 0.0))
        with torch.no_grad(), torch.cuda.device(self.device):
            scan_pts = points
            if self.poses is not None:
                q, scan_pts = _posed_scans(self.poses, points, obs_idx)
            pts, mask = _pad_scans([p.reshape(-1, 3).to(dtype=torch.float32) for p in scan_pts])
            S, n = pts.shape[0], pts.shape[1]
            if self._ws is None or self._ws[0] != (S, n):
                self._ws = ((S, n), self.engine.fit_workspace(S, n, self.device))
            terms, g_cond, g_xyz = self.engine.fit_surface_grad_batched(pts, self.latents, mask, clamp,
                                                                        want_xyz=self.poses is not None, workspace=self._ws[1])
            self.loss_terms.copy_(terms)
            if self.poses is not None:
                _pose_step(self, q, _rows_of_scans(g_xyz, q, points), obs_idx, lam_s, lr, apply_update)
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
    subjects per batch; the caller chooses S, nothing is split.  ``fixed_identity=True``: the identity codes (set by the caller)
    are held fixed, as in :class:`JointFitter`."""

    def __init__(self, decoder, decoder_expr, num_observations: List[int], device, fixed_identity: bool = False,
                 poses: ObservationPoses = None):
        self.device = device
        self.fixed_identity = fixed_identity
        self.poses, self.pose_lr0 = poses, None
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
            if self.poses is not None:                                                   # q: the Broyden target and start
                obs_all = self.poses.apply(obs_all, rows)
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
            if self.poses is not None:                                                   # d surface / d q = J^-T g_x = -u
                _pose_step(self, obs_all, u, rows, -lam_s, lr, apply_update)
            g_cond, _ = self.mlp.backward_inputs(p, cond, u, reuse_value_pass=True)
            g_zex = torch.zeros_like(self.z_ex)
            g_zex.index_add_(0, rows, lam_s * g_cond[:, D:] + (2.0 * lam_e / nb) * self.z_ex[rows])
            if self.fixed_identity:
                if not apply_update:
                    return None, [g_zex[o:o + c] for o, c in zip(self.offsets, self.num_observations)]
                return _adam_expressions(self, g_zex, lr, stream)
            g_zid = lam_s * (g_lat + g_cond[:, :D].reshape(S, nb, D).sum(1)) + (2.0 * lam_g) * self.z_id
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
                                                   lr_scale=1,
                                                   poses: List[ObservationPoses] = None):
    """:func:`inference_iterative_root_finding_joint` for several subjects (``subjects[k]``: the observations of subject k) at
    once.  Returns ``[(lat_rep (n_obs,1,E), lat_rep_shape (1,1,D), anchors)]`` in subject order, under the contract of
    :func:`inference_identity_space_batched`.  The ensemble configurations of :func:`_native_joint` run all subjects in one
    launch sequence per iteration (:class:`BatchedJointFitter`), and so does the NPM baseline (see :func:`_native_npm_joint`,
    :class:`BatchedNpmJointFitter`); anything else - CPU, other decoders or deformation modes, ``NPHM_JOINT_AUTOGRAD=1`` -
    calls the single-subject function subject by subject.  Memory grows linearly with the number of subjects; all subjects
    must fit on the device at once (nothing is split into smaller batches).  ``poses``: one :class:`ObservationPoses` per
    subject, fitted in place; all must share rates, ``fit_scale`` and ``fit`` (they update as one table)."""
    if not subjects:
        return []
    _batch_poses(poses, subjects, _scans_device(subjects))
    fit = _joint_batch_fit(decoder, decoder_expr, subjects, n_steps, schedule_cfg, step_scale, lr_scale)
    if fit is None:
        return _sequential(lambda e, lam: inference_iterative_root_finding_joint(decoder, decoder_expr, e[0], lam, n_steps,
                                                                                 schedule_cfg, step_scale, lr_scale, poses=e[1]),
                           list(zip(subjects, poses or [None] * len(subjects))), lambdas)
    return _fit_posed(fit, subjects, _sampling_plan(subjects, int(n_steps * step_scale)), lambdas, poses)


def _joint_batch_fit(decoder, decoder_expr, subjects, n_steps, schedule_cfg, step_scale, lr_scale):
    """``fit(subjects, gens, lambdas)``: the subject-batched joint fit with subject k drawing from ``gens[k]``, when a batched
    fitter takes these decoders on the subjects' device; None when the subjects are fitted one by one."""
    device = _scans_device(subjects)
    batched = None
    if device is not None and not os.environ.get('NPHM_JOINT_AUTOGRAD'):
        if _native_npm_joint(decoder, decoder_expr, device):
            batched = BatchedNpmJointFitter
        elif _native_joint(decoder, decoder_expr, device) and _tc_ensemble(decoder):
            batched = BatchedJointFitter
    if batched is None:
        return None
    return lambda chunk, gens, lambdas, poses=None: _fit_joint_batch(batched, decoder, decoder_expr, chunk, gens, lambdas,
                                                                     n_steps, schedule_cfg, step_scale, lr_scale, device, poses)


def _run_joint_batch(fitter, subjects, gens, lambdas, n_steps, schedule_cfg, step_scale, lr_scale):
    """:func:`_run_joint` for a subject-batched fitter, subject k drawing from ``gens[k]``."""
    device = fitter.device
    lr = 0.01 * lr_scale
    for j in range(int(n_steps * step_scale)):
        lr = _apply_schedule(j, step_scale, schedule_cfg, lambdas, lr)
        sample = [_sample_observations(all_obs, g) for all_obs, g in zip(subjects, gens)]
        fitter.step([o for o, _ in sample], [i.long().to(device) for _, i in sample], lambdas,
                    _clamp_for_iteration(j, step_scale), lr)


def _fit_joint_batch(batched, decoder, decoder_expr, subjects, gens, lambdas, n_steps, schedule_cfg, step_scale, lr_scale,
                     device, poses=None):
    fitter = batched(decoder, decoder_expr, [len(s) for s in subjects], device, poses=poses)
    _run_joint_batch(fitter, subjects, gens, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)
    out = []
    for k, (off, cnt) in enumerate(zip(fitter.offsets, fitter.num_observations)):
        lat_rep = fitter.z_ex[off:off + cnt].reshape(cnt, 1, -1).clone().requires_grad_(True)
        lat_rep_shape = fitter.z_id[k].reshape(1, 1, -1).clone().requires_grad_(True)
        out.append((lat_rep, lat_rep_shape, None if fitter.anchors is None else fitter.anchors[k:k + 1].clone()))
    return out


# ------------------------------------------------------------------------------ expressions of a subject whose identity is known
def _expression_fitter(decoder, decoder_expr, device, batched: bool):
    """The native fitter class that fits expressions with a fixed identity on ``device``, or None (the autograd mirror)."""
    if device is None or os.environ.get('NPHM_JOINT_AUTOGRAD'):
        return None
    if _native_npm_joint(decoder, decoder_expr, device):
        return BatchedNpmJointFitter if batched else NpmJointFitter
    if _native_joint(decoder, decoder_expr, device) and (not batched or _tc_ensemble(decoder)):
        return BatchedJointFitter if batched else JointFitter
    return None


def _identity_row(decoder, lat_rep_shape) -> torch.Tensor:
    z = lat_rep_shape.detach()
    if z.numel() != decoder.lat_dim:
        raise ValueError('lat_rep_shape has %d entries, the identity decoder takes %d' % (z.numel(), decoder.lat_dim))
    return z.reshape(-1)


def inference_expression_space(decoder,
                               decoder_expr,
                               lat_rep_shape: torch.Tensor,
                               all_obs: List[torch.Tensor],
                               lambdas,
                               n_steps,
                               schedule_cfg: Dict,
                               step_scale=1,
                               lr_scale=1,
                               lat_reps_expr_init=None,
                               poses: ObservationPoses = None):
    """Fit expression codes to the observations ``all_obs`` of a subject whose identity code ``lat_rep_shape`` (1,1,D) is
    known, e.g. from :func:`inference_identity_space` on a neutral scan.  The loop is the reference's joint loop (:14-177) with
    ``lat_rep_shape`` held fixed: the same 5-of-K observation draws from torch's global CPU generator, lr / lambda / clamp
    schedules (``lambdas`` is mutated as there), surface term at the Broyden roots with the implicit-differentiation correction,
    and ``reg_expr``; the identity regularisers have no gradient w.r.t. the expression codes.  ``z_ex`` starts at
    ``lat_reps_expr_init`` (K,1,E) or at zeros.  ``lat_rep_shape`` is not modified.  Returns ``(lat_reps_expr (K,1,E),
    anchors)``: the anchors of the identity code (None for a ``DeepSDF`` identity decoder).

    Runs natively (:class:`JointFitter` / :class:`NpmJointFitter` with ``fixed_identity=True``) for the configurations of
    :func:`inference_iterative_root_finding_joint`; anything else - CPU, other decoders, ``NPHM_JOINT_AUTOGRAD=1`` - runs the
    same loop on autograd.  ``poses``: each observation's similarity transform to the model frame, fitted with the
    expression codes as in :func:`inference_identity_space` (e.g. the frames of a capture in which the head moves)."""
    device = all_obs[0].device
    K = len(all_obs)
    check_poses(poses, K, device)
    z_id = _identity_row(decoder, lat_rep_shape)
    cls = _expression_fitter(decoder, decoder_expr, device, batched=False)
    if cls is None:
        lat_rep, _, anchors = _inference_joint_autograd(decoder, decoder_expr, all_obs, lambdas, n_steps, schedule_cfg,
                                                        step_scale, lr_scale, lat_rep_shape=z_id,
                                                        lat_rep_init=lat_reps_expr_init, poses=poses)
        return lat_rep, anchors
    fitter = cls(decoder, decoder_expr, K, device, fixed_identity=True, poses=poses)
    fitter.z_id.copy_(z_id)
    if lat_reps_expr_init is not None:
        fitter.z_ex.copy_(lat_reps_expr_init.detach().reshape(fitter.z_ex.shape))
    _run_joint(fitter, all_obs, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)
    return fitter.z_ex.reshape(K, 1, -1).clone().requires_grad_(True), fitter.anchors


def inference_expression_space_batched(decoder,
                                       decoder_expr,
                                       subjects,
                                       lambdas,
                                       n_steps,
                                       schedule_cfg: Dict,
                                       step_scale=1,
                                       lr_scale=1,
                                       poses: List[ObservationPoses] = None):
    """:func:`inference_expression_space` for several subjects at once.  ``subjects[k]`` is ``(lat_rep_shape, all_obs)`` or
    ``(lat_rep_shape, all_obs, lat_reps_expr_init)``; to track the T frames of one person, pass T single-observation entries
    that share one ``lat_rep_shape``.  Returns ``[(lat_reps_expr, anchors)]`` in subject order under the contract of
    :func:`inference_identity_space_batched`: what the single-subject function gives when called on each entry in turn, each
    call with a fresh copy of ``lambdas``, and the global CPU generator and ``lambdas`` end as those calls leave them.  The
    configurations of :func:`inference_iterative_root_finding_joint_batched` run all subjects in one launch sequence per
    iteration (:class:`BatchedJointFitter` / :class:`BatchedNpmJointFitter` with ``fixed_identity=True``); anything else calls
    the single-subject function subject by subject.  ``poses``: one :class:`ObservationPoses` per entry, fitted in place; all
    must share rates, ``fit_scale`` and ``fit`` (they update as one table)."""
    if not subjects:
        return []
    entries = [(e[0], e[1], e[2] if len(e) > 2 else None) for e in subjects]
    scans = [e[1] for e in entries]
    device = _scans_device(scans)
    _batch_poses(poses, scans, device)
    cls = _expression_fitter(decoder, decoder_expr, device, batched=True)
    if cls is None:
        return _sequential(lambda e, lam: inference_expression_space(decoder, decoder_expr, e[0], e[1], lam, n_steps,
                                                                     schedule_cfg, step_scale, lr_scale, e[2], poses=e[3]),
                           [e + (p,) for e, p in zip(entries, poses or [None] * len(entries))], lambdas)
    gens = _sampling_plan(scans, int(n_steps * step_scale))
    shared = None if poses is None else ObservationPoses.concat(poses)
    fitter = cls(decoder, decoder_expr, [len(o) for o in scans], device, fixed_identity=True, poses=shared)
    fitter.z_id.copy_(torch.stack([_identity_row(decoder, e[0]) for e in entries]))
    for (_, _, init), off, cnt in zip(entries, fitter.offsets, fitter.num_observations):
        if init is not None:
            fitter.z_ex[off:off + cnt].copy_(init.detach().reshape(cnt, -1))
    _run_joint_batch(fitter, scans, gens, lambdas, n_steps, schedule_cfg, step_scale, lr_scale)
    if shared is not None:
        shared.scatter(poses)
    return [(fitter.z_ex[off:off + cnt].reshape(cnt, 1, -1).clone().requires_grad_(True),
             None if fitter.anchors is None else fitter.anchors[k:k + 1].clone())
            for k, (off, cnt) in enumerate(zip(fitter.offsets, fitter.num_observations))]
