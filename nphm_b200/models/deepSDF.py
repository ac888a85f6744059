"""Drop-in mirror of the reference module ``NPHM.models.deepSDF``.

Reference interface (file:line):
  * ``DeepSDF``              src/NPHM/models/deepSDF.py:6-89
  * ``sample_point_feature`` src/NPHM/models/deepSDF.py:92-115 (duplicate of the ensemble one)
  * ``DeformationNetwork``   src/NPHM/models/deepSDF.py:118-239

Parameter names (``lin{i}.weight/bias``, ``compressor.0.*``, ``defDeepSDF.lin{i}.*``) and
constructor signatures are those of the reference so checkpoints load with ``strict=True``.
As in :mod:`.EnsembledDeepSDF`, CUDA no-grad calls with a per-query-constant condition run in
the native sm_90a MLP path; everything else uses a PyTorch composite that keeps autograd.
``forward_native_grad`` is the explicit first-order training path: native forward and native
backward (weight, bias, condition and point gradients), for a condition that is constant per query.
``DeepSDF.forward_with_gradient_native`` returns the SDF and its spatial gradient; its backward differentiates both
(the second-order terms of the stage-1 loss) natively.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from torch.autograd.function import once_differentiable

from .. import _native
from . import _composite
from .EnsembledDeepSDF import sample_point_feature  # same function in the reference (:92-115)

_SQRT2 = math.sqrt(2.0)


@once_differentiable
def _native_backward(ctx, engine_backward, p0, *upstream):
    """Backward of the native Functions below: ``engine_backward(workspace, *upstream, ...)`` computes what
    ``needs_input_grad`` asks for; the inputs are (engine, xyz, cond, [noise,] lin0.weight, lin0.bias, ...) with the
    parameters from index ``p0`` on."""
    ws, *params = ctx.saved_tensors                   # raises if a parameter was changed in place since the forward
    need = ctx.needs_input_grad
    gw, gb, g_cond, g_xyz = engine_backward(ws, *upstream, weights=any(need[p0::2]), biases=any(need[p0 + 1::2]),
                                            want_cond=need[2], want_xyz=need[1])
    grads = [None, g_xyz, g_cond] + [None] * (p0 - 3)
    for i in range(len(params) // 2):
        grads.append(gw[i] if need[p0 + 2 * i] else None)
        grads.append(gb[i] if need[p0 + 1 + 2 * i] else None)
    return tuple(grads)


class _NativeTrainFn(torch.autograd.Function):
    """``DeepSDF`` stack with a per-query condition on the native training kernels (``nphm_mlp_train_forward`` /
    ``_backward``): xyz B x N x 3, cond B x lat_dim, noise B x N x d (added to the leading ``d`` condition columns of each
    point, no gradient) or None, then the ``lin{l}.weight / bias`` parameters.  First order only."""

    @staticmethod
    def forward(ctx, engine, xyz, cond, noise, *params):
        out, ws = engine.train_forward(xyz, cond, noise)
        ctx.engine = engine
        ctx.noise_dim = 0 if noise is None else noise.shape[-1]
        ctx.save_for_backward(ws, *params)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if torch.is_grad_enabled():
            raise RuntimeError('forward_native_grad is differentiable to first order only: a double backward '
                               '(create_graph=True) through it is not supported; use the composite forward() instead')
        return _native_backward(ctx, ctx.engine.train_backward, 4, grad_out, ctx.noise_dim)


class _NativeSdfGradFn(torch.autograd.Function):
    """One-output ``DeepSDF`` stack on the native kernels (``nphm_mlp_sdfgrad_forward`` / ``_backward``): xyz B x N x 3,
    cond B x lat_dim, then the ``lin{l}.weight / bias`` parameters -> (sdf B x N x 1, d sdf / d xyz B x N x 3).  The backward
    takes upstream gradients of both outputs (the weight gradient of the gradient output is the second-order part);
    differentiable to first order only."""

    @staticmethod
    def forward(ctx, engine, xyz, cond, *params):
        sdf, grad, ws = engine.sdfgrad_forward(xyz, cond)
        ctx.engine = engine
        ctx.save_for_backward(ws, *params)
        return sdf, grad

    @staticmethod
    def backward(ctx, grad_sdf, grad_grad):
        if torch.is_grad_enabled():
            raise RuntimeError('forward_with_gradient_native is differentiable to first order only: a double backward '
                               '(create_graph=True) through it is not supported; use the composite forward() instead')
        return _native_backward(ctx, ctx.engine.sdfgrad_backward, 3, grad_sdf, grad_grad)


class DeepSDF(nn.Module):
    """Plain DeepSDF MLP: ``[xyz(+posenc) | latent] -> hidden x nlayers -> out_dim`` with the input
    re-injected (and the sum scaled by 1/sqrt(2)) at layer ``nlayers // 2``."""

    def __init__(
            self,
            lat_dim,
            hidden_dim,
            nlayers=8,
            geometric_init=True,
            radius_init=1,
            beta=100,
            out_dim=1,
            num_freq_bands=None,
            input_dim=3,
    ):
        super().__init__()
        d_spatial = input_dim if num_freq_bands is None else input_dim * (2 * num_freq_bands + 1)
        d_in = lat_dim + d_spatial
        self.lat_dim = lat_dim
        self.input_dim = input_dim
        self.out_dim_net = out_dim
        widths = [d_in] + [hidden_dim] * nlayers + [out_dim]
        self.num_layers = len(widths)
        self.skip_in = [nlayers // 2]
        self.num_freq_bands = num_freq_bands
        if num_freq_bands is not None:
            self.freq_bands = 2 ** torch.arange(num_freq_bands)

        for layer in range(self.num_layers - 1):
            fan_out = widths[layer + 1] - (d_in if layer + 1 in self.skip_in else 0)
            lin = nn.Linear(widths[layer], fan_out)
            if geometric_init and layer == self.num_layers - 2:
                # sphere-like initialisation of the output layer (reference :47-53)
                nn.init.normal_(lin.weight, mean=np.sqrt(np.pi) / np.sqrt(widths[layer]), std=0.00001)
                nn.init.constant_(lin.bias, -radius_init)
            setattr(self, 'lin' + str(layer), lin)

        self.beta = beta
        self.activation = nn.Softplus(beta=beta) if beta > 0 else nn.ReLU()
        self._engine = None

    def engine(self) -> "_native.MlpEngine":
        if self._engine is None:
            self._engine = _native.MlpEngine(self)
        self._engine.refresh(self)
        return self._engine

    def _fused_ok(self, xyz, lat_rep) -> bool:
        if not xyz.is_cuda or self.num_freq_bands is not None or self.beta != 100:
            return False
        n_lin = self.num_layers - 1
        hidden = _native.hidden_width(self, n_lin)
        if not _native.stack_supported(n_lin - 1, hidden, self.lat_dim, self.out_dim_net):
            return False             # shapes the native stack builder rejects: PyTorch composite path
        if torch.is_grad_enabled() and (xyz.requires_grad or lat_rep.requires_grad
                                        or any(p.requires_grad for p in self.parameters())):
            return False
        return xyz.dtype == torch.float32 and xyz.dim() == 3

    def native_grad_supported(self, xyz, lat_rep=None) -> bool:
        """Whether :meth:`forward_native_grad` takes these points: CUDA fp32 B x N x 3, no positional encoding, Softplus(100),
        a depth / width the native stack builder accepts (and, if given, a condition that is B x D or B x 1 x D)."""
        n_lin = self.num_layers - 1
        if lat_rep is not None and not (lat_rep.dim() == 2 or lat_rep.shape[1] == 1 or lat_rep.stride(1) == 0):
            return False
        return (xyz.is_cuda and xyz.dtype == torch.float32 and xyz.dim() == 3 and self.num_freq_bands is None
                and self.beta == 100 and next(self.parameters()).dtype == torch.float32
                and _native.stack_supported(n_lin - 1, _native.hidden_width(self, n_lin), self.lat_dim, self.out_dim_net))

    def _native_train(self, xyz, cond, noise=None):
        """xyz B x N x 3, cond B x lat_dim (differentiable), noise B x N x d or None -> B x N x out_dim."""
        if not self.native_grad_supported(xyz):
            raise _native.NativeError('forward_native_grad: unsupported input or network (needs CUDA fp32 B x N x 3 points, '
                                      'no positional encoding, Softplus(beta=100), a stack the native builder accepts)')
        params = []
        for i in range(self.num_layers - 1):
            lin = getattr(self, 'lin%d' % i)
            params += [lin.weight, lin.bias]
        return _NativeTrainFn.apply(self.engine(), xyz, cond, None if noise is None else noise.detach(), *params)

    def forward_native_grad(self, xyz, lat_rep, anchors=None):
        """:meth:`forward` on the native training kernels, differentiable to first order (weights, biases, ``lat_rep``,
        ``xyz``).  ``lat_rep``: B x D, B x 1 x D, or B x N x D equal for all points of a query; of a B x N x D tensor the
        gradient reaches the first row (an ``expand`` / ``repeat`` of a B x 1 x D code passes the reference's gradient on)."""
        cond = _native.constant_latent_rows(lat_rep)
        if cond is None:
            raise ValueError('forward_native_grad: the condition must be constant over the points of a query')
        return self._native_train(xyz, cond), None

    def sdfgrad_supported(self, xyz, lat_rep=None) -> bool:
        """Whether :meth:`forward_with_gradient_native` takes these points: what :meth:`native_grad_supported` asks, and
        one output."""
        return self.out_dim_net == 1 and self.native_grad_supported(xyz, lat_rep)

    def forward_with_gradient_native(self, xyz, lat_rep):
        """``(sdf B x N x 1, d sdf / d xyz B x N x 3)`` on the native kernels: the reference's ``forward`` followed by
        ``gradient(sdf, xyz)`` (diff_operators.py), differentiable to first order in the parameters, ``lat_rep`` and ``xyz``,
        so a loss on the gradient (normals, eikonal) trains the weights without a double backward in PyTorch.  ``lat_rep``
        as in :meth:`forward_native_grad`.  Raises ``ValueError`` for a stack or input it does not support (more than one
        output, ReLU, positional encoding, not CUDA fp32)."""
        if not self.sdfgrad_supported(xyz, lat_rep):
            raise ValueError('forward_with_gradient_native: unsupported input or network (needs CUDA fp32 B x N x 3 points, '
                             'one output, no positional encoding, Softplus(beta=100), a stack the native builder accepts)')
        cond = _native.constant_latent_rows(lat_rep)
        if cond is None:
            raise ValueError('forward_with_gradient_native: the condition must be constant over the points of a query')
        params = []
        for i in range(self.num_layers - 1):
            lin = getattr(self, 'lin%d' % i)
            params += [lin.weight, lin.bias]
        return _NativeSdfGradFn.apply(self.engine(), xyz, cond, *params)

    def forward(self, xyz, lat_rep, anchors=None):
        if self._fused_ok(xyz, lat_rep):
            cond = _native.constant_latent_rows(lat_rep)
            if cond is not None:
                return self.engine().query(xyz, cond), None
        return self._forward_composite(xyz, lat_rep), None

    def _forward_composite(self, xyz, lat_rep):
        if self.num_freq_bands is not None:
            feats = [xyz]
            for freq in self.freq_bands:
                feats += [torch.sin(xyz * freq), torch.cos(xyz * freq)]
            xyz = torch.cat(feats, dim=-1)
        if lat_rep.shape[-2] == 1 and xyz.shape[-2] != 1:
            lat_rep = lat_rep.expand(*xyz.shape[:-1], lat_rep.shape[-1])
        layers = [getattr(self, 'lin%d' % i) for i in range(self.num_layers - 1)]
        return _composite.skip_mlp(torch.cat([xyz, lat_rep], dim=-1), layers, self.skip_in, self.activation)


def _input_jacobian(backbone: DeepSDF, xyz, cond):
    """Forward-mode derivative of the backbone output w.r.t. ``xyz`` (the condition does not depend on the point):
    returns ``(out  ... x out_dim,  J  ... x out_dim x 3)``.  Same function as three reverse-mode passes through
    :meth:`DeepSDF._forward_composite` (what the reference's ``jac`` does, diff_operators.py:26-54) at a third of the
    launches: the three tangents ride through the layers as one batched matmul,
    ``T_{l+1} = sigmoid(beta z_l) * (T_l W_l^T)``."""
    if cond.shape[-2] == 1 and xyz.shape[-2] != 1:
        cond = cond.expand(*xyz.shape[:-1], cond.shape[-1])
    inp = torch.cat([xyz, cond], dim=-1)
    h, T = inp, None
    last = backbone.num_layers - 2
    for layer in range(last + 1):
        lin = getattr(backbone, 'lin' + str(layer))
        W = lin.weight
        if layer in backbone.skip_in:
            wh = h.shape[-1]
            h = torch.cat([h, inp], dim=-1) / _SQRT2
            dz = (torch.matmul(T, W[:, :wh].t()) + W[:, wh:wh + 3].t()) / _SQRT2
        elif T is None:
            dz = W[:, :3].t().expand(*xyz.shape[:-1], 3, W.shape[0])
        else:
            dz = torch.matmul(T, W.t())
        z = lin(h)
        if layer < last:
            h = backbone.activation(z)
            T = torch.sigmoid(backbone.beta * z).unsqueeze(-2) * dz
        else:
            return z, dz.transpose(-1, -2)


class DeformationNetwork(nn.Module):
    """Forward deformation field F_ex(x; z_ex, z_id): canonical point -> offset.

    ``mode='compress'`` (the shipped configuration, ``scripts/configs/nphm_def.yaml``) conditions a
    :class:`DeepSDF` backbone on ``[Linear([z_id | anchors]) (32) | z_ex]``; the other four modes of the
    reference are kept for API completeness (composite path only)."""

    def __init__(
            self,
            mode,
            lat_dim_expr,
            lat_dim_id,
            lat_dim_glob_shape,
            lat_dim_loc_shape,
            n_loc,
            anchors,
            hidden_dim,
            nlayers=8,
            out_dim=1,
            input_dim=3,
    ):
        super().__init__()
        self.mode = mode
        self.lat_dim_glob_shape = lat_dim_glob_shape
        self.lat_dim_loc_shape = lat_dim_loc_shape
        self.lat_dim_expr = lat_dim_expr
        self.input_dim = input_dim
        self.num_kps = n_loc
        self.out_dim = out_dim + 1

        if mode == 'glob_only':
            self.lat_dim = lat_dim_glob_shape + lat_dim_expr
        elif mode == 'expr_only':
            self.lat_dim = lat_dim_expr
        elif mode == 'interpolate':
            self.lat_dim = lat_dim_glob_shape + lat_dim_expr + lat_dim_loc_shape
        elif mode == 'compress':
            self.lat_dim = lat_dim_expr + lat_dim_id
            self.compressor = nn.Sequential(
                nn.Linear((lat_dim_loc_shape + 3) * n_loc + lat_dim_loc_shape + lat_dim_glob_shape, 32))
        elif mode == 'GNN':
            self.lat_dim = lat_dim_expr * 2
            self.pos_enc = nn.Sequential(nn.Linear(3, lat_dim_loc_shape), nn.ReLU(),
                                         nn.Linear(lat_dim_loc_shape, lat_dim_loc_shape))
            self.local_combiner = nn.Sequential(nn.Linear(lat_dim_loc_shape, lat_dim_loc_shape), nn.ReLU(),
                                                nn.Linear(lat_dim_loc_shape, lat_dim_loc_shape))
            self.global_combiner = nn.Sequential(
                nn.Linear(lat_dim_glob_shape + n_loc * lat_dim_loc_shape, 512), nn.ReLU(),
                nn.Linear(512, lat_dim_expr))
        else:
            raise ValueError('Unknown mode!')

        self.defDeepSDF = DeepSDF(lat_dim=self.lat_dim,
                                  hidden_dim=hidden_dim,
                                  nlayers=nlayers,
                                  geometric_init=False,
                                  out_dim=out_dim,
                                  input_dim=input_dim).float()
        self.anchors = anchors

    # ------------------------------------------------------------------
    def _condition(self, xyz, lat_rep, anchors, per_point: bool):
        """Condition vector of the backbone.  ``per_point=False`` returns ``B x 1 x C`` when the
        mode allows a per-query constant (used by the fused path)."""
        B, N, _ = xyz.shape
        E = self.lat_dim_expr
        if self.mode == 'glob_only':
            return torch.cat([lat_rep[..., :self.lat_dim_glob_shape], lat_rep[..., -E:]], dim=-1)
        if self.mode == 'expr_only':
            return lat_rep[..., -E:]
        if self.mode == 'interpolate':
            loc = lat_rep[:, 0, self.lat_dim_glob_shape:-E - self.lat_dim_loc_shape] \
                .reshape(B, self.num_kps, self.lat_dim_loc_shape)
            a0 = anchors[:, 0] if anchors.dim() == 4 else anchors
            interp = sample_point_feature(xyz[..., :3], a0[..., :3], loc.unsqueeze(1), background=False)
            lat_n = lat_rep.expand(B, N, lat_rep.shape[-1])
            return torch.cat([lat_n[..., :self.lat_dim_glob_shape], interp, lat_n[..., -E:]], dim=-1)
        if self.mode == 'compress':
            # uses the identity code and anchors of point 0 only (reference :218-219)
            a0 = anchors[:, 0] if anchors.dim() == 4 else anchors                 # B x K x 3
            first = torch.cat([lat_rep[:, 0, :-E], a0.reshape(B, -1)], dim=-1)     # B x 1461
            compressed = self.compressor(first).unsqueeze(1)                      # B x 1 x 32
            if per_point or self.training:
                compressed = compressed.expand(B, N, compressed.shape[-1])
                if self.training:
                    compressed = compressed + torch.randn(compressed.shape, device=compressed.device) / 200
                return torch.cat([compressed, lat_rep[..., -E:].expand(B, N, E)], dim=-1)
            return torch.cat([compressed, lat_rep[:, :1, -E:]], dim=-1)           # B x 1 x 232
        if self.mode == 'GNN':
            a0 = anchors[:, 0] if anchors.dim() == 4 else anchors
            offs = self.pos_enc(a0)
            g = self.lat_dim_glob_shape
            loc = lat_rep[:, 0, g:g + self.num_kps * self.lat_dim_loc_shape] \
                .reshape(B, self.num_kps, self.lat_dim_loc_shape)
            combined = self.global_combiner(
                torch.cat([lat_rep[:, 0, :g], self.local_combiner(offs + loc).reshape(B, -1)], dim=-1))
            return torch.cat([combined.unsqueeze(1).expand(B, N, combined.shape[-1]),
                              lat_rep[..., -E:].expand(B, N, E)], dim=-1)
        raise ValueError('Unknown mode')

    def offset_jacobian(self, xyz, lat_rep, anchors):
        """``d offsets / d xyz`` (B x N x 3 x 3) by forward-mode differentiation, or ``None`` when the fast path does not
        apply (condition depends on the point, positional encoding, ReLU backbone, training-mode noise)."""
        backbone = self.defDeepSDF
        if (self.training or self.mode not in ('compress', 'expr_only', 'glob_only') or backbone.num_freq_bands is not None
                or backbone.beta <= 0 or 0 in backbone.skip_in or xyz.dim() != 3):
            return None
        cond = self._condition(xyz, lat_rep, anchors, per_point=lat_rep.shape[1] != 1)
        _, J = _input_jacobian(backbone, xyz, cond)
        return J[..., :3, :]

    def native_grad_supported(self, xyz, lat_rep) -> bool:
        """Whether :meth:`forward_native_grad` takes this call (mode, backbone, points, a condition constant per query)."""
        if xyz.dim() < 3:
            xyz = xyz.unsqueeze(0)
        return (self.mode in ('compress', 'expr_only', 'glob_only') and self.defDeepSDF.native_grad_supported(xyz)
                and (lat_rep.dim() == 2 or lat_rep.shape[1] == 1 or lat_rep.stride(1) == 0))

    def forward_native_grad(self, xyz, lat_rep, anchors):
        """:meth:`forward` on the native training kernels, differentiable to first order.  ``lat_rep``: B x 1 x D (or B x D,
        or B x N x D equal over the points; see :meth:`DeepSDF.forward_native_grad` for its gradient).  In ``compress`` mode
        ``compressor([z_id | anchors])`` stays in autograd, and in train mode the noise is drawn by the reference's own call
        (``torch.randn(B, N, 32) / 200``, deepSDF.py:220-221), so a seeded run sees the same noise as :meth:`forward`."""
        if xyz.dim() < 3:
            xyz = xyz.unsqueeze(0)
        if self.mode not in ('compress', 'expr_only', 'glob_only'):
            raise ValueError('forward_native_grad: mode %r keeps the composite path' % self.mode)
        lat = _native.constant_latent_rows(lat_rep)
        if lat is None:
            raise ValueError('forward_native_grad: the condition must be constant over the points of a query')
        B, N, _ = xyz.shape
        E = self.lat_dim_expr
        noise = None
        if self.mode == 'compress':
            a0 = anchors[:, 0] if anchors.dim() == 4 else anchors
            compressed = self.compressor(torch.cat([lat[:, :-E], a0.reshape(B, -1)], dim=-1))          # B x 32
            if self.training:
                noise = torch.randn((B, N, compressed.shape[-1]), device=compressed.device) / 200
            cond = torch.cat([compressed, lat[:, -E:]], dim=-1)
        elif self.mode == 'glob_only':
            cond = torch.cat([lat[:, :self.lat_dim_glob_shape], lat[:, -E:]], dim=-1)
        else:
            cond = lat[:, -E:]
        pred = self.defDeepSDF._native_train(xyz, cond, noise)
        return pred[..., :3], pred[..., -1:]

    def forward(self,
                xyz: torch.Tensor,
                lat_rep: torch.Tensor,
                anchors: Optional[torch.Tensor]) -> (torch.Tensor, torch.Tensor):
        """xyz: B x N x 3; lat_rep: B x N|1 x (lat_id + lat_expr) = ``[z_id | z_ex]``;
        anchors: B x N x K x 3 or B x K x 3.  Returns ``(offsets B x N x 3, last channel B x N x 1)``."""
        if xyz.dim() < 3:
            xyz = xyz.unsqueeze(0)
        backbone = self.defDeepSDF
        fused = (backbone._fused_ok(xyz, lat_rep) and not self.training
                 and self.mode in ('compress', 'expr_only', 'glob_only')
                 and not (anchors is not None and torch.is_grad_enabled() and anchors.requires_grad))
        if fused:
            lat = _native.constant_latent_rows(lat_rep)
            if lat is not None:
                cond = self._condition(xyz, lat.unsqueeze(1), anchors, per_point=False)   # B x 1 x C
                pred = backbone.engine().query(xyz, cond[:, 0])
                return pred[..., :3], pred[..., -1:]
        cond = self._condition(xyz, lat_rep, anchors, per_point=True)
        pred = backbone._forward_composite(xyz, cond)
        return pred[..., :3], pred[..., -1:]
