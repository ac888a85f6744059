"""Drop-in mirror of the reference module ``NPHM.models.EnsembledDeepSDF``.

Reference interface (file:line, relative to the reference checkout):
  * ``EnsembledLinear``            src/NPHM/models/EnsembledDeepSDF.py:8-55
  * ``EnsembledDeepSDF``           src/NPHM/models/EnsembledDeepSDF.py:58-126
  * ``sample_point_feature``       src/NPHM/models/EnsembledDeepSDF.py:129-150
  * ``FastEnsembleDeepSDFMirrored`` src/NPHM/models/EnsembledDeepSDF.py:153-267

Same class names, constructor signatures, parameter names/shapes (``state_dict`` loads with
``strict=True``), attributes and return values.  Two execution paths:

  * **fused**  - CUDA tensors, autograd not recording: one call into ``libnphm_b200.so``
    (hand-written sm_90a kernels, see ``nphm_b200/csrc``).  This is the product path; it raises
    if the native library is missing, it never falls back.
  * **composite** - anything that needs autograd (training, double backward for the eikonal /
    normal losses of ``scripts/training``) or runs on CPU tensors (host-logic tests): stock
    PyTorch ops, written independently of the reference but computing the same function.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from .. import _native
from . import _composite


class _NativeEnsembleSdfGradFn(torch.autograd.Function):
    """The members of ``FastEnsembleDeepSDFMirrored`` on the native kernels (``nphm_ensemble_sdfgrad_forward`` /
    ``_backward``): xyz_local members x B x N x 3 (each member's frame, mirror applied), cond members x B x (G + L), then the
    ``ensembled_deep_sdf.lin{l}.weight / bias`` parameters -> (s members x B x N, grad_local s members x B x N x 3).  The
    backward takes upstream gradients of both outputs; differentiable to first order only."""

    @staticmethod
    def forward(ctx, engine, xyz_local, cond, *params):
        s, g, ws = engine.sdfgrad_forward(xyz_local, cond)
        ctx.engine = engine
        ctx.layer_shapes = [tuple(p.shape) for p in params[0::2]]
        ctx.save_for_backward(ws, *params)
        return s, g

    @staticmethod
    def backward(ctx, grad_s, grad_g):
        if torch.is_grad_enabled():
            raise RuntimeError('forward_with_gradient_native is differentiable to first order only: a double backward '
                               '(create_graph=True) through it is not supported; use the composite forward() instead')
        from .deepSDF import _native_backward

        def engine_backward(ws, gs, gg, **kw):
            return ctx.engine.sdfgrad_backward(ws, gs, gg, ctx.layer_shapes, **kw)
        return _native_backward(ctx, engine_backward, 3, grad_s, grad_g)


def _member_to_set(ensemble_size: int, n_symm: int) -> torch.Tensor:
    """member k -> weight-set index (reference :43-45): pairs (2i,2i+1), i<n_symm share set i."""
    k = torch.arange(ensemble_size)
    return torch.where(k < 2 * n_symm, k // 2, k - n_symm)


class EnsembledLinear(nn.Module):
    """``ensemble_size`` independent affine maps evaluated at once; the first ``n_symm`` weight
    sets are shared by two (mirror-symmetric) members each.  Parameters hold
    ``ensemble_size - n_symm`` sets, exactly as the reference (:21-23)."""

    def __init__(self, ensemble_size, n_symm, in_features, out_features, bias=True):
        super().__init__()
        self.ensemble_size = ensemble_size
        self.n_symm = n_symm
        self.in_features = in_features
        self.out_features = out_features
        n_sets = ensemble_size - n_symm
        self.weight = nn.Parameter(torch.empty(n_sets, out_features, in_features))
        if bias:
            self.bias = nn.Parameter(torch.empty(n_sets, out_features))
        else:
            self.register_parameter('bias', None)
        self.register_buffer('_set_of_member', _member_to_set(ensemble_size, n_symm), persistent=False)
        self.reset_parameters()

    def reset_parameters(self):
        # one nn.Linear-style init per weight set, consuming the RNG in the reference's order
        # (:28-35) so that equal seeds give equal parameters.
        with torch.no_grad():
            for s in range(self.weight.shape[0]):
                nn.init.kaiming_uniform_(self.weight[s], a=math.sqrt(5))
                if self.bias is not None:
                    bound = 1.0 / math.sqrt(self.in_features) if self.in_features > 0 else 0.0
                    nn.init.uniform_(self.bias[s], -bound, bound)

    def forward(self, input):
        """A x M x D_in -> A x M x D_out."""
        return _composite.ensembled_affine(input, self.weight, self.bias, self._set_of_member)


class EnsembledDeepSDF(nn.Module):
    """A stack of :class:`EnsembledLinear` with one skip re-injection of the input at layer
    ``nlayers // 2`` and ``Softplus(beta=100)`` between layers (reference :58-126)."""

    def __init__(self, ensemble_size, n_symm, lat_dim, hidden_dim, nlayers, out_dim=1, input_dim=3):
        super().__init__()
        d_in = input_dim + lat_dim
        self.ensemble_size = ensemble_size
        self.n_symm = n_symm
        self.lat_dim = lat_dim
        self.input_dim = input_dim
        widths = [d_in] + [hidden_dim] * nlayers + [out_dim]
        self.num_layers = len(widths)
        self.skip_in = [nlayers // 2]
        for layer in range(self.num_layers - 1):
            fan_out = widths[layer + 1]
            if layer + 1 in self.skip_in:
                fan_out -= d_in          # leave room for the re-injected input
            setattr(self, 'lin' + str(layer),
                    EnsembledLinear(ensemble_size, n_symm, widths[layer], fan_out))
        self.activation = nn.Softplus(beta=100)

    def forward(self, xyz, lat_rep):
        """xyz: A x B x nP x 3, lat_rep: A x B x nP x F  ->  A x B x nP x out_dim (A = ensemble members)."""
        A, B, nP, _ = xyz.shape
        layers = [getattr(self, 'lin%d' % i) for i in range(self.num_layers - 1)]
        inp = torch.cat([xyz, lat_rep], dim=-1).reshape(A, B * nP, -1)
        return _composite.skip_mlp(inp, layers, self.skip_in, self.activation).reshape(A, B, nP, -1)


def sample_point_feature(q, p, fea, var=0.1 ** 2, background=False):
    """Gaussian blend of per-anchor features (reference :129-150).

    q: B x N x 3, p: B x K x 3, fea: B x N x K(+1) x C  ->  B x N x C.
    ``-(|p-q| + 1e-5)^2 / var`` logits, optional constant background logit ``-0.2/var``,
    normalised by ``sum + 1e-6``."""
    return _composite.gaussian_blend(q, p, fea, var, background)


class FastEnsembleDeepSDFMirrored(nn.Module):
    """Identity SDF of NPHM: ``n_loc`` anchor-local MLPs + 1 global MLP, blended by distance
    to the (latent-dependent) anchors.  Reference :153-267."""

    def __init__(
            self,
            lat_dim_glob: int,
            lat_dim_loc: int,
            n_loc: int,
            n_symm_pairs: int,
            anchors: torch.Tensor,
            hidden_dim: int,
            n_layers: int,
            pos_mlp_dim: int = 256,
            out_dim: int = 1,
            input_dim: int = 3,
    ):
        super().__init__()
        self.lat_dim_glob = lat_dim_glob
        self.lat_dim_loc = lat_dim_loc
        self.lat_dim = lat_dim_glob + (n_loc + 1) * lat_dim_loc
        self.input_dim = input_dim
        self.out_dim = out_dim
        self.pos_mlp_dim = pos_mlp_dim
        self.num_kps = n_loc
        self.num_symm_pairs = n_symm_pairs

        self.ensembled_deep_sdf = EnsembledDeepSDF(ensemble_size=n_loc + 1,
                                                   n_symm=n_symm_pairs,
                                                   lat_dim=lat_dim_glob + lat_dim_loc,
                                                   hidden_dim=hidden_dim,
                                                   nlayers=n_layers,
                                                   out_dim=out_dim,
                                                   input_dim=input_dim).float()
        # plain attribute like the reference (:192): not a buffer, not in state_dict
        self.anchors = anchors
        self.mlp_pos = nn.Sequential(
            nn.Linear(lat_dim_glob, pos_mlp_dim),
            nn.ReLU(),
            nn.Linear(pos_mlp_dim, pos_mlp_dim),
            nn.ReLU(),
            nn.Linear(pos_mlp_dim, n_loc * 3),
        )
        self._engine = None          # lazily built native handle (see _native.EnsembleEngine)

    # ------------------------------------------------------------------ fused path plumbing
    def _fused_ok(self, xyz: torch.Tensor, lat_rep: torch.Tensor) -> bool:
        if not xyz.is_cuda:
            return False
        if torch.is_grad_enabled() and (xyz.requires_grad or lat_rep.requires_grad
                                        or any(p.requires_grad for p in self.parameters())):
            return False             # someone may call backward(): keep the autograd graph
        e = self.ensembled_deep_sdf
        n_lin = e.num_layers - 1
        if not _native.stack_supported(n_lin - 1, _native.hidden_width(e, n_lin), self.lat_dim_glob + self.lat_dim_loc):
            return False             # depth / width the native stack builder rejects: composite path
        return (xyz.dtype == torch.float32 and self.out_dim == 1 and self.input_dim == 3)

    def _sdfgrad_unsupported(self, xyz: torch.Tensor, lat_rep: torch.Tensor, call_sizes=None) -> Optional[str]:
        if not (xyz.is_cuda and lat_rep.is_cuda):
            return 'needs CUDA points and codes'
        if xyz.dtype != torch.float32 or any(p.dtype != torch.float32 for p in self.parameters()):
            return 'needs fp32 points and parameters'
        if not self.training and call_sizes is None:
            return ('needs training mode, or call_sizes in eval mode (the eval-mode forward overwrites the last point of '
                    'every decoder call, so its result depends on where the calls end)')
        if call_sizes is not None and (any(int(n) < 1 for n in call_sizes) or sum(int(n) for n in call_sizes) != xyz.shape[-2]):
            return 'needs call_sizes of at least one point each that add up to the points of a batch element'
        e = self.ensembled_deep_sdf
        n_lin = e.num_layers - 1
        if not (self.out_dim == 1 and self.input_dim == 3 and
                _native.stack_supported(n_lin - 1, _native.hidden_width(e, n_lin), self.lat_dim_glob + self.lat_dim_loc)):
            return 'needs a one-output member stack the native builder accepts'
        if xyz.dim() != 3 or xyz.shape[-1] != 3 or lat_rep.dim() != 3 or lat_rep.shape[-1] != self.lat_dim:
            return 'needs B x N x 3 points and B x 1 x lat_dim codes'
        if lat_rep.shape[1] != 1 and lat_rep.stride(1) != 0:
            return 'needs one code per batch element (B x 1 x lat_dim)'
        return None

    def sdfgrad_supported(self, xyz: torch.Tensor, lat_rep: torch.Tensor, call_sizes=None) -> bool:
        """Whether :meth:`forward_with_gradient_native` takes these inputs."""
        return self._sdfgrad_unsupported(xyz, lat_rep, call_sizes) is None

    def forward_with_gradient_native(self, xyz: torch.Tensor, lat_rep: torch.Tensor, call_sizes=None):
        """``(sdf B x N x 1, d sdf / d xyz B x N x 3, anchors B x n_loc x 3)``: the forward followed by
        ``gradient(sdf, xyz)``, with the members' values, gradients and second-order backward on the native kernels (one
        launch per pass for all members) and the anchors, frames and Gaussian blend in autograd
        (``_composite.ensemble_blend_with_gradient``).  Differentiable to first order in the parameters and ``lat_rep``; the
        points get no gradient.  Raises ``ValueError`` naming what it does not support.

        In eval mode ``call_sizes`` is required: the points of each batch element stand for consecutive decoder calls of
        ``call_sizes[i]`` points each (they add up to N), and the reference's eval-mode forward sets every member's output to 1
        at the last point of each call (EnsembledDeepSDF.py:260-261).  There s_k = 1 and grad s_k = 0 before the blend, so
        the members' native passes see a zero upstream gradient at those rows.  In training mode ``call_sizes`` only
        has to be consistent; it changes nothing."""
        reason = self._sdfgrad_unsupported(xyz, lat_rep, call_sizes)
        if reason is not None:
            raise ValueError('forward_with_gradient_native: ' + reason)
        lat = lat_rep[:, :1]
        anchors, local, cond = _composite.member_frames(self, xyz.detach(), lat)
        e = self.ensembled_deep_sdf
        params = []
        for i in range(e.num_layers - 1):
            lin = getattr(e, 'lin%d' % i)
            params += [lin.weight, lin.bias]
        s, g = _NativeEnsembleSdfGradFn.apply(self.engine(), local, cond[:, :, 0], *params)
        if not self.training:
            s, g = _composite.apply_eval_quirk(s, g, call_sizes)
        sdf, grad = _composite.ensemble_blend_with_gradient(self, xyz.detach(), anchors, s, g)
        return sdf, grad, anchors

    def engine(self) -> "_native.EnsembleEngine":
        """Native handle holding the packed weights; rebuilt when parameters change."""
        if self._engine is None:
            self._engine = _native.EnsembleEngine(self)
        self._engine.refresh(self)
        return self._engine

    def mean_anchors(self, device, dtype=torch.float32) -> torch.Tensor:
        a = self.anchors
        if a is None:
            raise ValueError('FastEnsembleDeepSDFMirrored needs mean anchors')
        return a.reshape(self.num_kps, 3).to(device=device, dtype=dtype)

    def predict_anchors(self, lat_rep: torch.Tensor) -> torch.Tensor:
        """Anchors ``B x n_loc x 3`` of the codes ``lat_rep`` (B x * x lat_dim): ``mlp_pos(z_glob) + mean anchors``.  The same
        values as the second return of :meth:`forward` (which the reference's fitters obtain by evaluating the whole ensemble
        on a dummy point), differentiable w.r.t. the code."""
        z_glob = lat_rep.reshape(lat_rep.shape[0], -1, self.lat_dim)[:, 0, :self.lat_dim_glob]
        out = self.mlp_pos(z_glob).view(-1, self.num_kps, 3)
        return out + self.mean_anchors(out.device, out.dtype)[None]

    # ------------------------------------------------------------------ forward
    def forward(self,
                xyz: torch.Tensor,
                lat_rep: torch.Tensor,
                anchors_gt: Optional[torch.Tensor]) -> (torch.Tensor, torch.Tensor):
        """xyz: B x N x 3 (or N x 3); lat_rep: B x N x lat_dim or B x 1 x lat_dim, laid out
        ``[z_glob, z_0 .. z_{n_loc-1}, z_global_member]``; ``anchors_gt`` is ignored (as in the
        reference).  Returns ``(sdf B x N x 1, anchors B x n_loc x 3)``."""
        if xyz.dim() < 3:
            xyz = xyz.unsqueeze(0)
        B, N, _ = xyz.shape
        assert self.lat_dim == lat_rep.shape[-1], \
            'lat dim {}, lat_rep {}'.format(self.lat_dim, lat_rep.shape)

        if self._fused_ok(xyz, lat_rep):
            lat = _native.constant_latent_rows(lat_rep)      # B x lat_dim, or None if per-point
            if lat is not None:
                return self.engine().query(xyz, lat, eval_quirk=not self.training)
        return self._forward_composite(xyz, lat_rep)

    def _forward_composite(self, xyz, lat_rep):
        return _composite.ensemble_sdf(self, xyz, lat_rep)
