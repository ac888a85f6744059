"""PyTorch-composite implementations shared by the mirrored modules (autograd / CPU path).

The fused kernels are the product path; these functions compute the same maps with stock torch ops so that training
(double backward for the eikonal / normal losses), CPU tests and odd configurations keep working.  They are written
against the maths in SURVEY.md section 8a', not against the reference's code, and are pinned to the reference's outputs by
the golden fixtures (tests/test_host.py)."""
from __future__ import annotations

import math
from typing import Sequence

import torch

SQRT2 = math.sqrt(2.0)


def ensembled_affine(x, weight, bias, set_of_member):
    """x: A x M x D_in; weight: S x D_out x D_in; member a uses weight set ``set_of_member[a]``  ->  A x M x D_out."""
    w = weight.index_select(0, set_of_member)
    y = torch.einsum('amk,ank->amn', x, w)
    if bias is not None:
        y = y + bias.index_select(0, set_of_member)[:, None, :]
    return y


def skip_mlp(inp, layers: Sequence, skip_in, activation):
    """DeepSDF-style stack: ``layers[i]`` are callables, the network input is re-injected (concatenated, the sum scaled by
    1/sqrt(2)) in front of every layer listed in ``skip_in``; ``activation`` after all layers but the last."""
    h = inp
    for i, layer in enumerate(layers):
        if i in skip_in:
            h = torch.cat([h, inp], dim=-1) / SQRT2
        h = layer(h)
        if i + 1 < len(layers):
            h = activation(h)
    return h


BLEND_VAR = 0.1 ** 2          # variance of the ensemble's Gaussian blend
BLEND_BACKGROUND = -0.2       # logit (before the division by the variance) of the global member


def gaussian_blend(queries, centres, features, var, background):
    """Blend per-centre features with weights exp(-(|c - q| + 1e-5)^2 / var) (plus a constant -0.2/var logit for an extra
    background feature), normalised by sum + 1e-6.  queries B x N x 3, centres B x K x 3, features B x N x K(+1) x C."""
    gap = (centres[:, None, :, :] - queries[:, :, None, :]).norm(dim=-1) + 10e-6
    logits = -(gap * gap)
    if background:
        logits = torch.cat([logits, logits.new_full(logits.shape[:2] + (1,), BLEND_BACKGROUND)], dim=-1)
    w = torch.exp(logits / var)
    w = w / (w.sum(dim=-1, keepdim=True) + 1e-6)
    return (features * w[..., None]).sum(dim=2)


def member_signs(module, like):
    """(K + 1) x 3: the x-mirror of the odd members of the symmetric pairs (-1 in their x column), 1 elsewhere."""
    sign = like.new_ones(module.num_kps + 1, 3)
    sign[1:2 * module.num_symm_pairs:2, 0] = -1.0
    return sign


def member_frames(module, xyz, lat_rep):
    """The inputs of the members of ``FastEnsembleDeepSDFMirrored``: anchors from the global code (B x K x 3), member-local
    coordinates (members x B x N x 3: anchor-centred for the K local members, the world frame for the last one, x-mirrored
    for the odd members of the symmetric pairs) and per-member conditions [z_glob | z_k] (members x B x N x (G + L))."""
    B, N, _ = xyz.shape
    K, G, L = module.num_kps, module.lat_dim_glob, module.lat_dim_loc
    if lat_rep.shape[1] == 1:
        lat_rep = lat_rep.expand(B, N, module.lat_dim)
    anchors = module.mlp_pos(lat_rep[:, 0, :G]).view(B, K, 3) + module.mean_anchors(xyz.device, xyz.dtype)[None]
    origin = torch.cat([anchors, anchors.new_zeros(B, 1, 3)], dim=1)
    local = (xyz[:, :, None, :] - origin[:, None, :, :]) * member_signs(module, xyz)
    cond = torch.cat([lat_rep[:, :, None, :G].expand(B, N, K + 1, G), lat_rep[:, :, G:].reshape(B, N, K + 1, L)], dim=-1)
    return anchors, local.permute(2, 0, 1, 3), cond.permute(2, 0, 1, 3)


def ensemble_sdf(module, xyz, lat_rep):
    """Composite forward of ``FastEnsembleDeepSDFMirrored``: anchors from the global code, member-local (mirrored)
    coordinates, per-member condition [z_glob | z_k], member MLPs, Gaussian blend.  Returns (sdf B x N x 1, anchors)."""
    anchors, local, cond = member_frames(module, xyz, lat_rep)
    s = module.ensembled_deep_sdf(local, cond)                                               # members x B x N x 1
    if not module.training:
        # the reference's eval-mode hack (EnsembledDeepSDF.py:260-261) hits the POINT axis: last point of the call -> 1
        s = s.clone()
        s[:, :, -1, 0] = 1
    return gaussian_blend(xyz[..., :3], anchors, s.permute(1, 2, 0, 3), var=BLEND_VAR, background=True), anchors


def call_ends(call_sizes):
    """Indices along the point axis of the last point of each of consecutive decoder calls of ``call_sizes`` points: the rows
    the eval-mode forward overwrites (EnsembledDeepSDF.py:260-261)."""
    ends, end = [], 0
    for n in call_sizes:
        end += int(n)
        ends.append(end - 1)
    return ends


def apply_eval_quirk(s, g, call_sizes):
    """The eval-mode quirk on the members' values s (members x B x N (x 1)) and local gradients g (members x B x N x 3):
    s_k = 1 and grad s_k = 0 at the last point of every call, as a differentiable select (those rows get no upstream)."""
    s, g = s.clone(), g.clone()
    for e in call_ends(call_sizes):
        s[:, :, e] = 1
        g[:, :, e] = 0
    return s, g


def ensemble_blend_with_gradient(module, xyz, anchors, s, g):
    """The blend of ``ensemble_sdf`` and its spatial gradient from the members' values and local-frame gradients.

    xyz B x N x 3 (data points), anchors B x K x 3, s members x B x N (x 1) = s_k, g members x B x N x 3 = grad_local s_k,
    both at the coordinates of ``member_frames``.  With w_k = exp(-(|x - A_k| + 1e-5)^2 / var) (the global member: the
    constant background weight), W = sum_j w_j + 1e-6 and wt_k = w_k / W:
        sdf      = sum_k wt_k s_k
        grad sdf = sum_k wt_k (sign_k * g_k) + sum_k s_k grad wt_k,   grad wt_k = (grad w_k - wt_k sum_j grad w_j) / W,
        grad w_k = -(2 (|x - A_k| + 1e-5) / var) w_k (x - A_k) / |x - A_k|   (0 at x = A_k, as torch's norm backward).
    Plain torch ops: autograd through it gives the upstream gradients of s_k and g_k and carries the point gradients of the
    members (through the frames of ``member_frames``) to the anchors.  Returns (sdf B x N x 1, grad sdf B x N x 3)."""
    n_members = s.shape[0]
    sign = member_signs(module, xyz)
    d = xyz[:, :, None, :] - anchors[:, None, :, :]                                          # B x N x K x 3: x - A_k
    r = d.norm(dim=-1)
    gap = r + 10e-6
    logits = -(gap * gap)
    logits = torch.cat([logits, logits.new_full(logits.shape[:2] + (1,), BLEND_BACKGROUND)], dim=-1)
    w = torch.exp(logits / BLEND_VAR)                                                       # B x N x (K + 1)
    total = w.sum(dim=-1, keepdim=True) + 1e-6
    wt = w / total
    s_b = s.reshape(n_members, *s.shape[1:3]).permute(1, 2, 0)                               # B x N x (K + 1)
    g_b = (g * sign[:, None, None, :]).permute(1, 2, 0, 3)                                   # B x N x (K + 1) x 3, world frame
    unit = d / torch.where(r > 0, r, torch.ones_like(r))[..., None]
    dw = (-2.0 / BLEND_VAR) * (gap * w[..., :-1])[..., None] * unit
    dw = torch.cat([dw, dw.new_zeros(dw.shape[:2] + (1, 3))], dim=2)                         # background: constant weight
    dwt = (dw - wt[..., None] * dw.sum(dim=2, keepdim=True)) / total[..., None]
    sdf = (wt * s_b).sum(dim=-1, keepdim=True)
    grad = (wt[..., None] * g_b).sum(dim=2) + (s_b[..., None] * dwt).sum(dim=2)
    return sdf, grad
