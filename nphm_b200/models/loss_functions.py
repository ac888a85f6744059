"""Training / validation losses of the reference, ``NPHM.models.loss_functions``:

  * ``compute_loss``                  src/NPHM/models/loss_functions.py:7-17
  * ``actual_compute_loss``           src/NPHM/models/loss_functions.py:20-110   (SURVEY.md 8f-3)
  * ``compute_loss_corresp_forward``  src/NPHM/models/loss_functions.py:282-322  (stage 2: the expression space)

Same inputs (a batch dict with ``points_face``, ``points_non_face``, ``sup_grad_far``, ``sup_grad_near``, the normals and
``gt_anchors``), same returned dict (``surf_sdf``, ``normals``, ``space_sdf``, ``grad``, ``lat_reg`` and - for the
ensemble - ``anchors``, ``symm_dist``, ``middle_dist``).  Two ways to get the SDF values and their spatial gradient:

  * **native** (no autograd graph: validation, monitoring, loss curves of a frozen model): one call per batch element and
    point set into ``nphm_ensemble_backward_inputs`` with an upstream gradient of ones - a point's SDF depends on its own
    coordinates only, so that vector-Jacobian product IS the per-point spatial gradient (tensor-core forward and backward,
    ``csrc/fit.cu``).  Used when autograd is not recording (the reference cannot evaluate these losses at all under
    ``torch.no_grad()``: its ``gradient`` needs a graph) or with ``native=True``.  In eval mode the call is
    ``nphm_ensemble_backward_inputs_quirk`` with the period of one reference call (its last point gets the eval-mode quirk,
    EnsembledDeepSDF.py:260-261); that form needs the tensor-core configuration, other eval-mode ensembles stay composite.
  * **composite** (training): the decoder's autograd path and ``diff_operators.gradient`` with ``create_graph=True`` -
    weight gradients of the normal / eikonal terms need the double backward, which stays in PyTorch.

With ``native=True`` and a ``DeepSDF`` decoder (the NPM baseline) the loss takes a third way, with or without autograd:
``DeepSDF.forward_with_gradient_native`` evaluates the four point sets in one call (concatenated along the points of each
query) and differentiates the SDF and its spatial gradient natively, second-order terms included.  ``native=None`` keeps the
composite path for it.  With ``native=True``, the ensemble in training mode on CUDA and autograd recording, the ensemble takes
the same way: ``FastEnsembleDeepSDFMirrored.forward_with_gradient_native`` runs the members' passes natively (one launch per
pass for all members) and the anchors and blend in autograd.  Under ``torch.no_grad()`` ``native=True`` keeps the evaluation
path above.  Both take the ensemble in eval mode too - the validation step of the reference's stage 1
(``TrainerAutoDecoder.compute_val_loss``, training.py:250-268, calls ``decoder.eval()`` and then differentiates this loss): the
four point sets are the reference's four decoder calls, so the last point of each set, per batch element, gets the quirk.

``compute_loss_corresp_forward`` is first order (no gradient with respect to the points is used), so its decoder calls run
natively to the weights: ``DeformationNetwork.forward_native_grad`` (forward and backward on the tensor cores, the compressor
and the embeddings in autograd).  ``native=None`` picks that path for a CUDA fp32 decoder the native chain supports,
``native=False`` keeps the composite one.

This module is NOT installed over ``NPHM.models.loss_functions`` by ``install_as_nphm`` (the reference's own file keeps
working on top of the drop-in decoder); import it explicitly.
"""
from __future__ import annotations

import torch

from .EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
from .deepSDF import DeepSDF, DeformationNetwork
from .diff_operators import gradient

_POINT_SETS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far')


def compute_loss(batch, decoder, latent_codes, device, native=None):
    """Moves the batch to ``device``, looks the latent codes up by ``batch['idx']`` and evaluates the losses."""
    batch = {k: v for k, v in batch.items() if k != 'path'}
    on_device = {k: v.to(device).float() for k, v in batch.items()}
    glob_cond = latent_codes(batch['idx'].to(device))
    return actual_compute_loss(on_device, decoder, glob_cond, native=native)


def _native_values_and_gradients(decoder, points, glob_cond):
    """points B x N x 3, glob_cond B x 1 x lat_dim -> (sdf B x N x 1, d sdf / d x  B x N x 3), no graph.  Each batch element
    is one decoder call, as in the reference (its last point carries the eval-mode quirk)."""
    engine = decoder.engine()
    period = 0 if decoder.training else points.shape[1]
    sdf, grad = [], []
    for b in range(points.shape[0]):
        pts = points[b].contiguous()
        ones = torch.ones(pts.shape[0], device=pts.device, dtype=torch.float32)
        s, _, g = engine.backward_inputs(pts, glob_cond[b].reshape(-1), ones, quirk_period=period)
        sdf.append(s)
        grad.append(g)
    return torch.stack(sdf)[..., None], torch.stack(grad)


def _composite_values_and_gradients(decoder, points, glob_cond, anchor_preds):
    pts = points.clone().detach().requires_grad_()
    pred, anchors = decoder(pts, glob_cond.repeat(1, pts.shape[1], 1), anchor_preds)
    return pred, gradient(pred, pts), anchors


def _pair_distance(latents):
    """mean over (batch, pairs) of || z_{2i} - z_{2i+1} ||; an odd trailing block is ignored (reference :84-87)."""
    n = latents.shape[1] - latents.shape[1] % 2
    return torch.norm(latents[:, 0:n:2, :] - latents[:, 1:n:2, :], dim=-1).mean()


def _sdfgrad_native(decoder, batch_cuda, glob_cond):
    """All four point sets in one ``forward_with_gradient_native`` call -> ({name: sdf}, {name: d sdf / d x})."""
    sets = [batch_cuda[name] for name in _POINT_SETS]
    pts = torch.cat(sets, dim=1)
    if not (glob_cond.dim() == 3 and glob_cond.shape[1] == 1 and decoder.sdfgrad_supported(pts, glob_cond)):
        raise ValueError('actual_compute_loss(native=True): this DeepSDF decoder / batch is not supported natively (needs '
                         'CUDA fp32 points, one output, Softplus(beta=100), no positional encoding, B x 1 x D codes)')
    sdf, g = decoder.forward_with_gradient_native(pts, glob_cond)
    sizes = [p.shape[1] for p in sets]
    return dict(zip(_POINT_SETS, sdf.split(sizes, dim=1))), dict(zip(_POINT_SETS, g.split(sizes, dim=1)))


def _ensemble_sdfgrad_native(decoder, batch_cuda, glob_cond):
    """The ensemble's ``forward_with_gradient_native`` on all four point sets in one call -> ({name: sdf},
    {name: d sdf / d x}, anchors)."""
    sets = [batch_cuda[name] for name in _POINT_SETS]
    pts = torch.cat(sets, dim=1)
    sizes = [p.shape[1] for p in sets]
    sdf, g, anchors = decoder.forward_with_gradient_native(pts, glob_cond, call_sizes=sizes)
    return dict(zip(_POINT_SETS, sdf.split(sizes, dim=1))), dict(zip(_POINT_SETS, g.split(sizes, dim=1))), anchors


def actual_compute_loss(batch_cuda, decoder, glob_cond, native=None):
    is_ensemble = isinstance(decoder, FastEnsembleDeepSDFMirrored)
    anchor_preds = batch_cuda['gt_anchors'] if hasattr(decoder, 'anchors') else None
    sdfgrad = native is not None and bool(native) and isinstance(decoder, DeepSDF)
    explicit = native is not None and bool(native)
    if native is None:
        native = not torch.is_grad_enabled()
    native = bool(native) and is_ensemble and batch_cuda['points_face'].is_cuda
    ensemble_sdfgrad = native and explicit and torch.is_grad_enabled()
    if native and not ensemble_sdfgrad:
        from .fitting import _fused_identity
        native = _fused_identity(decoder, grad_points=True)      # the vector-Jacobian product needs the tensor-core configuration

    pred, grad, anchors = {}, {}, None
    if sdfgrad:
        pred, grad = _sdfgrad_native(decoder, batch_cuda, glob_cond)
    elif ensemble_sdfgrad:
        pred, grad, anchors = _ensemble_sdfgrad_native(decoder, batch_cuda, glob_cond)
    elif native:
        with torch.no_grad():
            for name in _POINT_SETS:
                pred[name], grad[name] = _native_values_and_gradients(decoder, batch_cuda[name], glob_cond)
            anchors = decoder.engine().anchors(glob_cond[:, 0, :])
    else:
        with torch.enable_grad():
            for name in _POINT_SETS:
                pred[name], grad[name], a = _composite_values_and_gradients(decoder, batch_cuda[name], glob_cond, anchor_preds)
                if name != 'sup_grad_far':
                    anchors = a                      # the reference keeps the anchors of its third call (sup_grad_near)

    # geometry terms
    sdf_face = pred['points_face'].abs().squeeze()
    sdf_outer = pred['points_non_face'].abs().squeeze()
    normal_face = (grad['points_face'] - batch_cuda['normals_face']).norm(2, dim=-1)
    normal_outer = torch.clamp((grad['points_non_face'] - batch_cuda['normals_non_face']).norm(2, dim=-1), None, 0.75) / 2
    eikonal = torch.cat([(grad[name].norm(dim=-1) - 1).abs()
                         for name in ('points_face', 'points_non_face', 'sup_grad_far', 'sup_grad_near')], dim=-1)
    space_sdf = torch.exp(-1e1 * pred['sup_grad_far'].abs())

    losses = {'surf_sdf': torch.cat([sdf_face, sdf_outer], dim=-1).mean(),
              'normals': torch.cat([normal_face.squeeze(), normal_outer.squeeze()], dim=-1).mean(),
              'space_sdf': space_sdf.mean(),
              'grad': eikonal.mean(),
              'lat_reg': (torch.norm(glob_cond, dim=-1) ** 2).mean()}
    if anchors is None:
        return losses

    symm_dist = middle_dist = None
    if hasattr(decoder, 'lat_dim_glob'):
        z = glob_cond.squeeze(1)
        G, L, n_symm = decoder.lat_dim_glob, decoder.lat_dim_loc, decoder.num_symm_pairs
        symm = z[:, G:G + 2 * n_symm * L].view(z.shape[0], 2 * n_symm, L)
        middle = z[:, G + 2 * n_symm * L:-L].view(z.shape[0], decoder.num_kps - 2 * n_symm, L)
        symm_dist = _pair_distance(symm)
        middle_dist = _pair_distance(middle)
    losses['anchors'] = (anchors - batch_cuda['gt_anchors']).square().mean()
    losses['symm_dist'] = symm_dist
    losses['middle_dist'] = middle_dist
    return losses


def _corresp_native_ok(decoder, points, glob_cond) -> bool:
    return (hasattr(decoder, 'native_grad_supported') and points.is_cuda and points.dtype == torch.float32
            and glob_cond.dim() == 3 and glob_cond.shape[1] == 1 and decoder.native_grad_supported(points, glob_cond))


def corresp_forward_draws(decoder, n_rows, n_points, device, dtype):
    """The random draws of :func:`compute_loss_corresp_forward` on a batch of ``n_rows`` x ``n_points`` points, in its order,
    without evaluating anything: a rank of a data-parallel step that holds no rows keeps its generators in step this way."""
    noisy = isinstance(decoder, DeformationNetwork) and decoder.mode == 'compress' and decoder.training
    width = decoder.compressor[0].out_features if noisy else 0
    if noisy:
        torch.randn((n_rows, n_points, width), device=device)
    torch.rand(n_rows, 100, 3, device=device, dtype=dtype)
    if noisy:
        torch.randn((n_rows, 100, width), device=device)


def compute_loss_corresp_forward(batch, decoder, decoder_shape, latent_codes, latent_codes_shape, device, epoch=-1,
                                 exp_path=None, native=None, rows=None):
    """Stage-2 loss of the reference (same arguments, same random draws in the same order, same returned dict:
    ``corresp``, ``lat_reg``, ``loss_reg_zero``).  ``native``: None = the native first-order decoder path when it supports
    the call, False = the composite path, True = the native path (raises if unsupported).

    ``rows=(r0, r1)``: the losses of batch rows [r0, r1) only, each a mean over those rows.  Every random draw is made for the
    whole batch and these rows are kept, so the rows see the draws of a whole-batch call and the generators end in its state
    (the data-parallel step, :mod:`nphm_b200.training_sharded`)."""
    if 'path' in batch:
        del batch['path']
    batch_rows = None
    if rows is not None:
        r0, r1 = rows
        batch_rows = (r0, batch['idx'].shape[0])
        batch = {k: v[r0:r1] for k, v in batch.items()}
    noise_rows = {} if batch_rows is None or not isinstance(decoder, DeformationNetwork) else {'batch_rows': batch_rows}
    batch_cuda = {k: v.to(device).float() for (k, v) in zip(batch.keys(), batch.values())}
    glob_cond_shape = latent_codes_shape(batch['subj_ind'].to(device))
    glob_cond_pose = latent_codes(batch['idx'].to(device))

    if 'gt_anchors' in batch_cuda and decoder_shape is not None and decoder_shape.mlp_pos is None:
        gt_anchors = batch_cuda['gt_anchors']
    elif decoder_shape is not None and decoder_shape.mlp_pos is not None:
        gt_anchors = decoder_shape.mlp_pos(glob_cond_shape[..., :decoder_shape.lat_dim_glob]).view(glob_cond_pose.shape[0], -1, 3)
        gt_anchors += decoder.anchors.squeeze(0)
    else:
        gt_anchors = batch_cuda['gt_anchors']

    glob_cond = torch.cat([glob_cond_shape, glob_cond_pose], dim=-1)
    points_neutral = batch_cuda['points_neutral'].clone().detach().requires_grad_()
    if native is None:
        native = _corresp_native_ok(decoder, points_neutral, glob_cond)
    elif native and not _corresp_native_ok(decoder, points_neutral, glob_cond):
        raise ValueError('compute_loss_corresp_forward(native=True): the decoder / batch is not supported natively')

    if native:
        # B x 1 x D condition: its gradient is the sum over the points, which is what the reference's repeat() passes on
        decoder_call = lambda x, n: decoder.forward_native_grad(x, glob_cond, gt_anchors, **noise_rows)     # noqa: E731
    else:
        cond = glob_cond.repeat(1, points_neutral.shape[1], 1)
        decoder_call = lambda x, n: decoder(x, cond[:, :n, :], gt_anchors, **noise_rows)                    # noqa: E731

    delta, _ = decoder_call(points_neutral, points_neutral.shape[1])
    pred_posed = points_neutral + delta.squeeze()
    points_posed = batch_cuda['points_posed']
    loss_corresp = (pred_posed - points_posed[:, :, :3]) ** 2

    lat_mag = torch.norm(glob_cond_pose, dim=-1) ** 2

    # enforce deformation field to be zero elsewhere
    if batch_rows is None:
        samps = (torch.rand(glob_cond.shape[0], 100, 3, device=glob_cond.device, dtype=glob_cond.dtype) - 0.5) * 2.5
    else:
        whole = torch.rand(batch_rows[1], 100, 3, device=glob_cond.device, dtype=glob_cond.dtype)
        samps = (whole[batch_rows[0]:batch_rows[0] + glob_cond.shape[0]] - 0.5) * 2.5
    delta, _ = decoder_call(samps, 100)
    loss_reg_zero = (delta ** 2).mean()

    return {'corresp': loss_corresp.mean(),
            'lat_reg': lat_mag.mean(),
            'loss_reg_zero': loss_reg_zero}
