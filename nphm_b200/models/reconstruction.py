"""Drop-in mirror of the reference module ``NPHM.models.reconstruction``.

  * ``get_logits``           src/NPHM/models/reconstruction.py:6-25
  * ``get_logits_backward``  src/NPHM/models/reconstruction.py:28-56
  * ``deform_mesh``          src/NPHM/models/reconstruction.py:59-88

The reference evaluates the decoder chunk by chunk (``nbatch_points``) to bound its activation memory and
copies every chunk to the host.  The fused kernels keep activations on chip, so one launch covers all
points; the only chunk-size dependence of the reference's RESULT - in eval mode the last point of every
chunk gets s_k = 1 (EnsembledDeepSDF.py:260-261) - is reproduced through ``quirk_period``.
"""
from __future__ import annotations

import numpy as np
import torch

from .EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
from ..utils.mesh import make_mesh
from ..utils.reconstruction import _to_host


def _as_row(encoding: torch.Tensor) -> torch.Tensor:
    """1-D ``(D,)`` or ``(1,1,D)`` latent -> ``(1, D)``."""
    return encoding.reshape(1, -1)


def _per_point(code: torch.Tensor, n: int) -> torch.Tensor:
    """latent of any shape -> ``(1, n, D)`` view (the layout the reference's modules are called with)."""
    code = code.reshape(1, 1, -1)
    return code.expand(1, n, code.shape[-1])


def _sweep(grid_points, chunk, evaluate):
    """Run ``evaluate(points) -> (values, anchors)`` over ``chunk``-sized pieces of the point axis; the values of every
    piece go to the host.  Returns (numpy (N,), anchors of the last piece)."""
    pieces, anchors = [], None
    with torch.no_grad():
        for start in range(0, grid_points.shape[1], chunk):
            values, anchors = evaluate(grid_points[:, start:start + chunk])
            pieces.append(values.reshape(-1).detach().cpu())
    return torch.cat(pieces).numpy(), anchors


def get_logits(decoder, encoding, grid_points, nbatch_points=100000, return_anchors=False):
    """SDF of ``grid_points`` (1 x N x 3) under latent ``encoding`` -> numpy (N,) float32 [, anchors]."""
    fused = (isinstance(decoder, FastEnsembleDeepSDFMirrored) and grid_points.is_cuda
             and grid_points.dtype == torch.float32)
    if fused:
        # one launch over all points; the chunk size only matters through the eval-mode last-point-of-chunk quirk
        with torch.no_grad():
            pts = grid_points.reshape(1, -1, 3)
            sdf, anchors = decoder.engine().query(pts, _as_row(encoding).to(pts.device), eval_quirk=not decoder.training,
                                                  quirk_period=None if decoder.training else int(nbatch_points))
            logits = _to_host(sdf.reshape(-1))
    else:
        logits, anchors = _sweep(grid_points, nbatch_points,
                                 lambda pts: decoder(pts, _per_point(encoding, pts.shape[1]), None))
    return (logits, anchors) if return_anchors else logits


def get_logits_backward(decoder_shape, decoder_expr, encoding_shape, encoding_expr, grid_points,
                        nbatch_points=100000, return_anchors=False):
    """Backward-warp query: points are first offset by ``decoder_expr`` (called with ``anchors=None`` as in the
    reference, so a 'compress' DeformationNetwork fails here exactly like upstream), then ``decoder_shape``."""
    def evaluate(pts):
        if encoding_expr is not None:
            pts = pts + decoder_expr(pts, _per_point(encoding_expr, pts.shape[1]), None)[0]
        return decoder_shape(pts, _per_point(encoding_shape, pts.shape[1]), None)

    logits, anchors = _sweep(grid_points, nbatch_points, evaluate)
    return (logits, anchors) if return_anchors else logits


def deform_mesh(mesh, deformer, lat_rep, anchors, lat_rep_shape=None):
    """Forward-deform the vertices of a canonical mesh with ``deformer`` (one fused launch instead of the
    reference's 5000-vertex chunks + ``empty_cache``)."""
    cached = getattr(mesh, '_nphm_device_vertices', None)
    if (cached is not None and cached.device == lat_rep.device and cached.shape[0] == len(mesh.vertices)):
        rest = cached[None]                      # vertices never left the device since marching cubes (mesh_from_logits)
    else:
        rest = torch.as_tensor(np.asarray(mesh.vertices), dtype=torch.float32, device=lat_rep.device)[None]
    code = lat_rep if lat_rep_shape is None else torch.cat([lat_rep_shape, lat_rep], dim=-1)
    with torch.no_grad():
        if anchors is None:
            shift = deformer(rest, _per_point(code, rest.shape[1]), None)[0]
        else:
            shift = deformer(rest, code.reshape(1, 1, -1), anchors.reshape(1, -1, 3))[0]
    posed = (rest[..., :3] + shift.reshape(1, -1, 3))[0]
    return make_mesh(posed.cpu().numpy(), mesh.faces, process=False)


# ------------------------------------------------------------------------------------------ posed queries
# rows (points x expressions) the native posed query handles at once: bounds the Broyden workspace (~150 bytes per row) and
# the decoder's scratch; the result does not depend on it, because every row is computed independently of the others
POSED_PIECE_ROWS = 1 << 20


def _expression_codes(lat_reps_expr):
    """``(S, E)``, ``(S, 1, E)`` or ``(E,)`` -> (``S x E`` tensor, whether the input was one code)."""
    single = lat_reps_expr.dim() == 1
    codes = lat_reps_expr.reshape(1 if single else lat_reps_expr.shape[0], -1)
    if codes.shape[0] == 0:
        raise ValueError('get_logits_posed: no expression codes')
    return codes, single


def posed_parts(decoder_shape, decoder_expr, lat_rep_shape, codes):
    """The native pieces of the posed query of expressions ``codes`` (S x E), or None when the decoders have none:
    ``(device, cond S x C, search_engine, identity)`` with ``identity(xc S x n x 3, quirk) -> sdf S x n`` the identity decoder at
    canonical points.  ``shape_engine`` and ``z_id`` (1 x D) are attributes of ``identity``."""
    from .deepSDF import DeepSDF, DeformationNetwork
    from .fitting import NPM_EXPR_DIM, _native_npm_decoder
    from .iterative_root_finding import _fused_search_condition
    device = next(decoder_shape.parameters()).device
    if device.type != 'cuda' or decoder_expr.training or next(decoder_expr.parameters()).device != device:
        return None
    S = codes.shape[0]
    z_id = lat_rep_shape.reshape(1, -1).to(device=device, dtype=torch.float32)
    codes = codes.to(device=device, dtype=torch.float32)
    with torch.no_grad():
        if isinstance(decoder_shape, FastEnsembleDeepSDFMirrored) and isinstance(decoder_expr, DeformationNetwork):
            shape_engine = decoder_shape.engine()
            anchors = shape_engine.anchors(z_id)                                            # fitting.py:59
            # one row per call: the compressor's GEMM rounds differently for different batch sizes, and a row must not depend
            # on the other expressions of the call
            rows = [_fused_search_condition(decoder_expr, torch.zeros(1, 1, 3, device=device),
                                            torch.cat([z_id, codes[s:s + 1]], dim=-1)[:, None], anchors[:, None])  # fitting.py:72
                    for s in range(S)]
            if any(r is None for r in rows):
                return None
            cond = torch.cat(rows).contiguous()
            search_engine = decoder_expr.defDeepSDF.engine()
            lat = z_id.expand(S, -1).contiguous()

            def identity(xc, quirk):
                sdf, _ = shape_engine.query(xc, lat, eval_quirk=quirk, quirk_period=1 if quirk else None)
                return sdf.reshape(S, -1)
        elif (isinstance(decoder_shape, DeepSDF) and isinstance(decoder_expr, DeepSDF) and _native_npm_decoder(decoder_shape, 1)
              and _native_npm_decoder(decoder_expr, 3) and not hasattr(decoder_expr, 'lat_dim_expr')
              and decoder_expr.lat_dim == z_id.shape[1] + codes.shape[1] and codes.shape[1] == NPM_EXPR_DIM):
            cond = torch.cat([z_id.expand(S, -1), codes], dim=-1).contiguous()
            search_engine, shape_engine = decoder_expr.engine(), decoder_shape.engine()
            lat = z_id.expand(S, -1).contiguous()

            def identity(xc, quirk):
                return shape_engine.query(xc, lat).reshape(S, -1)
        else:
            return None
    identity.shape_engine, identity.z_id = shape_engine, z_id
    return device, cond, search_engine, identity


def posed_evaluator(decoder_shape, decoder_expr, lat_rep_shape, codes):
    """The native posed query of expressions ``codes`` (S x E), or None when the decoders have none (see
    :func:`get_logits_posed`): a function ``(points S x n x 3 float32 CUDA, quirk) -> (sdf S x n, valid S x n bool)``, row
    (s, i) the posed SDF of ``points[s, i]`` under expression s.  ``quirk``: every row takes the ensemble's eval-mode
    last-point-of-call value.  Each row depends on its own point and code only: J0^-1 at the point
    (``nphm_mlp_inverse_jacobian``), the compacting Broyden search (``nphm_mlp_broyden_search_compact``) and the identity query at
    the root, in pieces of :data:`POSED_PIECE_ROWS` rows."""
    parts = posed_parts(decoder_shape, decoder_expr, lat_rep_shape, codes)
    if parts is None:
        return None
    device, cond, search_engine, identity = parts
    S = codes.shape[0]

    def evaluate(points, quirk=False):
        n = points.shape[1]
        sdf = torch.empty(S, n, device=device, dtype=torch.float32)
        valid = torch.empty(S, n, device=device, dtype=torch.bool)
        piece = max(1, int(POSED_PIECE_ROWS) // S)
        with torch.no_grad(), torch.cuda.device(device):
            for a in range(0, n, piece):
                pts = points[:, a:a + piece].to(torch.float32).contiguous()
                _, j0_inv = search_engine.inverse_jacobian(pts, cond)
                xc, _, ok, _ = search_engine.broyden_search(pts, cond, pts, j0_inv, max_steps=15, cvg_thresh=1e-6,
                                                            dvg_thresh=0.2, compact=True)
                sdf[:, a:a + piece] = identity(xc, quirk)
                valid[:, a:a + piece] = ok
        return sdf, valid
    return evaluate


def _quirk_rows(n: int, nbatch_points: int) -> np.ndarray:
    """Rows that are the last of a chunk of ``nbatch_points`` (and the last row): the eval-mode quirk rows of get_logits."""
    return np.unique(np.append(np.arange(nbatch_points - 1, n, nbatch_points), n - 1))


def get_logits_posed(decoder_shape, decoder_expr, lat_rep_shape, lat_reps_expr, grid_points, nbatch_points=100000,
                     return_valid=False):
    """Posed SDF: the identity decoder at the canonical correspondence of every point of ``grid_points`` (1 x N x 3) under each
    expression code of ``lat_reps_expr`` ((S, E), (S, 1, E) or (E,)).  Row i of expression s is the reference joint fitter's
    composition (fitting.py:59-114) on the chunk of ``nbatch_points`` rows holding it:
        anchors = decoder_shape(0, lat_rep_shape)[1]  (ensemble only),  cond = [lat_rep_shape | lat_reps_expr[s]]
        xc, res = search(chunk, cond, decoder_expr, anchors, multi_corresp=False)  (Broyden on x + F_ex(x) = point)
        sdf     = decoder_shape(xc, lat_rep_shape)
    at every row, converged or not; ``valid`` is ``res['valid_ids']``.  ``decoder_shape.training`` is honoured: in eval mode the
    ensemble's last-point-of-call quirk falls on the last row of every chunk, as in :func:`get_logits`.  Deterministic (no random
    starts).

    The ensemble with an eval-mode ``DeformationNetwork`` (modes compress / expr_only / glob_only) and the NPM pair of DeepSDF
    decoders run natively on CUDA (:func:`posed_evaluator`); anything else takes the composite path (the mirror's ``search`` and
    the modules, chunk by chunk), which computes the same function.  Returns numpy float32 ``(S, N)`` (``(N,)`` for an ``(E,)``
    code) and, with ``return_valid``, bool of the same shape."""
    codes, single = _expression_codes(lat_reps_expr)
    S, N = codes.shape[0], grid_points.shape[1]
    fn = posed_evaluator(decoder_shape, decoder_expr, lat_rep_shape, codes) if grid_points.is_cuda else None
    if fn is not None:
        pts = grid_points.reshape(1, -1, 3).to(torch.float32)
        sdf, valid = fn(pts.expand(S, N, 3))
        if not decoder_shape.training and isinstance(decoder_shape, FastEnsembleDeepSDFMirrored) and N > 0:
            rows = torch.from_numpy(_quirk_rows(N, int(nbatch_points))).to(pts.device)
            sdf[:, rows] = fn(pts[:, rows].expand(S, -1, 3), quirk=True)[0]
        logits, ok = _to_host(sdf), _to_host(valid)
    else:
        logits, ok = _posed_composite(decoder_shape, decoder_expr, lat_rep_shape, codes, grid_points, int(nbatch_points))
    if single:
        logits, ok = logits[0], ok[0]
    return (logits, ok) if return_valid else logits


def _posed_composite(decoder_shape, decoder_expr, lat_rep_shape, codes, grid_points, nbatch_points):
    """:func:`get_logits_posed` through the mirror's modules, chunk by chunk as the reference calls them."""
    from .iterative_root_finding import search
    dev = grid_points.device
    z_id = lat_rep_shape.reshape(1, 1, -1).to(dev)
    ensemble = isinstance(decoder_shape, FastEnsembleDeepSDFMirrored)
    anchors = None
    if ensemble:
        with torch.no_grad():
            _, anchors = decoder_shape(torch.zeros(1, 1, 3, device=dev), z_id, None)
    N = grid_points.shape[1]
    logits = np.empty((codes.shape[0], N), dtype=np.float32)
    valid = np.empty((codes.shape[0], N), dtype=bool)
    for s in range(codes.shape[0]):
        glob_cond = torch.cat([z_id, codes[s].reshape(1, 1, -1).to(dev)], dim=-1)
        for a in range(0, N, nbatch_points):
            chunk = grid_points[:, a:a + nbatch_points]
            n = chunk.shape[1]
            xc, res = search(chunk, glob_cond.repeat(1, n, 1), decoder_expr,
                             None if anchors is None else anchors.unsqueeze(1).repeat(1, n, 1, 1), multi_corresp=False)
            with torch.no_grad():
                sdf, _ = decoder_shape(xc.detach(), z_id if ensemble else z_id.repeat(1, n, 1), None)
            logits[s, a:a + n] = sdf.reshape(-1).detach().cpu().numpy()
            valid[s, a:a + n] = res['valid_ids'].reshape(-1).cpu().numpy()
    return logits, valid
