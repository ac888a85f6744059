"""Depth and normal images of SDF heads by sphere tracing on the GPU, in the format of ``render_views`` (DESIGN.md §4.23).

``render_sdf_views`` renders the zero level set of a decoder directly, without a mesh: S canonical heads (one latent code each),
or one subject posed in S expressions.  Cameras and images follow ``render_views``: camera-to-world poses, the eye ray
``((c + 0.5 - cx)/fx, (cy - r - 0.5)/fy, -1)`` of pixel (r, c), eye depth in [znear, zfar] (0 = background) and render.cu's
uint8 normal encoding ((0, 0, 0) = background), so the images go unchanged into ``glcam_images`` and ``samples_from_images``.

March contract (tests/sdf_trace_common.py restates it in float64):
  * a ray is clipped to the box ``[mini, maxi]`` (decoder coordinates; a world point x is queried at ``scale x``) and to eye depth
    [znear, zfar]; a ray that misses is background without any query;
  * from the entry, with s the arc length and f = sigma sdf(scale x(s)), sigma the sign at the first sample (so a ray that enters
    the box inside the solid finds its first crossing, as the mesh of the box's grid shows it):  f < 0 after a positive sample
    brackets a crossing;  f < hit_eps is a hit;  else s += step_factor max(f / scale, min_step), a miss past the exit, out of
    steps after max_steps;
  * a bracket gets ``refine_steps`` secant steps (fraction clamped to [0.1, 0.9]); the hit is the last secant point;
  * posed heads: every sample is pulled back with the posed query's search (J0^-1 at the sample, Broyden 15 steps, cvg 1e-6,
    dvg 0.2); a sample whose search does not converge makes the ray invalid (as does the hit point's own search).
Normals: grad_x sdf at the hit (canonical), (I + dF/dx_c)^-T grad_{x_c} sdf at the root (posed), normalised and rounded as
render.cu rounds face normals.  The ensemble's eval-mode last-point-of-call quirk is not applied: the images are a render of the
field, not the mirror of a reference call.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _native

MINI = (-.55, -.5, -.95)            # the fitting grid's bounds (fitting_pointclouds.py)
MAXI = (0.55, 0.75, 0.4)
POSED_SEARCH = dict(max_steps=15, cvg_thresh=1e-6, dvg_thresh=0.2)
NORMAL_ROWS = 1 << 15               # rows of one normal evaluation: the ensemble backward's scratch grows with its rows
RAY_BYTES = 512                      # device bytes per ray and head that a chunk may take (state, queries, posed search)


def _cameras(poses, K, n, device):
    c2w = torch.from_numpy(np.stack([np.asarray(Rt, np.float64)[:3, :4].reshape(12) for Rt in poses])).to(device)
    k = np.asarray(K, np.float64)
    intr = torch.from_numpy(np.tile(np.array([k[0][0], k[1][1], k[0][2], k[1][2]]), (n, 1))).to(device)
    return c2w.contiguous(), intr.contiguous()


def trace(field, normal_fn, n_heads, poses, K, rend_size, znear=0.1, zfar=2.0, scale=1.0, mini=MINI, maxi=MAXI, max_steps=128,
          step_factor=0.6, hit_eps=5e-4, refine_steps=6, min_step=1e-4, check_every=8, max_rays=None, device=None):
    """The tracer for any field.  ``field(points (S, n, 3) float32) -> (sdf (S, n), valid (S, n) | None)`` evaluates the sample
    points of a step (rows past a head's count are padding); ``normal_fn(points (S, N, 3)) -> (grad (S, N, 3), jinv (S, N, 3, 3)
    | None, valid (S, N) | None)`` is called once per chunk at the scaled hit points.  ``check_every`` > 0: every that many march
    steps one read-back of the live counts ends the march when no ray is live and narrows the queries to the largest count;
    0: no read-back at all, every step queries every ray of the chunk.  Returns ``(depth (S, V, H, W), normals (S, V, H, W, 3)
    uint8, points (S, V, H, W, 3) world, status (S, V, H, W) uint8, steps (S, V, H, W) int32)``."""
    dev = device or torch.device('cuda', torch.cuda.current_device())
    H, W = int(rend_size[0]), int(rend_size[1])
    V, S = len(poses), int(n_heads)
    n_pix = V * H * W
    c2w, intr = _cameras(poses, K, V, dev)
    if max_rays is None:
        free, _ = torch.cuda.mem_get_info(dev)
        max_rays = max(S, min(free // (2 * RAY_BYTES), 1 << 22))
    N = max(1, min(n_pix, int(max_rays) // S))
    depth = torch.empty(S, n_pix, device=dev, dtype=torch.float32)
    normals = torch.empty(S, n_pix, 3, device=dev, dtype=torch.uint8)
    points = torch.empty(S, n_pix, 3, device=dev, dtype=torch.float32)
    status = torch.empty(S, n_pix, device=dev, dtype=torch.uint8)
    steps = torch.empty(S, n_pix, device=dev, dtype=torch.int32)
    with torch.no_grad():
        for p0 in range(0, n_pix, N):
            n = min(N, n_pix - p0)
            tr = _native.SdfTrace(S, n, mini, maxi, scale, znear, zfar, step_factor, min_step, hit_eps, max_steps, dev)
            buf = torch.empty(S, n, 3, device=dev, dtype=torch.float32)
            tr.begin(c2w, intr, H, W, p0)
            cols = n
            for k in range(int(max_steps)):
                tr.compact(refine=False)
                if check_every and k % check_every == 0:
                    cols = max(tr.counts())
                    if cols == 0:
                        break
                pts = tr.gather(cols, buf)
                sdf, valid = field(pts)
                tr.advance(False, sdf, valid)
            if refine_steps:
                tr.compact(refine=True)
                cols = max(tr.counts()) if check_every else n
                for _ in range(int(refine_steps) if cols else 0):
                    pts = tr.gather(cols, buf)
                    sdf, valid = field(pts)
                    tr.advance(True, sdf, valid)
            hits, piece = tr.points(), max(1, NORMAL_ROWS // S)
            parts = [normal_fn(hits[:, a:a + piece].contiguous()) for a in range(0, n, piece)]
            grad = torch.cat([g for g, _, _ in parts], dim=1)
            jinv = None if parts[0][1] is None else torch.cat([j for _, j, _ in parts], dim=1)
            valid = None if parts[0][2] is None else torch.cat([v for _, _, v in parts], dim=1)
            tr.finish(grad, jinv, valid, p0, depth, normals, points, status, steps)
    shape = (S, V, H, W)
    return depth.view(shape), normals.view(*shape, 3), points.view(*shape, 3), status.view(shape), steps.view(shape)


def _canonical_fns(decoder, lat):
    """(field, normal_fn) of S canonical heads, latents lat (S, D)."""
    from ..models.deepSDF import DeepSDF
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.fitting import _native_npm_decoder
    S = lat.shape[0]
    if isinstance(decoder, FastEnsembleDeepSDFMirrored):
        eng = decoder.engine()

        def field(pts):
            return eng.query(pts, lat, eval_quirk=False)[0].reshape(S, -1), None

        def normal_fn(pts):
            ones = torch.ones(pts.shape[1], device=pts.device)
            return torch.stack([eng.backward_inputs(pts[h], lat[h], ones)[2] for h in range(S)]), None, None
        return field, normal_fn
    if isinstance(decoder, DeepSDF) and _native_npm_decoder(decoder, 1):
        eng = decoder.engine()

        def field(pts):
            return eng.query(pts, lat).reshape(S, -1), None

        def normal_fn(pts):
            ones = torch.ones(pts.shape[0], pts.shape[1], 1, device=pts.device)
            return eng.backward_inputs(pts, lat, ones, want_xyz=True)[1], None, None
        return field, normal_fn
    raise ValueError('render_sdf_views: %s is not a decoder the tracer takes (FastEnsembleDeepSDFMirrored, or a native one-output '
                     'DeepSDF on CUDA)' % type(decoder).__name__)


def _posed_fns(decoder, decoder_expr, lat_rep_shape, codes):
    """(field, normal_fn) of one subject posed in the S expressions ``codes`` - the pieces of ``posed_evaluator``, with the Broyden
    search run without its early-exit read-back."""
    from ..models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from ..models.reconstruction import posed_parts
    parts = posed_parts(decoder, decoder_expr, lat_rep_shape, codes)
    if parts is None:
        raise ValueError('render_sdf_views: the decoder pair (%s, %s) has no native posed query (FastEnsembleDeepSDFMirrored with an '
                         'eval-mode DeformationNetwork, or the NPM DeepSDF pair, on one CUDA device)'
                         % (type(decoder).__name__, type(decoder_expr).__name__))
    _, cond, search, identity = parts
    S = codes.shape[0]
    ensemble = isinstance(decoder, FastEnsembleDeepSDFMirrored)

    def pull_back(pts):
        _, j0 = search.inverse_jacobian(pts, cond)
        xc, _, ok, _ = search.broyden_search(pts, cond, pts, j0, early_exit=False, compact=True, **POSED_SEARCH)
        return xc, ok

    def field(pts):
        xc, ok = pull_back(pts)
        return identity(xc, False), ok

    def normal_fn(pts):
        xc, ok = pull_back(pts)
        eng, z = identity.shape_engine, identity.z_id
        if ensemble:
            ones = torch.ones(S * xc.shape[1], device=xc.device)
            g = eng.backward_inputs(xc.reshape(-1, 3), z.reshape(-1), ones)[2].reshape(S, -1, 3)
        else:
            ones = torch.ones(S, xc.shape[1], 1, device=xc.device)
            g = eng.backward_inputs(xc, z.expand(S, -1).contiguous(), ones, want_xyz=True)[1]
        _, jinv = search.inverse_jacobian(xc, cond)
        return g, jinv, ok
    return field, normal_fn


def render_sdf_views(decoder, lat_rep_shape, poses, K, rend_size, znear=0.1, zfar=2.0, scale=1.0, decoder_expr=None,
                     lat_reps_expr=None, mini=None, maxi=None, max_steps=128, step_factor=0.6, hit_eps=5e-4, refine_steps=6,
                     min_step=1e-4, check_every=8, max_rays=None, return_points=False, return_stats=False):
    """Sphere-traced ``(depth (S, V, H, W) float32, normals (S, V, H, W, 3) uint8)`` of S heads in the views ``poses``
    (camera-to-world 4 x 4) with intrinsics K, in ``render_views``' format; pixel rays hit ``{x : sdf(scale x) = 0}``.

    Heads: ``lat_rep_shape`` is one code or S codes (``(D,)``, ``(S, D)`` or ``(S, 1, D)``) of ``decoder``
    (``FastEnsembleDeepSDFMirrored`` or a native one-output ``DeepSDF``).  With ``decoder_expr`` and ``lat_reps_expr`` (S expression
    codes): the one subject ``lat_rep_shape`` posed in each expression, for the decoder pairs ``posed_evaluator`` takes.  Anything
    else raises ``ValueError``.  The box defaults to the fitting grid's bounds; the march parameters are the module docstring's.
    The ensemble's eval-mode last-point quirk is not applied.

    ``return_points``: also the world hit points (S, V, H, W, 3) float32 (also set on invalid rays: the failing sample; 0 elsewhere).
    ``return_stats``: also a dict with ``status`` (S, V, H, W) uint8 (``_native.TRACE_*``), ``hit`` and ``valid`` masks, ``steps``
    (march steps per ray), and the counts ``n_hit``, ``n_miss``, ``n_out_of_steps``, ``n_invalid`` with ``steps_mean`` and
    ``steps_p99`` over the rays that entered the box."""
    if not torch.cuda.is_available():
        raise _native.NativeError('render_sdf_views traces on a CUDA device (no CPU fallback)')
    dev = next(decoder.parameters()).device
    if dev.type != 'cuda':
        raise ValueError('render_sdf_views: the decoder must be on a CUDA device (got %s)' % dev)
    if (decoder_expr is None) != (lat_reps_expr is None):
        raise ValueError('render_sdf_views: give both decoder_expr and lat_reps_expr, or neither')
    if decoder_expr is None:
        lat = lat_rep_shape.reshape(-1, lat_rep_shape.shape[-1]).to(device=dev, dtype=torch.float32).contiguous()
        field, normal_fn = _canonical_fns(decoder, lat)
        S = lat.shape[0]
    else:
        codes = lat_reps_expr.reshape(-1, lat_reps_expr.shape[-1]).to(device=dev, dtype=torch.float32)
        field, normal_fn = _posed_fns(decoder, decoder_expr, lat_rep_shape, codes)
        S = codes.shape[0]
    with torch.cuda.device(dev):
        depth, normals, points, status, steps = trace(
            field, normal_fn, S, poses, K, rend_size, znear, zfar, scale, MINI if mini is None else mini,
            MAXI if maxi is None else maxi, max_steps, step_factor, hit_eps, refine_steps, min_step, check_every, max_rays, dev)
    out = (depth, normals)
    if return_points:
        out += (points,)
    if return_stats:
        out += (trace_stats(status, steps),)
    return out


def trace_stats(status, steps):
    """The counts and step statistics of a trace (one read-back)."""
    hist = torch.bincount(steps.reshape(-1).long()).cpu().numpy()[1:]           # rays that entered the box: steps >= 1
    n = int(hist.sum())
    counts = torch.bincount(status.reshape(-1).long(), minlength=6).tolist()
    return dict(status=status, steps=steps, hit=status == _native.TRACE_HIT, valid=status != _native.TRACE_INVALID,
                n_hit=counts[_native.TRACE_HIT], n_miss=counts[_native.TRACE_MISS], n_out_of_steps=counts[_native.TRACE_OUT_OF_STEPS],
                n_invalid=counts[_native.TRACE_INVALID],
                steps_mean=float((hist * np.arange(1, len(hist) + 1)).sum() / n) if n else 0.0,
                steps_p99=float(np.searchsorted(np.cumsum(hist), 0.99 * n) + 1) if n else 0.0)
