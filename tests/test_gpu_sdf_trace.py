"""Sphere tracing on the GPU (csrc/sdf_trace.cu, evaluation/sdf_render.py): the step kernels against the float64 mirror on an
analytic field, seeded NPHM and NPM heads against float64 (surface, first hit, background, normals), posed heads, batching,
determinism, chunking and the sync-free march."""
import numpy as np
import pytest
import torch

import sdf_trace_common as T
from conftest import MAXI, MINI, make_deformation, make_ensemble, sample_latent

pytestmark = pytest.mark.gpu

H, W, SCALE = 160, 120, 4.0
# measured bounds (H100): the float64 SDF at a hit is within SURF of 0 (hit_eps 5e-4 plus the fp32 field's error and what a
# refined bracket leaves), normals within NORMAL_DEG of the float64 gradient
SURF = 2.5e-3
NORMAL_DEG = 3.0


def _cams(n=3):
    from nphm_b200.evaluation.render_utils import KK, render_cameras
    K = KK.astype(np.float64).copy()
    K[:2] /= 8.0                                                     # the evaluation cameras at 1/8 resolution: 160 x 120
    cams, poses = render_cameras(10)
    return [cams[i] for i in (0, 4, 7)][:n], [poses[i] for i in (0, 4, 7)][:n], K


def _f64_ensemble(device):
    """conftest.make_ensemble(0) in float64 (its forward then takes the composite path)."""
    d = make_ensemble(0, device=device).double().train()
    d.anchors = d.anchors.double()
    return d


def _f64_sdf(dec64, lat, x, grad=False, chunk=20000):
    """float64 composite SDF (and autograd gradient) of the training-mode forward at points x (n, 3)."""
    out, g = [], []
    lat = lat.double().reshape(1, 1, -1)
    for a in range(0, len(x), chunk):
        with torch.enable_grad():
            p = x[a:a + chunk].double().detach().requires_grad_(grad)
            s = dec64(p[None], lat.expand(1, len(p), -1), None)
            s = (s[0] if isinstance(s, tuple) else s).reshape(-1)
            if grad:
                g.append(torch.autograd.grad(s.sum(), p)[0])
        out.append(s.detach())
    return (torch.cat(out), torch.cat(g)) if grad else torch.cat(out)


def _hits(points, status):
    hit = status == T.HIT
    return points[hit], hit


def _decode_normals(n):
    return n.double() / 255 * 2 - 1


def test_step_kernels_match_the_float64_mirror(cuda_device):
    from nphm_b200.evaluation.sdf_render import trace
    _, poses, K = _cams()
    centres = torch.tensor([[0.02, 0.05, 0.1], [-0.05, 0.0, -0.25]], dtype=torch.float64)
    radii = (0.3, 0.35)

    def f64(x):
        return torch.minimum((x - centres[0].to(x)).norm(dim=-1) - radii[0], (x - centres[1].to(x)).norm(dim=-1) - radii[1])

    def field(pts):
        return f64(pts.double()).float(), None

    def normal_fn(pts):
        return pts.clone(), None, None
    kw = dict(scale=SCALE, max_steps=64, step_factor=0.9, hit_eps=5e-4, refine_steps=4)
    depth, _, _, status, steps = trace(field, normal_fn, 1, poses, K, (H, W), check_every=0, device=cuda_device, **kw)
    o, u, cos = [a.reshape(-1, a.shape[-1]) if a.ndim == 4 else a.reshape(-1) for a in T.pixel_rays(poses, K, (H, W))]
    s_in, s_out = T.box_interval(o, u, cos, MINI, MAXI, SCALE, 0.1, 2.0)
    ref_status, s, ref_steps = T.march(lambda x: f64(torch.from_numpy(x)).numpy(), o, u, s_in, s_out, scale=SCALE, min_step=1e-4,
                                       **{k: v for k, v in kw.items() if k != 'scale'})
    st = status.reshape(-1).cpu().numpy()
    # rays whose closest approach to a sphere is within hit_eps of tangency may classify either way
    tangent = np.zeros(len(st), bool)
    for c, r in zip(centres.numpy(), radii):
        oc = o * SCALE - c
        b = (oc * u).sum(-1)
        dist = np.sqrt(np.maximum((oc * oc).sum(-1) - b * b, 0))
        tangent |= np.abs(dist - r) < 5e-4 * 4
    differ = (st != ref_status) & ~tangent
    print('mirror: %d rays, %d hits, %d tangent-exempt, %d class differences: %s' % (len(st), (st == T.HIT).sum(), tangent.sum(),
                                                                                  differ.sum(), np.nonzero(differ)[0][:20]))
    assert differ.sum() == 0
    both = (st == T.HIT) & (ref_status == T.HIT) & ~tangent
    d = depth.reshape(-1).double().cpu().numpy()
    err = np.abs(d[both] - s[both] * cos[both])
    print('mirror depth: max |err| %.3g, steps equal on %.4f' % (err.max(), (steps.reshape(-1).cpu().numpy() == ref_steps)[both].mean()))
    # measured on the H100: max 1.1e-4 (a ray whose fp32 and float64 samples straddle hit_eps once), 99 % within 2e-6
    assert err.max() < 2.5e-4 and (err < 2e-6).mean() > 0.99


def test_seeded_ensemble_surface_first_hit_background_normals(cuda_device):
    from nphm_b200.evaluation.render_utils import render_sdf_views
    dec = make_ensemble(0, device=cuda_device).train()
    lat = sample_latent(1).to(cuda_device)
    _, poses, K = _cams()
    depth, normals, points, stats = render_sdf_views(dec, lat, poses, K, (H, W), scale=SCALE, return_points=True, return_stats=True)
    print('ensemble stats', {k: v for k, v in stats.items() if not torch.is_tensor(v)})
    assert stats['n_hit'] > 0.05 * depth.numel() and stats['n_out_of_steps'] < 0.1 * depth.numel()
    dec64 = _f64_ensemble(cuda_device)
    st = stats['status'][0]
    hit = st == T.HIT
    x = points[0][hit].double() * SCALE
    s, g = _f64_sdf(dec64, lat, x, grad=True)
    print('surface: max |sdf64| at hits %.3g' % float(s.abs().max()))
    assert float(s.abs().max()) < SURF
    n = _decode_normals(normals[0][hit])
    cosang = (torch.nn.functional.normalize(n, dim=-1) * torch.nn.functional.normalize(g, dim=-1)).sum(-1).clamp(-1, 1)
    ang = torch.rad2deg(torch.acos(cosang))
    print('normals: max angle %.3f deg, p99 %.3f' % (float(ang.max()), float(torch.quantile(ang, 0.99))))
    assert float(ang.max()) < NORMAL_DEG
    # first hit and background: dense float64 samples of a subset of rays from the box entry to the hit (or the exit)
    o, u, cos = [torch.from_numpy(a.reshape(-1, a.shape[-1]) if a.ndim == 4 else a.reshape(-1)).to(cuda_device)
                 for a in T.pixel_rays(poses, K, (H, W))]
    s_in, s_out = [torch.from_numpy(a).to(cuda_device) for a in T.box_interval(o.cpu().numpy(), u.cpu().numpy(), cos.cpu().numpy(),
                                                                                MINI, MAXI, SCALE, 0.1, 2.0)]
    flat_hit = hit.reshape(-1)
    rng = np.random.RandomState(0)
    inside = torch.nonzero(s_in <= s_out)[:, 0].cpu().numpy()
    sel = torch.from_numpy(rng.choice(inside, min(1500, len(inside)), replace=False)).to(cuda_device)
    end = torch.where(flat_hit[sel], depth[0].reshape(-1)[sel].double() / cos[sel], s_out[sel])
    k = torch.linspace(0, 1, 257, device=cuda_device, dtype=torch.float64)[:-1]
    ss = s_in[sel, None] + (end - s_in[sel])[:, None] * k[None]
    xs = SCALE * (o[sel, None] + ss[..., None] * u[sel, None])
    f = _f64_sdf(dec64, lat, xs.reshape(-1, 3)).reshape(len(sel), -1)
    f = f * torch.where(f[:, :1] < 0, -1.0, 1.0)                     # the march runs on the sign at the entry
    early = (f[flat_hit[sel]] < -SURF).any(dim=1)
    miss = st.reshape(-1)[sel] == T.MISS                             # out-of-steps rays are reported, not background
    bg = (f[miss] < -SURF).any(dim=1)
    print('first hit: %d of %d hit rays cross earlier; background: %d of %d missed rays dip below -%g'
          % (int(early.sum()), int(flat_hit[sel].sum()), int(bg.sum()), int(miss.sum()), SURF))
    assert int(early.sum()) == 0 and int(bg.sum()) == 0


def test_seeded_ensemble_agrees_with_the_mesh_path(cuda_device):
    """Against render_views of the 256^3 narrow-band mesh, on the rays whose field stays clear of hit_eps until its first sign
    change (or everywhere, for rays without one).

    The seeded head's field comes within hit_eps of 0 without changing sign over much of the box (its median |sdf| at the box
    entries of these views is 5e-5 on the H100): by the contract the march stops there, while marching cubes only meshes sign
    changes, so the two paths differ on those rays by design.  A dense fp32 sampling of every ray (1024 samples from the box
    entry to the exit) finds them; on all other rays both paths must see the same first crossing."""
    from nphm_b200.evaluation.render_utils import render_sdf_views, render_views
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    hit_eps = 5e-4
    dec = make_ensemble(0, device=cuda_device).train()
    lat = sample_latent(1).to(cuda_device)
    _, poses, K = _cams()
    depth, _, stats = render_sdf_views(dec, lat, poses, K, (H, W), scale=SCALE, hit_eps=hit_eps, max_steps=512, return_stats=True)
    mesh = extract_mesh_narrowband(dec, lat.reshape(1, 1, -1), MINI, MAXI, 256)
    d_mesh, _ = render_views(np.asarray(mesh.vertices) / SCALE, mesh.faces, poses, K, (H, W))
    voxel = (np.asarray(MAXI) - np.asarray(MINI)).max() / 255 / SCALE
    o, u, cos = [torch.from_numpy(a.reshape(-1, a.shape[-1]) if a.ndim == 4 else a.reshape(-1)).to(cuda_device)
                 for a in T.pixel_rays(poses, K, (H, W))]
    s_in, s_out = [torch.from_numpy(a).to(cuda_device) for a in T.box_interval(o.cpu().numpy(), u.cpu().numpy(), cos.cpu().numpy(),
                                                                                MINI, MAXI, SCALE, 0.1, 2.0)]
    rays = torch.nonzero(s_in <= s_out)[:, 0]
    k = torch.linspace(0, 1, 1024, device=cuda_device, dtype=torch.float64)
    clean = torch.zeros_like(s_in, dtype=torch.bool)
    eng = dec.engine()
    for piece in rays.split(4096):
        ss = s_in[piece, None] + (s_out - s_in)[piece, None] * k[None]
        xs = SCALE * (o[piece, None] + ss[..., None] * u[piece, None])
        f = eng.query(xs.reshape(1, -1, 3).float(), lat.reshape(1, -1), eval_quirk=False)[0].reshape(len(piece), -1).double()
        g = f * torch.where(f[:, :1] < 0, -1.0, 1.0)
        neg = g < 0
        s_cross = torch.where(neg.any(1), ss.gather(1, neg.double().argmax(1, keepdim=True))[:, 0], s_out[piece] + 1.0)
        before = ss < (s_cross - 2 * voxel)[:, None]                # the approach to the crossing itself is left to the tolerance
        clean[piece] = ~((f.abs() < hit_eps) & before).any(1)
    clean &= stats['status'][0].reshape(-1) != T.OUT_OF_STEPS
    a, b = (depth[0].reshape(-1) > 0) & clean, (d_mesh.reshape(-1) > 0) & clean
    both = a & b
    err = (depth[0].reshape(-1)[both] - d_mesh.reshape(-1)[both]).abs()
    close = float((err <= 2 * voxel).double().mean())
    share = float((a ^ b).double().sum() / (a | b).double().sum())
    print('mesh path: %d of %d rays in the box clear of hit_eps before their first crossing, %d hit by both; %.4f within 2 voxels '
          '(max %.3g, voxel %.3g); hit masks differ on %.4f of the hit pixels'
          % (int(clean.sum()), len(rays), int(both.sum()), close, float(err.max()), voxel, share))
    assert int(both.sum()) > 1000 and close > 0.99 and share < 0.02


def test_batching_determinism_chunking_and_no_read_back(cuda_device):
    from nphm_b200.evaluation.render_utils import render_sdf_views
    from nphm_b200.evaluation.sdf_render import _canonical_fns, trace
    dec = make_ensemble(0, device=cuda_device).train()
    lats = torch.stack([sample_latent(s) for s in (1, 2, 3)]).to(cuda_device)
    _, poses, K = _cams(2)
    together = render_sdf_views(dec, lats, poses, K, (H, W), scale=SCALE)
    again = render_sdf_views(dec, lats, poses, K, (H, W), scale=SCALE)
    chunked = render_sdf_views(dec, lats, poses, K, (H, W), scale=SCALE, max_rays=3 * 7001)
    no_sync = render_sdf_views(dec, lats, poses, K, (H, W), scale=SCALE, check_every=0)
    for h in range(3):
        one = render_sdf_views(dec, lats[h], poses, K, (H, W), scale=SCALE)
        assert torch.equal(one[0][0], together[0][h]) and torch.equal(one[1][0], together[1][h])
    for other in (again, chunked, no_sync):
        assert torch.equal(other[0], together[0]) and torch.equal(other[1], together[1])
    # a march step reads nothing back: the sync-free trace with torch's sync check set to error
    field, normal_fn = _canonical_fns(dec, lats)
    steps = []

    def checked(pts):
        torch.cuda.set_sync_debug_mode('error')
        try:
            out = field(pts)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        steps.append(1)
        return out
    d = trace(checked, normal_fn, 3, poses, K, (H, W), scale=SCALE, check_every=0, max_steps=8, refine_steps=0, device=cuda_device)
    assert len(steps) == 8 and d[0].shape == (3, 2, H, W)


def test_synthetic_single_view_observation(cuda_device):
    from nphm_b200.evaluation.render_utils import render_sdf_views, samples_from_images
    dec = make_ensemble(0, device=cuda_device).train()
    lat = sample_latent(1).to(cuda_device)
    cams, poses, K = _cams(1)
    depth, normals = render_sdf_views(dec, lat, poses, K, (H, W), scale=SCALE)
    pts, _ = samples_from_images(depth[0], normals[0], cams, poses, SCALE, K=K, rend_size=(H, W))
    s = _f64_sdf(_f64_ensemble(cuda_device), lat, pts)
    print('single view: %d points, max |sdf64| %.3g' % (len(pts), float(s.abs().max())))
    assert len(pts) > 1000 and float(s.abs().max()) < 4 * SURF


def test_npm_canonical(cuda_device):
    import posed_common as P
    from nphm_b200.evaluation.render_utils import render_sdf_views
    dec, _, lat, _, _, _ = P.npm_case(cuda_device)                   # the identity decoder and code of the NPM posed case
    _, poses, K = _cams()
    depth, normals, points, stats = render_sdf_views(dec, lat, poses, K, (H, W), scale=SCALE, return_points=True, return_stats=True)
    print('npm stats', {k: v for k, v in stats.items() if not torch.is_tensor(v)})
    hit = stats['hit'][0]
    assert stats['n_hit'] > 1000
    d64 = P.npm_case(cuda_device)[0].double()
    with torch.enable_grad():
        x = (points[0][hit].double() * SCALE).requires_grad_(True)
        s = d64(x[None], lat.double().reshape(1, 1, -1).expand(1, len(x), -1), None)
        s = (s[0] if isinstance(s, tuple) else s).reshape(-1)
        g = torch.autograd.grad(s.sum(), x)[0]
    n = _decode_normals(normals[0][hit])
    ang = torch.rad2deg(torch.acos((torch.nn.functional.normalize(n, dim=-1) * torch.nn.functional.normalize(g, dim=-1)).sum(-1)
                                   .clamp(-1, 1)))
    print('npm: max |sdf64| %.3g, max normal angle %.3f' % (float(s.abs().max()), float(ang.max())))
    assert float(s.abs().max()) < SURF and float(ang.max()) < NORMAL_DEG


@pytest.mark.parametrize('pair', ['ensemble', 'npm'])
def test_posed_heads(cuda_device, pair):
    import posed_common as P
    from nphm_b200.evaluation.render_utils import render_sdf_views
    from nphm_b200.models.reconstruction import get_logits_posed
    if pair == 'ensemble':
        dec, dfn, _, z_ex, _, _ = P.ensemble_case(cuda_device, training=True)
        lat = sample_latent(1).to(cuda_device).reshape(1, 1, -1)     # the seeded head of the canonical tests
    else:
        dec, dfn, lat, z_ex, _, _ = P.npm_case(cuda_device)
    _, poses, K = _cams(2)
    depth, normals, points, stats = render_sdf_views(dec, lat, poses, K, (H, W), scale=SCALE, decoder_expr=dfn, lat_reps_expr=z_ex,
                                                     return_points=True, return_stats=True)
    print('posed %s stats' % pair, {k: v for k, v in stats.items() if not torch.is_tensor(v)})
    assert depth.shape[0] == z_ex.shape[0] and stats['n_hit'] > 500
    for e in range(z_ex.shape[0]):
        st = stats['status'][e]
        for want, label in ((T.HIT, 'hit'), (T.INVALID, 'invalid')):
            sel = st == want
            if not sel.any():
                continue
            x = (points[e][sel] * SCALE).reshape(1, -1, 3)
            sdf, valid = get_logits_posed(dec, dfn, lat, z_ex[e], x, nbatch_points=x.shape[1] + 1, return_valid=True)
            if want == T.HIT:
                print('posed %s expr %d: %d hits, valid %.4f, max |sdf| %.3g' % (pair, e, sel.sum(), valid.mean(), np.abs(sdf).max()))
                assert valid.mean() > 0.999 and np.abs(sdf[valid]).max() < SURF
            else:
                print('posed %s expr %d: %d invalid rays, search valid at %.4f of their samples' % (pair, e, sel.sum(), valid.mean()))
                assert valid.mean() < 0.01
        # normals against float64 central differences of the posed field (through the fp32 posed query, h = 1e-3)
        hit = st == T.HIT
        idx = torch.nonzero(hit.reshape(-1))[:, 0][:300]
        x = (points[e].reshape(-1, 3)[idx] * SCALE).double()
        h = 1e-3
        g = torch.zeros_like(x)
        for a in range(3):
            dx = torch.zeros(3, dtype=torch.float64, device=x.device)
            dx[a] = h
            fp = get_logits_posed(dec, dfn, lat, z_ex[e], (x + dx).float()[None], nbatch_points=10 ** 6)
            fm = get_logits_posed(dec, dfn, lat, z_ex[e], (x - dx).float()[None], nbatch_points=10 ** 6)
            g[:, a] = torch.from_numpy((fp.astype(np.float64) - fm) / (2 * h)).to(x.device)
        n = _decode_normals(normals[e].reshape(-1, 3)[idx])
        ang = torch.rad2deg(torch.acos((torch.nn.functional.normalize(n, dim=-1) * torch.nn.functional.normalize(g, dim=-1)).sum(-1)
                                       .clamp(-1, 1)))
        print('posed %s expr %d: normal angle max %.3f, p99 %.3f deg' % (pair, e, float(ang.max()), float(torch.quantile(ang, 0.99))))
        assert float(torch.quantile(ang, 0.99)) < 2 * NORMAL_DEG


def test_rejects_other_decoders(cuda_device):
    from nphm_b200.evaluation.render_utils import render_sdf_views
    _, poses, K = _cams(1)
    with pytest.raises(ValueError):
        render_sdf_views(torch.nn.Linear(3, 1).to(cuda_device), torch.zeros(4, device=cuda_device), poses, K, (8, 8))
    dec = make_ensemble(0, device=cuda_device)
    dfn = make_deformation(cuda_device).train()                      # a training-mode deformation network has no native query
    with pytest.raises(ValueError):
        render_sdf_views(dec, sample_latent(1).to(cuda_device), poses, K, (8, 8), decoder_expr=dfn,
                         lat_reps_expr=torch.zeros(1, 200, device=cuda_device))
