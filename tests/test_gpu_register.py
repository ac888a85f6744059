"""Global registration on the GPU (csrc/register.cu, models/registration.py, DESIGN.md §4.25): the kernels against the float64
mirror, bitwise repeatability and batch independence, recovery of random similarities on an analytic volume, the ambiguity
statistic, the head volume, and register_scans followed by the pose fit on a distance-like decoder head."""
import math

import numpy as np
import pytest
import torch

import register_common as RC
from conftest import MAXI, MINI, make_ensemble, make_npm
from pose_common import clamp_in_a_gap, similarity
from nphm_b200.models import registration as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def asym(cuda_device):
    return RC.volume(RC.ASYMMETRIC, 128, cuda_device), RC.surface_points(RC.ASYMMETRIC, 6000, seed=1)


def test_prepare_equals_the_mirror_bit_for_bit(cuda_device, asym):
    vol, _ = asym
    noise = torch.from_numpy(np.random.RandomState(2).uniform(-1, 1, 37 ** 3).astype(np.float32)).to(cuda_device)
    for v, res in ((vol, 128), (noise, 37)):
        grid = G.Grid(res, MINI, MAXI)
        assert torch.equal(G.prepare(v, grid), G.prepare_torch(v, grid))


def _near_poses(pts, n, seed):
    """n scans of the points under random similarities and, per scan, a table row within ~5 degrees / 0.02 / 3 % of its
    inverse, with every moved point inside the grid."""
    rng = np.random.RandomState(seed)
    rows, scans = [], []
    for k in range(n):
        R, t, ls = RC.random_similarity(rng, max_trans=0.2)
        scans.append(RC.to_scan(pts, R, t, ls).float())
        W, _, _ = similarity(3.0 + k, rng.randn(3), (0, 0, 0), 1.0)
        Rinv = W @ R.T
        rows.append(torch.cat([Rinv.reshape(9), -math.exp(-ls) * Rinv @ t + torch.from_numpy(rng.randn(3) * 0.01),
                               torch.tensor([-ls + 0.02 * rng.randn()])]))
    return torch.stack(rows), scans


def _stage_inputs(scans, device):
    points = torch.cat(scans).to(device).contiguous()
    counts_h = [s.shape[0] for s in scans]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts_h)[:-1]]), dtype=torch.int64, device=device)
    return points, offsets, torch.tensor(counts_h, dtype=torch.int32, device=device)


def _rot_err(a, b):
    Ra, Rb = a[:, :9].reshape(-1, 3, 3), b[:, :9].reshape(-1, 3, 3)
    c = (((Ra.transpose(1, 2) @ Rb).diagonal(dim1=1, dim2=2).sum(-1) - 1) / 2).clamp(-1, 1)
    return float(torch.arccos(c).max())


def test_one_iteration_matches_the_mirror(cuda_device, asym):
    vol, (pts, _) = asym
    grid = G.Grid(128, MINI, MAXI)
    field = G.prepare(vol, grid)
    table, scans = _near_poses(pts[:3000], 6, seed=3)
    points, offsets, counts = _stage_inputs(scans, cuda_device)
    hyp_obs = torch.arange(6, dtype=torch.int32, device=cuda_device)
    unit = torch.linspace(0.8, 1.2, 6, dtype=torch.float64, device=cuda_device)
    table = table.to(cuda_device)
    seed = table[:, 12].clone()
    p, mask = G._hypothesis_points(points, offsets, counts, hyp_obs, 3000)
    inside, r0, _, _ = G.residuals_f64(field, grid, table, p, unit)
    assert bool(inside.all())
    gap_tau = clamp_in_a_gap(r0.abs())
    for fit_scale in (True, False):
        for tau in (math.inf, gap_tau):
            got, want = table.clone(), table.clone()
            sg, ig = G.search(field, grid, points, offsets, counts, unit, got, seed, hyp_obs, 3000, 1, (tau, tau), 1e-3,
                              fit_scale, 3000)
            sw, iw = G.search_f64(field, grid, points, offsets, counts, unit, want, seed, hyp_obs, 3000, 1, (tau, tau), 1e-3,
                                  fit_scale)
            step = _rot_err(table, want)
            e = (_rot_err(got, want), float((got[:, 9:12] - want[:, 9:12]).abs().max()),
                 float((got[:, 12] - want[:, 12]).abs().max()))
            print('one iteration (fit_scale %d, tau %.3g): step %.3g rad; kernel - mirror: %.2e rad, %.2e units, %.2e log scale; '
                  'score %.2e rel' % (fit_scale, tau, step, *e, float(((sg - sw).abs() / sw).max())))
            assert step > 1e-3 and max(e) < 1e-6
            assert torch.equal(ig, iw)
            assert float(((sg - sw).abs() / sw).max()) < 1e-4


def _register(vol, scans, **kw):
    return G.register_observations(vol, MINI, MAXI, scans, return_stats=True, **kw)


def test_bitwise_repeatable_and_independent_of_the_batch(cuda_device, asym):
    vol, (pts, nrm) = asym
    rng = np.random.RandomState(5)
    moves = [RC.random_similarity(rng) for _ in range(6)]
    obs = [RC.to_scan(pts[:2000 + 300 * k], *m).float().to(cuda_device) for k, m in enumerate(moves)]
    scans = [obs[:3], obs[3:]]
    poses, stats = _register(vol, scans)
    again, stats2 = _register(vol, scans)
    for a, b, sa, sb in zip(poses, again, stats, stats2):
        assert torch.equal(a.table, b.table) and all(torch.equal(sa[k], sb[k]) for k in sa)
    for k in range(6):
        single, st = _register(vol, [[obs[k]]])
        assert torch.equal(single[0].table[0], poses[k // 3].table[k % 3])
        assert torch.equal(st[0]['score'][0], stats[k // 3]['score'][k % 3])
    # hypothesis counts per observation that are not multiples of a CTA's 8 warps: some CTAs hold hypotheses of two
    # observations, and those of the second read their points from global memory
    odd = dict(n_rotations=1021, fine=dict(top_k=5))
    poses, stats = _register(vol, [obs[:2]], **odd)
    for k in range(2):
        single, st = _register(vol, [[obs[k]]], **odd)
        assert torch.equal(single[0].table[0], poses[0].table[k]) and torch.equal(st[0]['score'][0], stats[0]['score'][k])


def _errors(poses, moves):
    return [RC.pose_error(poses[0], o, *m) for o, m in enumerate(moves)]


def test_recovers_random_similarities_on_the_asymmetric_volume(cuda_device, asym):
    vol, (pts, nrm) = asym
    rng = np.random.RandomState(7)
    moves = [RC.random_similarity(rng) for _ in range(32)]
    g = torch.Generator().manual_seed(8)
    full = [RC.to_scan(pts[torch.randperm(pts.shape[0], generator=g)[:4000]], *m).float().to(cuda_device) for m in moves]
    patches = [RC.to_scan(RC.patch(pts, nrm, 100 + o, 4000), *m).float().to(cuda_device) for o, m in enumerate(moves)]
    for name, obs, bounds in (('full', full, (1.0, 5e-3, 5e-3)), ('patch', patches, (2.0, 1e-2, 1e-2))):
        poses, stats = _register(vol, [obs])
        errs = np.array(_errors(poses, moves))
        print('%s surfaces (%d..%d points): worst %.3g deg, %.3g units, %.3g scale; median %.3g deg; inliers >= %.3f'
              % (name, min(len(o) for o in obs), max(len(o) for o in obs), *errs.max(0), float(np.median(errs[:, 0])),
                 float(stats[0]['inlier_fraction'].min())))
        bad = [(o, tuple(e)) for o, e in enumerate(errs) if not (e < np.array(bounds)).all()]
        assert not bad, bad
    # millimetre-like: the scan 1000 times larger (pose scale 1e-3), turned upside down and moved half a head away
    R, t, _ = similarity(170.0, (0.2, 0.1, 1.0), (150.0, -200.0, 100.0), 1.0)
    mm = RC.to_scan(pts[:4000], R, t, math.log(1000.0)).float().to(cuda_device)
    poses, _ = _register(vol, [[mm]])
    e_mm = RC.pose_error(poses[0], 0, R, t, math.log(1000.0))
    # known scale: a rigid search
    Rk, tk, lk = moves[0]
    poses_k, _ = _register(vol, [[full[0]]], log_scale=-lk)
    e_k = RC.pose_error(poses_k[0], 0, Rk, tk, lk)
    print('millimetre scan: %.3g deg, %.3g units, %.3g scale; known log scale: %.3g deg, %.3g units' % (*e_mm, *e_k[:2]))
    assert e_mm[0] < 1.0 and e_mm[1] < 5e-3 and e_mm[2] < 5e-3
    assert not poses_k[0].fit_scale and e_k[0] < 1.0 and e_k[1] < 5e-3


def test_runner_up_flags_ambiguity(cuda_device, asym):
    vol, (pts, _) = asym
    rev = RC.volume(RC.REVOLUTION, 128, cuda_device)
    rpts, _ = RC.surface_points(RC.REVOLUTION, 4000, seed=9)
    rng = np.random.RandomState(10)
    m = RC.random_similarity(rng)
    _, st_rev = _register(rev, [[RC.to_scan(rpts, *m).float().to(cuda_device)]])
    _, st_asym = _register(vol, [[RC.to_scan(pts[:4000], *m).float().to(cuda_device)]])
    sr, ur = float(st_rev[0]['score'][0]), float(st_rev[0]['runner_up'][0])
    sa, ua = float(st_asym[0]['score'][0]), float(st_asym[0]['runner_up'][0])
    print('ambiguity: revolution score %.3g runner-up %.3g; asymmetric score %.3g runner-up %.3g' % (sr, ur, sa, ua))
    assert ur <= 1.1 * sr
    assert ua >= 3 * sa


# ------------------------------------------------------------------------------------------------------------ decoder heads
def test_head_volume_is_the_native_grid_query(cuda_device):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    dec = make_ensemble(0, device=cuda_device).train()
    vol = G.head_volume(dec, None, 48, MINI, MAXI, cuda_device)
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, 48)).to(cuda_device, torch.float32).reshape(1, -1, 3)
    want = get_logits(dec, torch.zeros(1, 1, dec.lat_dim, device=cuda_device), grid)     # training mode: no quirk
    assert np.array_equal(vol.cpu().numpy(), want)
    npm = make_npm(cuda_device)
    assert G.head_volume(npm, None, 24, MINI, MAXI, cuda_device).shape == (24 ** 3,)


ID_LAMBDAS = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2}, 'symm_dist': {200: 10}, 'reg_glob': {200: 3}, 'reg_loc': {200: 3}, 'reg_expr': {200: 10}}
MOVES = [((120.0, (0.3, 1.0, 0.2)), (0.3, 0.0, 0.0)), ((170.0, (1.0, -0.2, 0.4)), (0.0, -0.3, 0.0)),
         ((65.0, (-0.5, 0.3, 1.0)), (0.0, 0.0, 0.3))]


def _surface_points(dec, device, n_obs, n_points, seed):
    """test_gpu_pose.py's fixture: vertices of the decoder's zero-code mesh at 128^3, n_points per observation."""
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    z = torch.zeros(1, 1, dec.lat_dim, device=device)
    mesh = extract_mesh_narrowband(dec, z, MINI, MAXI, 128)
    v = torch.from_numpy(np.asarray(mesh.vertices, dtype=np.float64))
    g = torch.Generator().manual_seed(seed)
    return [v[torch.randint(0, v.shape[0], (n_points,), generator=g)] for _ in range(n_obs)]


def _rms_sdf(dec, z, pts_model):
    with torch.no_grad():
        sdf = dec.engine().query(pts_model.reshape(1, -1, 3).float().to(z.device), z.reshape(1, -1))
    return float(sdf.double().square().mean().sqrt())


def test_register_then_fit_a_millimetre_scan(cuda_device):
    """The pipeline on a distance-like decoder head (the DeepSDF fitted to the asymmetric head): 3 observations moved by 120,
    170 and 65 degrees about tilted axes and 0.3 units, the scan 1000 times larger than the model (millimetre-like).
    register_scans, then inference_identity_space with the poses, meets test_gpu_pose.py's recovery bounds and fits as
    well as the aligned scan without poses; the same fit from the identity pose does not."""
    from nphm_b200.models import fitting as F
    from nphm_b200.models.pose import ObservationPoses
    dec = RC.fitted_head(cuda_device)
    model_pts = _surface_points(dec, cuda_device, 3, 4000, seed=13)
    moves = [similarity(a, ax, np.array(t) * 1000.0, 1000.0) for (a, ax), t in MOVES]
    scan = [RC.to_scan(p, R, t, ls).float().to(cuda_device) for p, (R, t, ls) in zip(model_pts, moves)]
    aligned = [p.float().to(cuda_device) for p in model_pts]
    out = {}
    for mode in ('registered', 'identity', 'unposed', 'aligned'):
        poses = (G.register_scans(dec, [scan])[0] if mode == 'registered' else
                 ObservationPoses(3, cuda_device) if mode == 'identity' else None)
        if mode == 'registered':
            out['registration'] = np.array([RC.pose_error(poses, o, *m) for o, m in enumerate(moves)]).max(0)
        obs = aligned if mode == 'aligned' else scan
        torch.manual_seed(14)
        z, _ = F.inference_identity_space(dec, obs, dict(ID_LAMBDAS), 600, SCHEDULE, 1, poses=poses)
        to_model = (lambda p, o: poses.to_model(p.double(), o)) if poses is not None else (lambda p, o: p.double())
        rms = _rms_sdf(dec, z, torch.cat([to_model(s, o) for o, s in enumerate(obs)]))
        errs = (np.array([RC.pose_error(poses, o, *m) for o, m in enumerate(moves)]).max(0) if poses is not None else None)
        out[mode] = (rms, errs)
    (rms_reg, err), (rms_id, err_id) = out['registered'], out['identity']
    rms_un, rms_al = out['unposed'][0], out['aligned'][0]
    print('register -> fit: registration alone (%.3g deg, %.3g units, %.3g scale); after the fit rms %.3g (aligned scan '
          'without poses %.3g, unposed %.3g, from the identity pose %.3g); pose (%.3g deg, %.3g units, %.3g scale), from the '
          'identity pose (%.3g deg, %.3g units, %.3g scale)'
          % (*out['registration'], rms_reg, rms_al, rms_un, rms_id, *err, *err_id))
    assert rms_reg < 0.05 * rms_un and err[0] < 0.5 and err[1] < 5e-3 and err[2] < 5e-3
    assert rms_reg <= 2 * rms_al + 1e-4
    assert not (rms_id < 0.05 * rms_un and err_id[0] < 0.5 and err_id[1] < 5e-3 and err_id[2] < 5e-3)


def test_single_sphere_traced_view(cuda_device):
    """One sphere-traced view of the fitted head, back-projected and turned by 150 degrees: after register_scans the RMS SDF
    of the points is within twice its value at the true pose plus 1e-3."""
    from nphm_b200.evaluation.render_utils import render_sdf_views, samples_from_images
    from test_gpu_sdf_trace import H, SCALE, W, _cams
    dec = RC.fitted_head(cuda_device)
    z = torch.zeros(1, dec.lat_dim, device=cuda_device)
    cams, views, K = _cams(1)
    depth, normals = render_sdf_views(dec, z, views, K, (H, W), scale=SCALE)
    pts, _ = samples_from_images(depth[0], normals[0], cams, views, SCALE, K=K, rend_size=(H, W))
    R, t, ls = similarity(150.0, (0.4, 1.0, -0.3), (0.2, -0.1, 0.25), 1.0)
    scan = RC.to_scan(pts.double().cpu(), R, t, ls).float().to(cuda_device)
    state = torch.cuda.get_rng_state()
    poses, stats = G.register_scans(dec, [[scan]], return_stats=True)
    assert torch.equal(torch.cuda.get_rng_state(), state)
    rms_true = _rms_sdf(dec, z, pts.double())
    rms_reg = _rms_sdf(dec, z, poses[0].to_model(scan.double(), 0))
    e = RC.pose_error(poses[0], 0, R, t, ls)
    s, u = float(stats[0]['score'][0]), float(stats[0]['runner_up'][0])
    print('single view (%d points): rms sdf at the true pose %.3g, after registration %.3g; pose error %.3g deg, %.3g units, '
          '%.3g scale; score %.3g, runner-up %.3g, inliers %.3f'
          % (len(pts), rms_true, rms_reg, *e, s, u, float(stats[0]['inlier_fraction'][0])))
    assert rms_reg <= 2 * rms_true + 1e-3
    assert 0 < s <= u
