"""Observation poses on the GPU (csrc/pose.cu, DESIGN.md §4.24): the three kernels against their float64 statements, frozen
poses leaving the native fitters' results unchanged, batched against single-scan posed fits, sync-free posed steps, and the
recovery of a known similarity from surface points of a seeded head."""
import math

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, load_golden, make_deformation, make_ensemble, make_npm
from pose_common import (clamp_in_a_gap, identity_pose_gradient, joint_pose_gradient, random_poses, random_rotation,
                         random_rows, similarity)
from nphm_b200.models import fitting as F
from nphm_b200.models.pose import ObservationPoses, adam_f64, apply_f64, grad_f64

pytestmark = pytest.mark.gpu

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
ID_LAMBDAS = {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
SCHEDULE = {'lr': {200: 2, 400: 2}, 'symm_dist': {200: 10}, 'reg_glob': {200: 3}, 'reg_loc': {200: 3}, 'reg_expr': {200: 10}}


def _scans(sizes, seed, device):
    rng = np.random.RandomState(seed)
    return [torch.from_numpy((rng.randn(n, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32)).to(device)
            for n in sizes]


# ------------------------------------------------------------------------------------------------------------ kernels
def test_apply_is_the_float64_transform_rounded_once(cuda_device):
    poses = random_poses(4, seed=1, device=cuda_device)
    pts, rows, _ = random_rows(12, 777, 4, seed=2)
    rows[3], rows[7] = -1, 4                                   # padding and an index past the table: passed through
    pts, rows = pts.to(cuda_device), rows.to(cuda_device)
    q = poses.apply(pts, rows)
    assert torch.equal(q, apply_f64(poses.table, pts, rows))  # the same float64 operations, exp on the same device
    assert torch.equal(q[3], pts[3]) and torch.equal(q[7], pts[7])
    assert torch.equal(ObservationPoses(4, cuda_device).apply(pts, rows), pts)
    assert torch.equal(poses.apply(pts, rows), q)


def test_grad_is_the_float64_sum_and_repeatable(cuda_device):
    poses = random_poses(5, seed=3, device=cuda_device)
    pts, rows, g = random_rows(40, 1000, 5, seed=4)
    rows[5], rows[9] = -1, 5
    rows[rows == 2] = 3                                        # observation 2 has no rows: gradient 0
    q = poses.apply(pts.to(cuda_device), rows.to(cuda_device))
    poses.gradient(q, g.to(cuda_device), rows.to(cuda_device), 1.7)
    got = poses.grad.clone()
    want = grad_f64(poses.table.cpu(), q.cpu(), g, rows, 1.7)
    assert torch.equal(got[2].cpu(), torch.zeros(7, dtype=torch.float64))
    assert ((got.cpu() - want).abs() <= 1e-12 * want.abs().clamp_min(1e-9)).all(), (got.cpu() - want).abs().max()
    for _ in range(3):
        poses.gradient(q, g.to(cuda_device), rows.to(cuda_device), 1.7)
        assert torch.equal(poses.grad, got)


def test_adam_is_the_float64_mirror(cuda_device):
    for fit_scale in (True, False):
        poses = random_poses(6, seed=5, device=cuda_device, fit_scale=fit_scale, lr=(3e-3, 2e-3, 1e-3))
        table, m, v = poses.table.cpu(), poses.m.cpu(), poses.v.cpu()
        gen = torch.Generator().manual_seed(6)
        for step in range(1, 21):
            grad = torch.randn(6, 7, generator=gen, dtype=torch.float64)
            poses.grad.copy_(grad)
            poses.update(0.5, step)
            adam_f64(table, m, v, grad, poses.rates(0.5), fit_scale, step)
        assert (poses.table.cpu() - table).abs().max() < 1e-12
        assert (poses.m.cpu() - m).abs().max() < 1e-12 and (poses.v.cpu() - v).abs().max() < 1e-12


# ------------------------------------------------------------------------------------------------------------ frozen poses
def _frozen_pair(fit, n_obs, device, lambdas=LAMBDAS, repeat=False):
    """``fit`` without poses (twice with ``repeat``) and with a frozen identity pose: (result, generator state, lambdas)."""
    out = []
    for poses in ([None] * (1 + repeat)) + [ObservationPoses(n_obs, device, lr=(0.0, 0.0, 0.0))]:
        torch.manual_seed(5)
        lam = dict(lambdas)
        out.append((fit(lam, poses), torch.get_rng_state(), lam))
    return out


def _tensors(res):
    if isinstance(res, torch.Tensor):
        return [res]
    if isinstance(res, (tuple, list)):
        return [t for r in res for t in _tensors(r)]
    return []


def _max_diff(ra, rb):
    return max(float((x.detach() - y.detach()).abs().max()) for x, y in zip(_tensors(ra), _tensors(rb)))


def _assert_bitwise(runs, what):
    """A frozen pose gives the plain fit's result bit for bit wherever the plain fit repeats itself bit for bit."""
    (ra, ga, la), (rr, _, _), (rb, gb, lb) = runs
    assert torch.equal(ga, gb) and la == lb
    repeat, frozen = _max_diff(ra, rr), _max_diff(ra, rb)
    print('frozen pose, %s: plain vs plain %.3g, plain vs frozen %.3g' % (what, repeat, frozen))
    if repeat == 0.0:
        assert frozen == 0.0
    assert frozen <= 4 * repeat + 1e-6


def _npm_pair(device):
    from npm_fit_common import make_decoders
    from nphm_b200.models.deepSDF import DeepSDF
    return make_decoders(DeepSDF, device)


def test_frozen_pose_joint_and_expression_fits_are_bitwise_unchanged(cuda_device):
    dec, dfn = make_ensemble(0, device=cuda_device).train(), make_deformation(cuda_device)
    npm, npm_expr = _npm_pair(cuda_device)
    obs = _scans((1100, 1300, 1050), seed=7, device=cuda_device)
    for name, d, e in (('ensemble', dec, dfn), ('npm', npm, npm_expr)):
        _assert_bitwise(_frozen_pair(lambda l, p: F.inference_iterative_root_finding_joint(d, e, obs, l, 500, SCHEDULE, 0.01,
                                                                                           poses=p), 3, cuda_device, repeat=True),
                        name + ' joint')
        z_id = torch.randn(1, 1, d.lat_dim, generator=torch.Generator().manual_seed(1)).to(cuda_device) * 0.01
        _assert_bitwise(_frozen_pair(lambda l, p: F.inference_expression_space(d, e, z_id, obs, l, 500, SCHEDULE, 0.01,
                                                                               poses=p), 3, cuda_device, repeat=True),
                        name + ' expression')
        subjects = [obs, obs[:2]]

        def batched(l, p):
            return F.inference_iterative_root_finding_joint_batched(
                d, e, subjects, l, 500, SCHEDULE, 0.01,
                poses=None if p is None else [ObservationPoses(len(s), cuda_device, lr=(0.0, 0.0, 0.0)) for s in subjects])
        _assert_bitwise(_frozen_pair(batched, 3, cuda_device, repeat=True), name + ' batched joint')


def test_frozen_pose_identity_fits_stay_within_the_fit_bounds(cuda_device):
    """The ensemble switches from the fused step to surface_grad + apply_gradient, NPM to want_xyz: the same math."""
    obs = _scans((1100, 1300, 1050), seed=8, device=cuda_device)
    for dec in (make_ensemble(0, device=cuda_device).train(), make_ensemble(0, device=cuda_device).eval(),
                make_npm(cuda_device)):
        (ra, ga, la), (rb, gb, lb) = _frozen_pair(
            lambda l, p: F.inference_identity_space(dec, obs, l, 800, SCHEDULE, 0.01, poses=p), 3, cuda_device, ID_LAMBDAS)
        assert torch.equal(ga, gb) and la == lb
        dz = (ra[0] - rb[0]).detach().abs()
        close = float((dz < 5e-4).double().mean())
        print('frozen identity route switch (%s, %s): max |dz| %.3g, %.4f of the code within 5e-4'
              % (type(dec).__name__, 'train' if dec.training else 'eval', float(dz.max()), close))
        assert close > 0.99 and float(dz.max()) < 5e-3


# ------------------------------------------------------------------------------------------------------------ batched
@pytest.mark.parametrize('kind', ['identity', 'joint', 'expression'])
@pytest.mark.parametrize('decoder', ['nphm', 'npm'])
def test_batched_posed_fits_equal_single_scan_posed_fits(decoder, kind, cuda_device):
    if decoder == 'nphm':
        dec, dfn = make_ensemble(0, device=cuda_device).train(), make_deformation(cuda_device)
    else:
        dec, dfn = _npm_pair(cuda_device)
    # the second scan's observations have fewer points than a sampled row, so the batched fitters pad
    scans = [_scans((1100, 1300), seed=9, device=cuda_device), _scans((900, 900, 900), seed=10, device=cuda_device)]
    z_ids = [torch.randn(1, 1, dec.lat_dim, generator=torch.Generator().manual_seed(30 + k)).to(cuda_device) * 0.01
             for k in range(2)]

    def fit_batched(lam, poses):
        if kind == 'identity':
            return F.inference_identity_space_batched(dec, scans, lam, 500, SCHEDULE, 0.01, poses=poses)
        if kind == 'joint':
            return F.inference_iterative_root_finding_joint_batched(dec, dfn, scans, lam, 500, SCHEDULE, 0.01, poses=poses)
        return F.inference_expression_space_batched(dec, dfn, list(zip(z_ids, scans)), lam, 500, SCHEDULE, 0.01, poses=poses)

    def fit_single(k, lam, poses):
        if kind == 'identity':
            return F.inference_identity_space(dec, scans[k], lam, 500, SCHEDULE, 0.01, poses=poses)
        if kind == 'joint':
            return F.inference_iterative_root_finding_joint(dec, dfn, scans[k], lam, 500, SCHEDULE, 0.01, poses=poses)
        return F.inference_expression_space(dec, dfn, z_ids[k], scans[k], lam, 500, SCHEDULE, 0.01, poses=poses)

    base = ID_LAMBDAS if kind == 'identity' else LAMBDAS
    batched = [random_poses(len(s), seed=20 + k, device=cuda_device) for k, s in enumerate(scans)]
    torch.manual_seed(3)
    out_b = fit_batched(dict(base), batched)
    torch.manual_seed(3)
    single = [random_poses(len(s), seed=20 + k, device=cuda_device) for k, s in enumerate(scans)]
    out_s = [fit_single(k, dict(base), single[k]) for k in range(len(scans))]
    for pb, ps, rb, rs in zip(batched, single, out_b, out_s):
        assert not torch.equal(pb.table, random_poses(pb.n, seed=0, device=cuda_device).table)
        dt = float((pb.table - ps.table).abs().max())
        dz = torch.cat([(a - b).detach().abs().reshape(-1) for a, b in zip(_tensors(rb), _tensors(rs))])
        close = float((dz < 5e-4).double().mean())
        print('batched vs single posed %s %s: max |d table| %.3g, max |d code| %.3g, %.4f within 5e-4'
              % (decoder, kind, dt, float(dz.max()), close))
        # test_gpu_fit_batched.py's bound on whole fits: the share of code entries within 5e-4
        assert dt < 1e-4 and close > 0.95, (dt, close)


# ------------------------------------------------------------------------------------------------------------ no host sync
@pytest.mark.parametrize('decoder', ['nphm', 'npm'])
def test_posed_steps_do_not_synchronise_with_the_host(decoder, cuda_device):
    """Single and batched posed identity and joint steps (one scan of the batch padded) enqueue without a host sync."""
    if decoder == 'nphm':
        dec, dfn = make_ensemble(0, device=cuda_device).train(), make_deformation(cuda_device)
        classes = (F.IdentityFitter, F.JointFitter, F.BatchedIdentityFitter, F.BatchedJointFitter)
    else:
        dec, dfn = _npm_pair(cuda_device)
        classes = (F.NpmIdentityFitter, F.NpmJointFitter, F.BatchedNpmIdentityFitter, F.BatchedNpmJointFitter)
    scans = [_scans((1100, 1300, 1050), seed=11, device=cuda_device), _scans((900, 900, 900), seed=12, device=cuda_device)]
    single_poses = random_poses(3, seed=12, device=cuda_device)
    shared = ObservationPoses.concat([random_poses(3, seed=13 + k, device=cuda_device) for k in range(2)])
    torch.manual_seed(0)
    sample = [F._sample_observations(s) for s in scans]
    obs = [o for o, _ in sample]
    idx = [i.to(cuda_device) for _, i in sample]
    rows = torch.cat([i + 3 * k for k, i in enumerate(idx)]).to(torch.int32)
    lam_id = dict(ID_LAMBDAS)
    fit_id, fit_j = classes[0](dec, cuda_device, single_poses), classes[1](dec, dfn, 3, cuda_device, poses=single_poses)
    fit_bid, fit_bj = classes[2](dec, 2, cuda_device, shared), classes[3](dec, dfn, [3, 3], cuda_device, poses=shared)
    steps = [lambda: fit_id.step(obs[0], lam_id, 0.1, 0.01, obs_idx=idx[0].to(torch.int32)),
             lambda: fit_j.step(obs[0], idx[0], dict(LAMBDAS), 0.1, 0.01),
             lambda: fit_bid.step(obs, lam_id, 0.1, 0.01, obs_idx=rows),
             lambda: fit_bj.step(obs, idx, dict(LAMBDAS), 0.1, 0.01)]
    for step in steps:                                      # warm-up: workspaces, engines
        step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for step in steps:
            step()
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert torch.isfinite(single_poses.table).all() and torch.isfinite(shared.table).all()


# ------------------------------------------------------------------------------------------------------------ recovery
def _surface_points(dec, device, n_obs, n_points, seed):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband
    z = torch.zeros(1, 1, dec.lat_dim, device=device)
    mesh = extract_mesh_narrowband(dec, z, MINI, MAXI, 128)
    v = torch.from_numpy(np.asarray(mesh.vertices, dtype=np.float64))
    g = torch.Generator().manual_seed(seed)
    return [v[torch.randint(0, v.shape[0], (n_points,), generator=g)] for _ in range(n_obs)]


def _rms_sdf(dec, z, pts_model):
    with torch.no_grad():
        sdf = dec.engine().query(pts_model.reshape(1, -1, 3).float(), z.reshape(1, -1), eval_quirk=False)[0]
    return float(sdf.double().square().mean().sqrt())


def test_recovers_a_known_similarity(cuda_device):
    dec = make_ensemble(0, device=cuda_device).train()
    model_pts = _surface_points(dec, cuda_device, 3, 4000, seed=13)
    R_a, t_a, ls_a = similarity(8.0, (0.3, 1.0, 0.2), (0.03, -0.02, 0.04), 1.04)
    scan = [(math.exp(ls_a) * p @ R_a.T + t_a).float().to(cuda_device) for p in model_pts]
    results = {}
    for posed in (False, True):
        poses = ObservationPoses(3, cuda_device) if posed else None
        torch.manual_seed(14)
        z, _ = F.inference_identity_space(dec, scan, dict(ID_LAMBDAS), 600, SCHEDULE, 1, poses=poses)
        to_model = (lambda p, o: poses.to_model(p.double(), o)) if posed else (lambda p, o: p.double())
        rms = _rms_sdf(dec, z, torch.cat([to_model(s, o) for o, s in enumerate(scan)]))
        results[posed] = rms
        if posed:
            M = poses.matrices().cpu()
            A = torch.eye(4, dtype=torch.float64)
            A[:3, :3], A[:3, 3] = math.exp(ls_a) * R_a, t_a
            E = M @ A                                         # ~ identity when the pose inverts the applied similarity
            s = E[:, :3, :3].det().abs() ** (1 / 3)
            Rn = E[:, :3, :3] / s[:, None, None]
            ang = torch.rad2deg(torch.arccos(((Rn.diagonal(dim1=1, dim2=2).sum(-1) - 1) / 2).clamp(-1, 1)))
            results['angle'], results['trans'] = float(ang.max()), float(E[:, :3, 3].norm(dim=-1).max())
            results['scale'] = float((s - 1).abs().max())
    print('recovery: rms sdf posed %.3g, unposed %.3g; pose error %.3g deg, %.3g trans, %.3g scale'
          % (results[True], results[False], results['angle'], results['trans'], results['scale']))
    # H100 run: rms 1.1e-4 posed against 0.022 unposed; 0.02 degrees, 1.8e-4 translation and 2e-4 scale from the inverse
    assert results[True] < 0.05 * results[False]
    assert results['angle'] < 0.5 and results['trans'] < 5e-3 and results['scale'] < 5e-3


# ------------------------------------------------------------------------------- pose gradients at fixed correspondences
OBS_IDX = [2, 0, 2, 3, 0]                 # 4 observations: 0 and 2 sampled twice, 1 never (its gradient must be exactly 0)
K_F32 = {'nphm': (64.0, 2e-5), 'npm': (64.0, 1e-4)}      # as tests/test_gpu_joint_f64.py: K x the fp32 error, or a floor


@pytest.fixture
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _case(decoder, device):
    """Decoders, their float64 / float32 parameters (joint_f64_common), golden-near codes and sampled rows, a small pose."""
    import joint_f64_common as J
    if decoder == 'nphm':
        dec, expr = make_ensemble(0, device=device).train(), make_deformation(device)
        Q64, Q32 = J.NphmParams(dec, expr, torch.float64), J.NphmParams(dec, expr, torch.float32)
        g, key = load_golden('fit_joint.npz'), 'z_id_before'
    else:
        dec, expr = _npm_pair(device)
        Q64, Q32 = J.NpmParams(dec, expr, torch.float64), J.NpmParams(dec, expr, torch.float32)
        g, key = load_golden('fit_npm.npz'), 'joint_z_id_before'
    z_id = torch.from_numpy(g[key][2]).float().to(device)
    z_ex = torch.from_numpy(g[key.replace('id', 'ex')][2]).float()
    z_ex = torch.cat([z_ex, z_ex[:1]]).to(device)
    obs = torch.from_numpy(g['obs'])
    gen = torch.Generator().manual_seed(3)
    scans = [obs[k][torch.randint(0, obs.shape[1], (1000,), generator=gen)] + 0.002 * torch.randn(1000, 3, generator=gen)
             for k in (0, 1, 2, 0)]
    rows = torch.tensor(OBS_IDX, device=device)
    sample = torch.stack([scans[i] for i in OBS_IDX]).to(device)
    rng = np.random.RandomState(4)
    poses = ObservationPoses(4, device, R=torch.stack([random_rotation(rng, 0.03) for _ in range(4)]).to(device),
                             t=torch.from_numpy(rng.randn(4, 3) * 0.003).to(device),
                             log_scale=torch.from_numpy(rng.randn(4) * 0.005).to(device))
    return dec, expr, Q64, Q32, z_id, z_ex, sample, rows, poses


def _check_pose_grad(what, got, g64, g32, decoder):
    k, floor = K_F32[decoder]
    got = got.cpu()
    assert torch.equal(got[1], torch.zeros(7, dtype=torch.float64)), (what, 'unsampled observation')
    for o in (0, 2, 3):
        for part, sl in (('omega', slice(0, 3)), ('t', slice(3, 6)), ('sigma', slice(6, 7))):
            ref = float(g64[o, sl].norm())
            err = float((got[o, sl] - g64[o, sl].cpu()).norm()) / ref
            err32 = float((g32[o, sl].cpu() - g64[o, sl].cpu()).norm()) / ref
            print('POSE GRAD %-22s obs %d %-5s |g| %.3e  native %.2e  fp32 autograd %.2e' % (what, o, part, ref, err, err32))
            assert err <= max(k * err32, floor), (what, o, part, err, err32)


@pytest.mark.parametrize('kind', ['identity', 'joint'])
@pytest.mark.parametrize('decoder', ['nphm', 'npm'])
def test_pose_gradient_at_fixed_correspondences_matches_float64(decoder, kind, cuda_device, _no_tf32):
    """One ``apply_update=False`` step's ``poses.grad`` against float64 autograd of the composite formulation at the same
    sampled points (and, for the joint fitters, the same Broyden roots): the sign and scale of g_q = -u and of every route."""
    dec, expr, Q64, Q32, z_id, z_ex, obs, rows, poses = _case(decoder, cuda_device)
    lam = dict(LAMBDAS)
    lam_s = lam['surface']
    if kind == 'identity':
        fitter = (F.IdentityFitter(dec, cuda_device, poses) if decoder == 'nphm'
                  else F.NpmIdentityFitter(dec, cuda_device, poses))
        fitter.latent.copy_(z_id)
        import joint_f64_common as J
        with torch.no_grad():
            q64 = poses.apply(obs, rows).double()
            clamp = clamp_in_a_gap(J.identity_sdf(Q64, q64, z_id.double()).abs())
        fitter.step(obs, {k: v for k, v in lam.items() if k != 'reg_expr'}, clamp, 0.01, apply_update=False,
                    obs_idx=rows.to(torch.int32))
        g64, n64 = identity_pose_gradient(Q64, obs, rows, poses.table, z_id, lam_s, clamp)
        g32, n32 = identity_pose_gradient(Q32, obs, rows, poses.table, z_id, lam_s, clamp)
    else:
        cls = F.JointFitter if decoder == 'nphm' else F.NpmJointFitter
        fitter = cls(dec, expr, 4, cuda_device, poses=poses)
        fitter.z_id.copy_(z_id)
        fitter.z_ex.copy_(z_ex)
        roots, search = [], fitter.mlp.broyden_search

        def capture(*a, **k):
            out = search(*a, **k)
            roots.append((out[0].clone(), out[2].clone()))
            return out
        fitter.mlp.broyden_search = capture
        try:
            fitter.step(obs, rows, lam, 0.1, 0.01, apply_update=False)
            p, valid = roots[-1]
            import joint_f64_common as J
            a = J.sdf_at_roots(Q64, p, z_id).abs()
            clamp = clamp_in_a_gap(a[valid.reshape(-1)])
            fitter.step(obs, rows, lam, clamp, 0.01, apply_update=False)
            assert torch.equal(roots[-1][0], p) and torch.equal(roots[-1][1], valid)
        finally:
            del fitter.mlp.broyden_search
        g64, n64 = joint_pose_gradient(Q64, obs, rows, poses.table, p, valid, z_id, z_ex, rows, lam_s, clamp)
        g32, n32 = joint_pose_gradient(Q32, obs, rows, poses.table, p, valid, z_id, z_ex, rows, lam_s, clamp)
    assert n64 == n32 > 0
    _check_pose_grad('%s %s' % (decoder, kind), poses.grad, g64, g32, decoder)


# ------------------------------------------------------------------------------- recovery per observation: posed expressions
def test_recovers_per_observation_similarities_of_posed_expressions(cuda_device):
    """Surface points of two posed expressions (zero identity and expression codes, the fitters' start), each observation
    moved by its own similarity; ``inference_expression_space`` with poses brings them onto the posed surfaces."""
    from nphm_b200.utils.reconstruction import extract_posed_meshes_narrowband
    dec, dfn = make_ensemble(0, device=cuda_device).train(), make_deformation(cuda_device)
    z_id = torch.zeros(1, 1, dec.lat_dim, device=cuda_device)
    meshes = extract_posed_meshes_narrowband(dec, dfn, z_id, torch.zeros(2, dfn.lat_dim_expr, device=cuda_device), MINI, MAXI,
                                             128)
    gen = torch.Generator().manual_seed(15)
    surf = [torch.from_numpy(np.asarray(m.vertices, dtype=np.float64)).to(cuda_device) for m in meshes]
    model_pts = [v[torch.randint(0, v.shape[0], (4000,), generator=gen).to(cuda_device)] for v in surf]
    moves = [similarity(8.0, (0.3, 1.0, 0.2), (0.03, -0.02, 0.04), 1.04),
             similarity(6.0, (-1.0, 0.4, 0.5), (-0.04, 0.01, 0.02), 0.97)]
    scan = [(math.exp(ls) * p @ R.to(cuda_device).T + t.to(cuda_device)).float() for p, (R, t, ls) in zip(model_pts, moves)]

    def rms_to_surface(points):
        return float(torch.cat([torch.cdist(pt.double(), v).min(1).values for pt, v in zip(points, surf)]).square().mean().sqrt())

    poses = ObservationPoses(2, cuda_device)
    torch.manual_seed(16)
    F.inference_expression_space(dec, dfn, z_id, scan, dict(LAMBDAS), 600, SCHEDULE, 1, poses=poses)
    posed = rms_to_surface([poses.to_model(s.double(), o) for o, s in enumerate(scan)])
    unposed = rms_to_surface(scan)
    M = poses.matrices().cpu()
    errs = []
    for o, (R, t, ls) in enumerate(moves):
        A = torch.eye(4, dtype=torch.float64)
        A[:3, :3], A[:3, 3] = math.exp(ls) * R, t
        E = M[o] @ A
        s = E[:3, :3].det().abs() ** (1 / 3)
        ang = math.degrees(math.acos(max(-1.0, min(1.0, (float((E[:3, :3] / s).trace()) - 1) / 2))))
        errs.append((ang, float(E[:3, 3].norm()), abs(float(s) - 1)))
    print('expression recovery: rms to the posed surfaces %.3g posed, %.3g unposed; per observation (deg, trans, scale) %s'
          % (posed, unposed, ['(%.3g, %.3g, %.3g)' % e for e in errs]))
    assert posed < 0.1 * unposed
    for ang, tr, sc in errs:
        assert ang < 1.0 and tr < 1e-2 and sc < 1e-2


# ------------------------------------------------------------------------------- devices and inputs
def test_index_less_cuda_device_and_host_inputs_are_accepted(cuda_device):
    poses = ObservationPoses(2, 'cuda', R=torch.eye(3, dtype=torch.float64, device='cuda').repeat(2, 1, 1))
    assert poses.device == cuda_device
    pts, rows, g = random_rows(3, 50, 2, seed=17)
    q = poses.apply(pts, rows)                                 # host tensors are copied to the device
    assert q.device == cuda_device and torch.equal(q.cpu(), pts)
    poses.gradient(q, g, rows, 1.0)
    assert torch.isfinite(poses.grad).all()
    with pytest.raises(ValueError):
        poses.apply(pts.reshape(-1, 3), rows)
    dec = make_npm(cuda_device)
    obs = _scans((1100, 1200), seed=18, device=cuda_device)
    F.inference_identity_space(dec, obs, dict(ID_LAMBDAS), 200, SCHEDULE, 0.01, poses=ObservationPoses(2, 'cuda'))
