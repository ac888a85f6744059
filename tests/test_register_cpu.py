"""Global registration on the CPU (models/registration.py, DESIGN.md §4.25): the hypothesis set, the float64 mirror of the
kernels (prepare, the normal equations, the search), and the public functions' contract on generators and arguments."""
import math

import numpy as np
import pytest
import torch

import register_common as RC
from conftest import MAXI, MINI
from nphm_b200.models import registration as G


def test_rotation_set_is_deterministic_unit_and_covers_so3():
    q = G.rotation_set(G.N_ROTATIONS)
    assert torch.equal(q, G.rotation_set(G.N_ROTATIONS))
    assert float((q.norm(dim=1) - 1).abs().max()) < 1e-12
    rng = np.random.RandomState(0)
    x = torch.from_numpy(rng.randn(20000, 4))
    x = x / x.norm(dim=1, keepdim=True)
    gap = torch.rad2deg(2 * torch.arccos((x @ q.T).abs().max(1).values.clamp(max=1.0)))
    print('rotation set: largest gap %.2f deg, p99 %.2f deg' % (float(gap.max()), float(gap.quantile(0.99))))
    assert float(gap.max()) <= 23.0
    R = G.quaternion_matrices(q[:50])
    assert float((R.transpose(1, 2) @ R - torch.eye(3, dtype=torch.float64)).abs().max()) < 1e-12
    assert float((torch.linalg.det(R) - 1).abs().max()) < 1e-12


def test_prepare_is_exact_on_a_linear_field():
    res, a = 5, (0.5, -0.25, 2.0)                      # spacing 0.25: every value and difference is exact in fp32
    grid = G.Grid(res, (0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
    x = grid.coordinates('cpu')
    vol = (x @ torch.tensor(a, dtype=torch.float64) + 0.125).float()
    field = G.prepare_torch(vol, grid)
    assert torch.equal(field[:, 0], vol)
    assert torch.equal(field[:, 1:], torch.tensor(a, dtype=torch.float32).expand(res ** 3, 3))
    inside, f, n = G.sample_f64(field, grid, torch.tensor([[0.3, 0.6, 0.9], [1.2, 0.5, 0.5]], dtype=torch.float64))
    assert inside.tolist() == [True, False]
    assert abs(float(f[0]) - (0.15 - 0.15 + 1.8 + 0.125)) < 1e-12
    assert float((n[0] - torch.tensor(a, dtype=torch.float64)).abs().max()) < 1e-12


def _fixture(n_hyp=4, n_pts=300, seed=3, res=40):
    grid = G.Grid(res, MINI, MAXI)
    field = G.prepare_torch(RC.volume(RC.ASYMMETRIC, res), grid)
    pts, _ = RC.surface_points(RC.ASYMMETRIC, n_pts, seed=seed)
    rng = np.random.RandomState(seed)
    rows, scans = [], []
    for _ in range(n_hyp):
        R, t, ls = RC.random_similarity(rng, max_trans=0.1, scale_range=(0.8, 1.25))
        scans.append(RC.to_scan(pts, R, t, ls))
        Rp, tp, lp = RC.random_similarity(rng, max_trans=0.02, scale_range=(0.97, 1.03))
        Rw = torch.linalg.matrix_exp(torch.tensor([[0, -.05, .03], [.05, 0, -.02], [-.03, .02, 0]], dtype=torch.float64))
        Rinv = Rw @ R.T                                          # near the inverse rotation
        rows.append(torch.cat([Rinv.reshape(9), -math.exp(-ls) * Rinv @ t + tp, torch.tensor([-ls + lp])]))
    return grid, field, torch.stack(rows), torch.stack(scans)


def test_normal_equations_equal_float64_autograd_at_fixed_weights():
    grid, field, table, p = _fixture()
    unit = torch.tensor([1.1, 0.9, 1.0, 1.3], dtype=torch.float64)
    mask = torch.ones(p.shape[:2], dtype=torch.bool)
    mask[1, -50:] = False
    tau = 0.02
    for fit_scale in (True, False):
        A, b, count = G.normal_equations_f64(field, grid, table, p, mask, unit, tau, fit_scale)
        inside, r0, _, (a0, f0, n0) = G.residuals_f64(field, grid, table, p, unit)
        w = (mask & inside & (r0.abs() < tau)).to(torch.float64)
        assert torch.equal(count, w.sum(1)) and bool((count > 50).all())
        D = 7 if fit_scale else 6
        q0 = a0 + table[:, None, 9:12]

        def residual(xi):
            """r = (f0 + n0 . (q(xi) - q0)) u / s(xi): the sampled field to first order, exact value and slope at 0."""
            R = torch.linalg.matrix_exp(G_cross(xi[:, :3])) @ table[:, :9].reshape(-1, 3, 3)
            sig = table[:, 12] + (xi[:, 6] if D == 7 else 0.0)
            q = torch.exp(sig)[:, None, None] * torch.einsum('hij,hmj->hmi', R, p) + (table[:, 9:12] + xi[:, 3:6])[:, None]
            return (f0 + (n0 * (q - q0)).sum(-1)) * (unit / torch.exp(sig))[:, None]

        xi0 = torch.zeros(table.shape[0], D, dtype=torch.float64)
        Jfull = torch.autograd.functional.jacobian(residual, xi0)            # H x M x H x D
        J = torch.stack([Jfull[h, :, h] for h in range(table.shape[0])])
        r = residual(xi0)
        assert float((r - r0).abs().max()) < 1e-14
        A_ref = torch.einsum('hm,hmi,hmj->hij', w, J, J)
        b_ref = torch.einsum('hm,hmi,hm->hi', w, J, r)
        ea = float(((A - A_ref).abs().amax((1, 2)) / A_ref.abs().amax((1, 2))).max())
        eb = float(((b - b_ref).abs().amax(1) / b_ref.abs().amax(1)).max())
        print('normal equations (D = %d): relative error A %.2e, b %.2e' % (D, ea, eb))
        assert ea < 1e-10 and eb < 1e-10


def G_cross(w):
    z = torch.zeros_like(w[:, 0])
    return torch.stack([torch.stack([z, -w[:, 2], w[:, 1]], -1), torch.stack([w[:, 2], z, -w[:, 0]], -1),
                        torch.stack([-w[:, 1], w[:, 0], z], -1)], -2)


def test_small_search_recovers_known_similarities():
    vol = RC.volume(RC.ASYMMETRIC, 48)
    pts, _ = RC.surface_points(RC.ASYMMETRIC, 2000, seed=1)
    rng = np.random.RandomState(0)
    moves = [RC.random_similarity(rng) for _ in range(3)]
    scan = [RC.to_scan(pts, *m).float() for m in moves]
    poses, stats = G.register_observations(vol, MINI, MAXI, [scan[:2], scan[2:]], n_rotations=256, return_stats=True,
                                           coarse=dict(points=256), fine=dict(points=1000, top_k=4))
    errs = [RC.pose_error(poses[0], 0, *moves[0]), RC.pose_error(poses[0], 1, *moves[1]), RC.pose_error(poses[1], 0, *moves[2])]
    print('CPU search at 48^3, 256 rotations:', ['(%.3g deg, %.3g, %.3g)' % e for e in errs])
    for ang, tr, sc in errs:           # the 48^3 grid's trilinear bias bounds the accuracy here; the GPU tests run 128^3
        assert ang < 0.5 and tr < 3e-3 and sc < 5e-3
    assert all(p.fit_scale for p in poses) and [p.n for p in poses] == [2, 1]
    assert all(bool((s['inlier_fraction'] > 0.99).all()) for s in stats)


def test_known_log_scale_gives_a_rigid_search():
    vol = RC.volume(RC.ASYMMETRIC, 40)
    pts, _ = RC.surface_points(RC.ASYMMETRIC, 800, seed=2)
    R, t, ls = RC.random_similarity(np.random.RandomState(4))
    poses = G.register_observations(vol, MINI, MAXI, [[RC.to_scan(pts, R, t, ls).float()]], log_scale=-ls, n_rotations=256,
                                    coarse=dict(points=200), fine=dict(points=800, top_k=4))
    assert not poses[0].fit_scale
    assert float(poses[0].table[0, 12]) == -ls
    ang, tr, _ = RC.pose_error(poses[0], 0, R, t, ls)
    assert ang < 1.0 and tr < 5e-3


def test_global_generators_are_untouched():
    vol = RC.volume(RC.ASYMMETRIC, 24)
    pts, _ = RC.surface_points(RC.ASYMMETRIC, 300, seed=5)
    torch.manual_seed(123)
    cpu = torch.get_rng_state()
    cuda = torch.cuda.get_rng_state_all() if torch.cuda.is_available() else None
    G.register_observations(vol, MINI, MAXI, [[pts.float()]], n_rotations=16, coarse=dict(points=64, iters=2),
                            fine=dict(points=128, iters=2, top_k=2))
    assert torch.equal(torch.get_rng_state(), cpu)
    if cuda is not None:
        assert all(torch.equal(a, b) for a, b in zip(torch.cuda.get_rng_state_all(), cuda))


def test_bad_arguments_raise_value_error():
    vol = RC.volume(RC.ASYMMETRIC, 16)
    obs = [[torch.zeros(10, 3)]]
    small = dict(n_rotations=4, coarse=dict(points=8, iters=1), fine=dict(points=8, iters=1, top_k=1))
    bad = [
        (vol, [[torch.zeros(0, 3)]], {}),                                    # empty observation
        (vol, [[]], {}),                                                     # empty scan
        (vol, [], {}),                                                       # no scans
        (vol, [[torch.full((5, 3), float('nan'))]], {}),                    # non-finite points
        (vol, [[torch.zeros(5, 2)]], {}),                                    # not (n, 3)
        (vol[:-1], obs, {}),                                                 # not res^3
        (vol.reshape(16, 256), obs, {}),                                     # res^3 values but not a cube
        (torch.zeros(1), obs, {}),                                           # res < 2
        (vol, obs, dict(log_scale=float('inf'))),
        (vol, obs, dict(log_scale=[0.0, 1.0])),                              # one per scan: one scan here
        (vol, obs, dict(log_scale='mm')),
        (vol, obs, dict(log_scale=True)),
        (vol, obs, dict(fine=dict(points=8, iters=1, top_k=0))),
    ]
    for v, scans, kw in bad:
        with pytest.raises(ValueError):
            G.register_observations(v, MINI, MAXI, scans, **dict(small, **kw))
    with pytest.raises(ValueError):
        G.register_observations(vol, MAXI, MINI, obs, **small)              # inverted box
    with pytest.raises(ValueError):
        G.register_observations(vol.abs() + 1.0, MINI, MAXI, obs, **small)  # no surface in the volume
    if torch.cuda.is_available():
        with pytest.raises(ValueError):
            G.register_observations(vol, MINI, MAXI, [[torch.zeros(10, 3, device='cuda')]], **small)   # mixed devices
    else:
        with pytest.raises(ValueError):
            G.register_observations(vol.to('meta'), MINI, MAXI, obs, **small)                      # mixed devices


def test_mirror_chunks_give_the_unchunked_search():
    grid, field, table, p = _fixture()
    scans = [x.float() for x in p]
    points = torch.cat(scans)
    offsets = torch.tensor([0, 300, 600, 900])
    counts = torch.tensor([300, 300, 250, 300], dtype=torch.int32)
    hyp_obs = torch.tensor([0, 1, 2, 3, 1, 2], dtype=torch.int32)
    tab = torch.cat([table, table[1:3]])
    unit = torch.tensor([1.1, 0.9, 1.0, 1.3], dtype=torch.float64)
    args = (field, grid, points, offsets, counts, unit)
    whole, chunked = tab.clone(), tab.clone()
    s0, i0 = G.search_f64(*args, whole, tab[:, 12].clone(), hyp_obs, 512, 4, (0.1, 0.02), 1e-3, True)
    s1, i1 = G.search_f64(*args, chunked, tab[:, 12].clone(), hyp_obs, 512, 4, (0.1, 0.02), 1e-3, True, chunk_points=700)
    assert float((whole - chunked).abs().max()) < 1e-12 and float((s0 - s1).abs().max()) < 1e-15 and torch.equal(i0, i1)


def test_cpu_head_volume_has_no_eval_mode_quirk():
    from conftest import make_ensemble
    dec = make_ensemble(0).eval()
    vol = G.head_volume(dec, None, 12, MINI, MAXI, torch.device('cpu'))
    assert not dec.training
    assert torch.equal(vol, G.head_volume(make_ensemble(0).train(), None, 12, MINI, MAXI, torch.device('cpu')))
