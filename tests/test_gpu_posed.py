"""GPU tests of the posed queries: the compacting Broyden search (nphm_mlp_broyden_search_compact) against the dense one, the
native get_logits_posed against the reference (tests/golden/posed.npz) and the composite path, and the posed narrow band
against the dense posed mesh."""
import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_deformation, make_ensemble, sample_latent
from posed_common import check_against_golden, ensemble_case, npm_case
import npm_fit_common as C
from nphm_b200.models import reconstruction as R
from nphm_b200.utils.reconstruction import (create_grid_points_from_bounds, default_margin, extract_posed_meshes_narrowband,
                                            mesh_from_logits)

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------ compacting search
def _search_net(kind, dev):
    """(MlpEngine, condition width, spread of the points) of the three network dispatches: the tc backbone, the FFMA kernel, the
    layer chain; output layers scaled so that the searches take several steps and (tc, FFMA) some samples fail."""
    from nphm_b200.models.deepSDF import DeepSDF
    if kind == 'tc':
        dfn = make_deformation(dev)
        with torch.no_grad():                       # large deformations: some samples need many steps, some diverge
            dfn.defDeepSDF.lin6.weight.mul_(80.0)
            dfn.defDeepSDF.lin6.bias.mul_(80.0)
        return dfn.defDeepSDF.engine(), 232, 0.2
    if kind == 'ffma':
        torch.manual_seed(31)
        net = DeepSDF(lat_dim=37, hidden_dim=75, nlayers=4, out_dim=3).to(dev)
        with torch.no_grad():
            net.lin4.weight.mul_(3.5)
        return net.engine(), 37, 0.5
    _, expr = C.make_decoders(DeepSDF, dev)
    with torch.no_grad():
        expr.lin8.weight.mul_(400.0)
        expr.lin8.bias.mul_(400.0)
    return expr.engine(), 712, 0.3


def _assert_same_search(eng, obs, cond, x0, j0, **kw):
    a = eng.broyden_search(obs, cond, x0, j0, compact=False, **kw)
    b = eng.broyden_search(obs, cond, x0, j0, compact=True, **kw)
    for u, v in zip(a[:3], b[:3]):
        assert u.shape == v.shape and torch.equal(u, v)
    assert a[3] == b[3]
    return a


@pytest.mark.parametrize('kind', ['tc', 'ffma', 'chain'])
@pytest.mark.parametrize('S', [1, 3])
def test_compact_search_equals_dense_bitwise(cuda_device, kind, S):
    eng, cw, spread = _search_net(kind, cuda_device)
    if kind == 'tc':
        assert eng.fused_shape
    elif kind == 'ffma':
        assert eng.simt_ok and not eng.fused_shape
    else:
        assert not eng.simt_ok
    torch.manual_seed(5)
    cond = torch.randn(S, cw, device=cuda_device) * 0.1
    n = 1000 + 77                                    # not a multiple of 128
    obs = (torch.randn(S, n, 3, device=cuda_device) * spread).contiguous()
    _, j0 = eng.inverse_jacobian(obs, cond)
    converged, failed = 0, 0
    for early_exit in (True, False):
        x, diff, valid, steps = _assert_same_search(eng, obs, cond, obs, j0, early_exit=early_exit)
        converged, failed = int(valid.sum()), int((~valid).sum())
    assert converged > 0 and (failed > 0 or kind == 'chain')      # both exit paths of the loop are taken
    # max_steps = 0; every sample converged at the start; no samples
    _assert_same_search(eng, obs, cond, obs, j0, max_steps=0)
    x_root = x.clone()
    exact = x_root + eng.query(x_root, cond)
    _, j1 = eng.inverse_jacobian(x_root, cond)
    _, _, ok, _ = _assert_same_search(eng, exact, cond, x_root, j1)
    assert ok.all()
    empty = torch.zeros(S, 0, 3, device=cuda_device)
    _assert_same_search(eng, empty, cond, empty, torch.zeros(S, 0, 3, 3, device=cuda_device))


# ------------------------------------------------------------------------------------------ posed logits
@pytest.mark.parametrize('training', [True, False])
def test_native_posed_logits_match_reference(cuda_device, training):
    dec, dfn, lat, z_ex, grid, g = ensemble_case(cuda_device, training)
    assert R.posed_evaluator(dec, dfn, lat, z_ex) is not None
    sdf, valid = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=int(g['nbatch_points']), return_valid=True)
    check_against_golden(sdf, valid, g['sdf_train'] if training else g['sdf_eval'], g['valid'])


def test_native_posed_logits_npm_match_reference(cuda_device):
    dec, expr, lat, z_ex, pts, g = npm_case(cuda_device)
    assert R.posed_evaluator(dec, expr, lat, z_ex) is not None
    sdf, valid = R.get_logits_posed(dec, expr, lat, z_ex, pts, nbatch_points=1000, return_valid=True)
    check_against_golden(sdf, valid, g['npm_sdf'], g['npm_valid'])


def _composite(fn, *args, **kw):
    saved = R.posed_evaluator
    R.posed_evaluator = lambda *a, **k: None
    try:
        return fn(*args, **kw)
    finally:
        R.posed_evaluator = saved


def test_native_posed_logits_match_composite_on_larger_grid(cuda_device):
    """On the seeded (unscaled) deformation network: with the x 80 field of posed.npz, 3 % of this grid's rows end their search
    within the rounding of J0 (autograd against the native forward-mode pass) of the 1e-6 threshold and flip their valid flag."""
    dec, _, lat, z_ex, _, _ = ensemble_case(cuda_device, training=False)
    dfn = make_deformation(cuda_device)
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, 30)).to(cuda_device, torch.float32)[None]
    a, va = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=9000, return_valid=True)
    b, vb = _composite(R.get_logits_posed, dec, dfn, lat, z_ex, grid, nbatch_points=9000, return_valid=True)
    check_against_golden(a, va, b, vb)


def test_posed_logits_batch_and_piece_invariance(cuda_device, monkeypatch):
    """An S-expression call equals S one-expression calls, and no result depends on the piece size, bitwise."""
    dec, dfn, lat, z_ex, grid, g = ensemble_case(cuda_device, training=False)
    z3 = torch.cat([z_ex, z_ex[:1] * -1.5])
    nb = int(g['nbatch_points'])
    full, vfull = R.get_logits_posed(dec, dfn, lat, z3, grid, nbatch_points=nb, return_valid=True)
    for s in range(3):
        one, vone = R.get_logits_posed(dec, dfn, lat, z3[s], grid, nbatch_points=nb, return_valid=True)
        assert np.array_equal(one, full[s]) and np.array_equal(vone, vfull[s])
    for piece in (1000, 777 * 3, 128):
        monkeypatch.setattr(R, 'POSED_PIECE_ROWS', piece)
        other, vother = R.get_logits_posed(dec, dfn, lat, z3, grid, nbatch_points=nb, return_valid=True)
        assert np.array_equal(other, full) and np.array_equal(vother, vfull)


def test_posed_logits_of_a_translation(cuda_device):
    """F == t (zero output weight, bias t): the posed SDF is the canonical SDF at x - t, and every row converges."""
    dec = make_ensemble(0, device=cuda_device).eval()
    dfn = make_deformation(cuda_device)
    t = torch.tensor([0.03, -0.02, 0.05], device=cuda_device)
    with torch.no_grad():
        dfn.defDeepSDF.lin6.weight.zero_()
        dfn.defDeepSDF.lin6.bias.copy_(t)
    lat = sample_latent(1).to(cuda_device)
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, 20)).to(cuda_device, torch.float32)[None]
    z_ex = torch.randn(2, 200, device=cuda_device) * 0.1
    sdf, valid = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=3000, return_valid=True)
    canon = R.get_logits(dec, lat, grid - t, nbatch_points=3000)
    assert valid.all()
    assert np.abs(sdf - canon[None]).max() < 1e-5


# ------------------------------------------------------------------------------------------ posed meshes
def _margin_for(dec, dfn, lat, z_ex, res, nbatch, lo, hi):
    """The default margin, or more when the posed field's gradient bound measured on the dense grid exceeds 2 (the default
    margin's assumption): max |grad sdf| (finite differences of the canonical grid, times sqrt 3 for the diagonal) times
    max ||(I + dF/dx)^-1|| at the roots."""
    grid = torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(lat.device, torch.float32)[None]
    if hasattr(dfn, 'defDeepSDF'):
        canon = R.get_logits(dec, lat, grid, nbatch_points=nbatch)
    else:
        with torch.no_grad():
            canon = dec(grid, lat.reshape(1, 1, -1).expand(1, grid.shape[1], -1))[0].cpu().numpy()
    canon = canon.reshape(res, res, res)
    h = (np.asarray(hi) - np.asarray(lo)) / (res - 1)
    g_sdf = max(float(np.abs(np.diff(canon, axis=a)).max() / h[a]) for a in range(3)) * np.sqrt(3)
    fn = R.posed_evaluator(dec, dfn, lat, z_ex)
    assert fn is not None
    eng = dfn.defDeepSDF.engine() if hasattr(dfn, 'defDeepSDF') else dfn.engine()
    return default_margin(lo, hi, res) * max(1.0, g_sdf * _max_inverse_norm(eng, dec, dfn, lat, z_ex, grid) / 2.0)


def _max_inverse_norm(eng, dec, dfn, lat, z_ex, grid):
    from nphm_b200.models.iterative_root_finding import _fused_search_condition
    S = z_ex.shape[0]
    if hasattr(dfn, 'defDeepSDF'):
        anchors = dec.engine().anchors(lat.reshape(1, -1))
        cond = _fused_search_condition(dfn, torch.zeros(S, 1, 3, device=lat.device),
                                       torch.cat([lat.reshape(1, -1).expand(S, -1), z_ex], -1)[:, None],
                                       anchors[:, None].expand(S, 1, *anchors.shape[1:]))
    else:
        cond = torch.cat([lat.reshape(1, -1).expand(S, -1), z_ex], -1).contiguous()
    pts = grid.expand(S, -1, 3).contiguous()
    _, j0 = eng.inverse_jacobian(pts, cond)
    xc, _, ok, _ = eng.broyden_search(pts, cond, pts, j0, compact=True)
    _, j = eng.inverse_jacobian(xc, cond)
    return float(torch.linalg.matrix_norm(j[ok], ord=2).max())


def _assert_same_mesh(a, b):
    assert np.array_equal(np.asarray(a.faces), np.asarray(b.faces))
    assert np.array_equal(np.asarray(a.vertices), np.asarray(b.vertices))


@pytest.mark.parametrize('case', ['train-1', 'train-3', 'eval-1', 'eval-3', 'npm-2'])
def test_posed_band_meshes_equal_dense(cuda_device, case):
    mode, S = case.split('-')
    S = int(S)
    res, nbatch = 40, 7000
    if mode == 'npm':
        dec, dfn, lat, z_ex, _, _ = npm_case(cuda_device)
        lo, hi = [-0.35, -0.3, -0.45], [0.35, 0.4, 0.25]
    else:
        dec = make_ensemble(0, device=cuda_device).train(mode == 'train')
        dfn = make_deformation(cuda_device)
        lat = sample_latent(1).to(cuda_device)
        torch.manual_seed(8)
        z_ex = torch.randn(3, 200, device=cuda_device)[:S] * 0.1
        lo, hi = MINI, MAXI
    margin = _margin_for(dec, dfn, lat, z_ex, res, nbatch, lo, hi)
    meshes, stats = extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, lo, hi, res, nbatch_points=nbatch, margin=margin,
                                                    return_stats=True)
    grid = torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(cuda_device, torch.float32)[None]
    dense = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=nbatch)
    assert len(meshes) == S
    for s in range(S):
        ref = mesh_from_logits(dense[s], lo, hi, res)
        assert len(ref.faces) > 0
        _assert_same_mesh(meshes[s], ref)
        assert stats[s]['voxels_evaluated'] <= res ** 3 and stats[s]['margin'] == margin
