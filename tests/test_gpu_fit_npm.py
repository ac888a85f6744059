"""GPU tests of fitting with the NPM baseline's DeepSDF decoders: the surface-term entry point nphm_mlp_fit_surface_grad against a
float64 autograd reference, the device Broyden search on the 1024-wide expression decoder against the Python-loop mirror, and
the native identity / joint fitters against the reference's own runs (tests/golden/fit_npm.npz)."""
import copy

import numpy as np
import pytest
import torch

import npm_fit_common as C
from conftest import load_golden

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _npm_decoders(dev):
    from nphm_b200.models.deepSDF import DeepSDF
    return C.make_decoders(DeepSDF, dev)


def _odd_decoder(dev):
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(31)
    dec = DeepSDF(lat_dim=37, hidden_dim=75, nlayers=4, geometric_init=True).to(dev)
    with torch.no_grad():                       # zero level set through the points (as npm_fit_common does for the NPM stack)
        s = dec(torch.zeros(1, 1, 3, device=dev), torch.zeros(1, 1, 37, device=dev))[0]
        dec.lin4.bias.sub_(s.reshape(-1))
        dec.lin4.weight.mul_(20.0); dec.lin4.bias.mul_(20.0)
    return dec


def _check_surface_grad(dec, xyz, cond, mask, clamp, xyz_tol=3e-5):
    """nphm_mlp_fit_surface_grad against autograd through a float64 copy of the composite module: the loss to 5e-6 absolute,
    the gradients to 3e-5 of their max abs (``xyz_tol`` for the point gradient).  The comparison uses the native kept set
    (the rows with a nonzero point gradient); where it differs from the float64 one, |s| must be within 1e-5 of the clamp."""
    eng = dec.engine()
    terms, g_cond, g_xyz = eng.fit_surface_grad(xyz, cond, mask, clamp)
    terms, g_cond, g_xyz = terms.cpu().numpy(), g_cond.cpu().numpy(), g_xyz.cpu().numpy()
    B, N, _ = xyz.shape
    kept = np.abs(g_xyz).max(-1) > 0
    assert int(terms[5]) == int(kept.sum()) > 0
    saved, dec._engine = dec._engine, None                 # the native handle does not copy
    try:
        d64 = copy.deepcopy(dec).double()
    finally:
        dec._engine = saved
    x64 = xyz.double().clone().requires_grad_(True)
    c64 = cond.double().clone().requires_grad_(True)
    s = d64._forward_composite(x64, c64[:, None, :].expand(B, N, cond.shape[-1]))[..., 0]
    s_np = s.detach().cpu().numpy()
    m = np.ones((B, N), bool) if mask is None else mask.cpu().numpy().astype(bool)
    kept64 = m & (np.abs(s_np) < clamp)
    s_nat = eng.train_forward(xyz, cond)[0][..., 0].cpu().numpy()
    print('value pass: max |s - s64| %.3g, sign differences %d, kept %d / %d'
          % (np.abs(s_nat - s_np).max(), int((np.sign(s_nat) != np.sign(s_np)).sum()), int(kept.sum()), B * N))
    assert (np.abs(np.abs(s_np[kept != kept64]) - clamp) < 1e-5).all()
    loss = s.abs()[torch.from_numpy(kept).to(s.device)].mean()
    loss.backward()
    assert abs(float(terms[0]) - loss.item()) < 5e-6, (terms[0], loss.item())
    for got, ref, tol in ((g_cond, c64.grad.cpu().numpy(), 3e-5), (g_xyz, x64.grad.cpu().numpy(), xyz_tol)):
        print('gradient error %.3g of max abs (bound %g)' % (_rel(got, ref), tol))
        assert np.abs(got - ref).max() <= tol * np.abs(ref).max(), _rel(got, ref)
    return int(kept.sum())


# The NPM test decoder's xyz input columns carry a gain of 3000 (npm_fit_common.XYZ_GAIN: without it the random stack is flat
# over the points and the sign of s is not resolved).  The point gradient ends in W_0[:, :3]^T d_0, a sum of 1024 terms that
# carry that gain, so its error relative to its max abs is larger than for an untouched stack: 4.1e-5 to 4.6e-5 measured on the
# H100.  The condition gradient and the odd stack keep the 3e-5 bar.
NPM_XYZ_TOL = 6e-5


def test_fit_surface_grad_npm_size_matches_float64_autograd(cuda_device):
    """The NPM identity decoder at the reference's batch (5 scans x 1000 points, one condition per scan), two clamps, a mask."""
    dec, _ = _npm_decoders(cuda_device)
    torch.manual_seed(2)
    xyz = torch.randn(5, 1000, 3, device=cuda_device) * 0.1 + torch.tensor([0.0, 0.05, -0.1], device=cuda_device)
    cond = torch.randn(5, 512, device=cuda_device) * 0.01
    mask = torch.rand(5, 1000, device=cuda_device) > 0.1
    counts = [_check_surface_grad(dec, xyz, cond, mask, clamp, NPM_XYZ_TOL) for clamp in (0.1, 0.01)]
    assert counts[0] > counts[1] > 200, counts


@pytest.mark.parametrize('stack,B,N', [('npm', 1, 1000), ('npm', 1, 5000), ('odd', 2, 333)])
def test_fit_surface_grad_point_counts_and_odd_stack(cuda_device, stack, B, N):
    dec = _npm_decoders(cuda_device)[0] if stack == 'npm' else _odd_decoder(cuda_device)
    torch.manual_seed(3)
    xyz = torch.randn(B, N, 3, device=cuda_device) * 0.1 + torch.tensor([0.0, 0.05, -0.1], device=cuda_device)
    cond = torch.randn(B, dec.lat_dim, device=cuda_device) * 0.01
    _check_surface_grad(dec, xyz, cond, None, 0.02, NPM_XYZ_TOL if stack == 'npm' else 3e-5)


def test_fit_surface_grad_edge_cases(cuda_device):
    """Nothing kept: NaN loss and exactly zero gradients.  A 3-output stack and a wrong workspace size are rejected.  Two calls
    give bitwise-equal results."""
    from nphm_b200 import _native
    dec, expr = _npm_decoders(cuda_device)
    eng = dec.engine()
    torch.manual_seed(4)
    xyz = torch.randn(2, 700, 3, device=cuda_device) * 0.1
    cond = torch.randn(2, 512, device=cuda_device) * 0.01
    terms, g_cond, g_xyz = eng.fit_surface_grad(xyz, cond, torch.zeros(2, 700, dtype=torch.bool, device=cuda_device), 0.1)
    assert torch.isnan(terms[0]) and float(terms[5]) == 0.0
    assert float(g_cond.abs().max()) == 0.0 and float(g_xyz.abs().max()) == 0.0
    terms, g_cond, g_xyz = eng.fit_surface_grad(xyz, cond, None, 1e-9)
    assert torch.isnan(terms[0]) and float(g_cond.abs().max()) == 0.0
    with pytest.raises(_native.NativeError, match=r'\(-3\)'):
        expr.engine().fit_surface_grad(xyz, torch.zeros(2, 712, device=cuda_device), None, 0.1)
    ws = eng.fit_workspace(2, 700, cuda_device)
    with pytest.raises(_native.NativeError, match=r'\(-1\)'):
        eng.fit_surface_grad(xyz, cond, None, 0.1, workspace=ws[:-256])
    with pytest.raises(_native.NativeError, match=r'\(-1\)'):
        eng.fit_surface_grad(xyz[:, :600], cond, None, 0.1, workspace=ws)
    a = eng.fit_surface_grad(xyz, cond, None, 0.1, workspace=ws)
    a = [t.clone() for t in a]
    b = eng.fit_surface_grad(xyz, cond, None, 0.1, workspace=ws)
    assert int(a[0][5]) > 0
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_device_broyden_search_on_npm_expression_stack(cuda_device):
    """nphm_mlp_broyden_search on the 715 -> 1024 x 8 -> 3 expression decoder (too wide for the FFMA kernel, so its network
    evaluations run on the layer chain) against the Python-loop mirror of `broyden` on the same inputs: 5e-5 on the roots that
    both find, >= 97 % identical valid flags; with the host-side early exit and in the sync-free mode."""
    from nphm_b200.models import iterative_root_finding as irf
    _, expr = _npm_decoders(cuda_device)
    eng = expr.engine()
    assert not eng.simt_ok
    obs = torch.from_numpy(np.stack(C.make_scans())).to(cuda_device)
    B, N, _ = obs.shape
    torch.manual_seed(6)
    cond = torch.randn(B, 712, device=cuda_device) * 0.05
    with torch.no_grad():
        _, j0 = eng.inverse_jacobian(obs, cond)

        def residual(flat_x, mask=None):
            pts = flat_x.reshape(B, N, 3)
            out = (expr(pts, cond[:, None, :].expand(B, N, 712))[0] + pts - obs).reshape(B * N, 3, 1)
            return out if mask is None else out[mask]

        ref = irf.broyden(residual, obs.reshape(-1, 3, 1), j0.reshape(-1, 3, 3), cvg_thresh=1e-6, dvg_thresh=0.2, max_steps=15)
        x_ref, v_ref = ref['result'].reshape(B, N, 3).cpu().numpy(), ref['valid_ids'].reshape(B, N).cpu().numpy()
        assert v_ref.mean() > 0.9
        for early_exit in (True, False):
            x, diff, valid, steps = eng.broyden_search(obs, cond, obs, j0, early_exit=early_exit)
            x, valid = x.cpu().numpy(), valid.cpu().numpy()
            assert (valid == v_ref).mean() >= 0.97
            both = valid & v_ref
            assert np.abs(x[both] - x_ref[both]).max() < 5e-5
            assert (diff.cpu().numpy()[valid] < 1e-6).all()
            if not early_exit:
                assert steps == 0                 # sync-free: the step count is not read back


def _replay(all_obs, n_iter, lambdas):
    from nphm_b200.models.fitting import _apply_schedule, _clamp_for_iteration, _sample_observations
    np.random.seed(0)
    torch.manual_seed(0)
    lr = 0.01
    for j in range(n_iter):
        lr = _apply_schedule(j, C.STEP_SCALE, C.SCHEDULE, lambdas, lr)
        obs, idx = _sample_observations(all_obs)
        yield j, obs, idx, _clamp_for_iteration(j, C.STEP_SCALE), lr


def test_npm_identity_fitter_gradients_match_reference_autograd(cuda_device):
    """The native identity iteration from the reference's own latents against the gradient it handed to Adam (fit_npm.npz)."""
    from nphm_b200.models.fitting import NpmIdentityFitter
    g = load_golden('fit_npm.npz')
    dec, _ = _npm_decoders(cuda_device)
    fitter = NpmIdentityFitter(dec, cuda_device)
    lambdas = dict(C.LAMBDAS_IDENTITY)
    all_obs = [torch.from_numpy(o).to(cuda_device) for o in g['obs']]
    for j, obs, _, clamp, lr in _replay(all_obs, C.N_ITER_IDENTITY, lambdas):
        fitter.latent.copy_(torch.from_numpy(g['id_z_before'][j]))
        fitter.step(obs, lambdas, clamp, lr, apply_update=False)
        err = _rel(fitter.grad.cpu().numpy(), g['id_grads'][j])
        print('identity iteration %d: %d kept, rel err of d loss/d z %.3g' % (j, int(fitter.loss_terms[5]), err))
        assert err < 2e-3, (j, err)


def test_npm_joint_fitter_gradients_match_reference_autograd(cuda_device):
    """The autograd-free NPM joint iteration (NpmJointFitter) from the reference's own latents against the gradients the
    reference handed to its two Adam.step() calls, with the tolerances of the NPHM joint fitter's test
    (test_joint_fitter_gradients_match_reference_autograd) and the reasons given there."""
    from nphm_b200.models.fitting import NpmJointFitter, _native_npm_joint
    g = load_golden('fit_npm.npz')
    dec, expr = _npm_decoders(cuda_device)
    assert _native_npm_joint(dec, expr, cuda_device)
    all_obs = [torch.from_numpy(o).to(cuda_device) for o in g['obs']]
    fitter = NpmJointFitter(dec, expr, len(all_obs), cuda_device)
    lambdas = dict(C.LAMBDAS_JOINT)
    for j, obs, idx, clamp, lr in _replay(all_obs, C.N_ITER_JOINT, lambdas):
        fitter.z_id.copy_(torch.from_numpy(g['joint_z_id_before'][j]))
        fitter.z_ex.copy_(torch.from_numpy(g['joint_z_ex_before'][j]))
        g_id, g_ex = fitter.step(obs, idx.long().to(cuda_device), lambdas, clamp, lr, apply_update=False)
        e_id, e_ex = _rel(g_id.cpu().numpy(), g['joint_grads_id'][j]), _rel(g_ex.cpu().numpy(), g['joint_grads_ex'][j])
        print('joint iteration %d: %d kept, rel err of d loss/d z_id %.3g, d loss/d z_ex %.3g (|g_ex| max %.3g)'
              % (j, int(fitter.loss_terms[5]), e_id, e_ex, np.abs(g['joint_grads_ex'][j]).max()))
        assert e_id < 2e-3 and e_ex < 3e-2, (j, e_id, e_ex)


def test_npm_fitters_dropin_follow_reference(cuda_device):
    """The public functions with DeepSDF decoders on CUDA (native fitters) against the reference's final codes."""
    from nphm_b200.models.fitting import inference_identity_space, inference_iterative_root_finding_joint
    g = load_golden('fit_npm.npz')
    dec, expr = _npm_decoders(cuda_device)
    all_obs = [torch.from_numpy(o).to(cuda_device) for o in g['obs']]
    lambdas = dict(C.LAMBDAS_IDENTITY)
    np.random.seed(0)
    torch.manual_seed(0)
    z, anchors = inference_identity_space(dec, all_obs, lambdas, n_steps=C.N_ITER_IDENTITY * 100, schedule_cfg=C.SCHEDULE,
                                          step_scale=C.STEP_SCALE)
    assert anchors is None and z.shape == (1, 1, 512) and z.requires_grad
    assert np.allclose([lambdas[k] for k in sorted(lambdas)], g['id_lambdas_final'])
    ci = (np.abs(z.detach().cpu().numpy().reshape(-1) - g['id_z_final']) < 5e-4).mean()
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, z_id, anchors = inference_iterative_root_finding_joint(dec, expr, all_obs, lambdas, n_steps=C.N_ITER_JOINT * 100,
                                                                 schedule_cfg=C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert anchors is None and z_ex.shape == (3, 1, 200) and z_id.shape == (1, 1, 512)
    cj = (np.abs(z_id.detach().cpu().numpy().reshape(-1) - g['joint_z_id_final']) < 5e-4).mean()
    ce = (np.abs(z_ex.detach().cpu().numpy().reshape(3, 200) - g['joint_z_ex_final']) < 5e-4).mean()
    print('NPM drop-in fits: %.1f%% of z (identity), %.1f%% of z_id and %.1f%% of z_ex (joint) within 5e-4 of the reference'
          % (100 * ci, 100 * cj, 100 * ce))
    assert ci > 0.95 and cj > 0.9 and ce > 0.9


def test_npm_joint_iteration_has_no_host_sync(cuda_device):
    """One native NPM joint iteration is a pure launch sequence: no host synchronisation (sampling excluded)."""
    from nphm_b200.models.fitting import NpmJointFitter, _sample_observations
    g = load_golden('fit_npm.npz')
    dec, expr = _npm_decoders(cuda_device)
    all_obs = [torch.from_numpy(o).to(cuda_device) for o in g['obs']]
    fitter = NpmJointFitter(dec, expr, len(all_obs), cuda_device)
    lambdas = dict(C.LAMBDAS_JOINT)
    torch.manual_seed(0)
    obs, idx = _sample_observations(all_obs)
    idx = idx.long().to(cuda_device)
    fitter.step(obs, idx, lambdas, 0.1, 0.01)                     # warm-up: buffers and workspaces
    obs, idx = _sample_observations(all_obs)
    idx = idx.long().to(cuda_device)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        fitter.step(obs, idx, lambdas, 0.1, 0.01)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(fitter.z_id).all() and torch.isfinite(fitter.z_ex).all()
