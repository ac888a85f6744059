"""GPU tests of the native joint fitters with a DeformationNetwork in the expr_only and glob_only modes (JointFitter,
BatchedJointFitter, their fixed_identity mode, and the public functions that dispatch to them).  Every check runs in both modes.

* dispatch: the public functions take the native fitters; the autograd mirror is made to raise;
* per-step gradients from the reference's own codes against the gradients the reference handed to Adam (fit_joint_modes.npz),
  with the identity decoder in training and in eval mode, and with the identity held fixed;
* float64 at fixed correspondences (the scheme of test_gpu_joint_f64.py, with the condition of each mode restated here): d/d
  z_id, d/d z_ex, no anchor term, and the condition gradient of nphm_mlp_backward_inputs at the widths 200 and 264 by itself;
* the scan-batched fitter against the single fitter, step by step and as whole fits, with and without a fixed identity;
* a step reads nothing back from the device;
* the sharded fitter at world 1 is the batched call.
"""
import numpy as np
import pytest
import torch

import chain_shapes_common as CS
import ensemble_f64_common as E
import fit_modes_common as C
import joint_f64_common as J
from conftest import load_golden, make_ensemble, mean_anchors, sample_latent
from f64_check import Check
from test_gpu_joint_f64 import (K, FLOOR, LAMBDAS, N_POINT, OBS_IDX, SURFACE_ONLY, _Capture, _check_adjoint, _latent_parts,
                                _report_u, _sample, _scans, _two_steps, _clamp_in_a_gap)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64
GOLDEN = 'fit_joint_modes.npz'


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _decoders(mode, training=True):
    dec = make_ensemble(0, device=DEV).train(training)
    return dec, C.make_deformation(mode, mean_anchors(), device=DEV)


def _golden_obs():
    return [torch.from_numpy(o).to(DEV) for o in load_golden(GOLDEN)['obs']]


def _replay(all_obs, lambdas, n_iter=C.N_ITER):
    """(j, obs, idx, clamp, lr) of the reference's loop from seed 0."""
    from nphm_b200.models.fitting import _apply_schedule, _clamp_for_iteration, _sample_observations
    np.random.seed(0)
    torch.manual_seed(0)
    lr = 0.01
    for j in range(n_iter):
        lr = _apply_schedule(j, C.STEP_SCALE, C.SCHEDULE, lambdas, lr)
        obs, idx = _sample_observations(all_obs)
        yield j, obs, idx.long().to(DEV), _clamp_for_iteration(j, C.STEP_SCALE), lr


# ------------------------------------------------------------------------------------------------ dispatch
@pytest.mark.parametrize('mode', C.MODES)
def test_public_functions_take_the_native_fitters(mode, monkeypatch):
    from nphm_b200.models import fitting as F
    monkeypatch.delenv('NPHM_JOINT_AUTOGRAD', raising=False)
    dec, dfn = _decoders(mode)
    assert F._native_joint(dec, dfn, torch.device(DEV))
    assert F._expression_fitter(dec, dfn, torch.device(DEV), batched=True) is F.BatchedJointFitter
    assert F._joint_batch_fit(dec, dfn, [_golden_obs()], 100, C.SCHEDULE, C.STEP_SCALE, 1) is not None

    def mirror(*a, **k):
        raise AssertionError('the autograd mirror was called')
    monkeypatch.setattr(F, '_inference_joint_autograd', mirror)
    obs = _golden_obs()
    subjects = [obs, obs[:2]]
    z_id = sample_latent(C.ID_SEED).to(DEV).reshape(1, 1, -1)
    lam = dict(C.LAMBDAS_JOINT)
    z_ex, z, anchors = F.inference_iterative_root_finding_joint(dec, dfn, obs, lam, 200, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert z_ex.shape == (3, 1, 200) and z.shape == (1, 1, dec.lat_dim) and anchors.shape == (1, 39, 3)
    out = F.inference_iterative_root_finding_joint_batched(dec, dfn, subjects, lam, 200, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert [r[0].shape[0] for r in out] == [3, 2]
    z_ex, anchors = F.inference_expression_space(dec, dfn, z_id, obs, lam, 200, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert z_ex.shape == (3, 1, 200) and anchors.shape == (1, 39, 3)
    out = F.inference_expression_space_batched(dec, dfn, [(z_id, obs), (z_id, obs[:2])], lam, 200, C.SCHEDULE,
                                               step_scale=C.STEP_SCALE)
    assert [r[0].shape[0] for r in out] == [3, 2]
    # what keeps the mirror: a training-mode deformation network, glob_only with a global code of another width, the switch
    dfn.train()
    assert not F._native_joint(dec, dfn, torch.device(DEV))
    dfn.eval()
    if mode == 'glob_only':
        from nphm_b200.models.deepSDF import DeformationNetwork
        other = DeformationNetwork(mode=mode, lat_dim_expr=200, lat_dim_id=32, lat_dim_glob_shape=32, lat_dim_loc_shape=32,
                                   n_loc=39, anchors=mean_anchors(), hidden_dim=512, nlayers=6, out_dim=3).eval().to(DEV)
        assert not F._native_joint(dec, other, torch.device(DEV))
    monkeypatch.setenv('NPHM_JOINT_AUTOGRAD', '1')
    with pytest.raises(AssertionError, match='autograd mirror'):
        F.inference_iterative_root_finding_joint(dec, dfn, obs, dict(C.LAMBDAS_JOINT), 100, C.SCHEDULE,
                                                 step_scale=C.STEP_SCALE)


# ------------------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('mode', C.MODES)
def test_joint_fitter_gradients_match_reference(mode, training):
    """JointFitter from the reference's own codes at every iteration, against the gradients it handed to its two Adam.step()
    calls, with the bounds of test_gpu_fit.py::test_joint_fitter_gradients_match_reference_autograd (which gives the reasons)."""
    from nphm_b200.models.fitting import JointFitter
    g = load_golden(GOLDEN)
    key = mode + ('_' if training else '_eval_')
    dec, dfn = _decoders(mode, training)
    obs = _golden_obs()
    fitter = JointFitter(dec, dfn, len(obs), torch.device(DEV))
    lambdas = dict(C.LAMBDAS_JOINT)
    for j, o, idx, clamp, lr in _replay(obs, lambdas):
        fitter.z_id.copy_(torch.from_numpy(g[key + 'z_id_before'][j]))
        fitter.z_ex.copy_(torch.from_numpy(g[key + 'z_ex_before'][j]))
        g_id, g_ex = fitter.step(o, idx, lambdas, clamp, lr, apply_update=False)
        e_id, e_ex = _rel(g_id.cpu().numpy(), g[key + 'grads_id'][j]), _rel(g_ex.cpu().numpy(), g[key + 'grads_ex'][j])
        print('%s %s iteration %d: rel err d loss/d z_id %.3g, d loss/d z_ex %.3g' % (mode, key, j, e_id, e_ex))
        assert e_id < 2e-3 and e_ex < 3e-2, (j, e_id, e_ex)
    assert [lambdas[k] for k in sorted(lambdas)] == list(g[key + 'lambdas_final'])


def _fixed_fitters(mode, dec, dfn, obs, z_id):
    """The single fixed-identity fitter on the golden scans, and the batched one with them as subject 0 of 2."""
    from nphm_b200.models.fitting import BatchedJointFitter, JointFitter
    single = JointFitter(dec, dfn, len(obs), torch.device(DEV), fixed_identity=True)
    single.z_id.copy_(z_id)
    batched = BatchedJointFitter(dec, dfn, [len(obs), 2], torch.device(DEV), fixed_identity=True)
    batched.z_id.copy_(torch.stack([z_id, sample_latent(40).to(DEV)]))
    return single, batched


@pytest.mark.parametrize('mode', C.MODES)
def test_fixed_identity_matches_reference(mode):
    """fixed_identity, single and batched (the reference's scans as subject 0 of 2): per-step d/d z_ex against the reference's
    loop with the identity held fixed, then whole fits: z_id untouched, the codes near the reference's."""
    from nphm_b200.models.fitting import _sample_observations, inference_expression_space
    g = load_golden(GOLDEN)
    key = mode + '_fixed_'
    dec, dfn = _decoders(mode)
    obs = _golden_obs()
    z_id = torch.from_numpy(g['z_id_fixed']).to(DEV)
    single, batched = _fixed_fitters(mode, dec, dfn, obs, z_id)
    other = torch.Generator().manual_seed(6)
    lambdas = dict(C.LAMBDAS_JOINT)
    for j, o, idx, clamp, lr in _replay(obs, lambdas):
        single.z_ex.copy_(torch.from_numpy(g[key + 'z_ex_before'][j]))
        g_id, g_ex = single.step(o, idx, lambdas, clamp, lr, apply_update=False)
        assert g_id is None
        o2, i2 = _sample_observations(obs[1:], other)
        batched.z_ex[:3].copy_(single.z_ex)
        batched.z_ex[3:].copy_(single.z_ex[1:] * 0.5)
        b_id, b_ex = batched.step([o, o2], [idx, i2.long().to(DEV)], lambdas, clamp, lr, apply_update=False)
        e, eb = _rel(g_ex.cpu().numpy(), g[key + 'grads_ex'][j]), _rel(b_ex[0].cpu().numpy(), g[key + 'grads_ex'][j])
        print('%s fixed identity iteration %d: rel err d loss/d z_ex %.3g (batched %.3g)' % (mode, j, e, eb))
        assert b_id is None and e < 3e-2 and eb < 3e-2, (j, e, eb)
    # whole fits: the native single function against the reference's final codes and anchors
    z_in = z_id.reshape(1, 1, -1).clone()
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, anchors = inference_expression_space(dec, dfn, z_in, obs, lambdas, C.N_ITER * 100, C.SCHEDULE,
                                               step_scale=C.STEP_SCALE)
    assert torch.equal(z_in.reshape(-1), z_id)
    assert np.array_equal(torch.get_rng_state().numpy(), g[key + 'rng_after'])
    assert [lambdas[k] for k in sorted(lambdas)] == list(g[key + 'lambdas_final'])
    close = (np.abs(z_ex.detach().cpu().numpy().reshape(3, -1) - g[key + 'z_ex_final']) < 5e-4).mean()
    print('%s fixed identity: %.1f%% of z_ex within 5e-4 of the reference' % (mode, 100 * close))
    assert close > 0.9
    assert float(np.abs(anchors.cpu().numpy().reshape(-1, 3) - g[key + 'anchors_final']).max()) < 1e-5
    # the fitters' own updates leave the identity codes alone
    z_before = batched.z_id.clone()
    for j, o, idx, clamp, lr in _replay(obs, dict(C.LAMBDAS_JOINT), 2):
        single.step(o, idx, dict(C.LAMBDAS_JOINT), clamp, lr)
        batched.step([o, o[:, :200]], [idx, idx % 2], dict(C.LAMBDAS_JOINT), clamp, lr)
    assert torch.equal(single.z_id, z_id) and torch.equal(batched.z_id, z_before)
    assert torch.isfinite(single.z_ex).all() and torch.isfinite(batched.z_ex).all()


# ------------------------------------------------------------------------------------------------ float64, fixed roots
class _ModeParams(J.NphmParams):
    """J.NphmParams for a deformation network in expr_only or glob_only mode (no compressor)."""

    def __init__(self, dec, dfn, dtype):
        self.id = E.Params(dec, dtype)
        self.expr = CS.params_of(dfn.defDeepSDF, dtype)
        self.width = {'expr_only': 0, 'glob_only': dfn.lat_dim_glob_shape}[dfn.mode]
        self.dtype = dtype


def _mode_gradients(Q, p, valid, z_id, z_ex, obs_idx, lambdas, clamp, period=0):
    """J.joint_gradients with this mode's condition rows [z_id[:P] | z_ex[b]] (deepSDF.py:203-209): the reference's implicit
    differentiation of the root, the clamped surface term, reg_expr and the identity regularisers, by autograd."""
    dt = Q.dtype
    p = p.to(dt)
    zid = z_id.to(dt).clone().requires_grad_()
    zex = z_ex.to(dt).clone().requires_grad_()
    nb = obs_idx.shape[0]
    cond = torch.cat([zid[:Q.width][None, :].expand(nb, -1), zex[obs_idx]], dim=1)
    _, j_inv = CS.ref_inverse_jacobian(Q.expr, p, cond.detach())
    posed = CS.stack_forward(Q.expr, p, cond) + p
    xc = p + torch.einsum('bnij,bnj->bni', -j_inv.detach(), posed - posed.detach())
    a = J.identity_sdf(Q, xc, zid, period).abs()
    kept = valid.reshape(-1) & (a.detach() < clamp)
    terms = {'surface': a[kept].mean(), 'reg_expr': (zex[obs_idx] * zex[obs_idx]).sum(-1).mean()}
    terms.update(zip(('reg_global', 'reg_loc', 'reg_unobserved', 'symm_dist'), E.regularisers(Q.id, zid)))
    loss = sum(float(lam) * terms[k] for k, lam in lambdas.items() if k in terms)
    g_id, g_ex = torch.autograd.grad(loss, [zid, zex])
    return g_id, g_ex, int(kept.sum())


@pytest.fixture
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _codes(j, seed):
    """(z_id, z_ex 4 x E) near the reference's own codes at iteration j of the golden run."""
    g = load_golden(GOLDEN)
    gen = torch.Generator().manual_seed(seed)
    z_id = torch.from_numpy(g['glob_only_z_id_before'][j])
    z_ex = torch.from_numpy(g['glob_only_z_ex_before'][j])
    z_id = z_id + 0.01 * z_id.abs().max() * torch.randn(z_id.shape, generator=gen)
    z_ex = torch.cat([z_ex, z_ex[:1]]) + 0.02 * torch.randn(4, z_ex.shape[1], generator=gen)
    return z_id.to(DEV), z_ex.to(DEV)


class _AnchorSpy:
    """Records the anchor gradients the fitter hands to nphm_fit_apply_gradient*."""

    def __init__(self, fitter):
        self.seen, route = [], fitter.route
        real = route.identity_gradients

        def identity_gradients(*a):
            out = real(*a)
            self.seen.append(out[1].clone())
            return out
        route.identity_gradients = identity_gradients


def _check_f64(chk, what, fitter, Q64, Q32, obs, idx, lambdas, subjects):
    """Two no-update steps at the same roots, then every subject's d/d z_id and d/d z_ex against float64, no anchor term, and
    the adjoint pass's condition gradient.  subjects: [(z_id, z_ex, own(tensor) -> that subject's points, quirk period)]."""
    spy = _AnchorSpy(fitter)
    cap = _Capture(fitter.mlp)
    try:
        def clamp_of(p, v):
            a = torch.cat([J.sdf_at_roots(Q64, own(p), z, period).abs() for z, _, own, period in subjects])
            return _clamp_in_a_gap(a, torch.cat([own(v).reshape(-1) for _, _, own, _ in subjects]))
        single = fitter.z_id.dim() == 1                                          # JointFitter: one subject, one row tensor
        (g_id, g_ex), p, valid, clamp = _two_steps(fitter, cap, obs, idx[0] if single else idx, lambdas, clamp_of)
        assert cap.adjoint[1].shape[1] == C.CONDITION_WIDTH[fitter.dfn.mode]
        _report_u(chk, what, cap.adjoint[2])
        if single:
            g_id, g_ex = g_id[None], [g_ex]
        for k, (z_id, z_ex, own, period) in enumerate(subjects):
            r64 = _mode_gradients(Q64, own(p).double(), own(valid), z_id.double(), z_ex.double(), idx[k], lambdas, clamp,
                                  period)
            r32 = _mode_gradients(Q32, own(p), own(valid), z_id, z_ex, idx[k], lambdas, clamp, period)
            assert r64[2] == r32[2] > 0, (what, k, r64[2], r32[2])
            chk('%s subject %d z_id' % (what, k), g_id[k], r64[0], r32[0], kind='scalar', parts=_latent_parts(Q64))
            rows = idx[k].tolist()
            chk('%s subject %d z_ex' % (what, k), g_ex[k], r64[1], r32[1], kind='scalar',
                parts=[('row %d' % r, r) for r in sorted(set(rows))])
            assert all(bool((g_ex[k][r] == 0).all()) for r in range(z_ex.shape[0]) if r not in rows)
        _check_adjoint(chk, what, Q64, Q32, cap)
        assert spy.seen and all(not bool(a.any()) for a in spy.seen), 'an anchor term outside compress'
    finally:
        cap.release()


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('lambdas', [LAMBDAS, SURFACE_ONLY], ids=['fitting-yaml', 'surface-only'])
@pytest.mark.parametrize('mode', C.MODES)
def test_joint_fitter_float64(mode, lambdas, training, _fp32_without_tf32):
    """JointFitter at its own roots against float64; the adjoint pass at condition width 200 (expr_only) / 264 (glob_only)."""
    from nphm_b200.models.fitting import JointFitter
    dec, dfn = _decoders(mode, training)
    Q64, Q32 = _ModeParams(dec, dfn, F64), _ModeParams(dec, dfn, F32)
    chk = Check('JointFitter', K, FLOOR, prefix='JOINT')
    fitter = JointFitter(dec, dfn, 4, torch.device(DEV))
    z_id, z_ex = _codes(2, 0)
    fitter.z_id.copy_(z_id)
    fitter.z_ex.copy_(z_ex)
    idx = torch.tensor(OBS_IDX, device=DEV)
    obs = _sample(_scans(GOLDEN, 0), OBS_IDX, N_POINT)
    what = '%s %s %s' % (mode, 'train' if training else 'eval', 'yaml' if len(lambdas) > 1 else 'surface')
    _check_f64(chk, what, fitter, Q64, Q32, obs, [idx], lambdas, [(z_id, z_ex, lambda t: t, 0 if training else N_POINT)])
    chk.done()


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('mode', C.MODES)
def test_batched_joint_fitter_float64(mode, training, _fp32_without_tf32):
    """BatchedJointFitter, three subjects of unequal lengths (padded behind in training mode, in front in eval mode)."""
    from nphm_b200.models.fitting import BatchedJointFitter
    dec, dfn = _decoders(mode, training)
    Q64, Q32 = _ModeParams(dec, dfn, F64), _ModeParams(dec, dfn, F32)
    chk = Check('BatchedJoint', K, FLOOR, prefix='JOINT')
    S, ns = 3, (N_POINT, 613, 250)
    fitter = BatchedJointFitter(dec, dfn, [4] * S, torch.device(DEV))
    codes = [_codes(1 + k % 3, 10 + k) for k in range(S)]
    for k, (z_id, z_ex) in enumerate(codes):
        fitter.z_id[k].copy_(z_id)
        fitter.z_ex[4 * k:4 * k + 4].copy_(z_ex)
    idx = [torch.tensor(OBS_IDX[k:] + OBS_IDX[:k], device=DEV) for k in range(S)]
    obs = [_sample(_scans(GOLDEN, 20 + k), idx[k].tolist(), ns[k]) for k in range(S)]
    front = not training

    def own(k):
        def view(t):
            t = t.reshape(S, 5, N_POINT, *t.shape[2:])[k]
            return t[:, N_POINT - ns[k]:] if front else t[:, :ns[k]]
        return view
    # in eval mode every subject's quirk period is its own row length: the fitter pads in front, so its last point stays last
    subjects = [(z_id, z_ex, own(k), 0 if training else ns[k]) for k, (z_id, z_ex) in enumerate(codes)]
    _check_f64(chk, '%s S=%d %s' % (mode, S, 'train' if training else 'eval'), fitter, Q64, Q32, obs, idx, LAMBDAS, subjects)
    chk.done()


# ------------------------------------------------------------------------------------------------ batched = single
def _subjects():
    obs = _golden_obs()
    return [obs, [o * 1.03 + 0.01 for o in obs], [o[:200] for o in obs[:2]]]    # 3, 3 and 2 observations, 300 / 200 points


@pytest.mark.parametrize('mode', C.MODES)
def test_batched_step_matches_single_fitter(mode):
    """One step of BatchedJointFitter (free and fixed identity) against JointFitter on each subject, same codes and draws."""
    from nphm_b200.models.fitting import BatchedJointFitter, JointFitter, _sample_observations
    dec, dfn = _decoders(mode)
    subjects = _subjects()
    gen = torch.Generator().manual_seed(3)
    dgen = torch.Generator(device=DEV).manual_seed(4)
    z_id = torch.stack([sample_latent(30 + k) for k in range(3)]).to(DEV) * 0.3
    z_ex = [torch.randn(len(s), 200, device=DEV, generator=dgen) * 0.05 for s in subjects]
    for fixed in (False, True):
        bj = BatchedJointFitter(dec, dfn, [len(s) for s in subjects], torch.device(DEV), fixed_identity=fixed)
        bj.z_id.copy_(z_id)
        bj.z_ex.copy_(torch.cat(z_ex))
        samples = [_sample_observations(s, gen) for s in subjects]
        idx = [i.long().to(DEV) for _, i in samples]
        g_id, g_ex = bj.step([o for o, _ in samples], idx, dict(C.LAMBDAS_JOINT), 0.1, 0.01, apply_update=False)
        assert (g_id is None) == fixed
        for k in range(3):
            jf = JointFitter(dec, dfn, len(subjects[k]), torch.device(DEV), fixed_identity=fixed)
            jf.z_id.copy_(z_id[k])
            jf.z_ex.copy_(z_ex[k])
            s_id, s_ex = jf.step(samples[k][0], idx[k], dict(C.LAMBDAS_JOINT), 0.1, 0.01, apply_update=False)
            e_ex = float((g_ex[k] - s_ex).abs().max() / s_ex.abs().max())
            e_id = 0.0 if fixed else float((g_id[k] - s_id).abs().max() / s_id.abs().max())
            print('%s fixed=%s subject %d: batched vs single rel err z_id %.3g z_ex %.3g' % (mode, fixed, k, e_id, e_ex))
            assert e_id < 1e-4 and e_ex < 1e-4, (fixed, k, e_id, e_ex)


def _close(a, b, tol=5e-4):
    return float((a.detach() - b.detach()).abs().lt(tol).float().mean())


@pytest.mark.parametrize('S', [1, 3])
@pytest.mark.parametrize('mode', C.MODES)
def test_batched_functions_equal_sequential_calls(mode, S):
    """inference_iterative_root_finding_joint_batched and inference_expression_space_batched against the single-subject
    functions called in turn: the generator state and lambdas end equal, the codes within the bounds of
    test_gpu_fit_batched.py."""
    from nphm_b200.models.fitting import (inference_expression_space, inference_expression_space_batched,
                                          inference_iterative_root_finding_joint,
                                          inference_iterative_root_finding_joint_batched)
    dec, dfn = _decoders(mode)
    subjects = _subjects()[-S:]
    args = (C.SCHEDULE,)
    torch.manual_seed(0)
    seq = [inference_iterative_root_finding_joint(dec, dfn, s, dict(C.LAMBDAS_JOINT), 400, *args, step_scale=C.STEP_SCALE)
           for s in subjects]
    state, lam_seq = torch.get_rng_state(), dict(C.LAMBDAS_JOINT)
    inference_iterative_root_finding_joint(dec, dfn, subjects[0], lam_seq, 400, *args, step_scale=C.STEP_SCALE)
    torch.manual_seed(0)
    lam = dict(C.LAMBDAS_JOINT)
    bat = inference_iterative_root_finding_joint_batched(dec, dfn, subjects, lam, 400, *args, step_scale=C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state) and lam == lam_seq
    for k, ((e1, i1, a1), (e2, i2, a2)) in enumerate(zip(seq, bat)):
        ci, ce = _close(i1, i2), _close(e1, e2)
        print('%s S=%d joint subject %d: %.4f of z_id, %.4f of z_ex within 5e-4 of the sequential call' % (mode, S, k, ci, ce))
        assert e1.shape == e2.shape and ci > 0.9 and ce > 0.9, k
        assert float((a1 - a2).abs().max()) < 1e-5, k
    # the identity held fixed, one warm-started entry
    ids = [sample_latent(50 + k).to(DEV).reshape(1, 1, -1) for k in range(S)]
    entries = [(ids[k], s) for k, s in enumerate(subjects)]
    entries[-1] = entries[-1] + (torch.randn(len(subjects[-1]), 1, 200, device=DEV) * 0.02,)
    torch.manual_seed(0)
    seq = [inference_expression_space(dec, dfn, e[0], e[1], dict(C.LAMBDAS_JOINT), 400, *args, step_scale=C.STEP_SCALE,
                                      lat_reps_expr_init=e[2] if len(e) > 2 else None) for e in entries]
    state = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(C.LAMBDAS_JOINT)
    bat = inference_expression_space_batched(dec, dfn, entries, lam, 400, *args, step_scale=C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state) and lam == lam_seq
    for k, ((e1, a1), (e2, a2)) in enumerate(zip(seq, bat)):
        ce = _close(e1, e2)
        print('%s S=%d fixed identity subject %d: %.4f of z_ex within 5e-4 of the sequential call' % (mode, S, k, ce))
        assert ce > 0.9 and float((a1 - a2).abs().max()) < 1e-5, k
    assert all(torch.equal(e[0], i) for e, i in zip(entries, ids))


# ------------------------------------------------------------------------------------------------ launch sequences
@pytest.mark.parametrize('mode', C.MODES)
def test_steps_do_not_synchronise_with_the_host(mode):
    from nphm_b200.models.fitting import BatchedJointFitter, JointFitter, _sample_observations
    dec, dfn = _decoders(mode)
    subjects = _subjects()
    z_id = sample_latent(C.ID_SEED).to(DEV)
    fitters = []
    for fixed in (False, True):
        single = JointFitter(dec, dfn, 3, torch.device(DEV), fixed_identity=fixed)
        batched = BatchedJointFitter(dec, dfn, [len(s) for s in subjects], torch.device(DEV), fixed_identity=fixed)
        single.z_id.copy_(z_id)
        batched.z_id.copy_(z_id.expand(3, -1))
        fitters += [(single, False), (batched, True)]
    torch.manual_seed(0)
    samples = [_sample_observations(s) for s in subjects]
    args = {False: (samples[0][0], samples[0][1].long().to(DEV)),
            True: ([o for o, _ in samples], [i.long().to(DEV) for _, i in samples])}
    for f, b in fitters:
        f.step(*args[b], dict(C.LAMBDAS_JOINT), 0.1, 0.01)            # warm-up: workspaces, anchors, condition prefix
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for f, b in fitters:
            f.step(*args[b], dict(C.LAMBDAS_JOINT), 0.1, 0.01)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    for f, _ in fitters:
        assert torch.isfinite(f.z_id).all() and torch.isfinite(f.z_ex).all()
        if f.fixed_identity:
            assert torch.equal(f.z_id.reshape(-1, z_id.numel()), z_id.expand(f.z_id.reshape(-1, z_id.numel()).shape[0], -1))


# ------------------------------------------------------------------------------------------------ sharded fitter
@pytest.mark.parametrize('mode', C.MODES)
def test_sharded_world_one_is_the_batched_call(mode, monkeypatch):
    from nphm_b200.fitting_sharded import inference_iterative_root_finding_joint_batched_sharded
    from nphm_b200.models import fitting as F
    from test_gpu_fit_sharded import _assert_close, _record_steps
    dec, dfn = _decoders(mode)
    subjects = _subjects()
    assert F._joint_batch_fit(dec, dfn, subjects, 400, C.SCHEDULE, C.STEP_SCALE, 1) is not None
    log = _record_steps(monkeypatch)

    def run(fn, **kw):
        torch.manual_seed(0)
        lam = dict(C.LAMBDAS_JOINT)
        out = fn(dec, dfn, subjects, lam, 400, C.SCHEDULE, step_scale=C.STEP_SCALE, **kw)
        return out, torch.get_rng_state(), lam
    want = run(F.inference_iterative_root_finding_joint_batched)
    steps_want = list(log)
    log.clear()
    got = run(inference_iterative_root_finding_joint_batched_sharded, batch_size=len(subjects))
    assert len(steps_want) == 4 and log == steps_want
    assert all(name == 'BatchedJointFitter' for name, _, _ in log)
    _assert_close(got, want, mode)
