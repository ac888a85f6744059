"""CPU check of inference_expression_space's autograd mirror against the reference's own joint loop run with the identity code
held fixed (tests/golden/fit_expression.npz from make_golden_fit_expression.py): for the NPHM ensemble with its deformation
network and for the NPM pair of DeepSDF decoders, the expression gradients the reference handed to Adam at every step, the
final codes, the anchors, the mutated lambdas and torch's CPU generator afterwards.  The batched form is checked against
sequential calls.  The native fitters are checked against the same golden on the GPU (test_gpu_fit_expression.py)."""
import numpy as np
import pytest
import torch

import fit_expression_common as C
import npm_fit_common as N
from conftest import load_golden, make_deformation, make_ensemble


def _pair(which):
    g = load_golden('fit_expression.npz')
    if which == 'nphm':
        dec, expr = make_ensemble(0).train(), make_deformation()
    else:
        from nphm_b200.models.deepSDF import DeepSDF
        dec, expr = N.make_decoders(DeepSDF)
    assert N.state_dict_sha256(dec) == str(g[which + '_sha256_id'])
    assert N.state_dict_sha256(expr) == str(g[which + '_sha256_ex'])
    scans, i = [], 0
    while '%s_scan%d' % (which, i) in g.files:
        scans.append(torch.from_numpy(g['%s_scan%d' % (which, i)]))
        i += 1
    z_id = torch.from_numpy(g[which + '_z_id']).reshape(1, 1, -1)
    return g, dec, expr, scans, z_id


def _recording_adam(monkeypatch, record):
    real = torch.optim.Adam

    class RecordingAdam(real):
        def step(self, closure=None):
            p = self.param_groups[0]['params'][0]
            record.append((p.grad.detach().clone().double(), p.detach().clone().double()))
            return super().step(closure)
    monkeypatch.setattr(torch.optim, 'Adam', RecordingAdam)


@pytest.mark.parametrize('which', ['nphm', 'npm'])
def test_mirror_follows_reference_with_the_identity_held_fixed(which, monkeypatch):
    from nphm_b200.models.fitting import inference_expression_space
    g, dec, expr, scans, z_id = _pair(which)
    z_id_before = z_id.clone()
    record = []
    _recording_adam(monkeypatch, record)
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, anchors = inference_expression_space(dec, expr, z_id, scans, lambdas, n_steps=C.N_ITER * 100,
                                               schedule_cfg=C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert torch.equal(z_id, z_id_before)
    assert np.array_equal(torch.get_rng_state().numpy(), g[which + '_rng_after'])
    assert [lambdas[k] for k in sorted(lambdas)] == list(g[which + '_lambdas_final'])
    K = len(scans)
    assert z_ex.shape == (K, 1, g[which + '_z_ex_final'].shape[1]) and z_ex.requires_grad
    # one optimizer, over the expression codes: one record per iteration
    assert len(record) == C.N_ITER
    ref_g, ref_z = g[which + '_grads'], g[which + '_codes_before']
    for j, (grad, code) in enumerate(record):
        grad, code = grad.numpy().reshape(K, -1), code.numpy().reshape(K, -1)
        e_g = np.abs(grad - ref_g[j]).max() / np.abs(ref_g[j]).max()
        e_z = np.abs(code - ref_z[j]).max()
        print('%s iteration %d: rel err of d loss/d z_ex %.3g, max |z_ex - ref| %.3g' % (which, j, e_g, e_z))
        assert e_g < 1e-3 and e_z < 1e-4, (j, e_g, e_z)
    err = np.abs(z_ex.detach().double().numpy().reshape(K, -1) - g[which + '_z_ex_final'])
    assert err.max() < 1e-4, err.max()
    if which == 'nphm':
        assert np.abs(anchors.detach().double().numpy().reshape(-1, 3) - g['nphm_anchors']).max() < 1e-6
    else:
        assert anchors is None


def test_mirror_batched_equals_sequential_calls():
    """The batched function without a native fitter (CPU): one call per entry, warm starts honoured, the generator and the
    lambdas left as the sequential calls leave them."""
    from nphm_b200.models.fitting import inference_expression_space, inference_expression_space_batched
    g, dec, expr, scans, z_id = _pair('npm')
    torch.manual_seed(5)
    warm = torch.randn(2, 1, 200) * 0.01
    subjects = [(z_id, scans[:2], warm), (z_id * 0.5, scans[2:])]
    lam0 = dict(C.LAMBDAS_JOINT)
    torch.manual_seed(0)
    seq = [inference_expression_space(dec, expr, s[0], s[1], dict(lam0), 300, C.SCHEDULE, step_scale=C.STEP_SCALE,
                                      lat_reps_expr_init=s[2] if len(s) > 2 else None) for s in subjects]
    state = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lam0)
    bat = inference_expression_space_batched(dec, expr, subjects, lam, 300, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state)
    one = dict(lam0)
    inference_expression_space(dec, expr, z_id, scans[:1], one, 300, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert lam == one != lam0
    for (a, _), (b, _) in zip(seq, bat):
        assert torch.equal(a, b)
