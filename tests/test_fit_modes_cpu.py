"""CPU checks of joint fitting with a DeformationNetwork in the expr_only and glob_only modes.

* The autograd mirror (the path every configuration without a native fitter takes) against the reference's own joint loop in
  both modes (tests/golden/fit_joint_modes.npz from make_golden_fit_joint_modes.py): the gradients the reference handed to its
  two Adam.step() calls at every step, the final codes and anchors, the mutated lambdas and torch's CPU generator afterwards; the
  same for the loop with the identity code held fixed (inference_expression_space).
* The routing of the native fitters (fitting._IdentityRoute) restated in float64 on the composite modules: the condition prefix
  is what DeformationNetwork._condition puts in front of z_ex, and the identity and anchor gradients it hands on are autograd's
  through that condition, with no anchor term outside compress.  The native fitters are checked on the GPU
  (test_gpu_fit_modes.py).
"""
import numpy as np
import pytest
import torch

import fit_modes_common as C
import npm_fit_common as N
from conftest import load_golden, make_ensemble, mean_anchors, sample_latent


def _recording_adam(monkeypatch, record):
    real = torch.optim.Adam

    class RecordingAdam(real):
        def step(self, closure=None):
            p = self.param_groups[0]['params'][0]
            record.append((p.grad.detach().clone().double(), p.detach().clone().double()))
            return super().step(closure)
    monkeypatch.setattr(torch.optim, 'Adam', RecordingAdam)


def _setup(mode):
    g = load_golden('fit_joint_modes.npz')
    dfn = C.make_deformation(mode, mean_anchors())
    assert N.state_dict_sha256(dfn) == str(g[mode + '_sha256'])
    return g, make_ensemble(0).train(), dfn, [torch.from_numpy(o) for o in g['obs']]


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _check_end_state(g, key, lambdas, z_ex, anchors):
    assert np.array_equal(torch.get_rng_state().numpy(), g[key + 'rng_after'])
    assert [lambdas[k] for k in sorted(lambdas)] == list(g[key + 'lambdas_final'])
    assert np.abs(z_ex.detach().double().numpy().reshape(C.N_OBS, -1) - g[key + 'z_ex_final']).max() < 1e-4
    assert np.abs(anchors.detach().double().numpy().reshape(-1, 3) - g[key + 'anchors_final']).max() < 1e-5


@pytest.mark.parametrize('mode', C.MODES)
def test_joint_mirror_follows_reference(mode, monkeypatch):
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint
    g, dec, dfn, obs = _setup(mode)
    record = []
    _recording_adam(monkeypatch, record)
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, z_id, anchors = inference_iterative_root_finding_joint(dec, dfn, obs, lambdas, C.N_ITER * 100, C.SCHEDULE,
                                                                 step_scale=C.STEP_SCALE)
    key = mode + '_'
    _check_end_state(g, key, lambdas, z_ex, anchors)
    assert np.abs(z_id.detach().double().numpy().reshape(-1) - g[key + 'z_id_final']).max() < 1e-4
    # two optimizers, the identity's first: records alternate
    assert len(record) == 2 * C.N_ITER
    for j in range(C.N_ITER):
        (gi, zi), (ge, ze) = record[2 * j], record[2 * j + 1]
        e_id = _rel(gi.numpy().reshape(-1), g[key + 'grads_id'][j])
        e_ex = _rel(ge.numpy().reshape(C.N_OBS, -1), g[key + 'grads_ex'][j])
        print('%s iteration %d: rel err d loss/d z_id %.3g, d loss/d z_ex %.3g' % (mode, j, e_id, e_ex))
        assert e_id < 1e-3 and e_ex < 1e-3, (j, e_id, e_ex)
        assert np.abs(zi.numpy().reshape(-1) - g[key + 'z_id_before'][j]).max() < 1e-4
        assert np.abs(ze.numpy().reshape(C.N_OBS, -1) - g[key + 'z_ex_before'][j]).max() < 1e-4


@pytest.mark.parametrize('mode', C.MODES)
def test_fixed_identity_mirror_follows_reference(mode, monkeypatch):
    from nphm_b200.models.fitting import inference_expression_space
    g, dec, dfn, obs = _setup(mode)
    z_id = torch.from_numpy(g['z_id_fixed']).reshape(1, 1, -1)
    z_before = z_id.clone()
    record = []
    _recording_adam(monkeypatch, record)
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, anchors = inference_expression_space(dec, dfn, z_id, obs, lambdas, C.N_ITER * 100, C.SCHEDULE,
                                               step_scale=C.STEP_SCALE)
    assert torch.equal(z_id, z_before)
    key = mode + '_fixed_'
    _check_end_state(g, key, lambdas, z_ex, anchors)
    assert len(record) == C.N_ITER
    for j, (ge, ze) in enumerate(record):
        e_ex = _rel(ge.numpy().reshape(C.N_OBS, -1), g[key + 'grads_ex'][j])
        print('%s fixed identity iteration %d: rel err d loss/d z_ex %.3g' % (mode, j, e_ex))
        assert e_ex < 1e-3, (j, e_ex)
        assert np.abs(ze.numpy().reshape(C.N_OBS, -1) - g[key + 'z_ex_before'][j]).max() < 1e-4


# ------------------------------------------------------------------------------------------------ routing in float64
def _composite_rows(dfn, z_id, z_ex, anchors):
    """DeformationNetwork._condition of the rows [z_id | z_ex[b]] (float64, with graph): nb x C."""
    nb = z_ex.shape[0]
    lat = torch.cat([z_id[None, :].expand(nb, -1), z_ex], dim=1)[:, None, :]
    a = anchors.reshape(1, -1, 3).expand(nb, -1, -1)
    return dfn._condition(torch.zeros(nb, 1, 3, dtype=z_id.dtype), lat, a, per_point=False)[:, 0]


@pytest.mark.parametrize('mode', ('compress',) + C.MODES)
def test_identity_route_restates_the_condition_in_float64(mode):
    """Prefix width and values, d/d z_id and d/d anchors of the single- and S-subject forms against autograd through the
    composite condition, for an arbitrary upstream on the condition's prefix columns."""
    from nphm_b200.models.fitting import _IdentityRoute
    dec = make_ensemble(0).double()
    dfn = C.make_deformation(mode, mean_anchors()).double()
    route = _IdentityRoute(dfn)
    P, E = route.width, dfn.lat_dim_expr
    assert P + E == C.CONDITION_WIDTH[mode] == dfn.defDeepSDF.lat_dim
    assert P == {'compress': 32, 'glob_only': 64, 'expr_only': 0}[mode]
    gen = torch.Generator().manual_seed(4)
    S, nb = 3, 5
    z_ids = [sample_latent(20 + k).double() for k in range(S)]
    with torch.no_grad():
        anchors = [dec.predict_anchors(z.reshape(1, 1, -1)).reshape(1, -1, 3) for z in z_ids]       # 1 x K x 3
    K3 = anchors[0].numel()
    z_ex = torch.randn(S, nb, E, generator=gen, dtype=torch.float64) * 0.1
    g_rows = torch.randn(S, nb, P, generator=gen, dtype=torch.float64)
    g_lat = torch.randn(S, dec.lat_dim, generator=gen, dtype=torch.float64)
    singles = []
    for k in range(S):
        zi = z_ids[k].clone().requires_grad_(True)
        ak = anchors[k].clone().requires_grad_(True)
        rows = _composite_rows(dfn, zi, z_ex[k], ak)
        assert rows.shape == (nb, P + E) and torch.equal(rows[:, P:], z_ex[k])
        prefix = route.prefix(z_ids[k], anchors[k])
        assert prefix.shape == (P,)
        assert torch.allclose(rows[:, :P].detach(), prefix[None].expand(nb, -1), rtol=1e-12, atol=1e-12)
        (rows[:, :P] * g_rows[k]).sum().backward()
        want_id = g_lat[k] + (zi.grad if zi.grad is not None else 0)
        want_anc = ak.grad.reshape(-1) if ak.grad is not None else torch.zeros(K3, dtype=torch.float64)
        got_id, got_anc = route.identity_gradients(g_lat[k], g_rows[k], anchors[k])
        assert got_id.shape == (dec.lat_dim,) and got_anc.shape == (K3,)
        assert torch.allclose(got_id, want_id, rtol=1e-12, atol=1e-12), mode
        assert torch.allclose(got_anc, want_anc, rtol=1e-12, atol=1e-12), mode
        if mode != 'compress':
            assert not got_anc.any()                                         # no anchor term
            assert torch.equal(got_id[P:], g_lat[k][P:])                       # only z_id[:P] is routed
        singles.append((prefix, got_id, got_anc))
    # the S-subject form: the same per subject
    z_all, a_all = torch.stack(z_ids), torch.cat(anchors)
    prefix = route.prefix(z_all, a_all)
    got_id, got_anc = route.identity_gradients(g_lat, g_rows.reshape(S * nb, P), a_all)
    assert prefix.shape == (S, P) and got_id.shape == g_lat.shape and got_anc.shape == (S, K3)
    for k, (p1, i1, a1) in enumerate(singles):
        assert torch.allclose(prefix[k], p1, rtol=1e-12, atol=1e-12)
        assert torch.allclose(got_id[k], i1, rtol=1e-12, atol=1e-12)
        assert torch.allclose(got_anc[k], a1, rtol=1e-12, atol=1e-12)
