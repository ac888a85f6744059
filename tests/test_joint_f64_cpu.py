"""The float64 joint-iteration reference of tests/joint_f64_common.py against the graph ``_inference_joint_autograd`` builds
at the same roots (no GPU needed): the fitters' composite path, run in float64 with its correspondence search, sampling and
optimisers replaced, for both decoders and both modes of the identity ensemble."""
import copy
import types

import pytest
import torch

import joint_f64_common as J
from conftest import load_golden, make_deformation, make_ensemble


class _Recorder:
    """Stands in for torch.optim.Adam inside the fitter: sets its parameter to the code under test and records the gradient
    the reference would hand to Adam.step()."""
    codes, grads = {}, {}

    def __init__(self, params, lr):
        self.p = params[0]
        with torch.no_grad():
            self.p.copy_(self.codes[tuple(self.p.shape)])
        self.param_groups = []

    def zero_grad(self):
        self.p.grad = None

    def step(self):
        self.grads[tuple(self.p.shape)] = self.p.grad.detach().clone()


def _composite_grads(monkeypatch, dec, dfn, obs, obs_idx, p, valid, z_id, z_ex, lambdas):
    """(d loss / d z_id, d loss / d z_ex) of one iteration of the composite joint fitter at roots p (clamp 0.1, iteration 0)."""
    from nphm_b200.models import fitting
    _Recorder.codes = {(1, 1, z_id.shape[0]): z_id.reshape(1, 1, -1), (z_ex.shape[0], 1, z_ex.shape[1]): z_ex[:, None, :]}
    _Recorder.grads = {}
    monkeypatch.setattr(fitting, 'optim', types.SimpleNamespace(Adam=_Recorder))
    monkeypatch.setattr(fitting, '_sample_observations', lambda all_obs: (obs, obs_idx))
    monkeypatch.setattr(fitting, 'search', lambda *a, **k: (p.clone(), {'valid_ids': valid}))
    all_obs = [torch.zeros(4, 3, dtype=torch.float64) for _ in range(z_ex.shape[0])]
    fitting._inference_joint_autograd(dec, dfn, all_obs, dict(lambdas), 1, {})
    return _Recorder.grads[(1, 1, z_id.shape[0])].reshape(-1), _Recorder.grads[tuple(z_ex[:, None, :].shape)][:, 0]


def _roots(obs, seed):
    g = torch.Generator().manual_seed(seed)
    p = obs + 0.01 * torch.randn(obs.shape, generator=g, dtype=torch.float64)
    valid = torch.rand(obs.shape[:2], generator=g) < 0.8
    return p, valid


LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
OBS_IDX = torch.tensor([2, 0, 2, 1, 0])


@pytest.fixture
def float64_default():
    saved = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(saved)


@pytest.mark.parametrize('training', [True, False])
def test_reference_equals_the_composite_joint_iteration_nphm(monkeypatch, float64_default, training):
    """Identity ensemble + 'compress' DeformationNetwork: both gradients to 1e-10 of their largest entry; in eval mode the
    last point of every row carries the ensemble's quirk."""
    dec = make_ensemble(0).train(training)
    dfn = make_deformation()
    Q = J.NphmParams(dec, dfn, torch.float64)
    dec64 = copy.deepcopy(dec).double()
    dec64.anchors = dec64.anchors.double()
    dfn64 = copy.deepcopy(dfn).double()
    g = load_golden('fit_joint.npz')
    z_id = torch.from_numpy(g['z_id_before'][2]).double()
    z_ex = torch.cat([torch.from_numpy(g['z_ex_before'][2]).double(), 0.05 * torch.ones(1, 200, dtype=torch.float64)])
    obs = torch.from_numpy(g['obs']).double()[OBS_IDX % 3][:, :40]
    p, valid = _roots(obs, 1)
    want_id, want_ex = _composite_grads(monkeypatch, dec64, dfn64, obs, OBS_IDX, p, valid, z_id, z_ex, LAMBDAS)
    got_id, got_ex, kept = J.joint_gradients(Q, p, valid, z_id, z_ex, OBS_IDX, LAMBDAS, 0.1, 0 if training else 40)
    assert kept > 0 and (training or kept < int(valid.sum())), kept         # eval mode: the quirk rows (|s| ~ 1) drop out
    assert float((got_id - want_id).abs().max()) <= 1e-10 * float(want_id.abs().max())
    assert float((got_ex - want_ex).abs().max()) <= 1e-10 * float(want_ex.abs().max())
    assert bool((got_ex[3] == 0).all()) and bool((want_ex[3] == 0).all())          # row 3 is not sampled


def test_reference_equals_the_composite_joint_iteration_npm(monkeypatch, float64_default):
    """NPM baseline (DeepSDF identity and expression decoders of fitting_npm.yaml)."""
    import npm_fit_common as NC
    from nphm_b200.models.deepSDF import DeepSDF
    dec, expr = NC.make_decoders(DeepSDF)
    Q = J.NpmParams(dec, expr, torch.float64)
    g = load_golden('fit_npm.npz')
    z_id = torch.from_numpy(g['joint_z_id_before'][3]).double()
    z_ex = torch.cat([torch.from_numpy(g['joint_z_ex_before'][3]).double(), 0.05 * torch.ones(1, 200, dtype=torch.float64)])
    obs = torch.from_numpy(g['obs']).double()[OBS_IDX % 3][:, :24]
    p, valid = _roots(obs, 2)
    want_id, want_ex = _composite_grads(monkeypatch, copy.deepcopy(dec).double(), copy.deepcopy(expr).double(), obs, OBS_IDX,
                                        p, valid, z_id, z_ex, LAMBDAS)
    got_id, got_ex, kept = J.joint_gradients(Q, p, valid, z_id, z_ex, OBS_IDX, LAMBDAS, 0.1)
    assert kept > 0
    assert float((got_id - want_id).abs().max()) <= 1e-10 * float(want_id.abs().max())
    assert float((got_ex - want_ex).abs().max()) <= 1e-10 * float(want_ex.abs().max())
    assert bool((got_ex[3] == 0).all()) and bool((want_ex[3] == 0).all())
