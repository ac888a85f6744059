"""CPU tests of scan-batched fitting: the sampling plan replays the sequential global-generator stream, and the batched
fitting functions on CPU (the composite fallback) equal sequential calls bitwise."""
import torch

from conftest import make_ensemble
from fit_common import golden_fit_setup


def _scans():
    _, obs, _, _ = golden_fit_setup()
    return [obs, [o[:700] * 1.02 for o in obs], [o + 0.01 for o in obs[:2]]]


def test_sampling_plan_replays_the_sequential_stream():
    from nphm_b200.models.fitting import _sample_indices, _sampling_plan
    scans = _scans()
    sizes = [[o.shape[0] for o in s] for s in scans]
    n_iters = 7
    torch.manual_seed(0)
    seq = [[_sample_indices(sz) for _ in range(n_iters)] for sz in sizes]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    gens = _sampling_plan(scans, n_iters)
    assert torch.equal(torch.get_rng_state(), state_seq)
    for k, (sz, g) in enumerate(zip(sizes, gens)):
        for j in range(n_iters):
            idx, sub = _sample_indices(sz, g)
            assert torch.equal(idx, seq[k][j][0]), (k, j)
            assert all(torch.equal(a, b) for a, b in zip(sub, seq[k][j][1])), (k, j)
    # drawing from the plan's generators leaves the global generator alone
    assert torch.equal(torch.get_rng_state(), state_seq)


def test_identity_space_batched_on_cpu_equals_sequential_calls():
    from nphm_b200.models.fitting import inference_identity_space, inference_identity_space_batched
    _, _, lambdas, _ = golden_fit_setup()
    schedule = {'lr': {100: 2}, 'symm_dist': {100: 10}, 'reg_glob': {100: 3}}
    dec = make_ensemble(0).train()
    scans = _scans()
    torch.manual_seed(0)
    seq = [inference_identity_space(dec, s, dict(lambdas), 200, schedule, step_scale=0.01) for s in scans]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lambdas)
    bat = inference_identity_space_batched(dec, scans, lam, 200, schedule, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    one = dict(lambdas)
    inference_identity_space(dec, scans[0], one, 200, schedule, step_scale=0.01)
    assert lam == one and lam != lambdas
    assert len(bat) == len(scans)
    for (z1, a1), (z2, a2) in zip(seq, bat):
        assert torch.equal(z1, z2) and torch.equal(a1, a2)
    assert inference_identity_space_batched(dec, [], dict(lambdas), 200, schedule) == []


def test_joint_batched_on_cpu_equals_sequential_calls():
    from conftest import make_deformation
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint, inference_iterative_root_finding_joint_batched
    lambdas = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    schedule = {'lr': {100: 2}, 'reg_expr': {100: 10}}
    dec = make_ensemble(0).train()
    dfn = make_deformation()
    subjects = [[o[:200] for o in s] for s in _scans()[:2]]
    torch.manual_seed(0)
    seq = [inference_iterative_root_finding_joint(dec, dfn, s, dict(lambdas), 200, schedule, step_scale=0.01)
           for s in subjects]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lambdas)
    bat = inference_iterative_root_finding_joint_batched(dec, dfn, subjects, lam, 200, schedule, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    assert lam['reg_expr'] == lambdas['reg_expr'] / 10
    for r1, r2 in zip(seq, bat):
        for a, b in zip(r1, r2):
            assert torch.equal(a, b)
