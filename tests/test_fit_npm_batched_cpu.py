"""CPU tests of scan-batched fitting with DeepSDF decoders (the NPM baseline): on CPU the batched fitting functions fit the scans
one after another on the composite path, and equal sequential calls of the single-scan functions bitwise, with the same
global-generator state and the same ``lambdas``."""
import torch

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SCHEDULE = {'lr': {100: 2}, 'reg_glob': {100: 3}, 'reg_expr': {100: 10}}


def _decoders():
    """A small identity DeepSDF (13 -> 32 x 3 -> 1) and expression DeepSDF ([13 | 200] -> 256 x 3 -> 3, output scaled down)."""
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(3)
    dec = DeepSDF(lat_dim=13, hidden_dim=32, nlayers=4, geometric_init=True)
    expr = DeepSDF(lat_dim=13 + 200, hidden_dim=256, nlayers=4, out_dim=3)
    with torch.no_grad():
        expr.lin4.weight.mul_(0.02)
        expr.lin4.bias.mul_(0.02)
    return dec.train(), expr.eval()


def _scans():
    g = torch.Generator().manual_seed(8)
    base = [torch.randn(300, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.05, -0.1]) for _ in range(3)]
    return [base, [o[:120] * 1.02 for o in base], [o + 0.01 for o in base[:2]]]


def test_npm_identity_space_batched_on_cpu_equals_sequential_calls():
    from nphm_b200.models.fitting import inference_identity_space, inference_identity_space_batched
    dec, _ = _decoders()
    lambdas = {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
    scans = _scans()
    torch.manual_seed(0)
    seq = [inference_identity_space(dec, s, dict(lambdas), 200, SCHEDULE, step_scale=0.01) for s in scans]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lambdas)
    bat = inference_identity_space_batched(dec, scans, lam, 200, SCHEDULE, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    one = dict(lambdas)
    inference_identity_space(dec, scans[0], one, 200, SCHEDULE, step_scale=0.01)
    assert lam == one and lam != lambdas
    assert len(bat) == len(scans)
    for (z1, a1), (z2, a2) in zip(seq, bat):
        assert a1 is None and a2 is None and torch.equal(z1, z2)


def test_npm_joint_batched_on_cpu_equals_sequential_calls():
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint, inference_iterative_root_finding_joint_batched
    dec, expr = _decoders()
    subjects = [[o[:100] for o in s] for s in _scans()]
    torch.manual_seed(0)
    seq = [inference_iterative_root_finding_joint(dec, expr, s, dict(LAMBDAS), 200, SCHEDULE, step_scale=0.01) for s in subjects]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(LAMBDAS)
    bat = inference_iterative_root_finding_joint_batched(dec, expr, subjects, lam, 200, SCHEDULE, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    one = dict(LAMBDAS)
    inference_iterative_root_finding_joint(dec, expr, subjects[0], one, 200, SCHEDULE, step_scale=0.01)
    assert lam == one and lam['reg_expr'] == LAMBDAS['reg_expr'] / 10
    assert len(bat) == len(subjects)
    for (e1, i1, a1), (e2, i2, a2) in zip(seq, bat):
        assert a1 is None and a2 is None and torch.equal(e1, e2) and torch.equal(i1, i2)
