"""GPU tests of expression fitting with a fixed identity code (inference_expression_space and its batched form, the
fitters' fixed_identity mode, nphm_fit_surface_grad* without the identity-code gradient): per-step gradients against the
reference's own loop (fit_expression.npz) and the autograd mirror, trajectories, batched versus sequential calls, and a step
that reads nothing back from the device."""
import numpy as np
import pytest
import torch

import fit_expression_common as C
import npm_fit_common as N
from conftest import load_golden, make_deformation, make_ensemble, sample_latent

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _pair(which, dev, train=True):
    g = load_golden('fit_expression.npz')
    if which == 'nphm':
        dec, expr = make_ensemble(0, device=dev), make_deformation(dev)
    else:
        from nphm_b200.models.deepSDF import DeepSDF
        dec, expr = N.make_decoders(DeepSDF, dev)
    dec.train(train)
    scans, i = [], 0
    while '%s_scan%d' % (which, i) in g.files:
        scans.append(torch.from_numpy(g['%s_scan%d' % (which, i)]).to(dev))
        i += 1
    return g, dec, expr, scans, torch.from_numpy(g[which + '_z_id']).to(dev).reshape(1, 1, -1)


def _fixed_fitter(which, dec, expr, K, dev, z_id):
    from nphm_b200.models.fitting import JointFitter, NpmJointFitter
    f = (JointFitter if which == 'nphm' else NpmJointFitter)(dec, expr, K, dev, fixed_identity=True)
    f.z_id.copy_(z_id.reshape(-1))
    return f


def _replay(all_obs, lambdas):
    from nphm_b200.models.fitting import _apply_schedule, _clamp_for_iteration, _sample_observations
    np.random.seed(0)
    torch.manual_seed(0)
    lr = 0.01
    for j in range(C.N_ITER):
        lr = _apply_schedule(j, C.STEP_SCALE, C.SCHEDULE, lambdas, lr)
        obs, idx = _sample_observations(all_obs)
        yield j, obs, idx.long().to(all_obs[0].device), _clamp_for_iteration(j, C.STEP_SCALE), lr


@pytest.mark.parametrize('which', ['nphm', 'npm'])
def test_fixed_identity_gradients_match_reference(which, cuda_device):
    """The native fixed-identity step from the reference's own expression codes against the gradient it handed to Adam, with
    the z_ex tolerance of the joint fitters' tests (test_joint_fitter_gradients_match_reference_autograd gives the reasons)."""
    g, dec, expr, scans, z_id = _pair(which, cuda_device)
    f = _fixed_fitter(which, dec, expr, len(scans), cuda_device, z_id)
    lambdas = dict(C.LAMBDAS_JOINT)
    for j, obs, idx, clamp, lr in _replay(scans, lambdas):
        f.z_ex.copy_(torch.from_numpy(g[which + '_codes_before'][j]))
        g_id, g_ex = f.step(obs, idx, lambdas, clamp, lr, apply_update=False)
        assert g_id is None
        err = _rel(g_ex.cpu().numpy(), g[which + '_grads'][j])
        print('%s iteration %d: rel err of d loss/d z_ex %.3g' % (which, j, err))
        assert err < 3e-2, (j, err)


@pytest.mark.parametrize('which', ['nphm', 'npm'])
def test_expression_fit_follows_reference(which, cuda_device):
    """The public function on CUDA (native) against the reference's final codes; the identity code, the generator and the
    lambdas as the contract says."""
    from nphm_b200.models.fitting import inference_expression_space
    g, dec, expr, scans, z_id = _pair(which, cuda_device)
    z_before = z_id.clone()
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, anchors = inference_expression_space(dec, expr, z_id, scans, lambdas, C.N_ITER * 100, C.SCHEDULE,
                                               step_scale=C.STEP_SCALE)
    assert torch.equal(z_id, z_before)
    assert np.array_equal(torch.get_rng_state().numpy(), g[which + '_rng_after'])
    assert [lambdas[k] for k in sorted(lambdas)] == list(g[which + '_lambdas_final'])
    close = (np.abs(z_ex.detach().cpu().numpy().reshape(len(scans), -1) - g[which + '_z_ex_final']) < 5e-4).mean()
    print('%s: %.1f%% of z_ex within 5e-4 of the reference' % (which, 100 * close))
    assert close > 0.9
    if which == 'nphm':
        assert float(np.abs(anchors.cpu().numpy().reshape(-1, 3) - g['nphm_anchors']).max()) < 1e-5
    else:
        assert anchors is None


@pytest.mark.parametrize('which,train', [('nphm', True), ('nphm', False), ('npm', True), ('npm', False)])
def test_native_matches_mirror(which, train, cuda_device, monkeypatch):
    """Native versus the autograd mirror on the same device, in training and eval mode (the NPHM ensemble's eval mode has the
    last-point quirk rows): a short trajectory from a warm start, and the first step's gradient from the same codes."""
    from nphm_b200.models import fitting as F
    g, dec, expr, scans, z_id = _pair(which, cuda_device, train)
    torch.manual_seed(3)
    warm = torch.randn(len(scans), 1, g[which + '_z_ex_final'].shape[1], device=cuda_device) * 0.01
    runs = {}
    for mode in ('native', 'mirror'):
        if mode == 'mirror':
            monkeypatch.setenv('NPHM_JOINT_AUTOGRAD', '1')
        torch.manual_seed(0)
        runs[mode] = F.inference_expression_space(dec, expr, z_id, scans, dict(C.LAMBDAS_JOINT), 400, C.SCHEDULE,
                                                  step_scale=C.STEP_SCALE, lat_reps_expr_init=warm)[0]
        monkeypatch.delenv('NPHM_JOINT_AUTOGRAD', raising=False)
    close = (runs['native'] - runs['mirror']).abs().lt(5e-4).float().mean().item()
    print('%s train=%s: %.1f%% of z_ex within 5e-4 of the mirror' % (which, train, 100 * close))
    assert close > 0.9
    # the first step's gradient from the same codes: the mirror's is what its loop hands to Adam at iteration 0
    recorded = []
    real = torch.optim.Adam

    class RecordingAdam(real):
        def step(self, closure=None):
            recorded.append(self.param_groups[0]['params'][0].grad.detach().clone())
    monkeypatch.setattr(torch.optim, 'Adam', RecordingAdam)
    torch.manual_seed(0)
    F._inference_joint_autograd(dec, expr, scans, dict(C.LAMBDAS_JOINT), 100, C.SCHEDULE, C.STEP_SCALE, 1,
                                lat_rep_shape=z_id, lat_rep_init=warm)
    monkeypatch.setattr(torch.optim, 'Adam', real)
    f = _fixed_fitter(which, dec, expr, len(scans), cuda_device, z_id)
    f.z_ex.copy_(warm.reshape(len(scans), -1))
    _, obs, idx, clamp, lr = next(_replay(scans, dict(C.LAMBDAS_JOINT)))
    _, g_ex = f.step(obs, idx, dict(C.LAMBDAS_JOINT), clamp, lr, apply_update=False)
    [mirror] = recorded
    err = _rel(g_ex.cpu().numpy(), mirror.reshape(len(scans), -1).cpu().numpy())
    print('%s train=%s: rel err of the first step d loss/d z_ex against the mirror %.3g' % (which, train, err))
    assert err < 3e-2


def test_null_latent_surface_gradient_is_bitwise_the_full_call(cuda_device):
    """nphm_fit_surface_grad and its quirk, batched and batched-quirk forms with grad_latent_dev NULL: the loss terms and the
    point gradient are bitwise those of the call with a latent gradient, and two full calls agree bitwise too."""
    from nphm_b200 import _native
    from nphm_b200.models.fitting import _pad_scans
    dec = make_ensemble(0, device=cuda_device).train()
    eng = dec.engine()
    lib = _native.lib()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    gen = torch.Generator().manual_seed(8)
    clouds = [(torch.randn(n, 3, generator=gen) * 0.15 + torch.tensor([0.0, 0.05, -0.1])).to(cuda_device) for n in (5000, 3300, 4200)]
    z = torch.stack([sample_latent(s) for s in (3, 4, 5)]).to(cuda_device).contiguous()
    D = dec.lat_dim
    p1 = clouds[0].contiguous()
    m1 = (torch.rand(p1.shape[0], generator=gen) > 0.1).to(torch.uint8).to(cuda_device)

    def single(quirk, with_latent):
        terms, g_pts = torch.full((8,), -1.0, device=cuda_device), torch.empty_like(p1)
        g_lat = torch.empty(D, device=cuda_device) if with_latent else None
        if quirk:
            _native.check(lib.nphm_fit_surface_grad_quirk(eng.handle, p1.data_ptr(), p1.shape[0], 1000, z[0].data_ptr(),
                                                          m1.data_ptr(), 0.1, terms.data_ptr(), _native._ptr(g_lat),
                                                          g_pts.data_ptr(), None, stream))
        else:
            _native.check(lib.nphm_fit_surface_grad(eng.handle, p1.data_ptr(), p1.shape[0], z[0].data_ptr(), m1.data_ptr(), 0.1,
                                                    terms.data_ptr(), _native._ptr(g_lat), g_pts.data_ptr(), None, stream))
        return terms, g_pts, g_lat

    pts, mask = _pad_scans(clouds)
    S, n = pts.shape[0], pts.shape[1]
    ws = torch.empty(lib.nphm_fit_batch_workspace_bytes(eng.handle, S, n), dtype=torch.uint8, device=cuda_device)
    periods = torch.tensor([1000, 700, 600], dtype=torch.int32, device=cuda_device)

    def batched(quirk, with_latent):
        terms, g_pts = torch.full((S, 8), -1.0, device=cuda_device), torch.empty_like(pts)
        g_lat = torch.empty(S, D, device=cuda_device) if with_latent else None
        if quirk:
            _native.check(lib.nphm_fit_surface_grad_batched_quirk(eng.handle, pts.data_ptr(), mask.data_ptr(), S, n,
                                                                  periods.data_ptr(), z.data_ptr(), 0.1, terms.data_ptr(),
                                                                  _native._ptr(g_lat), g_pts.data_ptr(), ws.data_ptr(),
                                                                  ws.numel(), stream))
        else:
            _native.check(lib.nphm_fit_surface_grad_batched(eng.handle, pts.data_ptr(), mask.data_ptr(), S, n, z.data_ptr(), 0.1,
                                                            terms.data_ptr(), _native._ptr(g_lat), g_pts.data_ptr(),
                                                            ws.data_ptr(), ws.numel(), stream))
        return terms, g_pts, g_lat

    for name, call in (('single', single), ('batched', batched)):
        for quirk in (False, True):
            full, again, null = call(quirk, True), call(quirk, True), call(quirk, False)
            assert float(full[0][..., 5].min()) > 100 and float(full[1].abs().max()) > 0 and float(full[2].abs().max()) > 0
            for a, b in ((full, again), (full, null)):
                assert torch.equal(a[0], b[0]), (name, quirk)
                assert torch.equal(a[1], b[1]), (name, quirk)
    # the NULL mode with no point gradient either: the loss terms alone
    terms = torch.empty(8, device=cuda_device)
    _native.check(lib.nphm_fit_surface_grad(eng.handle, p1.data_ptr(), p1.shape[0], z[0].data_ptr(), m1.data_ptr(), 0.1,
                                            terms.data_ptr(), None, None, None, stream))
    assert torch.equal(terms, single(False, True)[0])


def _subjects(which, dev):
    """Three subjects with 1, 3 and 2 observations; subject 1 shorter than 1000 points per scan, subject 2 warm-started."""
    g, dec, expr, scans, z_id = _pair(which, dev)
    E = g[which + '_z_ex_final'].shape[1]
    torch.manual_seed(9)
    short = [s[:700] for s in scans[:3]] if scans[0].shape[0] > 1000 else scans[:3]
    subjects = [(z_id, scans[:1]), (z_id * 0.8, short), (z_id, scans[1:3], torch.randn(2, 1, E, device=dev) * 0.02)]
    return dec, expr, subjects


@pytest.mark.parametrize('which', ['nphm', 'npm'])
@pytest.mark.parametrize('S', [1, 3])
def test_batched_equals_sequential_calls(which, S, cuda_device):
    from nphm_b200.models.fitting import inference_expression_space, inference_expression_space_batched
    dec, expr, subjects = _subjects(which, cuda_device)
    subjects = subjects[-S:]
    lam0 = dict(C.LAMBDAS_JOINT)
    ids = [s[0].clone() for s in subjects]
    torch.manual_seed(0)
    seq = [inference_expression_space(dec, expr, s[0], s[1], dict(lam0), 400, C.SCHEDULE, step_scale=C.STEP_SCALE,
                                      lat_reps_expr_init=s[2] if len(s) > 2 else None) for s in subjects]
    state = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lam0)
    bat = inference_expression_space_batched(dec, expr, subjects, lam, 400, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state)
    one = dict(lam0)
    torch.manual_seed(0)
    inference_expression_space(dec, expr, subjects[0][0], subjects[0][1], one, 400, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert lam == one
    assert all(torch.equal(a, s[0]) for a, s in zip(ids, subjects))
    for k, ((e1, a1), (e2, a2)) in enumerate(zip(seq, bat)):
        assert e1.shape == e2.shape and e2.requires_grad
        close = (e1 - e2).abs().lt(5e-4).float().mean().item()
        print('%s S=%d subject %d: %.1f%% of z_ex within 5e-4 of the sequential call' % (which, S, k, 100 * close))
        assert close > 0.9, k
        assert (a1 is None) == (a2 is None) and (a1 is None or float((a1 - a2).abs().max()) < 1e-5)


def _log_native_calls(monkeypatch):
    from nphm_b200 import _native
    L = _native.lib()
    log = []
    for name in _native.EXPORTED_SYMBOLS:
        fn = getattr(L, name)

        def wrapped(*args, _fn=fn, _name=name):
            log.append((_name, args))
            return _fn(*args)
        monkeypatch.setattr(L, name, wrapped)
    return log


@pytest.mark.parametrize('which', ['nphm', 'npm'])
@pytest.mark.parametrize('batched', [False, True])
def test_fixed_identity_step_reads_nothing_back(which, batched, cuda_device, monkeypatch):
    """A fixed-identity step, single or batched, is a pure launch sequence: no synchronising torch call, no stream
    synchronisation, no identity update (nphm_fit_apply_gradient*), no anchor recomputation, and the ensemble's surface call
    goes without the latent gradient."""
    from nphm_b200.models import fitting as F
    g, dec, expr, scans, z_id = _pair(which, cuda_device)
    if batched:
        cls = F.BatchedJointFitter if which == 'nphm' else F.BatchedNpmJointFitter
        f = cls(dec, expr, [2, 2], cuda_device, fixed_identity=True)
        f.z_id.copy_(z_id.reshape(1, -1).expand(2, -1))
        subjects = [scans[:2], scans[1:3]]
    else:
        f = _fixed_fitter(which, dec, expr, len(scans), cuda_device, z_id)

    def sample():
        if batched:
            s = [F._sample_observations(a) for a in subjects]
            return [o for o, _ in s], [i.long().to(cuda_device) for _, i in s]
        o, i = F._sample_observations(scans)
        return o, i.long().to(cuda_device)
    torch.manual_seed(0)
    f.step(*sample(), dict(C.LAMBDAS_JOINT), 0.1, 0.01)            # warm-up: workspaces, anchors, compressor row
    obs, idx = sample()
    syncs = []
    for owner in (torch.cuda, torch.cuda.Stream):
        real = owner.synchronize
        monkeypatch.setattr(owner, 'synchronize', lambda *a, _r=real, **k: (syncs.append(1), _r(*a, **k))[1])
    log = _log_native_calls(monkeypatch)
    torch.cuda.current_stream().synchronize()
    del syncs[:]
    torch.cuda.set_sync_debug_mode('error')
    try:
        f.step(obs, idx, dict(C.LAMBDAS_JOINT), 0.1, 0.01)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    names = [n for n, _ in log]
    print('%s batched=%s: native calls %s, stream synchronisations %d' % (which, batched, names, len(syncs)))
    assert len(syncs) == 0
    assert not any(n.startswith('nphm_fit_apply_gradient') or n == 'nphm_ensemble_anchors' for n in names)
    assert names.count('nphm_adam_step') == 1
    if which == 'nphm':
        [(_, args)] = [(n, a) for n, a in log if n.startswith('nphm_fit_surface_grad')]
        assert args[-5 if batched else -4] is None                  # grad_latent_dev
    torch.cuda.synchronize()
    z_rows = f.z_id.reshape(-1, z_id.numel())
    assert torch.isfinite(f.z_ex).all() and torch.equal(z_rows, z_id.reshape(1, -1).expand_as(z_rows))
