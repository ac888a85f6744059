"""GPU tests of scan-batched fitting with the NPM baseline's DeepSDF decoders (nphm_mlp_fit_surface_grad_batched,
BatchedNpmIdentityFitter, BatchedNpmJointFitter and the two *_batched fitting functions): every scan of a batch gets what the
single-scan native path gives it, and the reference's trajectory stays within its bounds as one scan of three."""
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
    """A small stack of odd widths (37 -> 75 x 3 -> 1) with its zero level set through the points."""
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(31)
    dec = DeepSDF(lat_dim=37, hidden_dim=75, nlayers=4, geometric_init=True).to(dev)
    with torch.no_grad():
        s = dec(torch.zeros(1, 1, 3, device=dev), torch.zeros(1, 1, 37, device=dev))[0]
        dec.lin4.bias.sub_(s.reshape(-1))
        dec.lin4.weight.mul_(20.0); dec.lin4.bias.mul_(20.0)
    return dec


def _cloud(seed, n, dev):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.05, -0.1])).to(dev)


def _codes(seed, shape, dev, scale=0.01):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dev)


def _batched_call(eng, pts, cond, mask, clamp, ws):
    return [t.clone() for t in eng.fit_surface_grad_batched(pts, cond, mask, clamp, workspace=ws)]


@pytest.mark.parametrize('stack,sizes', [('npm', [5000, 5000, 3500, 5000]), ('odd', [333, 250, 333])])
def test_batched_surface_grad_matches_single_calls(cuda_device, stack, sizes):
    """nphm_mlp_fit_surface_grad_batched against one nphm_mlp_fit_surface_grad call per scan (n_queries = 1): kept counts
    equal, losses within 1e-6, gradients within 1e-5 of their max abs, padded rows exactly 0.  A scan with nothing kept gets a
    NaN loss and exactly zero gradients and leaves the other scans bitwise unchanged.  S = 1 agrees with the single call."""
    from nphm_b200.models.fitting import _pad_scans
    dec = _npm_decoders(cuda_device)[0] if stack == 'npm' else _odd_decoder(cuda_device)
    eng = dec.engine()
    S, D = len(sizes), dec.lat_dim
    pts_list = [_cloud(40 + k, nk, cuda_device) for k, nk in enumerate(sizes)]
    torch.manual_seed(5)
    masks = [(torch.rand(nk, device=cuda_device) > 0.15).to(torch.uint8) for nk in sizes]
    pts, pad = _pad_scans(pts_list)
    n = pts.shape[1]
    assert pad is not None
    mask = torch.stack([torch.cat([m, torch.zeros(n - m.numel(), dtype=torch.uint8, device=cuda_device)]) for m in masks])
    cond = _codes(6, (S, D), cuda_device)
    ws = eng.fit_workspace(S, n, cuda_device)
    for clamp in (0.1, 0.02):
        terms, g_cond, g_xyz = _batched_call(eng, pts, cond, mask, clamp, ws)
        for k, nk in enumerate(sizes):
            t1, gc1, gx1 = eng.fit_surface_grad(pts_list[k][None], cond[k:k + 1], masks[k][None], clamp)
            a, b = t1.cpu().numpy(), terms[k].cpu().numpy()
            assert int(a[5]) == int(b[5]) > 20 and abs(a[0] - b[0]) < 1e-6, (k, clamp, a, b)
            assert np.array_equal(a[1:5], b[1:5])
            gc, gcb = gc1[0].cpu().numpy(), g_cond[k].cpu().numpy()
            assert np.abs(gc - gcb).max() <= 1e-5 * np.abs(gc).max(), (k, clamp, _rel(gcb, gc))
            gx, gxb = gx1[0].cpu().numpy(), g_xyz[k, :nk].cpu().numpy()
            assert np.abs(gx - gxb).max() <= 1e-5 * np.abs(gx).max(), (k, clamp, _rel(gxb, gx))
            if nk < n:
                assert float(g_xyz[k, nk:].abs().max()) == 0.0
    # scan 1 with nothing kept: NaN loss, exactly zero gradients; the other scans as before, bit for bit
    terms, g_cond, g_xyz = _batched_call(eng, pts, cond, mask, 0.1, ws)
    mask2 = mask.clone()
    mask2[1] = 0
    t2, gc2, gx2 = _batched_call(eng, pts, cond, mask2, 0.1, ws)
    assert torch.isnan(t2[1, 0]) and float(t2[1, 5]) == 0.0
    assert float(gc2[1].abs().max()) == 0.0 and float(gx2[1].abs().max()) == 0.0
    others = [k for k in range(S) if k != 1]
    for a, b in ((terms, t2), (g_cond, gc2), (g_xyz, gx2)):
        assert torch.equal(a[others], b[others])
    # S = 1
    ws1 = eng.fit_workspace(1, sizes[0], cuda_device)
    t1, gc1, gx1 = eng.fit_surface_grad(pts_list[0][None], cond[:1], masks[0][None], 0.1)
    tb, gcb, gxb = _batched_call(eng, pts_list[0][None], cond[:1], masks[0][None], 0.1, ws1)
    assert torch.equal(t1, tb[0])
    assert float((gc1 - gcb).abs().max()) <= 1e-5 * float(gc1.abs().max())
    assert float((gx1 - gxb).abs().max()) <= 1e-5 * float(gx1.abs().max())


def test_batched_npm_identity_step_matches_single_scan_steps(cuda_device):
    from nphm_b200.models.fitting import BatchedNpmIdentityFitter, NpmIdentityFitter
    dec, _ = _npm_decoders(cuda_device)
    pts = [_cloud(20 + k, 3500 if k == 2 else 5000, cuda_device) for k in range(4)]
    z0 = _codes(3, (4, 512), cuda_device, 0.05)
    lam = dict(C.LAMBDAS_IDENTITY)
    clamp, lr = 0.1, 0.01
    torch.manual_seed(1)
    m0 = torch.rand_like(z0) * 1e-4
    v0 = torch.rand_like(z0) * 1e-7
    bf = BatchedNpmIdentityFitter(dec, 4, cuda_device)
    bf.latents.copy_(z0)
    bf.step(pts, lam, clamp, lr, apply_update=False)
    assert torch.equal(bf.latents, z0) and bf.t == 0
    single = NpmIdentityFitter(dec, cuda_device)
    for k in range(4):
        single.latent.copy_(z0[k])
        single.step(pts[k], lam, clamp, lr, apply_update=False)
        lt, blt = single.loss_terms.cpu().numpy(), bf.loss_terms[k].cpu().numpy()
        assert int(lt[5]) == int(blt[5]) > 100, k
        assert np.abs(lt[:5] - blt[:5]).max() < 1e-6, (k, lt, blt)
        g, bg = single.grad.cpu().numpy(), bf.grad[k].cpu().numpy()
        assert np.abs(g - bg).max() < 1e-5 * np.abs(g).max(), (k, _rel(bg, g))
    # the update from one (z, m, v, t) state
    bf.latents.copy_(z0); bf.m.copy_(m0); bf.v.copy_(v0); bf.t = 3
    bf.step(pts, lam, clamp, lr, apply_update=True)
    for k in range(4):
        single.latent.copy_(z0[k]); single.m.copy_(m0[k]); single.v.copy_(v0[k]); single.t = 3
        single.step(pts[k], lam, clamp, lr, apply_update=True)
        close = (bf.latents[k] - single.latent).abs() < 1e-5
        assert float(close.float().mean()) > 0.985, k


def _replay(n_iter, lambdas):
    """The schedule of the reference's iterations (tests/golden/fit_npm.npz) from its seeds: the golden scan then draws from
    the global generator as the reference did."""
    from nphm_b200.models.fitting import _apply_schedule, _clamp_for_iteration
    np.random.seed(0)
    torch.manual_seed(0)
    lr = 0.01
    for j in range(n_iter):
        lr = _apply_schedule(j, C.STEP_SCALE, C.SCHEDULE, lambdas, lr)
        yield j, _clamp_for_iteration(j, C.STEP_SCALE), lr


def test_batched_npm_identity_keeps_the_reference_trajectory_scan_separate(cuda_device):
    """The reference's NPM identity trajectory as scan 1 of 3: its gradients stay within the single-scan test's 2e-3."""
    from nphm_b200.models.fitting import BatchedNpmIdentityFitter, _sample_observations
    g = load_golden('fit_npm.npz')
    dec, _ = _npm_decoders(cuda_device)
    all_obs = [torch.from_numpy(o).to(cuda_device) for o in g['obs']]
    bf = BatchedNpmIdentityFitter(dec, 3, cuda_device)
    others = _codes(11, (2, 512), cuda_device, 0.05)
    lambdas = dict(C.LAMBDAS_IDENTITY)
    for j, clamp, lr in _replay(C.N_ITER_IDENTITY, lambdas):
        obs, _ = _sample_observations(all_obs)
        bf.latents[0].copy_(others[0]); bf.latents[2].copy_(others[1])
        bf.latents[1].copy_(torch.from_numpy(g['id_z_before'][j]))
        bf.step([_cloud(j, 700, cuda_device), obs, _cloud(100 + j, 1000, cuda_device)], lambdas, clamp, lr, apply_update=False)
        err = _rel(bf.grad[1].cpu().numpy(), g['id_grads'][j])
        print('identity iteration %d: %d kept, rel err of d loss/d z %.3g' % (j, int(bf.loss_terms[1, 5]), err))
        assert err < 2e-3, (j, err)


def _joint_subjects(dev):
    g = load_golden('fit_npm.npz')
    golden = [torch.from_numpy(o).to(dev) for o in g['obs']]
    shifted = [o * 1.03 + 0.01 for o in golden]
    short = [o[:150] for o in golden[:2]]                   # fewer observations, fewer points each
    return g, [golden, shifted, short]


def test_batched_npm_joint_gradients_match_single_subject_fitter(cuda_device):
    """BatchedNpmJointFitter against NpmJointFitter per subject (relative gradient error < 1e-4); the golden subject (subject 0)
    against the reference's gradients within the single-subject test's 2e-3 (z_id) and 3e-2 (z_ex)."""
    from nphm_b200.models.fitting import BatchedNpmJointFitter, NpmJointFitter, _sample_observations
    g, subjects = _joint_subjects(cuda_device)
    dec, expr = _npm_decoders(cuda_device)
    S = len(subjects)
    bj = BatchedNpmJointFitter(dec, expr, [len(s) for s in subjects], cuda_device)
    singles = [NpmJointFitter(dec, expr, len(s), cuda_device) for s in subjects]
    lambdas = dict(C.LAMBDAS_JOINT)
    other = torch.Generator().manual_seed(1)
    for j, clamp, lr in _replay(C.N_ITER_JOINT, lambdas):
        samples = [_sample_observations(s, None if k == 0 else other) for k, s in enumerate(subjects)]
        z_id = [torch.from_numpy(g['joint_z_id_before'][j]).to(cuda_device), _codes(30 + j, (512,), cuda_device, 0.05),
                _codes(40 + j, (512,), cuda_device, 0.05)]
        z_ex = [torch.from_numpy(g['joint_z_ex_before'][j]).to(cuda_device), _codes(50 + j, (len(subjects[1]), 200), cuda_device, 0.05),
                _codes(60 + j, (len(subjects[2]), 200), cuda_device, 0.05)]
        bj.z_id.copy_(torch.stack(z_id))
        bj.z_ex.copy_(torch.cat(z_ex))
        g_id, g_ex = bj.step([o for o, _ in samples], [i.long().to(cuda_device) for _, i in samples], lambdas, clamp, lr,
                             apply_update=False)
        for k in range(S):
            jf = singles[k]
            jf.z_id.copy_(z_id[k]); jf.z_ex.copy_(z_ex[k])
            obs, idx = samples[k]
            s_id, s_ex = jf.step(obs, idx.long().to(cuda_device), lambdas, clamp, lr, apply_update=False)
            assert int(jf.loss_terms[5]) == int(bj.loss_terms[k, 5]) > 0, (j, k)
            e_id = float((g_id[k] - s_id).abs().max() / s_id.abs().max())
            e_ex = float((g_ex[k] - s_ex).abs().max() / s_ex.abs().max())
            print('joint iteration %d subject %d: batched vs single rel err z_id %.3g z_ex %.3g' % (j, k, e_id, e_ex))
            assert e_id < 1e-4 and e_ex < 1e-4, (j, k, e_id, e_ex)
        e_id, e_ex = _rel(g_id[0].cpu().numpy(), g['joint_grads_id'][j]), _rel(g_ex[0].cpu().numpy(), g['joint_grads_ex'][j])
        print('joint iteration %d golden subject: rel err vs reference z_id %.3g z_ex %.3g' % (j, e_id, e_ex))
        assert e_id < 2e-3 and e_ex < 3e-2, (j, e_id, e_ex)


def _identity_scans(dev):
    g = load_golden('fit_npm.npz')
    obs = [torch.from_numpy(o).to(dev) for o in g['obs']]
    return [obs, [o * 1.02 for o in obs], [o[:150] + 0.01 for o in obs]]


def test_npm_identity_space_batched_equals_sequential_calls(cuda_device, monkeypatch):
    from nphm_b200.models import fitting
    dec, _ = _npm_decoders(cuda_device)
    scans = _identity_scans(cuda_device)
    n_steps = C.N_ITER_IDENTITY * 100
    torch.manual_seed(0)
    seq = [fitting.inference_identity_space(dec, s, dict(C.LAMBDAS_IDENTITY), n_steps, C.SCHEDULE, step_scale=C.STEP_SCALE)
           for s in scans]
    state_seq = torch.get_rng_state()
    one = dict(C.LAMBDAS_IDENTITY)
    fitting.inference_identity_space(dec, scans[0], one, n_steps, C.SCHEDULE, step_scale=C.STEP_SCALE)
    torch.manual_seed(0)
    lam = dict(C.LAMBDAS_IDENTITY)
    made = []
    real = fitting.BatchedNpmIdentityFitter

    def spy(*args, **kwargs):
        made.append(real(*args, **kwargs))
        return made[-1]
    monkeypatch.setattr(fitting, 'BatchedNpmIdentityFitter', spy)
    bat = fitting.inference_identity_space_batched(dec, scans, lam, n_steps, C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert len(made) == 1 and made[0].t == int(n_steps * C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state_seq)
    assert lam == one != C.LAMBDAS_IDENTITY
    for k, ((z1, a1), (z2, a2)) in enumerate(zip(seq, bat)):
        assert a1 is None and a2 is None and z2.shape == (1, 1, 512) and z2.requires_grad
        z1, z2 = z1.detach().cpu().numpy().reshape(-1), z2.detach().cpu().numpy().reshape(-1)
        close = np.abs(z1 - z2) < 2e-5
        print('NPM identity scan %d: batched vs sequential %.4f of the entries within 2e-5, max diff %.3g'
              % (k, close.mean(), np.abs(z1 - z2).max()))
        assert close.mean() > 0.93, k


def test_npm_joint_batched_equals_sequential_calls(cuda_device, monkeypatch):
    from nphm_b200.models import fitting
    monkeypatch.delenv('NPHM_JOINT_AUTOGRAD', raising=False)
    _, subjects = _joint_subjects(cuda_device)
    dec, expr = _npm_decoders(cuda_device)
    n_steps = C.N_ITER_JOINT * 100
    torch.manual_seed(0)
    seq = [fitting.inference_iterative_root_finding_joint(dec, expr, s, dict(C.LAMBDAS_JOINT), n_steps, C.SCHEDULE,
                                                          step_scale=C.STEP_SCALE) for s in subjects]
    state_seq = torch.get_rng_state()
    one = dict(C.LAMBDAS_JOINT)
    fitting.inference_iterative_root_finding_joint(dec, expr, subjects[0], one, n_steps, C.SCHEDULE, step_scale=C.STEP_SCALE)
    torch.manual_seed(0)
    lam = dict(C.LAMBDAS_JOINT)
    made = []
    real = fitting.BatchedNpmJointFitter

    def spy(*args, **kwargs):
        made.append(real(*args, **kwargs))
        return made[-1]
    monkeypatch.setattr(fitting, 'BatchedNpmJointFitter', spy)
    bat = fitting.inference_iterative_root_finding_joint_batched(dec, expr, subjects, lam, n_steps, C.SCHEDULE,
                                                                 step_scale=C.STEP_SCALE)
    assert len(made) == 1 and made[0].t == int(n_steps * C.STEP_SCALE)
    assert torch.equal(torch.get_rng_state(), state_seq)
    assert lam == one != C.LAMBDAS_JOINT
    for k, ((e1, i1, a1), (e2, i2, a2)) in enumerate(zip(seq, bat)):
        assert a1 is None and a2 is None
        assert e1.shape == e2.shape == (len(subjects[k]), 1, 200) and i1.shape == i2.shape == (1, 1, 512)
        ci = (np.abs(i1.detach().cpu().numpy() - i2.detach().cpu().numpy()) < 5e-4).mean()
        ce = (np.abs(e1.detach().cpu().numpy() - e2.detach().cpu().numpy()) < 5e-4).mean()
        print('NPM joint subject %d: batched vs sequential %.4f of z_id, %.4f of z_ex within 5e-4' % (k, ci, ce))
        assert ci > 0.9 and ce > 0.9, k


def test_batched_npm_steps_do_not_synchronise_with_the_host(cuda_device):
    from nphm_b200.models.fitting import BatchedNpmIdentityFitter, BatchedNpmJointFitter, _sample_observations
    dec, expr = _npm_decoders(cuda_device)
    pts = [_cloud(20 + k, 3500 if k == 2 else 5000, cuda_device) for k in range(4)]
    lam = dict(C.LAMBDAS_IDENTITY)
    bf = BatchedNpmIdentityFitter(dec, 4, cuda_device)
    bf.step(pts, lam, 0.1, 0.01)                            # first call: workspace allocation
    _, subjects = _joint_subjects(cuda_device)
    bj = BatchedNpmJointFitter(dec, expr, [len(s) for s in subjects], cuda_device)
    torch.manual_seed(0)
    samples = [_sample_observations(s) for s in subjects]
    obs, idx = [o for o, _ in samples], [i.long().to(cuda_device) for _, i in samples]
    bj.step(obs, idx, dict(C.LAMBDAS_JOINT), 0.1, 0.01)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bf.step(pts, lam, 0.1, 0.01)
        bj.step(obs, idx, dict(C.LAMBDAS_JOINT), 0.1, 0.01)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert torch.isfinite(bf.latents).all() and torch.isfinite(bj.z_id).all() and torch.isfinite(bj.z_ex).all()


def test_batched_surface_grad_rejects_bad_arguments(cuda_device):
    from nphm_b200 import _native
    dec, expr = _npm_decoders(cuda_device)
    eng = dec.engine()
    lib = _native.lib()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    S, n, D = 2, 700, dec.lat_dim
    pts = torch.stack([_cloud(1, n, cuda_device), _cloud(2, n, cuda_device)]).contiguous()
    cond = _codes(3, (S, D), cuda_device)
    terms = torch.empty(S, 8, device=cuda_device)
    g_cond = torch.empty(S, D, device=cuda_device)
    g_xyz = torch.empty_like(pts)
    need = lib.nphm_mlp_fit_workspace_bytes(eng._h, S, n)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_device)

    def call(p=pts.data_ptr(), c=cond.data_ptr(), s=S, nn=n, t=terms.data_ptr(), gc=g_cond.data_ptr(), w=ws.data_ptr(),
             nbytes=need, h=eng._h):
        return lib.nphm_mlp_fit_surface_grad_batched(h, p, c, None, s, nn, 0.1, t, gc, g_xyz.data_ptr(), w, nbytes, stream)
    assert call() == 0
    assert call(nbytes=need - 256) == -1 and call(nbytes=need + 256) == -1       # workspace of another shape
    assert call(nn=n - 100) == -1                                                 # the workspace is for (S, n)
    assert call(s=0) == -1 and call(nn=0) == -1
    for bad in ('p', 'c', 't', 'gc', 'w'):
        assert call(**{bad: None}) == -1, bad
    # a stack with three outputs: unsupported
    e3 = expr.engine()
    need3 = lib.nphm_mlp_fit_workspace_bytes(e3._h, S, n)
    ws3 = torch.empty(need3, dtype=torch.uint8, device=cuda_device)
    cond3 = torch.zeros(S, expr.lat_dim, device=cuda_device)
    g3 = torch.empty(S, expr.lat_dim, device=cuda_device)
    assert call(h=e3._h, c=cond3.data_ptr(), gc=g3.data_ptr(), w=ws3.data_ptr(), nbytes=need3) == -3
    torch.cuda.synchronize()
    with pytest.raises(_native.NativeError, match=r'\(-3\)'):
        e3.fit_surface_grad_batched(pts, cond3, None, 0.1)
