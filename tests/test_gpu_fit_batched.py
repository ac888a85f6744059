"""GPU tests of scan-batched fitting (nphm_fit_*_batched, BatchedIdentityFitter, BatchedJointFitter and the two
*_batched fitting functions): every scan of a batch gets what the single-scan path gives it."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden, make_deformation, make_ensemble, mean_anchors, sample_latent
from fit_common import golden_fit_setup, replay_iterations

pytestmark = pytest.mark.gpu

JOINT_LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
JOINT_SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999},
                  'reg_glob': {200: 3, 600: 10}, 'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}


def _rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def _cloud(seed, n, dev):
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(n, 3, generator=g) * 0.15 + torch.tensor([0.0, 0.05, -0.1])
    return pts.to(dev)


def _scan_points(dev):
    """Four scans of different point clouds; scan 2 is shorter and padded."""
    return [_cloud(20 + k, 3500 if k == 2 else 5000, dev) for k in range(4)]


def _latents(seeds, dev):
    return torch.stack([sample_latent(s) for s in seeds]).to(dev).contiguous()


def test_batched_identity_step_matches_single_scan_steps(cuda_device):
    from nphm_b200.models.fitting import BatchedIdentityFitter, IdentityFitter
    dec = make_ensemble(0, device=cuda_device).train()
    pts = _scan_points(cuda_device)
    z0 = _latents([3, 4, 5, 6], cuda_device) * 0.3
    lam = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    clamp, lr = 0.1, 0.01
    torch.manual_seed(1)
    m0 = torch.rand_like(z0) * 1e-4
    v0 = torch.rand_like(z0) * 1e-7
    bf = BatchedIdentityFitter(dec, 4, cuda_device)
    bf.latents.copy_(z0)
    bf.step(pts, lam, clamp, lr, apply_update=False)
    single = IdentityFitter(dec, cuda_device)
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


def test_batched_surface_grad_matches_single_calls(cuda_device):
    from nphm_b200 import _native
    from nphm_b200.models.fitting import _pad_scans
    dec = make_ensemble(0, device=cuda_device).train()
    eng = dec.engine()
    lib = _native.lib()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    pts_list = _scan_points(cuda_device)[:3]
    S, D = 3, dec.lat_dim
    torch.manual_seed(2)
    masks = [(torch.rand(p.shape[0], device=cuda_device) > 0.2).to(torch.uint8) for p in pts_list]
    pts, pad = _pad_scans(pts_list)
    n = pts.shape[1]
    mask = torch.stack([torch.cat([m, torch.zeros(n - m.numel(), dtype=torch.uint8, device=cuda_device)]) for m in masks])
    assert pad is not None and torch.equal(mask.bool() & pad.bool(), mask.bool())
    z = _latents([7, 8, 9], cuda_device)
    for clamp in (0.1, 0.02):
        terms = torch.empty(S, 8, device=cuda_device)
        g_lat = torch.empty(S, D, device=cuda_device)
        g_pts = torch.empty_like(pts)
        ws = torch.empty(lib.nphm_fit_batch_workspace_bytes(eng.handle, S, n), dtype=torch.uint8, device=cuda_device)
        _native.check(lib.nphm_fit_surface_grad_batched(eng.handle, pts.data_ptr(), mask.data_ptr(), S, n, z.data_ptr(),
                                                        clamp, terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(),
                                                        ws.data_ptr(), ws.numel(), stream))
        for k in range(S):
            nk = pts_list[k].shape[0]
            p1 = pts_list[k].contiguous()
            t1 = torch.empty(8, device=cuda_device)
            gl1 = torch.empty(D, device=cuda_device)
            gp1 = torch.empty_like(p1)
            _native.check(lib.nphm_fit_surface_grad(eng.handle, p1.data_ptr(), nk, z[k].data_ptr(), masks[k].data_ptr(), clamp,
                                                    t1.data_ptr(), gl1.data_ptr(), gp1.data_ptr(), None, stream))
            a, b = t1.cpu().numpy(), terms[k].cpu().numpy()
            assert int(a[5]) == int(b[5]) > 20 and abs(a[0] - b[0]) < 1e-6, (k, clamp, a, b)
            gl, gb = gl1.cpu().numpy(), g_lat[k].cpu().numpy()
            assert np.abs(gl - gb).max() < 1e-5 * np.abs(gl).max(), (k, clamp)
            gp, gpb = gp1.cpu().numpy(), g_pts[k, :nk].cpu().numpy()
            assert np.abs(gp - gpb).max() < 1e-5 * np.abs(gp).max(), (k, clamp)
            assert float(g_pts[k, nk:].abs().max()) == 0.0 if nk < n else True
    # a scan with nothing kept: NaN loss and zero gradients for it, the others unaffected
    mask2 = mask.clone()
    mask2[1] = 0
    _native.check(lib.nphm_fit_surface_grad_batched(eng.handle, pts.data_ptr(), mask2.data_ptr(), S, n, z.data_ptr(), 0.1,
                                                    terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(),
                                                    ws.numel(), stream))
    assert torch.isnan(terms[1, 0]) and float(g_lat[1].abs().max()) == 0.0 and float(g_pts[1].abs().max()) == 0.0
    assert not torch.isnan(terms[0, 0]) and float(g_lat[0].abs().max()) > 0


def test_batched_step_keeps_the_reference_trajectory_scan_separate(cuda_device):
    """The reference's identity trajectory as scan 1 of 3: its gradients stay at the bound of the single-scan test."""
    from nphm_b200.models.fitting import BatchedIdentityFitter
    g, _, _, _ = golden_fit_setup()
    dec = make_ensemble(0, device=cuda_device).train()
    bf = BatchedIdentityFitter(dec, 3, cuda_device)
    others = _latents([11, 12], cuda_device)
    for j, pts, lam, clamp, lr in replay_iterations(12):
        bf.latents[0].copy_(others[0]); bf.latents[2].copy_(others[1])
        bf.latents[1].copy_(torch.from_numpy(g['z_before'][j]))
        p = torch.from_numpy(pts).to(cuda_device)
        bf.step([_cloud(j, 4000, cuda_device), p, _cloud(100 + j, 5000, cuda_device)], lam, clamp, lr, apply_update=False)
        err = _rel(bf.grad[1].cpu().numpy(), g['grads'][j])
        assert err < 2e-4, (j, err)


def _joint_subjects(dev):
    g = load_golden('fit_joint.npz')
    golden = [torch.from_numpy(o).to(dev) for o in g['obs']]
    shifted = [o * 1.03 + 0.01 for o in golden]
    short = [o[:600] for o in golden[:2]]                   # fewer observations, fewer points each
    return g, [golden, shifted, short]


def test_batched_joint_gradients_match_single_subject_fitter(cuda_device):
    from nphm_b200.models.fitting import (BatchedJointFitter, JointFitter, _apply_schedule, _clamp_for_iteration,
                                          _sample_observations)
    g, subjects = _joint_subjects(cuda_device)
    dec = make_ensemble(0, device=cuda_device).train()
    dfn = make_deformation(cuda_device)
    S = len(subjects)
    bj = BatchedJointFitter(dec, dfn, [len(s) for s in subjects], cuda_device)
    lambdas = dict(JOINT_LAMBDAS)
    others = [(sample_latent(30 + j).to(cuda_device) * 0.3, sample_latent(40 + j).to(cuda_device) * 0.3) for j in range(3)]
    other = torch.Generator().manual_seed(1)
    dgen = torch.Generator(device=cuda_device).manual_seed(2)
    torch.manual_seed(0)
    lr = 0.01
    for j in range(3):
        lr = _apply_schedule(j, 0.01, JOINT_SCHEDULE, lambdas, lr)
        # the golden subject draws from the global generator as the reference's run did; the others from their own
        samples = [_sample_observations(s, None if k == 0 else other) for k, s in enumerate(subjects)]
        z_id = [torch.from_numpy(g['z_id_before'][j]).to(cuda_device), others[j][0], others[j][1]]
        z_ex = [torch.from_numpy(g['z_ex_before'][j]).to(cuda_device),
                torch.randn(len(subjects[1]), 200, device=cuda_device, generator=dgen) * 0.05,
                torch.randn(len(subjects[2]), 200, device=cuda_device, generator=dgen) * 0.05]
        bj.z_id.copy_(torch.stack(z_id))
        bj.z_ex.copy_(torch.cat(z_ex))
        clamp = _clamp_for_iteration(j, 0.01)
        g_id, g_ex = bj.step([o for o, _ in samples], [i.long().to(cuda_device) for _, i in samples], lambdas, clamp, lr,
                             apply_update=False)
        for k in range(S):
            jf = JointFitter(dec, dfn, len(subjects[k]), cuda_device)
            jf.z_id.copy_(z_id[k]); jf.z_ex.copy_(z_ex[k])
            obs, idx = samples[k]
            s_id, s_ex = jf.step(obs, idx.long().to(cuda_device), lambdas, clamp, lr, apply_update=False)
            e_id = float((g_id[k] - s_id).abs().max() / s_id.abs().max())
            e_ex = float((g_ex[k] - s_ex).abs().max() / s_ex.abs().max())
            print('joint iteration %d subject %d: batched vs single rel err z_id %.3g z_ex %.3g' % (j, k, e_id, e_ex))
            assert e_id < 1e-4 and e_ex < 1e-4, (j, k, e_id, e_ex)
        e_id, e_ex = _rel(g_id[0].cpu().numpy(), g['grads_id'][j]), _rel(g_ex[0].cpu().numpy(), g['grads_ex'][j])
        assert e_id < 2e-3 and e_ex < 3e-2, (j, e_id, e_ex)


def _identity_scans(dev):
    _, obs, _, _ = golden_fit_setup()
    obs = [o.to(dev) for o in obs]
    return [obs, [o * 1.02 for o in obs], [o[:700] + 0.01 for o in obs]]


def test_identity_space_batched_equals_sequential_calls(cuda_device):
    from nphm_b200.models.fitting import inference_identity_space, inference_identity_space_batched
    _, _, lambdas, schedule = golden_fit_setup()
    dec = make_ensemble(0, device=cuda_device).train()
    scans = _identity_scans(cuda_device)
    torch.manual_seed(0)
    seq = [inference_identity_space(dec, s, dict(lambdas), 1200, schedule, step_scale=0.01) for s in scans]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(lambdas)
    bat = inference_identity_space_batched(dec, scans, lam, 1200, schedule, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    one = dict(lambdas)
    torch.manual_seed(0)
    inference_identity_space(dec, scans[0], one, 1200, schedule, step_scale=0.01)
    assert lam == one
    for k, ((z1, a1), (z2, a2)) in enumerate(zip(seq, bat)):
        z1, z2 = z1.detach().cpu().numpy().reshape(-1), z2.detach().cpu().numpy().reshape(-1)
        close = np.abs(z1 - z2) < 2e-5
        print('identity scan %d: batched vs sequential %.4f of the entries within 2e-5, max diff %.3g'
              % (k, close.mean(), np.abs(z1 - z2).max()))
        assert close.mean() > 0.93, k
        assert float((a1 - a2).abs().max()) < 1e-5, k
    # S = 1 is the single-scan function
    torch.manual_seed(0)
    z1, a1 = inference_identity_space(dec, scans[2], dict(lambdas), 1200, schedule, step_scale=0.01)
    torch.manual_seed(0)
    [(z2, a2)] = inference_identity_space_batched(dec, scans[2:], dict(lambdas), 1200, schedule, step_scale=0.01)
    assert (np.abs(z1.detach().cpu().numpy() - z2.detach().cpu().numpy()) < 2e-5).mean() > 0.93
    assert float((a1 - a2).abs().max()) < 1e-5


def test_joint_batched_equals_sequential_calls(cuda_device):
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint, inference_iterative_root_finding_joint_batched
    _, subjects = _joint_subjects(cuda_device)
    dec = make_ensemble(0, device=cuda_device).train()
    dfn = make_deformation(cuda_device)
    torch.manual_seed(0)
    seq = [inference_iterative_root_finding_joint(dec, dfn, s, dict(JOINT_LAMBDAS), 400, JOINT_SCHEDULE, step_scale=0.01)
           for s in subjects]
    state_seq = torch.get_rng_state()
    torch.manual_seed(0)
    lam = dict(JOINT_LAMBDAS)
    bat = inference_iterative_root_finding_joint_batched(dec, dfn, subjects, lam, 400, JOINT_SCHEDULE, step_scale=0.01)
    assert torch.equal(torch.get_rng_state(), state_seq)
    one = dict(JOINT_LAMBDAS)
    inference_iterative_root_finding_joint(dec, dfn, subjects[0], one, 400, JOINT_SCHEDULE, step_scale=0.01)
    assert lam == one
    for k, ((e1, i1, a1), (e2, i2, a2)) in enumerate(zip(seq, bat)):
        assert e1.shape == e2.shape and i1.shape == i2.shape and a1.shape == a2.shape
        ci = (np.abs(i1.detach().cpu().numpy() - i2.detach().cpu().numpy()) < 5e-4).mean()
        ce = (np.abs(e1.detach().cpu().numpy() - e2.detach().cpu().numpy()) < 5e-4).mean()
        print('joint subject %d: batched vs sequential %.4f of z_id, %.4f of z_ex within 5e-4' % (k, ci, ce))
        assert ci > 0.9 and ce > 0.9, k
        assert float((a1 - a2).abs().max()) < 1e-5, k


def test_batched_steps_do_not_synchronise_with_the_host(cuda_device):
    from nphm_b200.models.fitting import BatchedIdentityFitter, BatchedJointFitter, _sample_observations
    dec = make_ensemble(0, device=cuda_device).train()
    dfn = make_deformation(cuda_device)
    pts = _scan_points(cuda_device)
    lam = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    bf = BatchedIdentityFitter(dec, 4, cuda_device)
    bf.step(pts, lam, 0.1, 0.01)                            # first call: workspace allocation
    _, subjects = _joint_subjects(cuda_device)
    bj = BatchedJointFitter(dec, dfn, [len(s) for s in subjects], cuda_device)
    torch.manual_seed(0)
    samples = [_sample_observations(s) for s in subjects]
    obs, idx = [o for o, _ in samples], [i.long().to(cuda_device) for _, i in samples]
    bj.step(obs, idx, dict(JOINT_LAMBDAS), 0.1, 0.01)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        bf.step(pts, lam, 0.1, 0.01)
        bj.step(obs, idx, dict(JOINT_LAMBDAS), 0.1, 0.01)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert torch.isfinite(bf.latents).all() and torch.isfinite(bj.z_id).all() and torch.isfinite(bj.z_ex).all()


def test_batched_entry_points_reject_bad_arguments(cuda_device, monkeypatch):
    from nphm_b200 import _native
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from nphm_b200.models import fitting
    dec = make_ensemble(0, device=cuda_device).train()
    eng = dec.engine()
    lib = _native.lib()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    S, n, D = 2, 1000, dec.lat_dim
    pts = torch.stack([_cloud(1, n, cuda_device), _cloud(2, n, cuda_device)]).contiguous()
    z = torch.zeros(S, D, device=cuda_device)
    m, v = torch.zeros_like(z), torch.zeros_like(z)
    terms = torch.empty(S, 8, device=cuda_device)
    grad = torch.empty(S, D, device=cuda_device)
    need = lib.nphm_fit_batch_workspace_bytes(eng.handle, S, n)
    assert need > lib.nphm_fit_workspace_bytes(eng.handle, n) and lib.nphm_fit_batch_workspace_bytes(eng.handle, 0, n) == -1
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_device)
    fp = _native.FitParams(2.0, 0.25, 0.05, 10.0, 5.0, 0.1, 0.01, 1)

    def step(pp, s, nn, lat, wsp, nbytes, h=eng.handle):
        return lib.nphm_fit_identity_step_batched(h, pp, None, s, nn, lat, m.data_ptr(), v.data_ptr(), ctypes.byref(fp), 1,
                                                  terms.data_ptr(), grad.data_ptr(), wsp, nbytes, stream)
    assert step(pts.data_ptr(), S, n, z.data_ptr(), ws.data_ptr(), need) == 0
    assert step(pts.data_ptr(), 0, n, z.data_ptr(), ws.data_ptr(), need) == -1                # S < 1
    assert step(pts.data_ptr(), S, 0, z.data_ptr(), ws.data_ptr(), need) == -1                # no points
    assert step(pts.data_ptr(), S, n, None, ws.data_ptr(), need) == -1                        # NULL latents
    assert step(pts.data_ptr(), S, n, z.data_ptr(), ws.data_ptr(), need - 1) == -4            # short workspace
    assert step(pts.data_ptr(), S, n, z.data_ptr(), None, need) == -1                         # no workspace
    assert lib.nphm_fit_surface_grad_batched(eng.handle, pts.data_ptr(), None, S, n, z.data_ptr(), 0.1, terms.data_ptr(),
                                             grad.data_ptr(), None, ws.data_ptr(), need - 1, stream) == -4
    assert lib.nphm_fit_apply_gradient_batched(eng.handle, 0, z.data_ptr(), m.data_ptr(), v.data_ptr(), ctypes.byref(fp),
                                               grad.data_ptr(), terms.data_ptr(), None, 1, None, None, stream) == -1
    torch.cuda.synchronize()
    # no tensor-core configuration: the C call refuses, the Python function fits scan by scan
    torch.manual_seed(4)
    small = FastEnsembleDeepSDFMirrored(lat_dim_glob=16, lat_dim_loc=8, n_loc=39, n_symm_pairs=16, anchors=mean_anchors(),
                                        hidden_dim=128, n_layers=4, pos_mlp_dim=64).to(cuda_device).train()
    small.anchors = small.anchors.to(cuda_device)
    se = small.engine()
    zs = torch.zeros(S, small.lat_dim, device=cuda_device)
    ms, vs = torch.zeros_like(zs), torch.zeros_like(zs)
    wss = torch.empty(lib.nphm_fit_batch_workspace_bytes(se.handle, S, n), dtype=torch.uint8, device=cuda_device)
    rc = lib.nphm_fit_identity_step_batched(se.handle, pts.data_ptr(), None, S, n, zs.data_ptr(), ms.data_ptr(), vs.data_ptr(),
                                            ctypes.byref(fp), 1, None, None, wss.data_ptr(), wss.numel(), stream)
    assert rc == -3
    # The fallback must BE the single-scan calls: record them.  (Their results are not compared with a second sequential run:
    # the single-scan FFMA backward sums with float atomics, so two runs of the same calls differ in the last bits, and
    # Adam's first, sign-like steps turn that into whole steps for entries whose gradient is at round-off level.)
    scans = [[_cloud(5, 1200, cuda_device), _cloud(6, 1000, cuda_device)], [_cloud(7, 1100, cuda_device)]]
    lam0 = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
    schedule = {'lr': {100: 2}, 'symm_dist': {100: 10}}
    single = fitting.inference_identity_space
    calls = []

    def spy(decoder, all_obs, lambdas, *args, **kwargs):
        calls.append({'decoder': decoder, 'obs': all_obs, 'lambdas_in': dict(lambdas), 'lambdas': lambdas, 'args': args})
        calls[-1]['out'] = single(decoder, all_obs, lambdas, *args, **kwargs)
        return calls[-1]['out']
    torch.manual_seed(0)
    for s_ in scans:
        single(small, s_, dict(lam0), 300, schedule, step_scale=0.01)
    state_seq = torch.get_rng_state()
    lam_one = dict(lam0)
    single(small, scans[0], lam_one, 300, schedule, step_scale=0.01)
    monkeypatch.setattr(fitting, 'inference_identity_space', spy)
    torch.manual_seed(0)
    lam = dict(lam0)
    bat = fitting.inference_identity_space_batched(small, scans, lam, 300, schedule, step_scale=0.01)
    assert len(calls) == len(scans) and all(c['obs'] is s_ and c['decoder'] is small for c, s_ in zip(calls, scans))
    assert all(c['lambdas_in'] == lam0 and c['lambdas'] is not lam for c in calls)          # a fresh copy per scan
    assert all(c['args'] == (300, schedule, 0.01, 1) for c in calls)
    assert all(b_ is c['out'] for b_, c in zip(bat, calls))
    assert torch.equal(torch.get_rng_state(), state_seq) and lam == lam_one != lam0
