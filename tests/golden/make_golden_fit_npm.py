#!/usr/bin/env python
"""Generate fit_npm.npz: the reference's two fitters (src/NPHM/models/fitting.py) run UNMODIFIED on CPU with the NPM baseline
of scripts/configs/fitting_npm.yaml - identity DeepSDF(512, 1024), expression DeepSDF(512 + 200, 1024, out_dim=3) - at seeded
weights (tests/npm_fit_common.py), 3 scans of 200 points, the hard-coded lambdas and schedule of
fitting_pointclouds.py:253-266 and step_scale = 0.01, so that the lr / lambda / clamp events are crossed.

As in the fit_identity / fit_joint sections of make_golden.py, torch.optim.Adam is wrapped only to RECORD the gradient and the
latent it is handed at every step, and inference_iterative_root_finding_joint's two hard-coded `.cuda()` calls are made the
identity for the duration of the call.  Stores the state-dict sha256 of both decoders (the mirror must initialise the same
weights), the scans, per-iteration gradients and latents, the final codes and the fraction of valid correspondences of a search
at the zero codes.  tests/test_fit_npm_cpu.py checks the composite fitters against it, tests/test_gpu_fit_npm.py the native ones.
Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_fit_npm.py
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_loader as R      # noqa: E402
import npm_fit_common as C              # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count())
    ns = R.load()
    import torch.optim as optim_mod
    real_adam = optim_mod.Adam
    scans = C.make_scans()
    obs = [torch.from_numpy(o) for o in scans]
    out = {'obs': np.stack(scans)}

    # ---------------------------------------------------------------- identity fitting
    rec = {'grad': [], 'z': [], 'lr': []}

    class RecordingAdam(real_adam):
        def step(self, closure=None):
            p = self.param_groups[0]['params'][0]
            rec['grad'].append(p.grad.detach().clone().numpy().reshape(-1))
            rec['z'].append(p.detach().clone().numpy().reshape(-1))
            rec['lr'].append(self.param_groups[0]['lr'])
            return super().step(closure)

    dec, expr = C.make_decoders(ns.deepSDF.DeepSDF)
    out['sha256_id'] = np.array(C.state_dict_sha256(dec))
    out['sha256_ex'] = np.array(C.state_dict_sha256(expr))
    lambdas = dict(C.LAMBDAS_IDENTITY)
    optim_mod.Adam = RecordingAdam
    try:
        np.random.seed(0)
        torch.manual_seed(0)
        z, anchors = ns.fitting.inference_identity_space(dec, obs, lambdas, n_steps=C.N_ITER_IDENTITY * 100,
                                                         schedule_cfg=C.SCHEDULE, step_scale=C.STEP_SCALE)
    finally:
        optim_mod.Adam = real_adam
    assert anchors is None
    out['id_grads'] = np.stack(rec['grad'])
    out['id_z_before'] = np.stack(rec['z'])
    out['id_lrs'] = np.array(rec['lr'], np.float64)
    out['id_z_final'] = z.detach().numpy().reshape(-1)
    out['id_lambdas_final'] = np.array([lambdas[k] for k in sorted(lambdas)], np.float64)
    print('identity fit: %d iterations, |z| %.4g, grad norms %s' % (
        len(rec['grad']), float(z.detach().norm()), np.round(np.linalg.norm(out['id_grads'], axis=1), 5)))

    # ---------------------------------------------------------------- joint fitting
    rec2 = {'grads': [], 'params': []}

    class RecordingAdam2(real_adam):
        def step(self, closure=None):
            p_ = self.param_groups[0]['params'][0]
            rec2['grads'].append(p_.grad.detach().clone().numpy().copy())
            rec2['params'].append(p_.detach().clone().numpy().copy())
            return super().step(closure)

    dec, expr = C.make_decoders(ns.deepSDF.DeepSDF)
    # how much of the search converges at the zero codes (the start of the fit)
    cond = torch.zeros(3, 200, 712)
    _, res = ns.iterative_root_finding.search(torch.from_numpy(np.stack(scans)), cond, expr, None, multi_corresp=False)
    out['valid_fraction_start'] = np.array(float(res['valid_ids'].float().mean()))
    print('valid correspondences at the zero codes: %.4f' % float(out['valid_fraction_start']))
    assert float(out['valid_fraction_start']) > 0.9
    lambdas = dict(C.LAMBDAS_JOINT)
    optim_mod.Adam = RecordingAdam2
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        np.random.seed(0)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()) as log:
            z_ex, z_id, anchors = ns.fitting.inference_iterative_root_finding_joint(
                dec, expr, obs, lambdas, n_steps=C.N_ITER_JOINT * 100, schedule_cfg=C.SCHEDULE, step_scale=C.STEP_SCALE)
    finally:
        optim_mod.Adam = real_adam
        torch.Tensor.cuda = real_cuda
    assert anchors is None
    # the reference prints the number of valid correspondences at the end of every iteration line
    n_valid = [int(line.split()[-1]) for line in log.getvalue().splitlines() if line.startswith('Epoch')]
    out['joint_n_valid'] = np.array(n_valid)
    # opt.step() (identity) is called before opt_expr.step(): records alternate id, expr, id, expr ...
    out['joint_grads_id'] = np.stack([g.reshape(-1) for g in rec2['grads'][0::2]])
    out['joint_grads_ex'] = np.stack([g.reshape(3, 200) for g in rec2['grads'][1::2]])
    out['joint_z_id_before'] = np.stack([g.reshape(-1) for g in rec2['params'][0::2]])
    out['joint_z_ex_before'] = np.stack([g.reshape(3, 200) for g in rec2['params'][1::2]])
    out['joint_z_id_final'] = z_id.detach().numpy().reshape(-1)
    out['joint_z_ex_final'] = z_ex.detach().numpy().reshape(3, 200)
    out['joint_lambdas_final'] = np.array([lambdas[k] for k in sorted(lambdas)], np.float64)
    print('joint fit: %d iterations, valid correspondences %s of 1000, grad norms id %s ex %s' % (
        len(n_valid), n_valid, np.round(np.linalg.norm(out['joint_grads_id'], axis=1), 5),
        np.round(np.linalg.norm(out['joint_grads_ex'].reshape(len(n_valid), -1), axis=1), 6)))
    path = os.path.join(HERE, 'fit_npm.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
