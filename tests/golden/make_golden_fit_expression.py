#!/usr/bin/env python
"""Generate fit_expression.npz: the reference's joint fitter (src/NPHM/models/fitting.py:14-177) run UNMODIFIED on CPU with the
identity code held fixed - the contract of nphm_b200.models.fitting.inference_expression_space - for the NPHM ensemble with its
'compress' deformation network and for the NPM pair of DeepSDF decoders, at seeded weights.

As in the joint sections of make_golden.py and make_golden_fit_npm.py, `Tensor.cuda` is made the identity for the duration of
the call.  torch.optim.Adam is wrapped: the FIRST optimizer the loop builds is the one over `lat_rep_shape` (fitting.py:35);
its wrapper copies the seeded identity code into that tensor and never steps.  The second one, over the expression codes,
records the gradient and the codes it is handed at every step, then steps.  Stored per decoder pair ('nphm', 'npm'): the
decoders' state-dict sha256, the scans, the identity code, per-step expression gradients and codes, the final codes, the
anchors the loop returns, the lambdas it leaves behind and torch's CPU generator state after the call.
Needs the reference modules (oracle/_ref, made by oracle/make_ref.py, or a reference checkout):

    python tests/golden/make_golden_fit_expression.py
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
import fit_expression_common as C       # noqa: E402
import npm_fit_common as N              # noqa: E402


def run_fixed_identity(ns, dec, expr, scans, z_id):
    """The reference joint loop with lat_rep_shape := z_id and its optimizer never stepping."""
    import torch.optim as optim_mod
    real_adam, real_cuda = optim_mod.Adam, torch.Tensor.cuda
    rec = {'grads': [], 'codes': [], 'built': 0}

    class FixedIdentityAdam(real_adam):
        def __init__(self, params, *args, **kwargs):
            params = list(params)
            super().__init__(params, *args, **kwargs)
            self.identity = rec['built'] == 0
            rec['built'] += 1
            if self.identity:
                with torch.no_grad():
                    params[0].copy_(z_id.reshape(params[0].shape))

        def step(self, closure=None):
            if self.identity:
                return None
            p = self.param_groups[0]['params'][0]
            rec['grads'].append(p.grad.detach().clone().numpy().reshape(len(scans), -1))
            rec['codes'].append(p.detach().clone().numpy().reshape(len(scans), -1))
            return super().step(closure)

    lambdas = dict(C.LAMBDAS_JOINT)
    optim_mod.Adam = FixedIdentityAdam
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        np.random.seed(0)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            z_ex, z_id_out, anchors = ns.fitting.inference_iterative_root_finding_joint(
                dec, expr, [torch.from_numpy(o) for o in scans], lambdas, n_steps=C.N_ITER * 100, schedule_cfg=C.SCHEDULE,
                step_scale=C.STEP_SCALE)
    finally:
        optim_mod.Adam = real_adam
        torch.Tensor.cuda = real_cuda
    assert torch.equal(z_id_out.detach().reshape(-1), z_id.reshape(-1)), 'the identity code moved'
    out = {'grads': np.stack(rec['grads']), 'codes_before': np.stack(rec['codes']),
           'z_ex_final': z_ex.detach().numpy().reshape(len(scans), -1),
           'lambdas_final': np.array([lambdas[k] for k in sorted(lambdas)], np.float64),
           'rng_after': torch.get_rng_state().numpy()}
    if anchors is not None:
        out['anchors'] = anchors.detach().numpy().reshape(-1, 3)
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    ns = R.load()
    out = {}
    # ---------------------------------------------------------------- NPHM ensemble + 'compress' deformation network
    dec = R.make_ensemble(ns, 0).train()                      # fitting_pointclouds.py:268
    dfn = R.make_deformation(ns, 10)                          # eval mode (fitting_pointclouds.py:229)
    z_id = R.sample_latent(ns, 3).float()
    scans = C.make_scans(C.NPHM_SCAN_POINTS, 400)
    out['nphm_sha256_id'] = np.array(N.state_dict_sha256(dec))
    out['nphm_sha256_ex'] = np.array(N.state_dict_sha256(dfn))
    out['nphm_z_id'] = z_id.numpy().reshape(-1)
    for i, s in enumerate(scans):
        out['nphm_scan%d' % i] = s
    for k, v in run_fixed_identity(ns, dec, dfn, scans, z_id).items():
        out['nphm_' + k] = v
    print('nphm: %d iterations, |z_ex| %.4g, grad norms %s' % (
        len(out['nphm_grads']), np.linalg.norm(out['nphm_z_ex_final']),
        np.round(np.linalg.norm(out['nphm_grads'].reshape(C.N_ITER, -1), axis=1), 6)))

    # ---------------------------------------------------------------- NPM baseline (DeepSDF pair)
    dec, expr = N.make_decoders(ns.deepSDF.DeepSDF)
    torch.manual_seed(41)
    z_id = torch.randn(dec.lat_dim) * 0.05
    scans = C.make_scans(C.NPM_SCAN_POINTS, 401)
    out['npm_sha256_id'] = np.array(N.state_dict_sha256(dec))
    out['npm_sha256_ex'] = np.array(N.state_dict_sha256(expr))
    out['npm_z_id'] = z_id.numpy()
    for i, s in enumerate(scans):
        out['npm_scan%d' % i] = s
    for k, v in run_fixed_identity(ns, dec, expr, scans, z_id).items():
        out['npm_' + k] = v
    print('npm: %d iterations, |z_ex| %.4g, grad norms %s' % (
        len(out['npm_grads']), np.linalg.norm(out['npm_z_ex_final']),
        np.round(np.linalg.norm(out['npm_grads'].reshape(C.N_ITER, -1), axis=1), 6)))
    path = os.path.join(HERE, 'fit_expression.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
