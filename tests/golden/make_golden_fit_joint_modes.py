#!/usr/bin/env python
"""Generate fit_joint_modes.npz: the reference's joint fitter (src/NPHM/models/fitting.py:14-177) run UNMODIFIED on CPU with
the NPHM ensemble and a DeformationNetwork in each of the two other modes the reference names (deepSDF.py:146): expr_only
(condition z_ex) and glob_only (condition [z_id[:64] | z_ex]), at seeded weights (tests/fit_modes_common.py).

The recipe of make_golden.py's fit_joint.npz: seeded ensemble in training mode, 3 observations of 300 points, the hard-coded
lambdas and schedule of fitting_pointclouds.py:253-266 at step_scale = 0.01.  `Tensor.cuda` is made the identity for the
duration of the call, and torch.optim.Adam is wrapped:
  * the joint run, with the ensemble in training and in eval mode: every Adam only RECORDS the gradient and the code it is
    handed, then steps (the identity's optimizer steps first, :168-169);
  * the fixed-identity run (the contract of inference_expression_space, as in make_golden_fit_expression.py): the FIRST
    optimizer, over lat_rep_shape, copies sample_latent(3) into it and never steps; the second records and steps.
Stored per mode ('<mode>_'): the deformation network's state-dict sha256, per-step gradients and codes, the final codes and
anchors, the lambdas the loop leaves behind and torch's CPU generator state after the call; 'fixed_' for the fixed-identity
run, 'eval_' for the joint run with the ensemble in eval mode (its forward overwrites every member's output at the last point
of each decoder call, EnsembledDeepSDF.py:260-261).  Needs the reference modules (oracle/_ref, made by oracle/make_ref.py,
or a reference checkout):

    python tests/golden/make_golden_fit_joint_modes.py
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
import fit_modes_common as C            # noqa: E402
import npm_fit_common as N              # noqa: E402


def run_joint(ns, dec, dfn, scans, z_id=None):
    """The reference joint loop; with ``z_id`` the identity code is set to it and its optimizer never steps."""
    import torch.optim as optim_mod
    real_adam, real_cuda = optim_mod.Adam, torch.Tensor.cuda
    rec = {'grads': [], 'codes': [], 'built': 0}

    class RecordingAdam(real_adam):
        def __init__(self, params, *args, **kwargs):
            params = list(params)
            super().__init__(params, *args, **kwargs)
            self.slot = rec['built']
            rec['built'] += 1
            if z_id is not None and self.slot == 0:
                with torch.no_grad():
                    params[0].copy_(z_id.reshape(params[0].shape))

        def step(self, closure=None):
            if z_id is not None and self.slot == 0:
                return None
            p = self.param_groups[0]['params'][0]
            rec['grads'].append(p.grad.detach().clone().numpy().copy())
            rec['codes'].append(p.detach().clone().numpy().copy())
            return super().step(closure)

    lambdas = dict(C.LAMBDAS_JOINT)
    optim_mod.Adam = RecordingAdam
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        np.random.seed(0)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            z_ex, z_id_out, anchors = ns.fitting.inference_iterative_root_finding_joint(
                dec, dfn, [torch.from_numpy(o) for o in scans], lambdas, n_steps=C.N_ITER * 100, schedule_cfg=C.SCHEDULE,
                step_scale=C.STEP_SCALE)
    finally:
        optim_mod.Adam = real_adam
        torch.Tensor.cuda = real_cuda
    out = {'z_ex_final': z_ex.detach().numpy().reshape(len(scans), -1),
           'anchors_final': anchors.detach().numpy().reshape(-1, 3),
           'lambdas_final': np.array([lambdas[k] for k in sorted(lambdas)], np.float64),
           'rng_after': torch.get_rng_state().numpy()}
    if z_id is not None:
        assert torch.equal(z_id_out.detach().reshape(-1), z_id.reshape(-1)), 'the identity code moved'
        out['grads_ex'] = np.stack([g.reshape(len(scans), -1) for g in rec['grads']])
        out['z_ex_before'] = np.stack([c.reshape(len(scans), -1) for c in rec['codes']])
        return out
    # the identity's optimizer steps first: records alternate id, expr, id, expr ...
    out['z_id_final'] = z_id_out.detach().numpy().reshape(-1)
    out['grads_id'] = np.stack([g.reshape(-1) for g in rec['grads'][0::2]])
    out['grads_ex'] = np.stack([g.reshape(len(scans), -1) for g in rec['grads'][1::2]])
    out['z_id_before'] = np.stack([c.reshape(-1) for c in rec['codes'][0::2]])
    out['z_ex_before'] = np.stack([c.reshape(len(scans), -1) for c in rec['codes'][1::2]])
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    ns = R.load()
    scans = C.make_scans()
    out = {'obs': np.stack(scans)}
    z_id = R.sample_latent(ns, C.ID_SEED).float()
    out['z_id_fixed'] = z_id.numpy().reshape(-1)
    for mode in C.MODES:
        dfn = C.make_deformation(mode, R.mean_anchors(ns), cls=ns.deepSDF.DeformationNetwork)
        out[mode + '_sha256'] = np.array(N.state_dict_sha256(dfn))
        for tag, z, train in (('', None, True), ('eval_', None, False), ('fixed_', z_id, True)):
            dec = R.make_ensemble(ns, 0).train(train)             # fitting_pointclouds.py:268 trains; eval: the last-point quirk
            for k, v in run_joint(ns, dec, dfn, scans, z).items():
                out['%s_%s%s' % (mode, tag, k)] = v
        print('%s: |z_id| %.4f |z_ex| %.4f, grad norms id %s ex %s; fixed identity: |z_ex| %.4f' % (
            mode, np.linalg.norm(out[mode + '_z_id_final']), np.linalg.norm(out[mode + '_z_ex_final']),
            np.round(np.linalg.norm(out[mode + '_grads_id'], axis=1), 5),
            np.round(np.linalg.norm(out[mode + '_grads_ex'].reshape(C.N_ITER, -1), axis=1), 5),
            np.linalg.norm(out[mode + '_fixed_z_ex_final'])))
    path = os.path.join(HERE, 'fit_joint_modes.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
