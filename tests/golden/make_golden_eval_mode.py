#!/usr/bin/env python
"""Generate eval_mode.npz: the reference's ensemble differentiated in eval mode, where FastEnsembleDeepSDFMirrored.forward sets
every member's output to 1 at the last point of each call (src/NPHM/models/EnsembledDeepSDF.py:260-261).  Runs the unmodified
reference (oracle/ref_loader.py) in torch fp32 on CPU on the seeded make_ensemble decoder (torch.manual_seed(0), nphm.yaml
size):

  (a) one validation batch of stage 1 as TrainerAutoDecoder.compute_val_loss takes it (training.py:250-268: decoder.eval(),
      actual_compute_loss, backward with the nphm.yaml lambdas) on the small point sets of train_ensemble.npz's generator:
      the loss terms, the full code and mlp_pos gradients, and a seeded subsample plus the max-abs and norm of every ensembled
      weight and bias gradient (prefix ``val_``);
  (b) 12 iterations of inference_identity_space with the decoder in eval mode: the latent before each Adam step, the gradient
      Adam is handed and the final code (prefix ``id_``).  One of the three observations lies far from every anchor, so that
      quirk rows there (sdf ~ 0.002, the normalised background weight) pass the |sdf| < clamp test;
  (c) 4 iterations of inference_iterative_root_finding_joint with the identity decoder in eval mode: d/dz_id and d/dz_ex handed
      to the two Adam steps and the latents before them (prefix ``joint_``).

    python tests/golden/make_golden_eval_mode.py
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
import ensemble_train_common as E       # noqa: E402
import shape_common as S                # noqa: E402

ID_LAMBDAS = {'surface': 2.0, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
JOINT_LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05,
                 'symm_dist': 5.0}
SCHEDULE = {'lr': {200: 2, 400: 2, 600: 2, 800: 2}, 'symm_dist': {200: 10, 500: 9999},
            'reg_glob': {200: 3, 600: 10}, 'reg_loc': {500: 3, 600: 10}, 'reg_expr': {600: 10}}
ID_ITERS, JOINT_ITERS = 12, 4
# the val batch: SIZES points per set and batch element (the reference's four calls end at each set's last point)
VAL_SIZES = E.SIZES


def identity_observations():
    rng = np.random.RandomState(300)
    near = [(rng.randn(300, 3) * 0.12 + np.array([0.0, 0.05, -0.1])).astype(np.float32) for _ in range(2)]
    far = (rng.randn(300, 3) * 0.2 + np.array([1.8, -1.6, 2.0])).astype(np.float32)
    return near + [far]


def joint_observations():
    rng = np.random.RandomState(400)
    return [(rng.randn(200, 3) * 0.1 + np.array([0.0, 0.05, -0.1])).astype(np.float32) for _ in range(3)]


class _Recorder:
    """Wraps torch.optim.Adam.step to record the parameter and the gradient it is handed (the reference runs unmodified)."""

    def __init__(self):
        self.grads, self.params = [], []
        self._real = torch.optim.Adam
        rec = self

        class RecordingAdam(self._real):
            def step(self, closure=None):
                p = self.param_groups[0]['params'][0]
                rec.grads.append(p.grad.detach().clone().numpy().copy())
                rec.params.append(p.detach().clone().numpy().copy())
                return super().step(closure)
        self.cls = RecordingAdam

    def __enter__(self):
        torch.optim.Adam = self.cls
        return self

    def __exit__(self, *exc):
        torch.optim.Adam = self._real


NORMALS = {'points_face': 'normals_face', 'points_non_face': 'normals_non_face'}


def select_points(net, batch):
    """Per set and batch element, the first VAL_SIZES points (of twice as many drawn) where the reference's |sdf| >= 1e-4
    (closer to 0 the sign in the gradients of surf_sdf and space_sdf is not resolved by an fp32 evaluation).  The selecting
    call's own quirk point is its last one, which is never among the first half kept."""
    codes = torch.from_numpy(batch['codes'])
    gt = torch.from_numpy(batch['gt_anchors'])
    out = dict(batch)
    with torch.no_grad():
        for name, n in zip(E.POINT_SETS, VAL_SIZES):
            pts = torch.from_numpy(batch[name])
            s = net(pts, codes.repeat(1, pts.shape[1], 1), gt)[0][..., 0].abs().numpy()
            keep = [np.flatnonzero(s[b, :-1] >= E.MIN_ABS_SDF)[:n] for b in range(s.shape[0])]
            assert all(k.size == n for k in keep), '%s: too few points with |sdf| >= %g' % (name, E.MIN_ABS_SDF)
            for key in (name,) + ((NORMALS[name],) if name in NORMALS else ()):
                out[key] = np.stack([batch[key][b, k] for b, k in enumerate(keep)])
    return out


def validation_batch(ns, out):
    net = R.make_ensemble(ns, 0).eval()                            # compute_val_loss: self.decoder.eval()
    batch = select_points(net, E.make_batch(ns.assets['anchors_39'], sizes=[2 * n for n in VAL_SIZES], seed=5))
    out['sha256'] = np.array(S.state_dict_sha256(net))
    for k, v in batch.items():
        out['val_batch_' + k] = v
    bt = {k: torch.from_numpy(v) for k, v in batch.items() if k != 'codes'}
    codes = torch.from_numpy(batch['codes']).requires_grad_()
    losses = ns.loss_functions.actual_compute_loss(bt, net, codes)
    E.total_loss(losses).backward()
    names = sorted(losses)
    out['val_loss_names'] = np.array(names)
    out['val_loss_values'] = np.array([float(losses[k].detach()) for k in names])
    full, sampled = E.gradient_record(net, codes)
    for k, v in full.items():
        out['val_full_' + k] = v.astype(np.float32)
    for k, v in sampled.items():
        flat = v.reshape(-1)
        idx = S.sample_idx(k, flat.size)
        out['val_idx_' + k] = idx.astype(np.int64)
        out['val_sampled_' + k] = flat[idx].astype(np.float32)
        out['val_maxabs_' + k] = np.array(np.abs(flat).max(), np.float64)
        out['val_norm_' + k] = np.array(np.linalg.norm(flat.astype(np.float64)))
    print('val losses', dict(zip(names, out['val_loss_values'])))


def identity_fit(ns, out):
    obs = identity_observations()
    dec = R.make_ensemble(ns, 0).eval()
    lambdas = dict(ID_LAMBDAS)
    np.random.seed(0)
    torch.manual_seed(0)
    with _Recorder() as rec:
        z, _ = ns.fitting.inference_identity_space(dec, [torch.from_numpy(o) for o in obs], lambdas,
                                                   n_steps=ID_ITERS * 100, schedule_cfg=SCHEDULE, step_scale=0.01)
    out['id_obs'] = np.stack(obs)
    out['id_grads'] = np.stack([g.reshape(-1) for g in rec.grads])
    out['id_z_before'] = np.stack([p.reshape(-1) for p in rec.params])
    out['id_z_final'] = z.detach().numpy().reshape(-1)
    print('identity fit (eval): grad norms', np.linalg.norm(out['id_grads'], axis=1)[:4])


def joint_fit(ns, out):
    obs = joint_observations()
    dec = R.make_ensemble(ns, 0).eval()
    dfn = R.make_deformation(ns)
    lambdas = dict(JOINT_LAMBDAS)
    # inference_iterative_root_finding_joint hard-codes `.cuda()` on two index tensors (fitting.py:72,137): identity on CPU
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    np.random.seed(0)
    torch.manual_seed(0)
    try:
        with _Recorder() as rec, contextlib.redirect_stdout(io.StringIO()):
            ns.fitting.inference_iterative_root_finding_joint(dec, dfn, [torch.from_numpy(o) for o in obs], lambdas,
                                                              n_steps=JOINT_ITERS * 100, schedule_cfg=SCHEDULE,
                                                              step_scale=0.01)
    finally:
        torch.Tensor.cuda = real_cuda
    # opt.step() (identity) runs before opt_expr.step(): the records alternate id, expr, id, expr ...
    out['joint_obs'] = np.stack(obs)
    out['joint_grads_id'] = np.stack([g.reshape(-1) for g in rec.grads[0::2]])
    out['joint_grads_ex'] = np.stack([g.reshape(len(obs), -1) for g in rec.grads[1::2]])
    out['joint_z_id_before'] = np.stack([p.reshape(-1) for p in rec.params[0::2]])
    out['joint_z_ex_before'] = np.stack([p.reshape(len(obs), -1) for p in rec.params[1::2]])
    print('joint fit (eval): grad norms id', np.linalg.norm(out['joint_grads_id'], axis=1))


def main():
    torch.set_num_threads(os.cpu_count())
    ns = R.load()
    out = {}
    validation_batch(ns, out)
    identity_fit(ns, out)
    joint_fit(ns, out)
    path = os.path.join(HERE, 'eval_mode.npz')
    np.savez_compressed(path, **out)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    main()
