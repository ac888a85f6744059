"""CPU check of the composite fitters with the NPM baseline's DeepSDF decoders (nphm_b200.models.fitting on autograd) against
the reference's own runs (tests/golden/fit_npm.npz from make_golden_fit_npm.py): same initial weights (state-dict sha256), the
schedule's lambdas, and the latents and gradients the reference handed to Adam.  The native fitters are checked against the same
golden on the GPU (test_gpu_fit_npm.py)."""
import numpy as np
import torch

import npm_fit_common as C
from conftest import load_golden


def _decoders():
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('fit_npm.npz')
    dec, expr = C.make_decoders(DeepSDF)
    assert C.state_dict_sha256(dec) == str(g['sha256_id']) and C.state_dict_sha256(expr) == str(g['sha256_ex'])
    return g, dec, expr


def test_composite_identity_fit_follows_reference():
    from nphm_b200.models.fitting import inference_identity_space
    g, dec, _ = _decoders()
    lambdas = dict(C.LAMBDAS_IDENTITY)
    np.random.seed(0)
    torch.manual_seed(0)
    z, anchors = inference_identity_space(dec, [torch.from_numpy(o) for o in g['obs']], lambdas,
                                          n_steps=C.N_ITER_IDENTITY * 100, schedule_cfg=C.SCHEDULE, step_scale=C.STEP_SCALE)
    assert anchors is None and z.shape == (1, 1, 512) and z.requires_grad
    assert np.allclose([lambdas[k] for k in sorted(lambdas)], g['id_lambdas_final'])
    err = np.abs(z.detach().numpy().reshape(-1) - g['id_z_final'])
    print('composite identity fit: max |z - z_ref| %.3g' % err.max())
    assert (err < 2e-4).mean() > 0.98, (err < 2e-4).mean()


def test_composite_joint_fit_follows_reference():
    from nphm_b200.models.fitting import inference_iterative_root_finding_joint
    g, dec, expr = _decoders()
    lambdas = dict(C.LAMBDAS_JOINT)
    np.random.seed(0)
    torch.manual_seed(0)
    z_ex, z_id, anchors = inference_iterative_root_finding_joint(
        dec, expr, [torch.from_numpy(o) for o in g['obs']], lambdas, n_steps=C.N_ITER_JOINT * 100, schedule_cfg=C.SCHEDULE,
        step_scale=C.STEP_SCALE)
    assert anchors is None and z_ex.shape == (3, 1, 200) and z_id.shape == (1, 1, 512)
    assert np.allclose([lambdas[k] for k in sorted(lambdas)], g['joint_lambdas_final'])
    e_id = np.abs(z_id.detach().numpy().reshape(-1) - g['joint_z_id_final'])
    e_ex = np.abs(z_ex.detach().numpy().reshape(3, 200) - g['joint_z_ex_final'])
    print('composite joint fit: max |z_id - ref| %.3g, max |z_ex - ref| %.3g' % (e_id.max(), e_ex.max()))
    assert (e_id < 2e-4).mean() > 0.97 and (e_ex < 2e-4).mean() > 0.97, ((e_id < 2e-4).mean(), (e_ex < 2e-4).mean())
