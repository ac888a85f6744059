"""CPU check of the composite (autograd) path of nphm_b200.models.loss_functions against the reference's
actual_compute_loss (loss_functions.py:20-110) - same weights, same batch; the reference's values are stored in
tests/golden/losses.npz (make_golden_losses.py).  The native path needs a GPU (test_gpu_losses.py)."""
import numpy as np
import torch

from conftest import load_golden, make_ensemble

KEYS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far', 'normals_face', 'normals_non_face', 'gt_anchors')


def test_composite_training_losses_match_the_reference_function_on_cpu():
    from nphm_b200.models import loss_functions as L
    g = load_golden('losses.npz')
    ours = make_ensemble(0).train()
    batch = {k: torch.from_numpy(g['cpu_' + k]) for k in KEYS}
    cond = torch.from_numpy(g['cpu_cond']).requires_grad_()
    want = dict(zip(g['cpu_loss_names'], g['cpu_loss_values']))
    got = L.actual_compute_loss(batch, ours, cond)
    assert set(got) == set(want)
    for k in want:
        assert abs(float(got[k].detach()) - want[k]) <= 1e-5 * max(1.0, abs(want[k])), (k, float(got[k].detach()), want[k])
    # the graph reaches the weights through the spatial gradient (double backward), like the reference's
    total_g = sum(got[k] for k in ('surf_sdf', 'normals', 'grad'))
    gg = torch.autograd.grad(total_g, ours.ensembled_deep_sdf.lin1.weight)[0].reshape(-1).numpy()
    assert float(np.abs(gg[g['cpu_lin1_grad_idx']] - g['cpu_lin1_grad']).max()) <= 1e-4 * max(1e-6, float(g['cpu_lin1_grad_absmax']))
