"""SURVEY.md 8f-3: the identity-space training losses (reference loss_functions.py:20-110) evaluated natively - SDF values and
spatial gradients from nphm_ensemble_backward_inputs, no autograd graph - against the UNMODIFIED reference function running on
its own modules with autograd, same weights, same batch (its values: tests/golden/losses.npz, make_golden_losses.py)."""
import pytest
import torch

from conftest import load_golden, make_ensemble

pytestmark = pytest.mark.gpu
KEYS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far', 'normals_face', 'normals_non_face', 'gt_anchors')


def test_native_training_losses_match_the_reference_function(cuda_device):
    from nphm_b200.models import loss_functions as L
    g = load_golden('losses.npz')
    ours = make_ensemble(0, device=cuda_device).train()
    batch = {k: torch.from_numpy(g['gpu_' + k]).to(cuda_device) for k in KEYS}
    cond = torch.from_numpy(g['gpu_cond']).to(cuda_device)
    want = dict(zip(g['gpu_loss_names'], g['gpu_loss_values']))
    with torch.no_grad():
        got = L.actual_compute_loss(batch, ours, cond)                      # native: no graph
    got_graph = L.actual_compute_loss(batch, ours, cond)                    # composite: autograd, what training uses
    assert set(got) == set(want) == set(got_graph)
    for k, w in want.items():
        w = float(w)
        for name, gv in (('native', got[k]), ('composite', got_graph[k])):
            gv = float(gv.detach())
            assert abs(gv - w) <= 2e-5 * max(1.0, abs(w)), (k, name, gv, w)
        print('%-12s reference %.7f  native %.7f  composite %.7f' % (k, w, float(got[k].detach()), float(got_graph[k].detach())))
    assert not got['grad'].requires_grad and got_graph['grad'].requires_grad
