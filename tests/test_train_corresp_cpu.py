"""CPU check of the composite path of nphm_b200.models.loss_functions.compute_loss_corresp_forward against one stage-2 step
of the reference (loss_functions.py:282-322 + backward, tests/golden/train_corresp.npz from make_golden_train_corresp.py):
the recorded random draws are replayed, so the loss terms and every stored gradient (compressor, biases, mlp_pos, expression
and shape rows, weight-gradient samples and norms) must match.  The native path is checked against the same golden on the
GPU (test_gpu_train.py)."""
import torch

import corresp_common as C
from conftest import load_golden, make_deformation, make_ensemble


def test_composite_corresp_step_matches_the_reference_golden():
    from nphm_b200.models.loss_functions import compute_loss_corresp_forward
    g = load_golden('train_corresp.npz')
    dfn = make_deformation().train()
    shape_dec = make_ensemble(0).train()
    lat_expr, lat_shape = C.make_embeddings(expr=g['weights_expr'], shape=g['weights_shape'])
    batch = {k: g['batch_' + k] for k in ('points_neutral', 'points_posed', 'gt_anchors', 'idx', 'subj_ind')}
    kinds = [str(k) for k in g['draw_kinds']]
    with C.replay_draws(kinds, [g['draw_%d' % i] for i in range(len(kinds))]):
        losses = compute_loss_corresp_forward({k: torch.from_numpy(v) for k, v in batch.items()}, dfn, shape_dec, lat_expr,
                                              lat_shape, 'cpu', native=False)
    C.total_loss(losses).backward()
    full, sampled = C.gradient_record(dfn, shape_dec, lat_expr, lat_shape, batch)
    C.check_against_golden(g, losses, full, sampled, rtol=1e-4)
