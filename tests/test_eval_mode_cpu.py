"""Which rows carry the eval-mode quirk (every member's output set to 1 at the last point of each decoder call,
EnsembledDeepSDF.py:260-261) in the layouts the native eval-mode paths use, checked on the CPU against the reference's call
boundaries: the stage-1 point sets concatenated along the points (call_sizes), the fitters' flattened rows and the padded
per-scan layouts of the batched fitters (a period per scan, the kernels' rule i % p == p - 1)."""
import numpy as np
import torch

import ensemble_train_common as E
import shape_common as S
from conftest import load_golden, make_ensemble


def quirk_rows(n_rows, period):
    """The rule of csrc/fit.cu quirk_row(): row i (within its scan) is a quirk row when period > 0 and i % period == period - 1."""
    i = torch.arange(n_rows)
    return (i % period == period - 1) if period > 0 else torch.zeros(n_rows, dtype=torch.bool)


def _val_batch():
    g = load_golden('eval_mode.npz')
    return g, {k: torch.from_numpy(g['val_batch_' + k]) for k in E.BATCH_KEYS}, torch.from_numpy(g['val_batch_codes'])


def test_composite_eval_losses_match_the_reference_golden():
    """The reference's eval-mode validation losses from the composite mirror (one decoder call per point set)."""
    from nphm_b200.models.loss_functions import actual_compute_loss
    g, batch, codes = _val_batch()
    dec = make_ensemble(0).eval()
    codes = codes.clone().requires_grad_()
    losses = actual_compute_loss(batch, dec, codes)
    E.total_loss(losses).backward()
    full, sampled = E.gradient_record(dec, codes)
    S.check_against_golden({k[4:]: g[k] for k in g.files if k.startswith('val_')}, losses, full, sampled, rtol=1e-4,
                           native=False)


def test_concatenated_point_sets_quirk_the_last_point_of_each_call():
    """call_ends / apply_eval_quirk on the members of the four concatenated point sets give, value and gradient, what four
    separate eval-mode decoder calls give."""
    from nphm_b200.models import _composite as C
    from nphm_b200.models.diff_operators import gradient
    g, batch, codes = _val_batch()
    dec = make_ensemble(0).eval()
    sets = [batch[name] for name in E.POINT_SETS]
    sizes = [p.shape[1] for p in sets]
    assert C.call_ends(sizes) == list(np.cumsum(sizes) - 1)
    xyz = torch.cat(sets, 1)
    with torch.enable_grad():
        anchors, local, cond = C.member_frames(dec, xyz, codes)
        local = local.detach().requires_grad_()
        s = dec.ensembled_deep_sdf(local, cond.detach())[..., 0]
        gl = torch.autograd.grad(s.sum(), local)[0]
        s, gl = C.apply_eval_quirk(s.detach(), gl, sizes)
        sdf, grad = C.ensemble_blend_with_gradient(dec, xyz, anchors.detach(), s, gl)
        want_s, want_g = [], []
        for p in sets:
            x = p.clone().requires_grad_()
            v, _ = dec(x, codes.repeat(1, x.shape[1], 1), None)
            want_s.append(v.detach())
            want_g.append(gradient(v, x).detach())
    assert torch.allclose(sdf, torch.cat(want_s, 1), atol=1e-6, rtol=1e-5)
    assert torch.allclose(grad, torch.cat(want_g, 1), atol=1e-5, rtol=1e-4)
    # the rows that differ from the training-mode forward are exactly the call ends
    with torch.no_grad():
        train = torch.cat([dec.train()(p, codes.repeat(1, p.shape[1], 1), None)[0] for p in sets], 1)
    diff = (train - sdf.detach()).abs()[..., 0] > 1e-6
    assert torch.equal(diff.nonzero()[:, 1].unique(), torch.tensor(C.call_ends(sizes)))


def test_fitter_rows_follow_the_observation_rows():
    """A fitter's call ``decoder(obs)`` on rows x n points: the flattened rows with i % n == n - 1 are each row's last point."""
    obs = torch.randn(5, 37, 3)
    flat = obs.reshape(-1, 3)
    q = quirk_rows(flat.shape[0], obs.shape[1])
    assert int(q.sum()) == 5 and torch.equal(flat[q], obs[:, -1])


def test_batched_identity_layout_keeps_each_scans_quirk_rows():
    """_pad_scans pads every scan behind its 5 n_k rows: with scan k's own period n_k its quirk rows are its rows' last
    points, and every padding row is masked out."""
    from nphm_b200.models.fitting import _pad_scans
    sizes = [40, 23, 31]
    scans = [torch.randn(5, n, 3) for n in sizes]
    pts, mask = _pad_scans([s.reshape(-1, 3) for s in scans])
    for k, (s, n) in enumerate(zip(scans, sizes)):
        q = quirk_rows(pts.shape[1], n)
        real = torch.arange(pts.shape[1]) < 5 * n
        assert torch.equal(pts[k][q & real], s[:, -1])
        assert bool((mask[k][~real] == 0).all()) and bool((mask[k][real] == 1).all())


def test_batched_joint_layout_pads_in_front_in_eval_mode():
    """_pad_rows with ``front``: every row of every subject ends with that subject's last sampled point, so one period n_point
    marks each subject's quirk rows; the kept points are the subject's points in order.  Without ``front`` (training mode) the
    padding goes behind, the layout of the training-mode fitter."""
    from nphm_b200.models.fitting import _pad_rows
    sizes = [30, 18]
    obs = [torch.randn(5, n, 3) for n in sizes]
    n_point = max(sizes)
    for front in (True, False):
        rows, keep = _pad_rows(obs, n_point, front)
        rows = rows.reshape(len(sizes), 5, n_point, 3)
        for k, o in enumerate(obs):
            assert torch.equal(rows[k][keep[k]], o.reshape(-1, 3))
            if front:
                q = quirk_rows(5 * n_point, n_point).reshape(5, n_point)
                assert bool(keep[k][q].all()) and torch.equal(rows[k][q], o[:, -1])
            else:
                assert torch.equal(rows[k][:, :o.shape[1]], o)
    same, keep = _pad_rows([obs[0], obs[0]], n_point, True)
    assert keep is None and torch.equal(same, torch.cat([obs[0], obs[0]]))
