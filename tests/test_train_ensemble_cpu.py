"""CPU checks of the autograd half of native stage-1 training for the NPHM ensemble: the blend of the members' values and
local-frame gradients (``_composite.ensemble_blend_with_gradient``).  Fed (s_k, grad_local s_k) from an autograd evaluation
of the members with create_graph=True, it must reproduce the composite loss of ``actual_compute_loss`` and every gradient
of its double backward: in float64 to 1e-10, and in fp32 against one step of the reference (tests/golden/train_ensemble.npz,
make_golden_train_ensemble.py)."""
import pytest
import torch

import ensemble_train_common as E
import shape_common as S
from conftest import load_golden, make_ensemble


def _assembled_values_and_gradients(decoder, points, glob_cond, anchor_preds):
    """Drop-in for loss_functions._composite_values_and_gradients: members by autograd, blend and its gradient by formula."""
    from nphm_b200.models import _composite as C
    anchors, local, cond = C.member_frames(decoder, points, glob_cond)
    s = decoder.ensembled_deep_sdf(local, cond)
    g, = torch.autograd.grad(s.sum(), local, create_graph=True)
    sdf, grad = C.ensemble_blend_with_gradient(decoder, points, anchors, s, g)
    return sdf, grad, anchors


def _step(decoder, batch, codes, assembled, monkeypatch):
    from nphm_b200.models import loss_functions as L
    decoder.zero_grad(set_to_none=True)
    codes = codes.detach().clone().requires_grad_()
    with monkeypatch.context() as m:
        if assembled:
            m.setattr(L, '_composite_values_and_gradients', _assembled_values_and_gradients)
        losses = L.actual_compute_loss(batch, decoder, codes)
    E.total_loss(losses).backward()
    grads = {'codes': codes.grad.clone()}
    grads.update({k: p.grad.clone() for k, p in decoder.named_parameters()})
    return {k: float(v.detach()) for k, v in losses.items()}, grads


def _golden_batch(g, dtype):
    batch = {k: torch.from_numpy(g['batch_' + k]).to(dtype) for k in E.BATCH_KEYS}
    return batch, torch.from_numpy(g['batch_codes']).to(dtype)


def test_blend_reproduces_the_composite_double_backward_in_float64(monkeypatch):
    g = load_golden('train_ensemble.npz')
    dec = make_ensemble(0).double().train()
    batch, codes = _golden_batch(g, torch.float64)
    want_l, want_g = _step(dec, batch, codes, False, monkeypatch)
    got_l, got_g = _step(dec, batch, codes, True, monkeypatch)
    assert set(got_l) == set(want_l)
    for k, v in want_l.items():
        assert abs(got_l[k] - v) <= 1e-10 * abs(v), (k, got_l[k], v)
    assert set(got_g) == set(want_g) and len(want_g) == 1 + 6 + 10
    for k, v in want_g.items():
        scale = float(v.abs().max())
        assert scale > 0, k
        err = float((got_g[k] - v).abs().max())
        assert err <= 1e-10 * scale, (k, err / scale)


def test_blend_handles_a_point_on_an_anchor(monkeypatch):
    """At x = A_k the blend weight's gradient has the 0 direction of torch's norm backward, as in the composite."""
    dec = make_ensemble(0).double().train()
    codes = 0.05 * torch.randn(1, 1, dec.lat_dim, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    with torch.no_grad():
        anchors = dec.predict_anchors(codes)
    pts = torch.cat([anchors[:, :3], anchors[:, :3] + 0.01], dim=1)
    from nphm_b200.models import _composite as C
    from nphm_b200.models.diff_operators import gradient
    x = pts.clone().requires_grad_()
    want_s, _ = C.ensemble_sdf(dec, x, codes)
    want_g = gradient(want_s, x)
    got_s, got_g, _ = _assembled_values_and_gradients(dec, pts, codes, None)
    assert torch.isfinite(got_g).all()
    torch.testing.assert_close(got_s, want_s, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(got_g, want_g, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize('assembled', [False, True], ids=['composite', 'blend'])
def test_fp32_step_matches_the_reference_golden(assembled, monkeypatch):
    g = load_golden('train_ensemble.npz')
    dec = make_ensemble(0).train()
    assert S.state_dict_sha256(dec) == str(g['sha256'])
    batch, codes = _golden_batch(g, torch.float32)
    from nphm_b200.models import loss_functions as L
    codes = codes.requires_grad_()
    with monkeypatch.context() as m:
        if assembled:
            m.setattr(L, '_composite_values_and_gradients', _assembled_values_and_gradients)
        losses = L.actual_compute_loss(batch, dec, codes)
    E.total_loss(losses).backward()
    full, sampled = E.gradient_record(dec, codes)
    # same bounds as the NPM step's composite check (test_train_shape_cpu.py)
    S.check_against_golden(g, losses, full, sampled, rtol=1e-4, native=False)
