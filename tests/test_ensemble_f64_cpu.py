"""The float64 reference of tests/ensemble_f64_common.py against the composite module, the point sets against what they are
meant to reach, and which ensembles the fused fitters take (no GPU needed)."""
import copy

import pytest
import torch

import ensemble_f64_common as E

torch.set_default_dtype(torch.float32)


def _composite64(dec):
    ref = copy.deepcopy(dec).double()
    ref.anchors = ref.anchors.double()
    return ref


@pytest.mark.parametrize('name', list(E.CONFIGS))
def test_reference_equals_the_composite_module(name):
    """Member outputs, anchors and the blended SDF (training mode and one eval-mode call) to 1e-12 in float64."""
    from nphm_b200.models import _composite
    dec = E.make_decoder(name)
    ref = _composite64(dec)
    P = E.Params(dec, torch.float64)
    z = E.latent(name).double()
    xyz, _ = E.mixed_points(P, z, 130)
    out, s, anc = E.sdf(P, xyz, z, with_members=True)
    with torch.no_grad():
        want, want_anc = _composite.ensemble_sdf(ref, xyz[None], z[None, None])
        _, local, cond = _composite.member_frames(ref, xyz[None], z[None, None].expand(1, xyz.shape[0], -1))
        want_s = ref.ensembled_deep_sdf(local, cond)[:, 0, :, 0].T
    assert float((anc - want_anc[0]).abs().max()) <= 1e-12
    assert float((s - want_s).abs().max()) <= 1e-12 * max(1.0, float(want_s.abs().max()))
    assert float((out - want[0, :, 0]).abs().max()) <= 1e-12
    ref.eval()
    with torch.no_grad():
        want_q, _ = _composite.ensemble_sdf(ref, xyz[None], z[None, None])
    got_q = E.sdf(P, xyz, z, period=xyz.shape[0])
    assert float((got_q - want_q[0, :, 0]).abs().max()) <= 1e-12


def test_regularisers_equal_the_fitters_composite_terms():
    from nphm_b200.models.fitting import _latent_regularisers
    for name in ('prod', 'api', 'symm0'):
        dec = E.make_decoder(name)
        P = E.Params(dec, torch.float64)
        z = E.latent(name, seed=3).double()
        got = E.regularisers(P, z)
        want = _latent_regularisers(_composite64(dec), z.reshape(1, 1, -1))
        for g, k in zip(got, ('reg_global', 'reg_loc', 'reg_unobserved', 'symm_dist')):
            if k == 'symm_dist' and not P.n_symm:
                assert float(g) == 0.0                   # the kernels' convention; torch's mean over no pairs is NaN
                continue
            assert abs(float(g) - float(want[k])) <= 1e-12 * max(1.0, abs(float(want[k]))), (name, k)


def test_quirk_rows_by_period():
    assert E.quirk_rows(5, 0).tolist() == [False] * 5
    assert E.quirk_rows(5, 1).tolist() == [True] * 5
    assert E.quirk_rows(7, 3).tolist() == [False, False, True, False, False, True, False]
    assert E.quirk_rows(129, 128).nonzero().reshape(-1).tolist() == [127]


@pytest.mark.parametrize('name', list(E.CONFIGS))
def test_point_sets_reach_every_member_and_the_background(name):
    """Every local member, mirrored ones included, is the largest blend weight of one of its near rows; the background
    member is that of every far row, where the local weights are exactly zero in fp32."""
    dec = E.make_decoder(name)
    P = E.Params(dec, torch.float64)
    z = E.latent(name).double()
    near, owner, box, far = E.point_sets(P, z)
    anc = E.anchors(P, z)
    top = E.blend_weights(P, near, anc).argmax(dim=1)
    missing = sorted(set(range(P.n_loc)) - set(top[top == owner].tolist()))
    assert not missing, (name, missing)
    assert bool((E.blend_weights(P, far, anc).argmax(dim=1) == P.n_loc).all())
    w32 = E.blend_weights(E.Params(dec, torch.float32), far.float(), anc.float())
    assert bool((w32[:, :P.n_loc] == 0).all())
    assert float((anc[None] - far[:, None]).norm(dim=-1).min()) > 1.1


@pytest.mark.parametrize('name', [k for k, c in E.CONFIGS.items() if c[6] == 'stack'])
def test_rescaled_weights_reach_the_softplus_kink_and_its_saturated_end(name):
    dec = E.make_decoder(name)
    P = E.Params(dec, torch.float64)
    z = E.latent(name).double()
    xyz, _ = E.mixed_points(P, z, 300)
    pre = []
    E.members(P, xyz, z, preacts=pre)
    hidden = torch.cat([t.reshape(-1) for per_member in pre for t in per_member[:-1]]) * E.BETA
    assert int((hidden.abs() < 1).sum()) > 0, name               # the kink
    assert int((hidden > 20).sum()) > 0, name                    # the linear end (softplus threshold 20)
    assert int((hidden < -20).sum()) > 0, name                   # the flat end: derivative below exp(-20)


# ------------------------------------------------------------------------------------------------ fused fitter predicate
@pytest.mark.parametrize('name,training,grad_points,want', [
    ('prod', True, False, True), ('prod', True, True, True), ('prod', False, False, True), ('prod', False, True, True),
    ('tc-64m', False, True, True),
    ('tc-2m', True, True, True), ('tc-2m', False, True, True),
    ('tc-64m-nosymm', True, True, True), ('tc-64m-nosymm', False, True, True),
    ('tc-allpairs', False, True, True), ('tc-split-32-64', False, True, True), ('tc-split-80-16', False, True, True),
    # 65 members at the tensor-core widths: the FFMA step only (training mode, no point gradients)
    ('tc-65m', True, False, True), ('tc-65m', True, True, False), ('tc-65m', False, False, False),
    ('api', True, False, True), ('api', True, True, False), ('api', False, False, False),
    ('ffma-widest', True, False, True), ('ffma-over', True, False, False),
    ('depth3', True, False, False), ('depth6', True, False, False),
])
def test_fused_fit_predicate(name, training, grad_points, want):
    from nphm_b200.models.fitting import fused_fit_config
    dec = E.make_decoder(name).train(training)
    assert fused_fit_config(dec, grad_points) == want


def test_fused_fit_predicate_rejects_the_ffma_step_beyond_its_shared_memory():
    """hidden 256 with a condition of 96 (not the tensor-core width) needs 1067 rows of the FFMA step: autograd."""
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from nphm_b200.models.fitting import FFMA_FIT_MAX_ROWS, ffma_fit_rows, fused_fit_config
    assert ffma_fit_rows(256, 96) == 1067 > FFMA_FIT_MAX_ROWS == 908
    assert ffma_fit_rows(204, 48) == 907 and ffma_fit_rows(205, 48) == 911
    dec = FastEnsembleDeepSDFMirrored(64, 32, 39, 16, E.mean_anchors(39).float().reshape(1, 1, 39, 3), 256, 4, pos_mlp_dim=64)
    assert not fused_fit_config(dec.train())
