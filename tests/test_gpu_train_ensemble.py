"""Stage-1 training of the NPHM ensemble on the native member passes (nphm_ensemble_sdfgrad_*, one launch per pass for all
members) with the anchors, frames and blend in autograd (FastEnsembleDeepSDFMirrored.forward_with_gradient_native,
actual_compute_loss(..., native=True)).  Checked against 24 single-set DeepSDF calls, a float64 composite double backward,
the reference's step (train_ensemble.npz, losses.npz), a composite trajectory, for determinism, host syncs and its guards."""
import copy

import numpy as np
import pytest
import torch

import ensemble_train_common as E
import shape_common as S
from conftest import load_golden, make_ensemble

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _codes(B, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (0.05 * torch.randn(B, 1, 64 + 40 * 32, generator=g, dtype=torch.float64)).to(DEV, dtype)


def _points(dec, B, N, seed, spread=0.05, dtype=torch.float32):
    """Points scattered around the mean anchors."""
    g = torch.Generator().manual_seed(seed)
    a = dec.mean_anchors('cpu', torch.float64)
    idx = torch.randint(0, a.shape[0], (B, N), generator=g)
    return (a[idx] + spread * torch.randn(B, N, 3, generator=g, dtype=torch.float64)).to(DEV, dtype)


def _grads(dec, codes):
    out = {'codes': codes.grad.detach().double().clone()}
    out.update({k: p.grad.detach().double().clone() for k, p in dec.named_parameters()})
    return out


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300))


def test_batched_members_match_single_set_calls():
    """The native member Function against 24 single-set nphm_mlp_sdfgrad_* calls on DeepSDF(96, 200, 4) stacks."""
    from nphm_b200.models import _composite as C
    from nphm_b200.models.EnsembledDeepSDF import _NativeEnsembleSdfGradFn
    from nphm_b200.models.deepSDF import DeepSDF
    dec = make_ensemble(0, device=DEV).train()
    B, N = 2, 150
    codes = _codes(B, 1)
    xyz = _points(dec, B, N, 2)
    with torch.no_grad():
        _, local, cond = C.member_frames(dec, xyz, codes)
    local, cond = local.contiguous(), cond[:, :, 0].contiguous()
    e = dec.ensembled_deep_sdf
    params = [p for i in range(5) for p in (getattr(e, 'lin%d' % i).weight, getattr(e, 'lin%d' % i).bias)]
    gen = torch.Generator(device=DEV).manual_seed(3)
    K = local.shape[0]
    sets = dec.ensembled_deep_sdf.lin0._set_of_member.tolist()
    # upstreams many orders of magnitude apart between the weight sets, as the blend weights make them.  Both members of a
    # set get the same largest magnitude, a power of two: the set's fp16 scale is then the one a single-set call picks
    # for each member, and the comparison sees the batching alone.
    gs = torch.randn(K, B, N, device=DEV, generator=gen)
    gg = torch.randn(K, B, N, 3, device=DEV, generator=gen)
    for k in range(K):
        top = max(float(gs[k].abs().max()), float(gg[k].abs().max()))
        mag = 2.0 ** -(sets[k] * 20 // 24)
        gs[k] = gs[k] / top * mag
        gg[k] = gg[k] / top * mag
    xl, cd = local.clone().requires_grad_(), cond.clone().requires_grad_()
    s, g = _NativeEnsembleSdfGradFn.apply(dec.engine(), xl, cd, *params)
    torch.autograd.backward([s, g], [gs, gg])
    ref_w = [torch.zeros_like(p) for p in params]
    stack = DeepSDF(lat_dim=96, hidden_dim=200, nlayers=4, geometric_init=False).to(DEV).train()
    ref = {'s': [], 'g': [], 'cond': [], 'xyz': []}
    for k in range(K):
        with torch.no_grad():
            for i in range(5):
                getattr(stack, 'lin%d' % i).weight.copy_(params[2 * i][sets[k]])
                getattr(stack, 'lin%d' % i).bias.copy_(params[2 * i + 1][sets[k]])
        eng = stack.engine()
        s1, g1, ws = eng.sdfgrad_forward(local[k], cond[k])
        gw, gb, gc, gx = eng.sdfgrad_backward(ws, gs[k][..., None], gg[k], want_xyz=True)
        for name, v in (('s', s1[..., 0]), ('g', g1), ('cond', gc), ('xyz', gx)):
            ref[name].append(v)
        for i in range(5):
            ref_w[2 * i][sets[k]] += gw[i]
            ref_w[2 * i + 1][sets[k]] += gb[i]
    # every tensor within 1e-6 of its max abs
    for name, got in (('s', s.detach()), ('g', g.detach()), ('cond', cd.grad), ('xyz', xl.grad)):
        assert _rel(got, torch.stack(ref[name])) <= 1e-6, (name, _rel(got, torch.stack(ref[name])))
    # weight and bias gradients: 1e-5.  The single-set reference rounds each member's gradient to fp32 and then adds the
    # two members of a mirrored set, each summed over its own row splits; the batched launch sums both members' rows and
    # both operand pairs in one sequence with other split boundaries (measured on an H100: 1.1e-6 of max abs on
    # lin0.weight, 2.0e-6 on lin1.weight, 6.6e-6 on lin3.weight).  Against float64 both are held to 5e-5 below.
    for i, p in enumerate(params):
        assert _rel(p.grad, ref_w[i]) <= 1e-5, (i, _rel(p.grad, ref_w[i]))


def _loss(sdf, grad, anchors, w, scale):
    return scale * ((w[0] * sdf[..., 0]).sum() + (w[1] * grad).sum() + (w[2] * anchors).sum())


@pytest.mark.parametrize('scale', [1.0, 1e-6])
def test_native_gradient_matches_float64_composite(scale):
    from nphm_b200.models import _composite as C
    from nphm_b200.models.diff_operators import gradient
    dec = make_ensemble(0, device=DEV).train()
    ref = copy.deepcopy(dec).double()
    ref.anchors = ref.anchors.double()
    B, N = 2, 120
    codes = _codes(B, 4)
    xyz = _points(dec, B, N, 5)
    # batch element 1 also holds points far from every anchor: there the local members' weights underflow to 0
    xyz[1, -20:] = torch.tensor([2.5, 2.5, 2.5], device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(6)
    w = [torch.randn(B, N, device=DEV, generator=gen), torch.randn(B, N, 3, device=DEV, generator=gen),
         torch.randn(B, 39, 3, device=DEV, generator=gen)]
    c32 = codes.clone().requires_grad_()
    sdf, grad, anchors = dec.forward_with_gradient_native(xyz, c32)
    _loss(sdf, grad, anchors, w, scale).backward()
    got = _grads(dec, c32)
    c64 = codes.double().requires_grad_()
    x64 = xyz.double().requires_grad_()
    s64, a64 = C.ensemble_sdf(ref, x64, c64)
    g64 = gradient(s64, x64)
    _loss(s64, g64, a64, [v.double() for v in w], scale).backward()
    want = _grads(ref, c64)
    for k, v in want.items():
        assert torch.isfinite(got[k]).all(), k
        assert _rel(got[k], v) <= 5e-5, (k, _rel(got[k], v))


def test_underflowed_members_get_exactly_zero_gradients():
    """Points so far from the anchors that only the global member has weight: every other set's gradient is exactly 0."""
    dec = make_ensemble(0, device=DEV).train()
    B, N = 2, 64
    codes = _codes(B, 7).requires_grad_()
    xyz = torch.full((B, N, 3), 3.0, device=DEV) + 0.1 * torch.randn(B, N, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    sdf, grad, anchors = dec.forward_with_gradient_native(xyz, codes)
    (sdf.sum() + grad.square().sum()).backward()
    e = dec.ensembled_deep_sdf
    for i in range(5):
        for p in (getattr(e, 'lin%d' % i).weight, getattr(e, 'lin%d' % i).bias):
            assert torch.isfinite(p.grad).all()
            assert bool((p.grad[:-1] == 0).all()), i                 # every set but the global member's
            assert float(p.grad[-1].abs().max()) > 0, i


def _golden_batch(g, prefix, keys):
    return {k: torch.from_numpy(g[prefix + k]).to(DEV) for k in keys}


def test_native_step_matches_the_reference_golden():
    g = load_golden('train_ensemble.npz')
    dec = make_ensemble(0, device=DEV).train()
    assert S.state_dict_sha256(dec) == str(g['sha256'])
    from nphm_b200.models.loss_functions import actual_compute_loss
    batch = _golden_batch(g, 'batch_', E.BATCH_KEYS)
    codes = torch.from_numpy(g['batch_codes']).to(DEV).requires_grad_()
    losses = actual_compute_loss(batch, dec, codes, native=True)
    E.total_loss(losses).backward()
    full, sampled = E.gradient_record(dec, codes)
    # same bound as the NPM step's native check (test_gpu_train_shape.py)
    S.check_against_golden(g, losses, full, sampled, rtol=5e-4)


def test_native_losses_match_the_reference_on_the_losses_batch():
    g = load_golden('losses.npz')
    dec = make_ensemble(0, device=DEV).train()
    from nphm_b200.models.loss_functions import actual_compute_loss
    keys = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far', 'normals_face', 'normals_non_face', 'gt_anchors')
    batch = _golden_batch(g, 'gpu_', keys)
    cond = torch.from_numpy(g['gpu_cond']).to(DEV).requires_grad_()
    got = actual_compute_loss(batch, dec, cond, native=True)
    assert got['surf_sdf'].requires_grad and got['grad'].requires_grad
    for k, v in zip([str(n) for n in g['gpu_loss_names']], g['gpu_loss_values']):
        tol = 1e-4 if k in ('surf_sdf', 'space_sdf') else 1e-5
        assert abs(float(got[k].detach()) - v) <= tol * abs(v), (k, float(got[k].detach()), v)


def test_ten_steps_track_the_composite_trajectory():
    from nphm_b200.models.loss_functions import actual_compute_loss
    g = load_golden('train_ensemble.npz')
    batch = _golden_batch(g, 'batch_', E.BATCH_KEYS)
    runs = {}
    for native in (True, False):
        dec = make_ensemble(0, device=DEV).train()
        codes = torch.nn.Parameter(torch.from_numpy(g['batch_codes']).to(DEV))
        opt = torch.optim.Adam([{'params': dec.parameters(), 'lr': 5e-4}, {'params': [codes], 'lr': 1e-3}])
        hist = []
        for _ in range(10):
            opt.zero_grad()
            losses = actual_compute_loss(batch, dec, codes, native=native)
            tot = E.total_loss(losses)
            tot.backward()
            opt.step()
            hist.append(float(tot.detach()))
        runs[native] = (np.array(hist), codes.detach().clone())
    (hn, cn), (hc, cc) = runs[True], runs[False]
    # bounds: the losses to 1e-3 relative, the codes (10 Adam steps of lr 1e-3, at most 1e-2 of travel) to 1e-3
    assert np.abs(hn - hc).max() <= 1e-3 * np.abs(hc).max(), (hn, hc)
    assert float((cn - cc).abs().max()) <= 1e-3


def test_backward_is_deterministic_and_sync_free():
    from nphm_b200.models.loss_functions import actual_compute_loss
    g = load_golden('train_ensemble.npz')
    batch = _golden_batch(g, 'batch_', E.BATCH_KEYS)
    dec = make_ensemble(0, device=DEV).train()
    dec.engine()                                          # weights packed before the checked calls
    grads = []
    for run in range(2):
        dec.zero_grad(set_to_none=True)
        codes = torch.from_numpy(g['batch_codes']).to(DEV).requires_grad_()
        torch.cuda.synchronize()
        if run == 1:
            torch.cuda.set_sync_debug_mode('error')
        try:
            losses = actual_compute_loss(batch, dec, codes, native=True)
            E.total_loss(losses).backward()
        finally:
            torch.cuda.set_sync_debug_mode('default')
        grads.append(_grads(dec, codes))
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), k


def test_guards():
    from nphm_b200 import _native
    from nphm_b200.models import _composite as C
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from conftest import mean_anchors
    dec = make_ensemble(0, device=DEV).train()
    codes = _codes(1, 9)
    xyz = _points(dec, 1, 32, 10)
    # workspace of another shape
    with torch.no_grad():
        _, local, cond = C.member_frames(dec, xyz, codes)
    eng = dec.engine()
    s, gr, ws = eng.sdfgrad_forward(local, cond[:, :, 0])
    shapes = [tuple(getattr(dec.ensembled_deep_sdf, 'lin%d' % i).weight.shape) for i in range(5)]
    with pytest.raises(_native.NativeError):
        eng.sdfgrad_backward(ws[:-256], torch.ones_like(s), torch.ones_like(gr), shapes)
    # double backward
    c = codes.clone().requires_grad_()
    sdf, grad, _ = dec.forward_with_gradient_native(xyz, c)
    with pytest.raises(RuntimeError, match='first order'):
        torch.autograd.grad(grad.square().sum(), c, create_graph=True)
    # eval mode, CPU, per-point codes
    with pytest.raises(ValueError, match='training mode'):
        dec.eval().forward_with_gradient_native(xyz, codes)
    dec.train()
    with pytest.raises(ValueError, match='CUDA'):
        make_ensemble(0).train().forward_with_gradient_native(xyz.cpu(), codes.cpu())
    with pytest.raises(ValueError, match='one code per batch element'):
        dec.forward_with_gradient_native(xyz, codes.repeat(1, 32, 1).contiguous())
    # a stack the native builder rejects (11 hidden layers)
    deep = FastEnsembleDeepSDFMirrored(lat_dim_glob=64, lat_dim_loc=32, n_loc=39, n_symm_pairs=16, anchors=mean_anchors(),
                                       hidden_dim=200, n_layers=11, pos_mlp_dim=256).to(DEV).train()
    deep.anchors = deep.anchors.to(DEV)
    assert not deep.sdfgrad_supported(xyz, codes)
    with pytest.raises(ValueError, match='native builder'):
        deep.forward_with_gradient_native(xyz, codes)
    # no_grad keeps the evaluation path; CPU keeps the composite path
    from nphm_b200.models.loss_functions import actual_compute_loss
    g = load_golden('train_ensemble.npz')
    batch = _golden_batch(g, 'batch_', E.BATCH_KEYS)
    with torch.no_grad():
        ev = actual_compute_loss(batch, dec, torch.from_numpy(g['batch_codes']).to(DEV), native=True)
    assert not ev['surf_sdf'].requires_grad
