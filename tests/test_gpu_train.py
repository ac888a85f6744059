"""GPU tests of the native first-order training path (nphm_mlp_train_forward / _backward, tc_wgrad.cu): values and every
gradient against autograd through the composite PyTorch forward, the stage-2 loss and a few optimizer steps against the
composite path, and the guards (determinism, no double backward, workspace check)."""
import copy

import pytest
import torch
import torch.nn.functional as F

from conftest import make_deformation

pytestmark = pytest.mark.gpu


def _stack(kind, device):
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed({'deform': 10, 'npm': 12, 'odd': 14}[kind])
    if kind == 'deform':
        return make_deformation(device).defDeepSDF, 2e-4
    if kind == 'npm':          # -mode npm expression decoder: condition 712, 715 -> 1024 x 8 -> 3
        return DeepSDF(lat_dim=712, hidden_dim=1024, nlayers=8, geometric_init=False, out_dim=3).to(device), 5e-4
    return DeepSDF(lat_dim=21, hidden_dim=88, nlayers=5, out_dim=1).to(device), 2e-4


def _params(dec):
    ps = []
    for i in range(dec.num_layers - 1):
        lin = getattr(dec, 'lin%d' % i)
        ps += [lin.weight, lin.bias]
    return ps


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def _both(dec, xyz, cond, noise, g):
    """(native out, native grads), (composite out, composite grads) w.r.t. (xyz, cond, lin params)."""
    ps = _params(dec)
    xn, cn = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
    out_n = dec._native_train(xn, cn, noise)
    gn = torch.autograd.grad(out_n, [xn, cn] + ps, g)
    xc, cc = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
    B, N, _ = xyz.shape
    c = cc[:, None, :].expand(B, N, cc.shape[-1])
    if noise is not None:
        c = c + F.pad(noise, (0, cc.shape[-1] - noise.shape[-1]))
    out_c = dec._forward_composite(xc, c)
    gc = torch.autograd.grad(out_c, [xc, cc] + ps, g)
    return (out_n, gn), (out_c, gc)


@pytest.mark.parametrize('kind', ['deform', 'npm', 'odd'])
@pytest.mark.parametrize('with_noise', [False, True])
def test_native_train_function_matches_autograd(cuda_device, kind, with_noise):
    dec, tol = _stack(kind, cuda_device)
    dec.train()
    gen = torch.Generator(device=cuda_device).manual_seed(3)
    for B, N in ((3, 100), (2, 333), (2, 1000)):
        xyz = (torch.rand(B, N, 3, device=cuda_device, generator=gen) - 0.5) * 1.5
        cond = torch.randn(B, dec.lat_dim, device=cuda_device, generator=gen) * 0.1
        nd = min(32, dec.lat_dim - 8)
        noise = torch.randn(B, N, nd, device=cuda_device, generator=gen) / 200 if with_noise else None
        g = torch.randn(B, N, dec.out_dim_net, device=cuda_device, generator=gen)
        for g_scale in (1.0, 1e-6):
            (out_n, gn), (out_c, gc) = _both(dec, xyz, cond, noise, g * g_scale)
            assert (out_n - out_c).abs().max().item() <= 1e-5, (kind, B, N)
            names = ['xyz', 'cond'] + ['lin%d.%s' % (i // 2, 'weight' if i % 2 == 0 else 'bias') for i in range(len(gn) - 2)]
            for name, a, b in zip(names, gn, gc):
                err = _rel(a, b)
                print('%s N=%d noise=%s scale=%g %s rel %.3g' % (kind, N, with_noise, g_scale, name, err))
                assert err <= tol, (kind, B, N, g_scale, name, err)


def test_native_train_guards(cuda_device):
    from nphm_b200 import _native
    dec, _ = _stack('deform', cuda_device)
    eng = dec.engine()
    B, N = 2, 300
    xyz = torch.rand(B, N, 3, device=cuda_device) - 0.5
    cond = torch.randn(B, dec.lat_dim, device=cuda_device) * 0.1
    noise = torch.randn(B, N, 32, device=cuda_device) / 200
    g = torch.randn(B, N, 3, device=cuda_device) * 1e-5
    _, ws = eng.train_forward(xyz, cond, noise)
    r1 = eng.train_backward(ws, g, 32, want_xyz=True)
    r2 = eng.train_backward(ws, g, 32, want_xyz=True)
    for a, b in zip(r1[0] + r1[1] + [r1[2], r1[3]], r2[0] + r2[1] + [r2[2], r2[3]]):
        assert torch.equal(a, b)                           # bitwise: fixed reduction order, no float atomics
    # a workspace that does not match the stated shape (points, noise columns, size) is rejected
    L = _native.lib()
    gw = torch.empty(B, N + 1, 3, device=cuda_device)
    g_cond = torch.empty(B, dec.lat_dim, device=cuda_device)
    stream = torch.cuda.current_stream().cuda_stream
    for nbytes, nd, n, grad in ((ws.numel(), 32, N + 1, gw), (ws.numel(), 0, N, g), (ws.numel() - 256, 32, N, g)):
        rc = L.nphm_mlp_train_backward(eng._h, grad.data_ptr(), ws.data_ptr(), nbytes, nd, B, n, None, None, g_cond.data_ptr(),
                                       None, stream)
        assert rc == -1, (nbytes, nd, n)                   # NPHM_ERR_INVALID
    rc = L.nphm_mlp_train_backward(eng._h, g.data_ptr(), ws.data_ptr(), ws.numel(), 32, B, N, None, None, g_cond.data_ptr(),
                                   None, stream)
    assert rc == 0
    assert torch.equal(g_cond, r1[2])
    # first order only
    x = xyz.clone().requires_grad_()
    out = dec._native_train(x, cond, noise)
    with pytest.raises(RuntimeError, match='double backward'):
        torch.autograd.grad(out.square().sum(), x, create_graph=True)
    # a parameter changed in place between forward and backward is caught by autograd's version check
    out = dec._native_train(x, cond, noise)
    with torch.no_grad():
        dec.lin0.weight.add_(0.0)
    with pytest.raises(RuntimeError):
        out.sum().backward()


def test_native_corresp_step_matches_the_reference_golden(cuda_device):
    """One stage-2 step of the reference (tests/golden/train_corresp.npz: compress DeformationNetwork in train mode, the
    ensemble's mlp_pos for the anchors, nphm_def.yaml lambdas) with its random draws replayed through the NATIVE path: two
    decoder calls, one backward.  Loss terms and every stored gradient against the golden."""
    import corresp_common as C
    from conftest import load_golden, make_ensemble
    from nphm_b200.models.loss_functions import compute_loss_corresp_forward
    g = load_golden('train_corresp.npz')
    dfn = make_deformation(cuda_device).train()
    dfn.anchors = dfn.anchors.to(cuda_device)             # plain attribute (not moved by .to())
    shape_dec = make_ensemble(0, device=cuda_device).train()
    lat_expr, lat_shape = C.make_embeddings(cuda_device, expr=g['weights_expr'], shape=g['weights_shape'])
    batch = {k: g['batch_' + k] for k in ('points_neutral', 'points_posed', 'gt_anchors', 'idx', 'subj_ind')}
    kinds = [str(k) for k in g['draw_kinds']]
    with C.replay_draws(kinds, [g['draw_%d' % i] for i in range(len(kinds))]):
        losses = compute_loss_corresp_forward({k: torch.from_numpy(v) for k, v in batch.items()}, dfn, shape_dec, lat_expr,
                                              lat_shape, cuda_device, native=True)
    C.total_loss(losses).backward()
    full, sampled = C.gradient_record(dfn, shape_dec, lat_expr, lat_shape, batch)
    C.check_against_golden(g, losses, full, sampled, rtol=2e-4)


def _corresp_setup(device, B=4, N=300):
    dfn = make_deformation(device).train()
    torch.manual_seed(21)
    lat_expr = torch.nn.Embedding(8, 200, max_norm=1.0, sparse=True).to(device)
    lat_shape = torch.nn.Embedding(5, 32 * 39 + 32 + 64, max_norm=1.0).to(device)
    with torch.no_grad():
        lat_expr.weight.mul_(0.3)
    gen = torch.Generator().manual_seed(5)
    pts = (torch.rand(B, N, 3, generator=gen) - 0.5) * 1.2
    batch = {'points_neutral': pts, 'points_posed': pts + 0.02 * torch.randn(B, N, 3, generator=gen),
             'gt_anchors': torch.rand(B, 39, 3, generator=gen) - 0.5,
             'idx': torch.tensor([[1], [3], [0], [6]][:B]), 'subj_ind': torch.tensor([[0], [2], [4], [1]][:B])}
    return dfn, lat_expr, lat_shape, batch


def _corresp_step(dfn, lat_expr, lat_shape, batch, native, seed=7):
    from nphm_b200.models.loss_functions import compute_loss_corresp_forward
    torch.manual_seed(seed)
    losses = compute_loss_corresp_forward(dict(batch), dfn, None, lat_expr, lat_shape, 'cuda', native=native)
    tot = losses['corresp'] * 100 + losses['loss_reg_zero'] * 0.5 + losses['lat_reg'] * 1e-4
    return losses, tot


def test_corresp_loss_native_matches_composite(cuda_device):
    dfn, lat_expr, lat_shape, batch = _corresp_setup(cuda_device)
    out = {}
    for native in (True, False):
        d, e, s = copy.deepcopy(dfn), copy.deepcopy(lat_expr), copy.deepcopy(lat_shape)
        losses, tot = _corresp_step(d, e, s, batch, native)
        tot.backward()
        grads = {n: p.grad.to_dense() for n, p in list(d.named_parameters()) + [('expr', e.weight), ('shape', s.weight)]}
        out[native] = ({k: v.item() for k, v in losses.items()}, grads)
    for k in out[False][0]:
        assert abs(out[True][0][k] - out[False][0][k]) <= 1e-5 * max(1.0, abs(out[False][0][k])), k
    for name, ref in out[False][1].items():
        err = _rel(out[True][1][name], ref)
        print('corresp grad %s rel %.3g' % (name, err))
        assert err <= 2e-4, (name, err)


def test_corresp_training_trajectory_native_matches_composite(cuda_device):
    dfn, lat_expr, lat_shape, batch = _corresp_setup(cuda_device)
    start = {n: p.detach().clone() for n, p in dfn.named_parameters()}
    final = {}
    for native in (True, False):
        d, e, s = copy.deepcopy(dfn), copy.deepcopy(lat_expr), copy.deepcopy(lat_shape)
        opt = torch.optim.AdamW(d.parameters(), lr=1e-4, weight_decay=5e-4)
        opt_lat = torch.optim.SparseAdam(e.parameters(), lr=1e-3)
        for step in range(5):
            opt.zero_grad()
            opt_lat.zero_grad()
            _, tot = _corresp_step(d, e, s, batch, native, seed=100 + step)
            tot.backward()
            torch.nn.utils.clip_grad_norm_(d.parameters(), max_norm=0.025)
            opt.step()
            opt_lat.step()
        final[native] = {n: p.detach().clone() for n, p in d.named_parameters()}
    # over all parameters (Adam's first steps move every weight by ~lr * sign(g), so an element whose gradient is at the
    # rounding level may step either way on either path: compare the whole update, not element by element)
    change = torch.cat([(final[False][n] - start[n]).reshape(-1) for n in start]).norm().item()
    diff = torch.cat([(final[True][n] - final[False][n]).reshape(-1) for n in start]).norm().item()
    print('trajectory: total change %.4g, native - composite %.4g' % (change, diff))
    assert change > 0 and diff <= 1e-3 * change, (diff, change)
