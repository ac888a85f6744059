"""GPU tests of the native training path through the spatial gradient (nphm_mlp_sdfgrad_forward / _backward,
DeepSDF.forward_with_gradient_native): values, gradients and every parameter / input gradient against a float64 composite
double backward, the stage-1 loss against the composite path and the reference golden, a few optimizer steps, and the guards
(determinism, workspace check, no double backward, in-place change, unsupported decoders)."""
import copy

import pytest
import torch

import shape_common as S
from conftest import load_golden

pytestmark = pytest.mark.gpu


def _stack(kind, device):
    from nphm_b200.models.deepSDF import DeepSDF
    if kind == 'npm':          # npm.yaml: 515 -> 1024 x 8 -> 1, geometric init
        return S.make_decoder(DeepSDF, device)
    torch.manual_seed({'member': 16, 'odd': 14}[kind])
    if kind == 'member':       # one member of the NPHM ensemble: 99 -> 200 -> 101 -> [skip] 200 -> 200 -> 1
        return DeepSDF(lat_dim=96, hidden_dim=200, nlayers=4).to(device)
    return DeepSDF(lat_dim=21, hidden_dim=88, nlayers=5).to(device)


def _params(dec):
    ps = []
    for i in range(dec.num_layers - 1):
        lin = getattr(dec, 'lin%d' % i)
        ps += [lin.weight, lin.bias]
    return ps


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-300)).item()


def _native(dec, xyz, cond, s_bar, g_bar):
    x, c = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
    sdf, g = dec.forward_with_gradient_native(x, c)
    grads = torch.autograd.grad((sdf, g), [x, c] + _params(dec), (s_bar, g_bar))
    return sdf, g, grads


def _composite64(d, xyz, cond, s_bar, g_bar):
    """float64 reference on a float64 copy `d`: the composite forward, gradient() with create_graph=True, then the double
    backward."""
    x, c = xyz.double().requires_grad_(), cond.double().requires_grad_()
    B, N, _ = xyz.shape
    sdf = d._forward_composite(x, c[:, None, :].expand(B, N, c.shape[-1]))
    g = torch.autograd.grad(sdf, x, torch.ones_like(sdf), create_graph=True)[0]
    grads = torch.autograd.grad((sdf, g), [x, c] + _params(d), (s_bar.double(), g_bar.double()))
    return sdf, g, grads


@pytest.mark.parametrize('kind', ['npm', 'member', 'odd'])
def test_sdfgrad_function_matches_float64_double_backward(cuda_device, kind):
    dec = _stack(kind, cuda_device)
    dec64 = copy.deepcopy(dec).double()                    # before the native engine is attached
    gen = torch.Generator(device=cuda_device).manual_seed(3)
    for B, N in ((3, 100), (2, 333), (2, 1000)):
        xyz = (torch.rand(B, N, 3, device=cuda_device, generator=gen) - 0.5) * 1.5
        cond = torch.randn(B, dec.lat_dim, device=cuda_device, generator=gen) * 0.1
        s_bar = torch.randn(B, N, 1, device=cuda_device, generator=gen)
        g_bar = torch.randn(B, N, 3, device=cuda_device, generator=gen)
        for scale in (1.0, 1e-6):
            sdf_n, g_n, gn = _native(dec, xyz, cond, s_bar * scale, g_bar * scale)
            sdf_c, g_c, gc = _composite64(dec64, xyz, cond, s_bar * scale, g_bar * scale)
            assert (sdf_n.double() - sdf_c).abs().max().item() <= 1e-5, (kind, B, N)
            err = _rel(g_n, g_c)
            assert err <= 1e-4, (kind, B, N, 'grad_x sdf', err)
            names = ['xyz', 'cond'] + ['lin%d.%s' % (i // 2, 'weight' if i % 2 == 0 else 'bias') for i in range(len(gn) - 2)]
            for name, a, b in zip(names, gn, gc):
                err = _rel(a, b)
                print('%s B=%d N=%d scale=%g %s rel %.3g' % (kind, B, N, scale, name, err))
                assert err <= 5e-4, (kind, B, N, scale, name, err)


def _loss_setup(device, B=4, sizes=(150, 30, 160, 40)):
    from nphm_b200.models.deepSDF import DeepSDF
    dec = S.make_decoder(DeepSDF, device)
    b = S.make_batch(B=B, sizes=sizes, seed=9)
    torch.manual_seed(21)
    codes = torch.nn.Embedding(8, 512, max_norm=1.0, sparse=True).to(device)
    with torch.no_grad():
        codes.weight.mul_(0.05)
    batch = {k: torch.from_numpy(v).to(device) for k, v in b.items() if k != 'codes'}
    idx = torch.tensor([[1], [3], [0], [6]][:B], device=device)
    return dec, codes, batch, idx


def _loss_step(dec, codes, batch, idx, native):
    from nphm_b200.models.loss_functions import actual_compute_loss
    losses = actual_compute_loss(batch, dec, codes(idx), native=native)
    return losses, S.total_loss(losses)


def test_shape_loss_native_matches_composite(cuda_device):
    dec, codes, batch, idx = _loss_setup(cuda_device)
    out = {}
    for native in (True, False):
        d, e = copy.deepcopy(dec), copy.deepcopy(codes)
        losses, tot = _loss_step(d, e, batch, idx, native)
        tot.backward()
        grads = {n: p.grad for n, p in d.named_parameters()}
        grads['codes'] = e.weight.grad.to_dense()
        out[native] = ({k: v.item() for k, v in losses.items()}, grads)
    for k in out[False][0]:
        err = abs(out[True][0][k] - out[False][0][k]) / abs(out[False][0][k])
        print('shape loss %s rel %.3g' % (k, err))
        assert err <= S.loss_rtol(k), (k, err)
    for name, ref in out[False][1].items():
        err = _rel(out[True][1][name], ref)
        print('shape loss grad %s rel %.3g' % (name, err))
        assert err <= 5e-4, (name, err)


def test_native_shape_step_matches_the_reference_golden(cuda_device):
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('train_shape.npz')
    dec = S.make_decoder(DeepSDF, cuda_device)
    losses, codes = S.run_step(dec, g, cuda_device, native=True)
    full, sampled = S.gradient_record(dec, codes)
    S.check_against_golden(g, losses, full, sampled, rtol=5e-4)


def test_shape_training_trajectory_native_matches_composite(cuda_device):
    dec, codes, batch, idx = _loss_setup(cuda_device)
    start = {n: p.detach().clone() for n, p in dec.named_parameters()}
    final = {}
    for native in (True, False):
        d, e = copy.deepcopy(dec), copy.deepcopy(codes)
        opt = torch.optim.AdamW(d.parameters(), lr=5e-4, weight_decay=0.02)
        opt_lat = torch.optim.SparseAdam(e.parameters(), lr=1e-3)
        for _ in range(5):
            opt.zero_grad()
            opt_lat.zero_grad()
            _, tot = _loss_step(d, e, batch, idx, native)
            tot.backward()
            torch.nn.utils.clip_grad_norm_(d.parameters(), max_norm=0.1)
            opt.step()
            opt_lat.step()
        final[native] = {n: p.detach().clone() for n, p in d.named_parameters()}
    change = torch.cat([(final[False][n] - start[n]).reshape(-1) for n in start]).norm().item()
    diff = torch.cat([(final[True][n] - final[False][n]).reshape(-1) for n in start]).norm().item()
    print('trajectory: total change %.4g, native - composite %.4g' % (change, diff))
    assert change > 0 and diff <= 1e-3 * change, (diff, change)


def test_sdfgrad_guards(cuda_device):
    from nphm_b200 import _native
    from nphm_b200.models.deepSDF import DeepSDF
    dec = _stack('member', cuda_device)
    eng = dec.engine()
    B, N = 2, 300
    xyz = torch.rand(B, N, 3, device=cuda_device) - 0.5
    cond = torch.randn(B, dec.lat_dim, device=cuda_device) * 0.1
    s_bar = torch.randn(B, N, 1, device=cuda_device) * 1e-5
    g_bar = torch.randn(B, N, 3, device=cuda_device) * 1e-5
    _, _, ws = eng.sdfgrad_forward(xyz, cond)
    r1 = eng.sdfgrad_backward(ws, s_bar, g_bar, want_xyz=True)
    r2 = eng.sdfgrad_backward(ws, s_bar, g_bar, want_xyz=True)
    for a, b in zip(r1[0] + r1[1] + [r1[2], r1[3]], r2[0] + r2[1] + [r2[2], r2[3]]):
        assert torch.equal(a, b)                           # bitwise: fixed reduction order, no float atomics
    # a workspace whose size does not match the stated shape is rejected (NPHM_ERR_INVALID; the size is what is checked:
    # N + 128 points need one more 128-row tile)
    L = _native.lib()
    g_cond = torch.empty(B, dec.lat_dim, device=cuda_device)
    big_s, big_g = torch.zeros(B, N + 128, 1, device=cuda_device), torch.zeros(B, N + 128, 3, device=cuda_device)
    stream = torch.cuda.current_stream().cuda_stream
    for nbytes, n, gs, gg in ((ws.numel(), N + 128, big_s, big_g), (ws.numel() - 256, N, s_bar, g_bar)):
        rc = L.nphm_mlp_sdfgrad_backward(eng._h, gs.data_ptr(), gg.data_ptr(), ws.data_ptr(), nbytes, B, n, None, None,
                                         g_cond.data_ptr(), None, stream)
        assert rc == -1, (nbytes, n)
    rc = L.nphm_mlp_sdfgrad_backward(eng._h, s_bar.data_ptr(), g_bar.data_ptr(), ws.data_ptr(), ws.numel(), B, N, None, None,
                                     g_cond.data_ptr(), None, stream)
    assert rc == 0
    assert torch.equal(g_cond, r1[2])
    # more than one output: NPHM_ERR_UNSUPPORTED from the library, ValueError from the module
    torch.manual_seed(1)
    dec3 = DeepSDF(lat_dim=21, hidden_dim=88, nlayers=5, out_dim=3).to(cuda_device)
    with pytest.raises(_native.NativeError, match=r'\(-3\)'):
        dec3.engine().sdfgrad_forward(xyz, torch.zeros(B, 21, device=cuda_device))
    # first order only
    x = xyz.clone().requires_grad_()
    sdf, g = dec.forward_with_gradient_native(x, cond)
    with pytest.raises(RuntimeError, match='double backward'):
        torch.autograd.grad((sdf.sum() + g.square().sum()), x, create_graph=True)
    # a parameter changed in place between forward and backward is caught by autograd's version check
    sdf, g = dec.forward_with_gradient_native(x, cond)
    with torch.no_grad():
        dec.lin0.weight.add_(0.0)
    with pytest.raises(RuntimeError):
        (sdf.sum() + g.sum()).backward()


@pytest.mark.parametrize('variant', ['out_dim3', 'relu', 'posenc'])
def test_native_shape_loss_rejects_unsupported_decoders(cuda_device, variant):
    from nphm_b200.models.deepSDF import DeepSDF
    kw = {'out_dim3': dict(out_dim=3), 'relu': dict(beta=0), 'posenc': dict(num_freq_bands=2)}[variant]
    torch.manual_seed(1)
    dec = DeepSDF(lat_dim=21, hidden_dim=88, nlayers=5, **kw).to(cuda_device)
    b = S.make_batch(B=2, sizes=(10, 5, 10, 5))
    batch = {k: torch.from_numpy(v).to(cuda_device) for k, v in b.items() if k != 'codes'}
    codes = torch.zeros(2, 1, 21, device=cuda_device, requires_grad=True)
    from nphm_b200.models.loss_functions import actual_compute_loss
    with pytest.raises(ValueError):
        actual_compute_loss(batch, dec, codes, native=True)
    with pytest.raises(ValueError):
        dec.forward_with_gradient_native(batch['points_face'], codes)
