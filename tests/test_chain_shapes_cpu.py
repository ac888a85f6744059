"""The float64 reference of tests/chain_shapes_common.py against ``DeepSDF._forward_composite`` (pinned to the reference's
outputs by the goldens) on a float64 copy of every stack of the shape matrix: values, first derivatives (w.r.t. the points,
the condition and every parameter, with and without condition noise) and the double backward through grad_x s.  It also
checks that the matrix's stacks reach both ends of the softplus (the kink and the saturated region)."""
import pytest
import torch
import torch.nn.functional as F

import chain_shapes_common as C


def _composite(net, xyz, cond, noise=None):
    B, N, _ = xyz.shape
    c = cond[:, None, :].expand(B, N, cond.shape[-1])
    if noise is not None:
        c = c + F.pad(noise, (0, cond.shape[-1] - noise.shape[-1]))
    return net._forward_composite(xyz, c)


def _close(a, b, what):
    err = float((a - b).abs().max())
    assert err <= 1e-12 * max(1.0, float(b.abs().max())), (what, err)


@pytest.mark.parametrize('cfg', C.CONFIGS, ids=C.config_id)
def test_reference_equals_composite_forward_float64(cfg):
    net = C.make_stack(cfg).double()
    P = C.params_of(net, torch.float64)
    xyz, cond = C.make_inputs(cfg, 2, 5, 'cpu')
    xyz, cond = xyz.double(), cond.double()
    nd = C.noise_dims(cfg)[-1]
    noise = torch.randn(2, 5, nd, dtype=torch.float64, generator=torch.Generator().manual_seed(1)) / 200
    params = [p for Wb in ((getattr(net, 'lin%d' % l).weight, getattr(net, 'lin%d' % l).bias) for l in range(net.num_layers - 1))
              for p in Wb]
    up = torch.randn(2, 5, cfg[3], dtype=torch.float64, generator=torch.Generator().manual_seed(2))

    # values, Jacobian and the first-order VJP (with and without noise)
    out_r, J_r = C.ref_jacobian(P, xyz, cond)
    x = xyz.clone().requires_grad_()
    out_c = _composite(net, x, cond)
    J_c = torch.stack([torch.autograd.grad(out_c[..., i].sum(), x, retain_graph=True)[0] for i in range(cfg[3])], dim=-2)
    _close(out_r, out_c.detach(), 'value')
    _close(J_r, J_c, 'jacobian')
    for nz in (None, noise):
        _, gc_r, gx_r, gw_r, gb_r = C.ref_vjp(P, xyz, cond, up, nz)
        x, c = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
        g = torch.autograd.grad((_composite(net, x, c, nz) * up).sum(), [c, x] + params)
        for name, a, b in zip(['cond', 'xyz'] + ['p%d' % i for i in range(len(params))], [gc_r, gx_r] + [t for Wb in zip(gw_r, gb_r)
                                                                                             for t in Wb], g):
            _close(a, b, ('vjp', nz is not None, name))

    # second order: d/d theta of (s sbar + grad_x s . gbar) through the first output
    sbar = torch.randn(2, 5, 1, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    gbar = torch.randn(2, 5, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    P1 = [(W, b) for W, b in P[:-1]] + [(P[-1][0][:1], P[-1][1][:1])]
    gc_r, gx_r, gw_r, gb_r = C.ref_sdfgrad_vjp(P1, xyz, cond, sbar, gbar)
    x, c = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
    s = _composite(net, x, c)[..., :1]
    gx = torch.autograd.grad(s.sum(), x, create_graph=True)[0]
    g = torch.autograd.grad((s * sbar).sum() + (gx * gbar).sum(), [c, x] + params)
    gw_last, gb_last = g[-2][:1], g[-1][:1]
    ours = [gc_r, gx_r] + [t for Wb in zip(gw_r, gb_r) for t in Wb]
    theirs = list(g[:-2]) + [gw_last, gb_last]
    for i, (a, b) in enumerate(zip(ours, theirs)):
        _close(a, b, ('double backward', i))


@pytest.mark.parametrize('cfg', C.CONFIGS, ids=C.config_id)
def test_matrix_stacks_cover_the_softplus_kink_and_saturation(cfg):
    P = C.params_of(C.make_stack(cfg), torch.float64)
    xyz, cond = C.make_inputs(cfg, 2, 200, 'cpu')
    zs = []
    C.stack_forward(P, xyz.double(), cond.double(), preacts=zs)
    z = torch.cat([t.reshape(-1) for t in zs[:-1]]) * C.BETA
    assert float(z.abs().max()) >= 100                   # where the exponential of the softplus underflows / saturates
    assert float((z.abs() < 1).double().mean()) >= 0.005   # and its kink
