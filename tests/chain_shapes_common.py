"""Shape matrix of the DeepSDF layer-chain tests and a float64 reference of the stack they check.

The reference is a plain per-layer loop over ``(W, b)`` pairs, written here and not taken from
``DeepSDF._forward_composite``, so it is independent of the module whose native kernels it checks;
tests/test_chain_shapes_cpu.py ties it to the composite forward, which the reference goldens pin.  Every quantity
an entry point of the layer chain returns (values, Jacobians, adjoints, weight gradients, the double backward
through ``grad_x s``, the fitting surface term) is derived from it with torch autograd, in whatever dtype the
parameters have: float64 is the yardstick, float32 the error a plain fp32 implementation makes.
"""
import math

import torch
import torch.nn.functional as F

SQRT2 = math.sqrt(2.0)
BETA = 100.0

# (lat_dim, hidden, n_layers, out_dim).  The skip connection sits in front of layer n_layers // 2; the layer before it
# has hidden - lat_dim - 3 output columns and gets [xyz | noise] (3 + nd columns) appended, so it packs hidden - lat_dim
# (+ nd) columns.  The chain's output tiles are 16-column units, at most 128 columns per tile; the FFMA kernel takes
# hidden <= 880 from Python (impl='simt') and hidden <= 905 in C (its shared memory, 2 * (hidden + 3) * 128 bytes).
CONFIGS = [
    (4, 8, 2, 1),           # narrowest legal width (hidden = lat + 4: 1 column before the skip), skip at layer 1
    (13, 30, 3, 2),         # skip at layer 1, 14 + 3 = 17 packed columns; 2 outputs
    (20, 36, 7, 4),         # 7 hidden layers, 13 + 3 = 16; 4 outputs
    (24, 39, 9, 8),         # 9 hidden layers, 12 + 3 = 15; 8 outputs (the upstream gradient's cp.async staging path)
    (14, 18, 4, 3),         # narrowest width with 3 outputs; noise as wide as the condition (nd = 14)
    (2, 129, 10, 3),        # 10 hidden layers (the deepest accepted), hidden 129: two column tiles; 124 + 3 = 127
    (1, 129, 5, 1),         # 125 + 3 = 128
    (128, 257, 6, 3),       # hidden 257: three column tiles; 126 + 3 = 129
    (40, 880, 4, 3),        # widest stack impl='simt' sends to the FFMA kernel
    (40, 881, 4, 1),        # narrowest one it sends to the layer chain
    (64, 905, 4, 3),        # widest stack the FFMA kernel holds (Broyden search, NPHM_IMPL_AUTO)
    (64, 906, 4, 3),        # narrowest one the search runs on the layer chain
    (232, 512, 6, 3),       # forward deformation backbone, 235 -> 512 x 6 -> 3 (nphm_def.yaml)
    (512, 1024, 8, 1),      # NPM identity decoder, 515 -> 1024 x 8 -> 1 (npm.yaml)
    (712, 1024, 8, 3),      # NPM expression decoder, 715 -> 1024 x 8 -> 3
]
PRODUCTION = [(232, 512, 6, 3), (512, 1024, 8, 1), (712, 1024, 8, 3)]

# (queries, points per query): 1 row; 127 / 128 / 129 / 257 rows around the 128-row tile; 9 queries of 37 points (several
# queries per tile, a ragged last tile); one query spanning four tiles
ROWS = [(1, 1), (1, 127), (1, 128), (1, 129), (1, 257), (9, 37), (2, 200)]
# rows of the chunked forward (65 536 rows per chunk): one query one row longer than a chunk, two queries of one chunk each
CHUNK_ROWS = [(1, 65537), (2, 65536)]
# production row counts: a stage-2 decoder call (32 x 1000 + 32 x 100 points, nphm_def.yaml) and a stage-1 call
# (32 x 1693 points, npm.yaml)
STAGE2_ROWS = (32, 1100)
STAGE1_ROWS = (32, 1693)


def config_id(cfg):
    return '%d-%dx%d-%d' % cfg


def noise_dims(cfg):
    """Noise widths the training forward is run with: 0, 1, 13, 14 (3 + nd = 16, 17) and the whole condition."""
    return sorted({nd for nd in (0, 1, 13, 14, cfg[0]) if nd <= cfg[0]})


def make_stack(cfg, device='cpu', seed=0):
    """A ``DeepSDF`` of this shape with the module's own initialisation (geometric for one output), then layers rescaled
    so that the pre-activations reach both the softplus kink (|100 z| < 1) and its saturated end (|100 z| ~ 200)."""
    from nphm_b200.models.deepSDF import DeepSDF
    lat, hidden, nl, out = cfg
    torch.manual_seed(1000 + 7 * seed + hidden + 13 * nl + 31 * out)
    net = DeepSDF(lat_dim=lat, hidden_dim=hidden, nlayers=nl, geometric_init=out == 1, out_dim=out)
    skip = nl // 2
    with torch.no_grad():
        for l in range(nl + 1):
            lin = getattr(net, 'lin%d' % l)
            if l == 0 or l == skip:
                lin.weight.mul_(3.0)
            elif l < nl:
                lin.weight.mul_(2.0)
                lin.bias.mul_(4.0)
            elif out != 1:
                lin.weight.mul_(0.5)
    return net.to(device)


def params_of(net, dtype):
    """[(W, b)] of the module's layers, detached copies in ``dtype``."""
    return [(getattr(net, 'lin%d' % l).weight.detach().to(dtype).clone(), getattr(net, 'lin%d' % l).bias.detach().to(dtype).clone())
            for l in range(net.num_layers - 1)]


def make_inputs(cfg, B, N, device, seed=0):
    g = torch.Generator().manual_seed(50 + seed + 17 * B + N)
    xyz = (torch.rand(B, N, 3, generator=g) - 0.5) * 1.6
    cond = torch.randn(B, cfg[0], generator=g) * 0.3
    return xyz.to(device), cond.to(device)


# ------------------------------------------------------------------------------------------------ the reference
def stack_forward(P, xyz, cond, noise=None, preacts=None):
    """xyz B x N x 3, cond B x D (the same for every point of a query), noise B x N x nd added to the leading condition
    columns, or None -> B x N x out.  The input is concatenated back (and the sum scaled by 1/sqrt(2)) in front of layer
    n_layers // 2; Softplus(beta=100) after every layer but the last.  ``preacts``: a list that receives z_l."""
    B, N, _ = xyz.shape
    c = cond[:, None, :].expand(B, N, cond.shape[-1])
    if noise is not None:
        c = c + F.pad(noise, (0, cond.shape[-1] - noise.shape[-1]))
    inp = torch.cat([xyz, c], dim=-1)
    skip = (len(P) - 1) // 2
    h = inp
    for l, (W, b) in enumerate(P):
        if l == skip:
            h = torch.cat([h, inp], dim=-1) / SQRT2
        z = h @ W.T + b
        if preacts is not None:
            preacts.append(z)
        h = F.softplus(z, beta=BETA) if l + 1 < len(P) else z
    return h


def _leaves(P, *ts):
    Pl = [(W.clone().requires_grad_(), b.clone().requires_grad_()) for W, b in P]
    return Pl, [t.clone().requires_grad_() for t in ts]


def _flat(P):
    return [t for Wb in P for t in Wb]


def ref_jacobian(P, xyz, cond):
    """(out, d out / d xyz  B x N x out x 3)."""
    x = xyz.clone().requires_grad_()
    out = stack_forward(P, x, cond)
    rows = [torch.autograd.grad(out[..., i].sum(), x, retain_graph=True)[0] for i in range(out.shape[-1])]
    return out.detach(), torch.stack(rows, dim=-2)


def ref_inverse_jacobian(P, xyz, cond):
    out, J = ref_jacobian(P, xyz, cond)
    return out, torch.linalg.inv(torch.eye(3, dtype=J.dtype, device=J.device) + J)


def ref_vjp(P, xyz, cond, up, noise=None):
    """(out, d/d cond, d/d xyz, [d/d W_l], [d/d b_l]) of (out * up).sum()."""
    Pl, (x, c) = _leaves(P, xyz, cond)
    out = stack_forward(Pl, x, c, noise)
    g = torch.autograd.grad((out * up).sum(), [c, x] + _flat(Pl))
    return out.detach(), g[0], g[1], list(g[2::2]), list(g[3::2])


def ref_sdfgrad(P, xyz, cond):
    """(s, grad_x s) of a one-output stack."""
    x = xyz.clone().requires_grad_()
    s = stack_forward(P, x, cond)
    return s.detach(), torch.autograd.grad(s.sum(), x)[0]


def ref_sdfgrad_vjp(P, xyz, cond, sbar, gbar):
    """(d/d cond, d/d xyz, [d/d W_l], [d/d b_l]) of (s * sbar + grad_x s . gbar).sum(): the double backward."""
    Pl, (x, c) = _leaves(P, xyz, cond)
    s = stack_forward(Pl, x, c)
    gx = torch.autograd.grad(s.sum(), x, create_graph=True)[0]
    g = torch.autograd.grad((s * sbar).sum() + (gx * gbar).sum(), [c, x] + _flat(Pl))
    return g[0], g[1], list(g[2::2]), list(g[3::2])


def ref_fit_surface(P, xyz, cond, mask, clamp):
    """(loss, kept count, d loss / d cond, d loss / d xyz): loss = mean |s| over the points with mask and |s| < clamp."""
    x, c = xyz.clone().requires_grad_(), cond.clone().requires_grad_()
    s = stack_forward(P, x, c)[..., 0]
    kept = mask & (s.detach().abs() < clamp)
    loss = s.abs()[kept].mean()
    gc, gx = torch.autograd.grad(loss, [c, x])
    return loss.detach(), int(kept.sum()), gc, gx


def ref_adjoints(P, xyz, cond, up, noise=None):
    """Pre-activation adjoints d_l = d (out * up).sum() / d z_l of the hidden layers (B x N x N_l each)."""
    zs = []
    out = stack_forward(P, xyz.clone().requires_grad_(), cond, noise, preacts=zs)
    return torch.autograd.grad((out * up).sum(), zs[:-1])


def ref_sdfgrad_adjoints(P, xyz, cond, sbar, gbar):
    """The two adjoints of the SDF-gradient backward per hidden layer: a_l = d s / d z_l (unit upstream) and
    zb_l = d (s * sbar + grad_x s . gbar).sum() / d z_l."""
    x = xyz.clone().requires_grad_()
    zs = []
    s = stack_forward(P, x, cond, preacts=zs)
    a = torch.autograd.grad(s.sum(), zs[:-1], retain_graph=True)
    gx = torch.autograd.grad(s.sum(), x, create_graph=True)[0]
    zb = torch.autograd.grad((s * sbar).sum() + (gx * gbar).sum(), zs[:-1])
    return a, zb


def broyden_residual(P, x, cond, obs):
    """x + F(x; cond) - obs."""
    return x + stack_forward(P, x, cond) - obs
