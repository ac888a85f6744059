"""Configuration matrix of the identity-ensemble tests and a float64 reference of ``FastEnsembleDeepSDFMirrored``.

The reference is a plain loop over the members, each through the ``(W, b)`` of its weight set, written here and not taken from
``nphm_b200.models._composite``; tests/test_ensemble_f64_cpu.py ties it to the composite forward, which the reference goldens
pin.  It runs in whatever dtype the parameters have: float64 is the yardstick, float32 (TF32 off) the error a plain fp32
implementation makes.  Every derived quantity (anchors, member outputs s_k, the blended SDF, the vector-Jacobian products with
respect to the latent code and the points, the fitting loss and the regularisers, the stage-1 double backward) comes from
torch autograd through it.
"""
import math

import torch
import torch.nn.functional as F

SQRT2 = math.sqrt(2.0)
BETA = 100.0
BLEND_VAR = 0.1 ** 2
BACKGROUND = -0.2
UNOBSERVED = (30, 31, 39)          # members whose codes the fitting regulariser reg_unobserved pulls to zero

# name -> (n_loc, n_symm, lat_dim_glob, lat_dim_loc, hidden, n_layers, weights).  weights: 'init' (the module's own), 'x2'
# (every member layer's weight doubled, as conftest.make_ensemble(scale=2)) or 'stack' (rescaled like
# chain_shapes_common.make_stack, so that the pre-activations reach both the softplus kink and its saturated end).
CONFIGS = {
    'prod': (39, 16, 64, 32, 200, 4, 'init'),          # nphm.yaml: the dense tensor-core kernel
    'prod-x2': (39, 16, 64, 32, 200, 4, 'x2'),
    'tc-64m': (63, 16, 64, 32, 200, 4, 'init'),        # 64 members: the most the tensor-core kernel's member masks hold
    'tc-65m': (64, 16, 64, 32, 200, 4, 'init'),        # 65 members at the tensor-core widths: the FFMA kernels
    # other member structures the tensor-core kernel takes (hidden 200, 4 layers, G + L = 96, at most 64 members)
    'tc-2m': (1, 0, 64, 32, 200, 4, 'init'),           # fewest members: one local member and the global one
    'tc-3m-pair': (2, 1, 64, 32, 200, 4, 'stack'),     # one mirrored pair and nothing else
    'tc-nosymm': (39, 0, 64, 32, 200, 4, 'init'),      # the production anchors without a mirror: 40 weight sets
    'tc-allpairs': (38, 19, 64, 32, 200, 4, 'init'),   # every local member mirrored or mirroring
    'tc-33m': (32, 8, 64, 32, 200, 4, 'x2'),           # the global member at mask bit 32, just past a 32-bit word
    'tc-64m-nosymm': (63, 0, 64, 32, 200, 4, 'init'),  # 64 members and 64 weight sets: mask bit 63, the most sets
    'tc-split-32-64': (39, 16, 32, 64, 200, 4, 'init'),    # another latent split: wide local codes
    'tc-split-80-16': (39, 16, 80, 16, 200, 4, 'stack'),   # another latent split: narrow local codes
    'api': (10, 3, 32, 16, 160, 4, 'init'),
    'fit': (39, 16, 16, 8, 128, 4, 'stack'),
    'symm0': (5, 0, 16, 8, 64, 4, 'stack'),
    'loc1': (1, 0, 16, 8, 64, 4, 'init'),
    'allpairs': (6, 3, 16, 8, 64, 4, 'stack'),         # 2 n_symm = n_loc: every local member is mirrored or mirrors
    'h77': (7, 2, 16, 8, 77, 4, 'stack'),              # hidden width not a multiple of 8
    'depth2': (7, 2, 16, 8, 64, 2, 'stack'),
    'depth3': (7, 2, 16, 8, 64, 3, 'stack'),
    'depth6': (7, 2, 16, 8, 64, 6, 'stack'),
    'depth10': (7, 2, 16, 8, 64, 10, 'stack'),
    'ffma-widest': (10, 3, 32, 16, 204, 4, 'init'),    # 139 + 4 H - C = 907 shared-memory rows: the widest FFMA fitting step
    'ffma-over': (10, 3, 32, 16, 205, 4, 'init'),      # 911 rows: rejected, fitting takes the autograd path
}
# the configurations the fitting kernels run on (4 hidden layers, within the FFMA step's shared memory)
FIT_CONFIGS = [k for k, c in CONFIGS.items() if c[5] == 4 and k != 'ffma-over']

# rows around the 128-row tile; several queries per call
ROWS = [(1, 1), (1, 63), (1, 64), (1, 65), (1, 127), (1, 128), (1, 129), (1, 257), (1, 1000), (3, 129), (5, 37)]


def quirk_periods(n):
    """Quirk periods of an n-row call: every row, around the tile, the whole call."""
    return sorted({p for p in (1, 127, 128, 129, n) if p <= n})


def n_members(cfg):
    return cfg[0] + 1


def mean_anchors(n_loc):
    """The shipped 39 mean anchors, cut to n_loc or extended by points of the head's box (fixed seed)."""
    from conftest import load_golden
    a = torch.from_numpy(load_golden('assets.npz')['anchors_39']).double()
    if n_loc <= 39:
        return a[:n_loc].clone()
    g = torch.Generator().manual_seed(39 + n_loc)
    extra = (torch.rand(n_loc - 39, 3, generator=g, dtype=torch.float64) - 0.5) * torch.tensor([1.0, 1.1, 1.2], dtype=torch.float64)
    return torch.cat([a, extra])


def make_decoder(name, device='cpu'):
    """The ``FastEnsembleDeepSDFMirrored`` of a configuration (fp32, training mode)."""
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    n_loc, n_symm, G, L, H, nl, weights = CONFIGS[name]
    torch.manual_seed(1000 + 7 * n_loc + H + 13 * nl)
    anchors = mean_anchors(n_loc).float().reshape(1, 1, n_loc, 3)
    dec = FastEnsembleDeepSDFMirrored(G, L, n_loc, n_symm, anchors, H, nl, pos_mlp_dim=256 if H == 200 else 64)
    e = dec.ensembled_deep_sdf
    skip = nl // 2
    with torch.no_grad():
        for l in range(nl + 1):
            lin = getattr(e, 'lin%d' % l)
            if weights == 'x2':
                lin.weight.mul_(2.0)
            elif weights == 'stack':
                if l == 0 or l == skip:
                    lin.weight.mul_(3.0)
                elif l < nl:
                    lin.weight.mul_(2.0)
                    lin.bias.mul_(4.0)
    dec.train()
    if device != 'cpu':
        dec = dec.to(device)
        dec.anchors = dec.anchors.to(device)
    return dec


def latent(name, seed=0, device='cpu'):
    """A code of the configuration: the fitting prior's distribution for 'prod', else 0.1 N(0, 1)."""
    cfg = CONFIGS[name]
    D = cfg[2] + n_members(cfg) * cfg[3]
    if D == 1344:
        from conftest import sample_latent
        return sample_latent(seed).reshape(-1).to(device)
    g = torch.Generator().manual_seed(77 + seed + D)
    return (0.1 * torch.randn(D, generator=g)).to(device)


# ------------------------------------------------------------------------------------------------ parameters
class Params:
    """Detached copies of a decoder's parameters in one dtype: member layers [(W S x N x K, b S x N)], mlp_pos
    [(W, b)] x 3, mean anchors n_loc x 3, and the shape constants."""

    def __init__(self, dec, dtype):
        e = dec.ensembled_deep_sdf
        self.n_loc, self.n_symm = dec.num_kps, dec.num_symm_pairs
        self.M = self.n_loc + 1
        self.G, self.L = dec.lat_dim_glob, dec.lat_dim_loc
        self.D = dec.lat_dim
        self.n_layers = e.num_layers - 2
        self.layers = [(getattr(e, 'lin%d' % l).weight.detach().to(dtype).clone(),
                        getattr(e, 'lin%d' % l).bias.detach().to(dtype).clone()) for l in range(e.num_layers - 1)]
        self.pos = [(dec.mlp_pos[i].weight.detach().to(dtype).clone(), dec.mlp_pos[i].bias.detach().to(dtype).clone())
                    for i in (0, 2, 4)]
        self.mean = dec.anchors.detach().reshape(self.n_loc, 3).to(dtype).clone()
        self.dtype = dtype

    def weight_set(self, m):
        """member m -> its weight set: the members 2i, 2i+1 of symmetric pair i share set i."""
        return m // 2 if m < 2 * self.n_symm else m - self.n_symm

    def mirrored(self, m):
        return m < 2 * self.n_symm and m % 2 == 1


# ------------------------------------------------------------------------------------------------ the reference
def anchors(P, z):
    """mlp_pos(z_glob) + mean anchors -> n_loc x 3 (ReLU between the three layers)."""
    h = z[:P.G]
    for i, (W, b) in enumerate(P.pos):
        h = W @ h + b
        if i < 2:
            h = torch.relu(h)
    return h.reshape(P.n_loc, 3) + P.mean


def member_mlp(P, m, inp, preacts=None):
    """One member's stack on its inputs [local xyz | z_glob | z_m] (rows x (3 + C)): the input concatenated back (the sum scaled
    by 1/sqrt(2)) in front of layer n_layers // 2, Softplus(beta=100, threshold=20) after every layer but the last."""
    s = P.weight_set(m)
    skip = P.n_layers // 2
    h = inp
    for l, (W, b) in enumerate(P.layers):
        if l == skip:
            h = torch.cat([h, inp], dim=-1) / SQRT2
        zl = h @ W[s].T + b[s]
        if preacts is not None:
            preacts.append(zl)
        h = F.softplus(zl, beta=BETA, threshold=20.0) if l + 1 < len(P.layers) else zl
    return h[:, 0]


def member_inputs(P, m, xyz, z, anc):
    """[local xyz | z_glob | z_m] of member m: anchor-centred for the local members, the world frame for the last one, the x
    column negated for the odd members of the symmetric pairs."""
    local = xyz - anc[m] if m < P.n_loc else xyz
    if P.mirrored(m):
        local = local * local.new_tensor([-1.0, 1.0, 1.0])
    cond = torch.cat([z[:P.G], z[P.G + m * P.L:P.G + (m + 1) * P.L]])
    return torch.cat([local, cond[None, :].expand(xyz.shape[0], -1)], dim=-1)


def members(P, xyz, z, anc=None, preacts=None):
    """s_k of every member at xyz (n x 3) -> n x M."""
    anc = anchors(P, z) if anc is None else anc
    cols = []
    for m in range(P.M):
        pa = [] if preacts is not None else None
        cols.append(member_mlp(P, m, member_inputs(P, m, xyz, z, anc), pa))
        if preacts is not None:
            preacts.append(pa)
    return torch.stack(cols, dim=1)


def blend_weights(P, xyz, anc):
    """Normalised blend weights n x M: exp(-(|x - A_k| + 10e-6)^2 / 0.01) for the local members, the constant
    exp(-0.2 / 0.01) for the background member, divided by their sum + 1e-6."""
    gap = (anc[None, :, :] - xyz[:, None, :]).norm(dim=-1) + 10e-6
    logits = torch.cat([-(gap * gap), gap.new_full((xyz.shape[0], 1), BACKGROUND)], dim=1)
    w = torch.exp(logits / BLEND_VAR)
    return w / (w.sum(dim=1, keepdim=True) + 1e-6)


def quirk_rows(n, period):
    """Rows the eval-mode forward overwrites: i % period == period - 1 (period 0: none)."""
    r = torch.zeros(n, dtype=torch.bool)
    if period:
        r[period - 1::period] = True
    return r


def query_quirk_rows(count, period, first=0, total=None):
    """Rows the eval-mode query overwrites, for rows [first, first + count) of a query of ``total`` points (a grid: its grid
    index): g % period == period - 1, and the query's last point g == total - 1, the end of the reference's last, partial
    decoder call."""
    total = first + count if total is None else total
    g = torch.arange(first, first + count)
    return (g % period == period - 1) | (g == total - 1) if period else torch.zeros(count, dtype=torch.bool)


def sdf(P, xyz, z, period=0, with_members=False, quirk=None):
    """The blended SDF at xyz (n x 3) for the code z (D,): every member's output is 1 at the quirk rows (those of
    :func:`quirk_rows` with ``period``, or the boolean mask ``quirk``)."""
    anc = anchors(P, z)
    s = members(P, xyz, z, anc)
    q = (quirk_rows(xyz.shape[0], period) if quirk is None else quirk).to(xyz.device)
    if q.any():
        s = torch.where(q[:, None], torch.ones_like(s), s)
    out = (blend_weights(P, xyz, anc) * s).sum(dim=1)
    return (out, s, anc) if with_members else out


def vjp(P, xyz, z, up, period=0):
    """(sdf, d (sdf . up) / d z, d (sdf . up) / d xyz)."""
    x, zz = xyz.clone().requires_grad_(), z.clone().requires_grad_()
    s = sdf(P, x, zz, period)
    gz, gx = torch.autograd.grad((s * up).sum(), [zz, x])
    return s.detach(), gz, gx


def surface_loss(s, mask, clamp):
    """Clamped mean |s| over the rows with mask and |s| < clamp: (loss, kept) - NaN when nothing is kept, like torch."""
    a = s.abs()
    kept = mask & (a.detach() < clamp)
    return a[kept].mean(), kept


def fit_surface(P, xyz, z, mask, clamp, period=0):
    """(loss, kept count, d loss / d z, d loss / d xyz).  Nothing kept: NaN loss and zero gradients."""
    x, zz = xyz.clone().requires_grad_(), z.clone().requires_grad_()
    loss, kept = surface_loss(sdf(P, x, zz, period), mask, clamp)
    if not bool(kept.any()):
        return loss.detach(), 0, torch.zeros_like(z), torch.zeros_like(xyz)
    gz, gx = torch.autograd.grad(loss, [zz, x])
    return loss.detach(), int(kept.sum()), gz, gx


def regularisers(P, z):
    """[reg_global, reg_loc, reg_unobserved, symm_dist] of the fitters: |z_glob|^2, |z_loc|^2, sum of |z_k|^2 over the
    unobserved members that exist, and the mean over the symmetric pairs of |z_2i - z_2i+1| (0 without pairs)."""
    loc = z[P.G:].reshape(P.M, P.L)
    ru = z.sum() * 0
    for k in UNOBSERVED:
        if k < P.M:
            ru = ru + (loc[k] * loc[k]).sum()
    symm = (loc[0:2 * P.n_symm:2] - loc[1:2 * P.n_symm:2]).norm(dim=-1).mean() if P.n_symm else z.sum() * 0
    return [(z[:P.G] * z[:P.G]).sum(), (z[P.G:] * z[P.G:]).sum(), ru, symm]


def identity_step(P, xyz, z, lambdas, clamp, period=0):
    """The identity fitter's objective lambda_s surface + lambda . regularisers: (terms [surface, reg_global, reg_loc,
    reg_unobserved, symm_dist, kept], d objective / d z)."""
    zz = z.clone().requires_grad_()
    loss, kept = surface_loss(sdf(P, xyz, zz, period), torch.ones(xyz.shape[0], dtype=torch.bool, device=xyz.device), clamp)
    regs = regularisers(P, zz)
    total = sum(l * r for l, r in zip(lambdas[1:], regs))
    if bool(kept.any()):
        total = total + lambdas[0] * loss
    g, = torch.autograd.grad(total, [zz])
    terms = [loss.detach()] + [r.detach() for r in regs] + [loss.new_tensor(float(kept.sum()))]
    return torch.stack(terms), g


def anchor_vjp(P, z, up):
    """d (anchors . up) / d z: the mlp_pos backward (ReLU masks)."""
    zz = z.clone().requires_grad_()
    g, = torch.autograd.grad((anchors(P, zz) * up).sum(), [zz])
    return g


# ------------------------------------------------------------------------------------------------ stage 1: member passes
def member_stack(P, m, xl, cond, layers=None):
    """Member m's stack on its own frame xl (rows x 3) and condition cond (C,), with ``layers`` in place of P.layers."""
    Q = P if layers is None else _with_layers(P, layers)
    return member_mlp(Q, m, torch.cat([xl, cond[None, :].expand(xl.shape[0], -1)], dim=-1))


def _with_layers(P, layers):
    q = Params.__new__(Params)
    q.__dict__.update(P.__dict__)
    q.layers = layers
    return q


def sdfgrad(P, xl, cond):
    """(s members x B x N, grad_local s members x B x N x 3) of the member passes: xl members x B x N x 3 (each member's
    frame), cond members x B x C."""
    x = xl.clone().requires_grad_()
    s = torch.stack([torch.stack([member_stack(P, m, x[m, b], cond[m, b]) for b in range(x.shape[1])])
                     for m in range(P.M)])
    g, = torch.autograd.grad(s.sum(), [x])
    return s.detach(), g


def sdfgrad_vjp(P, xl, cond, sbar, gbar):
    """The double backward of :func:`sdfgrad`: d (s . sbar + grad s . gbar) / d (W_l, b_l (per weight set), cond, xl)."""
    layers = [(W.clone().requires_grad_(), b.clone().requires_grad_()) for W, b in P.layers]
    x, c = xl.clone().requires_grad_(), cond.clone().requires_grad_()
    s = torch.stack([torch.stack([member_stack(P, m, x[m, b], c[m, b], layers) for b in range(x.shape[1])])
                     for m in range(P.M)])
    gx, = torch.autograd.grad(s.sum(), [x], create_graph=True)
    flat = [t for Wb in layers for t in Wb]
    g = torch.autograd.grad((s * sbar).sum() + (gx * gbar).sum(), flat + [c, x])
    return list(g[0:2 * len(layers):2]), list(g[1:2 * len(layers):2]), g[-2], g[-1]


# ------------------------------------------------------------------------------------------------ points
def point_sets(P, z, seed=0, near_per_member=3, n_box=200, n_far=40):
    """(near, the local member each near row was drawn at, box, far), float64 on the parameters' device.

    near: near_per_member points within 0.02 of every anchor; box: uniform in the head's box; far: more than 1.1 from every
    anchor, where only the background weight survives in fp32 (the background member's rows)."""
    g = torch.Generator().manual_seed(500 + seed)
    anc = anchors(P, z).detach().cpu()
    dt = torch.float64
    rows, owner = [], []
    for m in range(P.n_loc):
        d = torch.randn(near_per_member, 3, generator=g, dtype=dt)
        d = d / d.norm(dim=1, keepdim=True) * 0.02 * torch.rand(near_per_member, 1, generator=g, dtype=dt)
        rows.append(anc[m] + d)
        owner += [m] * near_per_member
    near = torch.cat(rows)
    box = (torch.rand(n_box, 3, generator=g, dtype=dt) - 0.5) * torch.tensor([1.1, 1.25, 1.35], dtype=dt) \
        + torch.tensor([0.0, 0.1, -0.3], dtype=dt)
    far = []
    while len(far) < n_far:
        p = (torch.rand(3, generator=g, dtype=dt) - 0.5) * 8.0
        if float((anc - p).norm(dim=1).min()) > 1.1:
            far.append(p)
    dev = P.mean.device
    return near.to(dev), torch.tensor(owner), box.to(dev), torch.stack(far).to(dev)


def mixed_points(P, z, n, seed=0):
    """n rows mixing the three point sets (near, box, far in turn), so that every 128-row tile holds each kind.  Returns
    (xyz n x 3 float64, kind n: 0 near / 1 box / 2 far)."""
    near, _, box, far = point_sets(P, z, seed, near_per_member=max(1, n // (3 * P.n_loc) + 1), n_box=n, n_far=max(1, n // 3 + 1))
    src = [near, box, far]
    idx = [0, 0, 0]
    out, kind = [], []
    for i in range(n):
        k = i % 3
        out.append(src[k][idx[k] % src[k].shape[0]])
        idx[k] += 1
        kind.append(k)
    return torch.stack(out), torch.tensor(kind)
