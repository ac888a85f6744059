"""A float64 reference of the posed SDF (get_logits_posed), written from the decoders' parameters.

It is the reference's composition (src/NPHM/models/fitting.py:59-114), not posed_evaluator's: for a point p and expression s,

    cond_s  = the deformation network's condition row of [z_id | z_ex[s]]
    x*      = the root of x + F(x; cond_s) = p
    sdf     = the identity decoder at x* (the ensemble's eval-mode quirk rows: every member's output is 1)

The condition row per deformation mode (DeformationNetwork._condition):
    compress   [Wc [z_id | anchors(z_id)] + bc | z_ex]       expr_only  z_ex
    glob_only  [z_id[:lat_dim_glob_shape] | z_ex]            NPM pair   [z_id | z_ex]

The pieces come from the existing references: the identity ensemble and its anchors from tests/ensemble_f64_common.py, the
DeepSDF stacks (deformation backbone, NPM decoders) from tests/chain_shapes_common.py.  Everything runs in the dtype of the
parameters: float64 is the yardstick, float32 (TF32 off) the error a plain fp32 implementation makes.
tests/test_posed_f64_cpu.py ties it to the mirror's modules.
"""
import torch

import chain_shapes_common as C
import ensemble_f64_common as E

CVG = 1e-6                      # the search's convergence threshold on |x + F(x) - p| (reference search(): cvg_thresh)
POLISH_TOL = 1e-13
POLISH_STEPS = 8

# the deformation networks of the posed tests: name -> (mode, output-layer scale)
DEFORMATIONS = {'compress': ('compress', 1.0), 'compress-x80': ('compress', 80.0), 'expr_only': ('expr_only', 1.0),
                'glob_only': ('glob_only', 1.0)}


def make_deformation(name, device='cpu'):
    """conftest.make_deformation with the mode of ``name`` (same sizes and seed; the condition of expr_only is 200 wide, that of
    glob_only 264) and its output layer scaled: x 80 makes searches take up to 15 steps and some rows diverge (posed.npz)."""
    from conftest import mean_anchors
    from nphm_b200.models.deepSDF import DeformationNetwork
    mode, scale = DEFORMATIONS[name]
    torch.manual_seed(10)
    dfn = DeformationNetwork(mode=mode, lat_dim_expr=200, lat_dim_id=32, lat_dim_glob_shape=64, lat_dim_loc_shape=32, n_loc=39,
                             anchors=mean_anchors(), hidden_dim=512, nlayers=6, out_dim=3, input_dim=3)
    if scale != 1.0:
        with torch.no_grad():
            dfn.defDeepSDF.lin6.weight.mul_(scale)
            dfn.defDeepSDF.lin6.bias.mul_(scale)
    dfn.eval()
    return dfn.to(device)


class Params:
    """Detached copies in ``dtype`` of an identity decoder and the deformation decoder it is posed with: the ensemble and a
    ``DeformationNetwork``, or the NPM pair of ``DeepSDF`` decoders."""

    def __init__(self, dec, dfn, dtype):
        from nphm_b200.models.deepSDF import DeformationNetwork
        self.nphm = isinstance(dfn, DeformationNetwork)
        self.dtype = dtype
        if self.nphm:
            self.id = E.Params(dec, dtype)
            self.expr = C.params_of(dfn.defDeepSDF, dtype)
            self.mode = dfn.mode
            self.glob = dfn.lat_dim_glob_shape
            if self.mode == 'compress':
                lin = dfn.compressor[0]
                self.Wc = lin.weight.detach().to(dtype).clone()
                self.bc = lin.bias.detach().to(dtype).clone()
        else:
            self.id = C.params_of(dec, dtype)
            self.expr = C.params_of(dfn, dtype)
            self.mode = 'npm'


def condition(Q, z_id, z_ex):
    """The S condition rows (S x C) of the identity code z_id (D,) under the expression codes z_ex (S x E)."""
    S = z_ex.shape[0]
    if Q.mode == 'compress':
        c = Q.Wc @ torch.cat([z_id, E.anchors(Q.id, z_id).reshape(-1)]) + Q.bc
        return torch.cat([c[None].expand(S, -1), z_ex], dim=1)
    if Q.mode == 'expr_only':
        return z_ex.clone()
    if Q.mode == 'glob_only':
        return torch.cat([z_id[None, :Q.glob].expand(S, -1), z_ex], dim=1)
    return torch.cat([z_id[None].expand(S, -1), z_ex], dim=1)


def residual(Q, x, cond, p):
    """x + F(x; cond) - p: x, p S x n x 3, cond S x C."""
    return C.broyden_residual(Q.expr, x, cond, p)


def inverse_jacobian(Q, x, cond):
    """(I + dF/dx)^-1 at x (S x n x 3) -> S x n x 3 x 3."""
    return C.ref_inverse_jacobian(Q.expr, x, cond)[1]


def polish(Q, x, cond, p, steps=POLISH_STEPS, tol=POLISH_TOL):
    """Newton's method on x + F(x; cond) = p from x, row by row (x, p m x 3, cond m x C: one condition row per point), until
    every |residual| < tol or ``steps`` steps.  Returns (x*, |residual| at x*)."""
    x = x.to(Q.dtype)[:, None]
    p = p.to(Q.dtype)[:, None]
    cond = cond.to(Q.dtype)
    with torch.no_grad():
        r = residual(Q, x, cond, p)
    for _ in range(steps):
        if x.shape[0] == 0 or float(r.norm(dim=-1).max()) < tol:
            break
        jinv = inverse_jacobian(Q, x, cond)
        with torch.no_grad():
            x = x - torch.einsum('mnij,mnj->mni', jinv, r)
            r = residual(Q, x, cond, p)
    return x[:, 0], r[:, 0].norm(dim=-1)


def quirk_mask(n, nbatch_points):
    """The rows of an n-point posed call that carry the ensemble's eval-mode quirk: the last row of every ``nbatch_points``
    chunk (one reference decoder call each) and the last row."""
    return E.query_quirk_rows(n, nbatch_points)


def identity_sdf(Q, x, z_id, quirk=None):
    """The identity decoder at x (n x 3) -> (n,).  quirk: the ensemble's eval-mode rows (boolean n), None in training mode."""
    if Q.nphm:
        q = torch.zeros(x.shape[0], dtype=torch.bool) if quirk is None else quirk
        return E.sdf(Q.id, x, z_id, quirk=q)
    return C.stack_forward(Q.id, x[None], z_id[None])[0, :, 0]


def identity_sdf_grad(Q, x, z_id, quirk=None):
    """(sdf (n,), d sdf / d x (n x 3)) of :func:`identity_sdf`."""
    xx = x.clone().requires_grad_()
    s = identity_sdf(Q, xx, z_id, quirk)
    g, = torch.autograd.grad(s.sum(), [xx])
    return s.detach(), g
