"""A float64 reference of one joint-fitting iteration at given correspondences, for both decoders of the fitters.

It is the reference's own formulation (src/NPHM/models/fitting.py:99-137), not the fitters' derivation: at the roots p of
x + F_ex(x; cond) = obs,

    xc = p - J^-1 (F_ex(p; cond) + p - stopgrad(F_ex(p; cond) + p)),    J = I + dF_ex/dx at p (held constant)

so that value(xc) = p and d xc / d theta = -J^-1 dF_ex / d theta; then the clamped surface term on xc, reg_expr over the
sampled expression rows and the identity regularisers, differentiated with torch autograd.  The chain the fitters write out by
hand (u = -J^-T g_x, the adjoint pass, the compressor and anchor route, index_add_ into the rows) never appears here.

The pieces come from the existing references: the identity ensemble, mlp_pos and the regularisers from
tests/ensemble_f64_common.py, the DeepSDF stacks (deformation backbone, NPM decoders) from tests/chain_shapes_common.py; the
'compress' condition [compressor([z_id | anchors]) | z_ex] is added here.  Everything runs in the dtype of the parameters:
float64 is the yardstick, float32 (TF32 off) the error a plain fp32 implementation of the same iteration makes.
tests/test_joint_f64_cpu.py ties it to the graph ``_inference_joint_autograd`` builds at the same roots.
"""
import torch

import chain_shapes_common as C
import ensemble_f64_common as E


class NphmParams:
    """The shipped configuration: the identity ensemble (``FastEnsembleDeepSDFMirrored``) and the 'compress'
    ``DeformationNetwork``, detached copies in ``dtype``."""
    nphm = True

    def __init__(self, dec, dfn, dtype):
        self.id = E.Params(dec, dtype)
        self.expr = C.params_of(dfn.defDeepSDF, dtype)
        lin = dfn.compressor[0] if isinstance(dfn.compressor, torch.nn.Sequential) else dfn.compressor
        self.Wc = lin.weight.detach().to(dtype).clone()
        self.bc = lin.bias.detach().to(dtype).clone()
        self.dtype = dtype


class NpmParams:
    """The NPM baseline: a one-output ``DeepSDF`` identity decoder and a three-output ``DeepSDF`` expression decoder
    conditioned on [z_id | z_ex]."""
    nphm = False

    def __init__(self, dec, expr, dtype):
        self.id = C.params_of(dec, dtype)
        self.expr = C.params_of(expr, dtype)
        self.dtype = dtype


def condition(Q, z_id, z_ex, obs_idx):
    """The per-row condition of the expression decoder (nb x C), with graph to z_id and z_ex."""
    nb = obs_idx.shape[0]
    if Q.nphm:
        anc = E.anchors(Q.id, z_id)
        c32 = Q.Wc @ torch.cat([z_id, anc.reshape(-1)]) + Q.bc
        return torch.cat([c32[None, :].expand(nb, -1), z_ex[obs_idx]], dim=1)
    return torch.cat([z_id[None, :].expand(nb, -1), z_ex[obs_idx]], dim=1)


def identity_sdf(Q, xc, z_id, period=0):
    """The identity decoder at xc (nb x n x 3) -> nb n values.  period: the eval-mode quirk period of the ensemble over the
    flattened points (one reference decoder call per row: n), 0 in training mode."""
    if Q.nphm:
        return E.sdf(Q.id, xc.reshape(-1, 3), z_id, period)
    return C.stack_forward(Q.id, xc, z_id[None, :].expand(xc.shape[0], -1))[..., 0].reshape(-1)


def sdf_at_roots(Q, p, z_id, period=0):
    """|s| at the roots themselves (value(xc) = p), for choosing the clamp."""
    with torch.no_grad():
        return identity_sdf(Q, p.to(Q.dtype), z_id.to(Q.dtype), period)


def joint_gradients(Q, p, valid, z_id, z_ex, obs_idx, lambdas, clamp, period=0):
    """d loss / d z_id (D,) and d loss / d z_ex (n_obs x E) of one joint iteration at the roots p (nb x n x 3) with the
    valid mask (nb x n), the codes z_id (D,), z_ex (n_obs x E), the sampled rows obs_idx (nb,), the lambdas dict and the clamp.
    Returns (g_id, g_ex, kept count)."""
    dt = Q.dtype
    p = p.to(dt)
    zid = z_id.to(dt).clone().requires_grad_()
    zex = z_ex.to(dt).clone().requires_grad_()
    cond = condition(Q, zid, zex, obs_idx)
    # implicit differentiation of the root (reference :99-106): J^-1 at p is a constant of the graph
    _, j_inv = C.ref_inverse_jacobian(Q.expr, p, cond.detach())
    posed = C.stack_forward(Q.expr, p, cond) + p
    xc = p + torch.einsum('bnij,bnj->bni', -j_inv.detach(), posed - posed.detach())
    # surface term (:111-136): clamped mean |s| over the valid points
    a = identity_sdf(Q, xc, zid, period).abs()
    kept = valid.reshape(-1) & (a.detach() < clamp)
    terms = {'surface': a[kept].mean(), 'reg_expr': (zex[obs_idx] * zex[obs_idx]).sum(-1).mean()}
    if Q.nphm:
        terms.update(zip(('reg_global', 'reg_loc', 'reg_unobserved', 'symm_dist'), E.regularisers(Q.id, zid)))
    else:
        terms['reg_global'] = (zid * zid).sum()            # a DeepSDF has no local codes: the other three are 0
    loss = sum(float(lam) * terms[k] for k, lam in lambdas.items() if k in terms)
    g_id, g_ex = torch.autograd.grad(loss, [zid, zex])
    return g_id, g_ex, int(kept.sum())
