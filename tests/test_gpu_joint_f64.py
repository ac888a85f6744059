"""The four joint fitters of nphm_b200/models/fitting.py (JointFitter, BatchedJointFitter, NpmJointFitter,
BatchedNpmJointFitter) against the float64 reference of one iteration at the same correspondences (tests/joint_f64_common.py).

The reference goldens of test_gpu_fit.py / test_gpu_fit_npm.py come from another Broyden run, so they can only pin the joint
gradients to a few percent.  Here the roots the fitter itself found are handed to the reference: the fitter's engine is
wrapped on the instance to capture p and the valid mask, ``step`` runs twice with ``apply_update=False`` and must find
bit-identical roots, and the clamp sits in a gap of |s(p)| so that no point is kept on one side and dropped on the other.
What is left is the chain's own arithmetic: the surface term, u = -J^-T g_x, the deformation adjoint (nphm_mlp_backward_inputs),
the compressor and anchor route, the regularisers and the rows of the expression codes.

The criterion is that of tests/f64_check.py, err_native <= K * err_fp32 + FLOOR * max|ref64|, with the same iteration in fp32
PyTorch (TF32 off) as the yardstick, applied to each part on its own: the z_glob block and every member's block of d/d z_id,
every sampled z_ex row, every subject of the batched fitters, and the condition gradient of the adjoint pass by itself (per
query, against float64 at the fitter's own u).  Unsampled rows must be exactly zero.  The upstream u of the adjoint pass is
d surface / d xc over the kept points, ~1e-4 at 5 x 1000 points: `-s` prints max|u| per case and the worst ratio per fitter and
part.
"""
import pytest
import torch

import chain_shapes_common as C
import joint_f64_common as J
from conftest import load_golden, make_deformation, make_ensemble
from f64_check import Check

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64

# Measured on an H100 80GB HBM3 (700 W power limit) over every case below: worst err_native / err_fp32 32 (g_cond) for the
# NPHM fitters, where no part needs a floor beyond K * err_fp32; 200 for the NPM fitters (the 1024-wide stacks), where a z_ex
# row of the surface-only case needs 3.9e-5 of its own max|ref|.  Before the adjoint pass scaled its upstream, the NPHM fitters
# measured ratios of 1e5 and 1.5e-2 (z_ex) to 9e-2 (g_cond) of max|ref|.
K = 64.0
FLOOR = 2e-5                    # NPHM: identity ensemble + deformation backbone
FLOOR_NPM = 1e-4                # NPM baseline: DeepSDF 515 -> 1024 x 8 -> 1 and 715 -> 1024 x 8 -> 3
LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
SURFACE_ONLY = {'surface': 2.0}
N_POINT = 1000                                  # points per sampled observation (fitting.NUM_POINTS_PER_OBSERVATION)
OBS_IDX = [2, 0, 2, 3, 0]                       # 4 observations: rows 0 and 2 sampled twice, row 1 never


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------ decoders and data
def _nphm():
    dec = make_ensemble(0, device=DEV)
    dfn = make_deformation(DEV)
    return dec, dfn, J.NphmParams(dec, dfn, F64), J.NphmParams(dec, dfn, F32)


def _npm():
    import npm_fit_common as NC
    from nphm_b200.models.deepSDF import DeepSDF
    dec, expr = NC.make_decoders(DeepSDF, DEV)
    return dec, expr, J.NpmParams(dec, expr, F64), J.NpmParams(dec, expr, F32)


def _scans(golden, seed):
    """4 observations of 1000 points around the golden scans (3 x 200 points: resampled with a 2 mm jitter; the fourth a
    shifted copy of the first)."""
    obs = torch.from_numpy(load_golden(golden)['obs'])
    g = torch.Generator().manual_seed(seed)
    out = []
    for k in (0, 1, 2, 0):
        pick = torch.randint(0, obs.shape[1], (N_POINT,), generator=g)
        out.append(obs[k][pick] + 0.002 * torch.randn(N_POINT, 3, generator=g) + (0.003 if len(out) == 3 else 0.0))
    return out


def _codes(golden, j, seed):
    """(z_id, z_ex 4 x E) near the reference's own codes at iteration j of the golden run."""
    g = load_golden(golden)
    key = 'z_id_before' if golden == 'fit_joint.npz' else 'joint_z_id_before'
    z_id = torch.from_numpy(g[key][j])
    z_ex = torch.from_numpy(g[key.replace('id', 'ex')][j])
    gen = torch.Generator().manual_seed(seed)
    z_id = z_id + 0.01 * z_id.abs().max() * torch.randn(z_id.shape, generator=gen)
    z_ex = torch.cat([z_ex, z_ex[:1]]) + 0.02 * torch.randn(4, z_ex.shape[1], generator=gen)
    return z_id.to(DEV), z_ex.to(DEV)


def _sample(scans, idx, n):
    """Rows idx of the scans with their first n points: 5 x n x 3 on the device."""
    return torch.stack([scans[i][:n] for i in idx]).to(DEV)


# ------------------------------------------------------------------------------------------------ capture
class _Capture:
    """Wraps the fitter's expression engine on the instance: the roots and valid mask of every Broyden search, and the
    arguments and condition gradient of every adjoint pass."""

    def __init__(self, eng):
        self.eng, self.roots, self.adjoint = eng, [], None
        search, backward = eng.broyden_search, eng.backward_inputs

        def broyden_search(*a, **k):
            out = search(*a, **k)
            self.roots.append((out[0].clone(), out[2].clone()))
            return out

        def backward_inputs(xyz, cond, grad_out, **k):
            out = backward(xyz, cond, grad_out, **k)
            self.adjoint = (xyz.clone(), cond.clone(), grad_out.clone(), out[0].clone())
            return out

        eng.broyden_search, eng.backward_inputs = broyden_search, backward_inputs

    def release(self):
        del self.eng.broyden_search, self.eng.backward_inputs


def _clamp_in_a_gap(a, keep):
    """A clamp in the widest gap between consecutive |s| (float64) of the points that may be kept, within the middle half of
    their range: fp32 rounding cannot move a point across it."""
    a = a[keep].sort().values
    lo, hi = a.numel() // 4, a.numel() * 3 // 4
    gaps = a[lo + 1:hi + 1] - a[lo:hi]
    i = int(gaps.argmax())
    return float((a[lo + i] + a[lo + i + 1]) / 2)


def _two_steps(fitter, cap, obs, idx, lambdas, clamp_of):
    """step twice (no update): the first finds the roots, clamp_of(roots, valid) picks the clamp of the second, whose roots must
    be bit-identical.  Returns (step output, p, valid, clamp)."""
    fitter.step(obs, idx, lambdas, 0.1, 0.01, apply_update=False)
    p, valid = cap.roots[-1]
    clamp = clamp_of(p, valid)
    out = fitter.step(obs, idx, lambdas, clamp, 0.01, apply_update=False)
    assert torch.equal(cap.roots[-1][0], p) and torch.equal(cap.roots[-1][1], valid), 'the Broyden roots changed between calls'
    return out, p, valid, clamp


def _latent_parts(Q):
    if Q.nphm:
        P = Q.id
        return [('z_glob', slice(0, P.G))] + [('z_%d' % m, slice(P.G + m * P.L, P.G + (m + 1) * P.L)) for m in range(P.M)]
    D = Q.id[0][0].shape[1] - 3
    return [('z[%d:%d]' % (a, a + 64), slice(a, a + 64)) for a in range(0, D, 64)]


def _check_subject(chk, what, Q64, Q32, g_id, g_ex, p, valid, z_id, z_ex, idx, lambdas, clamp, period):
    """One subject's d/d z_id (per block) and d/d z_ex (per sampled row; the others exactly zero) against float64."""
    r64 = J.joint_gradients(Q64, p.double(), valid, z_id.double(), z_ex.double(), idx, lambdas, clamp, period)
    r32 = J.joint_gradients(Q32, p, valid, z_id, z_ex, idx, lambdas, clamp, period)
    assert r64[2] == r32[2] > 0, (what, r64[2], r32[2])
    chk(what + ' z_id', g_id, r64[0], r32[0], kind='scalar', parts=_latent_parts(Q64))
    rows = idx.tolist()
    parts = [('row %d%s' % (r, ' (sampled twice)' if rows.count(r) > 1 else ''), r) for r in sorted(set(rows))]
    chk(what + ' z_ex', g_ex, r64[1], r32[1], kind='scalar', parts=parts)
    for r in range(z_ex.shape[0]):
        if r not in rows:
            assert bool((g_ex[r] == 0).all()), (what, 'unsampled row %d' % r)
    return r64[2]


def _check_adjoint(chk, what, Q64, Q32, cap):
    """The condition gradient of the fitter's adjoint pass against float64 at its own points, condition and upstream."""
    xyz, cond, up, g_cond = cap.adjoint
    gc64 = C.ref_vjp(Q64.expr, xyz.double(), cond.double(), up.double())[1]
    gc32 = C.ref_vjp(Q32.expr, xyz, cond, up)[1]
    chk(what + ' g_cond', g_cond, gc64, gc32, kind='cond')


def _report_u(chk, what, u):
    m = float(u.abs().max())
    print('JOINT %-16s %-44s max|u| %.3e' % (chk.tag, what, m))
    return m


# ------------------------------------------------------------------------------------------------ single-subject fitters
@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('lambdas', [LAMBDAS, SURFACE_ONLY], ids=['fitting-yaml', 'surface-only'])
def test_joint_fitter(training, lambdas):
    """JointFitter (identity ensemble + 'compress' deformation network); in eval mode the last point of every row carries the
    ensemble's quirk."""
    from nphm_b200.models.fitting import JointFitter, _native_joint
    dec, dfn, Q64, Q32 = _nphm()
    dec.train(training)
    assert _native_joint(dec, dfn, torch.device(DEV))
    chk = Check('JointFitter', K, FLOOR, prefix='JOINT')
    fitter = JointFitter(dec, dfn, 4, torch.device(DEV))
    z_id, z_ex = _codes('fit_joint.npz', 2, 0)
    fitter.z_id.copy_(z_id)
    fitter.z_ex.copy_(z_ex)
    idx = torch.tensor(OBS_IDX, device=DEV)
    obs = _sample(_scans('fit_joint.npz', 0), OBS_IDX, N_POINT)
    period = 0 if training else N_POINT
    cap = _Capture(fitter.mlp)
    try:
        clamp_of = lambda p, v: _clamp_in_a_gap(J.sdf_at_roots(Q64, p, z_id, period).abs(), v.reshape(-1))
        (g_id, g_ex), p, valid, clamp = _two_steps(fitter, cap, obs, idx, lambdas, clamp_of)
        what = '%s %s' % ('train' if training else 'eval', 'yaml' if len(lambdas) > 1 else 'surface')
        # the production range of the adjoint's upstream: d surface / d xc over thousands of kept points
        assert _report_u(chk, what, cap.adjoint[2]) < 1e-3
        kept = _check_subject(chk, what, Q64, Q32, g_id, g_ex, p, valid, z_id, z_ex, idx, lambdas, clamp, period)
        assert int(fitter.terms[5]) == kept, (int(fitter.terms[5]), kept)
        _check_adjoint(chk, what, Q64, Q32, cap)
    finally:
        cap.release()
    chk.done()


@pytest.mark.parametrize('lambdas', [LAMBDAS, SURFACE_ONLY], ids=['fitting-yaml', 'surface-only'])
def test_npm_joint_fitter(lambdas):
    """NpmJointFitter (DeepSDF identity and expression decoders of fitting_npm.yaml)."""
    from nphm_b200.models.fitting import NpmJointFitter, _native_npm_joint
    dec, expr, Q64, Q32 = _npm()
    assert _native_npm_joint(dec, expr, torch.device(DEV))
    chk = Check('NpmJointFitter', K, FLOOR_NPM, prefix='JOINT')
    fitter = NpmJointFitter(dec, expr, 4, torch.device(DEV))
    z_id, z_ex = _codes('fit_npm.npz', 3, 1)
    fitter.z_id.copy_(z_id)
    fitter.z_ex.copy_(z_ex)
    idx = torch.tensor(OBS_IDX, device=DEV)
    obs = _sample(_scans('fit_npm.npz', 1), OBS_IDX, N_POINT)
    cap = _Capture(fitter.mlp)
    try:
        clamp_of = lambda p, v: _clamp_in_a_gap(J.sdf_at_roots(Q64, p, z_id).abs(), v.reshape(-1))
        (g_id, g_ex), p, valid, clamp = _two_steps(fitter, cap, obs, idx, lambdas, clamp_of)
        what = 'yaml' if len(lambdas) > 1 else 'surface'
        _report_u(chk, what, cap.adjoint[2])
        kept = _check_subject(chk, what, Q64, Q32, g_id, g_ex, p, valid, z_id, z_ex, idx, lambdas, clamp, 0)
        assert int(fitter.loss_terms[5]) == kept, (int(fitter.loss_terms[5]), kept)
        _check_adjoint(chk, what, Q64, Q32, cap)
    finally:
        cap.release()
    chk.done()


# ------------------------------------------------------------------------------------------------ scan-batched fitters
SUBJECTS = [(1, (N_POINT,)), (3, (N_POINT, 613, 250))]


def _batched_case(fitter, Q64, Q32, chk, S, ns, training, lambdas, golden):
    """S subjects with n_k points per observation: padded behind (training) or in front (eval) by the fitter; each subject
    against float64 on its own roots, and the adjoint pass of all rows."""
    n_point = max(ns)
    codes = [_codes(golden, 1 + k % 3, 10 + k) for k in range(S)]
    for k, (z_id, z_ex) in enumerate(codes):
        fitter.z_id[k].copy_(z_id)
        fitter.z_ex[4 * k:4 * k + 4].copy_(z_ex)
    idx = [torch.tensor(OBS_IDX[k % 5:] + OBS_IDX[:k % 5], device=DEV) for k in range(S)]
    obs = [_sample(_scans(golden, 20 + k), idx[k].tolist(), ns[k]) for k in range(S)]
    front = not training
    period = lambda k: 0 if training else ns[k]

    def own(t, k):
        """Subject k's own points of a padded 5 S x n_point x ... tensor."""
        t = t.reshape(S, 5, n_point, *t.shape[2:])[k]
        return t[:, n_point - ns[k]:] if front else t[:, :ns[k]]

    def clamp_of(p, v):
        a = torch.cat([J.sdf_at_roots(Q64, own(p, k), codes[k][0], period(k)).abs() for k in range(S)])
        keep = torch.cat([own(v, k).reshape(-1) for k in range(S)])
        return _clamp_in_a_gap(a, keep)

    cap = _Capture(fitter.mlp)
    try:
        (g_id, g_ex), p, valid, clamp = _two_steps(fitter, cap, obs, idx, lambdas, clamp_of)
        mode = 'train' if training else 'eval'
        what = 'S=%d %s %s' % (S, mode, 'yaml' if len(lambdas) > 1 else 'surface')
        _report_u(chk, what, cap.adjoint[2])
        # the padding points repeat a row's first point and are searched like it: compared with each subject's own points
        # only, any contribution of theirs is an error
        for k in range(S):
            z_id, z_ex = codes[k]
            kept = _check_subject(chk, '%s subject %d (n %d)' % (what, k, ns[k]), Q64, Q32, g_id[k], g_ex[k], own(p, k),
                                  own(valid, k), z_id, z_ex, idx[k], lambdas, clamp, period(k))
            if not Q64.nphm:
                assert int(fitter.loss_terms[k, 5]) == kept, (k, int(fitter.loss_terms[k, 5]), kept)
        _check_adjoint(chk, what, Q64, Q32, cap)
    finally:
        cap.release()


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('S,ns', SUBJECTS, ids=['S1', 'S3'])
def test_batched_joint_fitter(S, ns, training):
    """BatchedJointFitter with one subject and with three of unequal lengths."""
    from nphm_b200.models.fitting import BatchedJointFitter
    dec, dfn, Q64, Q32 = _nphm()
    dec.train(training)
    chk = Check('BatchedJoint', K, FLOOR, prefix='JOINT')
    fitter = BatchedJointFitter(dec, dfn, [4] * S, torch.device(DEV))
    _batched_case(fitter, Q64, Q32, chk, S, ns, training, LAMBDAS, 'fit_joint.npz')
    chk.done()


@pytest.mark.parametrize('lambdas', [LAMBDAS, SURFACE_ONLY], ids=['fitting-yaml', 'surface-only'])
@pytest.mark.parametrize('S,ns', SUBJECTS, ids=['S1', 'S3'])
def test_batched_npm_joint_fitter(S, ns, lambdas):
    """BatchedNpmJointFitter with one subject and with three of unequal lengths (padded behind)."""
    from nphm_b200.models.fitting import BatchedNpmJointFitter
    dec, expr, Q64, Q32 = _npm()
    chk = Check('BatchedNpmJoint', K, FLOOR_NPM, prefix='JOINT')
    fitter = BatchedNpmJointFitter(dec, expr, [4] * S, torch.device(DEV))
    _batched_case(fitter, Q64, Q32, chk, S, ns, True, lambdas, 'fit_npm.npz')
    chk.done()

