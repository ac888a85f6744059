"""Every layer-chain entry point of a DeepSDF stack (csrc/mlp_chain.cu on tc_linear.cu / tc_wgrad.cu) on every stack shape
of tests/chain_shapes_common.py, against the float64 reference there.

Error criterion, per returned tensor: the same operation in fp32 PyTorch (TF32 off) is the yardstick of what fp32 arithmetic
costs at this shape, and

    err_native <= K * err_fp32 + FLOOR * max|ref64|

with both errors the maximum absolute difference from float64.  It is applied to the whole tensor and again, separately, to
the rows of the last 128-row tile, to the last 16-column unit (rows and columns) of every weight and bias gradient, and to
each query's condition gradient, each with its own err_fp32 and max|ref64|: a wrong value confined to one tile or unit is
not hidden by larger values elsewhere.  The kernels multiply in three fp16 passes (hi*hi + hi*lo + lo*hi, ~2^-22 per
product); a kernel that lost the lo terms would be ~2^11 times worse than fp32.  `-s` prints err_native, err_fp32 and their
ratio per configuration and tensor (the criterion: tests/f64_check.py)."""
import pytest
import torch

import chain_shapes_common as C
import f64_check
from f64_check import top_scale

pytestmark = pytest.mark.gpu

# Measured on an H100 80GB HBM3 (700 W power limit) over the whole matrix below (tensors and parts):
# - values, Jacobians, inverse Jacobians, point and condition gradients: worst err_native / err_fp32 123 on a whole tensor
#   (512-1024x8-1 forward, 1 x 257 rows); where the fp32 error happens to be small (a few rows), err_native / max|ref| up to
#   2.2e-5 (train out, 40-881x4-1);
# - weight and bias gradients whose adjoint stays in the range it is stored in (see f64_check.LO_NORMAL): worst err_native
#   beyond 64 * err_fp32, over the whole tensor and its last units, 5.0e-5 of the whole tensor's max|ref| (512-1024x8-1
#   lin7.bias, 1 x 257 rows; 8.5e-6 on the smaller stacks).  A unit of a gradient is a sum over the rows of d_l h_{l-1}
#   whose terms can cancel far below the tensor's largest entry, so its floor is relative to the whole tensor; the
#   64 * err_fp32 term stays the unit's own.
# A kernel that dropped a lo product measured ratios of 1200-4800 and 1.1e-3 of max|ref| on the forward; a weight-gradient
# GEMM that drops one lo pass reaches 1.2e-4 .. 9e-4 of max|ref|.
K = 64.0
FLOOR = 3e-5
FLOOR_GRAD = 6e-5


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def Check(cfg):
    """The criterion of tests/f64_check.py with this file's constants."""
    return f64_check.Check(C.config_id(cfg), K, FLOOR, FLOOR_GRAD)


def _setup(cfg, device):
    net = C.make_stack(cfg, device)
    return net, net.engine(), C.params_of(net, torch.float64), C.params_of(net, torch.float32)


def _inputs(cfg, B, N, device, seed=0):
    x, c = C.make_inputs(cfg, B, N, device, seed)
    return x, c, x.double(), c.double()


def _ids(pairs):
    return ['%s-nd%d' % (C.config_id(c), nd) for c, nd in pairs]


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize('cfg', C.CONFIGS, ids=C.config_id)
def test_forward(cuda_device, cfg):
    """query_layers (and query with impl='simt' where the FFMA kernel takes the width) on every row shape; the chunked
    forward at 65 536 / 65 537 points on two stacks."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    rows = list(C.ROWS) + (list(C.CHUNK_ROWS) if cfg in ((24, 39, 9, 8), (2, 129, 10, 3)) else [])
    for B, N in rows:
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        r64, r32 = C.stack_forward(P64, x64, c64), C.stack_forward(P32, x, c)
        chk('query_layers %dx%d' % (B, N), eng.query_layers(x, c), r64, r32)
        if eng.simt_ok:
            chk('query simt %dx%d' % (B, N), eng.query(x, c, impl='simt'), r64, r32)
    chk.done()


# ------------------------------------------------------------------------------------------------ Jacobian and adjoint
@pytest.mark.parametrize('cfg', C.CONFIGS, ids=C.config_id)
def test_jacobian_and_adjoint(cuda_device, cfg):
    """jacobian, inverse_jacobian (3 outputs), backward_inputs with fresh points and reusing the value pass of jacobian."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    for B, N in C.ROWS:
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        up = torch.randn(B, N, cfg[3], device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(B * N))
        o64, J64 = C.ref_jacobian(P64, x64, c64)
        o32, J32 = C.ref_jacobian(P32, x, c)
        out, J = eng.jacobian(x, c)
        chk('jacobian out %dx%d' % (B, N), out, o64, o32)
        chk('jacobian J %dx%d' % (B, N), J, J64, J32)
        if cfg[3] == 3:
            _, I64 = C.ref_inverse_jacobian(P64, x64, c64)
            _, I32 = C.ref_inverse_jacobian(P32, x, c)
            chk('inverse_jacobian %dx%d' % (B, N), eng.inverse_jacobian(x, c)[1], I64, I32)
        _, gc64, gx64, _, _ = C.ref_vjp(P64, x64, c64, up.double())
        _, gc32, gx32, _, _ = C.ref_vjp(P32, x, c, up)
        g_c, g_x = eng.backward_inputs(x, c, up, want_xyz=True)
        chk('backward_inputs cond %dx%d' % (B, N), g_c, gc64, gc32, 'cond')
        chk('backward_inputs xyz %dx%d' % (B, N), g_x, gx64, gx32)
        eng.jacobian(x, c)
        g_c, g_x = eng.backward_inputs(x, c, up, want_xyz=True, reuse_value_pass=True)
        chk('backward_inputs reuse cond %dx%d' % (B, N), g_c, gc64, gc32, 'cond')
        chk('backward_inputs reuse xyz %dx%d' % (B, N), g_x, gx64, gx32)
    chk.done()


# Upstream magnitudes of the adjoint pass: randn, the joint fitters' u = -J^-T g_x (d surface / d xc over a few thousand
# kept points, 1e-4 and below) and smaller still.  The pass holds every adjoint as an fp16 hi | lo pair, whose lo part is
# subnormal below 2^-3 and whose hi part is below 2^-14; it has to scale the upstream into that range itself.
UPSTREAM_SCALES = [1.0, 2.0 ** -12, 1e-4, 1e-6]


@pytest.mark.parametrize('cfg', C.PRODUCTION, ids=C.config_id)
def test_adjoint_upstream_range(cuda_device, cfg):
    """backward_inputs (condition and point gradients, fresh points and reusing the value pass of inverse_jacobian /
    jacobian) on the production stacks with upstreams of every magnitude in UPSTREAM_SCALES; no range-defect exemption."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    for B, N in ((1, 129), (9, 37), (5, 1000)):
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        base = torch.randn(B, N, cfg[3], device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(3 * B + N))
        for sc in UPSTREAM_SCALES:
            up = base * sc
            _, gc64, gx64, _, _ = C.ref_vjp(P64, x64, c64, up.double())
            _, gc32, gx32, _, _ = C.ref_vjp(P32, x, c, up)
            what = 'backward_inputs up %.0e %dx%d' % (sc, B, N)
            g_c, g_x = eng.backward_inputs(x, c, up, want_xyz=True)
            chk(what + ' cond', g_c, gc64, gc32, 'cond')
            chk(what + ' xyz', g_x, gx64, gx32)
            if cfg[3] == 3:
                eng.inverse_jacobian(x, c)
            else:
                eng.jacobian(x, c)
            g_c, g_x = eng.backward_inputs(x, c, up, want_xyz=True, reuse_value_pass=True)
            chk(what + ' reuse cond', g_c, gc64, gc32, 'cond')
            chk(what + ' reuse xyz', g_x, gx64, gx32)
    chk.done()


# ------------------------------------------------------------------------------------------------ first-order training
TRAIN = [(cfg, nd) for cfg in C.CONFIGS for nd in C.noise_dims(cfg)]


@pytest.mark.parametrize('cfg,nd', TRAIN, ids=_ids(TRAIN))
def test_train(cuda_device, cfg, nd):
    """train_forward / train_backward with nd noise columns: value, weight, bias, condition and point gradients."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    for B, N in C.ROWS:
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        gen = torch.Generator(cuda_device).manual_seed(7 * B + N + nd)
        noise = torch.randn(B, N, nd, device=cuda_device, generator=gen) / 200 if nd else None
        up = torch.randn(B, N, cfg[3], device=cuda_device, generator=gen) * 1e-4
        o64, gc64, gx64, gw64, gb64 = C.ref_vjp(P64, x64, c64, up.double(), None if noise is None else noise.double())
        o32, gc32, gx32, gw32, gb32 = C.ref_vjp(P32, x, c, up, noise)
        out, ws = eng.train_forward(x, c, noise)
        gw, gb, g_c, g_x = eng.train_backward(ws, up, nd, want_xyz=True)
        what = 'train nd=%d %dx%d' % (nd, B, N)
        chk(what + ' out', out, o64, o32)
        chk(what + ' cond', g_c, gc64, gc32, 'cond')
        chk(what + ' xyz', g_x, gx64, gx32)
        adj = C.ref_adjoints(P64, x64, c64, up.double(), None if noise is None else noise.double())
        chk.grads(what, gw, gb, (gw64, gb64), (gw32, gb32), [(adj, top_scale(up))])
    chk.done()


# ------------------------------------------------------------------------------------------------ one-output stacks
ONE_OUT = [cfg for cfg in C.CONFIGS if cfg[3] == 1]


@pytest.mark.parametrize('cfg', ONE_OUT, ids=C.config_id)
def test_sdfgrad(cuda_device, cfg):
    """sdfgrad_forward / sdfgrad_backward: s, grad_x s, and the double backward's weight, bias, condition and point
    gradients."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    for B, N in C.ROWS:
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        gen = torch.Generator(cuda_device).manual_seed(11 * B + N)
        sbar = torch.randn(B, N, 1, device=cuda_device, generator=gen) * 1e-4
        gbar = torch.randn(B, N, 3, device=cuda_device, generator=gen) * 1e-4
        s64, g64 = C.ref_sdfgrad(P64, x64, c64)
        s32, g32 = C.ref_sdfgrad(P32, x, c)
        gc64, gx64, gw64, gb64 = C.ref_sdfgrad_vjp(P64, x64, c64, sbar.double(), gbar.double())
        gc32, gx32, gw32, gb32 = C.ref_sdfgrad_vjp(P32, x, c, sbar, gbar)
        s, g, ws = eng.sdfgrad_forward(x, c)
        gw, gb, g_c, g_x = eng.sdfgrad_backward(ws, sbar, gbar, want_xyz=True)
        what = 'sdfgrad %dx%d' % (B, N)
        chk(what + ' s', s, s64, s32)
        chk(what + ' grad_x s', g, g64, g32)
        chk(what + ' cond', g_c, gc64, gc32, 'cond')
        chk(what + ' xyz', g_x, gx64, gx32)
        a, zb = C.ref_sdfgrad_adjoints(P64, x64, c64, sbar.double(), gbar.double())
        chk.grads(what, gw, gb, (gw64, gb64), (gw32, gb32), [(a, 2.0 ** 10), (zb, top_scale(sbar, gbar))])
    chk.done()


def _centre_output(net, P64, cfg, device):
    """Shift the output bias so that s changes sign over the test points (the surface term keeps |s| < clamp); returns the
    shift (the output's magnitude before it, what the rounding error of s scales with)."""
    x, c = C.make_inputs(cfg, 3, 100, device, seed=99)          # not the test's points: none of them lands on s = 0
    s = C.stack_forward(P64, x.double(), c.double())
    last = getattr(net, 'lin%d' % (net.num_layers - 2))
    with torch.no_grad():
        last.bias.sub_(float(s.median()))
    return abs(float(s.median()))


def _clamp_in_a_gap(s64, kept_mask):
    """A clamp in the widest gap between consecutive |s| of the masked points (middle half of their range), so that fp32
    rounding cannot move a point across it."""
    a = s64.abs()[kept_mask].sort().values
    if a.numel() < 4:
        return float(a.max()) * 2 + 1.0
    lo, hi = a.numel() // 4, max(a.numel() * 3 // 4, a.numel() // 4 + 1)
    gaps = a[lo + 1:hi + 1] - a[lo:hi]
    i = int(gaps.argmax())
    return float((a[lo + i] + a[lo + i + 1]) / 2)


@pytest.mark.parametrize('cfg', ONE_OUT, ids=C.config_id)
def test_fit_surface_grad(cuda_device, cfg):
    """fit_surface_grad with a mask and a clamp that drops part of the points: the loss, the kept count (exact) and the
    condition and point gradients."""
    net = C.make_stack(cfg, cuda_device)
    shift = _centre_output(net, C.params_of(net, torch.float64), cfg, cuda_device)
    eng, P64, P32 = net.engine(), C.params_of(net, torch.float64), C.params_of(net, torch.float32)
    chk = Check(cfg)
    for B, N in C.ROWS:
        x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
        mask = torch.rand(B, N, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(B + N)) < 0.8
        mask.view(-1)[0] = True
        s64 = C.stack_forward(P64, x64, c64)[..., 0]
        clamp = _clamp_in_a_gap(s64, mask)
        l64, n64, gc64, gx64 = C.ref_fit_surface(P64, x64, c64, mask, clamp)
        l32, n32, gc32, gx32 = C.ref_fit_surface(P32, x, c, mask, clamp)
        assert n32 == n64
        terms, g_c, g_x = eng.fit_surface_grad(x, c, mask, clamp)
        what = 'fit_surface_grad %dx%d' % (B, N)
        assert int(terms[5]) == n64, (what, int(terms[5]), n64)
        chk(what + ' loss', terms[0], l64, l32, 'scalar', scale=float(s64.abs().max()) + shift)
        chk(what + ' cond', g_c, gc64, gc32, 'cond')
        chk(what + ' xyz', g_x, gx64, gx32)
    chk.done()


# ------------------------------------------------------------------------------------------------ Broyden search
THREE_OUT = [cfg for cfg in C.CONFIGS if cfg[3] == 3]


@pytest.mark.parametrize('cfg', THREE_OUT, ids=C.config_id)
def test_broyden_search(cuda_device, cfg):
    """Roots of x + F(x) = obs (the FFMA kernel up to hidden 905, the layer chain above): the float64 residual at the
    returned roots against the reported ``diff`` of every converged point, and ``valid == (diff < cvg_thresh)``.  The
    trajectories themselves are not compared."""
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    cvg = 1e-5
    for B, N in ((1, 129), (9, 37), (2, 200)):
        x_true, c, _, c64 = _inputs(cfg, B, N, cuda_device, seed=1)
        x_true = x_true * 0.5
        obs = (x_true.double() + C.stack_forward(P64, x_true.double(), c64)).float()
        x0 = obs.clone()
        _, jinv = eng.inverse_jacobian(x0, c)
        x, diff, valid, _ = eng.broyden_search(obs, c, x0, jinv, max_steps=20, cvg_thresh=cvg)
        assert torch.equal(valid, diff < cvg)
        v = valid.reshape(-1)
        assert float(v.double().mean()) >= 0.9, (B, N, float(v.double().mean()))
        r64 = C.broyden_residual(P64, x.double(), c64, obs.double()).norm(dim=-1).reshape(-1)[v]
        r32 = C.broyden_residual(P32, x, c, obs).norm(dim=-1).reshape(-1)[v]
        assert float(r64.max()) <= cvg * 1.5, float(r64.max())
        en = float((diff.reshape(-1)[v].double() - r64).abs().max())
        ef = float((r32.double() - r64).abs().max())
        bound = K * ef + FLOOR * float(obs.abs().max())
        print('CHAIN %-16s broyden %dx%d: %d/%d converged, |diff - residual64| %.3e, fp32 residual err %.3e, bound %.3e'
              % (chk.tag, B, N, int(v.sum()), v.numel(), en, ef, bound))
        if not en <= bound:
            chk.bad.append('broyden %dx%d: |diff - residual64| %.3e > %.3e' % (B, N, en, bound))
    chk.done()


# ------------------------------------------------------------------------------------------------ production row counts
# The row counts of one decoder call in training: stage 2 (32 x 1100 points: the deformation backbone with 32 noise columns,
# the expression decoder's Jacobian and adjoint) and stage 1 (32 x 1693 points: the NPM identity decoder through grad_x s).
# At these counts the weight-gradient GEMM splits its rows differently and the per-query sums run over >1000 rows.
def test_production_rows_stage2_train(cuda_device):
    cfg = (232, 512, 6, 3)
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    B, N = C.STAGE2_ROWS
    x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
    gen = torch.Generator(cuda_device).manual_seed(5)
    noise = torch.randn(B, N, 32, device=cuda_device, generator=gen) / 200
    up = torch.randn(B, N, 3, device=cuda_device, generator=gen) * 1e-4
    o64, gc64, gx64, gw64, gb64 = C.ref_vjp(P64, x64, c64, up.double(), noise.double())
    o32, gc32, gx32, gw32, gb32 = C.ref_vjp(P32, x, c, up, noise)
    out, ws = eng.train_forward(x, c, noise)
    gw, gb, g_c, g_x = eng.train_backward(ws, up, 32, want_xyz=True)
    chk('stage-2 train out', out, o64, o32)
    chk('stage-2 train cond', g_c, gc64, gc32, 'cond')
    chk('stage-2 train xyz', g_x, gx64, gx32)
    del o64, o32, gx64, gx32
    adj = C.ref_adjoints(P64, x64, c64, up.double(), noise.double())
    chk.grads('stage-2 train', gw, gb, (gw64, gb64), (gw32, gb32), [(adj, top_scale(up))])
    chk.done()


def test_production_rows_stage2_jacobian_adjoint(cuda_device):
    cfg = (712, 1024, 8, 3)
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    B, N = C.STAGE2_ROWS
    x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
    up = torch.randn(B, N, 3, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(6))
    out, J = eng.jacobian(x, c)
    o64, J64 = C.ref_jacobian(P64, x64, c64)
    o32, J32 = C.ref_jacobian(P32, x, c)
    chk('stage-2 jacobian out', out, o64, o32)
    chk('stage-2 jacobian J', J, J64, J32)
    _, gc64, gx64, _, _ = C.ref_vjp(P64, x64, c64, up.double())
    _, gc32, gx32, _, _ = C.ref_vjp(P32, x, c, up)
    g_c, g_x = eng.backward_inputs(x, c, up, want_xyz=True, reuse_value_pass=True)
    chk('stage-2 backward_inputs cond', g_c, gc64, gc32, 'cond')
    chk('stage-2 backward_inputs xyz', g_x, gx64, gx32)
    chk.done()


def test_production_rows_stage1_sdfgrad(cuda_device):
    cfg = (512, 1024, 8, 1)
    net, eng, P64, P32 = _setup(cfg, cuda_device)
    chk = Check(cfg)
    B, N = C.STAGE1_ROWS
    x, c, x64, c64 = _inputs(cfg, B, N, cuda_device)
    gen = torch.Generator(cuda_device).manual_seed(7)
    sbar = torch.randn(B, N, 1, device=cuda_device, generator=gen) * 1e-5
    gbar = torch.randn(B, N, 3, device=cuda_device, generator=gen) * 1e-5
    s, g, ws = eng.sdfgrad_forward(x, c)
    gw, gb, g_c, g_x = eng.sdfgrad_backward(ws, sbar, gbar, want_xyz=True)
    s64, g64 = C.ref_sdfgrad(P64, x64, c64)
    s32, g32 = C.ref_sdfgrad(P32, x, c)
    chk('stage-1 sdfgrad s', s, s64, s32)
    chk('stage-1 sdfgrad grad_x s', g, g64, g32)
    del s64, g64, s32, g32
    gc64, gx64, gw64, gb64 = C.ref_sdfgrad_vjp(P64, x64, c64, sbar.double(), gbar.double())
    gc32, gx32, gw32, gb32 = C.ref_sdfgrad_vjp(P32, x, c, sbar, gbar)
    chk('stage-1 sdfgrad cond', g_c, gc64, gc32, 'cond')
    chk('stage-1 sdfgrad xyz', g_x, gx64, gx32)
    del gx64, gx32
    a, zb = C.ref_sdfgrad_adjoints(P64, x64, c64, sbar.double(), gbar.double())
    chk.grads('stage-1 sdfgrad', gw, gb, (gw64, gb64), (gw32, gb32), [(a, 2.0 ** 10), (zb, top_scale(sbar, gbar))])
    chk.done()
