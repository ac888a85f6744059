"""Every entry point of the identity ensemble (the dense tensor-core kernel, the FFMA kernels, the fitting pipeline of
csrc/fit.cu, Adam, the stage-1 member passes) against the float64 reference of tests/ensemble_f64_common.py, on the
configurations there.

The criterion is that of tests/f64_check.py, err_native <= K * err_fp32 + FLOOR * max|ref64|, applied to the whole tensor and
again to each of its parts, each with its own err_fp32 and max|ref64|: the last 128-row tile, the rows each member dominates
(one group per member), the far rows (only the background weight left) and the quirk rows; for a latent gradient the z_glob
block and every member's block; every anchor; every scan; for a stage-1 weight or bias gradient every weight set.  A member
whose anchor sees few points has a latent block 1e-2 .. 1e-4 of the tensor's largest entry, and the regulariser-only blocks of
the unobserved members are smaller still: checked on its own, such a block cannot hide behind the rest.  `-s` prints the
ratios per tensor and, at the end of each test, the worst ratio per entry point.
"""
import ctypes

import pytest
import torch

import ensemble_f64_common as E
from f64_check import Check

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F32, F64 = torch.float32, torch.float64

# Floors, each relative to the checked tensor's or part's own max|ref64|.  Measured on an H100 80GB HBM3 (700 W power limit)
# over every test below, the smallest floor each check needs beyond K * err_fp32 + 2^-24 max|ref64| of the whole tensor:
# - values: 1.1e-5 (backward_inputs sdf, the rows one member dominates), member outputs 4.8e-6, queries 3.0e-6, the
#   fitting loss 4.5e-7 (relative to the loss itself), everything else 0;
# - gradients: 6.6e-7 (the stage-1 output-layer bias of one weight set), everything else 0;
# - the latent blocks of the fitting backward: 0.  The fitting backward holds the member deltas as fp16 hi | lo pairs at the
#   fixed scale kDeltaScale = 64 (fit.cu), and a member whose anchor sees few points has a block 1e-2 .. 1e-4 of the largest
#   entry: there err_native / err_fp32 reaches 3.6e5, but every block's error stays within the criterion's other terms (64
#   x the block's own fp32 error, or 2^-24 of the whole gradient's max).  FLOOR_BLOCK bounds the blocks beyond that.
FLOOR = 2e-5                # values: SDFs, member outputs, anchors, loss terms
FLOOR_GRAD = 2e-6           # gradients w.r.t. points, codes and (stage 1) each weight set's parameters
FLOOR_BLOCK = 1e-6          # each member's block and the z_glob block of the fitting backward's latent gradient
# Query parts of the tensor-core structures with 'stack' weights (layer 0 and the skip layer x3, the other hidden layers x2
# and their biases x4).  Measured on tc-split-80-16: 2.06e-5 of the part's own max|ref|, at the rows member 22 dominates in
# one query of 37 rows, where |sdf| <= 3.3e-3, 1/60 of the query's max (err_native 1.82e-7, err_fp32 1.6e-9).  Its member
# outputs and every differentiated entry point pass FLOOR; the error is absolute, about 2^-22 of the larger internal
# magnitudes these weights give, so it shows as a relative error only where the blended SDF is small.
FLOOR_STACK_QUERY = 3e-5
K = 64.0
LAMBDAS = (2.0, 0.25, 0.05, 10.0, 5.0)      # surface, reg_global, reg_loc, reg_unobserved, symm_dist (fitting.yaml)


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _check(name):
    return Check(name, K, FLOOR, prefix='ENSEMBLE')


def _tc(name):
    n_loc, _, G, L, H, nl, _ = E.CONFIGS[name]
    return H == 200 and G + L == 96 and nl == 4 and n_loc + 1 <= 64


TC = [k for k in E.CONFIGS if _tc(k)]
TC_WIDTHS = [k for k, c in E.CONFIGS.items() if c[4] == 200 and c[2] + c[3] == 96]


def _setup(name):
    dec = E.make_decoder(name, DEV)
    return dec, dec.engine(), E.Params(dec, F64), E.Params(dec, F32)


def _lib():
    from nphm_b200 import _native
    return _native.lib()


def _run(rc, what):
    from nphm_b200 import _native
    _native.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _row_parts(P64, xyz64, z64, kind=None, period=0, prefix='', quirk=None):
    """(name, row index) of the rows each member dominates (float64 blend weights), the far rows and the quirk rows (those of
    the fitting kernels' period, or the mask ``quirk``)."""
    w = E.blend_weights(P64, xyz64, E.anchors(P64, z64))
    top = w.argmax(dim=1).cpu()
    parts = []
    for m in sorted(set(top.tolist())):
        parts.append(('%smember %d' % (prefix, m), (top == m).nonzero().reshape(-1).to(xyz64.device)))
    if kind is not None and bool((kind == 2).any()):
        parts.append((prefix + 'far', (kind == 2).nonzero().reshape(-1).to(xyz64.device)))
    q = E.quirk_rows(xyz64.shape[0], period) if quirk is None else quirk
    if bool(q.any()):
        parts.append((prefix + 'quirk', q.nonzero().reshape(-1).to(xyz64.device)))
    return parts


def _latent_parts(P):
    return [('z_glob', slice(0, P.G))] + [('z_%d' % m, slice(P.G + m * P.L, P.G + (m + 1) * P.L)) for m in range(P.M)]


def _points(P64, z64, n, seed=0):
    x64, kind = E.mixed_points(P64, z64, n, seed)
    x = x64.float()
    return x, x.double(), kind


# ------------------------------------------------------------------------------------------------ queries
@pytest.mark.parametrize('name', list(E.CONFIGS))
def test_query(name):
    """query with impl 'simt' on every configuration, 'tc' and 'auto' where the tensor-core kernel takes it; several queries
    per call, and the eval-mode quirk by period.  At 65 members the tensor-core kernel refuses the ensemble."""
    from nphm_b200 import _native
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    impls = ['simt'] + (['tc', 'auto'] if _tc(name) else [])
    if name in TC_WIDTHS and not _tc(name):
        with pytest.raises(_native.NativeError, match='tensor-core'):
            eng.query(torch.zeros(1, 4, 3, device=DEV), E.latent(name, device=DEV)[None], eval_quirk=False, impl='tc')
    rows = E.ROWS if _tc(name) or name in ('api', 'fit') else [(1, 129), (3, 129), (1, 257)]
    for B, N in rows:
        zs = [E.latent(name, seed=b, device=DEV) for b in range(B)]
        pts = [_points(P64, z.double(), N, seed=b) for b, z in enumerate(zs)]
        x = torch.stack([p[0] for p in pts])
        lat = torch.stack(zs)
        periods = [0] + ([p for p in E.quirk_periods(N) if p in (1, 128, N)] if N > 1 or B > 1 else [1])
        for period in periods:
            q = E.query_quirk_rows(N, period)
            r64 = torch.stack([E.sdf(P64, p[1], z.double(), quirk=q) for p, z in zip(pts, zs)]).detach()
            r32 = torch.stack([E.sdf(P32, p[0], z, quirk=q) for p, z in zip(pts, zs)]).detach()
            parts = []
            for b, (p, z) in enumerate(zip(pts, zs)):
                parts += [(nm, (b, i)) for nm, i in _row_parts(P64, p[1], z.double(), p[2], prefix='q%d ' % b, quirk=q)]
            for impl in impls:
                got = eng.query(x, lat, eval_quirk=period > 0, quirk_period=period or None, impl=impl)[0][..., 0]
                part_floor = FLOOR_STACK_QUERY if impl != 'simt' and E.CONFIGS[name][6] == 'stack' else None
                chk('query %s %dx%d p%d' % (impl, B, N, period), got, r64, r32, parts=parts, part_floor=part_floor)
    chk.done()


def _grid_points(res, first, count):
    from conftest import MAXI, MINI
    import numpy as np
    axes = [torch.from_numpy(np.linspace(MINI[a], MAXI[a], res).astype('float32')) for a in range(3)]
    xyz = torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=-1).reshape(-1, 3)[first:first + count]
    return xyz.to(DEV)


def _chunked(f, x, step=65536):
    return torch.cat([f(x[i:i + step]) for i in range(0, x.shape[0], step)])


@pytest.mark.parametrize('name', ['prod', 'prod-x2', 'tc-64m', 'tc-64m-nosymm'])
def test_query_grid(name):
    """query_grid over a whole 64^3 grid (blocked tiles, zero-weight members skipped), x-slabs, an unaligned range with the
    quirk, and the pruned kernel against its bound n_members * tau * max_k |s_k| (max over float64 s_k per point)."""
    from conftest import MAXI, MINI
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    z = E.latent(name, seed=5, device=DEV)
    res = 64
    with torch.no_grad():
        whole = _grid_points(res, 0, res ** 3)
        s64 = _chunked(lambda x: E.sdf(P64, x.double(), z.double(), with_members=True)[0], whole)
        s32 = _chunked(lambda x: E.sdf(P32, x, z), whole)
        smax = _chunked(lambda x: E.sdf(P64, x.double(), z.double(), with_members=True)[1].abs().max(dim=1).values, whole)
    for impl in ('tc', 'simt'):
        got = eng.query_grid(z, MINI, MAXI, res, 0, res ** 3, 0, impl=impl)[0]
        chk('grid %s whole' % impl, got, s64, s32, parts=[('x-plane %d' % i, slice(i * res * res, (i + 1) * res * res))
                                                         for i in (0, 17, 31, 63)])
        for x0, x1 in ((0, 8), (27, 40), (60, 64)):
            a, b = x0 * res * res, x1 * res * res
            got = eng.query_grid(z, MINI, MAXI, res, a, b - a, 0, impl=impl)[0]
            chk('grid %s x-slab %d-%d' % (impl, x0, x1), got, s64[a:b], s32[a:b])
        first, count = 12345, 50001
        for period in (0, 129, 4096):
            got = eng.query_grid(z, MINI, MAXI, res, first, count, period, impl=impl)[0]
            x = whole[first:first + count]
            q = E.query_quirk_rows(count, period, first, res ** 3)          # by grid index
            with torch.no_grad():
                r64 = E.sdf(P64, x.double(), z.double(), quirk=q)
                r32 = E.sdf(P32, x, z, quirk=q)
            chk('grid %s unaligned p%d' % (impl, period), got, r64, r32,
                parts=[('quirk', q.nonzero().reshape(-1).to(DEV))] if period else ())
    for tau in (1e-8, 1e-4):
        eng.set_prune_threshold(tau)
        got = eng.query_grid(z, MINI, MAXI, res, 0, res ** 3, 0, impl='tc_pruned')[0]
        bound = P64.M * tau * smax + K * (s32.double() - s64).abs() + FLOOR * float(s64.abs().max())
        err = (got.double() - s64).abs()
        bad = int((err > bound).sum())
        print('ENSEMBLE %-16s tc_pruned tau %.0e: max err %.3e, max err / bound %.3f, max_k |s_k| up to %.3f'
              % (name, tau, float(err.max()), float((err / bound).max()), float(smax.max())))
        if bad:
            chk.bad.append('tc_pruned tau %g: %d points beyond n_members * tau * max_k |s_k|' % (tau, bad))
    eng.set_prune_threshold(0.0)
    chk.done()


# ------------------------------------------------------------------------------------------------ fitting pipeline
def _surface_call(eng, dec, x, z, mask, clamp, period=0, grad_points=True):
    lib = _lib()
    n = x.shape[0]
    ws = torch.zeros(lib.nphm_fit_batch_workspace_bytes(eng.handle, 1, n), dtype=torch.uint8, device=DEV)
    terms = torch.full((8,), 7.0, device=DEV)
    g_lat = torch.empty(dec.lat_dim, device=DEV)
    g_pts = torch.empty(n, 3, device=DEV) if grad_points else None
    m = None if mask is None else mask.to(torch.uint8).contiguous()
    gp = g_pts.data_ptr() if grad_points else None
    if period:
        rc = lib.nphm_fit_surface_grad_quirk(eng.handle, x.data_ptr(), n, period, z.data_ptr(), None if m is None else m.data_ptr(),
                                             float(clamp), terms.data_ptr(), g_lat.data_ptr(), gp, ws.data_ptr(), _stream())
    else:
        rc = lib.nphm_fit_surface_grad(eng.handle, x.data_ptr(), n, z.data_ptr(), None if m is None else m.data_ptr(),
                                       float(clamp), terms.data_ptr(), g_lat.data_ptr(), gp, ws.data_ptr(), _stream())
    return rc, terms, g_lat, g_pts, ws


@pytest.mark.parametrize('name', TC)
def test_member_outputs_and_anchors(name):
    """The per-member outputs s_k the fitting forward leaves in the first block of its workspace (one column per member; at
    fitting sizes the members of a tile are split over CTAs) and nphm_ensemble_anchors, per anchor."""
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    for n in (1, 129, 300, 1000):
        z = E.latent(name, seed=n, device=DEV)
        x, x64, kind = _points(P64, z.double(), n, seed=n)
        rc, _, _, _, ws = _surface_call(eng, dec, x, z, None, 0.1)
        _run(rc, 'nphm_fit_surface_grad')
        got = ws.view(F32)[:n * P64.M].reshape(n, P64.M)
        with torch.no_grad():
            s64 = E.members(P64, x64, z.double())
            s32 = E.members(P32, x, z)
        chk('members %d' % n, got, s64, s32, parts=[('member %d' % m, (slice(None), m)) for m in range(P64.M)])
    lat = torch.stack([E.latent(name, seed=s, device=DEV) for s in range(4)] + [torch.zeros(dec.lat_dim, device=DEV)])
    got = eng.anchors(lat)
    with torch.no_grad():
        a64 = torch.stack([E.anchors(P64, z.double()) for z in lat])
        a32 = torch.stack([E.anchors(P32, z) for z in lat])
    chk('anchors', got, a64, a32, kind='scalar', parts=[('anchor %d' % k, (slice(None), k)) for k in range(P64.n_loc)])
    chk.done()


@pytest.mark.parametrize('name', TC)
def test_backward_inputs(name):
    """nphm_ensemble_backward_inputs(_quirk): sdf, the latent gradient per block and the point gradient per row group, with
    period 0, a period that splits the call and one eval-mode call."""
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    for n in (1, 127, 129, 1000):
        z = E.latent(name, seed=n, device=DEV)
        x, x64, kind = _points(P64, z.double(), n, seed=n)
        up = torch.randn(n, generator=torch.Generator().manual_seed(n)).to(DEV)
        for period in sorted({0, min(n, 129), n}):
            s, g_lat, g_pts = eng.backward_inputs(x, z, up, quirk_period=period)
            s64, gz64, gx64 = E.vjp(P64, x64, z.double(), up.double(), period)
            s32, gz32, gx32 = E.vjp(P32, x, z, up, period)
            rp = _row_parts(P64, x64, z.double(), kind, period)
            what = 'backward_inputs %d p%d' % (n, period)
            chk(what + ' sdf', s, s64, s32, parts=rp)
            chk(what + ' latent', g_lat, gz64, gz32, kind='scalar', parts=_latent_parts(P64), floor=FLOOR_GRAD,
                part_floor=FLOOR_BLOCK)
            chk(what + ' xyz', g_pts, gx64, gx32, parts=rp, floor=FLOOR_GRAD)
    chk.done()


def _clamp_away(s64, c):
    """c, moved to the middle of its gap between consecutive |s| if a value lies within 1e-5 of it (fp32 rounding must not move
    a point across the clamp)."""
    a = s64.abs().sort().values
    if not bool(((a - c).abs() < 1e-5).any()):
        return c
    lo, hi = a[a < c - 1e-5], a[a > c + 1e-5]
    lo = float(lo.max()) if lo.numel() else 0.0
    hi = float(hi.min()) if hi.numel() else 2 * c
    return (lo + hi) / 2


@pytest.mark.parametrize('name', TC)
def test_fit_surface_grad(name):
    """nphm_fit_surface_grad(_quirk) with masks and clamps 0.1, 0.02, 0.0075: loss, kept count (exact), latent and point
    gradients; with nothing kept a NaN loss and exactly zero gradients."""
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    for n in (1, 129, 1000):
        z = E.latent(name, seed=10 + n, device=DEV)
        x, x64, kind = _points(P64, z.double(), n, seed=10 + n)
        mask = torch.rand(n, generator=torch.Generator().manual_seed(n)).to(DEV) < 0.8
        mask[0] = True
        for period in sorted({0, n}):
            with torch.no_grad():
                s64 = E.sdf(P64, x64, z.double(), period)
            for c0 in (0.1, 0.02, 0.0075):
                clamp = _clamp_away(s64[mask], c0)
                l64, k64, gz64, gx64 = E.fit_surface(P64, x64, z.double(), mask, clamp, period)
                l32, k32, gz32, gx32 = E.fit_surface(P32, x, z, mask, clamp, period)
                rc, terms, g_lat, g_pts, _ = _surface_call(eng, dec, x, z, mask, clamp, period)
                _run(rc, 'nphm_fit_surface_grad')
                what = 'fit_surface_grad %d p%d c%g' % (n, period, c0)
                assert int(terms[5]) == k64 == k32, (what, float(terms[5]), k64, k32)
                if k64 == 0:
                    assert bool(torch.isnan(terms[0])), what
                    assert bool((g_lat == 0).all()) and bool((g_pts == 0).all()), what
                    continue
                rp = [(nm, i) for nm, i in _row_parts(P64, x64, z.double(), kind, period)]
                chk(what + ' loss', terms[0], l64, l32, kind='scalar')
                chk(what + ' latent', g_lat, gz64, gz32, kind='scalar', parts=_latent_parts(P64), floor=FLOOR_GRAD,
                    part_floor=FLOOR_BLOCK)
                chk(what + ' xyz', g_pts, gx64, gx32, parts=rp, floor=FLOOR_GRAD)
    # nothing kept: every row masked out, and a clamp of 0
    z = E.latent(name, device=DEV)
    x, _, _ = _points(P64, z.double(), 200)
    for mask, clamp in ((torch.zeros(200, dtype=torch.bool, device=DEV), 0.1), (None, 0.0)):
        rc, terms, g_lat, g_pts, _ = _surface_call(eng, dec, x, z, mask, clamp)
        _run(rc, 'nphm_fit_surface_grad')
        assert int(terms[5]) == 0 and bool(torch.isnan(terms[0]))
        assert bool((g_lat == 0).all()) and bool((g_pts == 0).all())
    chk.done()


def _identity_call(eng, dec, x, z, lambdas, clamp, period=0):
    from nphm_b200 import _native
    lib = _lib()
    fp = _native.FitParams(*[float(v) for v in lambdas], float(clamp), 0.01, 1)
    lat = z.clone()
    terms = torch.full((8,), 7.0, device=DEV)
    grad = torch.empty(dec.lat_dim, device=DEV)
    if period:
        rc = lib.nphm_fit_identity_step_quirk(eng.handle, x.data_ptr(), x.shape[0], period, lat.data_ptr(), None, None,
                                              ctypes.byref(fp), 0, terms.data_ptr(), grad.data_ptr(), None, _stream())
    else:
        rc = lib.nphm_fit_identity_step(eng.handle, x.data_ptr(), x.shape[0], lat.data_ptr(), None, None, ctypes.byref(fp), 0,
                                        terms.data_ptr(), grad.data_ptr(), None, _stream())
    return rc, terms, grad, lat


@pytest.mark.parametrize('name', E.FIT_CONFIGS)
def test_identity_step(name):
    """nphm_fit_identity_step with all five lambdas and no update (the FFMA step off the tensor-core configuration): loss
    terms and the latent gradient per block, also at the zero latent the fitters start from (identical symmetric pairs)."""
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    n = 500
    for seed, z in ((0, E.latent(name, seed=20, device=DEV)), (1, torch.zeros(dec.lat_dim, device=DEV))):
        x, x64, kind = _points(P64, z.double(), n, seed=20 + seed)
        for period in ((0, 100) if _tc(name) else (0,)):
            with torch.no_grad():
                s64 = E.sdf(P64, x64, z.double(), period)
            clamp = _clamp_away(s64, 0.1)
            t64, g64 = E.identity_step(P64, x64, z.double(), LAMBDAS, clamp, period)
            t32, g32 = E.identity_step(P32, x, z, LAMBDAS, clamp, period)
            rc, terms, grad, lat = _identity_call(eng, dec, x, z, LAMBDAS, clamp, period)
            _run(rc, 'nphm_fit_identity_step')
            assert torch.equal(lat, z)                          # apply_update = 0 leaves the latent alone
            what = 'identity_step %s p%d' % ('zero' if seed else 'code', period)
            assert int(terms[5]) == int(t64[5]), (what, float(terms[5]), float(t64[5]))
            for i, term in enumerate(('surface', 'reg_global', 'reg_loc', 'reg_unobserved', 'symm_dist')):
                chk('%s %s' % (what, term), terms[i], t64[i], t32[i], kind='scalar')
            chk(what + ' grad', grad, g64, g32, kind='scalar', parts=_latent_parts(P64), floor=FLOOR_GRAD, part_floor=FLOOR_BLOCK)
    chk.done()


# ------------------------------------------------------------------------------------------------ scan-batched
def _pad(points):
    from nphm_b200.models.fitting import _pad_scans
    return _pad_scans(points)


@pytest.mark.parametrize('S,ns', [(1, (127,)), (3, (1, 129, 300)), (5, (127, 129, 1, 300, 129))])
def test_batched_against_float64(S, ns):
    """nphm_fit_surface_grad_batched(_quirk) and nphm_fit_identity_step_batched with padding, masks, one scan with nothing
    kept and per-scan quirk periods: each scan against float64 on its own rows."""
    from nphm_b200 import _native
    name = 'prod'
    dec, eng, P64, P32 = _setup(name)
    chk = _check('prod S=%d' % S)
    lib = _lib()
    zs = [E.latent(name, seed=30 + k, device=DEV) for k in range(S)]
    pts = [_points(P64, zs[k].double(), ns[k], seed=30 + k) for k in range(S)]
    x, pad_mask = _pad([p[0] for p in pts])
    n = x.shape[1]
    masks = []
    for k in range(S):
        m = torch.rand(n, generator=torch.Generator().manual_seed(k)).to(DEV) < 0.85
        m[0] = True
        if pad_mask is not None:
            m &= pad_mask[k].bool()
        masks.append(m)
    if S > 2:
        masks[1][:] = False                                     # one scan with nothing kept
    mask = torch.stack(masks).to(torch.uint8).contiguous()
    lat = torch.stack(zs).contiguous()
    ws = torch.zeros(lib.nphm_fit_batch_workspace_bytes(eng.handle, S, n), dtype=torch.uint8, device=DEV)
    periods = [0] * S if S == 1 else [0] + [max(1, ns[k] // (1 + k % 2)) for k in range(1, S)]
    per_dev = torch.tensor(periods, dtype=torch.int32, device=DEV)
    terms = torch.full((S, 8), 7.0, device=DEV)
    g_lat = torch.empty(S, dec.lat_dim, device=DEV)
    g_pts = torch.empty(S, n, 3, device=DEV)
    with torch.no_grad():
        every = torch.cat([E.sdf(P64, pts[k][1], zs[k].double(), p) for k in range(S) for p in {0, periods[k]}])
    clamp = _clamp_away(every, 0.1)
    _run(lib.nphm_fit_surface_grad_batched_quirk(eng.handle, x.data_ptr(), mask.data_ptr(), S, n, per_dev.data_ptr(),
                                                 lat.data_ptr(), clamp, terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), _stream()), 'nphm_fit_surface_grad_batched_quirk')
    fp = _native.FitParams(*[float(v) for v in LAMBDAS], clamp, 0.01, 1)
    t_id = torch.full((S, 8), 7.0, device=DEV)
    g_id = torch.empty(S, dec.lat_dim, device=DEV)
    lat_id = lat.clone()
    _run(lib.nphm_fit_identity_step_batched(eng.handle, x.data_ptr(), mask.data_ptr(), S, n, lat_id.data_ptr(), None, None,
                                            ctypes.byref(fp), 0, t_id.data_ptr(), g_id.data_ptr(), ws.data_ptr(), ws.numel(),
                                            _stream()), 'nphm_fit_identity_step_batched')
    for k in range(S):
        nk, m = ns[k], masks[k][:ns[k]]
        xk, x64, kind = pts[k]
        what = 'batched scan %d n%d p%d' % (k, nk, periods[k])
        l64, k64, gz64, gx64 = E.fit_surface(P64, x64, zs[k].double(), m, clamp, periods[k])
        l32, k32, gz32, gx32 = E.fit_surface(P32, xk, zs[k], m, clamp, periods[k])
        assert int(terms[k, 5]) == k64, (what, float(terms[k, 5]), k64)
        if k64 == 0:
            assert bool(torch.isnan(terms[k, 0])) and bool((g_lat[k] == 0).all()) and bool((g_pts[k] == 0).all()), what
        else:
            chk(what + ' loss', terms[k, 0], l64, l32, kind='scalar')
            chk(what + ' latent', g_lat[k], gz64, gz32, kind='scalar', parts=_latent_parts(P64), floor=FLOOR_GRAD,
                part_floor=FLOOR_BLOCK)
            chk(what + ' xyz', g_pts[k, :nk], gx64, gx32, parts=_row_parts(P64, x64, zs[k].double(), kind, periods[k]),
                floor=FLOOR_GRAD)
            assert bool((g_pts[k, nk:] == 0).all()), what        # padding rows get no gradient
        # the identity step with the scan's mask (training mode)
        zz = zs[k].double().clone().requires_grad_()
        with torch.no_grad():
            s64 = E.sdf(P64, x64, zs[k].double())
        keep = m & (s64.abs() < clamp)
        z32 = zs[k].clone().requires_grad_()
        refs = []
        for P, zl, xx in ((P64, zz, x64), (P32, z32, xk)):
            s = E.sdf(P, xx, zl)
            regs = E.regularisers(P, zl)
            tot = sum(lm * r for lm, r in zip(LAMBDAS[1:], regs))
            if bool(keep.any()):
                tot = tot + LAMBDAS[0] * s.abs()[keep].mean()
            refs.append(torch.autograd.grad(tot, [zl])[0])
        assert int(t_id[k, 5]) == int(keep.sum()), (what, float(t_id[k, 5]), int(keep.sum()))
        chk(what + ' identity grad', g_id[k], refs[0], refs[1], kind='scalar', parts=_latent_parts(P64), floor=FLOOR_GRAD,
            part_floor=FLOOR_BLOCK)
    chk.done()


# ------------------------------------------------------------------------------------------------ Adam
def _ulps(got, ref, *operands):
    """Largest |got - ref| in fp32 ulps of the largest operand of the update at each element.  An update that cancels against
    the old value has a result far smaller than its operands, and its rounding error is that of the operands."""
    scale = torch.stack([t.abs().float() for t in operands] + [ref.abs()]).max(dim=0).values
    ulp = torch.ldexp(torch.ones_like(scale), torch.frexp(scale)[1] - 24).double()
    return float(((got.double() - ref.double()).abs() / ulp).max())


def _adam_ulps(got, want, p, g, m, v):
    """(param, exp_avg, exp_avg_sq) of the device against torch: the worst ulp difference of the three."""
    return max(_ulps(got[0], want[0], p, want[0] - p), _ulps(got[1], want[1], m, 0.1 * (g - m)),
               _ulps(got[2], want[2], 0.999 * v, 0.001 * g * g))


ADAM_TORCH_ULPS = 4         # against torch: FMA contraction of the moment and parameter updates, torch's division by a scalar


def _adam_fp32(p, g, m, v, lr, step, dense):
    """The kernels' Adam update in fp32, in their own order (adam_dense_kernel, fit_finalize_kernel): every operation rounded
    once to fp32, the three contracted ones as FMAs (the product exact in float64, one rounding of the sum), division and
    sqrt correctly rounded, the denominator sqrt(v) / sqrt(bc2) + eps.  dense: the constants of adam_dense_kernel (fp32
    literals), else those of fit_finalize_kernel (fp32 casts of 1 - beta).  Returns (param, exp_avg, exp_avg_sq)."""
    f = lambda x: x.float().double()
    one = lambda c: float(torch.tensor(c, dtype=F32))
    b1c, b2, b2c = (one(0.1), one(0.999), one(0.001)) if dense else (one(1.0 - 0.9), one(0.999), one(1.0 - 0.999))
    bc1, bc2 = 1.0 - 0.9 ** step, 1.0 - 0.999 ** step
    step_size, bc2_sqrt, eps = one(one(lr) / bc1), one(bc2 ** 0.5), one(1e-8)
    p, g, m, v = (t.double() for t in (p, g, m, v))
    v2 = f(g * f(b2c * g) + f(v * b2))                  # fma(g, (1 - beta2) g, beta2 v)
    m2 = f(f(g - m) * b1c + m)                           # fma(g - m, 1 - beta1, m)
    den = f(f(f(v2.sqrt()) / bc2_sqrt) + eps)
    p2 = f(p - f(m2 / den) * step_size)                  # fma(-(m / denom), step_size, p)
    return p2.float(), m2.float(), v2.float()


def _adam_exact(got, want, what, bad):
    """The device's (param, exp_avg, exp_avg_sq) against the fp32 emulation: equal, but for at most 1 ulp on at most one
    element in 10 000 (a float64 sum of an emulated FMA that lands on an fp32 midpoint rounds twice).  Returns the number of
    elements that differ."""
    n_diff = 0
    for name, a, b in zip(('param', 'exp_avg', 'exp_avg_sq'), got, want):
        d = a != b
        n_diff += int(d.sum())
        if bool(d.any()):
            u = _ulps(a[d], b[d])
            if u > 1 or int(d.sum()) > max(1, a.numel() // 10000):
                bad.append('%s %s: %d of %d elements differ from the fp32 emulation, up to %.2f ulp'
                           % (what, name, int(d.sum()), a.numel(), u))
    return n_diff


def _torch_adam(p, g, m, v, lr, step):
    """torch.optim.Adam(foreach=False) from the fp32 state (p, m, v) after step - 1 steps: one step with the gradient g."""
    param = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([param], lr=lr, foreach=False)
    opt.state[param] = {'step': torch.tensor(float(step - 1)), 'exp_avg': m.clone(), 'exp_avg_sq': v.clone()}
    param.grad = g.clone()
    opt.step()
    st = opt.state[param]
    return param.detach(), st['exp_avg'], st['exp_avg_sq']


def _adam_state(n, seed, gscale, zero=False):
    """(param, grad, exp_avg, exp_avg_sq) on the device; zero: the fitters' start, param and moments 0 (the update is the
    whole result)."""
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen)
    m = torch.randn(n, generator=gen) * 0.01
    v = torch.rand(n, generator=gen) * 1e-4
    g = torch.randn(n, generator=gen) * gscale
    if zero:
        p, m, v = p * 0, m * 0, v * 0
    return [t.to(DEV) for t in (p, m, v, g)]


@pytest.mark.parametrize('step', [1, 2, 10, 1000])
def test_adam_step(step):
    """nphm_adam_step and the fitting update (nphm_fit_apply_gradient, single scan and 3 scans, applying its own gradient)
    against an fp32 emulation in the kernels' order (bit for bit, see _adam_exact) and against torch.optim.Adam(foreach=False)
    on the same fp32 state (within ADAM_TORCH_ULPS of the update's operands); gradients from 0 and 1e-30 to 1e3, from a random
    state and from the fitters' zero start."""
    from nphm_b200 import _native
    lib = _lib()
    worst, n_diff, bad = 0.0, 0, []
    for zero in (False, True):
        for gscale in (0.0, 1e-30, 1e-8, 1e-3, 1.0, 1e3):
            p, m, v, g = _adam_state(1344, step, gscale, zero)
            if step == 1:
                m.zero_()
                v.zero_()
            want = _torch_adam(p, g, m, v, 0.01, step)
            pp, mm, vv = p.clone(), m.clone(), v.clone()
            _run(lib.nphm_adam_step(pp.data_ptr(), g.data_ptr(), mm.data_ptr(), vv.data_ptr(), pp.numel(), 0.01, step,
                                    _stream()), 'nphm_adam_step')
            what = 'nphm_adam_step %s gradient scale %g' % ('zero start' if zero else 'random state', gscale)
            n_diff += _adam_exact((pp, mm, vv), _adam_fp32(p, g, m, v, 0.01, step, True), what, bad)
            u = _adam_ulps((pp, mm, vv), want, p, g, m, v)
            worst = max(worst, u)
            if u > ADAM_TORCH_ULPS:
                bad.append('%s: %.2f ulp from torch' % (what, u))
    # the fitting update: surface gradient g (lambda_surface 1, no regulariser), single scan and 3 scans
    dec, eng, P64, P32 = _setup('prod')
    for S in (1, 3):
        for zero in (False, True):
            states = [_adam_state(dec.lat_dim, 10 * step + k, 1e-2, zero) for k in range(S)]
            if step == 1:
                for st in states:
                    st[1].zero_()
                    st[2].zero_()
            lat, m, v, g = (torch.stack([st[i] for st in states]).contiguous() for i in range(4))
            stats = torch.tensor([[10.0, 1.0]] * S, device=DEV)
            fp = _native.FitParams(1.0, 0.0, 0.0, 0.0, 0.0, 0.1, 0.01, step)
            terms = torch.empty(S, 8, device=DEV)
            gout = torch.empty(S, dec.lat_dim, device=DEV)
            if S == 1:
                rc = lib.nphm_fit_apply_gradient(eng.handle, lat.data_ptr(), m.data_ptr(), v.data_ptr(), ctypes.byref(fp),
                                                 g.data_ptr(), stats.data_ptr(), None, 1, terms.data_ptr(), gout.data_ptr(),
                                                 _stream())
            else:
                rc = lib.nphm_fit_apply_gradient_batched(eng.handle, S, lat.data_ptr(), m.data_ptr(), v.data_ptr(),
                                                         ctypes.byref(fp), g.data_ptr(), stats.data_ptr(), None, 1,
                                                         terms.data_ptr(), gout.data_ptr(), _stream())
            _run(rc, 'nphm_fit_apply_gradient')
            assert torch.equal(gout, g)
            for k in range(S):
                p0, m0, v0 = states[k][0], states[k][1], states[k][2]
                what = 'nphm_fit_apply_gradient S=%d scan %d %s' % (S, k, 'zero start' if zero else 'random state')
                n_diff += _adam_exact((lat[k], m[k], v[k]), _adam_fp32(p0, g[k], m0, v0, 0.01, step, False), what, bad)
                u = _adam_ulps((lat[k], m[k], v[k]), _torch_adam(p0, g[k], m0, v0, 0.01, step), p0, g[k], m0, v0)
                worst = max(worst, u)
                if u > ADAM_TORCH_ULPS:
                    bad.append('%s: %.2f ulp from torch' % (what, u))
    print('ENSEMBLE adam step %d: %d elements differ from the fp32 emulation; worst difference from torch.optim.Adam %.2f ulp'
          % (step, n_diff, worst))
    assert not bad, bad


def test_anchor_gradient_through_mlp_pos():
    """grad_anchors of nphm_fit_apply_gradient through the mlp_pos backward (ReLU masks) against float64, per block."""
    from nphm_b200 import _native
    lib = _lib()
    dec, eng, P64, P32 = _setup('prod')
    chk = _check('prod')
    for seed in range(3):
        z = E.latent('prod', seed=40 + seed, device=DEV)
        up = torch.randn(P64.n_loc, 3, generator=torch.Generator().manual_seed(seed)).to(DEV) * 10 ** (-seed)
        zero = torch.zeros(dec.lat_dim, device=DEV)
        stats = torch.tensor([1.0, 0.0], device=DEV)
        fp = _native.FitParams(1.0, 0.0, 0.0, 0.0, 0.0, 0.1, 0.0, 1)
        m, v = torch.zeros_like(z), torch.zeros_like(z)
        gout = torch.empty_like(z)
        terms = torch.empty(8, device=DEV)
        _run(lib.nphm_fit_apply_gradient(eng.handle, z.data_ptr(), m.data_ptr(), v.data_ptr(), ctypes.byref(fp), zero.data_ptr(),
                                         stats.data_ptr(), up.contiguous().data_ptr(), 0, terms.data_ptr(), gout.data_ptr(),
                                         _stream()), 'nphm_fit_apply_gradient')
        g64 = E.anchor_vjp(P64, z.double(), up.double())
        g32 = E.anchor_vjp(P32, z, up)
        chk('grad_anchors %d' % seed, gout, g64, g32, kind='scalar', parts=[('z_glob', slice(0, P64.G)),
                                                                              ('local', slice(P64.G, None))],
            floor=FLOOR_GRAD)
    chk.done()


# ------------------------------------------------------------------------------------------------ stage 1
@pytest.mark.parametrize('name', ['prod', 'api', 'depth3', 'tc-nosymm', 'tc-allpairs', 'tc-2m'])
def test_stage1_member_passes(name):
    """nphm_ensemble_sdfgrad_forward / _backward: s_k, grad_local s_k, and the double backward's weight and bias gradients
    per weight set, the condition and the point gradients."""
    dec, eng, P64, P32 = _setup(name)
    chk = _check(name)
    B, N = 2, 129
    gen = torch.Generator().manual_seed(3)
    xl = ((torch.rand(P64.M, B, N, 3, generator=gen) - 0.5) * 0.6).to(DEV)
    cond = (0.1 * torch.randn(P64.M, B, P64.G + P64.L, generator=gen)).to(DEV)
    sbar = (torch.randn(P64.M, B, N, generator=gen) * 1e-4).to(DEV)
    gbar = (torch.randn(P64.M, B, N, 3, generator=gen) * 1e-4).to(DEV)
    s, g, ws = eng.sdfgrad_forward(xl, cond)
    s64, g64 = E.sdfgrad(P64, xl.double(), cond.double())
    s32, g32 = E.sdfgrad(P32, xl, cond)
    members = [('member %d' % m, m) for m in range(P64.M)]
    chk('sdfgrad s', s, s64, s32, kind='scalar', parts=members)
    chk('sdfgrad grad_local', g, g64, g32, kind='scalar', parts=members, floor=FLOOR_GRAD)
    shapes = [tuple(W.shape) for W, _ in P64.layers]
    gw, gb, gc, gx = eng.sdfgrad_backward(ws, sbar, gbar, shapes)
    w64, b64, c64, x64 = E.sdfgrad_vjp(P64, xl.double(), cond.double(), sbar.double(), gbar.double())
    w32, b32, c32, x32 = E.sdfgrad_vjp(P32, xl, cond, sbar, gbar)
    chk('sdfgrad cond', gc, c64, c32, kind='scalar', parts=members, floor=FLOOR_GRAD)
    chk('sdfgrad xyz', gx, x64, x32, kind='scalar', parts=members, floor=FLOOR_GRAD)
    sets = [('set %d' % k, k) for k in range(P64.M - P64.n_symm)]
    for l in range(len(shapes)):
        chk('sdfgrad lin%d.weight' % l, gw[l], w64[l], w32[l], kind='scalar', parts=sets, floor=FLOOR_GRAD)
        chk('sdfgrad lin%d.bias' % l, gb[l], b64[l], b32[l], kind='scalar', parts=sets, floor=FLOOR_GRAD)
    chk.done()


# ------------------------------------------------------------------------------------------------ which ensembles the fitters take
PREDICATE = ['prod', 'tc-64m', 'tc-65m', 'tc-2m', 'tc-64m-nosymm', 'api', 'fit', 'symm0', 'h77', 'ffma-widest', 'ffma-over', 'depth3', 'depth6']


def _kernels_during(f):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc = f()
        torch.cuda.synchronize()
    return rc, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize('name', PREDICATE)
def test_fused_fit_predicate_matches_the_kernels(name):
    """For every shape and mode: fused_fit_config (what the fitters send to the fused kernels) is True exactly when the C entry
    points accept the call - the identity step, and the point-gradient call of the joint fitter and the stage-1 loss - and
    a rejected call launches nothing."""
    from nphm_b200 import _native
    from nphm_b200.models.fitting import fused_fit_config
    lib = _lib()
    dec = E.make_decoder(name, DEV)
    eng = dec.engine()
    P64 = E.Params(dec, F64)
    z = E.latent(name, device=DEV)
    x, _, _ = _points(P64, z.double(), 130)
    n = x.shape[0]
    ws = torch.zeros(lib.nphm_fit_batch_workspace_bytes(eng.handle, 1, n), dtype=torch.uint8, device=DEV)
    lat, terms, g_lat, g_pts = z.clone(), torch.empty(8, device=DEV), torch.empty_like(z), torch.empty(n, 3, device=DEV)
    fp = _native.FitParams(*[float(v) for v in LAMBDAS], 0.1, 0.01, 1)
    for training in (True, False):
        dec.train(training)
        period = 0 if training else n

        def identity():
            if period:
                return lib.nphm_fit_identity_step_quirk(eng.handle, x.data_ptr(), n, period, lat.data_ptr(), None, None,
                                                        ctypes.byref(fp), 0, terms.data_ptr(), g_lat.data_ptr(), ws.data_ptr(),
                                                        _stream())
            return lib.nphm_fit_identity_step(eng.handle, x.data_ptr(), n, lat.data_ptr(), None, None, ctypes.byref(fp), 0,
                                              terms.data_ptr(), g_lat.data_ptr(), ws.data_ptr(), _stream())

        def surface():
            if period:
                return lib.nphm_fit_surface_grad_quirk(eng.handle, x.data_ptr(), n, period, lat.data_ptr(), None, 0.1,
                                                       terms.data_ptr(), g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(),
                                                       _stream())
            return lib.nphm_fit_surface_grad(eng.handle, x.data_ptr(), n, lat.data_ptr(), None, 0.1, terms.data_ptr(),
                                             g_lat.data_ptr(), g_pts.data_ptr(), ws.data_ptr(), _stream())

        for grad_points, call in ((False, identity), (True, surface)):
            rc, kernels = _kernels_during(call)
            want = fused_fit_config(dec, grad_points)
            print('ENSEMBLE %-16s training %d grad_points %d: python %d, C rc %d, %d device activities'
                  % (name, training, grad_points, want, rc, len(kernels)))
            assert (rc == 0) == want, (name, training, grad_points, rc, lib.nphm_last_error())
            if rc:
                assert not kernels, (name, training, grad_points, kernels)
