"""The native posed query (get_logits_posed through posed_evaluator: nphm_mlp_inverse_jacobian, the compacting Broyden search
nphm_mlp_broyden_search_compact and the identity query at the roots) against the float64 reference of
tests/posed_f64_common.py, at every row.

test_gpu_posed.py compares the posed SDF with posed.npz and with the composite path, both from other Broyden runs: they can ask
for 5e-5 on the SDF and must let 3 % of the valid flags differ.  Here the search engine and the identity engine are wrapped on
their instances, so each call's condition rows, roots x^, residual norms and valid flags, and the points the identity decoder
was queried at (the eval-mode quirk rows' second search and query included), are handed to the reference:

1. the condition rows against float64 (the compressor row of 'compress' goes through the native anchors);
2. valid == (diff < 1e-6) bit for bit; for a valid row diff against |x^ + F(x^) - p| in float64, and that float64 residual
   below 1e-6 up to the same slack; a row reported unconverged is unconverged at the point it returns;
3. the identity decoder was queried at exactly x^, and the returned SDF is that query's (the quirk rows: the second one's);
4. the SDF against the float64 identity decoder at x^ with the call's quirk rows, converged rows or not;
5. end to end, for valid rows: x^ polished to the root x* in float64, |sdf - s64(x*)| within check 4's bound plus
   |grad s64(x*)| ||(I + dF/dx)^-1(x*)||_2 (1e-6 + slack), what the 1e-6 stopping rule allows;
6. posed_evaluator takes every case, so none falls back to the composite path.

The criterion of checks 1, 2 and 4 is that of tests/f64_check.py, err_native <= K * err_fp32 + FLOOR * max|ref64|, with the
same operation in fp32 PyTorch (TF32 off) as the yardstick, on the whole call and again on its parts: each expression, the quirk
rows, the first and last 128-row tile of each piece, and the invalid rows.  The matrix: the seeded ensemble in training and in
eval mode with four deformation networks (compress as seeded, compress with its output layer x 80, expr_only and glob_only,
whose searches run on the FFMA kernel at hidden 512), and the NPM pair; one expression, and three (one of them zero, one x 3);
a 20^3 grid with a ragged last chunk at the default piece size and with pieces that end on quirk rows and cut expressions
mid-tile, and 1, 127 and 129 points in and around the head's box.  `-s` prints the worst ratio and the floor each check needs,
per case, and the invalid and quirk rows of every call.
"""
import time

import numpy as np
import pytest
import torch

import posed_f64_common as P
from conftest import MAXI, MINI, make_ensemble, sample_latent
from f64_check import Check
from posed_common import npm_case
from nphm_b200.models import reconstruction as R
from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, extract_posed_meshes_narrowband, mesh_from_logits

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32, F64 = torch.float32, torch.float64

# Measured on an H100 80GB HBM3 (700 W power limit) over every case below, worst err_native / err_fp32 and the smallest floor
# each check needs beyond K * err_fp32: condition rows 1.0 (the compressor row; the other modes copy the codes exactly), floor 0;
# residual norms 12.4, floor 0; the ensemble's SDF 41 (a 129-row call), floor 0; the NPM SDF 813 (the 1024-wide layer chain
# against fp32 torch), floor 5.0e-5 of max|ref|; end to end at most 0.33 of the allowed error.  The whole file runs in 26 s.
# Inherent, not a defect: with the x 80 field |F| reaches ~10, so the fp32 residual itself is only resolved to ~1.6e-6, above
# the 1e-6 threshold; rows reported valid there have float64 residuals up to 4.3e-6, as a plain fp32 search would, and the
# slack of check 2 (K x the fp32 error of the row's tile) grows to match.  The seeded unscaled networks converge at every row,
# with the x 3 code too: only the x 80 field has invalid rows (845 of 8000 grid rows at S = 1, 3608 of 24000 at S = 3).
K = 64.0
FLOOR = 2e-5                    # the identity ensemble's values (test_gpu_ensemble_f64.py)
FLOOR_NPM = 1e-4                # the NPM DeepSDF stacks (test_gpu_joint_f64.py)
FLOOR_RES = 1e-8                # the residual norm, relative to max|p| (measured need: 0)
GRID_RES, GRID_NBATCH = 20, 3000                   # 8000 points: chunks of 3000, 3000 and 2000 rows
PIECE_ROWS = 3000               # pieces of 3000 // S points: they end on the quirk rows 2999 and 5999, and at S = 3 the 1000
                                # points of an expression end mid-tile
ROW_SETS = [(1, 1), (127, 100), (129, 100)]        # (points, nbatch_points)
DECODERS = ['%s-%s' % (m, d) for m in ('train', 'eval') for d in P.DEFORMATIONS] + ['npm']


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------ decoders, codes, points
class _Setup:
    """The decoders of a case (fp32 on the device), the codes, and the reference's parameters in float64 and float32."""

    def __init__(self, decoder, S):
        if decoder == 'npm':
            self.dec, self.dfn, lat, z_ex, _, _ = npm_case(DEV)
            z = z_ex[0]
            self.search_engine, self.shape_engine = self.dfn.engine(), self.dec.engine()
        else:
            mode, name = decoder.split('-', 1)
            self.dec = make_ensemble(0, device=DEV).train(mode == 'train')
            self.dfn = P.make_deformation(name, DEV)
            lat = sample_latent(1).to(DEV)
            torch.manual_seed(8)
            z = (torch.randn(200) * 0.1).to(DEV)
            self.search_engine, self.shape_engine = self.dfn.defDeepSDF.engine(), self.dec.engine()
        self.lat = lat.reshape(1, 1, -1).float()
        self.codes = torch.stack([z, 0 * z, 3 * z])[:S].float().contiguous()    # a zero code and one x 3
        self.Q64, self.Q32 = P.Params(self.dec, self.dfn, F64), P.Params(self.dec, self.dfn, F32)
        self.quirky = self.Q64.nphm and not self.dec.training
        self.floor = FLOOR if self.Q64.nphm else FLOOR_NPM


def _grid():
    return torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, GRID_RES)).to(DEV, F32)[None]


def _rows(n, seed):
    """n points in the head's box grown by half on every side: some lie outside it."""
    g = torch.Generator().manual_seed(600 + seed)
    lo, hi = torch.tensor(MINI), torch.tensor(MAXI)
    return ((lo + hi) / 2 + (torch.rand(n, 3, generator=g) * 2 - 1) * (hi - lo) / 2 * 1.5)[None].to(DEV)


# ------------------------------------------------------------------------------------------------ capture
class _Capture:
    """Wraps the cached search and identity engines on their instances.  ``pieces``: one dict per piece of posed_evaluator,
    with the points J0 was taken at, the search's arguments and results, and the identity query's points, flags and output."""

    def __init__(self, search_engine, shape_engine):
        self.engines = (search_engine, shape_engine)
        self.pieces = []
        ij, search, identity = search_engine.inverse_jacobian, search_engine.broyden_search, shape_engine.query

        def inverse_jacobian(xyz, cond):
            self.pieces.append({'j0_at': xyz.clone(), 'j0_cond': cond.clone()})
            return ij(xyz, cond)

        def broyden_search(obs, cond, x_init, j_inv, **kw):
            out = search(obs, cond, x_init, j_inv, **kw)
            self.pieces[-1].update(obs=obs.clone(), cond=cond.clone(), x0=x_init.clone(), x=out[0].clone(),
                                   diff=out[1].clone(), valid=out[2].clone())
            return out

        def query(xyz, lat, *a, **kw):
            out = identity(xyz, lat, *a, **kw)
            sdf = out[0] if isinstance(out, tuple) else out
            self.pieces[-1].update(at=xyz.clone(), lat=lat.clone(), quirk=bool(kw.get('eval_quirk', False)),
                                   period=kw.get('quirk_period'), sdf=sdf.reshape(xyz.shape[0], -1).clone())
            return out

        search_engine.inverse_jacobian, search_engine.broyden_search = inverse_jacobian, broyden_search
        shape_engine.query = query

    def release(self):
        se, sh = self.engines
        del se.inverse_jacobian, se.broyden_search, sh.query


def _posed(setup, pts, nbatch):
    """get_logits_posed with the engines captured: (sdf S x N, valid S x N on the device, pieces of the first pass, pieces of
    the quirk pass)."""
    cap = _Capture(setup.search_engine, setup.shape_engine)
    try:
        sdf, valid = R.get_logits_posed(setup.dec, setup.dfn, setup.lat, setup.codes, pts, nbatch_points=nbatch,
                                        return_valid=True)
    finally:
        cap.release()
    main = [c for c in cap.pieces if not c['quirk']]
    again = [c for c in cap.pieces if c['quirk']]
    return torch.from_numpy(sdf).to(DEV), torch.from_numpy(valid).to(DEV), main, again


# ------------------------------------------------------------------------------------------------ the checks
def _cat(pieces, key):
    return torch.cat([c[key] for c in pieces], dim=1)


def _piece_masks(pieces, S, N):
    """(name, mask S x N) of the first and last 128-row tile of each piece (rows q * n + k of a piece of n points)."""
    out, a = [], 0
    for k, c in enumerate(pieces):
        n = c['x'].shape[1]
        for name, r in (('first', torch.arange(min(128, S * n))), ('last', torch.arange((S * n - 1) // 128 * 128, S * n))):
            m = torch.zeros(S, N, dtype=torch.bool)
            m[r // n, a + r % n] = True
            out.append(('piece %d %s tile' % (k, name), m.to(DEV)))
        a += n
    return out


def _tile_max(t):
    """Every row of t (S x N) replaced by the maximum of its 128-row tile (rows s N + i)."""
    flat = t.reshape(-1)
    M = flat.numel()
    pad = torch.cat([flat, flat.new_zeros((-M) % 128)]).reshape(-1, 128)
    return pad.max(dim=1, keepdim=True).values.expand(-1, 128).reshape(-1)[:M].reshape(t.shape)


def _parts(masks, sel):
    """(name, index into the rows ``sel`` selects) of every part with rows there."""
    out = []
    for name, m in masks:
        idx = m.reshape(-1)[sel.reshape(-1)].nonzero().reshape(-1)
        if idx.numel():
            out.append((name, idx))
    return out


def _check_call(chk, tag, setup, pts, nbatch, stats):
    """Checks 1-5 on one get_logits_posed call; returns the per-row violations."""
    S, N = setup.codes.shape[0], pts.shape[1]
    Q64, Q32 = setup.Q64, setup.Q32
    sdf, valid, main, again = _posed(setup, pts, nbatch)
    bad = []
    p = pts.expand(S, N, 3)

    # ---- what each piece was asked and answered
    assert sum(c['x'].shape[1] for c in main) == N
    x, diff, ok = _cat(main, 'x'), _cat(main, 'diff'), _cat(main, 'valid')
    cond = main[0]['cond']
    for c in main + again:
        assert torch.equal(c['cond'], cond) and torch.equal(c['j0_cond'], cond)
        assert torch.equal(c['j0_at'], c['obs']) and torch.equal(c['x0'], c['obs'])      # J0 and the search start at p
    assert torch.equal(_cat(main, 'obs'), p)
    assert torch.equal(ok, valid)
    # check 3: the identity decoder was queried at the roots, and its output is the returned SDF
    assert torch.equal(_cat(main, 'at'), x)
    for c in main + again:
        assert torch.equal(c['lat'], setup.lat.reshape(1, -1).expand(S, -1))
    quirk = P.quirk_mask(N, nbatch).to(DEV) if setup.quirky else torch.zeros(N, dtype=torch.bool, device=DEV)
    rows = quirk.nonzero().reshape(-1)
    assert torch.equal(sdf[:, ~quirk], _cat(main, 'sdf')[:, ~quirk])
    if setup.quirky:
        assert all(c['period'] is None for c in main) and all(c['period'] == 1 for c in again)
        # the quirk rows' own search finds the same roots (rows are independent), and their query is the returned SDF
        assert torch.equal(_cat(again, 'obs'), p[:, rows])
        assert torch.equal(_cat(again, 'x'), x[:, rows]) and torch.equal(_cat(again, 'valid'), ok[:, rows])
        assert torch.equal(_cat(again, 'diff'), diff[:, rows])
        assert torch.equal(_cat(again, 'at'), x[:, rows]) and torch.equal(_cat(again, 'sdf'), sdf[:, rows])
    else:
        assert not again

    masks = [('expression %d' % s, torch.arange(S, device=DEV)[:, None].expand(S, N) == s) for s in range(S)]
    if setup.quirky:
        masks.append(('quirk', quirk[None].expand(S, N)))
    masks += _piece_masks(main, S, N)
    masks.append(('invalid', ~ok))
    everything = torch.ones(S, N, dtype=torch.bool, device=DEV)

    # ---- check 1: the condition rows
    z64, z32 = setup.lat.reshape(-1).double(), setup.lat.reshape(-1)
    c64, c32 = P.condition(Q64, z64, setup.codes.double()), P.condition(Q32, z32, setup.codes)
    chk('%s cond' % tag, cond, c64, c32, kind='cond')

    # ---- check 2: valid flags and the residual at the roots
    assert torch.equal(ok, diff < P.CVG)
    x64, p64 = x.double(), p.double()
    with torch.no_grad():
        r64 = P.residual(Q64, x64, c64, p64).norm(dim=-1)
        r32 = P.residual(Q32, x, c32, p).norm(dim=-1)
    pmax = float(p.abs().max())
    # what fp32 arithmetic allows a row: K x the fp32 error of its 128-row tile (one row's own fp32 error may be 0 by chance)
    e32 = torch.nan_to_num((r32.double() - r64).abs(), nan=0.0)
    slack = K * _tile_max(e32) + FLOOR_RES * pmax
    # relative to max|p| as a whole; the per-row bounds below hold every part to the same slack
    chk('%s residual' % tag, diff[ok], r64[ok], r32[ok], kind='scalar', scale=pmax, floor=FLOOR_RES)
    over = ok & ((diff.double() - r64).abs() > slack)
    bad += ['%s: valid row (%d, %d): diff %.3e, float64 residual %.3e, slack %.2e' % (tag, s, i, diff[s, i], r64[s, i], slack[s, i])
            for s, i in over.nonzero().tolist()[:5]]
    over = ok & (r64 > P.CVG + slack)
    bad += ['%s: valid row (%d, %d) unconverged in float64: residual %.3e' % (tag, s, i, r64[s, i])
            for s, i in over.nonzero().tolist()[:5]]
    finite = torch.isfinite(x).all(-1) & torch.isfinite(r64)
    under = ~ok & finite & (r64 < P.CVG - slack)
    bad += ['%s: invalid row (%d, %d) converged in float64: residual %.3e' % (tag, s, i, r64[s, i])
            for s, i in under.nonzero().tolist()[:5]]

    # ---- check 4: the SDF at the roots (converged or not), with the call's quirk rows
    q = quirk.cpu() if setup.quirky else None
    s64 = torch.stack([P.identity_sdf(Q64, x64[s], z64, q) for s in range(S)]).detach()
    s32 = torch.stack([P.identity_sdf(Q32, x[s], z32, q) for s in range(S)]).detach()
    fin = finite & torch.isfinite(s64)
    chk('%s sdf' % tag, sdf[fin], s64[fin], s32[fin], parts=_parts(masks, fin))
    bound4 = K * float((s32[fin].double() - s64[fin]).abs().max()) + setup.floor * float(s64[fin].abs().max())

    # ---- check 5: end to end, against the posed SDF at the polished root
    worst5 = 0.0
    idx = ok.nonzero()
    if idx.numel():
        sel_s, sel_i = idx[:, 0], idx[:, 1]
        xs, res = P.polish(Q64, x64[sel_s, sel_i], c64[sel_s], p64[sel_s, sel_i])
        assert float(res.max()) < P.POLISH_TOL, float(res.max())
        grad = torch.empty_like(xs)
        star = torch.empty(xs.shape[0], dtype=F64, device=DEV)
        for s in range(S):
            m = sel_s == s
            if bool(m.any()):
                sq = None if q is None else q[sel_i[m].cpu()]
                star[m], grad[m] = P.identity_sdf_grad(Q64, xs[m], z64, sq)
        jinv = P.inverse_jacobian(Q64, xs[:, None], c64[sel_s])[:, 0]
        lip = grad.norm(dim=-1) * torch.linalg.matrix_norm(jinv, ord=2)
        allowed = bound4 + lip * (P.CVG + slack[sel_s, sel_i])
        err = (sdf[sel_s, sel_i].double() - star).abs()
        worst5 = float((err / allowed).max())
        for j in (err > allowed).nonzero().reshape(-1).tolist()[:5]:
            bad.append('%s: row (%d, %d): |sdf - s64(x*)| %.3e > %.3e (|grad s| ||J^-1|| %.3e)'
                       % (tag, sel_s[j], sel_i[j], err[j], allowed[j], lip[j]))

    n_inv = int((~ok).sum())
    stats.append((tag, n_inv, int((~finite).sum()), int(quirk.sum()) * S, len(main), worst5))
    print('POSED %-20s %-10s rows %6d invalid %5d non-finite %d quirk %d pieces %d  end-to-end worst err / allowed %.3f'
          % (chk.tag, tag, S * N, n_inv, int((~finite).sum()), int(quirk.sum()) * S, len(main), worst5))
    return bad


@pytest.mark.parametrize('S', [1, 3])
@pytest.mark.parametrize('decoder', DECODERS)
def test_posed_against_float64(cuda_device, decoder, S, monkeypatch):
    t0 = time.time()
    setup = _Setup(decoder, S)
    # check 6: the native path takes the case
    assert R.posed_evaluator(setup.dec, setup.dfn, setup.lat, setup.codes) is not None
    chk = Check('%s S%d' % (decoder, S), K, setup.floor, prefix='POSED')
    stats, bad = [], []
    grid = _grid()
    bad += _check_call(chk, 'grid', setup, grid, GRID_NBATCH, stats)
    with monkeypatch.context() as m:
        m.setattr(R, 'POSED_PIECE_ROWS', PIECE_ROWS)
        bad += _check_call(chk, 'grid/piece', setup, grid, GRID_NBATCH, stats)
    for n, nb in ROW_SETS:
        bad += _check_call(chk, 'rows%d' % n, setup, _rows(n, n), nb, stats)
    print('POSED %-20s %.1f s' % (chk.tag, time.time() - t0))
    # the matrix reaches what it is for: several pieces, quirk rows in eval mode, rows that fail to converge under x 80
    assert stats[1][4] > 1
    if setup.quirky:
        assert all(st[3] > 0 for st in stats)
    if decoder.endswith('x80'):
        assert stats[0][1] > 0
    assert not bad, '\n'.join(bad[:40])
    chk.done()


# ------------------------------------------------------------------------------------------------ posed band, new modes
@pytest.mark.parametrize('name', ['expr_only', 'glob_only'])
def test_posed_band_meshes_equal_dense_modes(cuda_device, name):
    """extract_posed_meshes_narrowband with an expr_only / glob_only deformation network gives the dense posed mesh."""
    from test_gpu_posed import _assert_same_mesh, _margin_for
    res, nbatch = 40, 7000
    dec = make_ensemble(0, device=DEV).eval()
    dfn = P.make_deformation(name, DEV)
    lat = sample_latent(1).to(DEV)
    torch.manual_seed(8)
    z_ex = torch.randn(2, 200, device=DEV) * 0.1
    margin = _margin_for(dec, dfn, lat, z_ex, res, nbatch, MINI, MAXI)
    meshes = extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, MINI, MAXI, res, nbatch_points=nbatch, margin=margin)
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(DEV, F32)[None]
    dense = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=nbatch)
    assert len(meshes) == 2
    for s in range(2):
        ref = mesh_from_logits(dense[s], MINI, MAXI, res)
        assert len(ref.faces) > 0 and np.isfinite(dense[s]).all()
        _assert_same_mesh(meshes[s], ref)
