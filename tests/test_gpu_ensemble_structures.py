"""Grid queries of the dense ensemble kernel against float64 on every member structure the tensor-core kernel takes.

tc_ensemble_supported takes any ensemble of hidden width 200, 4 layers and lat_dim_glob + lat_dim_loc = 96 with at most 64
members, whatever its mirrored pairs and latent split.  STRUCTURES runs the configurations of tests/ensemble_f64_common.py
that reach the edges of that set: 2 members, one mirrored pair alone, no mirrored pair, every local member paired, the
global member at mask bit 32 and at bit 63 (64 members with and without pairs), two other latent splits, and one head with
its anchors moved in x (the mirrored members' sub-boxes then differ from their partners' reflected).  On each, in eval
mode, a subset of the layouts of tests/test_gpu_ensemble_grid_layouts.py (whole-grid cubes, a ragged x-slab, a partial
plane range, a short unaligned range and one rank of an 8-way sharded grid), with quirk periods 0 and 129, checks:

  * float64: the output against the float64 SDF (tests/f64_check.py, the K and FLOOR of tests/test_gpu_ensemble_f64.py),
    with the first and last x-plane, the ragged block row and the quirk rows as parts;
  * member by member: the query ran the member-major path (nphm_debug_ens_pair_counts is not empty) and gives the bits of
    the tile-major kernel (NPHM_ENS_ABSORB=0);
  * listed rows: no member lists more rows than the range has points where its float64 blend weight is above W_ZERO, and
    a member whose weight is below W_ZERO over the whole range lists none;
  * masks and writes: as tests/test_gpu_ensemble_grid_layouts.py, with the structure's member count (bit 63 at 64
    members); sentinel writes stay inside the range;
  * sub-box bounds (nphm_debug_ens_sub_bounds, period 0): each equals tools/absorbed_member_tiles.py member_bound on the
    sub-box's axis limits and the GPU's inputs (its anchors, fold_consts) to 1e-9 relative before the fp32 round-up, and is
    at least the float64 max |s_m| over the sub-box's grid points in the query's x-planes.  The sharded rank starts at x-slab
    1 of the sub-boxes (sub_x0 > 0) and crosses into slab 2.
The pruned kernel runs on the whole 64^3 grid against its bound n_members * tau * max_k |s_k| at both thresholds.  At 64
members without pairs one query crosses the 2^24-row chunk boundary of the member-major state (264^3), bits against the
tile-major kernel.  A negative control scales the bounds by 2^-40: the sub-box check must then fail and absorb on and off
must differ.

`-s` prints per case the worst err_native / err_fp32, the rows listed, and the smallest B / max |s_m| of the sub-boxes.
About 45 s on an H100 80GB HBM3 (700 W power limit).
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))

import absorbed_member_tiles as A  # noqa: E402
import test_gpu_ensemble_absorb_replay as R  # noqa: E402
import test_gpu_ensemble_grid_layouts as GL  # noqa: E402
import test_gpu_ensemble_member_major as MM  # noqa: E402
from f64_check import Check  # noqa: E402
from test_gpu_ensemble_f64 import FLOOR, K  # noqa: E402
from zero_member_tiles import tile_points  # noqa: E402

pytestmark = pytest.mark.gpu
F32, F64 = torch.float32, torch.float64
PERIODS = (0, 129)
STRUCTURES = ['tc-2m', 'tc-3m-pair', 'tc-nosymm', 'tc-allpairs', 'tc-33m', 'tc-64m', 'tc-64m-nosymm', 'tc-split-32-64',
              'tc-split-80-16', 'tc-allpairs:shift']


def _shard(res, world, rank):
    from nphm_b200.distributed import plan_slabs, slab_planes
    p0, n, _ = slab_planes(*plan_slabs(res, world)[rank])
    return p0 * res * res, n * res * res


# (id, layout the kernel must pick, res, first, count)
LAYOUTS = [
    ('cube-64-whole', 'cube', 64, 0, 64 ** 3),
    ('cube-134-x0-8', 'cube', 134, *GL._planes(134, 0, 8)),             # ragged y and z
    ('plane-64-partial-5-45', 'plane', 64, 5 * 64 ** 2 + 7, 40 * 64 ** 2),
    ('linear-64-unaligned', 'linear', 64, 12345, 50001),
    ('shard-128-w8-r3', 'plane', 128, *_shard(128, 8, 3)),             # x-planes 47 .. 64: sub-box x-slabs 1 and 2
]
CASES = [(s, c) for s in STRUCTURES for c in LAYOUTS]


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _head(dev, name):
    dec, eng, z, refs = GL._head(dev, name, sub_max=True)
    dec.eval()
    return dec, eng, z, refs


def sub_bounds(eng, M):
    """The sub-box bounds of the last query: (n_sub x M float32, sub_x0, sub_n); 0 x M when it ran tile-major."""
    L = R.lib()
    f = L.nphm_debug_ens_sub_bounds
    n, x0, sn = ctypes.c_longlong(0), ctypes.c_int(0), ctypes.c_int(0)
    from nphm_b200 import _native
    _native.check(f(eng.handle, None, 0, ctypes.byref(n), ctypes.byref(x0), ctypes.byref(sn)), 'sub bounds')
    buf = np.zeros(n.value, np.float32)
    _native.check(f(eng.handle, buf.ctypes.data_as(ctypes.c_void_p), n.value, ctypes.byref(n), ctypes.byref(x0),
                    ctypes.byref(sn)), 'sub bounds')
    return buf.reshape(-1, M), x0.value, sn.value


def check_sub_bounds(refs, z, anc, B, sub_x0, sub_n, res, first, count, what, bad):
    """The sub-box bounds B (n_sub x M) against member_bound on each sub-box's axis limits and the GPU's inputs, and against
    the float64 max |s_m| over the sub-box's points in the query's x-planes.  Returns the smallest B / max |s_m|."""
    M = refs.P64.M
    px0, px1 = first // (res * res), (first + count - 1) // (res * res)
    if sub_x0 != px0 >> 5 or sub_n != (res + 31) // 32 or B.shape[0] != ((px1 >> 5) - sub_x0 + 1) * sub_n * sub_n:
        bad.append('%s: %d sub-boxes from x-slab %d, %d per axis; the query spans x-planes %d .. %d'
                   % (what, B.shape[0], sub_x0, sub_n, px0, px1))
        return float('nan')
    from conftest import MAXI, MINI
    ax = R.grid_axes(MINI, MAXI, res)
    lim = [[(float(a[32 * c:32 * c + 32].min()), float(a[32 * c:32 * c + 32].max())) for c in range(sub_n)] for a in ax]
    Pc32, Pc64 = R.on_cpu(refs.P32), R.on_cpu(refs.P64)
    zc = z.reshape(-1).float().cpu()
    anc64 = anc.double().cpu().numpy()
    consts = [A.fold_consts(Pc32, zc, m) for m in range(M)]
    smax = refs.sub_boxes(res, range(px0, px1 + 1))
    n_eq = n_below = 0
    worst = float('inf')
    for b in range(B.shape[0]):
        sx, sy, sz = sub_x0 + b // (sub_n * sub_n), (b // sub_n) % sub_n, b % sub_n
        lo = np.array([lim[0][sx][0], lim[1][sy][0], lim[2][sz][0]])
        hi = np.array([lim[0][sx][1], lim[1][sy][1], lim[2][sz][1]])
        sm = smax[sx][sy, sz].cpu().numpy()
        for m in range(M):
            Bc = A.member_bound(Pc64, m, zc, anc64, lo, hi, consts[m])
            Bg = np.float32(B[b, m])
            if not np.isfinite(Bc):
                n_eq += Bg != np.inf
                continue
            below = float(np.nextafter(Bg, np.float32(0)))
            n_eq += not (float(Bg) >= Bc * (1 - 1e-9) and below < Bc * (1 + 1e-9))
            n_below += float(Bg) < sm[m]
            if sm[m] > 0:
                worst = min(worst, float(Bg) / float(sm[m]))
    if n_eq:
        bad.append('%s: %d of %d sub-box bounds differ from member_bound' % (what, n_eq, B.size))
    if n_below:
        bad.append('%s: %d of %d sub-box bounds below the float64 max |s_m| of their sub-box' % (what, n_below, B.size))
    print('STRUCT %-40s %s: %d sub-boxes from x-slab %d, %d differ from member_bound, %d below max |s_m|, min B / max |s_m| '
          '%.3g' % (what, 'sub-box bounds', B.shape[0], sub_x0, n_eq, n_below, worst))
    return worst


def listed_rows(counts, anc, res, first, count, M, what, bad):
    """Rows listed per member (summed over the chunks) against the range's points where its float64 weight is >= W_ZERO."""
    dev = anc.device
    X = GL._xyz(GL._axes(res, dev), res, torch.arange(first, first + count, device=dev))
    listed = counts.sum(axis=0)
    over = []
    for k in range(M):
        _, w64 = GL.emulated_weights(anc, X, k, M)
        n = int((w64 >= GL.W_ZERO).sum())
        if listed[k] > n:
            over.append((k, int(listed[k]), n))
    if over:
        bad.append('%s: members listing more rows than points with a float64 weight >= W_ZERO (member, listed, points): %s'
                   % (what, over[:8]))
    return int(listed.sum())


# ------------------------------------------------------------------------------------------------ the matrix
@pytest.mark.parametrize('name,case', CASES, ids=['%s-%s' % (s, c[0]) for s, c in CASES])
def test_structure_layout(cuda_device, name, case):
    label, layout, res, first, count = case
    dev = cuda_device
    dec, eng, z, refs = _head(dev, name)
    M = refs.P64.M
    lname, kind, block = GL.mirror_tiles(res, first, count, 'tc')
    assert lname == layout, (label, lname, layout)
    n_mirror = tile_points(res, first, count, kind, block)[0].shape[0]
    rows, g, ref = refs.rows(res, first, count, range(first // (res * res), (first + count - 1) // (res * res) + 1))
    tag = '%s %s' % (name, label)
    chk = Check(tag, K, FLOOR, prefix='STRUCT')
    bad = []
    for period in PERIODS:
        what = '%s p%d' % (tag, period)
        buf, pad, out = GL.sentinel_out(count, res, dev)
        _, anc = GL.grid_query(eng, z, res, first, count, period, out=out)
        masks = GL._debug_tile_masks(eng)
        counts = MM.pair_counts(eng, M)
        B, sub_x0, sub_n = sub_bounds(eng, M)
        if counts.shape[0] == 0 or B.shape[0] == 0:
            bad.append('%s: the query did not run member by member (%d pair-count chunks, %d sub-boxes)'
                       % (what, counts.shape[0], B.shape[0]))
        else:
            n_listed = listed_rows(counts, anc, res, first, count, M, what, bad)
            print('STRUCT %-40s %d rows listed in %d chunk(s); members listing none: %s'
                  % (what, n_listed, counts.shape[0], np.nonzero(counts.sum(axis=0) == 0)[0].tolist()))
            if period == 0:
                check_sub_bounds(refs, z, anc, B, sub_x0, sub_n, res, first, count, what, bad)
        if masks.size != n_mirror:
            bad.append('%s: the kernel ran %d tiles, tools/zero_member_tiles.py counts %d' % (what, masks.size, n_mirror))
        elif period == 0:
            n_in, n_beyond = GL.check_masks(masks, anc, res, first, count, kind, block, M, bad, what)
            print('STRUCT %-40s tiles %d; %d (tile, member) pairs in the masks, %d beyond the rule; bit %d in %d masks'
                  % (what, masks.size, n_in, n_beyond, M - 1, int(((masks >> np.uint64(M - 1)) & np.uint64(1)).sum())))
        GL.check_writes(buf, pad, count, what, bad)
        off, _ = GL.grid_query(eng, z, res, first, count, period, absorb=False)
        if MM.pair_counts(eng, M).shape[0] != 0:
            bad.append('%s: the query with NPHM_ENS_ABSORB=0 ran member by member' % what)
        n = int((off.view(torch.int32) != out.view(torch.int32)).sum())
        if n:
            bad.append('%s: %d outputs differ between member-major and tile-major' % (what, n))
        GL.check_f64(chk, 'tc p%d' % period, out[rows], g, ref, res, first, count, block, period, bad)
    if label.startswith('shard'):
        assert sub_x0 > 0, 'the sharded rank must start past the first x-slab of the sub-boxes'
    for b in bad:
        print('STRUCT %-40s FAIL %s' % (tag, b))
    chk.bad += bad
    chk.done()


@pytest.mark.parametrize('name', STRUCTURES)
def test_structure_pruned(cuda_device, name):
    """The pruned kernel on the whole 64^3 grid within n_members * tau * max_k |s_k| at both thresholds, with its masks."""
    dev = cuda_device
    dec, eng, z, refs = _head(dev, name)
    M = refs.P64.M
    res, first, count = 64, 0, 64 ** 3
    _, kind, block = GL.mirror_tiles(res, first, count, 'tc_pruned')
    rows, g, ref = refs.rows(res, first, count, range(res))
    chk = Check('%s pruned' % name, K, FLOOR, prefix='STRUCT')
    bad = []
    for tau in GL.TAUS:
        eng.set_prune_threshold(tau)
        try:
            for period in PERIODS:
                what = '%s pruned tau %g p%d' % (name, tau, period)
                out, anc = GL.grid_query(eng, z, res, first, count, period, impl='tc_pruned')
                if period == 0:
                    GL.check_masks(GL._debug_tile_masks(eng), anc, res, first, count, kind, block, M, bad, what, tau)
                GL.check_f64(chk, what, out[rows], g, ref, res, first, count, block, period, bad, tau=tau, M=M)
        finally:
            eng.set_prune_threshold(0.0)
    chk.bad += bad
    chk.done()


def test_chunk_boundary_at_64_members(cuda_device):
    """64 members without pairs across the 2^24-row chunk boundary of the member-major state (264^3: two chunks of
    n_members counters each): bits against the tile-major kernel."""
    dev = cuda_device
    dec, eng, z, refs = _head(dev, 'tc-64m-nosymm')
    M = refs.P64.M
    res = 264
    on, _ = GL.grid_query(eng, z, res, 0, res ** 3, MM.CHUNK)
    counts = MM.pair_counts(eng, M)
    off, _ = GL.grid_query(eng, z, res, 0, res ** 3, MM.CHUNK, absorb=False)
    n = int((on.view(torch.int32) != off.view(torch.int32)).sum())
    print('STRUCT tc-64m-nosymm 264^3: %s chunks x %d members, rows listed per chunk %s, %d outputs differ'
          % (counts.shape[0], counts.shape[1], counts.sum(axis=1).tolist(), n))
    assert counts.shape == (2, M), counts.shape
    assert n == 0, '%d of %d outputs differ between member-major and tile-major' % (n, on.numel())


def test_negative_control_sub_bounds(cuda_device):
    """Bounds scaled by 2^-40: the sub-box check must fail, and absorb on and off must differ."""
    dev = cuda_device
    name = 'tc-allpairs:shift'
    dec, eng, z, refs = _head(dev, name)
    M = refs.P64.M
    res, first, count = 64, 0, 64 ** 3
    L = R.lib()
    L.nphm_debug_ens_bound_scale(eng.handle, 2.0 ** -40)
    try:
        on, anc = GL.grid_query(eng, z, res, first, count, 0)
        B, sub_x0, sub_n = sub_bounds(eng, M)
        off, _ = GL.grid_query(eng, z, res, first, count, 0, absorb=False)
    finally:
        L.nphm_debug_ens_bound_scale(eng.handle, 1.0)
    bad = []
    check_sub_bounds(refs, z, anc, B, sub_x0, sub_n, res, first, count, '%s bounds x 2^-40' % name, bad)
    n = int((on.view(torch.int32) != off.view(torch.int32)).sum())
    print('STRUCT %s bounds x 2^-40: the sub-box check reports %s; %d of %d outputs differ between absorb on and off'
          % (name, bad, n, on.numel()))
    assert any('differ from member_bound' in b for b in bad) and any('below the float64 max' in b for b in bad), bad
    assert n > 0
    again, _ = GL.grid_query(eng, z, res, first, count, 0)
    assert torch.equal(again.view(torch.int32), off.view(torch.int32)), 'the bound scale was not reset'
