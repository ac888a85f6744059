"""Grid queries of the dense ensemble kernel against float64 on every tile layout the kernel picks (DESIGN 4.1).

tc_ensemble_launch tiles a grid query [first, first + count) in one of three layouts: 8 x 4 x 4 blocks ('cube': the pruned
kernel always, dense ranges of whole 8-plane groups), 1 x 16 x 8 blocks ('plane': other dense x-plane ranges) or 128
consecutive points ('linear': where blocks would add more than 3 % tiles).  tile_point maps each tile row to a grid index and
marks it valid only inside the grid and inside the range; that mapping places the output, the eval-mode quirk rows, the
zero-weight member masks and the fp32-absorption certificate.  CASES reaches every layout at aligned, ragged (the grid edge
cuts the last block row), partial-plane and sharded ranges (the x-slabs distributed.slab_planes issues, ghost planes
included), each with quirk period 0 and with periods that put quirk rows in most tiles.  Every case checks:

  * float64: the output against the float64 SDF with the quirk rows by grid index (tests/f64_check.py, the K and FLOOR of
    tests/test_gpu_ensemble_f64.py), and as parts the range's first and last x-plane and the points of the ragged last block
    row; the pruned kernel against its bound n_members * tau * max_k |s_k| at two thresholds;
  * xyz: with period 0 the grid output equals, bit for bit, an xyz query of the same points in flat order (linear tiles, no
    absorption; both skips are exact);
  * absorption: NPHM_ENS_ABSORB=1 and =0 give the same bits;
  * tile count: the kernel's (nphm_debug_ens_tile_masks) equals that of tools/zero_member_tiles.py tile_layout / tile_points;
  * masks: every member whose blend weight is non-zero at a valid point of a tile is in the tile's mask, and no member is in
    it that only a padding row could have put there (for the pruned kernel: its rule w_k >= tau (sum_k w_k + 1e-6));
  * writes: the query writes all of its range of an out= view into a sentinel-filled buffer and nothing outside it.

test_benchmark_configuration runs the query of bench.py (its head and latent, the whole 256^3 grid in 8 x 4 x 4 blocks,
quirk period CHUNK, out= preallocated) against float64 on every 16th x-plane and the last.

`-s` prints per case the layout, the tile counts, the err_native / err_fp32 ratios and the mask counts.  About 45 s on an
H100 80GB HBM3 (700 W power limit), most of it the float64 and fp32 references of the 256^3 x-slabs.
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))

import ensemble_f64_common as E  # noqa: E402
from f64_check import Check  # noqa: E402
from test_gpu_ensemble_f64 import FLOOR, K  # noqa: E402
from zero_member_tiles import tile_layout, tile_points  # noqa: E402

pytestmark = pytest.mark.gpu
F32, F64 = torch.float32, torch.float64
CHUNK = 25000                       # bench.py's nbatch_points: the quirk period of the benchmark
PERIODS = (0, 129, CHUNK)           # 129: a quirk row in almost every tile of every layout
TAUS = (1e-8, 1e-4)                 # thresholds of the pruned kernel
SENTINEL = 0x7FC0DEAD               # a NaN the kernel never writes
# blend weights in the fp32 underflow band, where the device's expf and torch's may round differently to +0 or a denormal:
# float64 weights above W_SURE are non-zero in fp32, those below W_ZERO are +0
W_SURE, W_ZERO = 2.0 ** -140, 2.0 ** -160
LAYOUTS = {(8, 4, 4): 'cube', (1, 16, 8): 'plane', None: 'linear'}


# ------------------------------------------------------------------------------------------------ the layout matrix
def _planes(res, p0, n):
    return p0 * res * res, n * res * res


def _sharded():
    from nphm_b200.distributed import plan_slabs, slab_planes
    out = []
    for res, world in ((128, 2), (128, 3), (128, 8), (256, 8)):
        for rank, (c0, c1) in enumerate(plan_slabs(res, world)):
            p0, n, _ = slab_planes(c0, c1)
            out.append(('shard-%d-w%d-r%d' % (res, world, rank), 'plane', res, *_planes(res, p0, n), 'tc'))
    return out


# (id, layout the kernel must pick, res, first, count, impl)
CASES = [
    ('cube-64-whole', 'cube', 64, 0, 64 ** 3, 'tc'),
    ('cube-64-x0-8', 'cube', 64, *_planes(64, 0, 8), 'tc'),
    ('cube-64-x24-40', 'cube', 64, *_planes(64, 24, 16), 'tc'),        # starts inside the grid
    ('cube-64-x20-36', 'cube', 64, *_planes(64, 20, 16), 'tc'),        # px0 off a multiple of 8
    ('cube-134-x0-8', 'cube', 134, *_planes(134, 0, 8), 'tc'),         # 134 = 33 * 4 + 2: ragged y and z
    ('cube-134-x4-12', 'cube', 134, *_planes(134, 4, 8), 'tc'),        # ragged, px0 off a multiple of 8
    ('cube-258-x64-72', 'cube', 258, *_planes(258, 64, 8), 'tc'),
    ('plane-64-partial-5-45', 'plane', 64, 5 * 64 ** 2 + 7, 40 * 64 ** 2, 'tc'),   # starts and ends inside x-planes
    ('plane-128-x27-40', 'plane', 128, *_planes(128, 27, 13), 'tc'),
    ('plane-264-x130-133', 'plane', 264, *_planes(264, 130, 3), 'tc'),  # 264 = 16 * 16 + 8: ragged y, 102.998 % tiles
    ('linear-66-whole', 'linear', 66, 0, 66 ** 3, 'tc'),
    ('linear-64-unaligned', 'linear', 64, 12345, 50001, 'tc'),
] + _sharded() + [
    ('pruned-37-whole', 'cube', 37, 0, 37 ** 3, 'tc_pruned'),           # ragged x, y and z
    ('pruned-66-whole', 'cube', 66, 0, 66 ** 3, 'tc_pruned'),
    ('pruned-64-x20-33', 'cube', 64, *_planes(64, 20, 13), 'tc_pruned'),
]


def mirror_tiles(res, first, count, impl):
    """(layout name, kind, block) of tools/zero_member_tiles.py for the kernel of impl: the pruned kernel always takes cubes."""
    kind, block = tile_layout(res, first, count, '8x4x4' if impl == 'tc_pruned' else 'auto')
    return LAYOUTS[block], kind, block


def ragged_rows(res, first, count, g, block):
    """Rows (grid indices g) in the last block row of a blocked layout over [first, first + count) where the grid's or the
    range's edge cuts it short."""
    rr = res * res
    if block is None:
        return torch.zeros_like(g, dtype=torch.bool)
    tbx, tby, tbz = block
    ix, iy, iz = g // rr, (g // res) % res, g % res
    r = torch.zeros_like(g, dtype=torch.bool)
    if res % tby:
        r |= iy >= res - res % tby
    if res % tbz:
        r |= iz >= res - res % tbz
    px0 = first // rr
    n_px = (first + count - 1) // rr - px0 + 1
    if n_px % tbx:
        r |= ix >= px0 + n_px - n_px % tbx
    return r


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _debug_tile_masks(eng):
    from test_gpu_ensemble_absorb_replay import debug_array
    return debug_array(eng, 'nphm_debug_ens_tile_masks', np.uint64)


def _axes(res, dev):
    from conftest import MAXI, MINI
    return [torch.from_numpy(np.linspace(MINI[a], MAXI[a], res).astype(np.float32)).to(dev) for a in range(3)]


def _xyz(ax, res, g):
    return torch.stack([ax[0][g // (res * res)], ax[1][(g // res) % res], ax[2][g % res]], dim=-1)


def _quirk(g, period, total):
    """Rows the eval-mode query overwrites, by grid index (tests/ensemble_f64_common.py query_quirk_rows)."""
    if not period:
        return torch.zeros_like(g, dtype=torch.bool)
    return (g % period == period - 1) | (g == total - 1)


def grid_query(eng, z, res, first, count, period, impl='tc', absorb=True, out=None):
    from conftest import MAXI, MINI
    old = os.environ.get('NPHM_ENS_ABSORB')
    os.environ['NPHM_ENS_ABSORB'] = '1' if absorb else '0'
    try:
        out, anc = eng.query_grid(z, MINI, MAXI, res, first, count, period, impl=impl, out=out)
        torch.cuda.synchronize()
    finally:
        if old is None:
            del os.environ['NPHM_ENS_ABSORB']
        else:
            os.environ['NPHM_ENS_ABSORB'] = old
    return out, anc


class Refs:
    """float64 and fp32 references per x-plane of a res^3 grid, for one head and code: the blended SDF, its value at a quirk
    row (every s_k = 1: the sum of the normalised weights) and max_k |s_k| (float64).  sub_max: also, per x-plane, the float64
    max |s_m| of every member over the plane's points in each 32 x 32 (y, z) block of the kernel's 32^3-point sub-boxes."""

    def __init__(self, dec, z, sub_max=False):
        self.P64, self.P32 = E.Params(dec, F64), E.Params(dec, F32)
        self.z = z.reshape(-1).float()
        self.cache = {}
        self.sub_max = sub_max
        self.sub_cache = {}

    def _compute(self, res, planes):
        ax = _axes(res, self.z.device)
        rr = res * res
        g = torch.cat([torch.arange(p * rr, (p + 1) * rr, device=self.z.device) for p in planes])
        cols = [[] for _ in range(5)]
        s_abs = []
        with torch.no_grad():
            for c0 in range(0, g.shape[0], 1 << 17):
                x = _xyz(ax, res, g[c0:c0 + (1 << 17)])
                for P, xx, zz, c in ((self.P64, x.double(), self.z.double(), 0), (self.P32, x, self.z, 2)):
                    anc = E.anchors(P, zz)
                    s = E.members(P, xx, zz, anc)
                    w = E.blend_weights(P, xx, anc)
                    cols[c].append((w * s).sum(dim=1))
                    cols[c + 1].append(w.sum(dim=1))
                    if P is self.P64:
                        cols[4].append(s.abs().max(dim=1).values)
                        if self.sub_max:
                            s_abs.append(s.abs())
        cols = [torch.cat(c) for c in cols]
        for i, p in enumerate(planes):
            self.cache[(res, p)] = [c[i * rr:(i + 1) * rr] for c in cols]
        if self.sub_max:
            n_sub, M = (res + 31) // 32, self.P64.M
            s = torch.cat(s_abs).reshape(len(planes), res, res, M)
            s = torch.nn.functional.pad(s, (0, 0, 0, 32 * n_sub - res, 0, 32 * n_sub - res))     # |s| >= 0: pad with 0
            s = s.reshape(len(planes), n_sub, 32, n_sub, 32, M).amax(dim=(2, 4))
            for i, p in enumerate(planes):
                self.sub_cache[(res, p)] = s[i]

    def sub_boxes(self, res, planes):
        """{sx: n_sub x n_sub x M float64 max |s_m| over the points of ``planes`` in the sub-boxes (sx, sy, sz)}."""
        todo = [p for p in planes if (res, p) not in self.sub_cache]
        for i in range(0, len(todo), max(1, (1 << 20) // (res * res))):
            self._compute(res, todo[i:i + max(1, (1 << 20) // (res * res))])
        out = {}
        for p in planes:
            out[p >> 5] = torch.maximum(out[p >> 5], self.sub_cache[(res, p)]) if (p >> 5) in out else self.sub_cache[(res, p)]
        return out

    def rows(self, res, first, count, planes):
        """(output rows, grid indices, [sdf64, quirk64, sdf32, quirk32, smax64]) over the range's points in ``planes``."""
        rr = res * res
        todo = [p for p in planes if (res, p) not in self.cache]
        for i in range(0, len(todo), max(1, (1 << 20) // rr)):
            self._compute(res, todo[i:i + max(1, (1 << 20) // rr)])
        gs, vals = [], [[] for _ in range(5)]
        for p in planes:
            lo, hi = max(first, p * rr), min(first + count, (p + 1) * rr)
            gs.append(torch.arange(lo, hi, device=self.z.device))
            for i, c in enumerate(self.cache[(res, p)]):
                vals[i].append(c[lo - p * rr:hi - p * rr])
        g = torch.cat(gs)
        return g - first, g, [torch.cat(v) for v in vals]


def check_f64(chk, what, got, g, ref, res, first, count, block, period, bad, tau=None, M=None):
    """got (rows of g) against float64 with the quirk rows of ``period`` by grid index; parts: the first and last x-plane,
    the ragged block row, the quirk rows.  tau: the pruned kernel's bound instead of the criterion."""
    sdf64, q64, sdf32, q32, smax = ref
    rr = res * res
    q = _quirk(g, period, res ** 3)
    r64, r32 = torch.where(q, q64, sdf64), torch.where(q, q32, sdf32)
    if tau is not None:
        smax = torch.where(q, torch.ones_like(smax), smax)
        bound = M * tau * smax + K * (r32.double() - r64).abs() + FLOOR * float(r64.abs().max())
        err = (got.double() - r64).abs()
        n = int((err > bound).sum())
        print('LAYOUT %-22s %s: max err %.3e, max err / bound %.3f' % (chk.tag, what, float(err.max()),
                                                                      float((err / bound).max())))
        if n:
            bad.append('%s: %d points beyond n_members * tau * max_k |s_k|' % (what, n))
        return
    px = g // rr
    parts = [('first x-plane', px == int(px.min())), ('last x-plane', px == int(px.max())),
             ('ragged block row', ragged_rows(res, first, count, g, block)), ('quirk', q)]
    chk(what, got, r64, r32, parts=[(nm, m.nonzero().reshape(-1)) for nm, m in parts if bool(m.any())])


def emulated_weights(anc, X, k, n_members):
    """(fp32 weight as blend_weight computes it, float64 weight) of member k at the points X (..., 3)."""
    if k == n_members - 1:
        w = torch.exp(torch.full(X.shape[:-1], -0.2, dtype=F32, device=X.device) / torch.tensor(0.01, device=X.device))
        return w, torch.full(X.shape[:-1], float(np.exp(-20.0)), dtype=F64, device=X.device)
    d = anc[k][None, None].float() - X
    inner = (d[..., 0].double() ** 2 + (d[..., 1] * d[..., 1]).double()).float()       # fma(dx, dx, dy * dy)
    d2 = (d[..., 2].double() ** 2 + inner.double()).float()                             # fma(dz, dz, .)
    nrm = torch.sqrt(d2) + np.float32(10e-6)
    w32 = torch.exp(-(nrm * nrm) / torch.tensor(0.01, device=X.device))
    n64 = d.double().norm(dim=-1) + 10e-6
    return w32, torch.exp(-(n64 * n64) / 0.01)


def check_masks(masks, anc, res, first, count, kind, block, M, bad, what, tau=None):
    """The tile masks against the dense rule (w_k != 0 at a valid point) or, with tau, the pruned rule (w_k >= tau (S + 1e-6)
    at a valid point, S = sum_k w_k in member order), on tile_points' rows.  Returns the number of (tile, member) pairs in a
    mask beyond the rule evaluated in fp32 at the valid points."""
    ix, iy, iz, valid = tile_points(res, first, count, kind, block)
    dev = anc.device
    ax = _axes(res, dev)
    X = torch.stack([ax[0][torch.from_numpy(ix).to(dev)], ax[1][torch.from_numpy(iy).to(dev)],
                     ax[2][torch.from_numpy(iz).to(dev)]], dim=-1)
    V = torch.from_numpy(valid).to(dev)
    mk = torch.from_numpy(((masks[:, None] >> np.arange(M, dtype=np.uint64)[None]) & np.uint64(1)).astype(bool)).to(dev)
    if not bool(mk[:, M - 1].all()):
        bad.append('%s: a tile mask without the global member' % what)
    W = [emulated_weights(anc, X, k, M) for k in range(M)] if tau is not None else None
    if tau is not None:
        S = torch.zeros_like(W[0][0])
        for k in range(M):
            S = S + W[k][0]
        thr = tau * (S + np.float32(1e-6))
    n_missing = n_extra = n_beyond = 0
    for k in range(M - 1):
        w32, w64 = W[k] if W is not None else emulated_weights(anc, X, k, M)
        if tau is None:
            rule, sure, possible = w32 != 0, w64 >= W_SURE, w64 >= W_ZERO
        else:
            rule, sure, possible = w32 >= thr, w32 >= thr * (1 + 1e-4), w32 >= thr * (1 - 1e-4)
        rule, sure, possible = ((c & V).any(dim=1) for c in (rule, sure, possible))
        n_missing += int((sure & ~mk[:, k]).sum())
        n_extra += int((mk[:, k] & ~possible).sum())
        n_beyond += int((mk[:, k] & ~rule).sum())
    if n_missing:
        bad.append('%s: %d (tile, member) pairs with a non-zero weight at a valid point missing from the mask'
                   % (what, n_missing))
    if n_extra:
        bad.append('%s: %d (tile, member) pairs in the mask that no valid point of the tile needs' % (what, n_extra))
    return int(mk[:, :M - 1].sum()), n_beyond


def check_writes(buf, pad, count, what, bad):
    """buf: the sentinel buffer, the range at [pad, pad + count)."""
    bits = buf.view(torch.int32)
    outside = int((bits[:pad] != SENTINEL).sum()) + int((bits[pad + count:] != SENTINEL).sum())
    unwritten = int((bits[pad:pad + count] == SENTINEL).sum())
    nonfinite = int((~torch.isfinite(buf[pad:pad + count])).sum())
    if outside or unwritten or nonfinite:
        bad.append('%s: %d writes outside the range, %d points of the range unwritten, %d non-finite'
                   % (what, outside, unwritten, nonfinite))


def sentinel_out(count, res, dev):
    pad = 2 * res * res + 256
    buf = torch.full((count + 2 * pad,), SENTINEL, dtype=torch.int32, device=dev).view(F32)
    return buf, pad, buf[pad:pad + count]


# ------------------------------------------------------------------------------------------------ the matrix on the GPU
_state = {}


def make_head(name, dev):
    """The decoder of a configuration of tests/ensemble_f64_common.py; '<name>:shift': with its anchors moved 0.13 in x, so
    that a mirrored member's boxes are not those of its unmirrored partner reflected."""
    base, _, variant = name.partition(':')
    dec = E.make_decoder(base, dev)
    if variant == 'shift':
        with torch.no_grad():
            dec.anchors = dec.anchors + torch.tensor([0.13, 0.0, 0.0], device=dec.anchors.device)
    else:
        assert not variant, name
    return dec


def _head(dev, name='prod', sub_max=False):
    """(decoder, engine, code, Refs) of one head at a time on the device (latent seed 5 of the configuration)."""
    if _state.get('name') != name:
        _state.clear()
        torch.cuda.empty_cache()
        dec = make_head(name, dev)
        z = E.latent(name.partition(':')[0], seed=5, device=dev)
        _state.update(name=name, dec=dec, eng=dec.engine(), z=z, refs=Refs(dec, z, sub_max))
    return _state['dec'], _state['eng'], _state['z'], _state['refs']


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_layout_against_float64(cuda_device, case):
    label, layout, res, first, count, impl = case
    dev = cuda_device
    dec, eng, z, refs = _head(dev)
    M = refs.P64.M
    name, kind, block = mirror_tiles(res, first, count, impl)
    assert name == layout, (label, name, layout)
    n_mirror = tile_points(res, first, count, kind, block)[0].shape[0]
    rows, g, ref = refs.rows(res, first, count, range(first // (res * res), (first + count - 1) // (res * res) + 1))
    chk = Check(label, K, FLOOR, prefix='LAYOUT')
    bad = []
    pruned = impl == 'tc_pruned'
    print('LAYOUT %-22s %d^3 points [%d, +%d) %s %s' % (label, res, first, count, impl,
                                                       name if block is None else '%s %dx%dx%d' % ((name,) + block)))
    for tau in (TAUS if pruned else (None,)):
        if pruned:
            eng.set_prune_threshold(tau)
        try:
            for period in PERIODS:
                what = '%s%s p%d' % (impl, ' tau %g' % tau if pruned else '', period)
                buf, pad, out = sentinel_out(count, res, dev)
                _, anc = grid_query(eng, z, res, first, count, period, impl=impl, out=out)
                masks = _debug_tile_masks(eng)
                if masks.size != n_mirror:
                    bad.append('%s: the kernel ran %d tiles, tools/zero_member_tiles.py counts %d' % (what, masks.size, n_mirror))
                elif period == 0:
                    n_in, n_beyond = check_masks(masks, anc, res, first, count, kind, block, M, bad, what, tau)
                    print('LAYOUT %-22s %s: tiles kernel %d, mirror %d; %d (tile, member) pairs in the masks, %d beyond '
                          'the rule at the valid points' % (label, what, masks.size, n_mirror, n_in, n_beyond))
                check_writes(buf, pad, count, what, bad)
                if not pruned:
                    off, _ = grid_query(eng, z, res, first, count, period, absorb=False)
                    n = int((off.view(torch.int32) != out.view(torch.int32)).sum())
                    if n:
                        bad.append('%s: %d outputs differ between NPHM_ENS_ABSORB=1 and =0' % (what, n))
                if period == 0 and not pruned:
                    xyz = _xyz(_axes(res, dev), res, torch.arange(first, first + count, device=dev))
                    flat = eng.query(xyz[None], z[None], eval_quirk=False, impl='tc')[0].reshape(-1)
                    n = int((flat.view(torch.int32) != out.view(torch.int32)).sum())
                    if n:
                        bad.append('%s: %d outputs differ from the xyz query of the same points' % (what, n))
                check_f64(chk, what, out[rows], g, ref, res, first, count, block, period, bad, tau=tau, M=M)
        finally:
            if pruned:
                eng.set_prune_threshold(0.0)
    for b in bad:
        print('LAYOUT %-22s FAIL %s' % (label, b))
    chk.bad += bad
    chk.done()


# ------------------------------------------------------------------------------------------------ bench.py's query
def test_benchmark_configuration(cuda_device):
    """The query bench.py times: make_ensemble(0) in eval mode, sample_latent(1), the whole 256^3 grid, quirk period CHUNK,
    out= preallocated; against float64 on x-planes 0, 16, ..., 240 and 255, each plane a part.  On an H100 80GB HBM3 (700 W
    power limit) the query took 301 ms (CUDA events) and the references of the 17 planes 1.6 s."""
    from conftest import MAXI, MINI, make_ensemble, sample_latent
    dev = cuda_device
    res, total = 256, 256 ** 3
    dec = make_ensemble(0, device=dev).eval()
    eng = dec.engine()
    lat = sample_latent(1).to(dev)
    volume = torch.empty(total, device=dev, dtype=F32)
    eng.query_grid(lat, MINI, MAXI, res, 0, total, quirk_period=CHUNK, out=volume)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    eng.query_grid(lat, MINI, MAXI, res, 0, total, quirk_period=CHUNK, out=volume)
    ev[1].record()
    torch.cuda.synchronize()
    masks = _debug_tile_masks(eng)
    name, kind, block = mirror_tiles(res, 0, total, 'tc')
    n_mirror = tile_points(res, 0, total, kind, block)[0].shape[0]
    assert name == 'cube' and masks.size == n_mirror, (name, masks.size, n_mirror)
    planes = list(range(0, res, 16)) + [res - 1]
    t0 = time.perf_counter()
    refs = Refs(dec, lat)
    rows, g, ref = refs.rows(res, 0, total, planes)
    torch.cuda.synchronize()
    t_ref = time.perf_counter() - t0
    sdf64, q64, sdf32, q32, _ = ref
    q = _quirk(g, CHUNK, total)
    r64, r32 = torch.where(q, q64, sdf64), torch.where(q, q32, sdf32)
    chk = Check('bench 256^3', K, FLOOR, prefix='LAYOUT')
    px = g // (res * res)
    parts = [('x-plane %d' % p, (px == p).nonzero().reshape(-1)) for p in planes] + [('quirk', q.nonzero().reshape(-1))]
    chk('tc p%d' % CHUNK, volume[rows], r64, r32, parts=parts)
    print('LAYOUT bench 256^3: query %.1f ms (CUDA events, %s), %d tiles (kernel and mirror); float64 and fp32 references '
          'of %d x-planes (%d points) %.1f s' % (ev[0].elapsed_time(ev[1]), torch.cuda.get_device_name(dev), masks.size,
                                                 len(planes), g.numel(), t_ref))
    chk.done()
