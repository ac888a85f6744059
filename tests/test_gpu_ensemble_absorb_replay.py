"""The dense ensemble kernel's fp32-absorption skip (DESIGN 4.1), checked decision by decision against replays of itself.

Each case runs one grid query with the kernel's debug view on (nphm_debug_ens_*: member bounds, pre-pass masks, the members
the producer skipped by vote) and checks:
  * bounds: B_m equals tools/absorbed_member_tiles.py member_bound on the same inputs (the GPU's anchors and fp32 folded
    layer constants, fold_consts) to 1e-9 relative before the round-up to fp32, and B_m >= the float64 max of |s_m| over
    every grid point of the query;
  * structure: skipped ⊆ den-absorbed ⊆ tile mask, the global member is never skipped, and no member is skipped before two
    members of its tile were evaluated;
  * replay: the per-point rule (absorbed_member_tiles.replay) on the state the kernel had (its own skips drive num, the
    published |num| and the lag), with the kernel's tiles, quirk rows, weights and bounds; a (tile, member) on which the
    kernel and the replay disagree must be borderline: its verdict flips within the rounding differences between the
    replay's and the kernel's w, s and num (replay's docstring);
  * on / off: absorb on and off (NPHM_ENS_ABSORB=0) give the same bits, on more heads, latents, ranges and quirk periods;
  * a negative control: bounds scaled by 2^-40 make the on / off comparison fail, so that it can fail.
About 2 GPU-minutes on an H100 (117-123 s), most of it the float64 member outputs of the bound check and the fp32 ones of
the replay.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, 'golden'))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))

import absorbed_member_tiles as A  # noqa: E402
import ensemble_f64_common as E  # noqa: E402
from zero_member_tiles import tile_layout, tile_points  # noqa: E402

CHUNK = 25000                       # bench.py's nbatch_points: the quirk period of the benchmark
S_REL = 2.0 ** -14                  # |s_kernel - s_fp32 reference| <= S_REL max(1, |s|) (the kernel is pinned at 1e-5)


# ------------------------------------------------------------------------------------------------ heads and the debug view
def make_head(name, dev):
    from conftest import make_ensemble
    if name == 'prod':
        return E.make_decoder('prod', dev).eval()
    kind, seed, scale = name.split(':')
    dec = make_ensemble(int(seed), scale=float(scale), device=dev).eval()
    with torch.no_grad():
        if kind == 'shift':          # anchors moved in x: the mirrored members' boxes differ from the unmirrored ones
            dec.anchors = dec.anchors + torch.tensor([0.13, 0.0, 0.0], device=dev)
        elif kind in ('bias+', 'bias-'):      # the output layer's bias moved: num crosses zero in many tiles
            dec.ensembled_deep_sdf.lin4.bias.add_(0.05 if kind == 'bias+' else -0.05)
    return dec


HEADS = ['seed:0:1', 'seed:0:0.25', 'seed:0:4', 'seed:1:0.25', 'seed:1:1', 'seed:1:4', 'seed:2:0.25', 'seed:2:1',
         'seed:2:4', 'prod', 'shift:0:1']
_cache = {}


def head(name, dev):
    if name not in _cache:
        from nphm_b200 import _native
        dec = make_head(name, dev)
        eng = _native.EnsembleEngine(dec)
        eng.refresh(dec)
        _cache.clear()                # one head at a time on the device
        _cache[name] = (dec, eng)
    return _cache[name]


def lib():
    from nphm_b200 import _native
    L = _native.lib()
    for f in ('nphm_debug_ens_tile_masks', 'nphm_debug_ens_absorb_masks', 'nphm_debug_ens_skipped', 'nphm_debug_ens_bounds'):
        getattr(L, f).argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.POINTER(ctypes.c_longlong)]
    L.nphm_debug_ens_sub_bounds.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong,
                                            ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int),
                                            ctypes.POINTER(ctypes.c_int)]
    L.nphm_debug_ens_skip_log.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.nphm_debug_ens_bound_scale.argtypes = [ctypes.c_void_p, ctypes.c_double]
    return L


def debug_array(eng, fn, dtype):
    from nphm_b200 import _native
    f = getattr(lib(), fn)
    n = ctypes.c_longlong(0)
    _native.check(f(eng.handle, None, 0, ctypes.byref(n)), fn)
    buf = np.zeros(n.value, dtype)
    _native.check(f(eng.handle, buf.ctypes.data_as(ctypes.c_void_p), n.value, ctypes.byref(n)), fn)
    return buf


def query(eng, lat, mini, maxi, res, first, count, quirk, absorb=True):
    old = os.environ.get('NPHM_ENS_ABSORB')
    os.environ['NPHM_ENS_ABSORB'] = '1' if absorb else '0'
    try:
        out, anc = eng.query_grid(lat, mini, maxi, res, first, count, quirk, impl='tc')
        torch.cuda.synchronize()
        return out.clone(), anc.clone()
    finally:
        if old is None:
            del os.environ['NPHM_ENS_ABSORB']
        else:
            os.environ['NPHM_ENS_ABSORB'] = old


def bits(mask_u64, M):
    """uint64 masks (T,) -> T x M bool."""
    return ((mask_u64[:, None] >> np.arange(M, dtype=np.uint64)[None, :]) & np.uint64(1)) == 1


# ------------------------------------------------------------------------------------------------ the kernel's inputs, replayed
def grid_axes(mini, maxi, res):
    return [np.linspace(mini[a], maxi[a], res).astype(np.float32) for a in range(3)]


def tile_inputs(P32, z, anc, mini, maxi, res, first, count, quirk, dev):
    """W, S (T x 128 x M, fp32, S = 1 at quirk rows), V, s_err on the kernel's tiles of the query."""
    kind, block = tile_layout(res, first, count, 'auto')
    ix, iy, iz, valid = tile_points(res, first, count, kind, block)
    ax = grid_axes(mini, maxi, res)
    X = torch.from_numpy(np.stack([ax[0][ix], ax[1][iy], ax[2][iz]], axis=-1)).to(dev)        # T x 128 x 3
    T = X.shape[0]
    M = P32.M
    # blend_weight(): fma(dz, dz, fma(dx, dx, dy * dy)), sqrt + 1e-5, -(n * n) / 0.01, expf
    d = anc[None, None].float() - X[:, :, None, :]
    inner = (d[..., 0].double() ** 2 + (d[..., 1] * d[..., 1]).double()).float()
    d2 = (d[..., 2].double() ** 2 + inner.double()).float()
    nrm = torch.sqrt(d2) + np.float32(10e-6)
    W = torch.exp(-(nrm * nrm) / np.float32(0.01))
    gw = torch.exp(torch.tensor(-0.2, dtype=torch.float32, device=dev) / np.float32(0.01))
    W = torch.cat([W, gw.expand(T, 128, 1)], dim=2)
    S = torch.empty(T * 128, M, dtype=torch.float32, device=dev)
    pts = X.reshape(-1, 3)
    with torch.no_grad():
        for c0 in range(0, pts.shape[0], 1 << 18):
            S[c0:c0 + (1 << 18)] = E.members(P32, pts[c0:c0 + (1 << 18)], z, anc)
    S = S.reshape(T, 128, M)
    err = S_REL * S.abs().clamp_min(1.0)
    if quirk:
        g = torch.from_numpy((ix * res + iy) * res + iz).to(dev)
        q = ((g % quirk == quirk - 1) | (g == res ** 3 - 1)) & torch.from_numpy(valid).to(dev)
        S[q] = 1.0
        err[q] = 0.0
    return W, S, torch.from_numpy(valid).to(dev), err, (ix, iy, iz)


def on_cpu(P):
    """A copy of Params P with its tensors on the host (member_bound and fold_consts work in numpy)."""
    q = E.Params.__new__(E.Params)
    q.__dict__.update(P.__dict__)
    q.layers = [(W.cpu(), b.cpu()) for W, b in P.layers]
    q.pos = [(W.cpu(), b.cpu()) for W, b in P.pos]
    q.mean = P.mean.cpu()
    return q


def check_bounds(P32, P64, z, anc, B_gpu, mini, maxi, res, dev, tag):
    """B_gpu against member_bound on the GPU's inputs, and against the float64 max |s_m| over the res^3 grid."""
    ax = grid_axes(mini, maxi, res)
    lo = np.array([a.min() for a in ax], np.float64)
    hi = np.array([a.max() for a in ax], np.float64)
    anc64 = anc.double().cpu().numpy()
    Pc32, Pc64 = on_cpu(P32), on_cpu(P64)
    for m in range(P32.M):
        Bc = A.member_bound(Pc64, m, z.cpu(), anc64, lo, hi, A.fold_consts(Pc32, z.cpu(), m))
        Bg = np.float32(B_gpu[m])
        if not np.isfinite(Bc):
            assert Bg == np.inf, (tag, m)
            continue
        below = float(np.nextafter(Bg, np.float32(0)))
        assert float(Bg) >= Bc * (1 - 1e-9) and below < Bc * (1 + 1e-9), (tag, m, float(Bg), Bc)
    # float64 member outputs over every grid point
    g = torch.stack(torch.meshgrid(*[torch.from_numpy(a.astype(np.float64)) for a in ax], indexing='ij'), -1).reshape(-1, 3)
    Pd, z64, a64 = P64, z.double(), anc.double()
    smax = torch.zeros(P32.M, dtype=torch.float64, device=dev)
    with torch.no_grad():
        for c0 in range(0, g.shape[0], 1 << 17):
            s = E.members(Pd, g[c0:c0 + (1 << 17)].to(dev), z64, a64)
            smax = torch.maximum(smax, s.abs().max(dim=0).values)
    smax = smax.cpu().numpy()
    B64 = B_gpu.astype(np.float64)
    assert np.all(B64 >= smax), (tag, np.nonzero(B64 < smax))
    ratio = float((B64 / smax).min())
    print('  bounds %s: min B/max|s| %.3g, max |s| %.3g' % (tag, ratio, smax.max()))
    return float(smax.max())


def check_decisions(eng, P32, z, anc, mini, maxi, res, first, count, quirk, dev, tag, report=None):
    """Structure of the kernel's decisions and the replay; returns (kernel evaluated, replay-self evaluated, disagreements)."""
    M = P32.M
    masks = debug_array(eng, 'nphm_debug_ens_tile_masks', np.uint64)
    amask = debug_array(eng, 'nphm_debug_ens_absorb_masks', np.uint64)
    skipped = debug_array(eng, 'nphm_debug_ens_skipped', np.uint64)
    B = debug_array(eng, 'nphm_debug_ens_bounds', np.float32)
    assert masks.size == amask.size == skipped.size > 0 and B.size == M
    assert np.all(skipped & ~amask == 0), 'skipped a member outside the den-absorbed mask'
    assert np.all(amask & ~masks == 0), 'den-absorbed mask outside the tile mask'
    assert np.all(skipped >> np.uint64(M - 1) == 0), 'skipped the global member'
    mk, sk, ak = bits(masks, M), bits(skipped, M), bits(amask, M)
    ev = mk & ~sk
    before = np.cumsum(ev, axis=1) - ev                  # members evaluated before each member of the tile
    assert np.all(before[sk] >= 2), 'skipped a member before two of its tile were evaluated'
    W, S, V, err, (ix, iy, iz) = tile_inputs(P32, z, anc, mini, maxi, res, first, count, quirk, dev)
    assert W.shape[0] == masks.size
    Bt = torch.from_numpy(B).to(dev)
    T = lambda a: torch.from_numpy(a).to(dev)               # noqa: E731
    r = A.replay(W, S, V, T(mk), T(ak), Bt, follow=T(sk), s_err=err)
    kern = T(sk)
    assert not bool((kern & ~r['cand']).any()), 'skipped a member that is not a candidate'
    dis = (kern != r['skip'])
    border = ~r['sure_skip'] & ~r['sure_keep']
    bad = dis & ~border
    n_dis = int(dis.sum())
    print('  decisions %s: %d tiles, %d member-tiles evaluated, %d skipped by vote, %d disagreements with the replay '
          '(%d borderline)' % (tag, masks.size, int(ev.sum()), int(sk.sum()), n_dis, int((dis & border).sum())))
    for t, m in torch.nonzero(dis)[:8].tolist():
        print('    tile %d member %d: kernel %s, replay %s, margin %.3g' % (t, m, 'skip' if sk[t, m] else 'keep',
              'skip' if bool(r['skip'][t, m]) else 'keep', float(r['margin'][t, m])))
    assert not bool(bad.any()), ('disagreements outside the borderline set', torch.nonzero(bad)[:8].tolist())
    if report is not None:
        # the replay on its own decisions (the predictor), with and without the quirk rows
        own = A.replay(W, S, V, T(mk), T(ak), Bt)
        report['kernel'] = int(ev.sum())
        report['replay'] = int(mk.sum()) - int(own['skip'].sum())
        _, S0, _, _, _ = tile_inputs(P32, z, anc, mini, maxi, res, first, count, 0, dev)
        own0 = A.replay(W, S0, V, T(mk), T(ak), Bt)
        report['replay_no_quirk'] = int(mk.sum()) - int(own0['skip'].sum())
        diff = torch.nonzero(kern & ~own0['skip']).tolist()
        report['located'] = []
        for t, m in diff[:4]:
            rel = r['margin'][t, m]
            gq = ((ix[t] * res + iy[t]) * res + iz[t])
            quirk_rows = np.nonzero(((gq % quirk == quirk - 1) | (gq == res ** 3 - 1)) & V[t].cpu().numpy())[0] if quirk else []
            report['located'].append((t, m, list(map(int, quirk_rows)), float(rel)))
    return n_dis


GRIDS = [('64^3', None, 64, 0, 64 ** 3, CHUNK), ('128^3', None, 128, 0, 128 ** 3, CHUNK),
         ('wide 64^3', 'wide', 64, 0, 64 ** 3, 0), ('x-slab 128^3', None, 128, 47 * 128 ** 2, 34 * 128 ** 2, CHUNK)]


@pytest.mark.gpu
@pytest.mark.parametrize('name', HEADS)
def test_bounds_and_decisions(cuda_device, name):
    import make_golden_ensemble_zero_skip as Z
    from conftest import MAXI, MINI, sample_latent
    dev = cuda_device
    dec, eng = head(name, dev)
    P32, P64 = E.Params(dec, torch.float32), E.Params(dec, torch.float64)
    L = lib()
    L.nphm_debug_ens_skip_log(eng.handle, 1)
    smax = 0.0
    try:
        for ls in ((1, 2, 3) if name.startswith('seed:0') or name == 'prod' else (1,)):
            z = sample_latent(ls).reshape(-1).to(dev)
            for tag, box, res, first, count, quirk in GRIDS:
                mini, maxi = (Z.WIDE_MIN, Z.WIDE_MAX) if box == 'wide' else (MINI, MAXI)
                _, anc = query(eng, z, mini, maxi, res, first, count, quirk)
                B = debug_array(eng, 'nphm_debug_ens_bounds', np.float32)
                label = '%s latent %d %s' % (name, ls, tag)
                if first == 0 and (res == 64 or ls == 1):
                    smax = max(smax, check_bounds(P32, P64, z, anc, B, mini, maxi, res, dev, label))
                check_decisions(eng, P32, z, anc, mini, maxi, res, first, count, quirk, dev, label)
    finally:
        L.nphm_debug_ens_skip_log(eng.handle, 0)
    if name.endswith(':4'):
        assert smax > 1.0, 'the floor of B at 1 hides the bound check on this head'


@pytest.mark.gpu
def test_locate_the_128_trace_pair(cuda_device):
    """The benchmark head, latent 1, 128^3 with the benchmark's quirk period: the trace build's member-tile count, the
    replay's on its own decisions with and without the quirk rows, and the member-tiles the kernel skips that the replay
    without quirk rows keeps (DESIGN 5)."""
    from conftest import MAXI, MINI, sample_latent
    dev = cuda_device
    dec, eng = head('seed:0:1', dev)
    P32 = E.Params(dec, torch.float32)
    L = lib()
    L.nphm_debug_ens_skip_log(eng.handle, 1)
    try:
        z = sample_latent(1).reshape(-1).to(dev)
        _, anc = query(eng, z, MINI, MAXI, 128, 0, 128 ** 3, CHUNK)
        rep = {}
        check_decisions(eng, P32, z, anc, MINI, MAXI, 128, 0, 128 ** 3, CHUNK, dev, 'trace case', rep)
    finally:
        L.nphm_debug_ens_skip_log(eng.handle, 0)
    print('  128^3 latent 1, quirk period %d: kernel evaluates %d member-tiles, the replay on its own decisions %d, '
          'without the quirk rows %d' % (CHUNK, rep['kernel'], rep['replay'], rep['replay_no_quirk']))
    for t, m, qrows, margin in rep['located']:
        print('    kernel skips, the replay without quirk rows keeps: tile %d member %d, quirk rows %s, margin %.3g'
              % (t, m, qrows, margin))
    assert rep['kernel'] == rep['replay']


def both_equal(eng, lat, *args):
    on, _ = query(eng, lat, *args, absorb=True)
    off, _ = query(eng, lat, *args, absorb=False)
    assert torch.equal(on.view(torch.int32), off.view(torch.int32)), args
    return on, off


@pytest.mark.gpu
@pytest.mark.parametrize('name', HEADS + ['bias+:0:1', 'bias-:0:1', 'bias+:0:0.25'])
def test_on_off_bit_equal(cuda_device, name):
    from conftest import MAXI, MINI, sample_latent
    dev = cuda_device
    _, eng = head(name, dev)
    lat = [sample_latent(s).reshape(-1).to(dev) for s in range(1, 9)]
    for z in lat:                                                           # 8 latents
        both_equal(eng, z, MINI, MAXI, 64, 0, 64 ** 3, CHUNK)
    for res in (48, 100, 128):                                              # 100: not a multiple of the 16 x 8 block
        both_equal(eng, lat[0], MINI, MAXI, res, 0, res ** 3, CHUNK)
    both_equal(eng, lat[1], MINI, MAXI, 256, 120 * 256 ** 2, 3 * 256 ** 2, CHUNK)   # planes of the benchmark grid
    both_equal(eng, lat[2], MINI, MAXI, 100, 777, 100 ** 3 - 5000, 4097)             # a window not aligned to a plane
    both_equal(eng, lat[3], MINI, MAXI, 128, 40 * 128 ** 2 + 3001, 20 * 128 ** 2 + 77, CHUNK)
    for period in (0, 1, 2, 127, 128, 129, 4097, 25000):
        both_equal(eng, lat[0], MINI, MAXI, 100, 0, 100 ** 3, period)


@pytest.mark.gpu
def test_negative_control_bound_scale(cuda_device):
    """Bounds scaled by 2^-40 certify members that change num: the on / off comparison must see a difference."""
    from conftest import MAXI, MINI, sample_latent
    dev = cuda_device
    _, eng = head('seed:0:4', dev)
    L = lib()
    z = sample_latent(1).reshape(-1).to(dev)
    L.nphm_debug_ens_bound_scale(eng.handle, 2.0 ** -40)
    try:
        on, _ = query(eng, z, MINI, MAXI, 64, 0, 64 ** 3, CHUNK, absorb=True)
        off, _ = query(eng, z, MINI, MAXI, 64, 0, 64 ** 3, CHUNK, absorb=False)
    finally:
        L.nphm_debug_ens_bound_scale(eng.handle, 1.0)
    n = int((on.view(torch.int32) != off.view(torch.int32)).sum())
    print('  bounds x 2^-40: %d of %d outputs differ between absorb on and off' % (n, on.numel()))
    assert n > 0
    on2, _ = query(eng, z, MINI, MAXI, 64, 0, 64 ** 3, CHUNK, absorb=True)
    assert torch.equal(on2.view(torch.int32), off.view(torch.int32)), 'the bound scale was not reset'
