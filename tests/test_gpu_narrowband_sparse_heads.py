"""The block-sparse band of S heads (csrc/narrowband_sparse.cu nphm_band_sparse_heads_*, _native.SparseNarrowBandHeads,
extract_meshes_narrowband / extract_posed_meshes_narrowband with sparse=True) against the single sparse band of each head, the
dense-storage head band and the dense meshes: the same vertex ids, float64 positions, triangles and band stats, bit for bit."""
import math

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_deformation, make_ensemble, sample_latent
from narrowband_common import make_npm_head, tilted_plate

pytestmark = pytest.mark.gpu

SYNCING = ('nphm_band_sparse_heads_begin', 'nphm_band_sparse_heads_corners', 'nphm_band_sparse_heads_classify',
           'nphm_band_sparse_heads_grow', 'nphm_band_sparse_heads_mc_count')
BAND_STATS = ('blocks_active', 'blocks_total', 'voxels_evaluated', 'voxels_total', 'growth_rounds', 'margin')


def _same_mesh(a, b):
    va, vb = np.asarray(a.vertices), np.asarray(b.vertices)
    fa, fb = np.asarray(a.faces), np.asarray(b.faces)
    return va.shape == vb.shape and fa.shape == fb.shape and np.array_equal(fa, fb) and np.array_equal(va, vb)


def _band(st):
    return {k: st[k] for k in BAND_STATS}


def _dense_mesh(dec, lat, res, nbatch, dev):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, mesh_from_logits
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float32)[None]
    return mesh_from_logits(get_logits(dec, lat, grid, nbatch_points=nbatch), MINI, MAXI, res)


def _check_canonical(dec, codes, res, nbatch, dense=False, **kw):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_meshes_narrowband
    meshes, stats = extract_meshes_narrowband(dec, codes, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True, sparse=True, **kw)
    dmeshes, dstats = extract_meshes_narrowband(dec, codes, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True, **kw)
    assert len(meshes) == len(stats) == len(codes)
    for h, code in enumerate(codes):
        ref, ref_st = extract_mesh_narrowband(dec, code, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True, sparse=True)
        assert len(ref.vertices) > 0
        assert _same_mesh(meshes[h], ref) and _same_mesh(meshes[h], dmeshes[h]), 'head %d' % h
        assert _band(stats[h]) == _band(ref_st) == _band(dstats[h]), 'head %d' % h
        assert stats[h]['padded_rows'] == dstats[h]['padded_rows']
        assert stats[h]['device_bytes']['band'] > 0 and stats[h]['device_bytes']['heads'] >= 1
        assert torch.equal(meshes[h]._nphm_device_vertices, ref._nphm_device_vertices)
        if dense:
            assert _same_mesh(meshes[h], _dense_mesh(dec, code, res, nbatch, code.device)), 'head %d vs dense' % h
    return meshes, stats


@pytest.fixture(scope='module')
def ensemble(cuda_device):
    return make_ensemble(0, device=cuda_device).eval(), [sample_latent(s).to(cuda_device) for s in (1, 2, 3)]


@pytest.mark.parametrize('res,train,nbatch', [(64, False, 25000), (64, True, 25000), (66, False, 7000)])
def test_ensemble_heads_equal_single_sparse_dense_heads_and_dense(ensemble, res, train, nbatch):
    """S = 3 seeded heads in train and eval mode (the quirk, nbatch_points not dividing res^3); res 66: (res-1) % block != 0."""
    dec, codes = ensemble
    dec.train(train)
    try:
        meshes, _ = _check_canonical(dec, codes, res, nbatch, dense=True)
    finally:
        dec.eval()
    assert len({len(m.vertices) for m in meshes}) == 3


def test_npm_deepsdf_heads(cuda_device):
    dec, zero = make_npm_head(cuda_device)
    torch.manual_seed(3)
    codes = [zero, zero + 0.02 * torch.randn(512, device=cuda_device), zero + 0.02 * torch.randn(512, device=cuda_device)]
    _check_canonical(dec, codes, 64, 25000)


def test_s_heads_equal_s_single_calls_and_chunks_change_nothing(ensemble):
    from nphm_b200.utils.reconstruction import extract_meshes_narrowband
    dec, codes = ensemble
    codes5 = torch.stack(codes + [sample_latent(s).to(codes[0].device) for s in (4, 5)])
    kw = dict(nbatch_points=25000, return_stats=True, sparse=True)
    one, st_one = extract_meshes_narrowband(dec, codes5, MINI, MAXI, 48, **kw)
    two, st_two = extract_meshes_narrowband(dec, codes5, MINI, MAXI, 48, max_heads=2, **kw)
    assert [s['device_bytes']['heads'] for s in st_two] == [2, 2, 2, 2, 1]
    for h in range(5):
        (single,), (st_single,) = extract_meshes_narrowband(dec, codes5[h:h + 1], MINI, MAXI, 48, **kw)
        assert _same_mesh(one[h], two[h]) and _same_mesh(one[h], single)
        assert _band(st_one[h]) == _band(st_two[h]) == _band(st_single)


def test_tiny_pool_changes_no_mesh(ensemble, monkeypatch):
    """Pools of one brick per head: every allocating step finds them short, grows them and repeats."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import extract_meshes_narrowband
    dec, codes = ensemble
    ref, ref_st = extract_meshes_narrowband(dec, codes, MINI, MAXI, 48, nbatch_points=7000, return_stats=True, sparse=True)
    grown = []
    orig = _native.SparseNarrowBandHeads._set_pool

    def spy(self, slots, keep=0):
        grown.append((slots, keep))
        return orig(self, slots, keep)
    monkeypatch.setattr(_native.SparseNarrowBandHeads, 'default_slots', staticmethod(lambda res, block: 1))
    monkeypatch.setattr(_native.SparseNarrowBandHeads, '_set_pool', spy)
    got, st = extract_meshes_narrowband(dec, codes, MINI, MAXI, 48, nbatch_points=7000, return_stats=True, sparse=True)
    assert grown[0][0] == 1 and len(grown) >= 3 and any(k > 0 for _, k in grown)       # grown while keeping used bricks
    for a, b, sa, sb in zip(got, ref, st, ref_st):
        assert _same_mesh(a, b) and _band(sa) == _band(sb)


def _count_syncing_calls(monkeypatch):
    """Wrap the entry points that read counts back (and synchronise the stream) in the ctypes binding; returns the call log."""
    from nphm_b200 import _native
    L = _native.lib()
    log = []
    for name in SYNCING:
        fn = getattr(L, name)

        def wrapped(*args, _fn=fn, _name=name):
            log.append(_name)
            return _fn(*args)
        monkeypatch.setattr(L, name, wrapped)
    return log


@pytest.mark.parametrize('slots', [16 ** 3, 1])
def test_analytic_heads_finish_at_different_rounds(cuda_device, monkeypatch, slots):
    """Spheres of different radii, a head without a surface and a thin plate that needs growth rounds: each head's block states,
    stats and brick mesh equal its single sparse band's, and each listing step reads counts back once whatever S is (pools that
    hold every block), plus once per capacity retry (one-brick pools)."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import LocalExchange, _mc_pair, _slab_mesh, narrowband_heads_volumes, narrowband_volume
    res, block = 65, 4
    lo, hi = [-1.0] * 3, [1.0] * 3
    h = 2.0 / (res - 1)
    tau = 4 * math.sqrt(3) * h
    fields = [lambda p: (p.norm(dim=-1) - 0.5).float(),
              lambda p: (p.norm(dim=-1) + 5.0).float(),
              lambda p: tilted_plate(p, h, xp=torch).float(),
              lambda p: (p.norm(dim=-1) - 0.27).float()]
    S = len(fields)

    def evaluate(pts):
        assert pts.shape[0] == S and pts.shape[1] % 128 == 0
        return torch.stack([f(pts[i]) for i, f in enumerate(fields)])

    log = _count_syncing_calls(monkeypatch)
    bands = _native.SparseNarrowBandHeads(res, block, cuda_device, S, slots=slots)
    vols, stats = narrowband_heads_volumes(bands, evaluate, lo, hi, tau)
    rounds = [s['growth_rounds'] for s in stats]
    assert rounds[0] == rounds[1] == rounds[3] == 0 and rounds[2] >= 2
    if slots == 16 ** 3:
        assert tuple(log) == SYNCING[:3] + (SYNCING[3],) * (max(rounds) + 1)
    else:
        assert len(log) > 4 + max(rounds) and bands.slots > 1
    assert bands.readbacks == len(log)
    verts, tris, counts = bands.marching_cubes(vols)
    assert log[-1] == SYNCING[4]
    states = bands.block_states()
    v_off = t_off = 0
    for i, f in enumerate(fields):
        vol, st, band = narrowband_volume(f, lo, hi, res, cuda_device, block=block, margin=tau, sparse=True)
        assert torch.equal(states[i], band.block_states())
        assert {k: st[k] for k in ('blocks_active', 'voxels_evaluated', 'growth_rounds')} == \
            {k: stats[i][k] for k in ('blocks_active', 'voxels_evaluated', 'growth_rounds')}
        v_ref, t_ref = _slab_mesh([band], [vol], LocalExchange(1), *_mc_pair(True), cuda_device)
        nv, nt = counts[i]
        assert (nv, nt) == (v_ref.shape[0], t_ref.shape[0]) and (nv > 0) == (i != 1)
        assert torch.equal(verts[v_off:v_off + nv], v_ref) and torch.equal(tris[t_off:t_off + nt], t_ref)
        dense_ref, _ = _native.marching_cubes_device(band.dense_volume(), 0.0, negate=True)
        assert torch.equal(verts[v_off:v_off + nv], dense_ref)
        v_off, t_off = v_off + nv, t_off + nt
    assert v_off == verts.shape[0] and t_off == tris.shape[0]
    # padding: past its count a head's rows repeat its last listed voxel
    bands.begin(0)
    ns = bands.corners()
    from nphm_b200.utils.reconstruction import pad_rows
    xyz = bands.gather(pad_rows(ns), lo, hi)
    for i, n in enumerate(ns):
        assert n > 0 and torch.equal(xyz[i, n:], xyz[i, n - 1].expand(xyz.shape[1] - n, 3))


def test_sparse_heads_error_paths(cuda_device):
    from ctypes import byref, c_longlong
    from nphm_b200 import _native
    L = _native.lib()
    assert L.nphm_band_sparse_heads_workspace_bytes(64, 4, 0) == -1                 # S = 0
    assert L.nphm_band_sparse_heads_workspace_bytes(64, 4, 65536) == -1
    assert L.nphm_band_sparse_heads_workspace_bytes(64, 0, 2) == -1                 # bad block
    assert L.nphm_band_sparse_heads_workspace_bytes(8193, 8, 2) == -1               # res over 8192
    assert L.nphm_band_sparse_heads_workspace_bytes(2049, 1, 2) == -1               # 2049^3 corners: indices are u32
    assert L.nphm_band_sparse_heads_mc_workspace_bytes(64, 4, 0, 10) == -1
    assert L.nphm_band_sparse_heads_mc_workspace_bytes(64, 4, 2, -1) == -1
    with pytest.raises(_native.NativeError):
        _native.SparseNarrowBandHeads(64, 4, cuda_device, 0)
    band = _native.SparseNarrowBandHeads(32, 4, cuda_device, 3, slots=8)
    counts = (c_longlong * 12)()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    need = band.ws.numel()
    assert L.nphm_band_sparse_heads_begin(32, 4, 3, 0, band.ws.data_ptr(), need - 1, byref(band.pool), counts, stream) == -4
    assert L.nphm_band_sparse_heads_begin(32, 4, 3, -1, band.ws.data_ptr(), need, byref(band.pool), counts, stream) == -1
    assert L.nphm_band_sparse_heads_begin(32, 4, 0, 0, band.ws.data_ptr(), need, byref(band.pool), counts, stream) == -1
    with pytest.raises(ValueError):
        band.classify(0.1, None)                         # the volumes of a sparse band are the band itself


# ------------------------------------------------------------------------------------------ posed meshes
@pytest.mark.parametrize('case', ['compress-train-1', 'compress-train-3', 'compress-eval-3', 'expr_only-eval-2', 'glob_only-eval-2',
                                  'npm-2'])
def test_posed_sparse_equals_dense_storage_and_dense(cuda_device, case):
    import posed_f64_common as P
    from posed_common import npm_case
    from test_gpu_posed import _margin_for
    from nphm_b200.models import reconstruction as R
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, extract_posed_meshes_narrowband, mesh_from_logits
    name, mode, S = (case.split('-') + [None])[:3] if not case.startswith('npm') else ('npm', 'eval', case.split('-')[1])
    S = int(S)
    res, nbatch = 40, 7000
    if name == 'npm':
        dec, dfn, lat, z_ex, _, _ = npm_case(cuda_device)
        lo, hi = [-0.35, -0.3, -0.45], [0.35, 0.4, 0.25]
    else:
        dec = make_ensemble(0, device=cuda_device).train(mode == 'train')
        dfn = make_deformation(cuda_device) if name == 'compress' else P.make_deformation(name, cuda_device)
        lat = sample_latent(1).to(cuda_device)
        torch.manual_seed(8)
        z_ex = torch.randn(3, 200, device=cuda_device)[:S] * 0.1
        lo, hi = MINI, MAXI
    margin = _margin_for(dec, dfn, lat, z_ex, res, nbatch, lo, hi)
    kw = dict(nbatch_points=nbatch, margin=margin, return_stats=True)
    meshes, stats = extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, lo, hi, res, sparse=True, **kw)
    dmeshes, dstats = extract_posed_meshes_narrowband(dec, dfn, lat, z_ex, lo, hi, res, **kw)
    grid = torch.from_numpy(create_grid_points_from_bounds(lo, hi, res)).to(cuda_device, torch.float32)[None]
    dense = R.get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=nbatch)
    assert len(meshes) == S
    for s in range(S):
        ref = mesh_from_logits(dense[s], lo, hi, res)
        assert len(ref.faces) > 0
        assert _same_mesh(meshes[s], ref) and _same_mesh(meshes[s], dmeshes[s]), 'expression %d' % s
        assert _band(stats[s]) == _band(dstats[s]) and stats[s]['margin'] == margin
