"""Many heads in one band run (csrc/narrowband.cu nphm_band_heads_*, csrc/marching_cubes.cu nphm_mc_heads_*,
utils/reconstruction.extract_meshes_narrowband) against the single-head band ``extract_mesh_narrowband`` of each head: the same
vertex ids, float64 positions, triangles and stats, bit for bit."""
import math

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_ensemble, sample_latent
from narrowband_common import make_npm_head, tilted_plate

pytestmark = pytest.mark.gpu

SYNCING = ('nphm_band_heads_begin', 'nphm_band_heads_corners', 'nphm_band_heads_classify', 'nphm_band_heads_grow',
           'nphm_mc_heads_count')


def _same_mesh(a, b):
    va, vb = np.asarray(a.vertices), np.asarray(b.vertices)
    fa, fb = np.asarray(a.faces), np.asarray(b.faces)
    return va.shape == vb.shape and fa.shape == fb.shape and np.array_equal(fa, fb) and np.array_equal(va, vb)


def _without_padding(st):
    return {k: v for k, v in st.items() if k != 'padded_rows'}


def _dense_mesh(dec, lat, res, nbatch, dev):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, mesh_from_logits
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(dev, dtype=torch.float32)[None]
    return mesh_from_logits(get_logits(dec, lat, grid, nbatch_points=nbatch), MINI, MAXI, res)


def _check_against_single(dec, codes, res, nbatch, dense=False, **kw):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_meshes_narrowband
    meshes, stats = extract_meshes_narrowband(dec, codes, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True, **kw)
    assert len(meshes) == len(stats) == len(codes)
    for h, code in enumerate(codes):
        ref, ref_st = extract_mesh_narrowband(dec, code, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True)
        assert len(ref.vertices) > 0
        assert _same_mesh(meshes[h], ref), 'head %d' % h
        assert _without_padding(stats[h]) == ref_st, 'head %d' % h
        assert stats[h]['padded_rows'] >= 0
        cached = getattr(ref, '_nphm_device_vertices', None)
        if cached is not None:
            assert torch.equal(meshes[h]._nphm_device_vertices, cached)
        if dense:
            assert _same_mesh(meshes[h], _dense_mesh(dec, code, res, nbatch, code.device)), 'head %d vs dense' % h
    return meshes, stats


@pytest.fixture(scope='module')
def ensemble(cuda_device):
    return make_ensemble(0, device=cuda_device).eval(), [sample_latent(s).to(cuda_device) for s in (1, 2, 3)]


@pytest.mark.parametrize('res,train,nbatch', [(64, False, 25000), (64, True, 25000), (66, False, 7000), (66, True, 25000)])
def test_ensemble_heads_equal_single_and_dense(ensemble, res, train, nbatch):
    """S = 3 seeded heads, train and eval mode (the quirk with nbatch_points not dividing res^3), res 66: (res-1) % block != 0."""
    dec, codes = ensemble
    dec.train(train)
    try:
        meshes, _ = _check_against_single(dec, codes, res, nbatch, dense=True)
    finally:
        dec.eval()
    assert len({len(m.vertices) for m in meshes}) == 3                 # the heads differ


def test_npm_deepsdf_heads_equal_single(cuda_device):
    dec, zero = make_npm_head(cuda_device)
    torch.manual_seed(3)
    codes = [zero, zero + 0.02 * torch.randn(512, device=cuda_device), zero + 0.02 * torch.randn(512, device=cuda_device)]
    _check_against_single(dec, codes, 64, 25000)


def test_one_head_equals_single_call(ensemble):
    from nphm_b200.utils.reconstruction import extract_mesh_narrowband, extract_meshes_narrowband
    dec, codes = ensemble
    (mesh,), (st,) = extract_meshes_narrowband(dec, codes[:1], MINI, MAXI, 96, nbatch_points=25000, return_stats=True)
    ref, ref_st = extract_mesh_narrowband(dec, codes[0], MINI, MAXI, 96, nbatch_points=25000, return_stats=True)
    assert _same_mesh(mesh, ref) and _without_padding(st) == ref_st


def test_chunks_change_no_mesh(ensemble):
    from nphm_b200.utils.reconstruction import extract_meshes_narrowband
    dec, codes = ensemble
    codes5 = torch.stack(codes + [sample_latent(s).to(codes[0].device) for s in (4, 5)])
    one, st_one = extract_meshes_narrowband(dec, codes5, MINI, MAXI, 64, nbatch_points=25000, return_stats=True)
    two, st_two = extract_meshes_narrowband(dec, codes5, MINI, MAXI, 64, nbatch_points=25000, return_stats=True, max_heads=2)
    for a, b, sa, sb in zip(one, two, st_one, st_two):
        assert _same_mesh(a, b) and _without_padding(sa) == _without_padding(sb)


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


def test_analytic_heads_finish_at_different_rounds(cuda_device, monkeypatch):
    """Analytic fields through an evaluate callable: spheres of different radii, a head without a surface, and a thin plate that
    needs growth rounds.  Each head's volume, block states, stats and mesh equal its single band's, and the band reads counts back
    once per listing step whatever S is."""
    from nphm_b200 import _native
    from nphm_b200.utils.reconstruction import narrowband_heads_volumes, narrowband_volume, pad_rows
    res, block = 65, 4
    lo, hi = [-1.0] * 3, [1.0] * 3
    h = 2.0 / (res - 1)
    tau = 4 * math.sqrt(3) * h
    fields = [lambda p: (p.norm(dim=-1) - 0.5).float(),
              lambda p: (p.norm(dim=-1) + 5.0).float(),                              # no surface
              lambda p: tilted_plate(p, h, xp=torch).float(),
              lambda p: (p.norm(dim=-1) - 0.27).float()]
    S = len(fields)

    def evaluate(pts):                         # S x n x 3 -> S x n, elementwise: independent of the padding rows
        assert pts.shape[0] == S and pts.shape[1] % 128 == 0
        return torch.stack([f(pts[i]) for i, f in enumerate(fields)])

    log = _count_syncing_calls(monkeypatch)
    bands = _native.NarrowBandHeads(res, block, cuda_device, S)
    vols, stats = narrowband_heads_volumes(bands, evaluate, lo, hi, tau)
    rounds = [s['growth_rounds'] for s in stats]
    assert rounds[0] == rounds[1] == rounds[3] == 0 and rounds[2] >= 2
    assert tuple(log) == SYNCING[:3] + (SYNCING[3],) * (max(rounds) + 1) and bands.readbacks == len(log)
    verts, tris, counts = bands.marching_cubes(vols)
    assert log[-1] == SYNCING[4] and len(log) == 4 + max(rounds) + 1
    states = bands.block_states()
    v_off = t_off = 0
    for i, f in enumerate(fields):
        one = _native.NarrowBandHeads(res, block, cuda_device, 1)
        vol1, st1 = narrowband_heads_volumes(one, lambda p, f=f: f(p[0])[None], lo, hi, tau)
        assert one.readbacks == 4 + st1[0]['growth_rounds']
        assert st1 == [dict(stats[i], padded_rows=st1[0]['padded_rows'])]
        vol, st, band = narrowband_volume(f, lo, hi, res, cuda_device, block=block, margin=tau)
        assert torch.equal(vols[i], vol) and torch.equal(vol1[0], vol)
        assert torch.equal(states[i], band.block_states())
        assert {k: st[k] for k in ('blocks_active', 'voxels_evaluated', 'growth_rounds')} == \
            {k: stats[i][k] for k in ('blocks_active', 'voxels_evaluated', 'growth_rounds')}
        v_ref, t_ref = _native.marching_cubes_device(vol, 0.0, negate=True)
        nv, nt = counts[i]
        assert (nv, nt) == (v_ref.shape[0], t_ref.shape[0]) and (nv > 0) == (i != 1)
        assert torch.equal(verts[v_off:v_off + nv], v_ref) and torch.equal(tris[t_off:t_off + nt], t_ref)
        v_off, t_off = v_off + nv, t_off + nt
    assert v_off == verts.shape[0] and t_off == tris.shape[0]
    # padding: past its count a head's rows repeat its last listed voxel (voxel 0 when it listed nothing)
    bands.begin(0)
    ns = bands.corners()
    xyz = bands.gather(pad_rows(ns), lo, hi)
    for i, n in enumerate(ns):
        assert n > 0 and torch.equal(xyz[i, n:], xyz[i, n - 1].expand(xyz.shape[1] - n, 3))


def test_heads_error_paths(cuda_device):
    from ctypes import byref, c_longlong
    from nphm_b200 import _native
    L = _native.lib()
    assert L.nphm_band_heads_workspace_bytes(64, 4, 0) == -1 and L.nphm_band_heads_workspace_bytes(1, 4, 2) == -1
    assert L.nphm_band_heads_workspace_bytes(64, 0, 2) == -1
    p = _native.McParams(8, 8, 8, 0, 1, 1, 0.0)                                      # ghost_lo: not a whole volume
    assert L.nphm_mc_heads_workspace_bytes(byref(p), 2) == -1
    need = L.nphm_band_heads_workspace_bytes(32, 4, 3)
    ws = torch.empty(need - 1, device=cuda_device, dtype=torch.uint8)
    counts = (c_longlong * 6)()
    stream = torch.cuda.current_stream(cuda_device).cuda_stream
    assert L.nphm_band_heads_begin(32, 4, 3, 0, ws.data_ptr(), ws.numel(), counts, stream) == -4       # NPHM_ERR_CAPACITY
    assert L.nphm_band_heads_begin(32, 4, 3, -1, ws.data_ptr(), need, counts, stream) == -1            # negative quirk period
