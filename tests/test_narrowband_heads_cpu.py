"""Many heads in one band run (utils/reconstruction.extract_meshes_narrowband) without a GPU: the head-chunk planner, the padding
and split helpers, the argument checks, and the per-head fallback that decoders on the CPU take (each head the dense mesh)."""
import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, make_ensemble, make_npm, sample_latent


def test_plan_head_chunks_whole_chunks_in_order():
    from nphm_b200.utils.reconstruction import plan_head_chunks
    assert plan_head_chunks(10, 100, 350) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert plan_head_chunks(10, 100, 350, max_heads=2) == [(0, 2), (2, 4), (4, 6), (6, 8), (8, 10)]
    assert plan_head_chunks(4, 100, 10 ** 9) == [(0, 4)]
    assert plan_head_chunks(3, 100, 10) == [(0, 1), (1, 2), (2, 3)]          # a budget below one head still runs one at a time
    assert plan_head_chunks(1, 100, 0, max_heads=8) == [(0, 1)]
    for n, per, budget, mh in [(17, 7, 50, None), (17, 7, 50, 3), (5, 1, 5, 2)]:
        chunks = plan_head_chunks(n, per, budget, mh)
        assert [h for a, b in chunks for h in range(a, b)] == list(range(n))
        assert len({b - a for a, b in chunks[:-1]}) <= 1 and chunks[-1][1] - chunks[-1][0] <= chunks[0][1] - chunks[0][0]
    with pytest.raises(ValueError):
        plan_head_chunks(3, 1, 10, max_heads=0)


def test_pad_rows_and_split_heads():
    from nphm_b200.utils.reconstruction import pad_rows, split_heads
    assert pad_rows([0, 1, 5]) == 128 and pad_rows([128, 3]) == 128 and pad_rows([129]) == 256 and pad_rows([0, 0]) == 0
    assert pad_rows([10, 7], multiple=4) == 12
    flat = torch.arange(12).reshape(6, 2)
    parts = split_heads(flat, [2, 0, 3, 1])
    assert [p.shape[0] for p in parts] == [2, 0, 3, 1]
    assert torch.equal(torch.cat(parts), flat)


def test_argument_checks():
    from nphm_b200.utils.reconstruction import _as_codes, extract_meshes_narrowband
    dec = make_ensemble(0).eval()
    with pytest.raises(ValueError):
        extract_meshes_narrowband(dec, [], MINI, MAXI, 16)
    with pytest.raises(ValueError):
        extract_meshes_narrowband(dec, torch.zeros(0, 96), MINI, MAXI, 16)
    with pytest.raises(ValueError):
        extract_meshes_narrowband(dec, [torch.zeros(96), torch.zeros(64)], MINI, MAXI, 16)
    codes = _as_codes([torch.zeros(1, 1, 4), torch.ones(4)])
    assert codes.shape == (2, 4) and torch.equal(codes[1], torch.ones(4))
    assert _as_codes(torch.zeros(3, 1, 5)).shape == (3, 5)


def _cpu_mesh_from_logits(logits, mini, maxi, res):
    """mesh_from_logits with the C restatement of marching cubes (oracle/mc_oracle.c): the GPU kernels need a device."""
    from nphm_b200.utils.mesh import make_mesh
    from oracle import nphm_oracle as O
    v, t = O.mesh_from_logits(np.asarray(logits, dtype=np.float32).copy(), mini, maxi, res)
    return make_mesh(v, t)


def _dense_mesh(dec, code, res, nbatch):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).float()[None]
    return _cpu_mesh_from_logits(get_logits(dec, code, grid, nbatch_points=nbatch), MINI, MAXI, res)


@pytest.mark.parametrize('kind,res,train', [('ensemble', 16, False), ('ensemble', 20, True), ('npm', 24, False),
                                            ('npm', 18, True)])
def test_cpu_fallback_each_head_is_dense(kind, res, train, monkeypatch):
    """Decoders on the CPU take extract_mesh_narrowband's dense path head by head: each head the mesh of
    mesh_from_logits(get_logits(...)) under its own code, in order, in the decoder's mode."""
    from nphm_b200.utils import reconstruction as R
    monkeypatch.setattr(R, 'mesh_from_logits', _cpu_mesh_from_logits)
    if kind == 'ensemble':
        dec, codes = make_ensemble(0), [sample_latent(s) for s in (1, 2, 3)]
    else:
        dec = make_npm()
        with torch.no_grad():                        # a field that varies over the grid, with its zero level inside it
            dec.lin0.weight[:, :3].mul_(1000.0)
            dec.lin8.bias.add_(0.63)
        torch.manual_seed(5)
        codes = torch.randn(3, 64) * 0.1
    dec.train(train)
    nbatch = 1000
    meshes, stats = R.extract_meshes_narrowband(dec, codes, MINI, MAXI, res, nbatch_points=nbatch, return_stats=True,
                                                max_heads=2)
    assert len(meshes) == len(stats) == 3
    refs = [_dense_mesh(dec, codes[h], res, nbatch) for h in range(3)]
    assert len({len(r.vertices) for r in refs}) > 1 or kind == 'npm'        # the ensemble's heads differ
    for mesh, st, ref in zip(meshes, stats, refs):
        assert len(ref.vertices) > 0
        assert np.array_equal(np.asarray(mesh.faces), np.asarray(ref.faces))
        assert np.array_equal(np.asarray(mesh.vertices), np.asarray(ref.vertices))
        assert st['voxels_evaluated'] == res ** 3 and st['padded_rows'] == 0
