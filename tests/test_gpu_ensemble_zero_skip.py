"""The dense ensemble kernel skips the members whose blend weight is exactly zero on a whole tile; the outputs must stay what they
were bit for bit.  Against stored outputs of the kernel before the skip (tests/golden/ensemble_zero_skip.npz, written by
tests/golden/make_golden_ensemble_zero_skip.py), and inside one build: a grid query (compact tiles, most members skipped), the
same points as an xyz query in flat order (linear tiles, few skipped) and in a random order (almost none skipped)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))

CASES = ['grid64_latent1', 'grid64_latent2', 'grid64_latent3', 'grid128_latent1', 'grid128_latent2', 'grid128_latent3',
         'wide64', 'unaligned64', 'slab128', 'xyz_far']


@pytest.fixture(scope='module')
def outputs(cuda_device):
    import make_golden_ensemble_zero_skip as M
    return M.run_cases(cuda_device)


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASES)
def test_matches_golden(outputs, name):
    import make_golden_ensemble_zero_skip as M
    from conftest import load_golden
    ref = load_golden('ensemble_zero_skip.npz')
    assert name in outputs
    assert M.matches(ref, name, outputs[name]), name


@pytest.mark.gpu
@pytest.mark.parametrize('mini, maxi', [('bench', 'bench'), ('wide', 'wide')])
def test_grid_equals_xyz_in_any_order(cuda_device, mini, maxi):
    import make_golden_ensemble_zero_skip as M
    from conftest import MAXI, MINI
    lo, hi = (MINI, MAXI) if mini == 'bench' else (M.WIDE_MIN, M.WIDE_MAX)
    eng, lat = M.engine(cuda_device)
    res = 128
    grid = eng.query_grid(lat[0], lo, hi, res, 0, res ** 3, 0, impl='tc')[0]
    axes = [torch.from_numpy(np.linspace(lo[a], hi[a], res).astype(np.float32)) for a in range(3)]
    xyz = torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=-1).reshape(1, -1, 3).to(cuda_device)
    flat = eng.query(xyz, lat[:1], eval_quirk=False, impl='tc')[0].reshape(-1)
    perm = torch.randperm(res ** 3, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    shuffled = eng.query(xyz[:, perm], lat[:1], eval_quirk=False, impl='tc')[0].reshape(-1)
    unshuffled = torch.empty_like(shuffled)
    unshuffled[perm] = shuffled
    assert torch.equal(grid, flat)
    assert torch.equal(grid, unshuffled)
