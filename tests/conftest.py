import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')

MINI = [-.55, -.5, -.95]
MAXI = [0.55, 0.75, 0.4]


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name))


def mean_anchors():
    a = load_golden('assets.npz')['anchors_39']
    return torch.from_numpy(a).float().unsqueeze(0).unsqueeze(0)       # fitting_pointclouds.py:80


def make_ensemble(seed=0, scale=1.0, device='cpu'):
    """Same recipe as tests/golden/make_golden.py:make_ensemble, with the drop-in class."""
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    torch.manual_seed(seed)
    dec = FastEnsembleDeepSDFMirrored(lat_dim_glob=64, lat_dim_loc=32, n_loc=39, n_symm_pairs=16,
                                      anchors=mean_anchors(), hidden_dim=200, n_layers=4, pos_mlp_dim=256)
    if scale != 1.0:
        with torch.no_grad():
            for i in range(5):
                getattr(dec.ensembled_deep_sdf, 'lin%d' % i).weight.mul_(scale)
    if device != 'cpu':
        dec = dec.to(device)
        dec.anchors = dec.anchors.to(device)
    return dec


def make_deformation(device='cpu'):
    from nphm_b200.models.deepSDF import DeformationNetwork
    torch.manual_seed(10)
    dfn = DeformationNetwork(mode='compress', lat_dim_expr=200, lat_dim_id=32, lat_dim_glob_shape=64,
                             lat_dim_loc_shape=32, n_loc=39, anchors=mean_anchors(), hidden_dim=512, nlayers=6,
                             out_dim=3, input_dim=3)
    dfn.eval()
    return dfn.to(device)


def make_npm(device='cpu'):
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(12)
    return DeepSDF(lat_dim=64, hidden_dim=96, nlayers=8, geometric_init=True).to(device)


def sample_latent(seed):
    a = load_golden('assets.npz')
    torch.manual_seed(seed)
    mean, std = torch.from_numpy(a['nphm_lat_mean']), torch.from_numpy(a['nphm_lat_std'])
    return torch.randn(mean.shape) * std * 0.85 + mean                  # fitting_pointclouds.py:206


def sd_numpy(module):
    return {k: v.detach().cpu().numpy() for k, v in module.state_dict().items()}


def sphere_volume(res, radius=0.4, center=(0.03, -0.02, 0.01), shape=None):
    shape = shape or (res, res, res)
    ax = [np.linspace(-0.5, 0.5, n) for n in shape]
    X, Y, Z = np.meshgrid(*ax, indexing='ij')
    return (np.sqrt((X - center[0]) ** 2 + (Y - center[1]) ** 2 + (Z - center[2]) ** 2) - radius).astype(np.float32)


def noise_volume(shape, seed=7):
    rng = np.random.RandomState(seed)
    return rng.uniform(-1, 1, size=shape).astype(np.float32)


def mesh_edge_stats(tris):
    """(#directed half edges that appear more than once, #half edges without an opposite partner)."""
    t = np.asarray(tris).astype(np.int64)
    he = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]], axis=0)
    n = int(t.max()) + 1 if len(t) else 1
    key = he[:, 0] * n + he[:, 1]
    rkey = he[:, 1] * n + he[:, 0]
    uniq, counts = np.unique(key, return_counts=True)
    dup = int((counts > 1).sum())
    unmatched = int((~np.isin(rkey, uniq)).sum())
    return dup, unmatched


@pytest.fixture(scope='session')
def cuda_device():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return torch.device('cuda:0')
