"""GPU parity against outputs of the UNMODIFIED REFERENCE MODULES (torch fp32), stored in tests/golden/reference_configs.npz
by tests/golden/make_golden_reference.py, on BASELINE.json's own configurations:

  * configs[0]: the 64^3 grid in full, eval and train mode, through ``get_logits`` (seeded points + every chunk boundary)
  * configs[1]: the 256^3 grid - the in-kernel-grid path the bench times (``query_grid``) over the whole volume, compared on
    whole chunks of the reference's 672 (first, middle, far field, the ragged last one), plus the drop-in ``get_logits`` path
  * configs[2]: deformation network on a 64^3 grid, ``get_logits_backward`` with a DeepSDF-type expression decoder

The CUDA kernels are called through the C ABI.  Tolerance: 1e-5 abs (north_star)."""
import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, load_golden, make_deformation, make_ensemble, sample_latent

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.fixture(scope='module')
def ref():
    return load_golden('reference_configs.npz')


def _grid(res, dev):
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    g = create_grid_points_from_bounds(MINI, MAXI, res)
    return torch.from_numpy(g).to(dev, dtype=torch.float).reshape(1, -1, 3)          # fitting_pointclouds.py:168-170


def _fingerprint(module):
    fp = []
    for v in module.state_dict().values():
        a = v.detach().double().reshape(-1).cpu().numpy()
        head = np.zeros(8)
        head[:min(8, a.size)] = a[:8]
        fp.append(np.concatenate([[a.sum(), (a * a).sum()], head]))
    return list(module.state_dict().keys()), np.array(fp)


def test_mirror_initialises_like_the_reference(cuda_device, ref):
    for module, tag in ((make_ensemble(0), 'ens'), (make_deformation(), 'def')):
        keys, fp = _fingerprint(module)
        assert keys == list(ref[tag + '_keys'])
        assert np.array_equal(fp, ref[tag + '_fp'])


@pytest.mark.parametrize('train', [False, True])
def test_config1_64cube_full_vs_reference(cuda_device, ref, train):
    """BASELINE.json configs[0]: single-head SDF query on the 64^3 grid, nbatch_points 25 000 (-sample) and 20 000 (fitting)."""
    from nphm_b200.models.reconstruction import get_logits
    dec = make_ensemble(0, device=cuda_device)
    dec.train(train)
    lat = sample_latent(1).to(cuda_device)
    grid = _grid(64, cuda_device)
    for nb in (25000, 20000):
        got = get_logits(dec, lat, grid, nbatch_points=nb)
        assert got.shape == (64 ** 3,) and got.dtype == np.float32
        idx, want = ref['c1_%d_%d_idx' % (train, nb)], ref['c1_%d_%d_sdf' % (train, nb)]
        err = float(np.abs(got[idx] - want).max())
        print('64^3 train=%s nbatch=%d: max abs err %.3g' % (train, nb, err))
        assert err < TOL


def test_config2_256cube_full_volume_vs_reference(cuda_device, ref):
    """BASELINE.json configs[1]: the 16.7 M-point volume of the benchmark step against the reference's chunks."""
    from nphm_b200.models.reconstruction import get_logits
    res, nb = 256, 25000
    total = res ** 3
    dec = make_ensemble(0, device=cuda_device).eval()
    lat = sample_latent(1).to(cuda_device)
    # (a) the path bench.py times: grid generated in the kernel
    vol, _ = dec.engine().query_grid(lat, MINI, MAXI, res, 0, total, quirk_period=nb)
    got = vol.cpu().numpy()
    chunks = sorted(int(k.split('_')[-1]) for k in ref.files if k.startswith('c2_chunk_'))
    want = np.concatenate([ref['c2_chunk_%d' % c] for c in chunks])
    idx = np.concatenate([np.arange(c * nb, min((c + 1) * nb, total)) for c in chunks])
    diff = np.abs(got[idx] - want)
    worst = int(diff.argmax())
    print('256^3 in-kernel grid: max abs err %.3g at flat index %d (sdf %.4g)' % (diff.max(), idx[worst], want[worst]))
    assert diff.max() < TOL
    # every chunk's last index carries the eval-mode quirk value in both
    last = np.array([min((c + 1) * nb, total) - 1 for c in chunks])
    pos = np.searchsorted(idx, last)
    assert np.abs(got[last] - want[pos]).max() < TOL
    assert np.abs(want[pos] - want[pos - 1]).max() > 1e-4       # the quirk is visible in the reference's own output
    # far field (sum of anchor weights underflows, SDF ~ 0.002 * global member)
    far = np.abs(want) < 1e-2
    assert far.sum() > 1000 and diff[far].max() < TOL
    # (b) the drop-in get_logits on explicit points: whole chunks, incl. the ragged last one
    grid = _grid(res, cuda_device)
    for c in chunks:
        pts = grid[:, c * nb:min((c + 1) * nb, total)]
        g2 = get_logits(dec, lat, pts, nbatch_points=nb)
        assert np.abs(g2 - ref['c2_chunk_%d' % c]).max() < TOL
    # a window of the grid path equals the same window of the full volume (first/count addressing)
    part, _ = dec.engine().query_grid(lat, MINI, MAXI, res, 1234567, 300001, quirk_period=nb)
    assert torch.equal(part, vol[1234567:1234567 + 300001])


def test_config3_deformation_and_joint_vs_reference(cuda_device, ref):
    """BASELINE.json configs[2] at 64^3: forward-deformation field and the identity field at the deformed points."""
    dfn = make_deformation(cuda_device)
    dec = make_ensemble(0, device=cuda_device).eval()
    lat_id = sample_latent(1).to(cuda_device)
    lat_ex = torch.from_numpy(ref['c3_lat_ex']).to(cuda_device)
    cond = torch.cat([lat_id, lat_ex]).reshape(1, 1, -1)
    idx = torch.from_numpy(ref['c3_idx']).to(cuda_device)
    pts = _grid(64, cuda_device)[:, idx]
    n = pts.shape[1]
    with torch.no_grad():
        _, anchors = dec(pts[:, :1], lat_id.reshape(1, 1, -1), None)
        got_off, _ = dfn(pts, cond.repeat(1, n, 1), anchors)
        want_off = ref['c3_offsets']
        err = float(np.abs(got_off[0].cpu().numpy() - want_off).max())
        print('deformation 64^3: max abs err %.3g (|offset| max %.3g)' % (err, float(np.abs(want_off).max())))
        assert err < TOL
        warped = pts + torch.from_numpy(want_off).to(cuda_device).unsqueeze(0)
        dec.train()                                          # no chunk quirk: compare the plain field
        got_sdf, _ = dec(warped, lat_id.reshape(1, 1, -1).expand(1, n, -1), None)
        assert float(np.abs(got_sdf.reshape(-1).cpu().numpy() - ref['c3_sdf']).max()) < TOL


def test_get_logits_backward_vs_reference(cuda_device, ref):
    """models/reconstruction.py:28-56 with a DeepSDF-type expression decoder (the only kind it works with upstream)."""
    from nphm_b200.models.deepSDF import DeepSDF
    from nphm_b200.models.reconstruction import get_logits_backward
    torch.manual_seed(31)
    ex = DeepSDF(lat_dim=100, hidden_dim=128, nlayers=6, out_dim=3).to(cuda_device).eval()
    keys, fp = _fingerprint(ex)
    assert keys == list(ref['ex_keys']) and np.array_equal(fp, ref['ex_fp'])
    dec = make_ensemble(0, device=cuda_device).eval()
    lat_id = sample_latent(1).to(cuda_device)
    lat_ex = torch.from_numpy(ref['bw_lat_ex']).to(cuda_device)
    grid = _grid(24, cuda_device)
    got, anc_g = get_logits_backward(dec, ex, lat_id.reshape(1, 1, -1), lat_ex, grid, nbatch_points=5000,
                                     return_anchors=True)
    want = ref['bw_sdf']
    assert got.shape == want.shape and np.abs(got - want).max() < TOL
    assert float(np.abs(anc_g.detach().cpu().numpy() - ref['bw_anchors']).max()) < 1e-6
    # encoding_expr=None: plain get_logits
    got0 = get_logits_backward(dec, ex, lat_id.reshape(1, 1, -1), None, grid, nbatch_points=5000)
    assert np.abs(got0 - ref['bw_sdf_no_expr']).max() < TOL
