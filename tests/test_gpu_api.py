"""GPU tests of the C-ABI boundary behaviour: error codes/messages, empty inputs, unsupported configurations,
non-default streams, handle re-use across weight updates."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, load_golden, make_ensemble, mean_anchors, sample_latent, sd_numpy
from oracle import nphm_oracle as O

pytestmark = pytest.mark.gpu


def test_error_codes_and_messages(cuda_device):
    from nphm_b200 import _native
    L = _native.lib()
    h = ctypes.c_void_p()
    bad = _native.EnsembleConfig(39, 30, 64, 32, 200, 4, 256)            # 2*n_symm_pairs > n_loc
    rc = L.nphm_ensemble_create(ctypes.byref(bad), ctypes.byref(h))
    assert rc == -1 and b'anchor counts' in L.nphm_last_error()
    dec = make_ensemble(0, device=cuda_device).eval()
    eng = dec.engine()
    lat = sample_latent(1).to(cuda_device)
    with pytest.raises(_native.NativeError, match='outside'):
        eng.query_grid(lat, MINI, MAXI, 8, 500, 100, 0)                    # range beyond the 8^3 grid
    with pytest.raises(_native.NativeError, match='unknown impl'):
        eng.query_grid(lat, MINI, MAXI, 8, 0, 8, 0, impl=9)
    # a handle without weights refuses to run
    h2 = ctypes.c_void_p()
    cfg = _native.EnsembleConfig(39, 16, 64, 32, 200, 4, 256)
    assert L.nphm_ensemble_create(ctypes.byref(cfg), ctypes.byref(h2)) == 0
    out = torch.zeros(8, device=cuda_device)
    rc = L.nphm_ensemble_query(h2, out.data_ptr(), lat.data_ptr(), 1, 2, 0, out.data_ptr(), None, 0, None)
    assert rc == -1 and b'not loaded' in L.nphm_last_error()
    L.nphm_ensemble_destroy(h2)


def test_empty_and_tiny_queries(cuda_device):
    dec = make_ensemble(0, device=cuda_device).eval()
    eng = dec.engine()
    lat = sample_latent(1).to(cuda_device)
    for impl in ('simt', 'tc', 'tc_pruned'):
        s, a = eng.query(torch.zeros(1, 0, 3, device=cuda_device), lat.reshape(1, -1), eval_quirk=True, impl=impl)
        assert s.shape == (1, 0, 1) and a.shape == (1, 39, 3)
        out, _ = eng.query_grid(lat, MINI, MAXI, 4, 10, 0, 0, impl=impl)
        assert out.numel() == 0
        one, _ = eng.query(torch.tensor([[[0.01, 0.02, 0.03]]], device=cuda_device), lat.reshape(1, -1),
                           eval_quirk=False, impl=impl)
        p = O.EnsembleParams(sd_numpy(dec), load_golden('assets.npz')['anchors_39'])
        ref, _ = O.ensemble_forward(p, np.array([[0.01, 0.02, 0.03]], np.float32), lat.cpu().numpy(), eval_mode=False)
        assert abs(one.item() - ref[0]) < 1e-5


def test_unsupported_configuration_uses_ffma_and_tc_request_fails(cuda_device):
    """A non-NPHM ensemble shape (hidden 160, 10 anchors) runs on the general FFMA kernel; forcing the tensor-core kernel
    reports NPHM_ERR_UNSUPPORTED instead of silently doing something else."""
    from nphm_b200 import _native
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    torch.manual_seed(3)
    anchors = mean_anchors()[:, :, :10]
    dec = FastEnsembleDeepSDFMirrored(32, 16, 10, 3, anchors, 160, 4, pos_mlp_dim=64).to(cuda_device).eval()
    dec.anchors = dec.anchors.to(cuda_device)
    x = (torch.rand(1, 300, 3, device=cuda_device) - 0.5)
    lat = torch.randn(1, 1, dec.lat_dim, device=cuda_device) * 0.1
    with torch.no_grad():
        fused, anc = dec(x, lat, None)                                      # auto -> FFMA kernel
        ref, anc_ref = dec._forward_composite(x, lat)
    assert (fused - ref).abs().max().item() < 1e-5 and (anc - anc_ref).abs().max().item() < 1e-6
    with pytest.raises(_native.NativeError, match='does not support'):
        dec.engine().query(x, lat[:, 0], eval_quirk=True, impl='tc')


def test_non_default_stream_and_weight_update(cuda_device):
    dec = make_ensemble(0, device=cuda_device).eval()
    lat = sample_latent(1).to(cuda_device)
    eng = dec.engine()
    base, _ = eng.query_grid(lat, MINI, MAXI, 16, 0, 16 ** 3, 1000)
    stream = torch.cuda.Stream(device=cuda_device)
    with torch.cuda.stream(stream):
        other, _ = dec.engine().query_grid(lat, MINI, MAXI, 16, 0, 16 ** 3, 1000)
    stream.synchronize()
    assert torch.equal(base, other)
    # load_state_dict -> the engine repacks (same handle)
    dec2 = make_ensemble(5, 2.0, device=cuda_device).eval()
    dec.load_state_dict(dec2.state_dict(), strict=True)
    a, _ = dec.engine().query_grid(lat, MINI, MAXI, 16, 0, 16 ** 3, 1000)
    b, _ = dec2.engine().query_grid(lat, MINI, MAXI, 16, 0, 16 ** 3, 1000)
    assert dec.engine() is eng and torch.equal(a, b) and not torch.equal(a, base)
