"""GPU parity tests (run with -m gpu on an H100): the CUDA kernels, called through the C ABI
(nphm_b200._native -> libnphm_b200.so), against the oracle and the golden vectors of the reference.
Tolerance 1e-5 abs fp32 (north_star) - the kernels are expected to be ~1e-7."""
import numpy as np
import pytest
import torch

from conftest import (MAXI, MINI, load_golden, make_deformation, make_ensemble, make_npm, sample_latent, sd_numpy)
from oracle import nphm_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _impls():
    from nphm_b200 import _native
    return ['simt', 'tc']


def _engine_or_skip(dec, impl):
    from nphm_b200 import _native
    eng = dec.engine()
    return eng


@pytest.mark.parametrize('impl', ['simt', 'tc'])
@pytest.mark.parametrize('tag,seed,scale', [('a', 0, 1.0), ('b', 5, 2.0)])
def test_ensemble_query_matches_reference_golden(cuda_device, impl, tag, seed, scale):
    g = load_golden('ensemble.npz')
    dec = make_ensemble(seed, scale, device=cuda_device)
    x = torch.from_numpy(g['points_' + tag]).to(cuda_device).unsqueeze(0)
    lat = torch.from_numpy(g['latent_' + tag]).to(cuda_device).reshape(1, -1)
    eng = dec.engine()
    s_eval, anc = eng.query(x, lat, eval_quirk=True, impl=impl)
    s_train, _ = eng.query(x, lat, eval_quirk=False, impl=impl)
    assert np.abs(anc.cpu().numpy()[0] - g['anchors_' + tag]).max() < 1e-6
    e1 = np.abs(s_eval.cpu().numpy().reshape(-1) - g['sdf_eval_' + tag]).max()
    e2 = np.abs(s_train.cpu().numpy().reshape(-1) - g['sdf_train_' + tag]).max()
    print('ensemble %s %s max abs err eval %.3g train %.3g' % (impl, tag, e1, e2))
    assert e1 < TOL and e2 < TOL


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_ensemble_matches_oracle_on_seeded_inputs(cuda_device, impl):
    """Ragged sizes (not a multiple of the tile), batch of 3 queries with different latents, zero latent."""
    dec = make_ensemble(3, 1.5, device=cuda_device)
    p = O.EnsembleParams(sd_numpy(dec), load_golden('assets.npz')['anchors_39'])
    rng = np.random.RandomState(11)
    for n in (1, 37, 129, 1000):
        pts = (rng.rand(3, n, 3) * (np.array(MAXI) - np.array(MINI)) + np.array(MINI)).astype(np.float32)
        lats = np.stack([sample_latent(21).numpy() * 5, np.zeros(1344, np.float32), sample_latent(22).numpy() * 10])
        sdf, anc = dec.engine().query(torch.from_numpy(pts).to(cuda_device), torch.from_numpy(lats).to(cuda_device),
                                      eval_quirk=True, impl=impl)
        for b in range(3):
            ref, ref_anc = O.ensemble_forward(p, pts[b], lats[b], eval_mode=True)
            assert np.abs(anc[b].cpu().numpy() - ref_anc).max() < 1e-6
            err = np.abs(sdf[b].cpu().numpy().reshape(-1) - ref).max()
            assert err < TOL, (n, b, err)


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_module_forward_and_get_logits_dropin(cuda_device, impl, monkeypatch):
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    monkeypatch.setenv('NPHM_B200_IMPL', impl)
    g = load_golden('ensemble.npz')
    dec = make_ensemble(0, device=cuda_device).eval()
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, 20)).to(cuda_device, dtype=torch.float)
    grid = grid.reshape(1, -1, 3)
    lat = torch.from_numpy(g['latent_a']).to(cuda_device)
    logits, anchors = get_logits(dec, lat, grid, nbatch_points=3000, return_anchors=True)
    assert logits.shape == (8000,) and logits.dtype == np.float32 and anchors.shape == (1, 39, 3)
    assert np.abs(logits - g['logits20_a']).max() < TOL
    # plain module call under no_grad: B x N x lat (materialised repeat, like the reference's get_logits does)
    with torch.no_grad():
        s, a = dec(grid[:, :777], lat.reshape(1, 1, -1).repeat(1, 777, 1), None)
    assert s.shape == (1, 777, 1)
    ref, _ = O.ensemble_forward(O.EnsembleParams(sd_numpy(dec), load_golden('assets.npz')['anchors_39']),
                                grid[0, :777].cpu().numpy(), g['latent_a'], eval_mode=True)
    assert np.abs(s.cpu().numpy().reshape(-1) - ref).max() < TOL
    # weights updated in place -> engine repacks
    with torch.no_grad():
        dec.ensembled_deep_sdf.lin4.bias.add_(0.25)
        s2, _ = dec(grid[:, :777], lat.reshape(1, 1, -1), None)
    ref2, _ = O.ensemble_forward(O.EnsembleParams(sd_numpy(dec), load_golden('assets.npz')['anchors_39']),
                                 grid[0, :777].cpu().numpy(), g['latent_a'], eval_mode=True)
    assert np.abs(ref2 - ref).max() > 0.1
    assert np.abs(s2.cpu().numpy().reshape(-1) - ref2).max() < TOL


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_grid_query_equals_explicit_points_and_shards(cuda_device, impl):
    """In-kernel grid generation == float32(np.linspace) points; shards of the flat index range agree with the
    whole (quirk positions follow the GLOBAL index)."""
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds
    dec = make_ensemble(0, device=cuda_device).eval()
    lat = sample_latent(1).to(cuda_device)
    res = 24
    total = res ** 3
    eng = dec.engine()
    whole, _ = eng.query_grid(lat, MINI, MAXI, res, 0, total, quirk_period=2500, impl=impl)
    pts = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(cuda_device, dtype=torch.float)
    explicit, _ = eng.query(pts.reshape(1, -1, 3), lat.reshape(1, -1), eval_quirk=True, quirk_period=2500, impl=impl)
    assert torch.equal(whole, explicit.reshape(-1))
    parts = []
    bounds = [0, 5000, 5001, 9999, total]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        part, _ = eng.query_grid(lat, MINI, MAXI, res, lo, hi - lo, quirk_period=2500, impl=impl)
        parts.append(part)
    assert torch.equal(torch.cat(parts), whole)


def test_tc_and_simt_kernels_agree(cuda_device):
    dec = make_ensemble(0, device=cuda_device).eval()
    lat = sample_latent(1).to(cuda_device)
    eng = dec.engine()
    a, _ = eng.query_grid(lat, MINI, MAXI, 40, 0, 40 ** 3, quirk_period=25000, impl='simt')
    b, _ = eng.query_grid(lat, MINI, MAXI, 40, 0, 40 ** 3, quirk_period=25000, impl='tc')
    err = (a - b).abs().max().item()
    print('tc vs simt max abs diff %.3g' % err)
    assert err < 2e-6


def test_deformation_and_npm_match_reference_golden(cuda_device):
    d = load_golden('deform.npz')
    dfn = make_deformation(cuda_device)
    pts = torch.from_numpy(d['points']).to(cuda_device).unsqueeze(0)
    cond = torch.cat([torch.from_numpy(d['latent_id']), torch.from_numpy(d['z_ex'])]).reshape(1, 1, -1).to(cuda_device)
    anc = torch.from_numpy(d['anchors']).to(cuda_device).unsqueeze(0)
    with torch.no_grad():
        off, last = dfn(pts, cond, anc)
        off_rep, _ = dfn(pts, cond.repeat(1, pts.shape[1], 1), anc.unsqueeze(1).repeat(1, pts.shape[1], 1, 1))
    assert off.shape == (1, pts.shape[1], 3) and last.shape == (1, pts.shape[1], 1)
    err = np.abs(off.cpu().numpy()[0] - d['offsets']).max()
    print('deformation max abs err %.3g' % err)
    assert err < TOL and torch.equal(off, off_rep)
    assert np.abs(last.cpu().numpy().reshape(-1) - d['last']).max() < TOL
    npm = make_npm(cuda_device)
    with torch.no_grad():
        out, none = npm(pts, torch.from_numpy(d['z_npm']).to(cuda_device).reshape(1, 1, -1))
    assert none is None and np.abs(out.cpu().numpy().reshape(-1) - d['npm_out']).max() < TOL
    # oracle on a ragged batch of 2 queries
    rng = np.random.RandomState(5)
    x = (rng.rand(2, 333, 3) - 0.5).astype(np.float32)
    c = (rng.randn(2, 64) * 0.1).astype(np.float32)
    got = npm.engine().query(torch.from_numpy(x).to(cuda_device), torch.from_numpy(c).to(cuda_device)).cpu().numpy()
    mp = O.MlpParams(sd_numpy(npm))
    for b in range(2):
        assert np.abs(got[b] - O.mlp_forward(mp, x[b], c[b])).max() < TOL


def test_deform_mesh_dropin(cuda_device):
    from nphm_b200.models.reconstruction import deform_mesh
    from nphm_b200.utils.mesh import SimpleMesh
    d = load_golden('deform.npz')
    dfn = make_deformation(cuda_device)
    mesh = SimpleMesh(d['points'].astype(np.float64), np.array([[0, 1, 2], [2, 3, 4]]))
    out = deform_mesh(mesh, dfn, torch.from_numpy(d['z_ex']).to(cuda_device).reshape(1, 1, -1),
                      torch.from_numpy(d['anchors']).to(cuda_device).unsqueeze(0),
                      lat_rep_shape=torch.from_numpy(d['latent_id']).to(cuda_device).reshape(1, 1, -1))
    assert np.abs(np.asarray(out.vertices) - (d['points'] + d['offsets'])).max() < 2e-5
    assert np.array_equal(np.asarray(out.faces), mesh.faces)


def test_tensor_core_operand_plumbing(cuda_device):
    """D = A * B^T through the wgmma operand path (fp16 hi/lo split, A in registers, B slabs in shared memory)."""
    import ctypes
    from nphm_b200 import _native
    lib = _native.lib()
    lib.nphm_debug_tc_mma.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_void_p, ctypes.c_void_p]
    rng = np.random.RandomState(0)
    for n, ks in ((112, 13), (208, 7), (208, 13), (16, 1)):
        a = (rng.randn(128, 16 * ks) * 3).astype(np.float32)
        b = (rng.randn(n, 16 * ks) * 0.1).astype(np.float32)
        ref = a.astype(np.float64) @ b.astype(np.float64).T
        ad, bd = torch.from_numpy(a).to(cuda_device), torch.from_numpy(b).to(cuda_device)
        errs = {}
        for variant in range(4):
            d = torch.zeros(128, n, device=cuda_device)
            _native.check(lib.nphm_debug_tc_mma(ad.data_ptr(), bd.data_ptr(), n, ks, variant, d.data_ptr(), None))
            errs[variant] = float(np.abs(d.cpu().numpy() - ref).max())
        print('tc operand self-test n=%d ks=%d: max abs err by layout variant %s' % (n, ks, errs))
        assert errs[0] < 2e-5 * max(1.0, np.abs(ref).max()), errs


def test_pruned_kernel_is_opt_in_and_within_its_error_bound(cuda_device):
    """NPHM_IMPL_TC_PRUNED skips members with negligible blend weight: not bit-identical to the dense kernel, but
    within n_members * tau * max|s_k| of it (and of the reference)."""
    g = load_golden('ensemble.npz')
    for tag, seed, scale in (('a', 0, 1.0), ('b', 5, 2.0)):
        dec = make_ensemble(seed, scale, device=cuda_device).eval()
        lat = torch.from_numpy(g['latent_' + tag]).to(cuda_device)
        eng = dec.engine()
        for res, first, count in ((40, 0, 40 ** 3), (33, 33 * 33 * 5 + 7, 33 * 33 * 9 + 100)):
            dense, _ = eng.query_grid(lat, MINI, MAXI, res, first, count, quirk_period=2500, impl='tc')
            for tau in (1e-8, 1e-6):
                eng.set_prune_threshold(tau)
                pruned, _ = eng.query_grid(lat, MINI, MAXI, res, first, count, quirk_period=2500, impl='tc_pruned')
                err = (dense - pruned).abs().max().item()
                print('pruned %s res %d tau %g: max abs diff vs dense %.3g' % (tag, res, tau, err))
                assert err < 40 * tau * 1.0 + 2e-7
        eng.set_prune_threshold(1e-8)
        x = torch.from_numpy(g['points_' + tag]).to(cuda_device).unsqueeze(0)
        s, _ = eng.query(x, lat.reshape(1, -1), eval_quirk=True, impl='tc_pruned')       # explicit points (no blocks)
        assert np.abs(s.cpu().numpy().reshape(-1) - g['sdf_eval_' + tag]).max() < TOL


def test_deformation_tensor_core_kernel(cuda_device):
    """Tensor-core MLP path (layer chain on the wgmma linear layer) against the reference golden, the oracle and the FFMA kernel."""
    d = load_golden('deform.npz')
    dfn = make_deformation(cuda_device)
    eng = dfn.defDeepSDF.engine()
    pts = torch.from_numpy(d['points']).to(cuda_device).unsqueeze(0)
    cond_id = torch.cat([torch.from_numpy(d['latent_id']), torch.from_numpy(d['z_ex'])]).reshape(1, 1, -1).to(cuda_device)
    anc = torch.from_numpy(d['anchors']).to(cuda_device).unsqueeze(0)
    with torch.no_grad():
        cond = dfn._condition(pts, cond_id, anc, per_point=False)[:, 0]
    tc = eng.query(pts, cond, impl='tc')
    simt = eng.query(pts, cond, impl='simt')
    e_gold = np.abs(tc.cpu().numpy()[0] - d['offsets']).max()
    e_simt = (tc - simt).abs().max().item()
    print('deformation tc: max abs err vs reference golden %.3g, vs FFMA kernel %.3g' % (e_gold, e_simt))
    assert e_gold < TOL and e_simt < 2e-6
    # ragged sizes and a batch of queries with different conditions
    rng = np.random.RandomState(3)
    mp = O.MlpParams(sd_numpy(dfn), prefix='defDeepSDF.')
    for n in (1, 63, 64, 65, 1000):
        x = (rng.rand(2, n, 3) - 0.5).astype(np.float32)
        c = (rng.randn(2, 232) * 0.3).astype(np.float32)
        got = eng.query(torch.from_numpy(x).to(cuda_device), torch.from_numpy(c).to(cuda_device), impl='tc').cpu().numpy()
        for b in range(2):
            assert np.abs(got[b] - O.mlp_forward(mp, x[b], c[b])).max() < TOL, n


def test_deformation_forward_streams_rows_in_chunks(cuda_device):
    """The tensor-core forward runs in bounded chunks of 65 536 rows: queries longer than a chunk (ragged last chunk) and
    several short queries per chunk give what the FFMA kernel gives on the whole call."""
    dfn = make_deformation(cuda_device)
    eng = dfn.defDeepSDF.engine()
    rng = np.random.RandomState(4)
    for B, n in ((2, 70001), (3, 30000)):
        x = torch.from_numpy((rng.rand(B, n, 3) - 0.5).astype(np.float32)).to(cuda_device)
        c = torch.from_numpy((rng.randn(B, 232) * 0.3).astype(np.float32)).to(cuda_device)
        tc = eng.query(x, c, impl='tc')
        simt = eng.query(x, c, impl='simt')
        err = (tc - simt).abs().max().item()
        print('chunked deformation forward B=%d n=%d: max abs diff vs FFMA kernel %.3g' % (B, n, err))
        assert err < 2e-6


# ---------------------------------------------------------------------------------------------- layer chain (tc_linear)
def _chain_case(kind, device):
    from nphm_b200.models.deepSDF import DeepSDF
    if kind == 'deform':
        dfn = make_deformation(device)
        return dfn.defDeepSDF, 232, 3
    torch.manual_seed(12)
    if kind == 'npm':          # scripts/configs/npm.yaml:2-4: lat 512, hidden 1024, 8 layers
        return DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True).to(device), 512, 1
    return DeepSDF(lat_dim=40, hidden_dim=96, nlayers=5, geometric_init=False, out_dim=3).to(device), 40, 3


@pytest.mark.parametrize('kind', ['deform', 'npm', 'small'])
def test_layer_chain_forward_jacobian_adjoint_match_autograd(cuda_device, kind):
    """nphm_mlp_query_layers / nphm_mlp_jacobian / nphm_mlp_backward_inputs (generic wgmma linear layer) against the
    reference-pinned composite module under torch autograd: values <= 1e-5, Jacobian and gradients <= 2e-4 relative (5e-4 for
    the 8 x 1024 NPM stack, whose fp32 autograd reference itself carries that much round-off)."""
    net, lat_dim, out_dim = _chain_case(kind, cuda_device)
    torch.manual_seed(3)
    B, N = 2, 333
    xyz = (torch.rand(B, N, 3, device=cuda_device) - 0.5) * 0.8
    cond = torch.randn(B, lat_dim, device=cuda_device) * (0.05 if kind != 'npm' else 0.2)
    eng = net.engine()
    xa = xyz.clone().requires_grad_(True)
    ca = cond.clone().requires_grad_(True)
    ref = net._forward_composite(xa, ca[:, None, :])
    got = eng.query_layers(xyz, cond)
    err = float((got - ref.detach()).abs().max())
    print('%s chain forward max abs err %.3g (|out| max %.3g)' % (kind, err, float(ref.detach().abs().max())))
    assert err < TOL
    out, J = eng.jacobian(xyz, cond)
    assert float((out - ref.detach()).abs().max()) < TOL
    rows = [torch.autograd.grad(ref[..., i].sum(), xa, retain_graph=True)[0] for i in range(out_dim)]
    J_ref = torch.stack(rows, dim=-2)
    jerr = float((J - J_ref).abs().max() / J_ref.abs().max())
    rtol = 5e-4 if kind == 'npm' else 2e-4
    print('%s chain Jacobian rel err %.3g' % (kind, jerr))
    assert jerr < rtol
    up = torch.randn(B, N, out_dim, device=cuda_device)
    g_c_ref, g_x_ref = torch.autograd.grad((ref * up).sum(), [ca, xa])
    g_c, g_x = eng.backward_inputs(xyz, cond, up, want_xyz=True)
    cerr = float((g_c - g_c_ref).abs().max() / g_c_ref.abs().max())
    xerr = float((g_x - g_x_ref).abs().max() / g_x_ref.abs().max())
    print('%s chain adjoint rel err: cond %.3g xyz %.3g' % (kind, cerr, xerr))
    assert cerr < rtol and xerr < rtol


def test_npm_width_deepsdf_matches_reference_golden(cuda_device):
    """NPM baseline DeepSDF 515 -> 1024 x 8 -> 1 (scripts/configs/npm.yaml:2-4) through the module forward: it runs on the
    tensor-core layer chain (no fused kernel takes that width, no eager PyTorch either) and must match the golden produced
    by the unmodified reference (tests/golden/make_golden_npm.py)."""
    import hashlib
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('npm.npz')
    torch.manual_seed(12)
    net = DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True)
    h = hashlib.sha256()
    sd = net.state_dict()
    for k in sorted(sd):
        h.update(k.encode()); h.update(np.ascontiguousarray(sd[k].numpy()).tobytes())
    assert h.hexdigest() == str(g['sha256'])                 # same initialisation as the reference class
    net = net.to(cuda_device)
    pts = torch.from_numpy(g['points']).to(cuda_device)
    codes = torch.from_numpy(g['codes']).to(cuda_device)
    with torch.no_grad():
        assert net._fused_ok(pts, codes[:, None, :])
        out, none = net(pts, codes[:, None, :].repeat(1, pts.shape[1], 1))
    assert none is None and out.shape == (2, 700, 1)
    err = float((out.cpu() - torch.from_numpy(g['sdf'])).abs().max())
    print('NPM 1024 x 8 on the layer chain: max abs err vs reference golden %.3g' % err)
    assert err < TOL
    torch.manual_seed(14)
    net2 = DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=False, out_dim=3).to(cuda_device)
    with torch.no_grad():
        out2, _ = net2(pts, (codes * 5.0)[:, None, :].repeat(1, pts.shape[1], 1))
    err2 = float((out2.cpu() - torch.from_numpy(g['out_plain'])).abs().max())
    print('plain-init 1024 x 8, 3 outputs: max abs err %.3g (range of the golden %.3g)' % (err2, float(np.ptp(g['out_plain']))))
    assert err2 < TOL


def test_generic_linear_layer_packed_blocked_batched(cuda_device):
    """tc_linear.cu through its test entry: three chained layers per batch entry - row-major in -> packed -> (x blocked
    multiplier, streamed through the shared-memory ring) -> packed -> row-major out - batched over entries that share weight
    sets pairwise, rows not a multiple of the 128-row tile.  Against float64 torch."""
    import ctypes
    from nphm_b200 import _native
    lib = _native.lib()
    rng = np.random.RandomState(3)
    batch, pairs, M, K, N1, N2, N3 = 5, 2, 300, 40, 200, 101, 24
    sets = batch - pairs
    a = torch.from_numpy(rng.randn(batch, M, K).astype(np.float32)).to(cuda_device)
    w1 = torch.from_numpy((rng.randn(sets, N1, K) / np.sqrt(K)).astype(np.float32)).to(cuda_device)
    w2 = torch.from_numpy((rng.randn(sets, N2, N1) / np.sqrt(N1)).astype(np.float32)).to(cuda_device)
    w3 = torch.from_numpy((rng.randn(sets, N3, N2) / np.sqrt(N2)).astype(np.float32)).to(cuda_device)
    mul = torch.from_numpy(rng.rand(batch, M, N2).astype(np.float32)).to(cuda_device)
    tiles, ldm = (M + 127) // 128, (N2 + 3) // 4 * 4
    blocked = torch.zeros(batch, tiles, ldm, 128, device=cuda_device)
    padded = torch.zeros(batch, tiles * 128, N2, device=cuda_device)
    padded[:, :M] = mul
    blocked[:, :, :N2, :] = padded.reshape(batch, tiles, 128, N2).permute(0, 1, 3, 2)
    z = torch.empty(batch, M, N3, device=cuda_device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(cuda_device).cuda_stream)
    lib.nphm_debug_linear_chain.restype = ctypes.c_int
    lib.nphm_debug_linear_chain.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int, ctypes.c_int, ctypes.c_longlong] + \
        [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_void_p]
    rc = lib.nphm_debug_linear_chain(a.data_ptr(), w1.data_ptr(), w2.data_ptr(), w3.data_ptr(), blocked.data_ptr(), batch, pairs,
                                     M, K, N1, N2, N3, z.data_ptr(), stream)
    assert rc == 0, _native.last_error() if hasattr(_native, 'last_error') else rc
    torch.cuda.synchronize()
    worst = 0.0
    for b in range(batch):
        s = b // 2 if b < 2 * pairs else b - pairs
        h1 = a[b].double() @ w1[s].double().T
        h2 = (h1 @ w2[s].double().T) * mul[b].double()
        want = h2 @ w3[s].double().T
        err = float((z[b].double() - want).abs().max() / want.abs().max())
        worst = max(worst, err)
    print('generic linear layer chain (packed / blocked / batched): max rel err %.2e' % worst)
    assert worst < 5e-6            # three chained fp32-accurate layers (3-pass fp16 split: ~2^-22 per product)
