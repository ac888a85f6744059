"""GPU tests of the native depth / normal rasterizer (csrc/render.cu, nphm_render_depth_normals) and of the evaluation mirror
built on it (nphm_b200/evaluation/render_utils.py, sampling.py).

The rasterizer is checked against the float64 ray caster of oracle/render_oracle.py: the triangle index must agree on every pixel
whose centre lies more than 1e-4 px from a triangle boundary and whose winning depth does not tie the runner-up's to 1e-6
(relative); where it agrees, depth to 1e-6 relative and the uint8 normal exactly, unless 0.5 n + 0.5 lies within 1e-4 of a
rounding boundary."""
import numpy as np
import pytest
import torch

from conftest import MAXI, MINI, load_golden, make_ensemble, sample_latent
from render_common import adversarial_scene, icosphere, intrinsics_for, look_at_views

pytestmark = pytest.mark.gpu

SMALL = (320, 240)
FULL = (1280, 960)


def _native(v, f, w2e, intr, H, W, dev, want_tri=True):
    from nphm_b200 import _native
    d, n, t = _native.render_depth_normals(torch.from_numpy(np.asarray(v, np.float32)).to(dev), torch.from_numpy(np.asarray(f)).to(dev),
                                           torch.from_numpy(w2e), torch.from_numpy(intr), H, W, want_tri=want_tri)
    return d.cpu().numpy(), n.cpu().numpy(), None if t is None else t.cpu().numpy()


def _compare(v, f, w2e, intr, H, W, dev, subset=None, seed=0):
    from oracle import render_oracle as O
    d, n, t = _native(v, f, w2e, intr, H, W, dev)
    ref = O.render(v, f, w2e, intr, H, W)
    sel = np.ones(d.shape, bool)
    if subset:
        sel = np.zeros(d.size, bool)
        sel[np.random.RandomState(seed).choice(d.size, subset, replace=False)] = True
        sel = sel.reshape(d.shape)
    tie = np.abs(ref['second'] - ref['depth']) <= 1e-6 * ref['depth']
    strict = sel & (ref['edge_px'] > 1e-4) & ~tie
    assert np.array_equal(t[strict], ref['tri'][strict]), 'triangle index differs on %d of %d unambiguous pixels' % (
        int((t[strict] != ref['tri'][strict]).sum()), int(strict.sum()))
    agree = sel & (t == ref['tri']) & (t >= 0)
    assert np.all(np.abs(d[agree] - ref['depth'][agree]) <= 1e-6 * ref['depth'][agree])
    assert np.all(d[sel & (t < 0)] == 0) and np.all(n[sel & (t < 0)] == 0)
    g = 0.5 * ref['normal'][agree] + 0.5
    frac = g * 255 - np.floor(g * 255)
    clear = np.all(np.abs(frac - 0.5) * 1.0 / 255 > 1e-4, axis=-1)
    assert np.array_equal(n[agree][clear], O.quantize_normals(ref['normal'][agree][clear]))
    assert (t >= 0).any() and strict.sum() > 0.9 * sel.sum()
    return d, n, t, ref


def _cams():
    from nphm_b200.evaluation.render_utils import render_cameras
    cams, _ = render_cameras(10)
    return cams


@pytest.fixture(scope='module')
def head_mesh(cuda_device):
    """The golden ensemble's zero level set at 64^3, scaled by 1/4 as gen_render_samples scales a mesh."""
    from nphm_b200.models.reconstruction import get_logits
    from nphm_b200.utils.reconstruction import create_grid_points_from_bounds, mesh_from_logits
    dec = make_ensemble(0, device=cuda_device).eval()
    lat = sample_latent(1).to(cuda_device)
    res = 64
    grid = torch.from_numpy(create_grid_points_from_bounds(MINI, MAXI, res)).to(cuda_device, dtype=torch.float).reshape(1, -1, 3)
    mesh = mesh_from_logits(get_logits(dec, lat, grid, nbatch_points=100000), MINI, MAXI, res)
    v, f = np.asarray(mesh.vertices) / 4, np.asarray(mesh.faces).astype(np.int64)
    assert len(f) > 1000
    return v, f


def test_head_ten_views_against_oracle(cuda_device, head_mesh):
    v, f = head_mesh
    H, W = SMALL
    _compare(v, f, look_at_views(_cams()), intrinsics_for(H, W, 10), H, W, cuda_device)


def test_head_full_size_against_oracle(cuda_device, head_mesh):
    v, f = head_mesh
    H, W = FULL
    _compare(v, f, look_at_views(_cams()[:1]), intrinsics_for(H, W, 1), H, W, cuda_device, subset=20000)


def test_sphere_against_oracle_and_watertight(cuda_device):
    from scipy.ndimage import binary_erosion
    v, f = icosphere(5, radius=0.12, center=(0.01, -0.02, 0.015))
    H, W = SMALL
    d, n, t, ref = _compare(v, f, look_at_views(_cams()), intrinsics_for(H, W, 10), H, W, cuda_device)
    for i in range(10):
        fg_ref = ref['tri'][i] >= 0
        inner = binary_erosion(fg_ref, iterations=1)
        outer = binary_erosion(~fg_ref, iterations=1)
        assert np.all(t[i][inner] >= 0), 'hole in a closed mesh'
        assert np.all(t[i][outer] < 0)


def test_shared_edges_through_pixel_centres_leave_no_hole(cuda_device):
    """A grid of triangles whose edges run exactly through pixel centres (axis-aligned and diagonal), with both windings and
    shuffled face order, and a jittered version with generic shared edges: every pixel of the grid is covered, those on its
    outer boundary included (the edge test is inclusive), and nothing outside."""
    H, W = 40, 48
    rng = np.random.RandomState(3)
    n = 16
    xs = np.arange(n + 1) - n / 2 + 0.5                      # half-integers: pixel-centre rays at z = -1 with f = 1, cx = W/2
    X, Y = np.meshgrid(xs, xs)
    for jitter in (0.0, 0.3):
        P = np.stack([X, Y, -np.ones_like(X)], -1)
        P[1:-1, 1:-1, :2] += rng.uniform(-jitter, jitter, (n - 1, n - 1, 2))     # the border stays on the grid
        P = P.reshape(-1, 3)
        F = []
        for i in range(n):
            for j in range(n):
                a, b, c, dd = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j + 1, (i + 1) * (n + 1) + j
                tri = [(a, b, c), (a, c, dd)] if (i + j) % 2 else [(a, b, dd), (b, c, dd)]
                F += [t[::-1] if rng.rand() < 0.5 else t for t in tri]
        F = np.array(F)[rng.permutation(len(F))]
        P = P * rng.choice([0.5, 0.75, 1.0, 1.25, 1.5], (len(P), 1))   # same rays (exactly: few mantissa bits), other depths
        w2e = np.hstack([np.eye(3), np.zeros((3, 1))])[None]
        intr = np.array([[1.0, 1.0, W / 2, H / 2]])
        d, _, t = _native(P, F, w2e, intr, H, W, cuda_device)
        lo, hi = -n / 2 + 0.5, n / 2 + 0.5
        r = np.arange(H)[:, None]; c = np.arange(W)[None, :]
        x, y = c + 0.5 - W / 2 + 0 * r, H / 2 - r - 0.5 + 0 * c
        inside = (x >= lo) & (x <= hi) & (y >= lo) & (y <= hi)
        assert np.all(t[0][inside] >= 0), 'jitter %g: %d holes' % (jitter, int((t[0][inside] < 0).sum()))
        assert np.all(t[0][~inside] < 0)


def test_adversarial_scene_against_oracle(cuda_device):
    """Full-viewport quad behind an object, a triangle through the near plane and the eye plane, one beyond zfar, one behind the
    eye, zero-area triangles, both windings and coplanar duplicates; head-on at 1280 x 960 (20 k pixels checked) and from the 10
    gen_render_samples cameras at reduced size."""
    ov, of = icosphere(3, radius=0.05)
    v, f = adversarial_scene(ov, of)
    w2e = np.hstack([np.eye(3), [[0], [0], [-0.6]]])[None]
    H, W = FULL
    d, n, t, ref = _compare(v, f, w2e, intrinsics_for(H, W, 1), H, W, cuda_device, subset=20000)
    assert (t == len(of)).any() or (t == len(of) + 1).any()               # the quad is visible
    assert not np.isin(t, np.arange(len(f) - 8, len(f) - 6)).any()       # the zero-area triangles never win
    H, W = SMALL
    _compare(v, f, look_at_views(_cams()), intrinsics_for(H, W, 10), H, W, cuda_device)


def test_deterministic_and_batch_invariant(cuda_device):
    ov, of = icosphere(3, radius=0.05)
    v, f = adversarial_scene(ov, of)
    cams = _cams()
    w2e = np.concatenate([np.hstack([np.eye(3), [[0], [0], [-0.6]]])[None], look_at_views(cams)])
    H, W = SMALL
    intr = intrinsics_for(H, W, len(w2e))
    a = _native(v, f, w2e, intr, H, W, cuda_device)
    b = _native(v, f, w2e, intr, H, W, cuda_device)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for i in range(len(w2e)):
        s = _native(v, f, w2e[i:i + 1], intr[i:i + 1], H, W, cuda_device)
        for x, y in zip(a, s):
            assert np.array_equal(x[i], y[0])


def test_gen_render_samples_end_to_end(cuda_device, head_mesh):
    """gen_render_samples on the GPU == the CPU post-processing of the native images copied to the host."""
    from nphm_b200.evaluation import render_utils as ru
    from nphm_b200.utils.mesh import SimpleMesh
    v, f = head_mesh
    mesh = SimpleMesh(v * 4, f)
    pts, nrm = ru.gen_render_samples(mesh, 10)
    cams, poses = ru.render_cameras(10)
    depth, normals = ru.render_views((np.asarray(mesh.vertices) / 4).astype(np.float32), f, poses, ru.KK, FULL)
    want_p, want_n = ru.samples_from_images(depth.cpu(), normals.cpu(), cams, poses, 4)
    assert pts.shape == tuple(want_p.shape) and len(pts) > 10000
    assert np.array_equal(nrm, want_n.numpy())
    assert np.abs(pts - want_p.numpy()).max() < 1e-12
    ndc, nrm0 = ru.render_glcam(SimpleMesh(v, f), ru.KK, poses[0], rend_size=FULL)
    ref_ndc, ref_n = ru.glcam_images(depth[0].cpu(), normals[0].cpu())
    assert np.array_equal(ndc, ref_ndc.numpy()) and np.array_equal(nrm0, ref_n.numpy())


def test_sample_surface_points_matches_reference(cuda_device, monkeypatch):
    """sample_surface_points with the golden's oracle images in place of the native render: the reference's seeded draws."""
    from nphm_b200.evaluation import render_utils as ru
    from nphm_b200.evaluation import sampling
    from nphm_b200.utils.mesh import SimpleMesh
    from test_render_cpu import _images
    g = load_golden('render.npz')
    depth, normals = _images(g)
    monkeypatch.setattr(ru, 'render_views', lambda *a, **k: (depth.to(cuda_device), normals.to(cuda_device)))
    fv, fn = np.zeros((5023, 3)), np.zeros((5023, 3))
    fv[g['flame_rows']], fn[g['flame_rows']] = g['flame_verts'], g['flame_normals']
    flame = SimpleMesh(fv, np.zeros((0, 3), np.int64))
    flame.vertex_normals = fn
    mesh = SimpleMesh(*icosphere(4, radius=0.025, bumps=0.25))       # the golden's fixture; its render is the injected images
    pts, pts_n = ru.gen_render_samples(mesh, 10)
    assert len(pts) == int(g['n_points']) and np.abs(pts[g['point_rows']] - g['points']).max() < 1e-12
    samps, samps_n = sampling.slice_properly(flame, pts, extra=pts_n)
    assert len(samps) == int(g['n_samps'])
    valids = sampling.face_region_mask(samps, flame, g['face_idx'])
    want = np.unpackbits(g['valids'], count=len(samps)).astype(bool)
    assert (valids == want).mean() > 0.999                      # fp32 nearest-neighbour ties may pick the other vertex
    np.random.seed(int(g['seed']))
    p, n, pf, nf = sampling.sample_surface_points(mesh, flame, g['face_idx'], int(g['num_samps']))
    assert np.array_equal(p, samps[g['s_idx']]) and np.array_equal(n, samps_n[g['s_idx']])
    assert np.abs(p[:200] - g['s_points']).max() < 1e-12
    if np.array_equal(valids, want):
        assert np.array_equal(pf, samps[valids][g['s_idx_face']]) and np.array_equal(nf, samps_n[valids][g['s_idx_face']])
        assert np.abs(pf[:200] - g['s_points_face']).max() < 1e-12


def test_errors(cuda_device):
    from nphm_b200 import _native
    v = torch.rand(4, 3, device=cuda_device)
    w2e = torch.from_numpy(np.hstack([np.eye(3), [[0], [0], [-0.6]]])[None])
    intr = torch.tensor([[100.0, 100.0, 8.0, 8.0]], dtype=torch.float64)
    for bad in ([[0, 1, 4]], [[0, -1, 2]]):
        with pytest.raises(ValueError):
            _native.render_depth_normals(v, torch.tensor(bad), w2e, intr, 16, 16)
    d, n, t = _native.render_depth_normals(v, torch.zeros(0, 3, dtype=torch.int64), w2e, intr, 16, 16, want_tri=True)
    assert bool((d == 0).all()) and bool((n == 0).all()) and bool((t == -1).all())
    for H, W in ((0, 16), (16, 0)):
        with pytest.raises(_native.NativeError):
            _native.render_depth_normals(v, torch.tensor([[0, 1, 2]]), w2e, intr, H, W)
    L = _native.lib()
    need = L.nphm_render_workspace_bytes(1, 16, 16)
    assert need > 0 and L.nphm_render_workspace_bytes(0, 16, 16) == -1
    f = torch.tensor([[0, 1, 2]], dtype=torch.int32, device=cuda_device)
    w, k = w2e.reshape(-1).to(cuda_device), intr.reshape(-1).to(cuda_device)
    depth = torch.empty(16 * 16, dtype=torch.float32, device=cuda_device)
    normals = torch.empty(16 * 16 * 3, dtype=torch.uint8, device=cuda_device)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda_device)
    args = lambda nbytes: (v.data_ptr(), 4, f.data_ptr(), 1, w.data_ptr(), k.data_ptr(), 1, 0.1, 2.0, 16, 16,   # noqa: E731
                           depth.data_ptr(), normals.data_ptr(), None, ws.data_ptr(), nbytes, None)
    assert L.nphm_render_depth_normals(*args(need - 1)) == -4                              # NPHM_ERR_CAPACITY
    assert L.nphm_render_depth_normals(*args(need)) == 0
    torch.cuda.synchronize()
