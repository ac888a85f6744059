"""The rendering mirror's post-processing (nphm_b200/evaluation/render_utils.py) against the reference's own, run on the same images
(tests/golden/render.npz, made by tests/golden/make_golden_render.py from the unmodified reference with oracle images), and the
float64 ray caster of oracle/render_oracle.py on scenes with known answers.  CPU only: the native rasterizer is not involved."""
import numpy as np
import torch

from conftest import load_golden


UNIT = np.arange(256) / 255 * 2 - 1          # the reference's u8 / 255 * 2 - 1: the golden stores normals as their uint8 codes


def _foreground(g):
    return np.cumsum(g['img_index_step'].astype(np.int64))


def _images(g):
    V, H, W = (int(x) for x in g['img_shape'])
    depth = np.zeros(V * H * W, np.float32)
    normals = np.zeros((V * H * W, 3), np.uint8)
    depth[_foreground(g)] = g['img_depth']
    normals[_foreground(g)] = g['img_normals']
    return torch.from_numpy(depth.reshape(V, H, W)), torch.from_numpy(normals.reshape(V, H, W, 3))


def test_cameras_match_reference():
    from nphm_b200.evaluation import render_utils as ru
    g = load_golden('render.npz')
    fib = np.array(ru.fibonacci_sphere(12))
    assert np.array_equal(fib, g['fib'])
    look = np.stack([ru.m3dLookAt(np.array(c) * 0.6, np.zeros([3]), np.array([0, 1, 0])) for c in fib[1:-1]])
    assert np.array_equal(look, g['look'])
    cams, poses = ru.render_cameras(10)
    assert np.array_equal(np.array(cams), fib[1:-1][::-1]) and np.array_equal(np.stack(poses), g['look'][::-1])


def test_get_3d_points_matches_reference():
    from nphm_b200.evaluation import render_utils as ru
    g = load_golden('render.npz')
    size = tuple(int(x) for x in g['g_size'])
    got = ru.get_3d_points(g['g_depth'], g['g_K'], g['look'][3], rend_size=size)
    want = g['g_points']
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(want).any()
    ok = ~np.isnan(want)
    assert np.abs(got[ok] - want[ok]).max() < 1e-12


def test_unproject_points_pixel_mapping():
    """unproject_points keeps the reference's /(W - 1), /(H - 1) pixel mapping: it equals get_3d_points row for row."""
    from nphm_b200.evaluation import render_utils as ru
    g = load_golden('render.npz')
    H, W = (int(x) for x in g['g_size'])
    K = g['g_K']
    P = ru.projection_matrix(K[0][0], K[1][1], K[0][2], K[1][2], W, H, 0.1, 2.0)
    xx, yy = np.meshgrid(np.arange(H), np.arange(W))
    ppos = np.stack([xx.reshape(-1), yy.reshape(-1)], axis=-1).astype(np.int32)
    got = ru.unproject_points(ppos, g['g_depth'], (H, W), P, g['look'][3])
    assert np.array_equal(got, ru.get_3d_points(g['g_depth'], K, g['look'][3], rend_size=(H, W)), equal_nan=True)


def test_glcam_post_processing_matches_reference():
    from nphm_b200.evaluation import render_utils as ru
    g = load_golden('render.npz')
    depth, normals = _images(g)
    ndc, nrm = ru.glcam_images(depth[0], normals[0])
    assert ndc.dtype == torch.float32 and nrm.dtype == torch.float64
    H, W = depth.shape[1:]
    fg = _foreground(g)
    fg0 = fg[fg < H * W]
    assert np.array_equal(ndc.reshape(-1)[fg0].numpy(), g['glcam_ndc'])
    assert ndc.reshape(-1)[0].item() == g['glcam_ndc_bg']
    assert np.array_equal(nrm.reshape(-1, 3)[fg0][g['glcam_rows']].numpy(), g['glcam_normals'])


def test_gen_render_samples_post_processing_matches_reference():
    """samples_from_images (everything gen_render_samples does after the render) on the golden's oracle images: same points in
    the same order, identical normals, points within 1e-12."""
    from nphm_b200.evaluation import render_utils as ru
    g = load_golden('render.npz')
    depth, normals = _images(g)
    cams, poses = ru.render_cameras(10)
    pts, nrm = ru.samples_from_images(depth, normals, cams, poses, 4)
    assert pts.shape == (int(g['n_points']), 3) and len(pts) > 20000
    assert np.array_equal(nrm.numpy(), UNIT[g['normal_codes']])
    assert np.abs(pts.numpy()[g['point_rows']] - g['points']).max() < 1e-12


def test_oracle_plane_depth():
    """A plane z = z0 seen head-on: every pixel has depth dist - z0, the normal +z, and an edge distance far from 0."""
    from oracle import render_oracle as O
    H, W = 30, 40
    V = np.array([(-1, -1, -0.5), (1, -1, -0.5), (1, 1, -0.5), (-1, 1, -0.5)])
    F = np.array([(0, 1, 2), (0, 2, 3)])
    w2e = np.hstack([np.eye(3), [[0], [0], [-0.3]]])               # eye at z = 0.3
    out = O.render_view(V, F, w2e, (50.0, 50.0, W / 2, H / 2), H, W)
    assert np.all(out['tri'] >= 0)
    assert np.allclose(out['depth'], 0.8, rtol=0, atol=1e-12)
    assert np.allclose(out['normal'], [0, 0, 1])
    diag = np.abs(np.arange(W)[None, :] + 0.5 - W / 2 - (H / 2 - np.arange(H)[:, None] - 0.5)) < 1e-9
    assert np.all(out['edge_px'][diag] < 1e-6) and np.all(out['edge_px'][~diag] > 0.1)    # the shared diagonal


def test_oracle_sphere_silhouette():
    """A fine sphere: the covered pixels are those whose ray passes within the (inscribed) polyhedron, between the inscribed
    and the circumscribed radius of the true silhouette."""
    from oracle import render_oracle as O
    from render_common import icosphere
    v, f = icosphere(5, radius=0.1)
    H = W = 64
    fx = 200.0
    w2e = np.hstack([np.eye(3), [[0], [0], [-0.6]]])
    out = O.render_view(v, f, w2e, (fx, fx, W / 2, H / 2), H, W)
    c = np.arange(W) + 0.5 - W / 2
    rr = np.hypot(c[None, :], c[:, None]) / fx                        # tan of the ray's angle off the axis
    tan_sil = 0.1 / np.sqrt(0.6 ** 2 - 0.1 ** 2)
    inscribed = 0.1 * np.cos(np.deg2rad(1.2))                          # level-5 icosphere edges span well under 2.4 degrees
    tan_in = inscribed / np.sqrt(0.6 ** 2 - inscribed ** 2)
    assert np.all(out['tri'][rr < tan_in] >= 0) and np.all(out['tri'][rr > tan_sil] < 0)
    d = out['depth'][H // 2, W // 2]
    assert abs(d - 0.5) < 1e-3
