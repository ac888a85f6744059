"""Shared by tests/test_train_ensemble_cpu.py and tests/golden/make_golden_train_ensemble.py: the seeded batch of the golden
train_ensemble.npz (one stage-1 step of the NPHM ensemble at nphm.yaml size), the nphm.yaml lambdas and the gradients the
golden records."""
import numpy as np

# scripts/configs/nphm.yaml: lambdas of the stage-1 loss
LAMBDAS = {'surf_sdf': 2.0, 'normals': 0.3, 'space_sdf': 0.01, 'grad': 0.1, 'lat_reg': 0.01, 'anchors': 7.5,
           'symm_dist': 0.01, 'middle_dist': 0.0}
POINT_SETS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far')
BATCH_KEYS = POINT_SETS + ('normals_face', 'normals_non_face', 'gt_anchors')
SIZES = (40, 16, 40, 20)          # points per set and batch element
N_ENSEMBLE_LAYERS = 5
# no stored point has |s| below this: there the sign in the gradients of surf_sdf and space_sdf is not resolved in fp32
MIN_ABS_SDF = 1e-4


def make_batch(mean_anchors, sizes, B=2, seed=3):
    """Points centred on the mean anchors (so that many members carry blend weight), unit normals, far points in a box,
    ground-truth anchors near the mean ones, codes B x 1 x 1344.  mean_anchors: 39 x 3."""
    rng = np.random.RandomState(seed)
    a = np.asarray(mean_anchors, np.float64).reshape(-1, 3)

    def near_anchors(n, spread):
        idx = rng.randint(0, a.shape[0], size=(B, n))
        return (a[idx] + spread * rng.randn(B, n, 3)).astype(np.float32)

    def normals(n):
        v = rng.randn(B, n, 3)
        return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)

    return {'points_face': near_anchors(sizes[0], 0.04), 'normals_face': normals(sizes[0]),
            'points_non_face': near_anchors(sizes[1], 0.06), 'normals_non_face': normals(sizes[1]),
            'sup_grad_near': near_anchors(sizes[2], 0.05),
            'sup_grad_far': ((rng.rand(B, sizes[3], 3) - 0.5) * 1.2).astype(np.float32),
            'gt_anchors': (a[None] + 0.01 * rng.randn(B, a.shape[0], 3)).astype(np.float32),
            'codes': (0.05 * rng.randn(B, 1, 64 + 40 * 32)).astype(np.float32)}


def total_loss(losses):
    return sum(LAMBDAS[k] * losses[k] for k in LAMBDAS)


def gradient_record(decoder, codes):
    """Named gradients the golden stores in full (codes, mlp_pos) and the ensembled weights and biases it samples."""
    full = {'codes': codes.grad}
    for k, p in decoder.mlp_pos.named_parameters():
        full['mlp_pos.' + k] = p.grad
    e = decoder.ensembled_deep_sdf
    sampled = {}
    for i in range(N_ENSEMBLE_LAYERS):
        sampled['lin%d.weight' % i] = getattr(e, 'lin%d' % i).weight.grad
        sampled['lin%d.bias' % i] = getattr(e, 'lin%d' % i).bias.grad
    return {k: v.detach().cpu().numpy() for k, v in full.items()}, {k: v.detach().cpu().numpy() for k, v in sampled.items()}
