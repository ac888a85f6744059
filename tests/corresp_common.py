"""Shared by the stage-2 loss tests (test_train_corresp_cpu.py, test_gpu_train.py) and tests/golden/make_golden_train_corresp.py:
the seeded setup of the golden train_corresp.npz, and recording / replaying the random draws of compute_loss_corresp_forward."""
import contextlib

import numpy as np
import torch

# scripts/configs/nphm_def.yaml: lambdas of the stage-2 loss
LAMBDAS = {'corresp': 100.0, 'lat_reg': 5.0e-05, 'loss_reg_zero': 5.0e-05}
B, N, N_EXPR, N_SHAPE = 4, 300, 8, 5
GRAD_SAMPLES = 2000


def make_batch():
    rng = np.random.RandomState(5)
    pts = ((rng.rand(B, N, 3) - 0.5) * 1.2).astype(np.float32)
    return {'points_neutral': pts, 'points_posed': (pts + 0.02 * rng.randn(B, N, 3)).astype(np.float32),
            'gt_anchors': (rng.rand(B, 39, 3) - 0.5).astype(np.float32),
            'idx': np.array([[1], [3], [0], [6]], np.int64), 'subj_ind': np.array([[0], [2], [4], [1]], np.int64)}


def make_embeddings(device='cpu', expr=None, shape=None):
    """(expression codes: sparse Embedding(8, 200), shape codes: Embedding(5, 1344)); seeded, or the given weights."""
    torch.manual_seed(21)
    lat_expr = torch.nn.Embedding(N_EXPR, 200, sparse=True)
    lat_shape = torch.nn.Embedding(N_SHAPE, 32 * 39 + 32 + 64)
    with torch.no_grad():
        lat_expr.weight.mul_(0.05)
        lat_shape.weight.mul_(0.05)
        if expr is not None:
            lat_expr.weight.copy_(torch.from_numpy(expr))
            lat_shape.weight.copy_(torch.from_numpy(shape))
    return lat_expr.to(device), lat_shape.to(device)


def total_loss(losses):
    return sum(LAMBDAS[k] * losses[k] for k in LAMBDAS)


@contextlib.contextmanager
def record_draws(log):
    """Appends (kind, array) for every torch.randn / torch.rand call inside the block."""
    orig = {'randn': torch.randn, 'rand': torch.rand}

    def wrap(kind):
        def f(*a, **k):
            t = orig[kind](*a, **k)
            log.append((kind, t.detach().cpu().numpy().copy()))
            return t
        return f
    torch.randn, torch.rand = wrap('randn'), wrap('rand')
    try:
        yield log
    finally:
        torch.randn, torch.rand = orig['randn'], orig['rand']


@contextlib.contextmanager
def replay_draws(kinds, arrays):
    """torch.randn / torch.rand return the recorded draws, in order (kind and shape must match)."""
    orig = {'randn': torch.randn, 'rand': torch.rand}
    pending = list(zip(kinds, arrays))

    def wrap(kind):
        def f(*a, device=None, dtype=None, **k):
            assert pending, 'more random draws than recorded'
            want, arr = pending.pop(0)
            shape = tuple(a[0]) if len(a) == 1 and not isinstance(a[0], int) else tuple(a)
            assert want == kind and tuple(arr.shape) == shape, (want, kind, arr.shape, shape)
            return torch.from_numpy(arr).to(device=device, dtype=dtype or torch.float32)
        return f
    torch.randn, torch.rand = wrap('randn'), wrap('rand')
    try:
        yield
        assert not pending, 'fewer random draws than recorded'
    finally:
        torch.randn, torch.rand = orig['randn'], orig['rand']


def gradient_record(dfn, decoder_shape, lat_expr, lat_shape, batch):
    """Named gradients the golden stores (full tensors) and the weight matrices it samples."""
    full = {'compressor.0.weight': dfn.compressor[0].weight.grad, 'compressor.0.bias': dfn.compressor[0].bias.grad}
    for i in range(dfn.defDeepSDF.num_layers - 1):
        full['defDeepSDF.lin%d.bias' % i] = getattr(dfn.defDeepSDF, 'lin%d' % i).bias.grad
    for i in (0, 2, 4):
        full['mlp_pos.%d.bias' % i] = decoder_shape.mlp_pos[i].bias.grad
    full['expr_rows'] = lat_expr.weight.grad.to_dense()[torch.as_tensor(batch['idx'][:, 0])]
    full['shape_rows'] = lat_shape.weight.grad[torch.as_tensor(batch['subj_ind'][:, 0])]
    sampled = {'defDeepSDF.lin%d.weight' % i: getattr(dfn.defDeepSDF, 'lin%d' % i).weight.grad
               for i in range(dfn.defDeepSDF.num_layers - 1)}
    for i in (0, 2, 4):
        sampled['mlp_pos.%d.weight' % i] = decoder_shape.mlp_pos[i].weight.grad
    return {k: v.detach().cpu().numpy() for k, v in full.items()}, {k: v.detach().cpu().numpy() for k, v in sampled.items()}


def sample_idx(name, size):
    seed = sum(ord(c) for c in name)
    return np.sort(np.random.RandomState(seed).choice(size, min(GRAD_SAMPLES, size), replace=False))


def check_against_golden(g, losses, full, sampled, rtol):
    """Loss terms to 1e-5 (relative above 1), every stored gradient to `rtol` of its largest magnitude."""
    names = [str(n) for n in g['loss_names']]
    for n, v in zip(names, g['loss_values']):
        got = float(losses[n].detach())
        assert abs(got - v) <= 1e-5 * max(1.0, abs(v)), (n, got, v)
    errs = {}
    for k, v in full.items():
        ref = g['full_' + k]
        errs[k] = float(np.abs(v - ref).max() / max(np.abs(ref).max(), 1e-30))
    for k, v in sampled.items():
        flat = v.reshape(-1)
        ref = g['sampled_' + k]
        errs[k] = max(float(np.abs(flat[g['idx_' + k]] - ref).max() / max(np.abs(ref).max(), 1e-30)),
                      abs(float(np.linalg.norm(flat)) - float(g['norm_' + k])) / float(g['norm_' + k]))
    for k, e in sorted(errs.items()):
        print('golden %s rel %.3g' % (k, e))
    bad = {k: e for k, e in errs.items() if not e <= rtol}
    assert not bad, bad
