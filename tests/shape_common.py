"""Shared by the stage-1 loss tests (test_train_shape_cpu.py, test_gpu_train_shape.py) and
tests/golden/make_golden_train_shape.py: the seeded NPM decoder and batch of the golden train_shape.npz, and the gradients it
records."""
import hashlib

import numpy as np
import torch

# scripts/configs/npm.yaml: lambdas of the stage-1 loss (the anchor / symmetry terms do not exist for a plain DeepSDF)
LAMBDAS = {'surf_sdf': 2.0, 'normals': 0.3, 'space_sdf': 0.01, 'grad': 0.1, 'lat_reg': 0.002}
POINT_SETS = ('points_face', 'points_non_face', 'sup_grad_near', 'sup_grad_far')
GRAD_SAMPLES = 2000
# relative bounds of the loss terms: 1e-5, except the two terms that are functions of the SDF value itself.  The native value
# pass of the 1024-wide stack (fp16 hi | lo operands, MUFU softplus: the forward of nphm_mlp_query_layers) leaves ~5e-6 absolute
# error in s, which is 1.3e-5 of surf_sdf = mean |s| ~ 0.4 and, through the factor 10 in exp(-10 |s|), 5e-5 of space_sdf.
LOSS_RTOL = {'surf_sdf': 1e-4, 'space_sdf': 1e-4}


def make_decoder(cls, device='cpu'):
    """The NPM baseline of npm.yaml (lat_dim 512, hidden 1024, 8 layers, geometric init), seeded like tests/golden/npm.npz."""
    torch.manual_seed(12)
    return cls(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True).to(device)


def state_dict_sha256(module):
    h = hashlib.sha256()
    sd = module.state_dict()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(np.ascontiguousarray(sd[k].detach().cpu().numpy()).tobytes())
    return h.hexdigest()


def make_batch(B=2, sizes=(60, 20, 60, 25), seed=5):
    """Surface points near a sphere of radius 0.4 with unit normals, off-surface points around them, far points in the
    unit box; codes B x 1 x 512."""
    rng = np.random.RandomState(seed)

    def sphere(n):
        d = rng.randn(B, n, 3)
        d /= np.linalg.norm(d, axis=-1, keepdims=True)
        return (0.4 * d * (1 + 0.05 * rng.randn(B, n, 1))).astype(np.float32), d.astype(np.float32)

    face, n_face = sphere(sizes[0])
    non_face, n_non = sphere(sizes[1])
    near = sphere(sizes[2])[0] + (0.01 * rng.randn(B, sizes[2], 3)).astype(np.float32)
    far = ((rng.rand(B, sizes[3], 3) - 0.5) * 1.2).astype(np.float32)
    return {'points_face': face, 'normals_face': n_face, 'points_non_face': non_face, 'normals_non_face': n_non,
            'sup_grad_near': near, 'sup_grad_far': far,
            'codes': (0.05 * rng.randn(B, 1, 512)).astype(np.float32)}


def total_loss(losses):
    return sum(LAMBDAS[k] * losses[k] for k in LAMBDAS)


def gradient_record(decoder, codes):
    """Named gradients the golden stores in full (codes, biases) and the weight matrices it samples."""
    full = {'codes': codes.grad}
    for i in range(decoder.num_layers - 1):
        full['lin%d.bias' % i] = getattr(decoder, 'lin%d' % i).bias.grad
    sampled = {'lin%d.weight' % i: getattr(decoder, 'lin%d' % i).weight.grad for i in range(decoder.num_layers - 1)}
    return {k: v.detach().cpu().numpy() for k, v in full.items()}, {k: v.detach().cpu().numpy() for k, v in sampled.items()}


def sample_idx(name, size):
    seed = sum(ord(c) for c in name)
    return np.sort(np.random.RandomState(seed).choice(size, min(GRAD_SAMPLES, size), replace=False))


def run_step(decoder, g, device, native):
    """One loss evaluation and backward of the mirror on the golden's batch -> (losses, codes leaf)."""
    from nphm_b200.models.loss_functions import actual_compute_loss
    batch = {k: torch.from_numpy(g['batch_' + k]).to(device) for k in
             ('points_face', 'normals_face', 'points_non_face', 'normals_non_face', 'sup_grad_near', 'sup_grad_far')}
    codes = torch.from_numpy(g['batch_codes']).to(device).requires_grad_()
    losses = actual_compute_loss(batch, decoder, codes, native=native)
    total_loss(losses).backward()
    return losses, codes


def loss_rtol(name, native=True):
    return LOSS_RTOL.get(name, 1e-5) if native else 1e-5


def check_against_golden(g, losses, full, sampled, rtol, native=True):
    """Loss terms to `loss_rtol` (LOSS_RTOL), every stored gradient (and each weight gradient's max-abs and norm) to `rtol`
    of its largest magnitude."""
    for n, v in zip([str(n) for n in g['loss_names']], g['loss_values']):
        got = float(losses[n].detach())
        print('golden loss %s rel %.3g' % (n, abs(got - v) / abs(v)))
        assert abs(got - v) <= loss_rtol(n, native) * abs(v), (n, got, v)
    errs = {}
    for k, v in full.items():
        ref = g['full_' + k]
        errs[k] = float(np.abs(v - ref).max() / max(np.abs(ref).max(), 1e-30))
    for k, v in sampled.items():
        flat = v.reshape(-1)
        ref = g['sampled_' + k]
        errs[k] = max(float(np.abs(flat[g['idx_' + k]] - ref).max() / max(float(g['maxabs_' + k]), 1e-30)),
                      abs(float(np.abs(flat).max()) - float(g['maxabs_' + k])) / float(g['maxabs_' + k]),
                      abs(float(np.linalg.norm(flat)) - float(g['norm_' + k])) / float(g['norm_' + k]))
    for k, e in sorted(errs.items()):
        print('golden %s rel %.3g' % (k, e))
    bad = {k: e for k, e in errs.items() if not e <= rtol}
    assert not bad, bad
