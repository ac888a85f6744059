"""Shared by the data-parallel training tests (test_train_sharded_cpu.py, test_gpu_train_sharded.py) and
tools/bench_train_sharded.py: a trainer with the attributes and the one-process steps of the reference's TrainerAutoDecoder
(training.py:111-139 / :250-275, training_corresp.py:154-176 / :292-320) on this package's losses, seeded models of both
stages, batches, and comparisons of the trained state."""
import math

import numpy as np
import torch

import ensemble_train_common as E
from conftest import make_deformation, make_ensemble, make_npm, mean_anchors

LAMBDAS_NPM = {'surf_sdf': 2.0, 'normals': 0.3, 'space_sdf': 0.01, 'grad': 0.1, 'lat_reg': 0.002}        # npm.yaml
LAMBDAS_CORRESP = {'corresp': 100.0, 'lat_reg': 5.0e-05, 'loss_reg_zero': 5.0e-05}                       # nphm_def.yaml
KINDS = ('nphm', 'npm', 'compress', 'expr_npm')           # stage 1: ensemble, NPM DeepSDF; stage 2: compress, -mode npm
N_CODES, N_SUBJ = 64, 4


class Trainer:
    """What the sharded steps read from a reference TrainerAutoDecoder, and its one-process train_step / compute_val_loss
    with this package's losses: stage 1 natively on CUDA (composite on the CPU, in the codes' dtype), stage 2 through
    compute_loss_corresp_forward's own choice.  The codes' gradient is clipped as the sharded step clips it."""

    def __init__(self, decoder, codes, codes_val, cfg, device, decoder_shape=None, codes_shape=None, codes_shape_val=None,
                 val_batches=()):
        self.decoder, self.latent_codes, self.latent_codes_val = decoder, codes, codes_val
        self.cfg, self.device = cfg, device
        if codes_shape is not None:
            self.decoder_shape = decoder_shape
            self.latent_codes_shape, self.latent_codes_shape_val = codes_shape, codes_shape_val
            self.latent_codes_shape.requires_grad = False          # a module attribute, as in training_corresp.py:57
            self.latent_codes_shape_val.requires_grad = False
        self.optimizer_encoder = torch.optim.AdamW(params=list(decoder.parameters()), lr=cfg['lr'],
                                                   weight_decay=cfg['weight_decay'])
        self.optimizer_lat = torch.optim.SparseAdam(list(codes.parameters()), lr=cfg['lr_lat'])
        self.optimizer_lat_val = torch.optim.SparseAdam(list(codes_val.parameters()), lr=cfg['lr_lat'])
        self.val_data_loader = list(val_batches)
        self.exp_path = None

    def losses(self, batch, codes, codes_shape, epoch):
        from nphm_b200.models.loss_functions import actual_compute_loss, compute_loss_corresp_forward
        if codes_shape is not None:
            return compute_loss_corresp_forward(dict(batch), self.decoder, self.decoder_shape, codes, codes_shape, self.device,
                                                epoch, self.exp_path)
        dtype = codes.weight.dtype
        part = {k: v.to(self.device).to(dtype) for k, v in batch.items()}
        native = True if torch.device(self.device).type == 'cuda' else None
        return actual_compute_loss(part, self.decoder, codes(batch['idx'].to(self.device)), native=native)

    def train_step(self, batch, epoch):
        from nphm_b200.training_sharded import clip_sparse_grad_norm_
        self.decoder.train()
        self.optimizer_encoder.zero_grad()
        self.optimizer_lat.zero_grad()
        losses = self.losses(batch, self.latent_codes, getattr(self, 'latent_codes_shape', None), epoch)
        tot = 0
        for k in losses:
            tot = tot + self.cfg['lambdas'][k] * losses[k]
        tot.backward()
        torch.nn.utils.clip_grad_norm_(self.decoder.parameters(), max_norm=self.cfg['grad_clip'])
        clip_sparse_grad_norm_(self.latent_codes.weight, self.cfg['grad_clip_lat'])
        self.optimizer_encoder.step()
        self.optimizer_lat.step()
        out = {k: v.item() for k, v in losses.items()}
        out['loss'] = tot.item()
        return out

    def compute_val_loss(self, epoch):
        from nphm_b200.training_sharded import clip_sparse_grad_norm_
        self.decoder.eval()
        sums = {k: 0.0 for k in self.cfg['lambdas']}
        sums['loss'] = 0.0
        for b in self.val_data_loader:
            self.optimizer_lat_val.zero_grad()
            losses = self.losses(b, self.latent_codes_val, getattr(self, 'latent_codes_shape_val', None), None)
            tot = 0.0
            for k in losses:
                sums[k] += losses[k].item()
                tot = tot + self.cfg['lambdas'][k] * losses[k]
            tot.backward()
            clip_sparse_grad_norm_(self.latent_codes_val.weight, self.cfg['grad_clip_lat'])
            self.optimizer_lat_val.step()
            sums['loss'] += tot.item()
        return {k: v / len(self.val_data_loader) for k, v in sums.items()}


def _codes(n, dim, device, dtype, seed):
    """Embedding(n, dim, max_norm=1, sparse=True) whose rows have norms from about 0.3 to 1.9: about half of them are
    renormalised by a lookup."""
    g = torch.Generator().manual_seed(seed)
    e = torch.nn.Embedding(n, dim, max_norm=1.0, sparse=True)
    with torch.no_grad():
        e.weight.copy_(torch.randn(n, dim, generator=g) / math.sqrt(dim) * torch.linspace(0.3, 1.9, n)[:, None])
    return e.to(device=device, dtype=dtype)


def make_trainer(kind, device='cpu', dtype=torch.float64, val_batches=(), big=False):
    """Seeded trainer of one of KINDS.  big: the DeepSDF decoders at their configurations' sizes (stage 1: 515 -> 1024 x 8 -> 1,
    `-mode npm`: 715 -> 1024 x 8 -> 3) instead of small ones (the CPU tests run them in float64)."""
    from nphm_b200.models.deepSDF import DeepSDF
    if kind in ('nphm', 'npm'):
        if kind == 'nphm':
            dec = make_ensemble(0, device=device)
        elif big:                                            # the NPM DeepSDF of npm.yaml, 515 -> 1024 x 8 -> 1
            torch.manual_seed(12)
            dec = DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True).to(device)
        else:
            dec = make_npm(device)
        dec = dec.to(dtype)
        cfg = {'lambdas': E.LAMBDAS if kind == 'nphm' else LAMBDAS_NPM, 'lr': 5e-4, 'weight_decay': 0.01, 'lr_lat': 1e-3,
               'grad_clip': 0.1, 'grad_clip_lat': 0.1}
        return Trainer(dec, _codes(N_CODES, dec.lat_dim, device, dtype, 1), _codes(N_CODES, dec.lat_dim, device, dtype, 2),
                       cfg, device, val_batches=val_batches)
    cfg = {'lambdas': LAMBDAS_CORRESP, 'lr': 1e-4, 'weight_decay': 5e-4, 'lr_lat': 5e-4, 'grad_clip': 0.025,
           'grad_clip_lat': 0.025}
    if kind == 'compress':
        dec, dec_shape, d_shape, d_expr = make_deformation(device), make_ensemble(0, device=device), 32 * 39 + 32 + 64, 200
        dec.anchors = dec.anchors.to(device)
        dec_shape = dec_shape.to(dtype)
    else:
        torch.manual_seed(13)
        d_shape, d_expr = (512, 200) if big else (24, 16)
        dec = DeepSDF(lat_dim=d_shape + d_expr, hidden_dim=1024 if big else 48, nlayers=8 if big else 4, geometric_init=False,
                      out_dim=3).to(device)
        dec_shape = None
    dec = dec.to(dtype)
    return Trainer(dec, _codes(N_CODES, d_expr, device, dtype, 3), _codes(N_CODES, d_expr, device, dtype, 4), cfg, device,
                   decoder_shape=dec_shape, codes_shape=_codes(N_SUBJ, d_shape, device, dtype, 5),
                   codes_shape_val=_codes(N_SUBJ, d_shape, device, dtype, 6), val_batches=val_batches)


def make_batch(kind, B, seed, sizes=(12, 5, 12, 6), n_points=100):
    """A batch as the reference's loaders yield it (CPU tensors, float32 points, int64 B x 1 indices).  Stage 2's subj_ind
    repeats: rows share subjects."""
    rng = np.random.RandomState(seed)
    idx = torch.from_numpy(rng.permutation(N_CODES)[:B].reshape(B, 1).astype(np.int64))
    if kind in ('nphm', 'npm'):
        b = E.make_batch(mean_anchors().reshape(-1, 3).numpy(), sizes, B=B, seed=seed)
        del b['codes']
        out = {k: torch.from_numpy(v) for k, v in b.items()}
        out['idx'] = idx
        return out
    pts = ((rng.rand(B, n_points, 3) - 0.5) * 1.2).astype(np.float32)
    return {'points_neutral': torch.from_numpy(pts),
            'points_posed': torch.from_numpy((pts + 0.02 * rng.randn(B, n_points, 3)).astype(np.float32)),
            'gt_anchors': torch.from_numpy((rng.rand(B, 39, 3) - 0.5).astype(np.float32)), 'idx': idx,
            'subj_ind': torch.from_numpy((np.arange(B) % 3).reshape(B, 1).astype(np.int64))}


def state(trainer):
    """The trained state: decoder parameters, codes, optimizer states, generator states."""
    out = {'p.' + n: p.detach().clone() for n, p in trainer.decoder.named_parameters()}
    out['codes'] = trainer.latent_codes.weight.detach().clone()
    out['codes_val'] = trainer.latent_codes_val.weight.detach().clone()
    for name in ('optimizer_encoder', 'optimizer_lat', 'optimizer_lat_val'):
        for i, st in getattr(trainer, name).state_dict()['state'].items():
            for k, v in st.items():
                out['%s.%d.%s' % (name, i, k)] = torch.as_tensor(v).detach().clone()
    out['rng_cpu'] = torch.get_rng_state()
    if torch.device(trainer.device).type == 'cuda':
        out['rng_cuda'] = torch.cuda.get_rng_state(trainer.device)
    return out


def reduced_grads(trainer):
    """The gradients the last step's optimizers used (after clipping), the codes' coalesced to dense rows."""
    out = {n: p.grad.detach().clone() for n, p in trainer.decoder.named_parameters()}
    out['codes'] = trainer.latent_codes.weight.grad.coalesce().to_dense()
    return out


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def assert_bitwise(a, b):
    assert set(a) == set(b)
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, bad


def collect(q, procs, n, timeout=900):
    """n results from the spawned processes; fails as soon as one of them exits with an error instead of waiting for it."""
    import time
    out, t0 = [], time.time()
    while len(out) < n:
        if not q.empty():
            out.append(q.get())
            continue
        dead = [p.exitcode for p in procs if p.exitcode not in (None, 0)]
        assert not dead and time.time() - t0 < timeout, ('a rank failed or timed out', dead)
        time.sleep(0.2)
    return out


def to_host(d):
    """Tensors as numpy arrays, to leave a spawned process through a queue (a torch tensor there is shared memory that the
    exiting process takes with it)."""
    return {k: v.detach().cpu().numpy() for k, v in d.items()}


def from_host(d):
    return {k: torch.from_numpy(v) for k, v in d.items()}
