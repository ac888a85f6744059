#!/usr/bin/env python
"""Stage-2 training step (reference TrainerAutoDecoder.train_step, src/NPHM/models/training_corresp.py:154-176, loss
compute_loss_corresp_forward) at scripts/configs/nphm_def.yaml settings: 32 samples x 1000 points plus 32 x 100 `samps`,
lambdas corresp 100 / loss_reg_zero 5e-5 / lat_reg 5e-5, AdamW (lr 1e-4, weight decay 5e-4) on the decoder, SparseAdam
(lr_lat 5e-4) on the expression codes, clip_grad_norm_ 0.025 on the decoder and on the codes (grad_clip, grad_clip_lat),
codes as the reference makes them (sparse Embedding, max_norm 1.0; the codes' clip is done on the coalesced sparse
gradient, which torch's clip_grad_norm_ cannot take), and the per-step `.item()` of every loss term and of
the total.  Random weights and codes (no dataset): the step's work does not depend on the values.

    python tools/bench_train.py --steps 20 --warmup 3

Native (forward_native_grad: tensor-core forward and weight gradients) and composite (PyTorch autograd) steps alternate
in one process on one GPU, for the `compress` DeformationNetwork (235 -> 512 x 6 -> 3) and the `-mode npm` expression
decoder (715 -> 1024 x 8 -> 3).  CUDA events split a step into loss forward, backward and optimizer.  Prints one JSON line.

    python tools/bench_train.py --stage 1 --steps 20 --warmup 3

Stage 1 (reference scripts/training/train.py without -local -> TrainerAutoDecoder.train_step, src/NPHM/models/training.py:
112-139, loss actual_compute_loss) at scripts/configs/npm.yaml settings: the NPM DeepSDF (515 -> 1024 x 8 -> 1, geometric
init), 32 samples x (750 face + 50 non-face + 800 near + 93 far) points, the npm.yaml lambdas, AdamW (lr 5e-4, weight decay
0.02) on the decoder, SparseAdam (lr_lat 1e-3) on Embedding(., 512, max_norm 1, sparse) codes, clip_grad_norm_ 0.1 on both.
Native (forward_with_gradient_native: SDF, spatial gradient and their weight gradients on the tensor cores, one call per
loss) and composite (PyTorch double backward) steps alternate; also reports the peak device memory of each path (torch's
peak plus what the path holds outside torch's allocator) and, for the first step, the largest relative difference between
the native and the composite gradients.

    python tools/bench_train.py --stage 1 --decoder nphm --steps 10 --warmup 2

Stage 1 of the NPHM ensemble (train.py -local) at scripts/configs/nphm.yaml settings: FastEnsembleDeepSDFMirrored (39 local
+ 1 global member, 16 symmetric pairs, 99 -> 200 x 4 -> 1), the same 32 x (750 + 50 + 800 + 93) points with ground-truth
anchors, the nphm.yaml lambdas, AdamW (lr 5e-4, weight decay 0.01) on the decoder, SparseAdam (lr_lat 1e-3) on
Embedding(., 1344, max_norm 1, sparse) codes, clip_grad_norm_ 0.1 on both.  Native (forward_with_gradient_native: the
members' passes on the tensor cores, one launch per pass for all 40 members, anchors and blend in autograd) and composite
steps alternate, with peak memory and the first step's gradient difference as above.  If the batch does not fit, the line
says so and both are measured at the largest halved batch that does.  --profile --stage 1 --decoder nphm: the kernel
breakdown of native ensemble steps.

    python tools/bench_train.py --stage 1 --decoder nphm --eval --steps 10 --warmup 2

The reference's stage-1 validation step (TrainerAutoDecoder.compute_val_loss, src/NPHM/models/training.py:250-268) on the same
batches: the ensemble in eval mode, the loss and its backward, the codes' gradient clipped and a SparseAdam step on them.
Native (the members' passes with the eval-mode quirk applied before the blend) against composite, as above."""
import argparse, gc, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch

LAMBDAS = {'corresp': 100.0, 'loss_reg_zero': 5.0e-05, 'lat_reg': 5.0e-05}          # nphm_def.yaml
LAMBDAS_SHAPE = {'surf_sdf': 2.0, 'normals': 0.3, 'space_sdf': 0.01, 'grad': 0.1, 'lat_reg': 0.002}   # npm.yaml
LAMBDAS_NPHM = {'surf_sdf': 2.0, 'normals': 0.3, 'space_sdf': 0.01, 'grad': 0.1, 'lat_reg': 0.01, 'anchors': 7.5,
                'symm_dist': 0.01, 'middle_dist': 0.0}                                                       # nphm.yaml
SHAPE_SETS = (('points_face', 750), ('points_non_face', 50), ('sup_grad_near', 800), ('sup_grad_far', 93))

def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(',')]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), 'not measured'


def setup(mode, dev):
    from conftest import make_deformation
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(0)
    if mode == 'compress':
        dec = make_deformation(dev).train()
        lat_shape_dim = 32 * 39 + 32 + 64
    else:
        dec = DeepSDF(lat_dim=712, hidden_dim=1024, nlayers=8, geometric_init=False, out_dim=3).to(dev).train()
        lat_shape_dim = 512
    lat_expr = torch.nn.Embedding(64, 200, max_norm=1.0, sparse=True).to(dev)
    lat_shape = torch.nn.Embedding(16, lat_shape_dim, max_norm=1.0, sparse=True).to(dev)
    with torch.no_grad():
        lat_expr.weight.mul_(0.1)
        lat_shape.weight.mul_(0.1)
    opt = torch.optim.AdamW(dec.parameters(), lr=1e-4, weight_decay=5e-4)
    opt_lat = torch.optim.SparseAdam(lat_expr.parameters(), lr=5e-4)
    return dec, lat_expr, lat_shape, opt, opt_lat


def batch(B, N, dev, step):
    g = torch.Generator().manual_seed(step)
    pts = (torch.rand(B, N, 3, generator=g) - 0.5) * 1.2
    return {'points_neutral': pts, 'points_posed': pts + 0.02 * torch.randn(B, N, 3, generator=g),
            'gt_anchors': torch.rand(B, 39, 3, generator=g) - 0.5,
            'idx': torch.randint(0, 64, (B, 1), generator=g), 'subj_ind': torch.randint(0, 16, (B, 1), generator=g)}


def clip_sparse_grad_norm_(p, max_norm):
    """clip_grad_norm_ of the reference's grad_clip_lat for the sparse gradient of an Embedding(sparse=True): this torch's
    clip_grad_norm_ has no sparse norm kernel, the coalesced values carry the same norm."""
    g = p.grad.coalesce()
    coef = torch.clamp(max_norm / (g.values().norm() + 1e-6), max=1.0)
    p.grad = g * coef


def train_step(state, b, native, ev, keep=None):
    from nphm_b200.models.loss_functions import compute_loss_corresp_forward
    dec, lat_expr, lat_shape, opt, opt_lat = state
    ev[0].record()
    opt.zero_grad()
    opt_lat.zero_grad()
    losses = compute_loss_corresp_forward(dict(b), dec, None, lat_expr, lat_shape, 'cuda', native=native)
    tot = 0
    for k, lam in LAMBDAS.items():
        tot = tot + lam * losses[k]
    ev[1].record()
    tot.backward()
    ev[2].record()
    ev[4].record()
    torch.nn.utils.clip_grad_norm_(dec.parameters(), max_norm=0.025)
    clip_sparse_grad_norm_(lat_expr.weight, max_norm=0.025)
    opt.step()
    opt_lat.step()
    ev[3].record()
    values = {k: v.item() for k, v in losses.items()}                # the reference's per-step read-backs
    values['loss'] = tot.item()
    return values['loss']


def setup_shape(dev):
    from nphm_b200.models.deepSDF import DeepSDF
    torch.manual_seed(12)
    dec = DeepSDF(lat_dim=512, hidden_dim=1024, nlayers=8, geometric_init=True).to(dev).train()
    torch.manual_seed(0)
    codes = torch.nn.Embedding(64, 512, max_norm=1.0, sparse=True).to(dev)
    with torch.no_grad():
        codes.weight.mul_(0.01)
    opt = torch.optim.AdamW(dec.parameters(), lr=5e-4, weight_decay=0.02)
    opt_lat = torch.optim.SparseAdam(codes.parameters(), lr=1e-3)
    return dec, codes, opt, opt_lat


def setup_nphm(dev):
    from conftest import make_ensemble
    dec = make_ensemble(0, device=dev).train()
    torch.manual_seed(0)
    codes = torch.nn.Embedding(64, dec.lat_dim, max_norm=1.0, sparse=True).to(dev)
    with torch.no_grad():
        codes.weight.mul_(0.01)
    opt = torch.optim.AdamW(dec.parameters(), lr=5e-4, weight_decay=0.01)
    opt_lat = torch.optim.SparseAdam(codes.parameters(), lr=1e-3)
    return dec, codes, opt, opt_lat


def batch_shape(B, dev, step, anchors=False):
    """Sphere-like point sets of SHAPE_SETS with unit normals; anchors: also ground-truth anchors near the mean ones."""
    g = torch.Generator().manual_seed(step)
    out = {'idx': torch.randint(0, 64, (B, 1), generator=g)}
    if anchors:
        from conftest import mean_anchors
        out['gt_anchors'] = mean_anchors().reshape(1, 39, 3) + 0.01 * torch.randn(B, 39, 3, generator=g)
    for name, n in SHAPE_SETS:
        d = torch.randn(B, n, 3, generator=g)
        d = d / d.norm(dim=-1, keepdim=True)
        if name in ('points_face', 'points_non_face'):
            out[name] = 0.4 * d
            out['normals' + name[6:]] = d
        elif name == 'sup_grad_near':
            out[name] = 0.4 * d + 0.01 * torch.randn(B, n, 3, generator=g)
        else:
            out[name] = (torch.rand(B, n, 3, generator=g) - 0.5) * 1.2
    return out


def train_step_shape(state, b, native, ev, keep=None, lambdas=LAMBDAS_SHAPE):
    """One step; `keep` (a dict): receives copies of the gradients before clipping, taken between the timed phases."""
    from nphm_b200.models.loss_functions import compute_loss
    dec, codes, opt, opt_lat = state
    ev[0].record()
    opt.zero_grad()
    opt_lat.zero_grad()
    losses = compute_loss(dict(b), dec, codes, 'cuda', native=native)
    tot = 0
    for k, lam in lambdas.items():
        tot = tot + lam * losses[k]
    ev[1].record()
    tot.backward()
    ev[2].record()
    if keep is not None:
        keep.update({n: p.grad.detach().clone() for n, p in dec.named_parameters()})
        keep['codes'] = codes.weight.grad.coalesce().to_dense()
    ev[4].record()
    torch.nn.utils.clip_grad_norm_(dec.parameters(), max_norm=0.1)
    clip_sparse_grad_norm_(codes.weight, max_norm=0.1)
    opt.step()
    opt_lat.step()
    ev[3].record()
    values = {k: v.item() for k, v in losses.items()}                # the reference's per-step read-backs
    values['loss'] = tot.item()
    return values['loss']


def val_step_nphm(state, b, native, ev, keep=None):
    """One step of the reference's stage-1 validation (TrainerAutoDecoder.compute_val_loss, training.py:250-268): the decoder in
    eval mode, the loss and its backward, the codes' gradient clipped and one SparseAdam step on them.  The decoder's own
    gradients accumulate unused there, as in the reference."""
    from nphm_b200.models.loss_functions import compute_loss
    dec, codes, _, opt_lat = state
    dec.eval()
    ev[0].record()
    opt_lat.zero_grad()
    losses = compute_loss(dict(b), dec, codes, 'cuda', native=native)
    tot = 0
    for k, lam in LAMBDAS_NPHM.items():
        tot = tot + lam * losses[k]
    ev[1].record()
    tot.backward()
    ev[2].record()
    if keep is not None:
        keep['codes'] = codes.weight.grad.coalesce().to_dense()
    ev[4].record()
    clip_sparse_grad_norm_(codes.weight, max_norm=0.1)
    opt_lat.step()
    ev[3].record()
    values = {k: v.item() for k, v in losses.items()}                # the reference's per-step read-backs
    values['loss'] = tot.item()
    return values['loss']


def outside_torch_bytes():
    """Device memory in use that torch's caching allocator does not hold (native handles' buffers, CUDA context); read from
    the driver's free count, so other processes on the same GPU would show up here too."""
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return (total - free) - torch.cuda.memory_reserved()


def run(setup_fn, batch_fn, step_fn, args, compare_first=False):
    """Alternates native and composite steps on two identically initialised states; median CUDA-event times per phase
    (events: 0 start, 1 loss, 2 backward done, 4 optimizer start, 3 end; the gradient copies of the first-step comparison
    fall between 2 and 4, outside every reported time).  compare_first: also the peak device memory of each path (torch's
    peak of the step plus what the path added outside torch's allocator) and the first step's gradient difference."""
    res = {}
    states = {nat: setup_fn() for nat in (True, False)}
    times = {nat: [] for nat in (True, False)}
    peak = {nat: 0 for nat in (True, False)}
    outside = {nat: 0 for nat in (True, False)}
    first = {True: {}, False: {}}
    for step in range(args.warmup + args.steps):
        b = batch_fn(step)
        for nat in (True, False):                       # alternate native / composite
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            before = outside_torch_bytes() if compare_first else 0
            torch.cuda.reset_peak_memory_stats()
            tot = step_fn(states[nat], b, nat, ev, first[nat] if compare_first and step == 0 else None)
            torch.cuda.synchronize()
            if compare_first:
                # buffers allocated outside torch are not released within a step: what the step added was held at its peak
                outside[nat] += max(0, outside_torch_bytes() - before)
                peak[nat] = max(peak[nat], torch.cuda.max_memory_allocated())
            if step >= args.warmup:
                fwd, bwd, opt = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[4].elapsed_time(ev[3])
                times[nat].append([fwd + bwd + opt, fwd, bwd, opt])
            res.setdefault('finite', True)
            res['finite'] &= bool(tot == tot and abs(tot) != float('inf'))
    for nat in (True, False):
        t = torch.tensor(times[nat]).median(dim=0).values.tolist()
        r = res['native' if nat else 'composite'] = {'steps_per_s': 1000.0 / t[0], 'ms_step': t[0], 'ms_forward': t[1],
                                                     'ms_backward': t[2], 'ms_optimizer': t[3]}
        if compare_first:
            r['peak_memory_gib'] = (peak[nat] + outside[nat]) / 2 ** 30
            r['outside_torch_gib'] = outside[nat] / 2 ** 30
    res['speedup'] = res['native']['steps_per_s'] / res['composite']['steps_per_s']
    if compare_first:
        # largest over the tensors of max |native - composite| / max |composite| (first step, before clipping)
        res['first_step_grad_max_rel_diff'] = max(
            ((first[True][k] - v).abs().max() / v.abs().max().clamp_min(1e-30)).item() for k, v in first[False].items())
    return res


def run_mode(mode, args, dev):
    return run(lambda: setup(mode, dev), lambda step: batch(32, 1000, dev, step), train_step, args)


def run_nphm(args, dev, name, power, eval_mode=False):
    """Native and composite ensemble steps at B = 32, halving B after an out-of-memory error.  eval_mode: the validation step
    (:func:`val_step_nphm`) instead of the training step."""
    out = {'metric': 'stage1_nphm_val_step' if eval_mode else 'stage1_nphm_train_step', 'gpu': name, 'power_limit': power,
           'steps': args.steps, 'timing': 'median of CUDA-event times per step, native and composite alternated'}
    step_fn = val_step_nphm if eval_mode else (lambda *a: train_step_shape(*a, lambdas=LAMBDAS_NPHM))
    B = 32
    while B >= 1:
        oom = False
        try:
            out['nphm'] = run(lambda: setup_nphm(dev), lambda step: batch_shape(B, dev, step, anchors=True), step_fn, args,
                              compare_first=True)
            out['batch'] = '%d x (750 + 50 + 800 + 93) points' % B
            return out
        except torch.cuda.OutOfMemoryError:
            oom = True
        if oom:                                        # outside the handler: the failed attempt's frames are released
            out.setdefault('out_of_memory_at_batch', []).append(B)
            gc.collect()
            torch.cuda.empty_cache()
            B //= 2
    return out


def profile_native(dev, stage=2, steps=5, decoder='npm'):
    """CUDA time per kernel (ms per step, largest first) of native steps (stage 2: `compress`, stage 1: NPM), from
    torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    if stage == 1 and decoder == 'nphm':
        state, batch_fn = setup_nphm(dev), lambda step: batch_shape(32, dev, step, anchors=True)
        step_fn = lambda *a: train_step_shape(*a, lambdas=LAMBDAS_NPHM)           # noqa: E731
    elif stage == 1:
        state, step_fn, batch_fn = setup_shape(dev), train_step_shape, lambda step: batch_shape(32, dev, step)
    else:
        state, step_fn, batch_fn = setup('compress', dev), train_step, lambda step: batch(32, 1000, dev, step)
    for step in range(3):
        step_fn(state, batch_fn(step), True, [torch.cuda.Event(enable_timing=True) for _ in range(5)])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for step in range(steps):
            step_fn(state, batch_fn(100 + step), True, [torch.cuda.Event(enable_timing=True) for _ in range(5)])
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, 'device_time_total', None)
        if t is None:
            t = e.cuda_time_total
        if t > 0 and e.count > 0:
            rows[e.key[:90]] = (t / 1000.0 / steps, e.count // steps)
    top = sorted(rows.items(), key=lambda kv: -kv[1][0])
    total = sum(v[0] for _, v in top)
    return {'ms_per_step_kernels': total, 'kernels': [{'name': k, 'ms_per_step': round(v[0], 4), 'launches_per_step': v[1]}
                                                      for k, v in top[:25]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--stage', type=int, choices=(1, 2), default=2,
                    help='2: expression space (train_corresp.py), 1: NPM shape space (train.py without -local)')
    ap.add_argument('--decoder', choices=('npm', 'nphm'), default='npm',
                    help='stage 1: npm (DeepSDF, train.py) or nphm (the ensemble, train.py -local)')
    ap.add_argument('--eval', action='store_true',
                    help='--stage 1 --decoder nphm: time the eval-mode validation step (compute_val_loss) instead')
    ap.add_argument('--profile', action='store_true',
                    help='instead: torch.profiler over 5 native steps of the stage, CUDA time per kernel of the step (JSON)')
    args = ap.parse_args()
    if args.steps < 1:
        ap.error('--steps must be >= 1')
    if args.decoder == 'nphm' and args.stage != 1:
        ap.error('--decoder nphm: stage 1 only')
    if args.eval and (args.decoder != 'nphm' or args.profile):
        ap.error('--eval: --stage 1 --decoder nphm only, without --profile')
    dev = torch.device('cuda', torch.cuda.current_device())
    name, power = gpu_info()
    if args.profile:
        print(json.dumps({'metric': 'stage%d_native_kernels' % args.stage, 'gpu': name, 'power_limit': power,
                          **profile_native(dev, args.stage, decoder=args.decoder)}))
        return
    if args.stage == 1 and args.decoder == 'nphm':
        print(json.dumps(run_nphm(args, dev, name, power, eval_mode=args.eval)))
        return
    if args.stage == 1:
        out = {'metric': 'stage1_train_step', 'gpu': name, 'power_limit': power,
               'batch': '32 x (750 + 50 + 800 + 93) points', 'steps': args.steps,
               'timing': 'median of CUDA-event times per step, native and composite alternated'}
        out['npm'] = run(lambda: setup_shape(dev), lambda step: batch_shape(32, dev, step), train_step_shape, args,
                         compare_first=True)
        print(json.dumps(out))
        return
    out = {'metric': 'stage2_train_step', 'gpu': name, 'power_limit': power, 'batch': '32 x (1000 + 100) points',
           'steps': args.steps, 'timing': 'median of CUDA-event times per step, native and composite alternated'}
    for mode in ('compress', 'npm'):
        out[mode] = run_mode(mode, args, dev)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
