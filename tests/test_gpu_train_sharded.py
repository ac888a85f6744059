"""The data-parallel training steps (nphm_b200.training_sharded) on one H100, on the native paths: stage 1 of the NPHM ensemble
and of the NPM DeepSDF (forward_with_gradient_native), stage 2 with the `compress` deformation network and the `-mode npm`
DeepSDF (forward_native_grad).  One shard is the existing native step bit for bit; 2, 4 and 8 shards match the whole-batch
native step; two gloo processes sharing the GPU are LocalTrainGroup(2) bit for bit."""
import os
import socket

import pytest
import torch

import train_sharded_common as T

pytestmark = pytest.mark.gpu

B = 8
# native-vs-composite gradient bounds: test_gpu_train_ensemble.py (golden), test_gpu_train_shape.py, test_gpu_train.py
GRAD_RTOL = {'nphm': 5e-4, 'npm': 5e-4, 'compress': 2e-4, 'expr_npm': 2e-4}


def _trainer(kind, dev, val_batches=()):
    return T.make_trainer(kind, device=dev, dtype=torch.float32, val_batches=val_batches, big=True)


def _batches(kind, n, seed=0, batch_size=B):
    return [T.make_batch(kind, batch_size, seed + s, sizes=(750, 50, 800, 93), n_points=1000) for s in range(n)]


def _steps(kind, dev, batches, world):
    from nphm_b200.training_sharded import LocalTrainGroup, train_step_sharded
    tr = _trainer(kind, dev)
    torch.manual_seed(123)
    outs = [tr.train_step(dict(b), e) if world is None else train_step_sharded(tr, dict(b), e, LocalTrainGroup(world))
            for e, b in enumerate(batches)]
    return outs, T.state(tr), T.reduced_grads(tr)


@pytest.mark.parametrize('kind', T.KINDS)
def test_one_shard_is_the_native_step_bit_for_bit(kind, cuda_device):
    batches = _batches(kind, 3)
    want = _steps(kind, cuda_device, batches, None)
    got = _steps(kind, cuda_device, batches, 1)
    assert got[0] == want[0]
    T.assert_bitwise(got[1], want[1])
    T.assert_bitwise(got[2], want[2])


def _first_step_grads(kind, dev, batch, world):
    """Loss dict and the gradients before clipping of one step from the same state."""
    from nphm_b200.training_sharded import LocalTrainGroup, train_step_sharded
    tr = _trainer(kind, dev)
    tr.cfg = dict(tr.cfg, grad_clip=1e30, grad_clip_lat=1e30)         # the raw reduced gradients
    torch.manual_seed(123)
    out = tr.train_step(dict(batch), 0) if world is None else train_step_sharded(tr, dict(batch), 0, LocalTrainGroup(world))
    return out, T.reduced_grads(tr)


@pytest.mark.parametrize('world', [2, 4, 8])
@pytest.mark.parametrize('kind', T.KINDS)
def test_shards_match_the_whole_batch(kind, world, cuda_device):
    """Each tensor's gradient within the bound the native-vs-composite checks of the same decoder accept, relative to its
    largest magnitude (GRAD_RTOL); losses to 1e-6.  The native passes scale each point set's upstream by a power of two chosen
    from the set's largest entry and split fp16 operands into hi | lo parts: a shard's set has its own largest entry, so its
    partial sums round differently from the whole batch's.  Either is within the native path's own error of the exact
    gradient, hence within twice that of the other."""
    batch = _batches(kind, 1, seed=5)[0]
    want_l, want_g = _first_step_grads(kind, cuda_device, batch, None)
    got_l, got_g = _first_step_grads(kind, cuda_device, batch, world)
    for k, v in want_l.items():
        err = abs(got_l[k] - v) / max(abs(v), 1e-30)
        print('%s world %d loss %s rel %.3g' % (kind, world, k, err))
        assert err <= 1e-6 or abs(got_l[k] - v) <= 1e-12, (k, err)
    for k, v in want_g.items():
        err = T.rel_err(got_g[k], v)
        print('%s world %d grad %s rel %.3g' % (kind, world, k, err))
        assert err <= GRAD_RTOL[kind], (k, err)


def test_ten_ensemble_steps_track_the_whole_batch(cuda_device):
    batches = _batches('nphm', 10, seed=30, batch_size=4)
    start = _trainer('nphm', cuda_device)
    p0 = {n: p.detach().clone() for n, p in start.decoder.named_parameters()}
    want = _steps('nphm', cuda_device, batches, None)
    got = _steps('nphm', cuda_device, batches, 4)
    names = [k for k in want[1] if k.startswith('p.')]
    change = torch.cat([(want[1][k] - p0[k[2:]]).reshape(-1) for k in names]).norm().item()
    diff = torch.cat([(got[1][k] - want[1][k]).reshape(-1) for k in names]).norm().item()
    print('ten steps: total change %.4g, sharded - whole %.4g' % (change, diff))
    assert change > 0 and diff <= 1e-3 * change, (diff, change)
    for a, b in zip(got[0], want[0]):                  # the trajectories part at the gradients' rounding, ~1e-4 of a loss
        for k in b:
            assert abs(a[k] - b[k]) <= 1e-3 * abs(b[k]) + 1e-9, (k, a[k], b[k])


@pytest.mark.parametrize('world', [2, 4])
def test_validation_step_in_eval_mode(world, cuda_device):
    """The ensemble's eval-mode quirk at the last point of every batch row, rows sharded: the reduced validation losses and
    codes match the one-process compute_val_loss."""
    from nphm_b200.training_sharded import LocalTrainGroup, val_step_sharded
    batches = _batches('nphm', 2, seed=40)
    a, b = _trainer('nphm', cuda_device, batches), _trainer('nphm', cuda_device, batches)
    want = a.compute_val_loss(0)
    got = val_step_sharded(b, 0, LocalTrainGroup(world))
    for k, v in want.items():
        assert abs(got[k] - v) <= 1e-6 * abs(v) + 1e-12, (k, got[k], v)
    assert T.rel_err(b.latent_codes_val.weight, a.latent_codes_val.weight) <= 1e-5


# ---------------------------------------------------------------------------------------------- torch.distributed
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dist_worker(rank, world, port, backend, q):
    import torch.distributed as dist
    from nphm_b200.training_sharded import train_step_sharded
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = {'device_id': dev} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        for kind in ('nphm', 'compress'):
            tr = _trainer(kind, dev)
            torch.manual_seed(123)
            outs = [train_step_sharded(tr, dict(b), e) for e, b in enumerate(_batches(kind, 2))]
            q.put((rank, kind, outs, T.to_host(T.state(tr))))
    finally:
        dist.destroy_process_group()


def _run_ranks(world, backend):
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = T.collect(q, procs, 2 * world)
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    return res


def _check_ranks(res, dev, world):
    for kind in ('nphm', 'compress'):
        mine = [r for r in res if r[1] == kind]
        assert len(mine) == world
        want = _steps(kind, dev, _batches(kind, 2), world)
        for _, _, outs, st in mine:
            assert outs == want[0], kind
            T.assert_bitwise(T.from_host(st), {k: v.cpu() for k, v in want[1].items()})


def test_gloo_two_processes_share_the_gpu(cuda_device):
    _check_ranks(_run_ranks(2, 'gloo'), cuda_device, 2)


def test_nccl_two_gpus(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    _check_ranks(_run_ranks(2, 'nccl'), cuda_device, 2)
