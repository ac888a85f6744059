"""The scan-batched fitters over several ranks (nphm_b200.fitting_sharded) on one H100, on the native batched paths: the NPHM
ensemble with the `compress` deformation network and the NPM baseline's DeepSDF decoders, identity and joint fitting, with the
identity decoder in training and in eval mode (the quirk rows).

At world 1 every step of the batched fitters receives, bit for bit, the inputs (sampled points, observation indices, lambdas,
clamp, lr) it receives in the batched call on each chunk - and in the existing batched call when one chunk holds every subject
- and the generator state and lambdas end equal.  The results themselves are compared within a tolerance: the native fitting
kernels sum gradients with float atomics, so two runs of the same batched call differ in the last bits, and Adam's first,
sign-like steps turn that into part of a step for entries whose gradient is at round-off level (the bounds of
test_gpu_fit_batched.py).  Two gloo processes sharing the GPU are checked the same way against world 1."""
import hashlib
import os
import socket

import pytest
import torch

import npm_fit_common as C
from conftest import make_deformation, make_ensemble
from train_sharded_common import collect

pytestmark = pytest.mark.gpu

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
LAMBDAS_ID = {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
SCHEDULE = {'lr': {200: 2, 400: 2}, 'symm_dist': {200: 10}, 'reg_glob': {200: 3}, 'reg_loc': {400: 3}, 'reg_expr': {400: 10}}
N_STEPS, STEP_SCALE = 500, 0.01            # five iterations, the schedule fires at the third and fifth
BATCH_SIZE = 2


def _decoders(decoder, mode, dev):
    if decoder == 'nphm':
        dec, dfn = make_ensemble(0, device=dev), make_deformation(dev)
    else:
        from nphm_b200.models.deepSDF import DeepSDF
        dec, dfn = C.make_decoders(DeepSDF, dev)
    return (dec.train() if mode == 'train' else dec.eval()), dfn


def _subjects(dev):
    """Five subjects with 1 to 3 expressions; subject 2 has fewer than 1000 points per observation."""
    g = torch.Generator().manual_seed(7)
    sizes = [(2000, 1500, 1800), (1200,), (700, 700), (3000, 1000), (1100, 1400, 1000)]
    centre = torch.tensor([0.0, 0.05, -0.1])
    return [[(torch.randn(n, 3, generator=g) * 0.1 + centre).to(dev) for n in s] for s in sizes]


def _fit(kind, decoders, subjects, lambdas, **kw):
    from nphm_b200.fitting_sharded import (inference_identity_space_batched_sharded,
                                           inference_iterative_root_finding_joint_batched_sharded)
    from nphm_b200.models.fitting import inference_identity_space_batched, inference_iterative_root_finding_joint_batched
    dec, dfn = decoders
    if kind == 'identity':
        fn = inference_identity_space_batched_sharded if kw else inference_identity_space_batched
        return fn(dec, subjects, lambdas, N_STEPS, SCHEDULE, step_scale=STEP_SCALE, **kw)
    fn = inference_iterative_root_finding_joint_batched_sharded if kw else inference_iterative_root_finding_joint_batched
    return fn(dec, dfn, subjects, lambdas, N_STEPS, SCHEDULE, step_scale=STEP_SCALE, **kw)


def _lambdas(kind):
    return dict(LAMBDAS_ID if kind == 'identity' else LAMBDAS)


def _chunked(kind, decoders, subjects, batch_size):
    """The batched call on each chunk in turn from seed 0: each chunk starts where the sequential loop starts its first
    subject.  Returns (results, generator state, lambdas of the last call)."""
    torch.manual_seed(0)
    out, lam = [], None
    for lo in range(0, len(subjects), batch_size):
        lam = _lambdas(kind)
        out += _fit(kind, decoders, subjects[lo:lo + batch_size], lam)
    return out, torch.get_rng_state(), lam


def _sharded(kind, decoders, subjects, batch_size, group=None):
    torch.manual_seed(0)
    lam = _lambdas(kind)
    out = _fit(kind, decoders, subjects, lam, batch_size=batch_size, group=group)
    return out, torch.get_rng_state(), lam


def _assert_close(got, want, what):
    """Same shapes, dtypes and requires_grad flags, the generator state and lambdas exactly; codes with at least 93 % of the
    entries within 2e-5 and anchors within 1e-5 (test_gpu_fit_batched.py's bounds between the batched and sequential paths)."""
    assert len(got[0]) == len(want[0]), what
    worst = 0.0
    for k, (a, b) in enumerate(zip(got[0], want[0])):
        assert len(a) == len(b), (what, k)
        for i, (x, y) in enumerate(zip(a, b)):
            assert (x is None) == (y is None), (what, k)
            if x is None:
                continue
            assert x.shape == y.shape and x.dtype == y.dtype and x.requires_grad == y.requires_grad, (what, k)
            d = (x.detach().cpu() - y.detach().cpu()).abs()
            worst = max(worst, float(d.max()))
            if i == len(a) - 1 and x.shape[-1] == 3:                    # anchors
                assert float(d.max()) < 1e-5, (what, k, float(d.max()))
            else:
                assert float((d < 2e-5).double().mean()) > 0.93, (what, k, float(d.max()))
    print('%s: largest difference %.3g' % (what, worst))
    assert torch.equal(got[1], want[1]), what
    assert got[2] == want[2], what


def _digest(x):
    if isinstance(x, torch.Tensor):
        return hashlib.sha256(x.detach().cpu().contiguous().numpy().tobytes()).hexdigest() + str(tuple(x.shape))
    if isinstance(x, (list, tuple)):
        return [_digest(v) for v in x]
    if isinstance(x, dict):
        return repr(sorted(x.items()))
    return repr(x)


def _record_steps(monkeypatch):
    """A digest of the inputs of every batched fitter step, in call order."""
    from nphm_b200.models import fitting as F
    log = []
    for name in ('BatchedIdentityFitter', 'BatchedNpmIdentityFitter', 'BatchedJointFitter', 'BatchedNpmJointFitter'):
        cls = getattr(F, name)

        def step(self, *args, _real=cls.step, **kwargs):
            log.append((type(self).__name__, _digest(list(args)), _digest(kwargs)))
            return _real(self, *args, **kwargs)
        monkeypatch.setattr(cls, 'step', step)
    return log


@pytest.mark.parametrize('mode', ['train', 'eval'])
@pytest.mark.parametrize('kind', ['identity', 'joint'])
@pytest.mark.parametrize('decoder', ['nphm', 'npm'])
def test_world_one_is_the_batched_call_on_each_chunk(decoder, kind, mode, cuda_device, monkeypatch):
    from nphm_b200.models import fitting as F
    monkeypatch.delenv('NPHM_JOINT_AUTOGRAD', raising=False)
    decoders = _decoders(decoder, mode, cuda_device)
    subjects = _subjects(cuda_device)
    # the batched fitters run: the chunks are fitted natively, not subject by subject
    if kind == 'identity':
        assert F._identity_batch_fit(decoders[0], subjects, N_STEPS, SCHEDULE, STEP_SCALE, 1) is not None
    else:
        assert F._joint_batch_fit(*decoders, subjects, N_STEPS, SCHEDULE, STEP_SCALE, 1) is not None
    log = _record_steps(monkeypatch)
    for batch_size in (BATCH_SIZE, len(subjects)):
        log.clear()
        want = _chunked(kind, decoders, subjects, batch_size)
        steps_want = list(log)
        log.clear()
        got = _sharded(kind, decoders, subjects, batch_size)
        assert len(steps_want) == -(-len(subjects) // batch_size) * 5 and log == steps_want, (decoder, kind, mode, batch_size)
        _assert_close(got, want, (decoder, kind, mode, batch_size))
    # and the results are those of a fit: the codes moved, every subject differently
    codes = [r[-2 if kind == 'joint' else 0].detach() for r in got[0]]
    assert all(float(c.abs().max()) > 0 for c in codes)
    assert not torch.equal(codes[0], codes[1])


# ---------------------------------------------------------------------------------------------- torch.distributed
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


JOBS = [('nphm', 'identity', 'train'), ('nphm', 'joint', 'eval'), ('npm', 'joint', 'train')]


def _to_host(res):
    out, state, lam = res
    return ([tuple(None if t is None else (t.detach().cpu().numpy(), t.requires_grad) for t in r) for r in out],
            state.numpy(), lam)


def _from_host(res):
    out, state, lam = res
    return ([tuple(None if t is None else torch.from_numpy(t[0]).requires_grad_(t[1]) for t in r) for r in out],
            torch.from_numpy(state), lam)


def _dist_worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    os.environ.pop('NPHM_JOINT_AUTOGRAD', None)
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = {'device_id': dev} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        for decoder, kind, mode in JOBS:
            res = _sharded(kind, _decoders(decoder, mode, dev), _subjects(dev), BATCH_SIZE)
            for r in res[0]:
                assert all(t is None or t.device == dev for t in r)
            q.put((rank, (decoder, kind, mode), _to_host(res)))
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
        res = collect(q, procs, world * len(JOBS))
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
    for job in JOBS:
        mine = [r for r in res if r[1] == job]
        assert len(mine) == world
        decoder, kind, mode = job
        want = _sharded(kind, _decoders(decoder, mode, dev), _subjects(dev), BATCH_SIZE)
        want = ([tuple(None if t is None else t.detach().cpu().requires_grad_(t.requires_grad) for t in r) for r in want[0]],
                want[1], want[2])
        for rank, _, got in mine:
            _assert_close(_from_host(got), want, (job, rank))


def test_gloo_two_processes_share_the_gpu(cuda_device):
    """Chunks [0, 2) and [4, 5) on rank 0, [2, 4) on rank 1: every rank gets every subject's result."""
    _check_ranks(_run_ranks(2, 'gloo'), cuda_device, 2)


def test_nccl_two_gpus(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    _check_ranks(_run_ranks(2, 'nccl'), cuda_device, 2)
