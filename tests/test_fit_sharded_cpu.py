"""CPU checks of the scan-batched fitters over several ranks (nphm_b200.fitting_sharded) on the float64 composite path: the
chunk plan, and worlds of 1, 2 and 3 (gloo processes) against the one-process batched functions - which on the CPU fit the
subjects one after another - bit for bit, with the generator state and the lambdas of the sequential loop."""
import os
import socket

import pytest
import torch

from conftest import mean_anchors
from train_sharded_common import collect

LAMBDAS = {'surface': 2.0, 'reg_expr': 0.01, 'reg_global': 0.25, 'reg_unobserved': 10, 'reg_loc': 0.05, 'symm_dist': 5.0}
LAMBDAS_ID = {k: v for k, v in LAMBDAS.items() if k != 'reg_expr'}
SCHEDULE = {'lr': {100: 2}, 'symm_dist': {100: 10}, 'reg_glob': {100: 3}, 'reg_expr': {100: 10}}
N_STEPS, STEP_SCALE = 200, 0.01          # two iterations; the schedule fires at the second
BATCH_SIZES = (1, 2, 5)


def _decoders():
    """A small ensemble and a `compress` deformation network of matching sizes, float64 (the default dtype must be float64:
    the fitters make their codes with it)."""
    from nphm_b200.models.EnsembledDeepSDF import FastEnsembleDeepSDFMirrored
    from nphm_b200.models.deepSDF import DeformationNetwork
    torch.manual_seed(4)
    dec = FastEnsembleDeepSDFMirrored(lat_dim_glob=16, lat_dim_loc=8, n_loc=39, n_symm_pairs=16, anchors=mean_anchors(),
                                      hidden_dim=32, n_layers=4, pos_mlp_dim=32).double().train()
    dfn = DeformationNetwork(mode='compress', lat_dim_expr=16, lat_dim_id=32, lat_dim_glob_shape=16, lat_dim_loc_shape=8,
                             n_loc=39, anchors=mean_anchors(), hidden_dim=64, nlayers=4, out_dim=3, input_dim=3)
    return dec, dfn.double().eval()


def _subjects():
    """Five subjects with 1 to 4 expressions; only subject 0 has 1000 points or more per observation (all observations of a
    subject with fewer have the same number: the sampled rows are stacked)."""
    g = torch.Generator().manual_seed(0)
    sizes = [(1000, 1100, 1050), (300, 300), (400,), (150, 150, 150, 150), (200, 200)]
    return [[torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.1 for n in s] for s in sizes]


@pytest.fixture
def float64():
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    yield
    torch.set_default_dtype(old)


def _fit(kind, decoders, subjects, lambdas, **kw):
    from nphm_b200 import fitting_sharded as S
    from nphm_b200.models import fitting as F
    dec, dfn = decoders
    if kind == 'identity':
        fn = S.inference_identity_space_batched_sharded if kw else F.inference_identity_space_batched
        return fn(dec, subjects, lambdas, N_STEPS, SCHEDULE, step_scale=STEP_SCALE, **kw)
    fn = S.inference_iterative_root_finding_joint_batched_sharded if kw else F.inference_iterative_root_finding_joint_batched
    return fn(dec, dfn, subjects, lambdas, N_STEPS, SCHEDULE, step_scale=STEP_SCALE, **kw)


def _lambdas(kind):
    return dict(LAMBDAS_ID if kind == 'identity' else LAMBDAS)


def _reference(kind):
    """(results, generator state, lambdas) of the one-process batched call from seed 0, and the lambdas of one call."""
    subjects, decoders = _subjects(), _decoders()
    torch.manual_seed(0)
    lam = _lambdas(kind)
    out = _fit(kind, decoders, subjects, lam)
    return out, torch.get_rng_state(), lam


def _sharded(kind, batch_size, group=None):
    subjects, decoders = _subjects(), _decoders()
    torch.manual_seed(0)
    lam = _lambdas(kind)
    out = _fit(kind, decoders, subjects, lam, group=group, batch_size=batch_size)
    return out, torch.get_rng_state(), lam


def _assert_same(got, want):
    assert len(got[0]) == len(want[0])
    for a, b in zip(got[0], want[0]):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert (x is None) == (y is None)
            if x is not None:
                assert x.shape == y.shape and x.dtype == y.dtype and x.requires_grad == y.requires_grad
                assert torch.equal(x.detach(), y.detach())
    assert torch.equal(got[1], want[1])
    assert got[2] == want[2]


# ---------------------------------------------------------------------------------------------- the plan
@pytest.mark.parametrize('costs,batch_size', [([1] * 17, 4), ([1] * 5, 8), ([3, 1, 4, 1, 5, 9, 2, 6, 5, 3, 5], 2),
                                              ([2, 7, 1, 8, 2, 8, 1, 8], 3), ([1], 1), ([], 3)])
def test_plan_chunks_do_not_depend_on_the_world(costs, batch_size):
    from nphm_b200.fitting_sharded import fit_owner, plan_fit_chunks
    n = len(costs)
    want = [(lo, min(lo + batch_size, n)) for lo in range(0, n, batch_size)]
    for world in range(1, 10):
        plan = plan_fit_chunks(costs, batch_size, world)
        assert plan.chunks == want, world
        assert plan == plan_fit_chunks(list(costs), batch_size, world)
        assert len(plan.owners) == len(want) and all(0 <= r < world for r in plan.owners)
        load = [0] * world
        for (lo, hi), r in zip(plan.chunks, plan.owners):
            load[r] += sum(costs[lo:hi])
        chunk_costs = [sum(costs[lo:hi]) for lo, hi in plan.chunks] or [0]
        bound = max(sum(costs) / world, max(chunk_costs))        # no schedule does better than this
        assert max(load) <= bound + max(chunk_costs), (world, load)
        if world >= len(want):                                   # more ranks than chunks: one chunk per rank at most
            assert sorted(plan.owners) == list(range(len(want)))
        for k in range(n):
            lo, hi = plan.chunks[k // batch_size]
            assert fit_owner(plan, k) == plan.owners[k // batch_size] and lo <= k < hi
    with pytest.raises(IndexError):
        fit_owner(plan_fit_chunks(costs, batch_size, 2), n)


def test_plan_is_longest_processing_time_first():
    from nphm_b200.fitting_sharded import plan_fit_chunks
    # chunk costs 1, 5, 3, 3, taken 5, 3, 3, 1 (the tie in chunk order): 5 -> rank 0, 3 -> rank 1, 3 -> rank 1 (3 < 5),
    # 1 -> rank 0 (5 < 6)
    plan = plan_fit_chunks([1, 5, 3, 3], 1, 2)
    assert plan.owners == [0, 0, 1, 1]
    with pytest.raises(ValueError):
        plan_fit_chunks([1, 2], 0, 2)
    with pytest.raises(ValueError):
        plan_fit_chunks([1, 2], 1, 0)


# ---------------------------------------------------------------------------------------------- one process
@pytest.mark.parametrize('kind', ['identity', 'joint'])
def test_world_one_equals_the_batched_call(kind, float64):
    want = _reference(kind)
    for batch_size in BATCH_SIZES:
        _assert_same(_sharded(kind, batch_size), want)
    # the caller's lambdas end as one single-subject call leaves them
    from nphm_b200.models import fitting as F
    dec, dfn = _decoders()
    one = _lambdas(kind)
    if kind == 'identity':
        F.inference_identity_space(dec, _subjects()[2], one, N_STEPS, SCHEDULE, step_scale=STEP_SCALE)
    else:
        F.inference_iterative_root_finding_joint(dec, dfn, _subjects()[2], one, N_STEPS, SCHEDULE, step_scale=STEP_SCALE)
    assert want[2] == one != _lambdas(kind)


def test_the_batched_fitter_gets_the_chunks_and_their_generators(float64, monkeypatch):
    """Where a batched fitter takes the decoder (on the GPU) it receives the plan's chunks, each subject's generator in the
    state its sequential fit starts from, and a fresh copy of the lambdas.  A stand-in fitter records them and fits each
    subject with the single-subject function from that state."""
    from nphm_b200.models import fitting as F
    dec, _ = _decoders()
    torch.manual_seed(0)
    starts = []
    for s in _subjects():                                # the state each sequential fit starts from
        starts.append(torch.get_rng_state())
        F.inference_identity_space(dec, s, dict(LAMBDAS_ID), N_STEPS, SCHEDULE, step_scale=STEP_SCALE)
    want = _reference('identity')
    calls = []

    def batch_fit(dec_, scans, n_steps, schedule_cfg, step_scale, lr_scale):
        def fit(chunk, gens, lambdas):
            calls.append(([g.get_state() for g in gens], dict(lambdas)))
            out = []
            for all_obs, g in zip(chunk, gens):
                torch.set_rng_state(g.get_state())
                out.append(F.inference_identity_space(dec_, all_obs, dict(lambdas), n_steps, schedule_cfg, step_scale,
                                                      lr_scale))
            lambdas['surface'] = -1.0                    # what a fit does to its copy stays there
            return out
        return fit
    monkeypatch.setattr(F, '_identity_batch_fit', batch_fit)
    _assert_same(_sharded('identity', 2), want)
    assert [len(states) for states, _ in calls] == [2, 2, 1]
    assert all(lam == LAMBDAS_ID for _, lam in calls)
    states = [st for sts, _ in calls for st in sts]
    assert len(states) == len(starts) and all(torch.equal(a, b) for a, b in zip(states, starts))


def test_no_subjects_and_no_iterations(float64):
    from nphm_b200.fitting_sharded import inference_identity_space_batched_sharded
    dec, _ = _decoders()
    lam = dict(LAMBDAS_ID)
    assert inference_identity_space_batched_sharded(dec, [], lam, N_STEPS, SCHEDULE, step_scale=STEP_SCALE) == []
    assert lam == LAMBDAS_ID
    with pytest.raises(ValueError, match='no iteration'):
        inference_identity_space_batched_sharded(dec, _subjects()[:1], lam, 10, SCHEDULE, step_scale=STEP_SCALE)


# ---------------------------------------------------------------------------------------------- gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _to_host(res):
    out, state, lam = res
    return ([tuple(None if t is None else (t.detach().numpy(), t.requires_grad) for t in r) for r in out], state.numpy(),
            lam)


def _from_host(res):
    out, state, lam = res
    return ([tuple(None if t is None else torch.from_numpy(t[0]).requires_grad_(t[1]) for t in r) for r in out],
            torch.from_numpy(state), lam)


def _gloo_worker(rank, world, port, jobs, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.set_default_dtype(torch.float64)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        for kind, batch_size, bad in jobs:
            subjects, decoders = _subjects(), _decoders()
            lam = _lambdas(kind)
            if bad == 'points' and rank == world - 1:
                subjects[3][1] = subjects[3][1][:100]
            if bad == 'lambdas' and rank == world - 1:
                lam['reg_global'] *= 2
            torch.manual_seed(0)
            try:
                out = _fit(kind, decoders, subjects, lam, batch_size=batch_size)
            except ValueError as e:
                q.put((rank, kind, batch_size, 'ValueError: %s' % e))
                continue
            q.put((rank, kind, batch_size, _to_host((out, torch.get_rng_state(), lam))))
    finally:
        dist.destroy_process_group()


def _gloo(world, jobs):
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, jobs, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = collect(q, procs, world * len(jobs))
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    out = {}
    for rank, kind, batch_size, r in res:
        out.setdefault((kind, batch_size), {})[rank] = r
    return out


@pytest.mark.parametrize('world', [2, 3])
def test_gloo_ranks_equal_the_batched_call(world, float64):
    """Every rank gets every subject's result bit for bit, for chunk sizes that give one chunk per subject, chunks of two with a
    shorter last one, and one chunk for all (ranks without a chunk)."""
    jobs = [(kind, b, None) for kind in ('identity', 'joint') for b in BATCH_SIZES]
    out = _gloo(world, jobs)
    for kind in ('identity', 'joint'):
        want = _reference(kind)
        for b in BATCH_SIZES:
            for r in range(world):
                got = out[kind, b][r]
                assert not isinstance(got, str), got
                _assert_same(_from_host(got), want)


def test_gloo_ranks_called_differently_raise():
    out = _gloo(2, [('identity', 2, 'points'), ('joint', 2, 'lambdas')])
    for kind in ('identity', 'joint'):
        for r in range(2):
            msg = out[kind, 2][r]
            assert isinstance(msg, str) and msg.startswith('ValueError') and 'ranks [1]' in msg, msg
