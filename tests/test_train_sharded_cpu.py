"""CPU checks of the data-parallel training steps (nphm_b200.training_sharded) on the composite path in float64: the rows of
each batch split over 1, 2, 3, 5 and 7 shards (one-row shards at 5, empty ones at 7 with B = 5), in one process
(LocalTrainGroup) and over gloo ranks, against the one-process step of the reference trainer, for both stages and both
decoders of each."""
import os
import socket

import pytest
import torch

import train_sharded_common as T

STEPS = 3
B = 5


def _run(kind, world, batches, val=False):
    """(returned dicts, state, last reduced gradients) after the steps; world None: the one-process trainer."""
    from nphm_b200.training_sharded import LocalTrainGroup, train_step_sharded, val_step_sharded
    tr = T.make_trainer(kind, val_batches=batches if val else ())
    torch.manual_seed(123)
    outs = []
    for epoch, b in enumerate(batches if not val else range(2)):
        if val:
            outs.append(tr.compute_val_loss(epoch) if world is None else val_step_sharded(tr, epoch, LocalTrainGroup(world)))
        elif world is None:
            outs.append(tr.train_step(dict(b), epoch))
        else:
            outs.append(train_step_sharded(tr, dict(b), epoch, LocalTrainGroup(world)))
    return outs, T.state(tr), (None if val else T.reduced_grads(tr))


def _check_against_one_process(got, want, rtol=1e-12):
    for a, b in zip(got[0], want[0]):
        assert list(a) == list(b)
        for k in b:
            assert abs(a[k] - b[k]) <= rtol * abs(b[k]) + 1e-300, (k, a[k], b[k])
    for k, v in want[1].items():
        if k.startswith('rng'):
            assert torch.equal(got[1][k], v), k
        else:
            assert T.rel_err(got[1][k], v) <= rtol, (k, T.rel_err(got[1][k], v))
    if want[2] is not None:
        for k, v in want[2].items():
            assert T.rel_err(got[2][k], v) <= rtol, (k, T.rel_err(got[2][k], v))


@pytest.fixture(scope='module')
def one_process():
    cache = {}

    def get(kind, batch_size=B):
        if (kind, batch_size) not in cache:
            batches = [T.make_batch(kind, batch_size, seed) for seed in range(STEPS)]
            cache[kind, batch_size] = batches, _run(kind, None, batches)
        return cache[kind, batch_size]
    return get


@pytest.mark.parametrize('world', [1, 2, 3, 5, 7])
@pytest.mark.parametrize('kind', T.KINDS)
def test_local_group_matches_one_process(kind, world, one_process):
    batches, want = one_process(kind)
    got = _run(kind, world, batches)
    _check_against_one_process(got, want)


def test_one_row_shards_and_uneven_splits_use_every_row(one_process):
    """B = 5 over 2 and 3 shards is uneven; a change in the stage-2 rows that only one shard holds must move the result."""
    batches, want = one_process('compress')
    moved = [dict(b) for b in batches]
    moved[0]['points_posed'] = moved[0]['points_posed'].clone()
    moved[0]['points_posed'][4] += 0.1                      # the last row: the last shard's, for every world
    for world in (2, 3):
        got = _run('compress', world, moved)
        assert abs(got[0][0]['corresp'] - want[0][0]['corresp']) > 1e-6 * abs(want[0][0]['corresp'])


@pytest.mark.parametrize('kind', ['nphm', 'compress'])
def test_validation_step(kind):
    """Eval mode: the ensemble's last-point quirk per batch row, SparseAdam on the validation codes."""
    batches = [T.make_batch(kind, B, 10 + s) for s in range(2)]
    want = _run(kind, None, batches, val=True)
    for world in (2, 5):
        got = _run(kind, world, batches, val=True)
        _check_against_one_process(got, want)


def test_the_ensemble_quirk_stays_with_its_row():
    """Without the quirk (training mode) the eval-mode loss differs: the quirk changes what each shard evaluates."""
    from nphm_b200.training_sharded import LocalTrainGroup, val_step_sharded
    batches = [T.make_batch('nphm', B, 20)]
    tr = T.make_trainer('nphm', val_batches=batches)
    got = val_step_sharded(tr, 0, LocalTrainGroup(3))
    tr2 = T.make_trainer('nphm', val_batches=batches)
    tr2.decoder.train()
    losses = tr2.losses(batches[0], tr2.latent_codes_val, None, None)
    assert abs(got['surf_sdf'] - losses['surf_sdf'].item()) > 1e-9


# ---------------------------------------------------------------------------------------------- gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_worker(rank, world, port, jobs, q):
    import torch.distributed as dist
    from nphm_b200.training_sharded import train_step_sharded
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        for kind, batch_size, bad in jobs:
            tr = T.make_trainer(kind)
            torch.manual_seed(123)
            outs = []
            try:
                for epoch, seed in enumerate(range(STEPS)):
                    b = T.make_batch(kind, batch_size, seed)
                    if bad and rank == world - 1:
                        b['idx'] = b['idx'].flip(0)
                    outs.append(train_step_sharded(tr, b, epoch))
            except ValueError as e:
                q.put((rank, kind, batch_size, 'ValueError: %s' % e))
                continue
            q.put((rank, kind, batch_size, (outs, T.to_host(T.state(tr)), T.to_host(T.reduced_grads(tr)))))
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
        res = T.collect(q, procs, world * len(jobs))
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
        if not isinstance(r, str):
            r = (r[0], T.from_host(r[1]), T.from_host(r[2]))
        out.setdefault((kind, batch_size), {})[rank] = r
    return out


def test_gloo_ranks_equal_the_local_group_bit_for_bit(one_process):
    """Three gloo processes: every rank ends with the same state bit for bit, which is LocalTrainGroup(3)'s; with B = 2 one
    rank holds no rows and still joins the collectives and the random draws."""
    jobs = [(k, B, False) for k in T.KINDS] + [('compress', 2, False)]
    out = _gloo(3, jobs)
    for kind, batch_size, _ in jobs:
        ranks = out[kind, batch_size]
        batches, want = one_process(kind, batch_size)
        local = _run(kind, 3, batches)
        for r in range(3):
            assert ranks[r][0] == local[0], (kind, r)
            T.assert_bitwise(ranks[r][1], local[1])
            T.assert_bitwise(ranks[r][2], local[2])
        _check_against_one_process(ranks[0], want)


def test_gloo_ranks_with_different_batches_raise():
    out = _gloo(2, [('npm', B, True)])
    for r in range(2):
        msg = out['npm', B][r]
        assert isinstance(msg, str) and 'different batch' in msg, msg
