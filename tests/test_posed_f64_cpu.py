"""The float64 posed reference of tests/posed_f64_common.py against the mirror's modules, in float64 on the CPU (no GPU
needed): its condition rows equal DeformationNetwork._condition, its polished roots solve the modules' x + F(x) = p, and its
identity SDF equals decoder_shape called chunk by chunk as get_logits_posed's reference calls it, eval-mode quirk included.
Every deformation network of the posed float64 test (compress as seeded and with its output layer x 80, expr_only, glob_only)
and the NPM pair."""
import copy

import pytest
import torch

import posed_f64_common as P
from conftest import MAXI, MINI, make_ensemble, sample_latent
from posed_common import npm_case
from nphm_b200.models.iterative_root_finding import search
from nphm_b200.models.reconstruction import _quirk_rows

F64 = torch.float64
CASES = list(P.DEFORMATIONS) + ['npm']


def _double(module):
    m = copy.deepcopy(module).double()
    if getattr(m, 'anchors', None) is not None:
        m.anchors = m.anchors.double()
    return m


def _case(name):
    """(decoder_shape, decoder_expr (both float64), reference params, z_id (D,), z_ex (3 x E)): the seeded ensemble and
    deformation network with 0.1 N(0, 1) codes, or the NPM pair of posed.npz with a third code."""
    if name == 'npm':
        dec, dfn, lat, z_ex, _, _ = npm_case()
        z_ex = torch.cat([z_ex, -2.0 * z_ex[:1]])
    else:
        dec, dfn, lat = make_ensemble(0), P.make_deformation(name), sample_latent(1)
        torch.manual_seed(8)
        z_ex = torch.randn(3, 200) * 0.1
    dec64, dfn64 = _double(dec), _double(dfn)
    return dec64, dfn64, P.Params(dec64, dfn64, F64), lat.reshape(-1).double(), z_ex.double()


def _points(n, seed=0):
    """n points in the head's box grown by half on every side, so that some lie outside it (float64, 1 x n x 3)."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(MINI, dtype=F64), torch.tensor(MAXI, dtype=F64)
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    return (mid + (torch.rand(n, 3, generator=g, dtype=F64) * 2 - 1) * half * 1.5)[None]


def _anchors(dec64, z_id):
    """The anchors the reference's composition hands the deformation network (decoder_shape(0, z_id)[1]), or None."""
    if not hasattr(dec64, 'ensembled_deep_sdf'):
        return None
    with torch.no_grad():
        return dec64(torch.zeros(1, 1, 3, dtype=F64), z_id.reshape(1, 1, -1), None)[1]


def _module_offsets(dfn64, x, glob, anc):
    """F(x) of the float64 deformation module (n x 3) under the code [z_id | z_ex] ``glob`` (1 x 1 x D)."""
    n = x.shape[0]
    with torch.no_grad():
        return dfn64(x[None], glob.expand(1, n, -1), None if anc is None else anc.unsqueeze(1).repeat(1, n, 1, 1))[0][0]


def _close(a, b, rel=1e-12):
    scale = max(float(b.abs().max()), 1e-300)
    assert float((a - b).abs().max()) <= rel * scale, (float((a - b).abs().max()), scale)


@pytest.mark.parametrize('name', CASES)
def test_condition_rows_equal_the_module(name):
    dec64, dfn64, Q, z_id, z_ex = _case(name)
    got = P.condition(Q, z_id, z_ex)
    S = z_ex.shape[0]
    lat = torch.cat([z_id[None].expand(S, -1), z_ex], dim=1)[:, None]
    if name == 'npm':
        want = lat[:, 0]                                   # the NPM expression decoder is conditioned on [z_id | z_ex]
    else:
        anc = _anchors(dec64, z_id).expand(S, -1, -1)
        with torch.no_grad():
            want = dfn64._condition(torch.zeros(S, 1, 3, dtype=F64), lat, anc, per_point=False)[:, 0]
    assert got.shape == want.shape
    _close(got, want)
    if name.startswith('compress'):
        assert got.shape[1] == 232
    elif name in ('expr_only', 'glob_only'):
        assert got.shape[1] == {'expr_only': 200, 'glob_only': 264}[name]


@pytest.mark.parametrize('name', CASES)
def test_polished_roots_solve_the_module(name):
    """From the mirror's own search (float64) to roots whose residual through the modules is below 1e-12."""
    dec64, dfn64, Q, z_id, z_ex = _case(name)
    cond = P.condition(Q, z_id, z_ex)
    p = _points(40, seed=1)
    n = p.shape[1]
    anc = _anchors(dec64, z_id)
    solved = 0
    for s in range(z_ex.shape[0]):
        glob = torch.cat([z_id, z_ex[s]]).reshape(1, 1, -1)
        a = None if anc is None else anc.unsqueeze(1).repeat(1, n, 1, 1)
        xc, res = search(p, glob.repeat(1, n, 1), dfn64, a, multi_corresp=False)
        ok = res['valid_ids'].reshape(-1)
        x = xc.detach().reshape(-1, 3)[ok]
        if x.shape[0] == 0:
            continue
        xs, r = P.polish(Q, x, cond[s:s + 1].expand(x.shape[0], -1), p[0, ok])
        assert float(r.max()) < P.POLISH_TOL
        assert float((xs + _module_offsets(dfn64, xs, glob, anc) - p[0, ok]).norm(dim=-1).max()) < 1e-12
        # the reference's residual at the search's own roots is the module's
        want = x + _module_offsets(dfn64, x, glob, anc) - p[0, ok]
        got = P.residual(Q, x[:, None], cond[s:s + 1].expand(x.shape[0], -1), p[0, ok][:, None])[:, 0]
        assert float((got - want).abs().max()) < 1e-14
        solved += x.shape[0]
    assert solved > 0


@pytest.mark.parametrize('case', ['ensemble-train', 'ensemble-eval', 'npm'])
def test_identity_sdf_equals_the_module(case):
    """The identity SDF at given points equals decoder_shape called in chunks of nbatch_points: in eval mode the last row of
    every chunk and the last row carry the quirk, and the quirk mask is get_logits_posed's."""
    name = 'npm' if case == 'npm' else 'compress'
    dec64, _, Q, z_id, _ = _case(name)
    training = case != 'ensemble-eval'
    dec64.train(training)
    x = _points(50, seed=2)
    n, nb = x.shape[1], 16
    quirk = P.quirk_mask(n, nb)
    assert quirk.nonzero().reshape(-1).tolist() == _quirk_rows(n, nb).tolist()
    want = []
    with torch.no_grad():
        for a in range(0, n, nb):
            chunk = x[:, a:a + nb]
            lat = z_id.reshape(1, 1, -1) if Q.nphm else z_id.reshape(1, 1, -1).expand(1, chunk.shape[1], -1)
            want.append(dec64(chunk, lat, None)[0].reshape(-1))
    want = torch.cat(want)
    got = P.identity_sdf(Q, x[0], z_id, None if training or not Q.nphm else quirk)
    _close(got, want)
    if case == 'ensemble-eval':
        dec64.train(True)
        with torch.no_grad():
            plain = dec64(x, z_id.reshape(1, 1, -1), None)[0].reshape(-1)
        assert bool((plain != want)[quirk].all())
        _close(plain[~quirk], want[~quirk])
    s, g = P.identity_sdf_grad(Q, x[0], z_id, None if training or not Q.nphm else quirk)
    _close(s, want)
    assert g.shape == (n, 3) and bool(torch.isfinite(g).all())
