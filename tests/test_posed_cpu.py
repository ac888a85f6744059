"""The composite posed SDF (get_logits_posed on CPU tensors: the mirror's `search` and modules) against the reference's own
composition (tests/golden/posed.npz)."""
import numpy as np
import pytest
import torch

from posed_common import check_against_golden, ensemble_case, npm_case
from nphm_b200.models.reconstruction import _quirk_rows, get_logits_posed


@pytest.mark.parametrize('training', [True, False])
def test_composite_posed_logits_match_reference(training):
    dec, dfn, lat, z_ex, grid, g = ensemble_case(training=training)
    nb = int(g['nbatch_points'])
    sdf, valid = get_logits_posed(dec, dfn, lat, z_ex, grid, nbatch_points=nb, return_valid=True)
    assert sdf.dtype == np.float32 and sdf.shape == (2, grid.shape[1])
    ref = g['sdf_train'] if training else g['sdf_eval']
    check_against_golden(sdf, valid, ref, g['valid'])
    if not training:
        # the eval-mode quirk rows are the last rows of the chunks, and only those differ from the train-mode values
        rows = _quirk_rows(grid.shape[1], nb)
        assert list(rows) == [nb - 1, 2 * nb - 1, grid.shape[1] - 1]
        differ = np.flatnonzero((g['sdf_train'] != g['sdf_eval']).any(0))
        assert set(differ) <= set(rows) and len(differ) > 0


def test_composite_posed_logits_npm_match_reference():
    dec, expr, lat, z_ex, pts, g = npm_case()
    sdf, valid = get_logits_posed(dec, expr, lat, z_ex, pts, nbatch_points=1000, return_valid=True)
    check_against_golden(sdf, valid, g['npm_sdf'], g['npm_valid'])


def test_posed_code_shapes():
    """(E,) gives (N,), (S, 1, E) the same as (S, E)."""
    dec, dfn, lat, z_ex, grid, g = ensemble_case()
    pts = grid[:, :200]
    a = get_logits_posed(dec, dfn, lat, z_ex, pts)
    b = get_logits_posed(dec, dfn, lat, z_ex[:, None], pts)
    c = get_logits_posed(dec, dfn, lat, z_ex[1], pts)
    assert a.shape == (2, 200) and c.shape == (200,)
    assert np.array_equal(a, b) and np.array_equal(a[1], c)

