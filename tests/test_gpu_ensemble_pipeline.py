"""Bit-identity of the tensor-core ensemble kernel against stored outputs (tests/golden/ensemble_pipeline.npz, written by
tests/golden/make_golden_ensemble_pipeline.py): a single tile, three tiles, a ragged last tile, three queries with different
latents, a 64^3 grid slice with the reference's chunk quirk, the pruned kernel, and the fitting surface gradient (activation
dump with members split over CTAs, per-member outputs).  Scheduling changes of the kernel must not change a single bit; only
sums the fitting backward forms with atomics are compared with a tolerance."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))


@pytest.fixture(scope='module')
def outputs(cuda_device):
    import make_golden_ensemble_pipeline as M
    return M.run_cases(cuda_device)


CASES = ['one_tile', 'three_tiles', 'ragged', 'three_latents', 'grid64_quirk', 'grid64_pruned', 'fit_member_s',
         'fit_loss_terms', 'fit_grad_latent', 'fit_grad_points']


@pytest.mark.gpu
@pytest.mark.parametrize('name', CASES)
def test_matches_golden(outputs, name):
    import make_golden_ensemble_pipeline as M
    from conftest import load_golden
    ref = load_golden('ensemble_pipeline.npz')
    assert name in outputs
    assert M.matches(ref, name, outputs[name]), name
