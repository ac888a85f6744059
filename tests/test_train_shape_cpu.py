"""CPU check of the composite path of nphm_b200.models.loss_functions.actual_compute_loss on the DeepSDF mirror against one
stage-1 step of the reference (loss_functions.py:20-110 + backward, tests/golden/train_shape.npz from
make_golden_train_shape.py): same initial weights (state-dict sha256), loss terms, code and bias gradients, weight-gradient
samples, max-abs and norms.  The native path is checked against the same golden on the GPU (test_gpu_train_shape.py)."""
import shape_common as S
from conftest import load_golden


def test_composite_shape_step_matches_the_reference_golden():
    from nphm_b200.models.deepSDF import DeepSDF
    g = load_golden('train_shape.npz')
    dec = S.make_decoder(DeepSDF)
    assert S.state_dict_sha256(dec) == str(g['sha256'])
    losses, codes = S.run_step(dec, g, 'cpu', native=False)
    full, sampled = S.gradient_record(dec, codes)
    S.check_against_golden(g, losses, full, sampled, rtol=1e-4, native=False)
