"""GPU: the CUDA layers against the golden vectors produced by the REFERENCE's own layer code
(tests/golden/*.npz, see tests/golden/generate.py) - same constructor arguments, same inputs, the
reference's weights loaded by name (model_golden_checks' layer check).  fp32 tolerance 1e-4 relative (north_star).
CPU: the set holds the fixtures and layers its record in golden_models.LAYER_SETS names."""
import os

import numpy as np
import pytest

import model_golden_checks as C

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

test_layer_matches_reference_output = C.gpu_layer_test("root")
test_fixture_set = C.layer_tests("root").fixture_set


@pytest.mark.gpu
@pytest.mark.usefixtures("gemm_precision")
def test_hash_known_answer_vector(cuda, tmp_path):
    """tests/layers/utils_test.py:20-22 through this package's Hash layer."""
    from deepctr_b200.layers import Hash
    d = np.load(os.path.join(GOLD, "hash_vocab_kat.npz"))
    p = tmp_path / "vocab.csv"
    p.write_text(str(d["vocab"]))
    out = Hash(num_buckets=4, vocabulary_path=str(p))([[k] for k in d["keys"]])
    assert np.asarray(out).tolist() == d["out"].tolist()
