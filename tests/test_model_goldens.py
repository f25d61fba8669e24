"""CPU: model-level pinning of the five original builders (DeepFM, xDeepFM, DCN, AutoInt, DIN).

The fixtures under tests/golden/models/ were produced by the REFERENCE's own composition code
(deepctr/{feature_column,inputs}.py + the five builders, unmodified) under the torch-backed TF shim
(tests/golden/generate_models.py).  The checks are model_golden_checks' (shared by every fixture family):
oracle/models.py reproduces their logits, predictions, loss and every weight gradient, and the deepctr_b200
builders create exactly the reference's weight set (names, shapes, trainable flags, order).  The builder graphs and
keyword defaults are checked in tests/test_reference_builders_dropin.py.
"""
import numpy as np

import model_golden_checks as C

T = C.model_tests("models")
test_fixture_set_covers_the_five_builders = T.fixture_set
test_oracle_matches_reference_model = T.oracle
test_builders_create_the_reference_weight_set = T.weight_set


def test_hash_tf_documentation_example():
    """Third-party known-answer test for FarmHash Fingerprint64: the TensorFlow API documentation of
    tf.strings.to_hash_bucket_fast gives  to_hash_bucket_fast(["Hello", "TensorFlow", "2.x"], 3) -> [0, 2, 2]
    (1 of the 3 buckets per string: a weak pin, but it is the only published vector available offline).
    Checked for the oracle's restatement and the product's independent host copy."""
    from oracle import farmhash
    from deepctr_b200.layers.utils import host_hash_array
    strings = ["Hello", "TensorFlow", "2.x"]
    assert [farmhash.fingerprint64(s.encode()) % 3 for s in strings] == [0, 2, 2]
    got = host_hash_array(np.array(strings), 3, False, None, 0)
    assert np.asarray(got).reshape(-1).tolist() == [0, 2, 2]
