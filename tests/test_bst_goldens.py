"""The BST fixtures made by the reference's own code (tests/golden/generate_bst.py).

Model fixtures: model_golden_checks' checks (shared by every fixture family), bound below; on the GPU,
test_model_fixture_gpu is the one-SGD-step check.
Layer fixtures: model_golden_checks' layer checks, bound below.  CPU: the restatement of tests/bst_oracle.py
reproduces every layer fixture (outputs and all gradients).  GPU: the Transformer / PositionEncoding /
LayerNormalization layers reproduce the fixtures in both GEMM precisions: outputs and gradients.
"""
import golden_models as G
import model_golden_checks as C

T = C.model_tests("bst")
test_oracle_reproduces_model_fixture = T.oracle
test_builder_creates_the_reference_weight_set = T.weight_set
test_builder_carries_the_fixture_weights_and_the_reference_graph = T.graph
test_reference_default_arguments_are_the_same = T.defaults
T = C.gpu_model_tests("bst")
test_model_forward_matches_reference = T.forward
test_model_fixture_gpu = T.sgd_step
L = C.layer_tests("bst")
test_oracle_reproduces_layer_fixture = L.oracle
test_layer_fixture_gpu = C.gpu_layer_test("bst")


def test_fixture_sets():
    C.check_fixture_set(G.FAMILIES["bst"])
    L.fixture_set()
