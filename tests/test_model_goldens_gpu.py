"""GPU: the CUDA models of the five original builders against the MODEL-level golden vectors produced by the
reference's own unmodified feature_column.py / inputs.py / builders (tests/golden/models/*.npz,
tests/golden/generate_models.py), with model_golden_checks' forward and one-SGD-step checks (shared by every
fixture family): the reference's weights loaded by name, the same inputs, then

* logits and predictions within 1e-4 relative (north_star), in both GEMM precisions;
* one SGD step: the loss and every weight's update  -lr * dL/dw  against the gradient torch autograd
  took THROUGH the reference's graph (tables included: dense Keras semantics).
"""
import model_golden_checks as C

T = C.gpu_model_tests("models")
test_model_forward_matches_reference = T.forward
test_model_sgd_step_matches_reference_gradients = T.sgd_step
