"""TEST INFRASTRUCTURE - the ONN model-fixture family (tests/golden/models_onn, written by
tests/golden/generate_onn.py): how a fixture's weights map onto tests/onn_oracle.py, and its record in
golden_models.FAMILIES, added when this module is imported so that model_golden_checks.model_tests("onn") and
gpu_model_tests("onn") find it."""
import golden_models as G


def onn_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus W['bn'], the BatchNormalization's gamma and beta when the model has one."""
    W, leaves = G.oracle_weights(fx, requires_grad)
    for n in fx.layer_names("BatchNormalization"):
        W["bn"] = {k: G._leaf(fx, leaves, "%s/%s" % (n, k), requires_grad) for k in ("gamma", "beta")}
    return W, leaves


def onn_forward(fx, W):
    import onn_oracle as OO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return OO.onn(fx.inputs(), G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC), W,
                  use_bn=kw.get("use_bn", True), reduce_sum=kw.get("reduce_sum", False), task=fx.task)


FAMILY = G.Family("models_onn", "reference_builders_onn.json", ("ONN",), onn_weights, onn_forward, 9,
                  {"binary", "regression"},
                  # the reference creates each field's tables together; the graph looks them up pair by pair
                  graph_weight_order=("onn_defaults", "onn_f2", "onn_hashed", "onn_no_bn", "onn_no_dense",
                                      "onn_no_dnn", "onn_reduce_sum", "onn_regression", "onn_varlen"))
G.FAMILIES.setdefault("onn", FAMILY)
