"""TEST INFRASTRUCTURE - the EDCN model-fixture family (tests/golden/models_edcn, written by
tests/golden/generate_edcn.py): how a fixture's weights map onto tests/edcn_oracle.py, and its record in
golden_models.FAMILIES, added when this module is imported so that model_golden_checks.model_tests("edcn") and
gpu_model_tests("edcn") find it."""
import golden_models as G


def edcn_weights(fx, requires_grad=False):
    """golden_models.oracle_weights plus the gates, the per-layer CrossNet / DNN weights and the bridges' nested
    weights, in creation order."""
    W, leaves = G.oracle_weights(fx, requires_grad)

    def t(key):
        return G._leaf(fx, leaves, key, requires_grad)

    def numbered(prefix):
        n = len([k for k in fx.w if k.startswith(prefix + "kernel")])
        return [t("%skernel%d" % (prefix, i)) for i in range(n)], [t("%sbias%d" % (prefix, i)) for i in range(n)]

    W["regulation"] = [t("%s/%s_field_weight" % (n, n)) for n in fx.layer_names("RegulationModule")]
    W["cross"] = [numbered(n + "/") for n in fx.layer_names("CrossNet")]
    W["deep"] = []
    for n in fx.layer_names("DNN"):
        k, b = numbered(n + "/")
        bn = {p: t("%s/bn0/%s" % (n, p)) for p in ("gamma", "beta")} if n + "/bn0/gamma" in fx.w else None
        W["deep"].append((k, b, bn))
    W["bridges"] = []
    for n in fx.layer_names("BridgeModule"):
        d = {}
        if n + "/dense/kernel" in fx.w:
            d["dense"] = (t(n + "/dense/kernel"), t(n + "/dense/bias"))
        for sub in ("dense_x", "dense_h"):
            if "%s/%s/kernel0" % (n, sub) in fx.w:
                d[sub] = numbered("%s/%s/" % (n, sub))
        W["bridges"].append(d)
    return W, leaves


def edcn_forward(fx, W):
    import edcn_oracle as EO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return EO.edcn(fx.inputs(), G.columns(fx, "linear", FC), G.columns(fx, "dnn", FC), W,
                   cross_num=kw.get("cross_num", 2), parameterization=kw.get("cross_parameterization", "vector"),
                   bridge_type=kw.get("bridge_type", "concatenation"), tau=kw.get("tau", 1.0), task=fx.task)


FAMILY = G.Family("models_edcn", "reference_builders_edcn.json", ("EDCN",), edcn_weights, edcn_forward, 9,
                  {"binary", "regression"},
                  # every layer's gate is created with its block; the graph reaches each gate next to its consumer
                  graph_weight_order=("edcn_attention_pooling", "edcn_concatenation", "edcn_defaults", "edcn_dnn_bn",
                                      "edcn_hadamard_product", "edcn_pointwise_addition", "edcn_regression",
                                      "edcn_tau_half", "edcn_varlen"))
G.FAMILIES.setdefault("edcn", FAMILY)
