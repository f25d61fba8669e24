"""Shared loader for the MODEL-level golden fixtures (tests/golden/models*/*.npz, produced by the
reference's own feature_column.py / inputs.py / builders under the TF shim: see
tests/golden/generate_*.py), the table of fixture families, the table of LAYER-level fixture sets
(``LAYER_SETS``, tests/golden/*.npz and tests/golden/<set>/*.npz), and the mappings a test needs:

* ``oracle_weights``  fixture weight keys -> the dict oracle/models.py takes;
* ``assign_weights``  fixture weight keys -> the weights of a deepctr_b200 model built from the same columns.

Key convention of the fixtures: ``<top-level layer name>/<reference attribute path>/<weight name>``.
``linearsparse_emb_*`` tables are the reference's redundant second lookup pass inside get_linear_logit
(feature_column.py:185, SURVEY.md App. F.2): their outputs are discarded, their gradient is zero, and
neither the oracle nor this package materialises them.
"""
import glob
import itertools
import json
import os
import re

import numpy as np
import torch

import b2_helpers as H

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MODELS = os.path.join(GOLDEN, "models")


def _cases(models_dir):
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(models_dir, "*.npz")))


CASES = _cases(MODELS)


class Fixture(object):
    def __init__(self, name, models_dir=MODELS):
        d = np.load(os.path.join(models_dir, name + ".npz"))
        self.name = name
        self.meta = json.loads(str(d["meta"]))
        self.x = {k[2:]: d[k] for k in d.files if k.startswith("x_")}
        self.y = d["y"]
        self.w = {k[2:]: d[k] for k in d.files if k.startswith("w_")}
        self.g = {k[2:]: d[k] for k in d.files if k.startswith("g_")}
        self.out, self.logit, self.loss = d["out"], d["logit"], float(d["loss"])
        self.builder, self.kwargs = self.meta["builder"], self.meta["kwargs"]
        self.task = self.meta.get("task", "binary")
        self.training = bool(self.meta.get("training"))

    def layer_names(self, cls):
        return [n for c, n in self.meta["layers"] if c == cls]

    def inputs(self):
        """what a user passes: ints as int32/int64 arrays, strings as str arrays, floats as float32."""
        out = {}
        for k, a in self.x.items():
            out[k] = a.astype(np.int32) if a.dtype.kind in "iu" else a
        return out


def columns(fx, which, FC):
    """Rebuild the feature columns with module ``FC``'s SparseFeat / VarLenSparseFeat / DenseFeat."""
    def sparse(m):
        vp = os.path.join(MODELS, m["vocabulary_path"]) if m["vocabulary_path"] else None
        return FC.SparseFeat(m["name"], m["vocabulary_size"], m["embedding_dim"], use_hash=m["use_hash"],
                             vocabulary_path=vp, dtype=m["dtype"], embedding_name=m["embedding_name"],
                             group_name=m["group_name"], trainable=m["trainable"])
    out = []
    for m in fx.meta["columns"][which]:
        if m["kind"] == "sparse":
            out.append(sparse(m))
        elif m["kind"] == "varlen":
            out.append(FC.VarLenSparseFeat(sparse(m["sparsefeat"]), maxlen=m["maxlen"], combiner=m["combiner"],
                                           length_name=m["length_name"], weight_name=m["weight_name"],
                                           weight_norm=m["weight_norm"]))
        else:
            out.append(FC.DenseFeat(m["name"], m["dimension"]))
    return out


def _ignored(key):
    return key.startswith("linearsparse_")


def oracle_weights(fx, requires_grad=False):
    """-> (W for oracle/models.py, {fixture key: leaf tensor})."""
    leaves = {}

    def t(key):
        return _leaf(fx, leaves, key, requires_grad)

    W = {"tables": {}, "att": []}
    for name in fx.layer_names("Embedding"):
        if not _ignored(name):
            W["tables"][name] = t(name + "/embeddings")
    for name in fx.layer_names("DNN"):
        n = len([k for k in fx.w if k.startswith(name + "/kernel")])
        W["dnn_kernels"] = [t("%s/kernel%d" % (name, i)) for i in range(n)]
        W["dnn_biases"] = [t("%s/bias%d" % (name, i)) for i in range(n)]
    for name in fx.layer_names("Linear"):
        if name + "/linear_kernel" in fx.w:
            W["linear_kernel"] = t(name + "/linear_kernel")
    denses = fx.layer_names("Dense")
    if denses:
        W["dense_kernel"] = t(denses[0] + "/kernel")
    if len(denses) > 1:
        W["cin_dense_kernel"] = t(denses[1] + "/kernel")
    for name in fx.layer_names("PredictionLayer"):
        if name + "/global_bias" in fx.w:
            W["global_bias"] = t(name + "/global_bias")
    for name in fx.layer_names("CIN"):
        n = len([k for k in fx.w if k.startswith(name + "/filter")])
        W["cin_filters"] = [t("%s/filter%d" % (name, i)) for i in range(n)]
        W["cin_biases"] = [t("%s/bias%d" % (name, i)) for i in range(n)]
    for name in fx.layer_names("CrossNet"):
        n = len([k for k in fx.w if k.startswith(name + "/kernel")])
        W["cross_kernels"] = [t("%s/kernel%d" % (name, i)) for i in range(n)]
        W["cross_biases"] = [t("%s/bias%d" % (name, i)) for i in range(n)]
    for name in fx.layer_names("InteractingLayer"):
        d = {"query": t(name + "/query"), "key": t(name + "/key"), "value": t(name + "/value")}
        if name + "/res" in fx.w:
            d["res"] = t(name + "/res")
        W["att"].append(d)
    for name in fx.layer_names("AttentionSequencePoolingLayer"):
        p = name + "/local_att/"
        n = len([k for k in fx.w if k.startswith(p + "dnn/kernel")])
        d = {"dnn_kernels": [t("%sdnn/kernel%d" % (p, i)) for i in range(n)],
             "dnn_biases": [t("%sdnn/bias%d" % (p, i)) for i in range(n)],
             "kernel": t(p + "kernel"), "bias": t(p + "bias")}
        acts = []
        for i in range(n):
            a = "%sdnn/activation_layers%d/" % (p, i)
            if a + "dice_alpha" in fx.w:
                acts.append({"alphas": t(a + "dice_alpha"), "moving_mean": t(a + "bn/moving_mean"),
                             "moving_var": t(a + "bn/moving_variance")})
            else:
                acts.append(None)
        if any(a is not None for a in acts):
            d["act_params"] = acts
        W["lau"] = d
    return W, leaves


def oracle_forward(fx, W):
    """(logit, prediction) of oracle/models.py for this fixture's builder + kwargs."""
    from oracle import models as OM
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    x = fx.inputs()
    lin, dnn = columns(fx, "linear", FC), columns(fx, "dnn", FC)
    b = fx.builder
    if b == "DeepFM":
        return OM.deepfm(x, lin, dnn, W, fm_group=tuple(kw.get("fm_group", ("default_group",))), task=fx.task)
    if b == "xDeepFM":
        return OM.xdeepfm(x, lin, dnn, W, cin_layer_size=tuple(kw["cin_layer_size"]),
                          cin_split_half=kw["cin_split_half"], cin_activation=kw["cin_activation"], task=fx.task)
    if b == "DCN":
        return OM.dcn(x, lin, dnn, W, cross_num=kw["cross_num"], parameterization=kw["cross_parameterization"],
                      use_dnn=len(kw["dnn_hidden_units"]) > 0, task=fx.task)
    if b == "AutoInt":
        return OM.autoint(x, lin, dnn, W, att_layer_num=kw["att_layer_num"],
                          att_embedding_size=kw["att_embedding_size"], att_head_num=kw["att_head_num"],
                          att_res=kw["att_res"], use_dnn=len(kw["dnn_hidden_units"]) > 0, task=fx.task)
    if b == "DIN":
        return OM.din(x, dnn, ["item_id", "cate_id"], W, att_activation=kw["att_activation"],
                      att_weight_normalization=kw["att_weight_normalization"], task=fx.task,
                      training=fx.training)
    raise KeyError(b)


def loss_of(fx, pred):
    """Keras binary_crossentropy on probabilities / mse (SURVEY.md App. C)."""
    from oracle import ops as O
    if fx.task == "binary":
        return O.binary_crossentropy(fx.y, pred)
    y = torch.as_tensor(fx.y).reshape(-1, 1)
    return ((pred - y) ** 2).mean()


# ---- deepctr_b200 side -------------------------------------------------------------------------------
_RENAMES = [("/local_att/", "/local_activation_unit/"), ("/activation_layers", "/act")]


def builder_args(fx):
    """(positional, keyword) arguments of the fixture's builder call."""
    from deepctr_b200 import feature_column as FC
    kw = dict(fx.kwargs)
    for k in ("dnn_hidden_units", "cin_layer_size", "att_hidden_size", "fm_group"):
        if k in kw:
            kw[k] = tuple(kw[k])
    dnn = columns(fx, "dnn", FC)
    if fx.builder in ("DIN", "BST"):
        return (dnn, ["item_id", "cate_id"]), kw
    if fx.builder == "PNN":                  # PNN(dnn_feature_columns, **kwargs) (pnn.py:18)
        return (dnn,), kw
    return (columns(fx, "linear", FC), dnn), kw


def build(fx):
    """Build the deepctr_b200 model of this fixture (graph construction only: works without a GPU)."""
    from deepctr_b200 import engine as E
    from deepctr_b200 import models as M
    args, kw = builder_args(fx)
    E.clear_session()
    return getattr(M, fx.builder)(*args, **kw)


def signature(model):
    """What reference_builders*.json records of a built graph: inputs, layers, weights, planner slots."""
    from deepctr_b200 import engine as E
    layers = [(type(l).__name__, l.name) for l in model.layers if not isinstance(l, E.InputLayer)]
    weights = [(w.name, tuple(w.shape), w.trainable) for w in model.weights]
    slots = [(s.emb.name, s.input_name, s.maxlen, s.pool, s.mask_mode, s.len_name, s.weight_name, s.weight_mode,
              s.dim, s.buf, s.col) for s in model.planner.slots]
    sig = {"inputs": list(model.input_names), "layers": layers, "weights": weights, "slots": slots,
           "fast": (model.planner.fast, getattr(model.planner, "fast_n", 0))}
    return json.loads(json.dumps(sig))      # tuples -> lists, as stored


def weight_map(fx, model):
    """{fixture key: deepctr_b200 Weight}; raises if the two weight sets differ (names or shapes)."""
    mine = {w.name: w for w in model.weights}
    out, missing = {}, []
    for key, val in fx.w.items():
        if _ignored(key):
            continue
        k2 = key
        for a, b in _RENAMES:
            k2 = k2.replace(a, b)
        if k2 not in mine:
            missing.append((key, k2))
            continue
        if tuple(mine[k2].shape) != tuple(val.shape):
            raise AssertionError("shape of %s: reference %s, here %s" % (key, val.shape, mine[k2].shape))
        out[key] = mine.pop(k2)
    if missing or mine:
        raise AssertionError("weight sets differ: reference-only %s, here-only %s" % (missing, sorted(mine)))
    return out


def assign_weights(fx, model):
    wm = weight_map(fx, model)
    for key, w in wm.items():
        w.set_value(fx.w[key])
    return wm


# ---- the fixture families -----------------------------------------------------------------------------
def _leaf(fx, leaves, key, requires_grad):
    v = torch.tensor(fx.w[key], requires_grad=requires_grad and key in fx.g)
    leaves[key] = v
    return v


def _pairwise_weights(fx, requires_grad=False):
    """oracle_weights plus the AFMLayer weights (one dict per layer, in graph order)."""
    W, leaves = oracle_weights(fx, requires_grad)
    W["afm"] = [{k: _leaf(fx, leaves, "%s/%s" % (name, k), requires_grad)
                 for k in ("attention_W", "attention_b", "projection_h", "projection_p")}
                for name in fx.layer_names("AFMLayer")]
    return W, leaves


def _pairwise_forward(fx, W):
    import pairwise_oracle as PO
    from deepctr_b200 import feature_column as FC
    x = fx.inputs()
    lin, dnn = columns(fx, "linear", FC), columns(fx, "dnn", FC)
    if fx.builder == "NFM":
        return PO.nfm(x, lin, dnn, W, task=fx.task)
    kw = fx.kwargs
    fm_group = kw.get("fm_group", "default_group")
    return PO.afm_model(x, lin, dnn, W, fm_group=tuple(fm_group) if isinstance(fm_group, list) else fm_group,
                        use_attention=kw.get("use_attention", True), task=fx.task)


def _creation_order(name):
    m = re.search(r"_(\d+)$", name)
    return int(m.group(1)) if m else 0


def _fibinet_weights(fx, requires_grad=False):
    """oracle_weights plus the SENET weights and the two bilinear layers' weights (SENET branch first: the layer
    created first)."""
    W, leaves = oracle_weights(fx, requires_grad)
    senet = fx.layer_names("SENETLayer")[0]
    W["senet"] = (_leaf(fx, leaves, senet + "/W_1", requires_grad), _leaf(fx, leaves, senet + "/W_2", requires_grad))
    W["bilinear"] = [[_leaf(fx, leaves, k, requires_grad) for k in fx.w if k.startswith(name + "/bilinear_weight")]
                     for name in sorted(fx.layer_names("BilinearInteraction"), key=_creation_order)]
    W.setdefault("dnn_kernels", [])
    W.setdefault("dnn_biases", [])
    return W, leaves


def _fibinet_forward(fx, W):
    import fibinet_oracle as FO
    from deepctr_b200 import feature_column as FC
    lin, dnn = columns(fx, "linear", FC), columns(fx, "dnn", FC)
    return FO.fibinet(fx.inputs(), lin, dnn, W, bilinear_type=fx.kwargs.get("bilinear_type", "interaction"),
                      task=fx.task)


def _fefm_weights(fx, requires_grad=False):
    """oracle_weights plus W['fwfm'] (each FwFMLayer's strengths, in creation order) or W['fefm'] (the FEFMLayer's
    P matrices, in itertools.combinations order)."""
    W, leaves = oracle_weights(fx, requires_grad)
    W["fwfm"] = [_leaf(fx, leaves, n + "/field_pair_strengths", requires_grad) for n in fx.layer_names("FwFMLayer")]
    for n in fx.layer_names("FEFMLayer"):
        F = int(round((1 + np.sqrt(1 + 8 * len([k for k in fx.w if k.startswith(n + "/")]))) / 2))
        W["fefm"] = [_leaf(fx, leaves, "%s/field_embeddings%d-%d" % (n, i, j), requires_grad)
                     for i, j in itertools.combinations(range(F), 2)]
    return W, leaves


def _fefm_forward(fx, W):
    import fefm_oracle as FO
    from deepctr_b200 import feature_column as FC
    lin, dnn = columns(fx, "linear", FC), columns(fx, "dnn", FC)
    kw = fx.kwargs
    if fx.builder == "FwFM":
        return FO.fwfm_model(fx.inputs(), lin, dnn, W, fm_group=tuple(kw.get("fm_group", ("default_group",))),
                             task=fx.task)
    return FO.deepfefm(fx.inputs(), lin, dnn, W, use_fefm=kw.get("use_fefm", True),
                       use_linear=kw.get("use_linear", True),
                       use_fefm_embed_in_dnn=kw.get("use_fefm_embed_in_dnn", True),
                       exclude_feature_embed_in_dnn=kw.get("exclude_feature_embed_in_dnn", False), task=fx.task)


def _pnn_weights(fx, requires_grad=False):
    """oracle_weights plus W['outer'], the OutterProductLayer kernel when it is on the output path."""
    W, leaves = oracle_weights(fx, requires_grad)
    for n in fx.layer_names("OutterProductLayer"):
        W["outer"] = _leaf(fx, leaves, n + "/kernel", requires_grad)
    return W, leaves


def _pnn_forward(fx, W):
    import pnn_oracle as PO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return PO.pnn(fx.inputs(), columns(fx, "dnn", FC), W, use_inner=kw.get("use_inner", True),
                  use_outter=kw.get("use_outter", False), kernel_type=kw.get("kernel_type", "mat"), task=fx.task)


def _ifm_weights(fx, requires_grad=False):
    """oracle_weights plus W['m_kernels'], the Dense(F) kernels in creation order."""
    W, leaves = oracle_weights(fx, requires_grad)
    W["m_kernels"] = [leaves[n + "/kernel"] if n + "/kernel" in leaves else
                      _leaf(fx, leaves, n + "/kernel", requires_grad) for n in fx.layer_names("Dense")]
    return W, leaves


def _ifm_forward(fx, W):
    import ifm_oracle as IO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    args = (fx.inputs(), columns(fx, "linear", FC), columns(fx, "dnn", FC), W)
    if fx.builder == "IFM":
        return IO.ifm(*args, task=fx.task)
    return IO.difm(*args, att_embedding_size=kw.get("att_embedding_size", 8), att_head_num=kw.get("att_head_num", 8),
                   att_res=kw.get("att_res", True), task=fx.task)


def _bst_weights(fx, requires_grad=False):
    """The dict tests/bst_oracle.py takes; every fixture weight is a leaf."""
    leaves = {k: torch.tensor(v, requires_grad=requires_grad) for k, v in fx.w.items()}
    tables = {k.split("/")[0][len("sparse_emb_"):]: v for k, v in leaves.items() if k.endswith("/embeddings")}
    trs = []
    for name in fx.layer_names("Transformer"):
        trs.append({k[len(name) + 1:]: v for k, v in leaves.items() if k.startswith(name + "/")})
    p = fx.layer_names("AttentionSequencePoolingLayer")[0] + "/local_att/"
    n = len([k for k in leaves if k.startswith(p + "dnn/kernel")])
    lau = {"dnn_kernels": [leaves["%sdnn/kernel%d" % (p, i)] for i in range(n)],
           "dnn_biases": [leaves["%sdnn/bias%d" % (p, i)] for i in range(n)],
           "kernel": leaves[p + "kernel"], "bias": leaves[p + "bias"]}
    dnn = fx.layer_names("DNN")[-1]
    m = len([k for k in leaves if k.startswith(dnn + "/kernel")])
    W = {"tables": tables, "transformers": trs, "lau": lau,
         "dnn_kernels": [leaves["%s/kernel%d" % (dnn, i)] for i in range(m)],
         "dnn_biases": [leaves["%s/bias%d" % (dnn, i)] for i in range(m)],
         "dense_kernel": leaves[fx.layer_names("Dense")[-1] + "/kernel"],
         "global_bias": leaves[fx.layer_names("PredictionLayer")[-1] + "/global_bias"]}
    return W, leaves


def _bst_forward(fx, W):
    import bst_oracle as BO
    from deepctr_b200 import feature_column as FC
    kw = fx.kwargs
    return BO.bst(fx.inputs(), columns(fx, "dnn", FC), ["item_id", "cate_id"], W,
                  transformer_num=kw.get("transformer_num", 1), att_head_num=kw.get("att_head_num", 8))


class Family(object):
    """One directory of model fixtures, the builders that made them and the oracle that restates them.

    ``n_cases``, ``builders`` and ``tasks`` are what the fixture set holds.  The flags keep what legitimately differs
    between families:

    * ``graph_weight_order``: fixtures whose model lists its weights in graph order, which differs from the reference's
      creation order (the graph order itself is pinned against the reference-built graph);
    * ``placed``: the builders write their products into the DNN input in place, so the GPU fixture tests run with and
      without that placement;
    * ``predict_atol``: the absolute tolerance of the GPU predictions, where the family has its own.
    """

    def __init__(self, subdir, builders_json, builders, oracle_weights, oracle_forward, n_cases, tasks,
                 graph_weight_order=(), placed=False, predict_atol=None):
        self.models_dir = os.path.join(GOLDEN, subdir)
        self.cases = _cases(self.models_dir)
        self.builders_json = os.path.join(GOLDEN, builders_json)
        self.builders = builders
        self.oracle_weights, self.oracle_forward = oracle_weights, oracle_forward
        self.n_cases, self.tasks = n_cases, tasks
        self.graph_weight_order, self.placed, self.predict_atol = graph_weight_order, placed, predict_atol

    def fixture(self, name):
        return Fixture(name, self.models_dir)

    def reference_builders(self):
        with open(self.builders_json) as f:
            return json.load(f)


FAMILIES = {
    "models": Family("models", "reference_builders.json", ("DeepFM", "xDeepFM", "DCN", "AutoInt", "DIN"),
                     oracle_weights, oracle_forward, 17, {"binary", "regression"},
                     graph_weight_order=("autoint_2x2_res", "autoint_attonly", "dcn_crossonly", "dcn_empty_linear",
                                         "dcn_matrix1", "dcn_vector2", "deepfm_groups_varlen")),
    "pairwise": Family("models_pairwise", "reference_builders_pairwise.json", ("NFM", "AFM"),
                       _pairwise_weights, _pairwise_forward, 4, {"binary"},
                       graph_weight_order=("afm_fm_only", "afm_two_groups")),     # AFM looks up embeddings first
    "fibinet": Family("models_fibinet", "reference_builders_fibinet.json", ("FiBiNET",),
                      _fibinet_weights, _fibinet_forward, 5, {"binary"}, placed=True),
    "fefm": Family("models_fefm", "reference_builders_fefm.json", ("FwFM", "DeepFEFM"),
                   _fefm_weights, _fefm_forward, 10, {"binary", "regression"}, placed=True,
                   # a group's FwFMLayer is built before the next group's embeddings
                   graph_weight_order=("fwfm_two_groups",)),
    "pnn": Family("models_pnn", "reference_builders_pnn.json", ("PNN",),
                  _pnn_weights, _pnn_forward, 9, {"binary", "regression"}, placed=True),
    "ifm": Family("models_ifm", "reference_builders_ifm.json", ("IFM", "DIFM"),
                  _ifm_weights, _ifm_forward, 6, {"binary", "regression"},
                  graph_weight_order=("difm_defaults", "difm_no_att_res", "difm_two_heads_varlen", "ifm_criteo",
                                      "ifm_regression", "ifm_varlen")),
    "bst": Family("models_bst", "reference_builders_bst.json", ("BST",),
                  _bst_weights, _bst_forward, 4, {"binary"}, predict_atol=1e-5),
}


# ---- layer fixtures (tests/golden/*.npz, tests/golden/<set>/*.npz) -------------------------------------
# Key convention: ``w_<weight>`` / ``g_<weight>`` (the weight's path inside the layer), the inputs ``x`` [B,F,E],
# ``x_<i>`` or ``in_<i>`` with their gradients ``gx`` / ``gx_<i>``, ``out`` and, where there are gradients, the
# ``dout`` they were taken for.
def allclose(rtol, atol):
    """elementwise: |got - want| <= atol + rtol |want|."""
    def check(got, want, what):
        np.testing.assert_allclose(got, want, rtol=rtol, atol=atol, err_msg=what)
    return check


def max_rel(tol):
    """normwise: max |got - want| < tol x max |want| (b2_helpers.close)."""
    def check(got, want, what):
        H.close(got, want, what, tol)
    return check


def _root_out(got, want, what):
    """1e-4 relative; under the split-bf16 GEMMs the atol is normwise, 1e-4 x max |want| (see test_layers_gpu)."""
    from deepctr_b200 import ops, _lib as L
    atol = 2e-6
    if ops.GEMM_PRECISION == L.GEMM_BF16X3 and want.size:
        atol = max(atol, 1e-4 * float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=atol, err_msg=what)


def numbered(d, prefix):
    """``prefix``0, ``prefix``1, ... as far as the fixture has them."""
    return ["%s%d" % (prefix, i) for i in range(len([k for k in d if k.startswith(prefix)]))]


def _one_or_list(vs):
    return vs[0] if len(vs) == 1 else vs


# layers called on a list of F [B,1,E] tensors; the others of the x-format sets take the [B,F,E] tensor
_LIST_LAYERS = ("AFMLayer", "SENETLayer", "BilinearInteraction", "InnerProductLayer", "OutterProductLayer")


def _x_args(meta, d, device):
    """``x`` [B,F,E] as a model hands it to the layer, a [B, F*E] buffer read in place: F [B,1,E] windows of it
    (which ops.concat joins back without a copy) or one [B,F,E] window.  The buffer collects ``gx``."""
    from deepctr_b200 import engine as E, ops
    b, f, e = d["x"].shape
    buf = E.Var(torch.tensor(d["x"].reshape(b, f * e), device=device), requires_grad=True)
    if meta["layer"] in _LIST_LAYERS:
        return [ops._window(buf, i * e, e, (b, 1, e)) for i in range(f)], {"x": buf}
    return ops._window(buf, 0, f * e, (b, f, e)), {"x": buf}


def _x_i_args(meta, d, device):
    """BST's ``x_<i>``; masked fixtures carry each input's mask as ``mask_<i>`` [B,T], a prefix of valid steps."""
    from deepctr_b200 import engine as E
    vs = []
    for i, k in enumerate(numbered(d, "x_")):
        a = d[k]
        v = E.Var(torch.tensor(a, device=device), requires_grad=a.dtype == np.float32)
        if meta["masked"]:
            lengths = d["mask_%d" % i].sum(1).astype(np.int32)
            v.mask = E.KMask(lengths=torch.tensor(lengths, device=device), maxlen=a.shape[1])
        vs.append(v)
    return _one_or_list(vs), dict(zip(numbered(d, "x_"), vs))


def _in_args(meta, d, device):
    """``in_<i>``; a Keras mask in meta['extra']['mask'] (one per input, or one for the first) becomes the
    ``id != 0`` mask of its input."""
    from deepctr_b200 import engine as E
    vs = [E.to_var(d[k]) for k in numbered(d, "in_")]
    mask = meta["extra"].get("mask")
    if mask is not None:
        ms = mask if (isinstance(mask, list) and (mask[0] is None or isinstance(mask[0][0], list))) else [mask]
        for v, m in zip(vs, ms):
            if m is not None:
                v.mask = E.KMask(ids=[torch.as_tensor(np.asarray(m, dtype=np.int32)).to(v.data.device)])
    return _one_or_list(vs), {}


def _pairwise_layer(meta, xs, W, d):
    import pairwise_oracle as PO
    if meta["layer"] == "AFMLayer":
        return PO.afm(xs[0], **W)
    return PO.bi_interaction(xs[0])


def _fibinet_layer(meta, xs, W, d):
    import fibinet_oracle as FO
    if meta["layer"] == "SENETLayer":
        return FO.senet(xs[0], *W.values())
    return FO.bilinear(xs[0], meta["kwargs"]["bilinear_type"], list(W.values()))


def _fefm_layer(meta, xs, W, d):
    import fefm_oracle as FO
    if meta["layer"] == "FwFMLayer":
        return FO.fwfm(xs[0], W["field_pair_strengths"])
    return FO.fefm(xs[0], list(W.values()))


def _pnn_layer(meta, xs, W, d):
    import pnn_oracle as PO
    kw = meta["kwargs"]
    if meta["layer"] == "InnerProductLayer":
        return PO.inner(xs[0], kw.get("reduce_sum", True))
    return PO.outer(xs[0], W["kernel"], kw["kernel_type"])


def _bst_layer(meta, xs, W, d):
    import bst_oracle as BO
    kw = meta["kwargs"]
    cls = meta["layer"]
    if cls == "LayerNormalization":
        return BO.layer_norm(xs[0], W["gamma"], W["beta"])
    if cls == "PositionEncoding":
        return BO.position_encoding(xs[0], W["lookup_table"], kw.get("scale", True))
    T = xs[0].shape[1]
    if meta["masked"]:
        qv, kv = torch.as_tensor(d["mask_0"]), torch.as_tensor(d["mask_1"])
    else:
        ar = torch.arange(T)[None, :]
        qv, kv = ar < torch.as_tensor(xs[2]).long(), ar < torch.as_tensor(xs[3]).long()
    return BO.transformer(xs[0], xs[1], qv, kv, W, **kw)


class LayerSet(object):
    """One directory of layer fixtures: the reference's layer, built from meta's ``layer`` and ``kwargs``, run on the
    fixture's inputs and weights.

    * ``n_cases`` and ``layers`` are what the set holds;
    * ``args(meta, d, device)``: the layer's call argument and {input key: the Var its gradient lands in};
    * ``oracle(meta, xs, W, d)``: the CPU restatement (``xs`` the inputs ``x`` or ``x_<i>``, ``W`` {weight: tensor});
      the root set has none, test_oracle_pinning.py pins it layer by layer;
    * ``cpu`` / ``gpu``: (output check, gradient check), each ``check(got, want, what)``;
    * ``renames``: reference weight path -> path inside this package's layer.
    """

    def __init__(self, subdir, n_cases, layers, args, gpu, oracle=None, cpu=None, renames=(), skip=()):
        self.dir = os.path.join(GOLDEN, subdir)
        self.cases = [n for n in _cases(self.dir) if n not in skip]
        self.n_cases, self.layers, self.args = n_cases, layers, args
        self.oracle, self.cpu, self.gpu, self.renames = oracle, cpu, gpu, renames

    def load(self, name):
        """(meta, {key: array}); the keys keep the npz's order, the weights the layer's."""
        d = np.load(os.path.join(self.dir, name + ".npz"))
        return json.loads(str(d["meta"])), {k: d[k] for k in d.files if k != "meta"}

    def weight_name(self, key):
        for a, b in self.renames:
            key = key.replace(a, b)
        return key


_FAMILY_CPU = (allclose(1e-5, 1e-6), allclose(1e-4, 1e-6))
_FAMILY_GPU = allclose(1e-4, 1e-5)

LAYER_SETS = {
    "root": LayerSet("", 35, ("AttentionSequencePoolingLayer", "CIN", "CrossNet", "DNN", "Dice", "FM",
                              "InteractingLayer", "Linear", "LocalActivationUnit", "PredictionLayer",
                              "SequencePoolingLayer", "WeightedSequenceLayer"),
                     _in_args, gpu=(_root_out, None), skip=("hash_vocab_kat",),
                     renames=(("local_att/", "local_activation_unit/"), ("activation_layers", "act"))),
    "pairwise": LayerSet("pairwise", 6, ("AFMLayer", "BiInteractionPooling"), _x_args, oracle=_pairwise_layer,
                         cpu=_FAMILY_CPU, gpu=(allclose(1e-5, 1e-5), _FAMILY_GPU)),
    "fibinet": LayerSet("fibinet", 12, ("SENETLayer", "BilinearInteraction"), _x_args, oracle=_fibinet_layer,
                        cpu=_FAMILY_CPU, gpu=(_FAMILY_GPU, _FAMILY_GPU)),
    "fefm": LayerSet("fefm", 6, ("FwFMLayer", "FEFMLayer"), _x_args, oracle=_fefm_layer,
                     cpu=_FAMILY_CPU, gpu=(_FAMILY_GPU, _FAMILY_GPU)),
    "pnn": LayerSet("pnn", 15, ("InnerProductLayer", "OutterProductLayer"), _x_args, oracle=_pnn_layer,
                    cpu=_FAMILY_CPU, gpu=(_FAMILY_GPU, _FAMILY_GPU)),
    "bst": LayerSet("bst", 7, ("Transformer", "PositionEncoding", "LayerNormalization"), _x_i_args,
                    oracle=_bst_layer, cpu=(max_rel(1e-5), max_rel(1e-4)), gpu=(max_rel(2e-4), max_rel(2e-4))),
}
