"""Scaffolding shared by the tabular builders (DeepFM / xDeepFM / DCN / AutoInt): symbolic inputs, the
first-order (linear) logit, the embedding windows and the usual tower pieces.  Construction order is part of
the contract - layer and weight names are derived from it - so every accessor builds its sub-graph exactly
once, the first time it is asked for."""
from ..engine import Dense, Model
from ..feature_column import build_input_features, get_linear_logit, input_from_feature_columns
from ..layers.core import DNN, PredictionLayer
from ..layers.utils import add_func, combined_dnn_input, concat_func


class Tower(object):
    def __init__(self, input_columns, linear_columns, dnn_columns, seed, l2_linear, l2_embedding, grouped=False,
                 defer_linear=False):
        """``defer_linear``: the linear logit is not built here but by ``linear()``, after the embeddings (IFM / DIFM
        reweight it with field weights computed from them)."""
        self.seed = seed
        self.features = build_input_features(input_columns)
        self.inputs = list(self.features.values())
        self._linear = (linear_columns, l2_linear)
        self.linear_logit = None if defer_linear else self.linear()
        looked_up, self.dense_values = input_from_feature_columns(self.features, dnn_columns, l2_embedding, seed,
                                                                  support_group=grouped)
        self.groups = looked_up if grouped else None          # group name -> [B,1,E] tensors
        self.embeddings = [t for g in looked_up.values() for t in g] if grouped else looked_up
        self._flat = None

    def linear(self, refine_weight=None):
        """The first-order logit; ``refine_weight`` [B, F] scales the sparse lookups (sparse_feat_refine_weight)."""
        columns, l2_reg = self._linear
        return get_linear_logit(self.features, columns, seed=self.seed, prefix='linear', l2_reg=l2_reg,
                                sparse_feat_refine_weight=refine_weight)

    def field_matrix(self, embeddings=None):
        """[B, F, E] stack of per-field embeddings (a zero-copy window of the fused gather's buffer)."""
        return concat_func(self.embeddings if embeddings is None else embeddings, axis=1)

    def flat_input(self):
        """[B, F*E + n_dense]: the DNN / CrossNet operand."""
        if self._flat is None:
            self._flat = combined_dnn_input(self.embeddings, self.dense_values)
        return self._flat

    def mlp(self, hidden_units, activation, l2_reg, dropout, use_bn, inputs=None):
        layer = DNN(hidden_units, activation, l2_reg, dropout, use_bn, seed=self.seed)
        return layer(self.flat_input() if inputs is None else inputs)

    @staticmethod
    def project(x):
        """[B, d] -> [B, 1] without bias (the `Dense(1, use_bias=False)` every builder ends its branches with)."""
        return Dense(1, use_bias=False)(x)

    def finish(self, logit, task):
        return Model(inputs=self.inputs, outputs=PredictionLayer(task)(logit))


def total(logits):
    return add_func(list(logits))
