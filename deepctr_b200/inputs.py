"""Host mirror of deepctr/inputs.py plus the machinery that turns its per-feature ``Embedding``
calls into ONE fused launch per step.

Reference functions mirrored (same names / arguments / return structure):
``create_embedding_dict`` (inputs.py:44-71), ``create_embedding_matrix`` (:89-98),
``embedding_lookup`` (:101-117), ``varlen_embedding_lookup`` (:120-130),
``get_varlen_pooling_list`` (:133-158), ``get_dense_input`` (:161-172), ``mergeDict`` (:175-181),
``get_embedding_vec_list`` (:74-86), ``get_inputs_list`` (:40-41).

H100 design (DESIGN.md section 3): the builders still call ``Embedding`` once per feature, but the
``EmbeddingPlanner`` owned by the Model recognises, once per graph, every lookup whose ids are a
model input (optionally through ``Hash``) and every ``SequencePoolingLayer`` /
``WeightedSequenceLayer`` chain hanging off such a lookup, lays all their outputs out as adjacent
column windows of one [B, ld] buffer, and serves them from a single kernel launch
(``b2ctr_embed_gather_uniform_fwd`` for the Criteo shape, ``b2ctr_embed_gather_fwd`` otherwise).
Concatenations of those windows are then zero-copy views, and the backward pass is a single fused
scatter (+ SGD update) launch.
"""
from collections import defaultdict, OrderedDict
import itertools
from itertools import chain

import ctypes as C

import numpy as np
import torch

from . import _lib as L
from . import kernels as K
from . import engine as E
from .engine import Layer, l2


# ================================================================================================
# Embedding layer (tf.keras.layers.Embedding surface used by deepctr/inputs.py:19-26)
# ================================================================================================
class Embedding(Layer):
    def __init__(self, input_dim, output_dim, embeddings_initializer=None, embeddings_regularizer=None,
                 mask_zero=False, name=None, **kwargs):
        Layer.__init__(self, name=name, **kwargs)
        self.input_dim, self.output_dim = int(input_dim), int(output_dim)
        self.embeddings_initializer = embeddings_initializer or E.RandomNormal(0.0, 0.05)
        self.embeddings_regularizer = embeddings_regularizer
        self.mask_zero = mask_zero
        self.supports_masking = mask_zero
        # tables are created eagerly so that they exist (and can be set) before any call
        self.embeddings = self.add_weight("embeddings", (self.input_dim, self.output_dim),
                                          self.embeddings_initializer, self.embeddings_regularizer,
                                          trainable=self.trainable)
        self.built = True

    def _output_dtype(self, inputs):
        return "float32"

    def compute_output_shape(self, input_shape):
        return tuple(input_shape) + (self.output_dim,)

    def compute_mask(self, inputs, mask=None):
        if not self.mask_zero:
            return None
        return E.KMask(ids=[inputs.data])

    def call(self, inputs, **kwargs):
        """Unplanned (eager / computed ids) lookup: one generic-kernel launch for this table."""
        ids = inputs.data
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.to(torch.int64)
        ids2 = ids.reshape(ids.shape[0], -1).contiguous()
        b, t = ids2.shape
        table = self.embeddings.materialize()
        out = torch.empty((b, t * self.output_dim), dtype=torch.float32, device=ids.device)
        feat = K.make_feature(table, ids2, out, maxlen=t)
        K.embed_gather_fwd([feat], b)
        res = E.Var(out.reshape(tuple(ids.shape) + (self.output_dim,)))
        w = self.embeddings

        def bwd(grads):
            g = grads[0].reshape(b, t * self.output_dim).contiguous()
            tgt, scale = _grad_target(w, E.current_opt())
            fb = K.make_feature(tgt, ids2, g, maxlen=t)
            K.embed_scatter_add([fb], b, scale)

        E.record([res], [w], bwd)
        return res

    def get_config(self):
        c = Layer.get_config(self)
        c.update(input_dim=self.input_dim, output_dim=self.output_dim, mask_zero=self.mask_zero)
        return c


def _grad_target(w, opt_ctx):
    """Where a table gradient goes: the table itself (fused SGD, scale=-lr) or a dense .grad buffer."""
    if w.sparse_grad:
        lr = opt_ctx["optimizer"].lr if opt_ctx and opt_ctx.get("optimizer") else 0.0
        return w.data, -lr
    if w.grad is None:
        w.grad = torch.empty_like(w.data)
        K.fill(w.grad, 0.0)
    return w.grad, 1.0


# ================================================================================================
# the deepctr/inputs.py function surface (same names, arguments and return structures; bodies are
# this package's own: one table registry + one id resolver shared by every lookup flavour)
# ================================================================================================
_SHARED_ATTRS = ('vocabulary_size', 'embedding_dim', 'trainable')


def _check_embedding_compatible(embedding_name, existing_feat, feat):
    """Columns sharing an ``embedding_name`` share ONE table, so they must agree on its geometry
    (deepctr/inputs.py:29-37; the message is part of the interface, tests/feature_test.py:53-60)."""
    clash = [a for a in _SHARED_ATTRS if getattr(existing_feat, a) != getattr(feat, a)]
    if clash:
        a = clash[0]
        raise ValueError("Feature columns with the same embedding_name must share the same "
                         "{}. embedding_name='{}' has {} and {}.".format(
                             a, embedding_name, getattr(existing_feat, a), getattr(feat, a)))


class _TableRegistry(object):
    """embedding_name -> Embedding layer, first declaration wins (deepctr/inputs.py:44-71)."""

    def __init__(self, l2_reg, prefix):
        self.l2_reg, self.prefix = l2_reg, prefix
        self.tables, self.owner = {}, {}

    def declare(self, feat, kind, mask_zero):
        key = feat.embedding_name
        if key in self.tables:
            _check_embedding_compatible(key, self.owner[key], feat)
            return
        self.owner[key] = feat
        self.tables[key] = Embedding(feat.vocabulary_size, feat.embedding_dim,
                                     embeddings_initializer=feat.embeddings_initializer,
                                     embeddings_regularizer=l2(self.l2_reg),
                                     name="%s_%s_%s" % (self.prefix, kind, key),      # inputs.py:23
                                     mask_zero=mask_zero, trainable=feat.trainable)


def create_embedding_dict(sparse_feature_columns, varlen_sparse_feature_columns, seed, l2_reg,
                          prefix='sparse_', seq_mask_zero=True):
    """One table per distinct embedding_name.  A table is ``mask_zero`` when a VarLen column reads it
    (its own ``seq_emb`` table, or a SparseFeat table it shares: DIN's item_id / hist_item_id)."""
    varlen = list(varlen_sparse_feature_columns or ())
    read_by_sequences = set(f.embedding_name for f in varlen)
    reg = _TableRegistry(l2_reg, prefix)
    for feat in sparse_feature_columns:
        reg.declare(feat, 'emb', bool(seq_mask_zero and feat.embedding_name in read_by_sequences))
    for feat in varlen:
        reg.declare(feat, 'seq_emb', seq_mask_zero)
    return reg.tables


def create_embedding_matrix(feature_columns, l2_reg, seed, prefix="", seq_mask_zero=True):
    from . import feature_column as fc_lib
    cols = list(feature_columns or ())
    return create_embedding_dict([c for c in cols if isinstance(c, fc_lib.SparseFeat)],
                                 [c for c in cols if isinstance(c, fc_lib.VarLenSparseFeat)],
                                 seed, l2_reg, prefix=prefix + 'sparse', seq_mask_zero=seq_mask_zero)


def _ids_of(fc, tensor, mask_zero):
    """The id tensor a column looks up: the input itself, or Hash(...)(input) for ``use_hash`` columns
    (folded into the gather kernel / the Feeder by the planner whenever the input is a model input)."""
    if not fc.use_hash:
        return tensor
    from .layers.utils import Hash
    return Hash(fc.vocabulary_size, mask_zero=mask_zero, vocabulary_path=fc.vocabulary_path)(tensor)


def _selected(columns, return_feat_list):
    keep = set(return_feat_list)
    return [fc for fc in columns if not keep or fc.name in keep]


def get_inputs_list(inputs):
    return [t for d in inputs if d is not None for t in d.values()]


def get_embedding_vec_list(embedding_dict, input_dict, sparse_feature_columns, return_feat_list=(),
                           mask_feat_list=()):
    """Legacy flavour (inputs.py:74-86): tables keyed by FEATURE name, flat list out."""
    return [embedding_dict[fc.name](_ids_of(fc, input_dict[fc.name], fc.name in mask_feat_list))
            for fc in _selected(sparse_feature_columns, return_feat_list)]


def embedding_lookup(sparse_embedding_dict, sparse_input_dict, sparse_feature_columns, return_feat_list=(),
                     mask_feat_list=(), to_list=False):
    """[B,1,E] (or [B,T,E]) per selected column, grouped by ``group_name`` (inputs.py:101-117)."""
    groups = defaultdict(list)
    for fc in _selected(sparse_feature_columns, return_feat_list):
        ids = _ids_of(fc, sparse_input_dict[fc.name], fc.name in mask_feat_list)
        groups[fc.group_name].append(sparse_embedding_dict[fc.embedding_name](ids))
    return [t for g in groups.values() for t in g] if to_list else groups


def varlen_embedding_lookup(embedding_dict, sequence_input_dict, varlen_sparse_feature_columns):
    """feature name -> [B,T,E] (hashing always keeps 0 as the padding id; inputs.py:120-130)."""
    return {fc.name: embedding_dict[fc.embedding_name](_ids_of(fc, sequence_input_dict[fc.name], True))
            for fc in varlen_sparse_feature_columns}


def get_varlen_pooling_list(embedding_dict, features, varlen_sparse_feature_columns, to_list=False):
    """Pool every sequence to [B,1,E]: validity comes from ``length_name`` when the column has one,
    else from the Keras mask of its mask_zero table; an optional per-position weight is applied first
    (inputs.py:133-158).  The planner folds these chains into the fused gather."""
    from .layers.sequence import SequencePoolingLayer, WeightedSequenceLayer
    groups = defaultdict(list)
    for fc in varlen_sparse_feature_columns:
        by_length = fc.length_name is not None
        extent = [features[fc.length_name]] if by_length else []
        seq = embedding_dict[fc.name]
        if fc.weight_name is not None:
            seq = WeightedSequenceLayer(weight_normalization=fc.weight_norm, supports_masking=not by_length)(
                [seq] + extent + [features[fc.weight_name]])
        pool = SequencePoolingLayer(fc.combiner, supports_masking=not by_length)
        groups[fc.group_name].append(pool([seq] + extent if by_length else seq))
    return chain.from_iterable(groups.values()) if to_list else groups


def get_dense_input(features, feature_columns):
    from . import feature_column as fc_lib
    out = []
    for fc in (c for c in (feature_columns or ()) if isinstance(c, fc_lib.DenseFeat)):
        t = features[fc.name]
        out.append(t if fc.transform_fn is None else E.Lambda(fc.transform_fn)(t))
    return out


def mergeDict(a, b):
    merged = defaultdict(list)
    for d in (a, b):
        for k, v in d.items():
            merged[k].extend(v)
    return merged


# ================================================================================================
# EmbeddingPlanner: graph pattern -> one fused launch
# ================================================================================================
VIRTUAL = object()   # result of a node folded into a fused descriptor (never consumed)


class _Slot(object):
    """One planned output: a lookup (single / sequence) or a pooled bag."""
    __slots__ = ("node", "emb", "input_name", "hash", "maxlen", "pool", "mask_mode", "len_name",
                 "weight_name", "weight_mode", "dim", "col", "buf", "out_shape", "virtual_nodes",
                 "mask_zero")


class EmbeddingPlanner(object):
    def __init__(self, model):
        from .layers.utils import Hash
        from .layers.sequence import SequencePoolingLayer, WeightedSequenceLayer
        self.model = model
        self.slots = []
        self.results = {}
        self.optimizer = None
        self.mode = "auto"
        self.fm_hint = None        # (col0, ncols) of the main buffer an FM layer consumed
        self.lin_hint = False      # the linear buffer is only ever row-summed
        self.tail_hint = None      # (dense col0, ncols) appended behind the main buffer
        self.planes_hint = None    # ncols of the leading main-buffer window ops.dense split into bf16 planes
        self.fm_result = None
        self.lin_result = None
        self._plans = {}
        consumers = defaultdict(list)
        for node in model._order:
            for t in E._flatten(node.inputs):
                consumers[id(t)].append(node)
        out_ids = set(id(t) for t in E._flatten(model.outputs))
        input_names = set(t.name for t in model.inputs)

        def as_input(t):
            return t.name if (isinstance(t.node.layer, E.InputLayer) and t.name in input_names) else None

        # ONN's field-aware lookups and their products: one kernel pair of their own, never slots of the gather
        self.ffm = _plan_field_aware(model, consumers, out_ids, as_input)
        claimed = self.ffm.claimed if self.ffm is not None else ()
        for node in model._order:
            if not isinstance(node.layer, Embedding) or not isinstance(node.inputs, E.KTensor):
                continue
            if id(node) in claimed:
                continue
            src, hcfg, virt = node.inputs, None, []
            if isinstance(src.node.layer, Hash) and isinstance(src.node.inputs, E.KTensor):
                h = src.node.layer
                if len(consumers[id(src)]) == 1 and id(src) not in out_ids:
                    hcfg, virt, src = h, [src.node], src.node.inputs
            name = as_input(src)
            if name is None:
                continue
            if hcfg is not None and (hcfg.vocabulary_path or src.dtype in ("string", str)):
                hash_mode, prehashed = L.HASH_NONE, hcfg      # resolved on the host by the Feeder
            elif hcfg is not None:
                hash_mode, prehashed = (L.HASH_FARM_MASK_ZERO if hcfg.mask_zero else L.HASH_FARM), None
            else:
                hash_mode, prehashed = L.HASH_NONE, None
            s = _Slot()
            s.emb, s.input_name, s.hash = node.layer, name, (hash_mode, prehashed)
            s.maxlen = int(np.prod(src.shape[1:])) if len(src.shape) > 1 else 1
            s.dim, s.mask_zero = node.layer.output_dim, node.layer.mask_zero
            s.pool, s.mask_mode, s.len_name, s.weight_name, s.weight_mode = L.POOL_NONE, L.MASK_NONE, None, None, L.WEIGHT_NONE
            s.node, s.virtual_nodes = node, list(virt)
            out_t = node.outputs[0]
            cons = consumers[id(out_t)]
            # --- pooled-bag patterns of get_varlen_pooling_list (inputs.py:133-158) ----------------
            if len(cons) == 1 and id(out_t) not in out_ids:
                c = cons[0]
                wnode = None
                if isinstance(c.layer, WeightedSequenceLayer) and E._flatten(c.inputs)[0] is out_t:
                    wins = E._flatten(c.inputs)
                    wt = c.outputs[0]
                    wc = consumers[id(wt)]
                    if (len(wc) == 1 and id(wt) not in out_ids and isinstance(wc[0].layer, SequencePoolingLayer)
                            and all(as_input(t) for t in wins[1:])):
                        wnode, c = c, wc[0]
                if isinstance(c.layer, SequencePoolingLayer):
                    pins = E._flatten(c.inputs)
                    first = wnode.outputs[0] if wnode is not None else out_t
                    ok = pins[0] is first and all(as_input(t) for t in pins[1:])
                    pl = c.layer
                    if ok and pl.supports_masking and not s.mask_zero:
                        ok = False   # reference raises at run time: input must carry a mask
                    if ok and wnode is not None and wnode.layer.supports_masking != pl.supports_masking:
                        ok = False
                    if ok:
                        s.pool = L.POOL_BY_NAME[pl.mode]
                        if pl.supports_masking:
                            s.mask_mode = L.MASK_ZERO_ID
                        else:
                            s.mask_mode, s.len_name = L.MASK_LENGTH, pins[1].name
                        if wnode is not None:
                            wins = E._flatten(wnode.inputs)
                            s.weight_name = wins[-1].name
                            s.weight_mode = L.WEIGHT_SOFTMAX if wnode.layer.weight_normalization else L.WEIGHT_RAW
                            s.virtual_nodes.append(wnode)
                        s.virtual_nodes.append(node)
                        s.node = c
            self.slots.append(s)
        # ---- column layout: dim-1 lookups (linear terms) | everything else | sequences ------------
        self.main = [s for s in self.slots if not (s.pool == L.POOL_NONE and s.maxlen > 1) and s.dim > 1]
        self.lin = [s for s in self.slots if not (s.pool == L.POOL_NONE and s.maxlen > 1) and s.dim == 1]
        self.seq = [s for s in self.slots if s.pool == L.POOL_NONE and s.maxlen > 1]
        for group, tag in ((self.main, "main"), (self.lin, "lin")):
            col = 0
            for s in group:
                s.buf, s.col = tag, col
                col += s.dim
        self.main_width = sum(s.dim for s in self.main)
        self.lin_width = sum(s.dim for s in self.lin)
        for s in self.seq:
            s.buf, s.col = "seq", 0
        self.tail_reserve = 0
        for t in model.inputs:
            if t.dtype in ("float32", "float64", "float16") and len(t.shape) == 2:
                self.tail_reserve += int(t.shape[1])
        # DeepFEFM's FEFM scores go behind the dense columns (fefm_place): P more columns in the row pitch
        self.fefm_places = _plan_fefm_input(model, consumers, out_ids)
        # PNN's inner / outer products go between the embeddings and the dense columns (pnn_place): P per product
        # more columns in the row pitch
        self.pnn_places, self.pnn_cols = _plan_pnn_input(model, consumers, out_ids)
        self.main_ld = (self.main_width + self.tail_reserve + sum(self.fefm_places.values()) + self.pnn_cols
                        + 3) // 4 * 4
        self.lin_ld = max(1, (self.lin_width + 3) // 4 * 4)
        self.fast = self._fast_eligible()
        self.dnn_places = _plan_dnn_input(model, consumers, out_ids)
        # EDCN's RegulationModule pairs and the bridges in front of them: one b2ctr_regulate launch each
        self.regulate_plan = _plan_regulate(model, consumers, out_ids)
        # CCPM's Lambda(expand_dims) -> [Conv2D -> KMaxPooling(axis=1)] x l -> Flatten: one b2ctr_conv_stack launch
        self.conv_plan = _plan_conv_stack(model, consumers, out_ids)
        # FLEN's FieldWiseBiInteraction on concatenations of gather-buffer windows: one launch reading them in place
        self.field_wise_plan = _plan_field_wise(model, consumers, out_ids, self.main)
        # IFM / DIFM scale the linear lookups by per-sample field weights before Linear sums them: their rows are
        # needed, so they are never fused into the gather's row-sum (lin_hint)
        from .layers.utils import RefineWeight
        self.lin_refined = any(isinstance(node.layer, RefineWeight) for node in model._order)

    # ---- configuration ---------------------------------------------------------------------------
    def tables(self):
        seen, out = set(), []
        for s in self.slots:
            if id(s.emb.embeddings) not in seen:
                seen.add(id(s.emb.embeddings))
                out.append(s.emb.embeddings)
        return out

    def configure(self, optimizer, mode):
        self.optimizer, self.mode = optimizer, mode
        total = sum(w.numel() for w in self.tables()) + (self.ffm.numel() if self.ffm is not None else 0)
        sparse = mode in ("sparse", "sparse_deterministic") or (mode == "auto" and total > (1 << 22))
        # 'sparse_deterministic': sort + ordered segmented reduce instead of fp32 atomics (bit-identical from run
        # to run); it is also the path of row-state optimizers, i.e. Keras' lazy sparse Adagrad.  Keras' Adam
        # decays m and v of EVERY row each step (SURVEY.md App. C): it has no faithful row-wise form.
        self.sorted_update = bool(sparse and (mode == "sparse_deterministic" or optimizer.name == "adagrad"))
        if self.sorted_update and self.ffm is not None:
            raise ValueError("the deterministic / Adagrad row-wise update does not cover ONN's field-aware tables "
                             "(%s ..., %d tables): use embedding_update='dense', or 'sparse' with the 'sgd' optimizer"
                             % (self.ffm.tables[0][1].name, self.ffm.n_tables()))
        if sparse and optimizer.name not in ("sgd", "adagrad"):
            raise ValueError("row-wise (sparse) embedding updates support 'sgd' and 'adagrad'; %r keeps dense state "
                             "for every row of every table - use embedding_update='dense' (O(vocabulary) per step)"
                             % optimizer.name)
        if self.sorted_update and not (self.fast and self._all_fast_single()):
            if mode == "sparse_deterministic" or optimizer.name == "adagrad":
                raise ValueError("the deterministic / Adagrad row-wise update covers models whose sparse features are "
                                 "single-valued columns of one embedding_dim (the Criteo shape)")
        if self.sorted_update and self.lin and self.lin_refined:
            raise ValueError("the deterministic / Adagrad row-wise update sums the linear lookups inside the gather, "
                             "but this model scales them by field weights first (sparse_feat_refine_weight): use "
                             "embedding_update='dense', or 'sparse' with the 'sgd' optimizer")
        if self.sorted_update and self.lin:
            self.lin_hint = True        # the linear tables are updated by the same sorted pass from the first step on
        tabs = list(self.tables())
        for l in self.model.layers:          # unplanned Embedding layers follow the same policy
            if isinstance(l, Embedding) and all(l.embeddings is not w for w in tabs):
                tabs.append(l.embeddings)
        if sparse:
            # the fused row-wise update touches only the rows of the batch: a whole-table L2 penalty (the
            # builders' default l2_reg_embedding / l2_reg_linear = 1e-5, Keras semantics: SURVEY.md App. C)
            # cannot be part of it.  Never drop it silently.
            reg = sorted(w.name for w in tabs if w.trainable and w.l2 > 0)
            if reg and mode == "sparse":
                raise ValueError("embedding_update='sparse' applies row-wise updates and cannot apply the L2 "
                                 "regulariser of %s ... (%d tables): build the model with l2_reg_embedding=0 and "
                                 "l2_reg_linear=0, or use embedding_update='dense'" % (reg[0], len(reg)))
            if reg:
                import warnings
                warnings.warn("tables of %d elements take the row-wise (sparse) update path, which does NOT apply "
                              "the L2 regulariser of %s ... (%d tables); pass l2_reg_embedding=0 / l2_reg_linear=0 "
                              "to silence this, or embedding_update='dense' for Keras' O(vocabulary) semantics"
                              % (total, reg[0], len(reg)))
        for w in tabs:
            w.sparse_grad = bool(sparse and w.trainable)

    def set_dist(self, ctx):
        """Row-shard the fast-path tables (and their dim-1 linear twins) over the process group:
        row r -> rank r % world, local row r // world.  Everything else stays replicated."""
        from . import parallel
        self.dist = ctx
        self.exchange = parallel.ShardedExchange(ctx, K)
        self.sharded = False
        if ctx.world == 1:
            return
        lin_ok = self.fast and self._lin_matches_fast() and not self.lin_refined
        shardable = self.fast and (lin_ok or not self.lin)
        will_shard = set()
        if shardable:
            for s_ in list(self.main[:self.fast_n]) + (list(self.lin) if lin_ok else []):
                will_shard.add(id(s_.emb.embeddings))
        # Every table that stays REPLICATED must take the dense path: its gradient is then part of the bucket
        # all-reduced over the ranks.  A row-wise local update from this rank's mini-batch alone would let the
        # replicas drift apart.
        for l in self.model.layers:
            if isinstance(l, Embedding) and id(l.embeddings) not in will_shard:
                l.embeddings.sparse_grad = False
        if not shardable:
            return        # unusual graph: every table replicated, gradients all-reduced like the dense weights
        if self.optimizer is None or self.optimizer.name != "sgd":
            raise ValueError("row-sharded embeddings need the 'sgd' optimizer (fused row-wise update)")
        seen = set()
        for s_ in list(self.main[:self.fast_n]) + (list(self.lin) if lin_ok else []):
            w = s_.emb.embeddings
            if id(w) in seen:
                continue
            seen.add(id(w))
            full_v = w.shape_[0]
            if w.data is not None or w.host_value is not None:
                full = w.value()
                w.data = None
                w.host_value = np.ascontiguousarray(parallel.shard_rows(full, ctx.rank, ctx.world))
            w.shape_ = (parallel.shard_size(full_v, ctx.rank, ctx.world),) + tuple(w.shape_[1:])
            w.opt_state["shard"] = (ctx.rank, ctx.world, full_v)
            w.sparse_grad = bool(w.trainable)
        self.sharded = True
        if lin_ok:
            self.lin_hint = True     # the linear rows never leave their owner: only the per-sample sum exists
        import os
        mode = os.environ.get("B2CTR_SHARD_MODE", "auto")
        if mode == "auto":
            shard_bytes = sum(int(np.prod(w_.shape_)) * 4 for w_ in
                              {id(s_.emb.embeddings): s_.emb.embeddings
                               for s_ in list(self.main[:self.fast_n]) + (list(self.lin) if lin_ok else [])}.values())
            mode = parallel.choose_transport(shard_bytes, ctx.world)
        pow2 = ctx.world & (ctx.world - 1) == 0
        self.peer_mode = mode == "peer" and pow2 and ctx.backend == "nccl"
        self.peers = None            # built lazily (tables must be materialised on the device first)

    def _peer_tables(self, fast_slots, lin_fused):
        """(PeerTables of the embedding shards, PeerTables of the linear shards | None), built once."""
        if self.peers is None:
            from . import parallel
            tabs = [s.emb.embeddings.materialize() for s in fast_slots]
            emb = parallel.PeerTables(self.dist, tabs, L)
            lin = None
            if lin_fused:
                lin = parallel.PeerTables(self.dist, [s.emb.embeddings.materialize().reshape(-1) for s in self.lin], L)
            token = torch.zeros((1,), dtype=torch.float32, device=tabs[0].device)
            self.peers = (emb, lin, token)
        return self.peers

    def _fast_eligible(self):
        m = self.main
        if not m or len(m) > 64:
            return False
        d = m[0].dim
        if d not in (4, 8, 16, 32, 64, 128):
            return False
        # the leading run of plain single-valued features (rest of `main` goes through the generic kernel)
        n = 0
        for s in m:
            if s.dim == d and s.maxlen == 1 and s.pool == L.POOL_NONE and s.hash[0] == L.HASH_NONE:
                n += 1
            else:
                break
        self.fast_n = n
        return n >= 1

    def _all_fast_single(self):
        return len(self.main) == self.fast_n and not self.seq and (not self.lin or self._lin_matches_fast())

    def _lin_matches_fast(self):
        """linear (dim-1) lookups mirror the fast features one-to-one -> summed inside the kernel."""
        if not self.lin or len(self.lin) != self.fast_n or len(self.main) != self.fast_n:
            return False
        for a, b in zip(self.lin, self.main):
            if (a.input_name != b.input_name or a.maxlen != 1 or a.pool != L.POOL_NONE
                    or a.hash[0] != L.HASH_NONE):
                return False
        return True

    # ---- per-step execution ------------------------------------------------------------------------
    def begin_step(self, feed, training):
        self.results = {}
        self.fm_result = self.lin_result = None
        self.tail_done = None
        self.planes_result = None
        if self.ffm is not None:
            self.ffm.forward(feed, self.results, training and E.current_tape() is not None)
        if not self.slots:
            return
        some = feed[self.slots[0].input_name].data
        batch, dev = some.shape[0], some.device
        grad = training and E.current_tape() is not None
        bufs = {}
        if self.main:
            bufs["main"] = E.Var(torch.empty((batch, self.main_ld), dtype=torch.float32, device=dev),
                                 ncols=self.main_width, owner=self)
        lin_fused = self.fast and self.lin_hint and self._lin_matches_fast()
        if self.lin and not lin_fused:
            bufs["lin"] = E.Var(torch.empty((batch, self.lin_ld), dtype=torch.float32, device=dev),
                                ncols=self.lin_width, owner=self)
        generic = []
        for s in self.slots:
            if s.buf == "seq":
                bufs[id(s)] = E.Var(torch.empty((batch, s.maxlen * s.dim), dtype=torch.float32, device=dev),
                                    owner=self)
        fast_slots = self.main[:self.fast_n] if self.fast else []
        for s in self.slots:
            if s in fast_slots or (lin_fused and s.buf == "lin"):
                continue
            generic.append(s)
        tables_used = []
        # ---- fast path launch -----------------------------------------------------------------------
        plan = None
        if fast_slots:
            x = bufs["main"].data
            self.route = None
            peer = None
            if getattr(self, "sharded", False) and getattr(self, "peer_mode", False):
                # row-sharded tables addressed in place over NVLink peer mappings: same launch as one GPU
                peer = self._peer_tables(fast_slots, self.fast and self.lin_hint and self._lin_matches_fast())
                feats = [self._feature(s, feed, x, self.main_ld) for s in fast_slots]
                lin_tabs = None
            elif getattr(self, "sharded", False):
                # ids -> owners (all-to-all), rows -> back (all-to-all); the returned row buffer then plays
                # the role of the table and `pos` the role of the ids for the ordinary fused gather
                id_feats = [self._feature(s, feed, x, self.main_ld) for s in fast_slots]
                st = self.exchange.route(id_feats, batch)
                dimf = fast_slots[0].dim
                tabs = [s.emb.embeddings.materialize() for s in fast_slots]
                ltabs = [s.emb.embeddings.materialize().reshape(-1) for s in self.lin] if lin_fused else None
                rows, rlin = self.exchange.fetch(st, tabs, ltabs, dimf)
                self.route = (st, tabs, ltabs, dimf)
                pos = st["pos"]
                feats = [K.make_feature(rows, pos[:, f], x, out_col=s.col, out_ld=self.main_ld)
                         for f, s in enumerate(fast_slots)]
                lin_tabs = [rlin] * len(fast_slots) if lin_fused else None
            else:
                feats = [self._feature(s, feed, x, self.main_ld) for s in fast_slots]
                lin_tabs = [s.emb.embeddings.materialize().reshape(-1) for s in self.lin] if lin_fused else None
            only_fast = len(self.main) == self.fast_n
            dense = None
            if only_fast and self.tail_hint is not None and "__dense_pack__" in feed and not self.pnn_cols:
                c0, nd = self.tail_hint
                dp = feed["__dense_pack__"].data
                if c0 + nd <= dp.shape[1] and self.main_width + nd <= self.main_ld:
                    dense = dp[:, c0:c0 + nd]
                    self.tail_done = (c0, nd)
            linear = torch.empty((batch,), dtype=torch.float32, device=dev) if lin_fused else None
            fm, fm_mask = None, 0
            if self.fm_hint is not None:
                c0, nc = self.fm_hint
                d = fast_slots[0].dim
                if c0 % d == 0 and nc % d == 0 and c0 + nc <= self.fast_n * d:
                    fm = torch.empty((batch,), dtype=torch.float32, device=dev)
                    for f in range(c0 // d, (c0 + nc) // d):
                        fm_mask |= 1 << f
            plan = K.UniformPlan(feats, lin_tabs, dense, x, linear, fm, fm_mask)
            # with PNN's products placed, the gather's zero padding stops at the embeddings: the product columns
            # behind them are written by the product kernels, the dense columns by append_dense
            plan.g.x_cols = (self.main_ld if only_fast and not self.pnn_cols
                             else self.fast_n * fast_slots[0].dim)
            if peer is not None:
                plan.set_peers(self.dist.world, peer[0].table, peer[1].table if peer[1] is not None else None)
            from . import ops
            kd = self.main_width + (self.tail_done[1] if self.tail_done is not None else 0)
            if (self.planes_hint == kd and only_fast and not self.pnn_cols and batch >= 128
                    and ops.GEMM_PRECISION == L.GEMM_BF16X3):
                # the first Dense reads x[:, :kd] as its GEMM operand: the gather writes its bf16 planes too
                self.planes_result = (kd, plan.set_planes(kd))
            K.embed_gather_uniform_fwd(plan, batch)
            if fm is not None:
                self.fm_result = (self.fm_hint, E.Var(fm.reshape(batch, 1)))
            if linear is not None:
                self.lin_result = E.Var(linear.reshape(batch, 1))
        # ---- generic launch for everything else ------------------------------------------------------
        if generic:
            feats = []
            for s in generic:
                buf = bufs[id(s)] if s.buf == "seq" else bufs[s.buf]
                feats.append(self._feature(s, feed, buf.data, buf.data.stride(0)))
            K.embed_gather_fwd(feats, batch)
        # ---- hand the windows to the graph executor ---------------------------------------------------
        from . import ops
        vlin = E.Var(None, owner=self, name="__virtual_lin__")   # virtual: only its row-sum exists this step
        for s in self.slots:
            if s.buf == "lin" and lin_fused:
                base = vlin
                out = E.Var(None, base=base, col0=s.col, ncols=s.dim, owner=self, vshape=(batch, 1, s.dim))
            elif s.buf == "seq":
                base = bufs[id(s)]
                out = ops._window(base, 0, s.maxlen * s.dim, (batch, s.maxlen, s.dim))
            else:
                base = bufs[s.buf]
                out = ops._window(base, s.col, s.dim, (batch, 1, s.dim))
            if s.pool == L.POOL_NONE and s.mask_zero:
                out.mask = E.KMask(ids=[feed[s.input_name].data], hashed=s.hash)
            out.requires_grad = grad and s.emb.embeddings.trainable
            self.results[id(s.node)] = out
            for vn in s.virtual_nodes:
                if vn is not s.node:
                    self.results[id(vn)] = VIRTUAL
        for node in self.field_wise_plan.virtual:      # never formed: a Var without data
            self.results[id(node)] = E.Var(None, vshape=(batch,) + tuple(node.outputs[0].shape[1:]))
        if grad:
            outs = [b for b in bufs.values()]
            if self.fm_result is not None:
                outs.append(self.fm_result[1])
            if self.lin_result is not None:
                outs.append(self.lin_result)
            for o in outs:
                o.requires_grad = True
            tape = E.current_tape()
            tape.record(outs, lambda grads: self._backward(feed, bufs, plan, fast_slots, generic, lin_fused,
                                                           batch))

    def _feature(self, s, feed, out, out_ld, table=None, src_table=None):
        ids = feed[s.input_name].data
        length = feed[s.len_name].data if s.len_name else None
        weight = feed[s.weight_name].data if s.weight_name else None
        if length is not None and length.dtype != torch.int32:
            raise ValueError("sequence lengths must be int32")
        tab = table if table is not None else s.emb.embeddings.materialize()
        shard = s.emb.embeddings.opt_state.get("shard")        # (rank, world, full vocabulary) when row-sharded
        return K.make_feature(tab, ids, out, out_col=s.col if s.buf != "seq" else 0, out_ld=out_ld,
                              maxlen=s.maxlen, pool=s.pool, mask_mode=s.mask_mode, length=length,
                              weight=weight, weight_mode=s.weight_mode, hash_mode=s.hash[0],
                              src_table=src_table, vocab=shard[2] if shard else s.emb.input_dim)

    @staticmethod
    def _target(w, opt):
        """(buffer, scale) for a table in the fused scatter; frozen tables land in a scratch buffer."""
        if not w.trainable:
            scratch = w.opt_state.get("scratch")
            if scratch is None:
                scratch = w.opt_state["scratch"] = torch.empty_like(w.data)
            return scratch, 0.0
        return _grad_target(w, opt)

    def _backward(self, feed, bufs, plan, fast_slots, generic, lin_fused, batch):
        opt = E.current_opt()
        if fast_slots:
            main = bufs["main"]
            dx = main.grad
            dfm = self.fm_result[1].grad if self.fm_result is not None else None
            dlin = self.lin_result.grad if self.lin_result is not None else None
            if (dx is not None or dfm is not None or dlin is not None) and getattr(self, "route", None) is not None:
                # sharded: gradient rows are formed in request order, return to their owners over NVLink
                # and are applied there by the fused SGD scatter (scale = -lr / world: global-batch mean)
                st, tabs, ltabs, dimf = self.route
                dev = main.data.device
                # every (b, f) owns a distinct row of the buffers: the scatter writes (no zero-fill, no RMW)
                grows = torch.empty((st["n_send"], dimf), dtype=torch.float32, device=dev)
                glin = torch.empty((st["n_send"],), dtype=torch.float32, device=dev) if lin_fused else None
                if dlin is None and glin is not None:
                    K.fill(glin, 0.0)
                pos = st["pos"]
                feats = [K.make_feature(grows, pos[:, f], main.data, out_col=s.col, out_ld=self.main_ld)
                         for f, s in enumerate(fast_slots)]
                bplan = K.UniformPlan(feats, [glin] * len(fast_slots) if lin_fused else None, None, main.data,
                                      None, None, plan.g.fm_mask[0])
                bplan.g.x_cols = plan.g.x_cols
                bplan.g.flags = L.UNIFORM_STORE_GRADS
                K.embed_scatter_uniform_bwd(bplan, dx, None if dfm is None else dfm.reshape(-1).contiguous(),
                                            None if dlin is None else dlin.reshape(-1).contiguous(),
                                            1.0, 1.0, batch, fm_sum=plan.fm_sum)
                lr = opt["optimizer"].lr if opt and opt.get("optimizer") else 0.0
                sc = -lr / self.dist.world
                self.exchange.push(st, tabs, ltabs, dimf, grows, glin, sc, sc)
            elif (dx is not None or dfm is not None or dlin is not None) and plan.g.world > 1:
                # peer mode: every rank applies its gradient rows at the owners (red.add over NVLink) with
                # scale -lr / world (global-batch mean).  The all-reduce below separates the gathers of ALL
                # ranks from the first update; the dense-gradient all-reduce at the end of the step separates
                # the updates from the next step's gathers.
                from . import parallel
                emb, lin, token = self.peers
                parallel.device_barrier(self.dist, token)
                lr = opt["optimizer"].lr if opt and opt.get("optimizer") else 0.0
                sc = -lr / self.dist.world
                feats = [self._feature(s, feed, main.data, self.main_ld) for s in fast_slots]
                bplan = K.UniformPlan(feats, None, None, main.data, None, None, plan.g.fm_mask[0])
                bplan.g.x_cols = plan.g.x_cols
                bplan.set_peers(self.dist.world, emb.table, lin.table if (lin is not None and lin_fused) else None)
                K.embed_scatter_uniform_bwd(bplan, dx, None if dfm is None else dfm.reshape(-1).contiguous(),
                                            None if dlin is None else dlin.reshape(-1).contiguous(),
                                            sc, sc, batch, fm_sum=plan.fm_sum)
            elif dx is not None or dfm is not None or dlin is not None:
                tgts = [self._target(s.emb.embeddings, opt) for s in fast_slots]
                feats = [self._feature(s, feed, main.data, self.main_ld, table=tgt)
                         for s, (tgt, _) in zip(fast_slots, tgts)]
                scale = max(abs(sc) for _, sc in tgts) * (-1.0 if any(sc < 0 for _, sc in tgts) else 1.0)
                lin_tabs, lin_scale = None, 0.0
                if lin_fused:
                    lt = [self._target(s.emb.embeddings, opt) for s in self.lin]
                    lin_tabs = [t.reshape(-1) for t, _ in lt]
                    lin_scale = max(abs(sc) for _, sc in lt) * (-1.0 if any(sc < 0 for _, sc in lt) else 1.0)
                bplan = K.UniformPlan(feats, lin_tabs, None, main.data, None, None, plan.g.fm_mask[0])
                bplan.g.x_cols = plan.g.x_cols
                if getattr(self, "sorted_update", False) and all(sc < 0 for _, sc in tgts):
                    o = opt["optimizer"]
                    adagrad = o.name == "adagrad"
                    acc = lacc = None
                    if adagrad:
                        acc = [self._adagrad_state(s.emb.embeddings) for s in fast_slots]
                        lacc = [self._adagrad_state(s.emb.embeddings).reshape(-1) for s in self.lin] if lin_fused else None
                    K.embed_update_sorted(bplan, dx, None if dfm is None else dfm.reshape(-1).contiguous(),
                                          None if dlin is None else dlin.reshape(-1).contiguous(),
                                          1 if adagrad else 0, o.lr, o.lr, 1e-7, acc, lacc, batch)
                    return self._backward_generic(feed, bufs, generic, opt, batch)
                K.embed_scatter_uniform_bwd(bplan, dx, None if dfm is None else dfm.reshape(-1).contiguous(),
                                            None if dlin is None else dlin.reshape(-1).contiguous(),
                                            scale, lin_scale, batch, fm_sum=plan.fm_sum)
        self._backward_generic(feed, bufs, generic, opt, batch)

    @staticmethod
    def _adagrad_state(w):
        acc = w.opt_state.get("acc")
        if acc is None:
            acc = w.opt_state["acc"] = torch.empty_like(w.data)
            K.fill(acc, 0.1)               # Keras initial_accumulator_value
        return acc

    def _backward_generic(self, feed, bufs, generic, opt, batch):
        feats, scales = [], []
        flat = {}            # (rows, scale) -> features of plain sequences re-described as B*T single lookups
        for s in generic:
            if not s.emb.embeddings.trainable:
                continue
            buf = bufs[id(s)] if s.buf == "seq" else bufs[s.buf]
            if buf.grad is None:
                continue
            tgt, scale = _grad_target(s.emb.embeddings, opt)
            src = s.emb.embeddings.data if s.pool == L.POOL_MAX else None
            ids = feed[s.input_name].data
            g = buf.grad
            if (s.buf == "seq" and s.maxlen > 1 and s.hash[0] == L.HASH_NONE and ids.dim() == 2 and ids.is_contiguous()
                    and g.is_contiguous() and g.shape[1] == s.maxlen * s.dim):
                # a [B, T] behaviour sequence scattered as B*T independent rows: one sub-warp per ROW instead of
                # one per sample walking its T rows in sequence (8192 tasks x 50 dependent updates at C4)
                shard = s.emb.embeddings.opt_state.get("shard")
                f = K.make_feature(tgt, ids.reshape(-1), g.reshape(-1, s.dim), maxlen=1,
                                   vocab=shard[2] if shard else s.emb.input_dim)
                flat.setdefault((batch * s.maxlen, scale), []).append(f)
                continue
            feats.append(self._feature(s, feed, g, g.stride(0), table=tgt, src_table=src))
            scales.append(scale)
        # one launch per distinct scale (normally exactly one)
        for sc in sorted(set(scales)):
            K.embed_scatter_add([f for f, s_ in zip(feats, scales) if s_ == sc], batch, sc)
        for (rows, sc), fs in flat.items():
            K.embed_scatter_add(fs, rows, sc)

    # ---- fusion hooks used by layers ---------------------------------------------------------------
    def lookup_fm(self, x):
        """FM layer: return the in-kernel FM if this step computed it for exactly this window."""
        if x.base is None or x.base.owner is not self or x.ncols == -1:
            return None
        if x.base.ncols != self.main_width or x.base.data is None or x.base.data.shape[1] != self.main_ld:
            return None
        key = (x.col0, x.ncols)
        if self.fm_result is not None and self.fm_result[0] == key:
            return self.fm_result[1]
        if self.fast:
            self.fm_hint = key      # fused from the next step on
        return None

    def lookup_planes(self, x, t2):
        """ops.dense in BF16X3: the bf16 planes of ``x`` (2-D view ``t2``) if this step's gather wrote them, i.e. if
        ``x`` is the leading window of the main buffer that the planner learned on an earlier step."""
        base = x.base
        if (x.col0 != 0 or x.ncols == -1 or base.data is None or base.ncols != self.main_width
                or t2.data_ptr() != base.data.data_ptr() or t2.stride(0) != base.data.stride(0)):
            return None
        if self.planes_result is not None and self.planes_result[0] == t2.shape[1]:
            return self.planes_result[1]
        if self.fast:
            self.planes_hint = t2.shape[1]      # written by the gather from the next step on
        return None

    def lookup_rowsum(self, x):
        if x.base is None or x.base.owner is not self:
            return None
        if x.base.name == "__virtual_lin__":
            if x.col0 == 0 and x.ncols == self.lin_width and self.lin_result is not None:
                return self.lin_result
            raise L.B2ctrError("the linear-term lookups were fused into a row-sum but a layer asked for the rows")
        if (self.fast and x.base.ncols == self.lin_width and x.col0 == 0 and x.ncols == self.lin_width
                and x.base.data.shape[1] == self.lin_ld and self._lin_matches_fast()):
            self.lin_hint = True
        return None

    def dnn_input_place(self, layer):
        """(DnnInputPlacement, index) when ``layer`` writes its output into the first DNN layer's input."""
        return self.dnn_places.get(id(layer))

    def fefm_place(self, layer, x):
        """The [B, P] window of this step's main buffer, behind the dense columns, where the FEFMLayer ``layer``
        writes its scores (ops.fefm ``out``), or None.  With the embeddings at [0, main_width) and
        combined_dnn_input's dense columns behind them, DeepFEFM's concat([combined_dnn_input, scores]) is then the
        zero-copy window [0, main_width + n_dense + P) of the buffer, the first Dense reads it in place and its data
        gradient becomes the buffer's gradient, whose score columns the FEFM backward reads in place."""
        from . import ops
        P = self.fefm_places.get(id(layer))
        base = x.base
        if (P is None or base is None or base.owner is not self or base.data is None
                or base.ncols != self.main_width or base.data.shape[1] != self.main_ld):
            return None
        b = base.data.shape[0]
        return ops._window(base, self.main_width + self.tail_reserve, P, (b, P))

    def pnn_place(self, layer, x):
        """The [B, P] window of this step's main buffer where PNN's InnerProductLayer / OutterProductLayer ``layer``
        writes its scores (ops.pnn_inner / ops.pnn_outer ``out``), or None.  ``x`` must be the embeddings' window
        [0, main_width): the products then follow it in the order of PNN's concat([linear_signal, inner, outer]),
        so that concatenation is a zero-copy window, combined_dnn_input copies only the dense columns behind it
        (append_dense) and the first Dense reads the buffer in place.  Its data gradient becomes the buffer's
        gradient, whose product columns the product backwards read in place."""
        from . import ops
        rel = self.pnn_places.get(id(layer))
        base = x.base
        if (rel is None or base is None or base.owner is not self or base.data is None or x.ncols == -1
                or x.col0 != 0 or x.ncols != self.main_width or base.ncols != self.main_width
                or base.data.shape[1] != self.main_ld):
            return None
        b, f, _ = x.data.shape
        P = f * (f - 1) // 2
        return ops._window(base, self.main_width + rel, P, (b, P))

    def regulated(self, layer, x):
        """RegulationModule ``layer`` on ``x``: when the planner pairs it with a second module reading the same tensor,
        one launch writes both gated outputs; the partner's becomes that node's result.  Else None."""
        from . import ops
        p = self.regulate_plan.pairs.get(id(layer))
        if p is None:
            return None
        partner, node = p
        _, (y0, y1) = ops.regulate("copy", x, gates=[(layer.g, layer.tau), (partner.g, partner.tau)], want_u=False)
        self.results[id(node)] = y1
        return y0

    def bridged(self, layer, mode, operands):
        """BridgeModule ``layer`` whose output reaches only Reshape -> two RegulationModules: one launch writes the two
        gated outputs as those modules' results, the bridge output and its reshape are never written (VIRTUAL).
        Else None."""
        from . import ops
        plan = self.regulate_plan.bridges.get(id(layer))
        if plan is None:
            return None
        reshape, regs = plan
        _, ys = ops.regulate(mode, *operands, gates=[(l.g, l.tau) for l, _ in regs], want_u=False)
        self.results[id(reshape)] = VIRTUAL
        for (_, node), y in zip(regs, ys):
            self.results[id(node)] = y
        return VIRTUAL

    def conv_stacked(self, layer, x):
        """The first Conv2D of a chain the planner claimed (ConvStackPlan): one launch runs every Conv2D and
        KMaxPooling of the chain on ``x`` and becomes the last KMaxPooling's result; the maps between are never
        written (VIRTUAL).  Else None."""
        from . import ops
        chain = self.conv_plan.chains.get(id(layer))
        if chain is None:
            return None
        b, rows, dim, channels = x.data.shape
        last = chain[-1]
        res = ops.conv_stack(x, [n.layer.stage() for n in chain], rows, dim, channels,
                             (b,) + tuple(last.outputs[0].shape[1:]))
        for n in chain[1:-1]:
            self.results[id(n)] = VIRTUAL
        self.results[id(last)] = res
        return VIRTUAL

    def field_wise_groups(self, layer):
        """FieldWiseBiInteraction ``layer`` the planner claimed (FieldWisePlan): its groups as lists of this step's
        gather-buffer windows, to be read in place (the groups' concatenations are Vars without data).  Else None."""
        groups = self.field_wise_plan.groups.get(id(layer))
        if groups is None:
            return None
        return [[self.results[id(n)] for n in g] for g in groups]

    def append_dense(self, emb_flat, dense_flat):
        """combined_dnn_input: place the dense features behind the embeddings (and PNN's placed products) in the
        main buffer so the DNN input is a zero-copy window.  Returns the window or None."""
        from . import ops
        if emb_flat.base is not None and isinstance(emb_flat.base.owner, DnnInputPlacement):
            return emb_flat.base.owner.append_dense(emb_flat, dense_flat)
        if (emb_flat.base is None or emb_flat.base.owner is not self or emb_flat.ncols == -1
                or emb_flat.base.ncols != self.main_width or emb_flat.base.data is None
                or emb_flat.base.data.shape[1] != self.main_ld):
            return None
        width = self.main_width + self.pnn_cols if self.pnn_cols else self.main_width
        if emb_flat.col0 != 0 or emb_flat.ncols != width:
            return None
        b = emb_flat.data.shape[0]
        nd = dense_flat.data.shape[1]
        if width + nd > self.main_ld:
            return None
        base = emb_flat.base
        if self.pnn_cols:
            # the fused gather would write its dense tail at main_width, over the products: always copy
            src, ld = dense_flat.flat2d()
            if src is None:
                return None
            K.copy2d(src, ld, base.data, base.data.stride(0), b, nd, dst_off=width)
            return ops._window(base, 0, width + nd, (b, width + nd))
        is_pack = (dense_flat.base is not None and dense_flat.base.name == "__dense_pack__"
                   and dense_flat.ncols != -1)
        if is_pack and self.tail_done == (dense_flat.col0, nd):
            pass    # the gather kernel already wrote it
        else:
            src, ld = dense_flat.flat2d()
            if src is None:
                return None
            K.copy2d(src, ld, base.data, base.data.stride(0), b, nd, dst_off=self.main_width)
            if is_pack and self.fast and len(self.main) == self.fast_n:
                self.tail_hint = (dense_flat.col0, nd)
        return ops._window(base, 0, self.main_width + nd, (b, self.main_width + nd))


class DnnInputPlacement(object):
    """n BilinearInteraction layers whose [B,P,E] outputs reach the DNN only as Flatten(Concat(outputs, -1))
    (FiBiNET, deepctr/models/fibinet.py:58), possibly followed by combined_dnn_input's dense columns.  The layers
    write their pairs straight into one [B, ld] buffer, ld = round_up(n*P*E + n_dense, 4): pair p of layer k at
    columns p*n*E + k*E, which is exactly the layout of the concatenation.  The Concat is then a zero-copy window,
    combined_dnn_input copies only the dense columns behind it, and the first Dense reads the buffer in place; its
    data gradient is adopted as the buffer's gradient and each layer's backward reads its strided part."""

    def __init__(self, n, P, E, ndense):
        self.n, self.P, self.E, self.ndense = n, P, E, ndense
        self.width = n * P * E
        self.ld = (self.width + ndense + 3) // 4 * 4
        self.buf = None                 # this step's buffer Var, dropped once the backward has consumed it
        self.outs = [None] * n

    def _release(self):
        """Forget this step's buffer (5.46 GB at C2), so that it is freed with the step's last reference and never
        coexists with the next step's."""
        self.buf = None
        self.outs = [None] * self.n

    def out_view(self, k, b, device):
        """Where layer k writes its [B,P,E] output this step (a new buffer when a step starts)."""
        if self.buf is None or self.outs[k] is not None or self.buf.data.shape[0] != b:
            self._release()
            t = torch.empty((b, self.ld), dtype=torch.float32, device=device)
            self.buf = E.Var(t, ncols=self.width, owner=self, name="__dnn_input__")
            self.outs = [None] * self.n
        t = self.buf.data
        return t.as_strided((b, self.P, self.E), (self.ld, self.n * self.E, 1), t.storage_offset() + k * self.E)

    def placed(self, k, var):
        var.owner = self
        self.outs[k] = var

    def placed_concat(self, xs, axis):
        """ops.concat of the n placed outputs along the last axis: the window [0, n*P*E) of the buffer."""
        from . import ops
        if (self.buf is None or axis not in (-1, 2) or len(xs) != self.n
                or any(a is not b for a, b in zip(xs, self.outs))):
            return None
        base, b, n, E_ = self.buf, self.buf.data.shape[0], self.n, self.E

        def bwd(grads):
            g = grads[0]
            for k, v in enumerate(xs):
                E.add_grad(v, g.as_strided((b, self.P, E_), (g.stride(0), n * E_, 1), g.storage_offset() + k * E_))
            self._release()             # only the tape still holds the buffer; it goes when the backward ends

        E.record([base], xs, bwd)
        return ops._window(base, 0, self.width, (b, self.P, n * E_))

    def append_dense(self, emb_flat, dense_flat):
        from . import ops
        nd = dense_flat.data.shape[1]
        if (emb_flat.col0 != 0 or emb_flat.ncols != self.width or self.width + nd > self.ld
                or dense_flat.requires_grad):
            return None
        src, ld = dense_flat.flat2d()
        if src is None:
            return None
        base = emb_flat.base
        b = base.data.shape[0]
        K.copy2d(src, ld, base.data, self.ld, b, nd, dst_off=self.width)
        base.ncols = self.width + nd
        return ops._window(base, 0, self.width + nd, (b, self.width + nd))


# FiBiNET's bilinear outputs, DeepFEFM's FEFM scores and PNN's products written in place into the DNN input; False
# keeps every layer's own output buffer (same results, used by the tests to compare the two)
DNN_INPUT_PLACEMENT = True


def _plan_fefm_input(model, consumers, out_ids):
    """{id(FEFMLayer): P} for DeepFEFM's DNN input concat([combined_dnn_input(...), NoMask(FEFM(x))], axis=1)
    (deepctr/models/deepfefm.py:64-78) when that concatenation reaches only the DNN: the planner then reserves the
    P score columns behind the dense tail of the main buffer (fefm_place).  Decided once from the model's graph;
    every other graph plans nothing and keeps its row pitch."""
    if not DNN_INPUT_PLACEMENT:
        return {}
    from .layers.core import DNN
    from .layers.interaction import FEFMLayer
    from .layers.utils import Concat, NoMask, _CombinedDNNInput
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1
    places = {}
    for node in model._order:
        if not isinstance(node.layer, Concat) or node.layer.axis not in (1, -1):
            continue
        srcs = E._flatten(node.inputs)
        if len(srcs) != 2 or len(srcs[0].shape) != 2 or len(srcs[1].shape) != 2:
            continue
        head, tail = srcs
        if not isinstance(head.node.layer, (_CombinedDNNInput, E.Flatten)) or len(consumers[id(head)]) != 1:
            continue
        while isinstance(tail.node.layer, NoMask):                   # concat_func of the single FEFM output
            tail = E._flatten(tail.node.inputs)[0]
        fefm = tail.node.layer
        if not isinstance(fefm, FEFMLayer) or calls[id(fefm)] != 1 or id(fefm) in places:
            continue
        out = node.outputs[0]
        oc = consumers[id(out)]
        if len(oc) != 1 or id(out) in out_ids or not isinstance(oc[0].layer, DNN):
            continue
        places[id(fefm)] = int(tail.shape[1])
    return places


def _plan_pnn_input(model, consumers, out_ids):
    """({id(product layer): column offset behind the embeddings}, total product columns) for PNN's DNN input
    concat([linear_signal, Flatten(InnerProductLayer(...)), OutterProductLayer(...)]) (deepctr/models/pnn.py:46-63,
    either product or both) when that concatenation reaches the first DNN layer only through combined_dnn_input:
    the planner then reserves the product columns between the embeddings and the dense columns of the main buffer
    (pnn_place).  Decided once from the model's graph; every other graph plans nothing and keeps its row pitch."""
    if not DNN_INPUT_PLACEMENT:
        return {}, 0
    from .layers.core import DNN
    from .layers.interaction import InnerProductLayer, OutterProductLayer
    from .layers.utils import Concat, NoMask, _CombinedDNNInput
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1

    def only_use(t):
        return len(consumers[id(t)]) == 1 and id(t) not in out_ids

    for node in model._order:
        if not isinstance(node.layer, Concat) or node.layer.axis not in (1, -1):
            continue
        srcs = E._flatten(node.inputs)
        if not 2 <= len(srcs) <= 3 or any(len(t.shape) != 2 or not only_use(t) for t in srcs):
            continue
        if not isinstance(srcs[0].node.layer, E.Reshape):
            continue
        products = []
        for t in srcs[1:]:
            layer = t.node.layer
            if isinstance(layer, E.Flatten):                          # Flatten(InnerProductLayer()(...))
                inner = E._flatten(t.node.inputs)[0]
                layer = inner.node.layer
                if not (isinstance(layer, InnerProductLayer) and layer.reduce_sum and only_use(inner)):
                    break
            elif not isinstance(layer, OutterProductLayer):
                break
            if calls[id(layer)] != 1:
                break
            products.append((layer, int(t.shape[1])))
        if len(products) != len(srcs) - 1 or len(set(id(l) for l, _ in products)) != len(products):
            continue
        # combined_dnn_input: NoMask + Flatten of the single deep input, then _CombinedDNNInput with the dense
        # features or the DNN directly
        flat = node.outputs[0]
        while only_use(flat) and isinstance(consumers[id(flat)][0].layer, (NoMask, E.Flatten)):
            flat = consumers[id(flat)][0].outputs[0]
        if not only_use(flat):
            continue
        nxt = consumers[id(flat)][0]
        if isinstance(nxt.layer, _CombinedDNNInput):
            if E._flatten(nxt.inputs)[0] is not flat or not only_use(nxt.outputs[0]):
                continue
            nxt = consumers[id(nxt.outputs[0])][0]
        if not isinstance(nxt.layer, DNN):
            continue
        places, col = {}, 0
        for layer, w in products:
            places[id(layer)] = col
            col += w
        return places, col
    return {}, 0


def _plan_dnn_input(model, consumers, out_ids):
    """{id(BilinearInteraction layer): (DnnInputPlacement, index)}, decided once from the model's graph."""
    if not DNN_INPUT_PLACEMENT:
        return {}
    from .layers.core import DNN
    from .layers.interaction import BilinearInteraction
    from .layers.utils import Concat, NoMask, _CombinedDNNInput
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1
    places = {}
    for node in model._order:
        if not isinstance(node.layer, Concat) or node.layer.axis not in (-1, 2):
            continue
        srcs = E._flatten(node.inputs)
        layers = [t.node.layer for t in srcs]
        if (len(srcs) < 2 or not all(isinstance(l, BilinearInteraction) for l in layers)
                or len(set(id(l) for l in layers)) != len(layers) or any(calls[id(l)] != 1 for l in layers)
                or any(len(consumers[id(t)]) != 1 or id(t) in out_ids for t in srcs)
                or len(set(tuple(t.shape) for t in srcs)) != 1):
            continue
        # then only Flatten / NoMask (combined_dnn_input wraps the flattened concat in both) up to the DNN input
        flat, fc = node.outputs[0], None
        while True:
            fc = consumers[id(flat)]
            if len(fc) != 1 or id(flat) in out_ids or not isinstance(fc[0].layer, (E.Flatten, NoMask)):
                break
            flat = fc[0].outputs[0]
        if flat is node.outputs[0] or len(fc) != 1 or id(flat) in out_ids or len(flat.shape) != 2:
            continue
        ndense = 0
        if isinstance(fc[0].layer, _CombinedDNNInput):
            ins = E._flatten(fc[0].inputs)
            if ins[0] is not flat:
                continue
            ndense = int(np.prod(ins[1].shape[1:]))
        elif not isinstance(fc[0].layer, DNN):
            continue
        _, P, Ed = srcs[0].shape
        pl = DnnInputPlacement(len(srcs), int(P), int(Ed), ndense)
        for k, l in enumerate(layers):
            places[id(l)] = (pl, k)
    return places


class RegulatePlan(object):
    """EDCN's information sharing (deepctr/models/edcn.py:66-85) with fewer passes over [B, F*E]:

    * ``pairs`` {id(RegulationModule): (partner module, partner node)}: two RegulationModules reading one tensor (the
      embeddings' concat_func, a window of the gather buffer read in place, or the Reshape of a 'concatenation'
      bridge's Dense) are one 'copy' launch with both gates;
    * ``bridges`` {id(BridgeModule): (Reshape node, [(module, node)] * 2)}: a non-concatenation BridgeModule whose
      output reaches only Reshape([F, E]), which feeds only two RegulationModules, is one launch in the bridge's
      mode that writes the two gated outputs; bridge_out and its reshape are never written.

    Decided once from the model's graph; anything else runs layer by layer on the same kernel."""

    def __init__(self, pairs, bridges):
        self.pairs, self.bridges = pairs, bridges


def _plan_regulate(model, consumers, out_ids):
    from .layers.core import RegulationModule
    from .layers.interaction import BridgeModule
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1

    def regulators(t):
        """The two RegulationModule nodes that are all of ``t``'s consumers, or None."""
        cs = consumers[id(t)]
        if id(t) in out_ids or len(cs) != 2 or len(t.shape) != 3 or cs[0].layer is cs[1].layer:
            return None
        if all(isinstance(c.layer, RegulationModule) and calls[id(c.layer)] == 1 for c in cs):
            return cs
        return None

    pairs, bridges, claimed = {}, {}, set()
    for node in model._order:
        layer = node.layer
        if not isinstance(layer, BridgeModule) or layer.bridge_type == "concatenation" or calls[id(layer)] != 1:
            continue
        out = node.outputs[0]
        cs = consumers[id(out)]
        if id(out) in out_ids or len(cs) != 1 or not isinstance(cs[0].layer, E.Reshape):
            continue
        regs = regulators(cs[0].outputs[0])
        if regs is not None:
            bridges[id(layer)] = (cs[0], [(c.layer, c) for c in regs])
            claimed.add(id(cs[0].outputs[0]))
    for node in model._order:
        for t in node.outputs:
            regs = regulators(t) if id(t) not in claimed else None
            if regs is not None:
                pairs[id(regs[0].layer)] = (regs[1].layer, regs[1])
    return RegulatePlan(pairs, bridges)


class ConvStackPlan(object):
    """CCPM's convolution stack (deepctr/models/ccpm.py:58-70) served by one b2ctr_conv_stack launch: the chain
    concat_func(embeddings) -> Lambda(expand_dims(x, 3)) -> [Conv2D -> KMaxPooling(axis=1)] x l -> Flatten, every
    intermediate with this one consumer, runs when its first Conv2D is called.  The input is read in place (a
    window of the gather buffer), the per-layer maps are never written, and Flatten of the result is a view.

    ``chains`` {id(first Conv2D layer): [Conv2D node, KMaxPooling node, ...]}.  Decided once from the model's graph;
    any other graph, or a stack beyond the kernel's limits, runs layer by layer on the same kernel."""

    def __init__(self, chains):
        self.chains = chains


def _plan_conv_stack(model, consumers, out_ids):
    from . import kernels as K
    from .layers.sequence import KMaxPooling
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1

    def only(t, cls):
        """The single consumer node of ``t`` when it is a ``cls`` called once, else None."""
        cs = consumers[id(t)]
        if id(t) in out_ids or len(cs) != 1 or not isinstance(cs[0].layer, cls) or calls[id(cs[0].layer)] != 1:
            return None
        return cs[0]

    chains = {}
    for node in model._order:
        if not isinstance(node.layer, E.Lambda) or not isinstance(node.inputs, E.KTensor):
            continue
        src, out = node.inputs, node.outputs[0]
        if len(src.shape) != 3 or tuple(out.shape) != tuple(src.shape) + (1,):
            continue
        chain, t = [], out
        while True:
            conv = only(t, E.Conv2D)
            if conv is None:
                break
            pool = only(conv.outputs[0], KMaxPooling)
            if pool is None or pool.layer.axis != 1:
                break
            chain += [conv, pool]
            t = pool.outputs[0]
        if not chain or only(t, E.Flatten) is None:
            continue
        try:
            K.conv_stack_check(int(src.shape[1]), 1, [n.layer.stage()[:3] for n in chain])
        except ValueError:
            continue
        chains[id(chain[0].layer)] = chain
    return ConvStackPlan(chains)


class FieldWisePlan(object):
    """FLEN's FieldWiseBiInteraction (deepctr/models/flen.py:69-70) served in place: a FieldWiseBiInteraction called
    once, whose every input is concat_func(members, axis=1) (a Concat, or NoMask for a one-member group) of
    embedding or pooled windows of the gather buffer, each concatenation used by that layer only, runs as one
    b2ctr_field_wise_bi launch reading the members where the gather wrote them.  The concatenations are never
    formed (their results are Vars without data), whether or not a group's members are adjacent.

    ``groups`` {id(layer): [[member slot node, ...] per group]}, ``virtual`` the concatenation nodes.  Decided
    once from the model's graph; any other graph runs the layer on its concrete inputs, on the same kernel."""

    def __init__(self, groups, virtual):
        self.groups = groups
        self.virtual = virtual


def _plan_field_wise(model, consumers, out_ids, main_slots):
    from .layers.interaction import FieldWiseBiInteraction
    from .layers.utils import Concat, NoMask
    slot_out = {id(s.node.outputs[0]): s.node for s in main_slots}
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1
    groups, virtual = {}, []
    for node in model._order:
        if not isinstance(node.layer, FieldWiseBiInteraction) or calls[id(node.layer)] != 1:
            continue
        if not isinstance(node.inputs, (list, tuple)) or len(node.inputs) < 2:
            continue
        plan, concats = [], []
        for t in node.inputs:
            src = t.node
            if id(t) in out_ids or len(consumers[id(t)]) != 1:
                break
            if isinstance(src.layer, Concat) and src.layer.axis in (1, -2):
                members = E._flatten(src.inputs)
            elif isinstance(src.layer, NoMask) and isinstance(src.inputs, E.KTensor):
                members = [src.inputs]
            else:
                break
            if not all(id(m) in slot_out and len(m.shape) == 3 for m in members):
                break
            plan.append([slot_out[id(m)] for m in members])
            concats.append(src)
        else:
            dims = set(int(n.outputs[0].shape[-1]) for g in plan for n in g)
            nfield = sum(int(n.outputs[0].shape[1]) for g in plan for n in g)
            try:
                K.field_wise_bi_check(nfield, len(plan), dims.pop())
            except ValueError:
                continue
            if dims:
                continue
            groups[id(node.layer)] = plan
            virtual += concats
    return FieldWisePlan(groups, virtual)


class FieldAwarePlan(object):
    """ONN's field-aware products (deepctr/models/onn.py:79-97) served by one b2ctr_ffm_product_fwd launch: the
    output of pair p's ``multiply`` (or of the ``K.sum`` Lambda behind it) is the column window [p*E, (p+1)*E) (or
    [p, p+1)) of one [B, P*E] (or [B, P]) buffer, so concat_func + Flatten of the P outputs is a zero-copy view of
    it.  The backward is one tape node on that buffer: b2ctr_ffm_product_bwd writes every lookup's gradient row
    into a [B, F(F-1)*E] scratch at the tables' pre-step values, then b2ctr_embed_scatter_add applies the scratch,
    one single-valued or pooled feature per lookup, to the tables (fused SGD) or their dense gradients.

    A VarLenSparseFeat field is pooled per partner by the generic gather into a [B, (F-1)*E] operand that the
    product kernel reads; its gradient rows go back through the same scatter's pooling Jacobian.

    ``fields[a]``: (input name, maxlen, pool, hash mode, vocabulary); ``tables[a*F + b]``: (a, b) -> Embedding layer
    (None on the diagonal); ``pair_nodes[p]``: the node whose output pair p's window is; ``virtual``: every other
    node the plan replaces."""

    def __init__(self, fields, tables, E_, reduce_sum, pair_nodes, virtual, claimed):
        self.fields, self.E, self.reduce_sum = fields, E_, reduce_sum
        self.F = len(fields)
        self.table_of = tables
        self.tables = [(k, t) for k, t in enumerate(tables) if t is not None]
        self.pair_nodes, self.virtual, self.claimed = pair_nodes, virtual, claimed
        self.P = self.F * (self.F - 1) // 2
        self.width = self.P * (1 if reduce_sum else E_)
        self.ld = (self.width + 3) // 4 * 4
        self._ptrs, self._dev_ptrs = None, None

    def n_tables(self):
        return len(self.tables)

    def numel(self):
        return sum(t.embeddings.numel() for _, t in self.tables)

    def _slot(self, a, b):
        return b - (b > a)

    def _table_array(self, dev):
        """The device array [F*F] of table pointers, kept at one address (a captured step reads it) and rewritten
        in place only when a table moved."""
        ptrs = tuple(t.embeddings.materialize().data_ptr() if t is not None else 0 for t in self.table_of)
        if ptrs != self._ptrs:
            host = torch.tensor(ptrs, dtype=torch.int64)
            if self._dev_ptrs is None:
                self._dev_ptrs = host.to(dev)
            else:
                self._dev_ptrs.copy_(host)
            self._ptrs = ptrs
        return self._dev_ptrs

    def _bag_features(self, a, feed, buf, tables=None, scale_of=None):
        """The generic-gather features of pooled field a: one bag per partner, at its slot of ``buf``."""
        name, maxlen, pool, hash_mode, vocab = self.fields[a]
        ids = feed[name].data
        out = []
        for b in range(self.F):
            if b == a:
                continue
            emb = self.table_of[a * self.F + b].embeddings
            tab = emb.materialize() if tables is None or tables[a * self.F + b] is None else tables[a * self.F + b]
            col = self._slot(a, b) * self.E if tables is None else (a * (self.F - 1) + self._slot(a, b)) * self.E
            out.append(K.make_feature(tab, ids, buf, out_col=col, out_ld=buf.stride(0), maxlen=maxlen, pool=pool,
                                      mask_mode=L.MASK_ZERO_ID, hash_mode=hash_mode, vocab=vocab,
                                      src_table=emb.data if (tables is not None and pool == L.POOL_MAX) else None))
        return out

    def forward(self, feed, results, grad):
        F, E_ = self.F, self.E
        some = feed[self.fields[0][0]].data
        b, dev = some.shape[0], some.device
        ptrs = self._table_array(dev)
        pooled, kfields = {}, []
        bags = []
        for a, (name, maxlen, pool, hash_mode, vocab) in enumerate(self.fields):
            if pool == L.POOL_NONE:
                kfields.append(K.ffm_field(idx=feed[name].data.reshape(b, -1), vocab=vocab, hash_mode=hash_mode))
            else:
                pooled[a] = torch.empty((b, (F - 1) * E_), dtype=torch.float32, device=dev)
                bags.extend(self._bag_features(a, feed, pooled[a]))
                kfields.append(K.ffm_field(pooled=pooled[a]))
        for c in range(0, len(bags), L.MAX_FEATURES):
            K.embed_gather_fwd(bags[c:c + L.MAX_FEATURES], b)
        buf = E.Var(torch.empty((b, self.ld), dtype=torch.float32, device=dev), ncols=self.width, owner=self,
                    name="__ffm_products__")
        K.ffm_product_fwd(kfields, ptrs, E_, self.reduce_sum, buf.data, 0, b)
        trainable = any(t.embeddings.trainable for _, t in self.tables)
        buf.requires_grad = grad and trainable
        w = 1 if self.reduce_sum else E_
        for p, node in enumerate(self.pair_nodes):
            results[id(node)] = ops_window(buf, p * w, w, (b, 1) if self.reduce_sum else (b, 1, E_))
        for node in self.virtual:
            results[id(node)] = VIRTUAL
        if buf.requires_grad:
            E.current_tape().record([buf], lambda grads: self._backward(feed, buf, pooled, b))

    def _backward(self, feed, buf, pooled, b):
        g = buf.grad
        if g is None:
            return
        F, E_ = self.F, self.E
        opt = E.current_opt()
        ptrs = self._table_array(g.device)
        scratch = torch.empty((b, F * (F - 1) * E_), dtype=torch.float32, device=g.device)
        kfields = []
        for a, (name, maxlen, pool, hash_mode, vocab) in enumerate(self.fields):
            gv = scratch[:, a * (F - 1) * E_:]
            if pool == L.POOL_NONE:
                kfields.append(K.ffm_field(idx=feed[name].data.reshape(b, -1), vocab=vocab, hash_mode=hash_mode,
                                           grad=gv))
            else:
                kfields.append(K.ffm_field(pooled=pooled[a], grad=gv))
        K.ffm_product_bwd(kfields, ptrs, E_, self.reduce_sum, g, 0, b)
        # every lookup's row of the scratch, applied to its table: one feature each, grouped by update scale
        targets = [None] * (F * F)
        for k, t in self.tables:
            if t.embeddings.trainable:
                targets[k] = _grad_target(t.embeddings, opt)
        groups = defaultdict(list)
        for a, (name, maxlen, pool, hash_mode, vocab) in enumerate(self.fields):
            tabs = [tg[0] if tg is not None else None for tg in targets]
            if pool == L.POOL_NONE:
                ids = feed[name].data.reshape(b, -1)
                for c in range(F):
                    if c == a or targets[a * F + c] is None:
                        continue
                    f = K.make_feature(tabs[a * F + c], ids, scratch, out_col=(a * (F - 1) + self._slot(a, c)) * E_,
                                       out_ld=scratch.stride(0), hash_mode=hash_mode, vocab=vocab)
                    groups[targets[a * F + c][1]].append(f)
            else:
                keep = [c for c in range(F) if c != a]
                for c, f in zip(keep, self._bag_features(a, feed, scratch, tables=tabs)):
                    if targets[a * F + c] is not None:
                        groups[targets[a * F + c][1]].append(f)
        for sc, feats in sorted(groups.items()):
            for c in range(0, len(feats), L.MAX_FEATURES):
                K.embed_scatter_add(feats[c:c + L.MAX_FEATURES], b, sc)


def ops_window(base, col0, ncols, shape):
    from . import ops
    return ops._window(base, col0, ncols, shape)


MAX_FFM_FIELDS, MAX_FFM_DIM = 64, 64       # b2ctr_ffm_product_fwd's limits


def _plan_field_aware(model, consumers, out_ids, as_input):
    """The FieldAwarePlan of ONN's graph (deepctr/models/onn.py:79-97), or None.  Per pair (i, j) of
    itertools.combinations order: multiply([lookup_i, lookup_j]), optionally followed by Lambda(K.sum(., axis=-1)),
    where a lookup is NoMask(Embedding(ids)) for a single-valued field or SequencePoolingLayer(combiner,
    supports_masking=True)(Embedding(mask_zero=True)(ids)) for a varlen one, its ids a model input, optionally
    through Hash(vocabulary_size).  Every intermediate has exactly one consumer and every layer one call.  The pairs
    must name F fields and cover all F(F-1)/2 pairs in order, with one table per (field, partner); anything else
    plans nothing and each layer runs as itself."""
    from .layers.sequence import SequencePoolingLayer
    from .layers.utils import Hash, NoMask
    calls = defaultdict(int)
    for node in model._order:
        calls[id(node.layer)] += 1

    def only_use(t):
        return len(consumers[id(t)]) == 1 and id(t) not in out_ids

    def lookup(t):
        if not only_use(t) or calls[id(t.node.layer)] != 1 or not isinstance(t.node.inputs, E.KTensor):
            return None
        outer = t.node
        if isinstance(outer.layer, NoMask):
            pool = L.POOL_NONE
        elif isinstance(outer.layer, SequencePoolingLayer) and outer.layer.supports_masking:
            pool = L.POOL_BY_NAME[outer.layer.mode]
        else:
            return None
        e = outer.inputs
        emb = e.node.layer
        if (not only_use(e) or not isinstance(emb, Embedding) or calls[id(emb)] != 1
                or not isinstance(e.node.inputs, E.KTensor) or emb.mask_zero != (pool != L.POOL_NONE)):
            return None
        virt = [outer, e.node]
        src, hash_mode = e.node.inputs, L.HASH_NONE
        if isinstance(src.node.layer, Hash):
            h = src.node.layer
            if (not only_use(src) or h.mask_zero or h.vocabulary_path or calls[id(h)] != 1
                    or not isinstance(src.node.inputs, E.KTensor)):
                return None
            virt.append(src.node)
            src, hash_mode = src.node.inputs, L.HASH_FARM
            if src.dtype in ("string", str):
                return None
        name = as_input(src)
        if name is None:
            return None
        maxlen = int(np.prod(src.shape[1:])) if len(src.shape) > 1 else 1
        if (pool == L.POOL_NONE) != (maxlen == 1):
            return None
        return (name, maxlen, pool, hash_mode, emb.input_dim), emb, virt

    pairs = []
    for node in model._order:
        if not isinstance(node.layer, E.Multiply) or calls[id(node.layer)] != 1:
            continue
        ins = E._flatten(node.inputs)
        sides = [lookup(t) for t in ins] if len(ins) == 2 else [None]
        if any(sd is None for sd in sides):
            continue
        out, served, virt, reduce_sum = node.outputs[0], node, [node], False
        if only_use(out):
            nxt = consumers[id(out)][0]
            if isinstance(nxt.layer, E.Lambda) and getattr(nxt.layer, "reduces_last_axis", False):
                served, reduce_sum = nxt, True
            else:
                virt = []
        else:
            virt = []
        pairs.append((sides, served, virt if reduce_sum else [], reduce_sum))
    if not pairs:
        return None
    fields, index = [], {}
    for sides, _, _, _ in pairs:
        for fd, _, _ in sides:
            if fd[0] not in index:
                index[fd[0]] = len(fields)
                fields.append(fd)
    F = len(fields)
    combos = list(itertools.combinations(range(F), 2))
    if not 2 <= F <= MAX_FFM_FIELDS or len(pairs) != len(combos) or len(set(r for *_, r in pairs)) != 1:
        return None
    tables, pair_nodes, virtual, claimed = [None] * (F * F), [], [], set()
    E_ = None
    for (i, j), (sides, served, virt, _) in zip(combos, pairs):
        (fi, ei, vi), (fj, ej, vj) = sides
        if index[fi[0]] != i or index[fj[0]] != j or fi != fields[i] or fj != fields[j]:
            return None
        if E_ is None:
            E_ = ei.output_dim
        if ei.output_dim != E_ or ej.output_dim != E_ or not 1 <= E_ <= MAX_FFM_DIM:
            return None
        tables[i * F + j], tables[j * F + i] = ei, ej
        pair_nodes.append(served)
        virtual.extend(vi + vj + virt)
        claimed.update(id(n) for n in vi + vj if isinstance(n.layer, Embedding))
    if len(set(id(t) for t in tables if t is not None)) != F * (F - 1):
        return None
    return FieldAwarePlan(fields, tables, E_, pairs[0][3], pair_nodes, virtual, claimed)


# ================================================================================================
# Feeder: host arrays -> few packed, pinned H2D copies -> Vars
# ================================================================================================
def slice_inputs(x, sl):
    if isinstance(x, dict):
        return {k: _take(v, sl) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_take(v, sl) for v in x]
    return _take(x, sl)


def _take(v, sl):
    if hasattr(v, "iloc"):
        return v.iloc[sl]
    return v[sl]


class Feeder(object):
    """Packs the per-feature host arrays of one batch into at most three pinned staging buffers
    (int32 ids, int64 ids, fp32 dense/weights) so a step costs <= 3 H2D copies, and exposes every
    model input as a column window of those packs."""

    def __init__(self, model):
        self.model = model
        self.names = list(model.input_names)
        self.specs = {t.name: t for t in model.inputs}
        self.host_hash = {}
        for s in model.planner.slots:
            if s.hash[1] is not None:
                self.host_hash[s.input_name] = s.hash[1]
        self._meta = {}
        for name, spec in self.specs.items():
            tail = tuple(int(d) for d in spec.shape[1:])
            width = int(np.prod(tail)) if tail else 1
            self._meta[name] = (width, spec.dtype in ("float32", "float64", "float16"), spec.dtype == "int64", tail)
        self._pinned = {}
        self._carrays = {}
        self._plan = None
        self._views = {}
        self._copied_ev = {}
        self._consumed_ev = {}
        self.h2d_bytes = 0

    def _as_dict(self, x):
        if isinstance(x, dict):
            return x
        if isinstance(x, (list, tuple)):
            if len(x) != len(self.names):
                raise ValueError("model expects %d inputs %s, got %d arrays" % (len(self.names), self.names, len(x)))
            return dict(zip(self.names, x))
        if len(self.names) == 1:
            return {self.names[0]: x}
        raise ValueError("model inputs must be a dict or a list ordered like get_feature_names()")

    _RING = 3

    # Staging ring.  One feed() + labels() pair uses ONE slot: a pinned host buffer and a persistent device
    # buffer per dtype group.  Persistent device addresses are what lets the training step be replayed as a
    # CUDA graph (engine.Model._loss_step keys its graphs on them).  Two guards per slot:
    #   copied[slot]   - recorded after the H2D copies; the host waits on it before overwriting the pinned side
    #   consumed[slot] - recorded by the model on the compute stream after the step that read the device side;
    #                    the staging stream waits on it before the next H2D into that slot
    def _next_slot(self):
        self.slot = (getattr(self, "slot", -1) + 1) % self._RING
        ev = self._copied_ev.get(self.slot)
        if ev is not None:
            ev.synchronize()
        ev = self._consumed_ev.get(self.slot)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)
        return self.slot

    def consumed(self, slot):
        """The kernels reading slot `slot` have been enqueued on the current stream."""
        ev = self._consumed_ev.get(slot)
        if ev is None:
            ev = self._consumed_ev[slot] = torch.cuda.Event()
        ev.record()

    def _stage(self, key, shape, dtype):
        """(pinned host view, device view) of the current slot for dtype group `key`."""
        n = 1
        for d in shape:
            n *= int(d)
        bufs = self._pinned.setdefault((key, self.slot), [None, None])
        if bufs[0] is None or bufs[0].numel() < n:
            host = torch.empty(max(n, 1), dtype=dtype)
            try:
                host = host.pin_memory()
            except Exception:
                pass
            bufs[0] = host
            bufs[1] = torch.empty(max(n, 1), dtype=dtype, device=E.device())
            self._views.clear()          # cached per-slot views point at the replaced buffer
        return bufs[0][:n].reshape(shape), bufs[1][:n].reshape(shape)

    def _fill(self, sn, items, b):
        """Copy every input's [b, w] block into the flat pinned buffer: one b2ctr_host_pack call (persistent
        native thread pool, no GIL) - a single core moves ~6 GB/s, which would otherwise cap the input
        pipeline at ~1.7 ms per 10 MB batch, above the ~1.3 ms training step it feeds."""
        n = len(items)
        keep = []
        src = (C.c_void_p * n)()
        nbytes = (C.c_int64 * n)()
        offs = (C.c_int64 * n)()
        off = 0
        isz = sn.itemsize
        for i, (name, a, w) in enumerate(items):
            if not (a.flags.c_contiguous and a.dtype == sn.dtype):
                a = np.ascontiguousarray(a, dtype=sn.dtype)
                keep.append(a)
            src[i] = a.__array_interface__["data"][0]
            nbytes[i] = b * w * isz
            offs[i] = off * isz
            off += b * w
        L.check(L.lib().b2ctr_host_pack(src, nbytes, offs, n, C.c_void_p(sn.ctypes.data), _pack_threads()), "host_pack")

    def _upload(self, host, dev):
        dev.copy_(host, non_blocking=True)
        ev = self._copied_ev.get(self.slot)
        if ev is None:
            ev = self._copied_ev[self.slot] = torch.cuda.Event()
        ev.record()
        self.h2d_bytes += host.numel() * host.element_size()
        return dev

    # ---- steady-state path -------------------------------------------------------------------------------
    # fit() feeds thousands of batches of identical structure (one contiguous numpy array per feature, fixed
    # dtypes).  After a batch went through the general path below, its structure is remembered; the next batches
    # only have their array pointers collected (~2 us per input) before the native pack + the H2D copies: the
    # per-step Python cost of the input pipeline must stay well under the ~1.2 ms training step it feeds.
    def _feed_fast(self, xd):
        plan = getattr(self, "_plan", None)
        if plan is None:
            return None
        b = -1
        ptrs = {}
        for key, np_dt, items, _ in plan:
            col = []
            for name, w in items:
                a = xd.get(name)
                if type(a) is not np.ndarray or a.dtype != np_dt or not a.flags.c_contiguous:
                    return None
                if b < 0:
                    b = a.shape[0]
                if a.shape[0] != b or not ((a.ndim == 1 and w == 1) or (a.ndim == 2 and a.shape[1] == w)):
                    return None
                col.append(a.__array_interface__["data"][0])
            ptrs[key] = col
        slot = (getattr(self, "slot", -1) + 1) % self._RING
        for key, np_dt, items, names in plan:          # every view of the slot this batch will land in must exist
            if (slot, key, b, names) not in self._views:
                return None
        self._next_slot()
        feed = {}
        th_dt = {"i32": torch.int32, "i64": torch.int64, "f32": torch.float32}
        for key, np_dt, items, names in plan:
            total = sum(w for _, w in items)
            stage, dbuf = self._stage(key, (b * total,), th_dt[key])
            ck = (key, b)
            arrs = self._carrays.get(ck)
            if arrs is None:
                n = len(items)
                src, nbytes, offs = (C.c_void_p * n)(), (C.c_int64 * n)(), (C.c_int64 * n)()
                off, isz = 0, np.dtype(np_dt).itemsize
                for i, (_, w) in enumerate(items):
                    nbytes[i], offs[i] = b * w * isz, off * isz
                    off += b * w
                arrs = self._carrays[ck] = (src, nbytes, offs, n)
            src, nbytes, offs, n = arrs
            for i, pv in enumerate(ptrs[key]):
                src[i] = pv
            L.check(L.lib().b2ctr_host_pack(src, nbytes, offs, n, C.c_void_p(stage.data_ptr()), _pack_threads()),
                    "host_pack")
            pack = self._upload(stage, dbuf)
            cached = self._views[(self.slot, key, b, names)]
            if key == "f32":
                if len(items) > 1:
                    _, pbuf = self._stage("f32pack", (b, total), torch.float32)
                    K.pack_rows(pack, [w for _, w in items], b, out=pbuf)
                for v in cached.values():          # per-step state of a reused Var
                    v.grad = None
                    v.planes = None
            feed.update(cached)
        return feed

    def feed(self, x, batch_slice=None):
        xd = self._as_dict(x)
        fast = self._feed_fast(xd)
        if fast is not None:
            return fast
        self._next_slot()
        groups = {"i32": [], "i64": [], "f32": []}
        arrays = {}
        meta = self._meta
        for name in self.names:
            if name not in xd:
                raise ValueError("missing model input %r" % name)
            a = xd[name]
            width, is_float, want_i64, shape_tail = meta[name]
            if type(a) is not np.ndarray:
                if isinstance(a, torch.Tensor) and a.is_cuda:
                    arrays[name] = ("dev", a)
                    continue
                a = np.asarray(a.values if hasattr(a, "values") else a)
            if name in self.host_hash:
                a = host_hash(a, self.host_hash[name])
            kind = a.dtype.kind
            if kind in "USO":
                raise ValueError("input %r holds strings: declare the SparseFeat with use_hash=True" % name)
            # hot path (fit over per-feature 1-D columns): no reshape, _fill only needs pointer + contiguity
            if not (a.ndim == 1 and width == 1) and (a.ndim != 2 or a.shape[1] != width):
                a = a.reshape(a.shape[0], -1)
                if a.shape[1] != width:
                    raise ValueError("input %r: expected %d values per sample, got %s" % (name, width, a.shape))
            if is_float:
                groups["f32"].append((name, a, width))
            elif a.dtype == np.int64 and (want_i64 or a.size and
                                          (a.max(initial=0) > 2 ** 31 - 1 or a.min(initial=0) < -2 ** 31)):
                groups["i64"].append((name, a, width))
            else:
                groups["i32"].append((name, a, width))
        feed = {}
        np_dt = {"i32": np.int32, "i64": np.int64, "f32": np.float32}
        th_dt = {"i32": torch.int32, "i64": torch.int64, "f32": torch.float32}
        for key, items in groups.items():
            if not items:
                continue
            b = items[0][1].shape[0]
            total = sum(w for _, _, w in items)
            # the device side of a ring slot is persistent, so the per-input views (engine Vars) of a slot
            # are built once and reused for every batch that lands in it
            vkey = (self.slot, key, b, tuple(name for name, _, _ in items))
            cached = self._views.get(vkey)
            stage, dbuf = self._stage(key, (b * total,), th_dt[key])
            self._fill(stage.numpy(), items, b)
            pack = self._upload(stage, dbuf)
            if key != "f32":
                # ids: one flat staging buffer of per-input contiguous blocks (a plain memcpy per input on
                # the host, one H2D for all); the gather kernels take a pointer + stride per feature
                if cached is None:
                    cached = {}
                    off = 0
                    for name, a, w in items:
                        shape = (b,) + self._meta[name][3]
                        v = E.Var(pack[off:off + b * w].reshape(shape))
                        v.name = name
                        cached[name] = v
                        off += b * w
                    self._views[vkey] = cached
                feed.update(cached)
                continue
            # floats: contiguous per-input blocks on the host (plain memcpy), one H2D, then a device kernel
            # builds the row-major [B, total] dense pack (a strided host-side pack costs ~2 ms at B = 65536)
            flat = pack
            if len(items) > 64:
                raise ValueError("more than 64 dense inputs are not supported")
            if len(items) > 1:
                _, pbuf = self._stage("f32pack", (b, total), torch.float32)
                pack = K.pack_rows(flat, [w for _, _, w in items], b, out=pbuf)
            else:
                pack = flat.reshape(b, total)
            if cached is None:
                cached = {}
                base = E.Var(pack, name="__dense_pack__")
                cached["__dense_pack__"] = base
                col = 0
                for name, a, w in items:
                    shape = (b,) + self._meta[name][3]
                    view = pack[:, col:col + w]
                    v = E.Var(view.as_strided(shape, (pack.stride(0),) + _dense_strides(shape[1:]),
                                              pack.storage_offset() + col),
                              base=base, col0=col, ncols=w)
                    v.name = name
                    cached[name] = v
                    col += w
                self._views[vkey] = cached
            else:
                for v in cached.values():          # per-step state of a reused Var
                    v.grad = None
                    v.planes = None
            feed.update(cached)
        # remember the structure of an all-host batch for the steady-state path
        if not arrays and not self.host_hash:
            plan = []
            for key, items in groups.items():
                if items and all(type(a) is np.ndarray and a.dtype == np_dt[key] and a.flags.c_contiguous
                                 for _, a, _ in items):
                    plan.append((key, np.dtype(np_dt[key]), [(name, w) for name, _, w in items],
                                 tuple(name for name, _, _ in items)))
                elif items:
                    plan = None
                    break
            self._plan = plan or None
        # device-resident inputs: float columns that are views of one [B, nd] buffer form a dense pack
        packs = {}
        for name, (_, a) in arrays.items():
            if (a.dtype == torch.float32 and a.dim() == 2 and a.stride(1) == 1 and a.shape[0] > 1
                    and "__dense_pack__" not in feed):
                packs.setdefault((a.untyped_storage().data_ptr(), a.stride(0)), []).append((name, a))
        done = set()
        for (_, ld), items in packs.items():
            lo = min(a.storage_offset() for _, a in items)
            if len(items) < 2 or any(a.storage_offset() - lo + a.shape[1] > ld for _, a in items):
                continue
            first = items[0][1]
            base_t = first.as_strided((first.shape[0], ld), (ld, 1), lo)
            base = E.Var(base_t, name="__dense_pack__")
            feed["__dense_pack__"] = base
            for name, a in items:
                v = E.Var(a, base=base, col0=a.storage_offset() - lo, ncols=a.shape[1])
                v.name = name
                feed[name] = v
                done.add(name)
            break
        for name, (_, a) in arrays.items():
            if name not in done:
                feed[name] = E.Var(a)
        return feed

    def labels(self, y):
        if isinstance(y, torch.Tensor) and y.is_cuda:
            return y.reshape(-1).float()
        a = np.asarray(y, dtype=np.float32).reshape(-1)
        if not hasattr(self, "slot"):
            self._next_slot()
        stage, dbuf = self._stage("labels", (a.shape[0],), torch.float32)
        stage.numpy()[:] = a
        return self._upload(stage, dbuf)


_PACK_THREADS = None


def _pack_threads():
    """Size of the native staging pool: the cores THIS process may use (its affinity mask, shared between the
    ranks of the node under torchrun), leaving room for the Python threads; between 1 and 8."""
    global _PACK_THREADS
    if _PACK_THREADS is None:
        import os
        try:
            avail = len(os.sched_getaffinity(0))
        except AttributeError:
            avail = os.cpu_count() or 1
        local = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))
        _PACK_THREADS = max(1, min(8, (avail // local - 2) // 2))
    return _PACK_THREADS


def _dense_strides(shape):
    out, acc = [], 1
    for s in reversed(shape):
        out.append(acc)
        acc *= s
    return tuple(reversed(out))


def host_hash(a, hash_layer):
    """Host-side Hash for string ids / vocabulary files (deepctr/layers/utils.py:89-112): strings never
    reach the device; integers are hashed on the device by the gather kernel itself."""
    from .layers.utils import host_hash_array
    return host_hash_array(a, hash_layer.num_buckets, hash_layer.mask_zero, hash_layer.vocabulary_path,
                           hash_layer.default_value)
