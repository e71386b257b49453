"""DeepModel -- the reference's model object (deeptables/models/deepmodel.py) on the H100 engine.

Same constructor and public methods (fit / predict / evaluate / apply / save / release, attributes
``model``, ``model_desc``, ``config``), same graph (``__build_model``, reference deepmodel.py:259-317:
inputs -> MultiColumnEmbedding -> flatten/concat + BatchNormalization -> net builders -> stacking ->
``task_output``), same training contract (Adam(1e-3) + BCE/MSE/CCE when ``optimizer``/``loss`` are
'auto', reference deepmodel.py:319-346; SGD / RMSprop / Adagrad / Adam at other hyperparameters through
``optimizers.py``; ``steps_per_epoch`` / ``validation_steps`` arithmetic,
reference deepmodel.py:76-83).  The numerics run in hand-written sm_90a kernels behind the C ABI;
torch supplies device memory and the autograd tape only.

Multi-GPU: one process per GPU under ``torch.distributed`` (NCCL).  Each rank trains on its shard
of the global batch; dense-weight gradients are all-reduced in one bucket and the embedding
gradient is exchanged once per step (reference: tf.distribute.MirroredStrategy, deepmodel.py:88-103).
"""
import collections
import contextlib
import math
import os
import pickle
from collections import OrderedDict
from typing import Union

import numpy as np
import torch

from . import consts, deepnets, dp, engine as E, layers as L, optimizers as O, regularizers as R
from ._native import ptr, check, stream_ptr
from . import _native as N


class _Scope:
    """Active-forward-pass state: parameter store + Keras-style layer naming."""

    def __init__(self, device, seed=None):
        self.device = torch.device(device)
        self.generator = torch.Generator(device=self.device)
        self.generator.manual_seed(int(seed) if seed is not None else int.from_bytes(os.urandom(4), 'little'))
        self.params = OrderedDict()
        self.regularizers = OrderedDict()  # parameter name -> regularizers.RegSpec (Keras add_weight(regularizer=))
        self.reg_segments = []             # after freeze(): (offset, numel, l1, l2) of each regularized parameter
        self.stacked = {}                  # key of a param_stack() tensor -> the reference names of its slices
        self.buffers = OrderedDict()
        self.training = False
        self.frozen = False
        self.capture = None                # set of layer names whose outputs `apply` wants
        self.outputs = {}
        self.anchor = torch.zeros(1, dtype=torch.float32, device=self.device, requires_grad=True)
        self._counters = {}
        self._indices = {}
        self._prefix = []
        self._seed_counter = 0

    def next_seed(self):
        """Fresh dropout seed per call site and per pass (drawn from the model's generator stream)."""
        self._seed_counter += 1
        return (int(self.generator.initial_seed()) * 1000003 + self._seed_counter) & 0xFFFFFFFFFFFF

    def _begin_pass(self):
        self._counters = {}
        self._prefix = []
        self.outputs = {}
        self._indices = {}

    def next_index(self, counter_name):
        """utils/counter.py:next_num scoped to one forward pass of this model (index begins from 0)."""
        n = self._indices.get(counter_name, -1) + 1
        self._indices[counter_name] = n
        return n

    def full_name(self, given, base):
        prefix = '/'.join(self._prefix)
        if given is None:
            key = (prefix, base)
            n = self._counters.get(key, 0)
            self._counters[key] = n + 1
            given = base if n == 0 else f'{base}_{n}'
        return f'{prefix}/{given}' if prefix else given

    @contextlib.contextmanager
    def name_prefix(self, prefix):
        self._prefix.append(prefix.split('/')[-1] if self._prefix else prefix)
        try:
            yield
        finally:
            self._prefix.pop()

    def record_output(self, name, out):
        if self.capture is not None and name in self.capture:
            self.outputs[name] = out

    def param(self, name, shape, init, regularizer=None):
        p = self.params.get(name)
        if p is None:
            if self.frozen:
                raise RuntimeError(f'parameter {name!r} requested after the model was built')
            p = L.init_tensor(shape, init, self.device, self.generator).requires_grad_(True)
            self.params[name] = p
            spec = R.resolve(regularizer)
            if spec is not None:
                self.regularizers[name] = spec
        elif tuple(p.shape) != tuple(int(s) for s in shape):
            raise ValueError(f'parameter {name!r} has shape {tuple(p.shape)}, layer asked for {tuple(shape)}')
        return p

    def param_stack(self, names, shape, init):
        """One leaf tensor [len(names), *shape] for a family of same-shaped reference weights that a kernel wants contiguous
        (BilinearInteraction's per-pair matrices, layers.py:343-356).  ``state_dict`` exposes the slices under the reference's
        individual names; the optimiser sees one tensor."""
        key = names[0] + '[*]'
        p = self.params.get(key)
        if p is None:
            if self.frozen:
                raise RuntimeError(f'parameter {key!r} requested after the model was built')
            p = torch.stack([L.init_tensor(shape, init, self.device, self.generator) for _ in names]).requires_grad_(True)
            self.params[key] = p
            self.stacked[key] = list(names)
        elif tuple(p.shape) != (len(names),) + tuple(int(s) for s in shape):
            raise ValueError(f'parameter {key!r} has shape {tuple(p.shape)}, layer asked for {(len(names),) + tuple(shape)}')
        return p

    def buffer(self, name, shape, value):
        b = self.buffers.get(name)
        if b is None:
            if self.frozen:
                raise RuntimeError(f'buffer {name!r} requested after the model was built')
            b = torch.full(tuple(int(s) for s in shape), float(value), dtype=torch.float32, device=self.device)
            self.buffers[name] = b
        return b

    def flatten_embeddings(self, emb_list):
        mat = emb_list.block.materialize()
        return mat.reshape(mat.shape[0], -1)

    # ---- flat storage so Adam and the DP all-reduce are one launch / one bucket -------------------
    def freeze(self, slot_inits=None):
        """slot_inits: initial values of the SGD / RMSprop / Adagrad state slots (optimizers.slot_inits); None = Adam's
        flat_m, flat_v."""
        names = list(self.params)
        sizes = [self.params[n].numel() for n in names]
        total = sum(sizes)
        self.flat_p = torch.empty(total, dtype=torch.float32, device=self.device)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=self.device)
        if slot_inits is None:
            self.flat_m = torch.zeros(total, dtype=torch.float32, device=self.device)
            self.flat_v = torch.zeros(total, dtype=torch.float32, device=self.device)
        else:
            self.flat_slots = [None if s is None else torch.full((total,), s, dtype=torch.float32, device=self.device)
                               for s in slot_inits]
        off = 0
        self.reg_segments = []
        for n, sz in zip(names, sizes):
            old = self.params[n]
            view = self.flat_p[off:off + sz].view(old.shape)
            view.copy_(old.detach())
            p = view.detach().requires_grad_(True)
            p.grad = self.flat_g[off:off + sz].view(old.shape)
            self.params[n] = p
            if n in self.regularizers:
                self.reg_segments.append((off, sz, self.regularizers[n].l1, self.regularizers[n].l2))
            off += sz
        self.frozen = True


class _HostBatches:
    """Input pipeline for data sets that should not (or cannot) live in HBM: the encoded columns stay in PINNED host
    memory, a batch is gathered on the host into one of two pinned staging buffers and copied on a side stream while the
    previous step computes (double buffering).  Replaces the reference's ``tf.data`` path (utils/dataset_generator.py:36-72,
    241-257: ``from_tensor_slices`` over ``.tolist()`` of the whole frame, shuffle buffer = N, batch, prefetch); the default
    path keeps the whole encoded data set in HBM (160 B/row at the Criteo shape: 10 M rows = 1.6 GB of 180 GB)."""

    def __init__(self, device, *tensors):
        self.device = device
        self.src = [None if t is None else t.contiguous().pin_memory() for t in tensors]
        self.stream = torch.cuda.Stream(device=device)
        self.slots = [None, None]
        self.k = 0

    def prefetch(self, sel):
        """Start the gather + copy of the rows ``sel`` (CPU int64 tensor); returns a handle for ``get``."""
        slot = self.k & 1
        self.k += 1
        n = sel.numel()
        if self.slots[slot] is None or self.slots[slot][0] < n:
            self.slots[slot] = (n, [None if t is None else torch.empty((n,) + tuple(t.shape[1:]), dtype=t.dtype).pin_memory()
                                    for t in self.src], None)
        _, stage, prev = self.slots[slot]
        if prev is not None:
            prev.synchronize()                    # the copy that last used this staging buffer has finished
        outs = []
        with torch.cuda.stream(self.stream):
            for t, st in zip(self.src, stage):
                if t is None:
                    outs.append(None)
                    continue
                torch.index_select(t, 0, sel, out=st[:n])
                outs.append(st[:n].to(self.device, non_blocking=True))
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.slots[slot] = (self.slots[slot][0], stage, ev)
        return outs, ev

    @staticmethod
    def get(handle):
        outs, ev = handle
        torch.cuda.current_stream().wait_event(ev)
        for o in outs:
            if o is not None:
                o.record_stream(torch.cuda.current_stream())
        return outs


class KerasLikeModel:
    """What ``DeepModel.model`` holds: the built network (parameters + forward)."""

    def __init__(self, owner):
        self._owner = owner

    @property
    def weights(self):
        return self._owner.state_dict()

    def count_params(self):
        return sum(int(np.prod(v.shape)) for v in self._owner.state_dict().values())


class History:
    def __init__(self):
        self.history = {}
        self.epoch = []


class DeepModel:
    """Class for neural network models (reference deepmodel.py:26-58)."""

    def __init__(self, task, num_classes, config, categorical_columns, continuous_columns, model_file=None,
                 var_categorical_len_columns=None, custom_objects=None, device=None, seed=None):
        self.model_desc = ModelDesc()
        self.categorical_columns = list(categorical_columns or [])
        self.continuous_columns = list(continuous_columns or [])
        self.var_len_categorical_columns = var_categorical_len_columns
        if var_categorical_len_columns:
            raise NotImplementedError('var-len categorical columns are outside the hot path (SURVEY.md 8f)')
        self.task = task
        self.num_classes = num_classes
        self.config = config
        self.model_file = model_file
        self.model = None
        self.stop_training = False
        self._seed = seed
        self._step = 0
        if not torch.cuda.is_available():
            raise RuntimeError('deeptables_b200 needs a CUDA device (H100, sm_90a); there is no CPU path')
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self._dist = torch.distributed.is_available() and torch.distributed.is_initialized() and \
            torch.distributed.get_world_size() > 1
        self.world_size = torch.distributed.get_world_size() if self._dist else 1
        self.rank = torch.distributed.get_rank() if self._dist else 0
        self.emb_dims = [int(c.embeddings_output_dim) for c in self.categorical_columns]
        self.n_fields = len(self.categorical_columns)
        self.emb_dim = max(self.emb_dims) if self.emb_dims else 0     # stored row width of the embedding table
        self.n_cont = sum(c.input_dim for c in self.continuous_columns)
        self._scope = None
        self.table = None
        self._loss_acc = None
        self._focal = None                  # (gamma, alpha) when ModelConfig.loss is one of the focal losses
        self._alpha = None
        self._step_dev = None              # optimiser step counter in device memory (CUDA-graph replay of the train step)
        self._opt = None                   # optimizers.OptimizerSpec resolved from ModelConfig.optimizer
        self._opt_native = None            # its dtb_optim_params (SGD / RMSprop / Adagrad)
        self._emb_reg = None               # regularizers.RegSpec of ModelConfig.embeddings_regularizer
        self._graphs = {}
        self._graph_failed = False
        if model_file is not None:
            self._load_model(model_file)

    # ------------------------------------------------------------------------------------------
    # build  (reference deepmodel.py:259-317)
    # ------------------------------------------------------------------------------------------
    def _build_model(self):
        cfg = self.config
        self._opt = O.resolve(cfg.optimizer)
        self._opt_native = None if self._opt.kind == 'adam' else _native_optim_params(self._opt)
        slot_inits = None if self._opt.kind == 'adam' else O.slot_inits(self._opt)
        self._focal = None
        if isinstance(cfg.loss, L.CategoricalFocalLoss):
            if self.task != consts.TASK_MULTICLASS:
                raise ValueError('CategoricalFocalLoss needs a multiclass task')
            self._focal = (cfg.loss.gamma, cfg.loss.alpha)
        elif isinstance(cfg.loss, L.BinaryFocalLoss):
            if self.task not in (consts.TASK_BINARY, consts.TASK_MULTILABEL):
                raise ValueError('BinaryFocalLoss needs a binary or multilabel task')
            self._focal = (cfg.loss.gamma, cfg.loss.alpha)
        elif cfg.loss != 'auto':
            raise NotImplementedError("loss must be 'auto' or one of layers.BinaryFocalLoss / CategoricalFocalLoss")
        R.reject_activity(cfg.embeddings_activity_regularizer, 'embeddings_activity_regularizer')
        self._emb_reg = R.resolve(cfg.embeddings_regularizer, 'embeddings_regularizer')
        if self.task not in consts.ALL_TASKS:
            raise ValueError(f'Unknown task type:{self.task}')
        if len(set(self.emb_dims)) > 1:
            for net in cfg.nets:
                if isinstance(net, str) and net in deepnets.EQUAL_WIDTH_NETS:
                    raise ValueError(f'{net} concatenates the field embeddings on axis 1 and needs one embedding width '
                                     f'for every categorical column; got widths {self.emb_dims}')
        self._scope = _Scope(self.device, self._seed)
        if self.n_fields:
            self.table = E.EmbeddingTable([c.vocabulary_size for c in self.categorical_columns], self.emb_dim,
                                          self.device, cfg.embeddings_initializer, self._scope.generator,
                                          field_dims=self.emb_dims)
            self.table.slot_inits = slot_inits
            # a regularized table takes a non-zero gradient in every row every step: no exact-lazy row form
            self.table.lazy_active = self.table.lazy_adam and self._emb_reg is None
        self.model_desc = ModelDesc()
        if self.n_fields:
            self.model_desc.add_input('all_categorical_vars', self.n_fields)
            self.model_desc.set_embeddings([c.vocabulary_size for c in self.categorical_columns],
                                           list(self.emb_dims), cfg.embedding_dropout)
            if self.table.ragged:
                self.model_desc.set_embedding_storage(self.table.dim, self.table.padding_share())
            if self._emb_reg is not None:
                self.model_desc.embeddings += f'\nregularizer: {self._emb_reg}'
        for c in self.continuous_columns:
            self.model_desc.add_input(c.name, c.input_dim)
        self.model_desc.set_dense(cfg.dense_dropout, False)
        self.model_desc.nets = cfg.nets
        self.model_desc.stacking = cfg.stacking_op
        self.model_desc.optimizer = self._opt.keras_name
        self.model_desc.loss = {consts.TASK_BINARY: 'binary_crossentropy', consts.TASK_MULTILABEL:
                                'binary_crossentropy', consts.TASK_REGRESSION: 'mse'}.get(
            self.task, 'binary_crossentropy' if self.num_classes == 2 else 'categorical_crossentropy')
        if self._focal is not None:
            self.model_desc.loss = 'focal_loss'
        # dry run on two rows materialises every weight (define-by-run build)
        cat = torch.zeros(2, self.n_fields, dtype=torch.int32, device=self.device) if self.n_fields else None
        cont = torch.zeros(2, self.n_cont, dtype=torch.float32, device=self.device) if self.n_cont else None
        with torch.no_grad():
            self._forward(cat, cont, training=False, describe=True)
        self._scope.freeze(slot_inits)
        self.model_desc.regularizers = [f'{k}: {v}' for k, v in self._scope.regularizers.items()]
        dp.broadcast_parameters([self._scope.flat_p, self.table.weight if self.table is not None else None])
        self._loss_acc = torch.zeros(1, dtype=torch.float64, device=self.device)
        self.model = KerasLikeModel(self)
        return self.model

    def _forward(self, cat, cont, training, describe=False, capture=None):
        """inputs -> embeddings -> nets -> stacking -> task_output pre-activation z."""
        cfg = self.config
        scope = self._scope
        scope.training = training
        scope.capture = capture
        desc = self.model_desc if describe else _NullDesc()
        with L.scope_guard(scope):
            embeddings = []
            block = None
            if self.n_fields and self.table.ragged:
                # fields of different widths: one flat (B, sum D_i) gather feeds flatten_embeddings, the list items
                # (B, 1, D_i) and, with dropout, concat_embedding_dense, so they all share one mask
                block = E.RaggedFieldBlock(cat, self.table)
                if cfg.embedding_dropout > 0 and training:
                    dropped = E.DropoutFn.apply(block.materialize(), cfg.embedding_dropout, scope.next_seed())
                    block = E.RaggedFieldBlock(cat, self.table, flat=dropped)
                embeddings = E.RaggedEmbeddingList(block)
            elif self.n_fields:
                block = E.FieldBlock(cat, self.table)
                if cfg.embedding_dropout > 0 and training:
                    # SpatialDropout1D per field (reference layers.py:878-901): the mask must be shared by
                    # every consumer, so this (non-default-for-benchmarks) mode materialises the dropped
                    # block once and feeds the same fused kernels through the tensor-backed table facade
                    dropped = E.DropoutFn.apply(block.materialize(), cfg.embedding_dropout, scope.next_seed())
                    block = E.FieldBlock.from_tensor(dropped)
                embeddings = E.EmbeddingList(block)
            dense_layer = cont
            if dense_layer is not None and cfg.dense_dropout > 0:
                dense_layer = L.Dropout(cfg.dense_dropout, name='dropout_dense_input')(dense_layer)
            flatten_emb_layer = _LazyFlat(scope, embeddings) if self.n_fields else None
            if capture and 'flatten_embeddings' in capture and flatten_emb_layer is not None:
                flatten_emb_layer._get()
            # cin_nets is evaluated before anything else touches the embedding table: autograd runs nodes
            # in reverse creation order, so its backward comes last and its weight-gradient kernels can hide
            # the data-parallel exchange of the table gradient (engine._table_grad_done).  It does not use
            # concat_emb_dense (reference deepnets.py:69-81).
            results = {}
            if 'cin_nets' in cfg.nets and self.n_fields:
                results['cin_nets'] = deepnets.get('cin_nets')(embeddings, flatten_emb_layer, dense_layer, None, cfg, desc)
            # concat_embedding_dense + bn_concat_emb_dense (reference deepmodel.py:348-361)
            if isinstance(block, E.RaggedFieldBlock):
                if block._mat is None:
                    x = E.RaggedConcatEmbDenseFn.apply(block.table.anchor, dense_layer, block)
                else:
                    x = block._mat if dense_layer is None else torch.cat([block._mat, dense_layer], dim=1)
            elif block is not None:
                x = E.ConcatEmbDenseFn.apply(block.table.anchor, dense_layer, block)
            elif dense_layer is not None:
                x = dense_layer
            else:
                raise ValueError('No input layer exists.')
            scope.record_output('concat_embedding_dense', x)
            concat_emb_dense = L.BatchNormalization(name='bn_concat_emb_dense')(x)
            if describe:
                desc.set_concat_embed_dense(tuple(concat_emb_dense.shape))
            for net in cfg.nets:
                if net in results:
                    continue
                fn = deepnets.get(net)
                results[net] = fn(embeddings if self.n_fields else [], flatten_emb_layer, dense_layer,
                                  concat_emb_dense, cfg, desc)
            outs = OrderedDict((net, results[net]) for net in cfg.nets if results[net] is not None)
            if len(outs) > 1:
                logits = []
                for name, out in outs.items():
                    if out.dim() > 2:
                        out = L.Flatten(name=f'flatten_{name}_out')(out)
                    if out.shape[-1] > 1:
                        out = L.Dense(1, use_bias=False, activation=None, name=f'dense_logit_{name}')(out)
                    logits.append(out)
                if cfg.stacking_op == consts.STACKING_OP_ADD:
                    x = L.Add(name='add_logits')(logits)
                elif cfg.stacking_op == consts.STACKING_OP_CONCAT:
                    x = L.Concatenate(name='concat_logits')(logits)
                else:
                    raise ValueError(f'Unsupported stacking_op:{cfg.stacking_op}.')
            elif len(outs) == 1:
                name, out = next(iter(outs.items()))
                if out.dim() > 2:
                    out = L.Flatten(name=f'flatten_{name}_out')(out)
                x = out
            else:
                raise ValueError(f'Unexpected logit output.{outs}')
            out_dim = self._output_dim()
            z = L.Dense(out_dim, activation=None, name='task_output', use_bias=cfg.output_use_bias)(x)
            if describe:
                act = {consts.TASK_BINARY: 'sigmoid', consts.TASK_MULTILABEL: 'sigmoid',
                       consts.TASK_REGRESSION: None, consts.TASK_MULTICLASS: 'softmax'}[self.task]
                desc.set_output(act, tuple(z.shape), cfg.output_use_bias)
        return z

    def _output_dim(self):
        if self.task in (consts.TASK_BINARY, consts.TASK_REGRESSION):
            return 1
        if not self.num_classes:
            raise ValueError('"config.multiclass_classes" value must be provided for multi-class task.')
        return self.num_classes

    # ------------------------------------------------------------------------------------------
    # one optimiser step / one scoring pass on device-resident batches
    # ------------------------------------------------------------------------------------------
    def _alpha_table(self, upto):
        if self._alpha is None or self._alpha.numel() <= upto:
            n = max(4096, 2 * (upto + 1))
            o = self._opt
            vals = [0.0] + [E.adam_alpha(s, o.learning_rate, o.beta_1, o.beta_2) for s in range(1, n)]
            self._alpha = torch.tensor(vals, dtype=torch.float32, device=self.device)
        return self._alpha

    def _select_table_optimizer(self, n_refs):
        """Row-wise exact-lazy Adam visits every touched row (the UNION over ranks in data parallel);
        the dense sweep reads the whole table.  Both give identical bits, so pick the cheaper one:
        lazy while the references per step are a small fraction of the table, dense beyond that
        (large world sizes).  Switching flushes / re-stamps ``last_step`` so the trajectory is unchanged."""
        t = self.table
        want_lazy = bool(t.lazy_adam and n_refs * 6 <= t.total_rows)
        if getattr(self, '_table_mode_override', None) is not None:       # test hook
            want_lazy = bool(t.lazy_adam and self._table_mode_override == 'lazy')
        want_lazy = want_lazy and self._emb_reg is None
        if want_lazy == t.lazy_active:
            return
        if t.lazy_active:                       # lazy -> dense: bring every row up to date first
            t.lazy_active = True
            self.flush_optimizer_state()
            t.lazy_active = False
        else:                                   # dense -> lazy: every row is current as of this step
            t.last_step.fill_(self._step)
            t.lazy_active = True

    def _catch_up(self, cat, upto, dev_step=False):
        t = self.table
        if t is None or not t.lazy_active or t.last_step is None:
            return
        o = self._opt
        if o.kind != 'adam':
            s = [ptr(x) for x in t.slots]
            if dev_step:
                check(N.lib.dtb_optim_rows_catchup_dev(ptr(cat), ptr(t.row_offsets), ptr(t.weight), *s, ptr(t.last_step),
                                                       ptr(self._step_dev), self._opt_native, cat.shape[0], t.n_fields,
                                                       t.dim, stream_ptr()), 'optim_rows_catchup_dev')
            elif upto > 0:
                check(N.lib.dtb_optim_rows_catchup(ptr(cat), ptr(t.row_offsets), ptr(t.weight), *s, ptr(t.last_step), upto,
                                                   self._opt_native, cat.shape[0], t.n_fields, t.dim, stream_ptr()),
                      'optim_rows_catchup')
            return
        if dev_step:          # CUDA-graph form: "steps done so far" is read from device memory
            check(N.lib.dtb_adam_rows_catchup_dev(ptr(cat), ptr(t.row_offsets), ptr(t.weight), ptr(t.m), ptr(t.v),
                                                  ptr(t.last_step), ptr(self._alpha), ptr(self._step_dev), o.beta_1,
                                                  o.beta_2, o.epsilon, cat.shape[0], t.n_fields, t.dim, stream_ptr()),
                  'adam_rows_catchup_dev')
            return
        if upto <= 0:
            return
        check(N.lib.dtb_adam_rows_catchup(ptr(cat), ptr(t.row_offsets), ptr(t.weight), ptr(t.m), ptr(t.v),
                                          ptr(t.last_step), ptr(self._alpha_table(upto)), upto, o.beta_1,
                                          o.beta_2, o.epsilon, cat.shape[0], t.n_fields, t.dim, stream_ptr()),
              'adam_rows_catchup')

    def train_step(self, cat, cont, y, sample_weight=None):
        """forward + loss + backward + (DP exchange) + Adam on one device-resident batch.
        Returns the batch predictions; the summed loss accumulates in ``self._loss_acc``.

        Single-GPU steps without dropout or sample weights are captured ONCE per batch shape in a CUDA graph and replayed
        (``DTB_CUDA_GRAPH=0`` disables it): a step is ~90 launches of kernels that take microseconds at small batch sizes
        (DeepFM at 8 192 rows), where the host's launch path -- not the GPU -- would set the pace."""
        if self._graph_eligible(cat, cont, y, sample_weight):
            return self._train_step_graphed(cat, cont, y)
        prob = self._train_step_body(cat, cont, y, sample_weight, dev_step=False)
        self._step += 1
        if self._step_dev is not None:
            self._step_dev.fill_(self._step)
        return prob

    def _train_step_body(self, cat, cont, y, sample_weight, dev_step):
        scope = self._scope
        t = self.table
        if t is not None:
            t.ensure_training_state()
            self._select_table_optimizer(self.world_size * cat.shape[0] * t.n_fields)
            self._catch_up(cat, self._step, dev_step)
        if t is not None:
            t.pending_bwd = 0
            t.on_grad_final = (lambda: self._begin_table_exchange(cat)) if (self._dist and t.lazy_adam) else None
        self._early_exchange = None
        z = self._forward(cat, cont, training=True)
        prob, dz = E.loss_forward_backward(z, y, self.task, sample_weight, True, self._loss_acc, focal=self._focal)
        dp.scale_for_mean(dz)
        z.backward(dz)
        step = self._step + 1
        union_cat = cat
        if self._dist:
            union_cat = self._exchange_gradients(cat)
        rows = y.shape[0]
        self._reg_terms(scope.flat_g, self._loss_acc, rows)    # after the exchange: counted once, on every replica
        o = self._opt
        if o.kind != 'adam':
            self._optim_step(union_cat, step, dev_step, rows)
            if dev_step:
                check(N.lib.dtb_step_increment(ptr(self._step_dev), stream_ptr()), 'step_increment')
            return prob
        if dev_step:
            check(N.lib.dtb_adam_dense_dev(ptr(scope.flat_p), ptr(scope.flat_m), ptr(scope.flat_v), ptr(scope.flat_g),
                                           scope.flat_p.numel(), ptr(self._alpha), ptr(self._step_dev), o.beta_1,
                                           o.beta_2, o.epsilon, 1, stream_ptr()), 'adam_dense_dev')
            if t is not None:
                if t.lazy_active:
                    check(N.lib.dtb_adam_rows_apply_dev(ptr(union_cat), ptr(t.row_offsets), ptr(t.weight), ptr(t.m), ptr(t.v),
                                                        ptr(t.grad), ptr(t.last_step), ptr(self._alpha), ptr(self._step_dev),
                                                        o.beta_1, o.beta_2, o.epsilon, union_cat.shape[0], t.n_fields,
                                                        t.dim, stream_ptr()), 'adam_rows_apply_dev')
                elif self._emb_reg is not None:
                    r = self._emb_reg
                    check(N.lib.dtb_adam_dense_reg_dev(ptr(t.weight), ptr(t.m), ptr(t.v), ptr(t.grad), t.weight.numel(),
                                                       ptr(self._alpha), ptr(self._step_dev), o.beta_1, o.beta_2,
                                                       o.epsilon, 1, r.l1, r.l2, ptr(self._loss_acc), float(rows),
                                                       stream_ptr()), 'adam_dense_reg_dev(table)')
                else:
                    check(N.lib.dtb_adam_dense_dev(ptr(t.weight), ptr(t.m), ptr(t.v), ptr(t.grad), t.weight.numel(),
                                                   ptr(self._alpha), ptr(self._step_dev), o.beta_1, o.beta_2, o.epsilon, 1,
                                                   stream_ptr()), 'adam_dense_dev(table)')
            check(N.lib.dtb_step_increment(ptr(self._step_dev), stream_ptr()), 'step_increment')
            return prob
        alpha = E.adam_alpha(step, o.learning_rate, o.beta_1, o.beta_2)
        check(N.lib.dtb_adam_dense(ptr(scope.flat_p), ptr(scope.flat_m), ptr(scope.flat_v), ptr(scope.flat_g),
                                   scope.flat_p.numel(), alpha, o.beta_1, o.beta_2, o.epsilon, 1,
                                   stream_ptr()), 'adam_dense')
        if t is not None:
            if t.lazy_active:
                a = self._alpha_table(step)
                check(N.lib.dtb_adam_rows_apply(ptr(union_cat), ptr(t.row_offsets), ptr(t.weight), ptr(t.m),
                                                ptr(t.v), ptr(t.grad), ptr(t.last_step), ptr(a), step, o.beta_1,
                                                o.beta_2, o.epsilon, union_cat.shape[0], t.n_fields, t.dim,
                                                stream_ptr()), 'adam_rows_apply')
            elif self._emb_reg is not None:
                r = self._emb_reg
                check(N.lib.dtb_adam_dense_reg(ptr(t.weight), ptr(t.m), ptr(t.v), ptr(t.grad), t.weight.numel(), alpha,
                                               o.beta_1, o.beta_2, o.epsilon, 1, r.l1, r.l2, ptr(self._loss_acc),
                                               float(rows), stream_ptr()), 'adam_dense_reg(table)')
            else:
                check(N.lib.dtb_adam_dense(ptr(t.weight), ptr(t.m), ptr(t.v), ptr(t.grad), t.weight.numel(),
                                           alpha, o.beta_1, o.beta_2, o.epsilon, 1, stream_ptr()),
                      'adam_dense(table)')
        return prob

    def _optim_step(self, union_cat, step, dev_step, rows):
        """SGD / RMSprop / Adagrad step `step`: the dense sweep over the flat parameters, then the table's row-wise
        update (lazy) or dense sweep (with the table's regularization fused in; `rows` scales its loss term).  Only
        the row form needs the step number (to count skipped steps); its CUDA-graph form reads it from device
        memory."""
        scope, t, hp = self._scope, self.table, self._opt_native
        check(N.lib.dtb_optim_dense(ptr(scope.flat_p), ptr(scope.flat_g), *[ptr(x) for x in scope.flat_slots],
                                    scope.flat_p.numel(), hp, 1, stream_ptr()), 'optim_dense')
        if t is None:
            return
        s = [ptr(x) for x in t.slots]
        if self._emb_reg is not None:
            r = self._emb_reg
            check(N.lib.dtb_optim_dense_reg(ptr(t.weight), ptr(t.grad), *s, t.weight.numel(), hp, 1, r.l1, r.l2,
                                            ptr(self._loss_acc), float(rows), stream_ptr()), 'optim_dense_reg(table)')
        elif not t.lazy_active:
            check(N.lib.dtb_optim_dense(ptr(t.weight), ptr(t.grad), *s, t.weight.numel(), hp, 1, stream_ptr()),
                  'optim_dense(table)')
        elif dev_step:
            check(N.lib.dtb_optim_rows_apply_dev(ptr(union_cat), ptr(t.row_offsets), ptr(t.weight), *s, ptr(t.grad),
                                                 ptr(t.last_step), ptr(self._step_dev), hp, union_cat.shape[0], t.n_fields,
                                                 t.dim, stream_ptr()), 'optim_rows_apply_dev')
        else:
            check(N.lib.dtb_optim_rows_apply(ptr(union_cat), ptr(t.row_offsets), ptr(t.weight), *s, ptr(t.grad),
                                             ptr(t.last_step), step, hp, union_cat.shape[0], t.n_fields, t.dim,
                                             stream_ptr()), 'optim_rows_apply')

    def _reg_terms(self, flat_g, loss_acc, loss_scale):
        """Regularized dense weights (Dense kernels): flat_g += their regularization gradient and loss_acc +=
        loss_scale * their term, from the weights before the step.  flat_g None: the loss term only."""
        scope = self._scope
        for off, n, l1, l2 in scope.reg_segments:
            check(N.lib.dtb_reg_grad(ptr(scope.flat_p[off:]), None if flat_g is None else ptr(flat_g[off:]), n, l1, l2,
                                     ptr(loss_acc), float(loss_scale), stream_ptr()), 'reg_grad')

    def _reg_loss(self, loss_acc, loss_scale):
        """loss_acc += loss_scale * the regularization term of every regularized weight at the current weights."""
        self._reg_terms(None, loss_acc, loss_scale)
        if self._emb_reg is not None and self.table is not None:
            r = self._emb_reg
            check(N.lib.dtb_reg_grad(ptr(self.table.weight), None, self.table.weight.numel(), r.l1, r.l2, ptr(loss_acc),
                                     float(loss_scale), stream_ptr()), 'reg_grad(table)')

    # ---- CUDA-graph replay of the train step ---------------------------------------------------------------------------
    def _has_dropout(self):
        cfg = self.config
        if cfg.embedding_dropout or cfg.dense_dropout:
            return True
        if any(float(u[1]) > 0 for u in (cfg.dnn_params or {}).get('hidden_units', ())):
            return True
        return bool((cfg.autoint_params or {}).get('dropout_rate', 0)) and 'autoint_nets' in cfg.nets

    def _graph_eligible(self, cat, cont, y, sample_weight):
        if self._dist or sample_weight is not None or os.environ.get('DTB_CUDA_GRAPH', '1') == '0':
            return False
        if self._graph_failed or self._step < 1:       # the first step runs eagerly (allocations, lazy initialisation)
            return False
        if getattr(self, '_no_graph', None) is None:
            self._no_graph = self._has_dropout() or any(callable(n) for n in self.config.nets)
        return not self._no_graph

    def _train_step_graphed(self, cat, cont, y):
        t = self.table
        key = (None if cat is None else tuple(cat.shape), None if cont is None else tuple(cont.shape), tuple(y.shape),
               None if t is None else t.lazy_active)
        if self._step_dev is None:
            self._step_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
        if self._opt.kind == 'adam' and (self._alpha is None or self._alpha.numel() <= self._step + 2):
            self._graphs.clear()                       # the alpha table moves when it grows: captured pointers are stale
            self._alpha_table(self._step + 200000)
        if t is not None:
            t.ensure_training_state()
            self._select_table_optimizer(cat.shape[0] * t.n_fields)
            key = key[:3] + (t.lazy_active,)
        entry = self._graphs.get(key)
        if entry is None:
            sc = None if cat is None else torch.empty_like(cat)
            sx = None if cont is None else torch.empty_like(cont)
            sy = torch.empty_like(y)
            self._step_dev.fill_(self._step)
            try:
                import gc
                gc.collect()             # no autograd graph of an earlier (eager) step may outlive into the capture
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                l0 = N.lib.dtb_launch_count()
                with torch.cuda.graph(graph):
                    prob = self._train_step_body(sc, sx, sy, None, dev_step=True)
                n_launch = N.lib.dtb_launch_count() - l0          # kernels of this library inside one replay
            except Exception as exc:                       # capture unsupported here: say so once, run eagerly from now on
                self._graph_failed = True
                import warnings
                warnings.warn(f'deeptables_b200: CUDA-graph capture of the train step failed ({type(exc).__name__}: {exc}); '
                              f'continuing with eager launches')
                torch.cuda.synchronize()
                prob = self._train_step_body(cat, cont, y, None, dev_step=False)
                self._step += 1
                return prob
            N.lib.dtb_launch_count_add(-n_launch)                # counted at capture, not executed yet
            entry = self._graphs[key] = (graph, sc, sx, sy, prob, n_launch)
        graph, sc, sx, sy, prob, n_launch = entry
        if sc is not None:
            sc.copy_(cat)
        if sx is not None:
            sx.copy_(cont)
        sy.copy_(y)
        graph.replay()
        N.lib.dtb_launch_count_add(n_launch)
        self._step += 1
        return prob

    def _row_exchange_fns(self, cat):
        t = self.table
        step = self._step + 1
        if t.claim is None:
            t.claim = torch.zeros(t.total_rows, dtype=torch.int32, device=self.device)

        def pack():
            packed = torch.empty(cat.shape[0], t.n_fields, t.dim, dtype=torch.float32, device=self.device)
            check(N.lib.dtb_grad_rows_pack(ptr(cat), ptr(t.row_offsets), ptr(t.grad), ptr(t.claim), ptr(packed),
                                           step, cat.shape[0], t.n_fields, t.dim, stream_ptr()), 'grad_rows_pack')
            return packed

        def unpack(ids, packed):
            check(N.lib.dtb_grad_rows_unpack(ptr(ids), ptr(t.row_offsets), ptr(packed), ptr(t.grad), ids.shape[0],
                                             t.n_fields, t.dim, stream_ptr()), 'grad_rows_unpack')
        return pack, unpack

    def _begin_table_exchange(self, cat):
        """Called from inside backward the moment the table gradient is final (engine._table_grad_done):
        pack this rank's rows and start the all-gathers so they run under the remaining backward kernels."""
        pack, unpack = self._row_exchange_fns(cat)
        self._early_exchange = dp.TableExchange(cat, pack, unpack)

    def _exchange_gradients(self, cat):
        """Data-parallel exchange (dp.py): dense bucket all-reduce + row-wise table-gradient exchange; rows
        first touched by another rank this step are caught up before the row-wise Adam."""
        t = self.table
        early = getattr(self, '_early_exchange', None)
        self._early_exchange = None
        if early is not None:
            torch.distributed.all_reduce(self._scope.flat_g)
            union = early.finish()
        else:
            pack = unpack = None
            if t is not None and t.lazy_adam:
                pack, unpack = self._row_exchange_fns(cat)
            union = dp.exchange(self._scope.flat_g, t.grad if t is not None else None, cat, pack, unpack)
        if t is not None:
            self._catch_up(union, self._step)     # lazy mode: rows first touched by another rank this step
        return union

    def predict_step(self, cat, cont):
        if self.table is not None:
            self._catch_up(cat, self._step)
        with torch.no_grad():
            z = self._forward(cat, cont, training=False)
            prob, _ = E.loss_forward_backward(z, torch.zeros_like(z), self.task, None, False, None)
        return prob

    # ------------------------------------------------------------------------------------------
    # host <-> device input plumbing  (replaces utils/dataset_generator.py:36-72)
    # ------------------------------------------------------------------------------------------
    def _to_device_inputs(self, X, device=None):
        """DataFrame / dict of arrays -> (cat int32 [N,F] | None, cont float32 [N,C] | None) on ``device`` (default: the GPU)."""
        device = self.device if device is None else device
        cat = cont = None
        if self.n_fields:
            names = [c.name for c in self.categorical_columns]
            arr = _columns(X, names)
            if arr.dtype.kind == 'f':
                # the reference ships ids as float32 and casts back (dataset_generator.py:41-42,
                # layers.py:893-895); exact below 2**24
                arr = arr.astype(np.int64)
            cat = torch.as_tensor(np.ascontiguousarray(arr.astype(np.int32))).to(device, non_blocking=True)
        if self.n_cont:
            parts = [_columns(X, c.column_names).astype(np.float32) for c in self.continuous_columns]
            arr = parts[0] if len(parts) == 1 else np.concatenate(parts, axis=1)
            cont = torch.as_tensor(np.ascontiguousarray(arr)).to(device, non_blocking=True)
        return cat, cont

    def _to_device_labels(self, y, device=None):
        device = self.device if device is None else device
        y = np.asarray(y)
        if self.task == consts.TASK_MULTICLASS:
            onehot = np.zeros((len(y), self.num_classes), dtype=np.float32)
            onehot[np.arange(len(y)), y.astype(np.int64).reshape(-1)] = 1.0
            y = onehot
        y = y.astype(np.float32).reshape(len(y), -1)
        return torch.as_tensor(np.ascontiguousarray(y)).to(device, non_blocking=True)

    def train_on_batch(self, x_cat, x_cont, y, sample_weight=None):
        """Public per-batch entry (Keras ``Model.train_on_batch`` analogue): HOST arrays/tensors in,
        python float loss out -- includes the host->device copies and the device->host read."""
        cat = _host_to_device(x_cat, torch.int32, self.device) if self.n_fields else None
        cont = _host_to_device(x_cont, torch.float32, self.device) if self.n_cont else None
        yb = _host_to_device(y, torch.float32, self.device)
        yb = yb.view(yb.shape[0], -1)
        if self.model is None:
            self._build_model()
        self._loss_acc.zero_()
        sw = _host_to_device(sample_weight, torch.float32, self.device)
        self.train_step(cat, cont, yb, sw)
        return float(self._loss_acc.item()) / yb.shape[0]

    # ------------------------------------------------------------------------------------------
    # fit / predict / evaluate  (reference deepmodel.py:60-173)
    # ------------------------------------------------------------------------------------------
    def fit(self, X=None, y=None, batch_size=128, epochs=1, verbose=1, callbacks=None, validation_split=0.2,
            validation_data=None, shuffle=True, class_weight=None, sample_weight=None, initial_epoch=0,
            steps_per_epoch=None, validation_steps=None, validation_freq=1, max_queue_size=10, workers=1,
            use_multiprocessing=False):
        if sample_weight is not None and len(sample_weight) != _length(X):
            raise ValueError(f'sample_weight has {len(sample_weight)} entries for {_length(X)} rows')
        if validation_data is None:
            from sklearn.model_selection import train_test_split
            if sample_weight is not None:          # the weights follow their rows through the shuffle + split
                X, X_val, y, y_val, sample_weight, _ = train_test_split(X, y, np.asarray(sample_weight),
                                                                        test_size=validation_split)
            else:
                X, X_val, y, y_val = train_test_split(X, y, test_size=validation_split)
        else:
            if len(validation_data) != 2:
                raise ValueError(f'Unexpected validation_data length, expected 2 but {len(validation_data)}.')
            X_val, y_val = validation_data[0], validation_data[1]
        if batch_size is None:
            batch_size = 128
        n, n_val = _length(X), _length(X_val)
        if steps_per_epoch is None:
            steps_per_epoch = n // batch_size
            if steps_per_epoch == 0:
                steps_per_epoch = 1
        if validation_steps is None:
            validation_steps = n_val // batch_size - 1
            if validation_steps <= 1:
                validation_steps = 1
        if self.model is None:
            self._build_model()
        if self._dist:
            # every rank feeds its own shard; the ranks must agree on the number of collective steps
            agreed = torch.tensor([steps_per_epoch], dtype=torch.int64, device=self.device)
            torch.distributed.all_reduce(agreed, op=torch.distributed.ReduceOp.MIN)
            steps_per_epoch = int(agreed.item())
        # where the training rows live: HBM (default) or pinned host memory behind a double-buffered loader
        # (DTB_DATA_ON_HOST=1, or automatically when the encoded data set would take more than a quarter of the free HBM)
        row_bytes = 4 * (self.n_fields + self.n_cont + (self.num_classes if self.task == consts.TASK_MULTICLASS else 1))
        free_hbm = torch.cuda.mem_get_info(self.device)[0]
        on_host = os.environ.get('DTB_DATA_ON_HOST', '') == '1' or n * row_bytes > free_hbm // 4
        if on_host:
            cat, cont = self._to_device_inputs(X, device='cpu')
            yd = self._to_device_labels(y, device='cpu')
        else:
            cat, cont = self._to_device_inputs(X)
            yd = self._to_device_labels(y)
        vcat, vcont = self._to_device_inputs(X_val)
        vy = self._to_device_labels(y_val)
        sw = None
        if class_weight is not None:
            cw = torch.ones(int(max(class_weight)) + 1, dtype=torch.float32)
            for k, v in class_weight.items():
                cw[int(k)] = float(v)
            sw = cw[torch.as_tensor(np.asarray(y).astype(np.int64).reshape(-1))]
        if sample_weight is not None:
            s2 = torch.as_tensor(np.asarray(sample_weight, dtype=np.float32))
            sw = s2 if sw is None else sw * s2
        if sw is not None and not on_host:
            sw = sw.to(self.device)
        loader = _HostBatches(self.device, cat, cont, yd, sw) if on_host else None

        history = History()
        callbacks = list(callbacks or [])
        for cb in callbacks:
            if hasattr(cb, 'set_model'):
                cb.set_model(self)
        self.stop_training = False
        for cb in callbacks:
            _call(cb, 'on_train_begin', None)
        metric_fns = _resolve_metrics(self.config.metrics, self.task)
        # train batches drop the remainder only when there is at least one full batch
        # (reference dataset_generator.py:70)
        drop_remainder = n >= batch_size
        for epoch in range(initial_epoch, epochs):
            for cb in callbacks:
                _call(cb, 'on_epoch_begin', epoch, None)
            pdev = 'cpu' if on_host else self.device
            perm = torch.randperm(n, device=pdev) if shuffle else torch.arange(n, device=pdev)
            self._loss_acc.zero_()
            seen = 0
            probs, targets = [], []

            def rows_of(step):
                lo = (step * batch_size) % max(n, 1)
                sel = perm[lo:lo + batch_size]
                if drop_remainder and sel.numel() < batch_size:
                    sel = perm[:batch_size]
                return sel

            pending = loader.prefetch(rows_of(0)) if on_host and steps_per_epoch > 0 else None
            for step in range(steps_per_epoch):
                if on_host:
                    bc, bx, by, bw = loader.get(pending)
                    if step + 1 < steps_per_epoch:
                        pending = loader.prefetch(rows_of(step + 1))      # next batch travels while this step computes
                else:
                    sel = rows_of(step)
                    bc = cat[sel] if cat is not None else None
                    bx = cont[sel] if cont is not None else None
                    by = yd[sel]
                    bw = sw[sel] if sw is not None else None
                p = self.train_step(bc, bx, by, bw)
                seen += by.shape[0]
                if metric_fns:
                    probs.append(p)
                    targets.append(by)
            logs = {'loss': float(self._loss_acc.item()) / max(seen, 1)}
            if metric_fns:
                pp, tt = torch.cat(probs), torch.cat(targets)
                for name, fn in metric_fns.items():
                    logs[name] = fn(tt, pp)
            if self.table is not None:
                self.table.check_status()
            self.sync_replica_buffers()          # before validation / callbacks snapshot or score the model
            if (epoch + 1) % validation_freq == 0 and n_val > 0:
                vlogs = self._evaluate_tensors(vcat, vcont, vy, batch_size, validation_steps, metric_fns)
                if self._dist and vlogs:
                    # same validation logs on every rank (mean over the ranks' shards), so callbacks such as
                    # EarlyStopping(restore_best_weights) take identical decisions and the replicas stay identical
                    keys = sorted(vlogs)
                    vt = torch.tensor([float(vlogs[k]) for k in keys], dtype=torch.float64, device=self.device)
                    torch.distributed.all_reduce(vt)
                    vlogs = dict(zip(keys, (vt / self.world_size).tolist()))
                logs.update({f'val_{k}': v for k, v in vlogs.items()})
            history.epoch.append(epoch)
            for k, v in logs.items():
                history.history.setdefault(k, []).append(v)
            if verbose:
                msg = ' - '.join(f'{k}: {v:.4f}' for k, v in logs.items())
                print(f'Epoch {epoch + 1}/{epochs} - {steps_per_epoch} steps - {msg}')
            for cb in callbacks:
                _call(cb, 'on_epoch_end', epoch, logs)
            if self._dist:
                # early stopping looks at per-rank validation metrics: stop everywhere as soon as one rank stops
                flag = torch.tensor([1 if self.stop_training else 0], dtype=torch.int32, device=self.device)
                torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MAX)
                self.stop_training = bool(flag.item())
            if self.stop_training:
                break
        for cb in callbacks:
            _call(cb, 'on_train_end', None)
        history.history = IgnoreCaseDict(history.history)
        return history

    def _evaluate_tensors(self, cat, cont, y, batch_size, steps, metric_fns):
        n = y.shape[0]
        loss_acc = torch.zeros(1, dtype=torch.float64, device=self.device)
        probs, targets = [], []
        seen = 0
        for step in range(steps):
            lo = step * batch_size
            if lo >= n:
                break
            bc = cat[lo:lo + batch_size] if cat is not None else None
            bx = cont[lo:lo + batch_size] if cont is not None else None
            by = y[lo:lo + batch_size]
            if bc is not None:
                self._catch_up(bc, self._step)
            with torch.no_grad():
                z = self._forward(bc, bx, training=False)
                p, _ = E.loss_forward_backward(z, by, self.task, None, False, loss_acc, focal=self._focal)
            probs.append(p)
            targets.append(by)
            seen += by.shape[0]
        self._reg_loss(loss_acc, seen)          # Keras's compute_loss adds model.losses in evaluation too
        logs = {'loss': float(loss_acc.item()) / max(seen, 1)}
        pp, tt = torch.cat(probs), torch.cat(targets)
        for name, fn in metric_fns.items():
            logs[name] = fn(tt, pp)
        return logs

    def predict(self, X, batch_size=128, verbose=0):
        return self.__predict(X, batch_size=batch_size, verbose=verbose)

    def __predict(self, X, batch_size=128, verbose=0, capture=None):
        if self.model is None:
            raise RuntimeError('model is not built: call fit() or load a model first')
        cat, cont = self._to_device_inputs(X)
        n = _length(X)
        steps = math.ceil(n / batch_size)
        outs = []
        captured = {k: [] for k in (capture or [])}
        for step in range(steps):
            lo = step * batch_size
            bc = cat[lo:lo + batch_size] if cat is not None else None
            bx = cont[lo:lo + batch_size] if cont is not None else None
            if capture:
                if bc is not None:
                    self._catch_up(bc, self._step)
                with torch.no_grad():
                    self._forward(bc, bx, training=False, capture=set(capture))
                for k in capture:
                    if k not in self._scope.outputs:
                        raise ValueError(f'No layer found in the model:{k}')
                    o = self._scope.outputs[k]
                    captured[k].append(L._materialize(o).detach())
            else:
                outs.append(self.predict_step(bc, bx))
        if self.table is not None:
            self.table.check_status()
        if capture:
            return [torch.cat(captured[k]).cpu().numpy() for k in capture]
        return torch.cat(outs).cpu().numpy()

    def apply(self, X, output_layers=[], concat_outputs=False, batch_size=128, verbose=0, transformer=None):
        """Outputs of named intermediate layers (reference deepmodel.py:143-163)."""
        if len(output_layers) <= 0:
            raise ValueError('"output_layers" at least 1 element.')
        output = self.__predict(X, batch_size=batch_size, verbose=verbose, capture=list(output_layers))
        if len(output) > 1 and concat_outputs:
            output = np.concatenate([o.reshape(o.shape[0], -1) for o in output], axis=-1)
        elif len(output) == 1:
            output = output[0]
        if transformer is None:
            return output
        if isinstance(output, list):
            return [transformer.fit_transform(o.reshape(o.shape[0], -1) if o.ndim > 2 else o) for o in output]
        return transformer.fit_transform(output)

    def evaluate(self, X_test, y_test, batch_size=256, verbose=0, return_dict=True):
        if self.model is None:
            raise RuntimeError('model is not built: call fit() or load a model first')
        cat, cont = self._to_device_inputs(X_test)
        y = self._to_device_labels(y_test)
        steps = math.ceil(_length(X_test) / batch_size)
        logs = self._evaluate_tensors(cat, cont, y, batch_size, steps, _resolve_metrics(self.config.metrics, self.task))
        if return_dict:
            return IgnoreCaseDict(logs)
        return list(logs.values())

    # ------------------------------------------------------------------------------------------
    # weights in / out, keyed by the reference's layer/weight names
    # ------------------------------------------------------------------------------------------
    def flush_optimizer_state(self):
        """Bring every embedding row up to date (lazy row-wise optimiser) -- before export / save."""
        t = self.table
        if t is not None and t.lazy_active and t.last_step is not None and self._step > 0:
            o = self._opt
            if o.kind != 'adam':
                check(N.lib.dtb_optim_rows_flush(ptr(t.weight), *[ptr(x) for x in t.slots], ptr(t.last_step), self._step,
                                                 self._opt_native, t.total_rows, t.dim, stream_ptr()), 'optim_rows_flush')
                return
            check(N.lib.dtb_adam_rows_flush(ptr(t.weight), ptr(t.m), ptr(t.v), ptr(t.last_step),
                                            ptr(self._alpha_table(self._step)), self._step, o.beta_1, o.beta_2,
                                            o.epsilon, t.total_rows, t.dim, stream_ptr()), 'adam_rows_flush')

    def sync_replica_buffers(self):
        """Data parallel: BatchNormalization moving statistics are updated from each rank's own shard; average them
        over the replicas (tf.distribute.MirroredStrategy aggregates these variables with MEAN, reference
        deepmodel.py:88-103) so that inference, validation metrics and checkpoints do not depend on the rank."""
        if not self._dist or self._scope is None or not self._scope.buffers:
            return
        flat = torch.cat([b.reshape(-1) for b in self._scope.buffers.values()])
        torch.distributed.all_reduce(flat)
        flat /= self.world_size
        off = 0
        for b in self._scope.buffers.values():
            b.copy_(flat[off:off + b.numel()].view(b.shape))
            off += b.numel()

    def state_dict(self):
        self.flush_optimizer_state()
        sd = OrderedDict()
        if self.table is not None:
            for i in range(self.n_fields):
                sd[f'{consts.LAYER_PREFIX_EMBEDDING}categorical_vars_all/embeddings_{i}'] = self.table.field_weight(i)
        for k, v in self._scope.params.items():
            if k in self._scope.stacked:                 # a stacked family: one entry per reference weight name (views)
                for i, name in enumerate(self._scope.stacked[k]):
                    sd[name] = v.detach()[i]
            else:
                sd[k] = v.detach()
        for k, v in self._scope.buffers.items():
            sd[k] = v
        return sd

    def load_state_dict(self, sd, strict=True):
        own = self.state_dict()
        missing = [k for k in own if k not in sd]
        unexpected = [k for k in sd if k not in own]
        if strict and (missing or unexpected):
            raise KeyError(f'state dict mismatch: missing {missing}, unexpected {unexpected}')
        with torch.no_grad():
            for k, v in sd.items():
                if k in own:
                    src = torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v)
                    own[k].copy_(src.to(self.device, torch.float32).reshape(own[k].shape))

    def save(self, filepath):
        """Weights + architecture descriptor as .npz keyed by the reference's weight names (the
        reference writes Keras .h5, deepmodel.py:205-221; h5py is absent here -- SURVEY.md 8f rank 2)."""
        sd = {k: v.detach().cpu().numpy() for k, v in self.state_dict().items()}
        # optimiser state (the reference's .h5 keeps it too): Adam step, moments of the dense weights and of the
        # embedding rows (state_dict() flushed the lazy rows, so m/v are current for every row)
        # (SGD / RMSprop / Adagrad: their state slots under __opt_slot{i}__ / __opt_table_slot{i}__); __optimizer__ names
        # the optimiser and its hyperparameters, under which alone the state resumes
        opt = {'__step__': np.array(self._step), '__optimizer__': np.array(self._opt.describe())}
        if self._step > 0 and self._opt.kind != 'adam':
            for i, s in enumerate(self._scope.flat_slots):
                if s is not None:
                    opt[f'__opt_slot{i}__'] = s.cpu().numpy()
            if self.table is not None and self.table.slots is not None:
                for i, s in enumerate(self.table.slots):
                    if s is not None:
                        opt[f'__opt_table_slot{i}__'] = s.cpu().numpy()
        elif self._step > 0:
            opt['__adam_m__'] = self._scope.flat_m.cpu().numpy()
            opt['__adam_v__'] = self._scope.flat_v.cpu().numpy()
            if self.table is not None and self.table.m is not None:
                opt['__adam_table_m__'] = self.table.m.cpu().numpy()
                opt['__adam_table_v__'] = self.table.v.cpu().numpy()
        os.makedirs(os.path.dirname(os.path.abspath(filepath)) or '.', exist_ok=True)
        with open(filepath, 'wb') as f:
            np.savez(f, **opt, **sd)

    def _load_model(self, filepath):
        self._build_model()
        with np.load(filepath) as data:
            sd = {k: data[k] for k in data.files if not k.startswith('__')}
            opt = {k: data[k] for k in data.files if k.startswith('__')}
        self.load_state_dict(sd)
        self._restore_optimizer(opt)
        return self.model

    def _restore_optimizer(self, opt):
        """Resume the optimiser where the checkpoint left it.  A weights-only file, or one written under another optimiser
        or other hyperparameters, restarts it at step 0.  A file without __optimizer__ was written by Adam(1e-3)."""
        step = int(opt.get('__step__', 0))
        saved = str(opt['__optimizer__']) if '__optimizer__' in opt else O.resolve('auto').describe()
        if saved != self._opt.describe():
            step = 0
        if step > 0 and self._opt.kind != 'adam':
            t = self.table
            wanted = [f'__opt_slot{i}__' for i, s in enumerate(self._scope.flat_slots) if s is not None]
            if t is not None:
                t.ensure_training_state()
                wanted += [f'__opt_table_slot{i}__' for i, s in enumerate(t.slots) if s is not None]
            if all(k in opt for k in wanted):
                for i, s in enumerate(self._scope.flat_slots):
                    if s is not None:
                        s.copy_(torch.as_tensor(opt[f'__opt_slot{i}__']).to(self.device))
                if t is not None:
                    for i, s in enumerate(t.slots):
                        if s is not None:
                            s.copy_(torch.as_tensor(opt[f'__opt_table_slot{i}__']).to(self.device))
                    t.last_step.fill_(step)
                self._step = step
            else:
                self._step = 0
        elif step > 0 and '__adam_m__' in opt:
            self._scope.flat_m.copy_(torch.as_tensor(opt['__adam_m__']).to(self.device))
            self._scope.flat_v.copy_(torch.as_tensor(opt['__adam_v__']).to(self.device))
            if self.table is not None and '__adam_table_m__' in opt:
                t = self.table
                t.ensure_training_state()
                t.m.copy_(torch.as_tensor(opt['__adam_table_m__']).to(self.device))
                t.v.copy_(torch.as_tensor(opt['__adam_table_v__']).to(self.device))
                t.last_step.fill_(step)
            self._step = step
        else:
            self._step = 0
        if self._step_dev is not None:
            self._step_dev.fill_(self._step)

    def release(self):
        self.model = None
        self._scope = None
        self.table = None
        torch.cuda.empty_cache()


# -------------------------------------------------------------------------------------------------
# helpers
# -------------------------------------------------------------------------------------------------
class _LazyFlat:
    """``flatten_emb_layer`` argument of the net builders: materialised only if a builder uses it."""

    def __init__(self, scope, embeddings):
        self._scope, self._emb, self._val = scope, embeddings, None

    def _get(self):
        if self._val is None:
            self._val = self._scope.flatten_embeddings(self._emb)
            self._scope.record_output('flatten_embeddings', self._val)
        return self._val

    def __getattr__(self, item):
        return getattr(self._get(), item)

    def __torch_function__(self, func, types, args=(), kwargs=None):
        args = tuple(a._get() if isinstance(a, _LazyFlat) else a for a in args)
        return func(*args, **(kwargs or {}))


class _NullDesc:
    def __getattr__(self, item):
        return lambda *a, **k: None


def _native_optim_params(spec):
    """OptimizerSpec of SGD / RMSprop / Adagrad -> the kernels' dtb_optim_params."""
    kind = {'sgd': N.OPTIM_SGD, 'rmsprop': N.OPTIM_RMSPROP, 'adagrad': N.OPTIM_ADAGRAD}[spec.kind]
    flag = spec.nesterov if spec.kind == 'sgd' else spec.centered if spec.kind == 'rmsprop' else False
    return N.OptimParams(kind=kind, flag=int(bool(flag)), lr=spec.learning_rate, momentum=spec.momentum or 0.0,
                         rho=spec.rho or 0.0, eps=spec.epsilon or 0.0)


def _columns(X, names):
    if hasattr(X, 'iloc'):
        return X[list(names)].values
    if isinstance(X, dict):
        return np.stack([np.asarray(X[n]) for n in names], axis=1)
    raise TypeError(f'unsupported input container {type(X)}')


def _length(X):
    if hasattr(X, 'shape'):
        return X.shape[0]
    if isinstance(X, dict):
        return len(next(iter(X.values())))
    return len(X)


def _host_to_device(a, dtype, device):
    if a is None:
        return None
    t = a if torch.is_tensor(a) else torch.as_tensor(np.ascontiguousarray(a))
    return t.to(device=device, dtype=dtype, non_blocking=True)


def _call(cb, name, *args):
    fn = getattr(cb, name, None)
    if fn is not None:
        fn(*args)


def _auc(y_true, y_prob):
    """Rank-sum AUC on device (ties averaged)."""
    y = y_true.reshape(-1)
    p = y_prob.reshape(-1)
    n_pos = float((y > 0.5).sum())
    n_neg = float(y.numel()) - n_pos
    if n_pos == 0 or n_neg == 0:
        return 0.0
    vals, inv, counts = torch.unique(p, sorted=True, return_inverse=True, return_counts=True)
    csum = torch.cumsum(counts, 0).double()
    avg_rank = csum - (counts.double() - 1.0) / 2.0
    ranks = avg_rank[inv]
    s = float(ranks[y > 0.5].sum())
    return (s - n_pos * (n_pos + 1) / 2.0) / (n_pos * n_neg)


def _resolve_metrics(metrics, task):
    fns = OrderedDict()
    for m in (metrics or []):
        name = m if isinstance(m, str) else getattr(m, 'name', getattr(m, '__name__', str(m)))
        key = name.lower()
        if key in ('auc',):
            fns[name] = _auc
        elif key in ('accuracy', 'acc'):
            if task == consts.TASK_MULTICLASS:
                fns[name] = lambda t, p: float((p.argmax(-1) == t.argmax(-1)).float().mean())
            else:
                fns[name] = lambda t, p: float(((p > 0.5).float() == t).float().mean())
        elif key in ('mse', 'mean_squared_error'):
            fns[name] = lambda t, p: float(((p - t) ** 2).mean())
        elif key in ('rmse', 'rootmeansquarederror', 'root_mean_squared_error'):
            fns[name] = lambda t, p: float(((p - t) ** 2).mean().sqrt())
        elif key in ('mae', 'mean_absolute_error'):
            fns[name] = lambda t, p: float((p - t).abs().mean())
        elif callable(m):
            fns[name] = lambda t, p, _m=m: float(_m(t.cpu().numpy(), p.cpu().numpy()))
        else:
            raise NotImplementedError(f'metric {m!r}')
    return fns


class ModelDesc:
    """Human-readable description of the built model (reference deepmodel.py:460-532)."""

    def __init__(self):
        self.inputs, self.nets, self.nets_info = [], [], []
        self.embeddings = self.dense = self.concat_embed_dense = None
        self.stacking = self.output = self.loss = self.optimizer = None
        self.regularizers = []             # 'weight name: regularizer' of the regularized Dense kernels

    def add_input(self, name, num_columns):
        self.inputs.append(f'{name}: ({num_columns})')

    def set_embeddings(self, input_dims, output_dims, embedding_dropout):
        self.embeddings = f'input_dims: {input_dims}\noutput_dims: {output_dims}\ndropout: {embedding_dropout}'

    def set_embedding_storage(self, row_width, padding_share):
        """Columns of different widths share one table of the widest row; the rest of each row is padding."""
        self.embeddings += f'\nstored_width: {row_width}\npadding: {100.0 * padding_share:.1f}%'

    def set_dense(self, dense_dropout, use_batchnormalization):
        self.dense = f'dropout: {dense_dropout}\nbatch_normalization: {use_batchnormalization}'

    def set_concat_embed_dense(self, output_shape):
        self.concat_embed_dense = f'shape: {output_shape}'

    def add_net(self, name, input_shape, output_shape):
        self.nets_info.append(f'{name}: input_shape {input_shape}, output_shape {output_shape}')

    def set_output(self, activation, output_shape, use_bias):
        self.output = f'activation: {activation}, output_shape: {output_shape}, use_bias: {use_bias}'

    def nets_desc(self):
        return '\n'.join(self.nets_info)

    def optimizer_info(self):
        return self.optimizer

    def __str__(self):
        bar = '-' * 57
        rows = [('inputs', [c for c in self.inputs]), ('embeddings', self.embeddings), ('dense', self.dense),
                ('concat_embed_dense', self.concat_embed_dense), ('nets', f'{self.nets}\n{self.nets_desc()}'),
                ('stacking_op', self.stacking), ('output', self.output), ('loss', self.loss),
                ('optimizer', self.optimizer_info())]
        if self.regularizers:
            rows.insert(5, ('regularizers', '\n'.join(self.regularizers)))
        body = f'\n{bar}\n'.join(f'{k}: {v}' for k, v in rows)
        return f'>>>>>>>>>>>>>>>>>>>>>> Model Desc <<<<<<<<<<<<<<<<<<<<<<< \n{bar}\n{body}\n{bar}\n'


class IgnoreCaseDict(collections.UserDict):
    """dict with case-insensitive string keys (reference deepmodel.py:535-563)."""

    def __init__(self, inputs: Union[dict, collections.UserDict] = None):
        super().__init__()
        src = inputs.data if isinstance(inputs, collections.UserDict) else (inputs or {})
        for k, v in src.items():
            self[k] = v

    @staticmethod
    def _key(item):
        if not isinstance(item, str):
            raise KeyError(f'Key should be str but is {item}')
        return item.lower()

    def __contains__(self, item):
        return self._key(item) in self.data

    def __setitem__(self, item, value):
        self.data[self._key(item)] = value

    def __getitem__(self, item):
        return self.data[self._key(item)]
