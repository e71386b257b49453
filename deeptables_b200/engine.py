"""Device-side state and autograd glue over the C ABI (deeptables_b200/_native.py).

* ``EmbeddingTable`` -- the F per-column Keras variables ``embeddings_{i}`` of MultiColumnEmbedding
  (reference layers.py:853-877) stored as ONE ``[sum V, D]`` buffer plus row offsets, with its
  gradient accumulator and row-wise Adam state.  Gradients never travel through autograd: every
  fused backward kernel scatter-adds straight into ``table.grad``.
* ``FieldBlock`` / ``EmbeddingList`` -- lazy ``(B, F, D)`` views (ids + table) handed to the net
  builders so the gather is fused into each interaction kernel instead of materialised.
* autograd ``Function`` wrappers -- one per C-ABI op; torch is only the allocator / autograd tape.
"""
import math

import torch

from . import _native as N
from ._native import ptr, check, stream_ptr

ADAM_B1, ADAM_B2, ADAM_EPS = 0.9, 0.999, 1e-7     # keras.optimizers.Adam defaults (deepmodel.py:321)
BN_EPS, BN_MOMENTUM = 1e-3, 0.99                   # keras BatchNormalization defaults


def _f32(t):
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.contiguous().float()


class EmbeddingTable:
    """All categorical columns' embedding matrices in one HBM buffer of row width ``dim``.

    ``field_dims`` (default: ``dim`` for every field) gives each field's own width D_i <= dim
    (``fixed_embedding_dim=False``).  Field i then uses columns [0, D_i) of its rows; columns [D_i, dim) are
    padding that is zero in the weights and the gradient and at its initial value in every optimiser slot.  No
    kernel writes them, and a zero gradient on zero state is a zero update under every optimiser, so the dense
    sweeps, the row-wise optimiser kernels and the data-parallel row exchange run unchanged on ``dim``-wide rows."""

    def __init__(self, vocab_sizes, dim, device, initializer='uniform', generator=None, lazy_adam=True,
                 field_dims=None):
        self.vocab_sizes = [int(v) for v in vocab_sizes]
        self.n_fields = len(self.vocab_sizes)
        self.dim = int(dim)
        self.field_dims = [self.dim] * self.n_fields if field_dims is None else [int(d) for d in field_dims]
        if len(self.field_dims) != self.n_fields or not all(1 <= d <= self.dim for d in self.field_dims):
            raise ValueError(f'field widths {self.field_dims} must be {self.n_fields} values in [1, {self.dim}]')
        self.ragged = any(d != self.dim for d in self.field_dims)
        self.dims_host = N.int_array(self.field_dims)
        self.device = torch.device(device)
        offs = [0]
        for v in self.vocab_sizes:
            offs.append(offs[-1] + v)
        self.total_rows = offs[-1]
        self.row_offsets_host = offs
        self.row_offsets = torch.tensor(offs, dtype=torch.int64, device=self.device)
        self.weight = torch.empty(self.total_rows, self.dim, dtype=torch.float32, device=self.device)
        if initializer == 'uniform':          # keras 'uniform' = RandomUniform(-0.05, 0.05)
            self.weight.uniform_(-0.05, 0.05, generator=generator)
        elif initializer == 'zeros':
            self.weight.zero_()
        else:
            raise NotImplementedError(f'embeddings_initializer={initializer!r}')
        for i, d in enumerate(self.field_dims):
            if d < self.dim:
                self.weight[offs[i]:offs[i + 1], d:] = 0.0
        self.grad = None
        self.m = None
        self.v = None
        self.slot_inits = None     # SGD / RMSprop / Adagrad: initial values of state slots s0..s2 (None: Adam's m, v)
        self.slots = None
        self.last_step = None
        self.claim = None          # per-row claim stamps of the data-parallel row exchange
        self.status = torch.zeros(1, dtype=torch.int32, device=self.device)
        # lazy row-wise Adam needs dim = 4*2^k; otherwise dense Adam over the whole table
        q = self.dim // 4
        self.lazy_adam = bool(lazy_adam and self.dim % 4 == 0 and 1 <= q <= 32 and (q & (q - 1)) == 0)
        self.lazy_active = self.lazy_adam     # which optimiser form is live (DeepModel._select_table_optimizer)
        # autograd anchor: fused ops take it as an input so their backward always runs
        self.anchor = torch.zeros(1, dtype=torch.float32, device=self.device, requires_grad=True)

    def ensure_training_state(self):
        if self.grad is None:
            self.grad = torch.zeros_like(self.weight)
            if self.slot_inits is None:
                self.m = torch.zeros_like(self.weight)
                self.v = torch.zeros_like(self.weight)
            else:
                self.slots = [None if s is None else torch.full_like(self.weight, s) for s in self.slot_inits]
            self.last_step = torch.zeros(self.total_rows, dtype=torch.int32, device=self.device)

    def field_weight(self, i):
        """View of the reference's ``embeddings_{i}`` variable: (V_i, D_i)."""
        lo, hi = self.row_offsets_host[i], self.row_offsets_host[i + 1]
        return self.weight[lo:hi, :self.field_dims[i]] if self.ragged else self.weight[lo:hi]

    def padding_share(self):
        """Fraction of the stored floats that are padding."""
        pad = sum(v * (self.dim - d) for v, d in zip(self.vocab_sizes, self.field_dims))
        return pad / max(1, self.total_rows * self.dim)

    def check_status(self):
        """TF-CPU raises on an out-of-range id (layers.py:898); the kernels flag it instead."""
        bits = int(self.status.item())
        if bits:
            self.status.zero_()
            cols = [i for i in range(self.n_fields) if bits & (1 << (i & 31))]
            raise IndexError(f'categorical id out of range for column(s) {cols} (mod 32)')


class FieldBlock:
    """Lazy (B, F, D) block of field embeddings = ids + table (what Concatenate(axis=1) of the
    reference's embedding list would hold, deepnets.py:30-40)."""

    def __init__(self, idx, table):
        self.idx = idx
        self.table = table
        self._mat = None

    @property
    def shape(self):
        return (self.idx.shape[0], self.table.n_fields, self.table.dim)

    def materialize(self):
        if self._mat is None:
            self._mat = GatherFn.apply(self.table.anchor, self)
        return self._mat

    @staticmethod
    def from_tensor(x):
        """Wrap an already materialised (B, F, D) tensor so the fused kernels can consume it:
        stored field-major [F, B, D] it IS a table with vocab B per field and ids = row number."""
        b, f, d = x.shape
        return _TensorFieldBlock(x)


class _TensorFieldBlock(FieldBlock):
    def __init__(self, x):
        b, f, d = x.shape
        self.x = x
        tab = _TensorTable(x)
        idx = torch.arange(b, dtype=torch.int32, device=x.device).unsqueeze(1).expand(b, f).contiguous()
        super().__init__(idx, tab)

    def materialize(self):
        return self.x


class _TensorTable:
    """Table facade over a materialised (B,F,D) tensor (see FieldBlock.from_tensor)."""

    def __init__(self, x):
        b, f, d = x.shape
        self.src = x
        self.n_fields, self.dim, self.device = f, d, x.device
        self.weight = x.detach().permute(1, 0, 2).contiguous().view(f * b, d)
        self.row_offsets = torch.arange(f + 1, dtype=torch.int64, device=x.device) * b
        self.grad = torch.zeros_like(self.weight) if x.requires_grad else None
        self.status = None
        self.anchor = x        # gradient flows back into x through TensorTableGradFn
        self.is_tensor_table = True


class EmbeddingList:
    """What the reference passes to net builders as ``embeddings``: a list of F tensors (B,1,D)
    (layers.py:889-904).  Indexing materialises; the built-in builders use ``.block`` instead."""

    def __init__(self, block):
        self.block = block

    def __len__(self):
        return self.block.table.n_fields

    def __getitem__(self, i):
        mat = self.block.materialize()
        if isinstance(i, slice):
            return [mat[:, j:j + 1, :] for j in range(*i.indices(len(self)))]
        return mat[:, i:i + 1, :]

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]


class RaggedFieldBlock:
    """Embeddings of fields of different widths (ids + table, ``table.ragged``): what ``flatten_embeddings`` of the
    reference's embedding list holds, (B, sum D_i).  ``flat`` set: an already materialised (dropped-out) tensor."""

    def __init__(self, idx, table, flat=None):
        self.idx, self.table, self._mat = idx, table, flat

    def materialize(self):
        if self._mat is None:
            self._mat = RaggedConcatEmbDenseFn.apply(self.table.anchor, None, self)
        return self._mat


class RaggedEmbeddingList:
    """The reference's embedding list for fields of different widths: item i is (B, 1, D_i), a slice of the flat
    (B, sum D_i) block, so every consumer sees the same gather (and the same dropout mask)."""

    def __init__(self, block):
        self.block = block
        cols = [0]
        for d in block.table.field_dims:
            cols.append(cols[-1] + d)
        self._cols = cols

    def __len__(self):
        return self.block.table.n_fields

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        if i < 0:
            i += len(self)
        flat = self.block.materialize()
        return flat[:, self._cols[i]:self._cols[i + 1]].unsqueeze(1)

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]


def _tabs(block):
    t = block.table
    return t, block.idx, t.weight, t.row_offsets


def _grad_target(table):
    if getattr(table, 'is_tensor_table', False):
        return table.grad
    table.ensure_training_state()
    return table.grad


def _note_consumer(ctx, table):
    """Forward of a table-consuming op that autograd will differentiate (the anchor input requires grad
    and grad mode was on at apply time): one more backward will add into table.grad."""
    if ctx.needs_input_grad[0] and not getattr(table, 'is_tensor_table', False):
        table.pending_bwd = getattr(table, 'pending_bwd', 0) + 1


def _table_grad_done(table):
    """An op finished its contribution to table.grad.  When it was the last one of the step the table
    gradient is final and the data-parallel exchange may start -- possibly while weight-gradient kernels
    of the same op are still to be launched (CINFn)."""
    if getattr(table, 'is_tensor_table', False):
        return
    table.pending_bwd = getattr(table, 'pending_bwd', 1) - 1
    if table.pending_bwd == 0 and getattr(table, 'on_grad_final', None) is not None:
        table.on_grad_final()


class _TableBackwardMixin:
    @staticmethod
    def finish_tensor_table(table):
        """For tensor-backed blocks return the gradient wrt the source tensor (else None)."""
        if getattr(table, 'is_tensor_table', False) and table.grad is not None:
            f, d = table.n_fields, table.dim
            b = table.weight.shape[0] // f
            g = table.grad.view(f, b, d).permute(1, 0, 2).contiguous()
            table.grad = torch.zeros_like(table.weight)
            return g
        return None


class GatherFn(torch.autograd.Function):
    """MultiColumnEmbedding.call, materialising form (layers.py:889-904)."""

    @staticmethod
    def forward(ctx, anchor, block):
        t, idx, w, offs = _tabs(block)
        b = idx.shape[0]
        out = torch.empty(b, t.n_fields, t.dim, dtype=torch.float32, device=w.device)
        check(N.lib.dtb_embedding_gather(ptr(idx), ptr(w), ptr(offs), ptr(out), b, t.n_fields, t.dim,
                                         ptr(t.status), stream_ptr()), 'embedding_gather')
        # NOT ctx.block: the block caches this op's output (FieldBlock._mat), whose grad_fn owns ctx -- a reference cycle
        # that kept the whole autograd graph of a step (and the gradient accumulators bound to the stream it ran on)
        # alive until the next garbage collection, which invalidated CUDA-graph capture of the following step
        ctx.table, ctx.idx = t, idx
        _note_consumer(ctx, t)
        return out

    @staticmethod
    def backward(ctx, g):
        t, idx = ctx.table, ctx.idx
        gt = _grad_target(t)
        g = _f32(g)
        check(N.lib.dtb_embedding_scatter_add(ptr(idx), ptr(t.row_offsets), ptr(g), ptr(gt), idx.shape[0], t.n_fields,
                                              t.dim, stream_ptr()), 'embedding_scatter_add')
        _table_grad_done(t)
        return _TableBackwardMixin.finish_tensor_table(t), None


class FMLinearFn(torch.autograd.Function):
    """linear (deepnets.py:43-66) and/or FM (layers.py:53-62) with the gather fused."""

    @staticmethod
    def forward(ctx, anchor, dense, w_lin, block, want_lin, want_fm):
        if block is not None:
            t, idx, w, offs = _tabs(block)
            b, f, d = idx.shape[0], t.n_fields, t.dim
            status = t.status
        else:
            t = idx = w = offs = status = None
            b, f, d = dense.shape[0], 0, 0
        c = 0 if dense is None else dense.shape[1]
        dev = dense.device if dense is not None else w.device
        out_lin = torch.empty(b, 1, dtype=torch.float32, device=dev) if want_lin else None
        out_fm = torch.empty(b, 1, dtype=torch.float32, device=dev) if want_fm else None
        check(N.lib.dtb_fm_linear_fwd(ptr(idx), ptr(w), ptr(offs), ptr(dense), ptr(w_lin), ptr(out_lin),
                                      ptr(out_fm), b, f, d, c, ptr(status), stream_ptr()), 'fm_linear_fwd')
        ctx.block, ctx.dims = block, (b, f, d, c)
        ctx.save_for_backward(dense, w_lin)
        ctx.want = (want_lin, want_fm)
        if t is not None:
            _note_consumer(ctx, t)
        outs = tuple(o for o in (out_lin, out_fm) if o is not None)
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *grads):
        dense, w_lin = ctx.saved_tensors
        b, f, d, c = ctx.dims
        want_lin, want_fm = ctx.want
        grads = list(grads)
        g_lin = _f32(grads.pop(0)) if want_lin else None
        g_fm = _f32(grads.pop(0)) if want_fm else None
        block = ctx.block
        gt = idx = w = offs = t = None
        if block is not None:
            t, idx, w, offs = _tabs(block)
            gt = _grad_target(t)
        gw = torch.zeros_like(w_lin) if want_lin else None
        check(N.lib.dtb_fm_linear_bwd(ptr(idx), ptr(w), ptr(offs), ptr(dense), ptr(w_lin), ptr(g_lin),
                                      ptr(g_fm), ptr(gt), ptr(gw), b, f, d, c, stream_ptr()), 'fm_linear_bwd')
        if t is not None:
            _table_grad_done(t)
        ga = _TableBackwardMixin.finish_tensor_table(t) if t is not None else None
        gd = None
        if ctx.needs_input_grad[1] and want_lin:       # input gradients (explain.gradient_values); training never asks
            gd = torch.empty_like(dense)
            check(N.lib.dtb_linear_dense_grad(ptr(g_lin), ptr(w_lin[f:]), ptr(gd), b, c, stream_ptr()),
                  'linear_dense_grad')
        return ga, gd, gw, None, None, None


class ConcatEmbDenseFn(torch.autograd.Function):
    """flatten_embeddings + concat_embedding_dense (deepmodel.py:269-278, 348-357)."""

    @staticmethod
    def forward(ctx, anchor, dense, block):
        t, idx, w, offs = _tabs(block)
        b, f, d = idx.shape[0], t.n_fields, t.dim
        c = 0 if dense is None else dense.shape[1]
        x = torch.empty(b, f * d + c, dtype=torch.float32, device=w.device)
        check(N.lib.dtb_concat_emb_dense_fwd(ptr(idx), ptr(w), ptr(offs), ptr(dense), ptr(x), b, f, d, c,
                                             ptr(t.status), stream_ptr()), 'concat_emb_dense_fwd')
        ctx.block, ctx.dims = block, (b, f, d, c)
        _note_consumer(ctx, t)
        return x

    @staticmethod
    def backward(ctx, g):
        t, idx, w, offs = _tabs(ctx.block)
        b, f, d, c = ctx.dims
        gt = _grad_target(t)
        g = _f32(g)
        check(N.lib.dtb_concat_emb_dense_bwd(ptr(idx), ptr(offs), ptr(g), ptr(gt), b, f, d, c, stream_ptr()),
              'concat_emb_dense_bwd')
        _table_grad_done(t)
        gd = g[:, f * d:] if ctx.needs_input_grad[1] else None      # training never asks
        return _TableBackwardMixin.finish_tensor_table(t), gd, None


class RaggedConcatEmbDenseFn(torch.autograd.Function):
    """flatten_embeddings + concat_embedding_dense over fields of different widths: (B, sum D_i + C)."""

    @staticmethod
    def forward(ctx, anchor, dense, block):
        t, idx = block.table, block.idx
        b, sd = idx.shape[0], sum(t.field_dims)
        c = 0 if dense is None else dense.shape[1]
        x = torch.empty(b, sd + c, dtype=torch.float32, device=t.weight.device)
        check(N.lib.dtb_ragged_concat_emb_dense_fwd(ptr(idx), ptr(t.weight), ptr(t.row_offsets), t.dims_host, ptr(dense),
                                                    ptr(x), b, t.n_fields, t.dim, c, ptr(t.status), stream_ptr()),
              'ragged_concat_emb_dense_fwd')
        ctx.table, ctx.idx, ctx.c = t, idx, c
        _note_consumer(ctx, t)
        return x

    @staticmethod
    def backward(ctx, g):
        t, idx = ctx.table, ctx.idx
        gt = _grad_target(t)
        g = _f32(g)
        check(N.lib.dtb_ragged_concat_emb_dense_bwd(ptr(idx), ptr(t.row_offsets), t.dims_host, ptr(g), ptr(gt),
                                                    idx.shape[0], t.n_fields, t.dim, ctx.c, stream_ptr()),
              'ragged_concat_emb_dense_bwd')
        _table_grad_done(t)
        gd = g[:, sum(t.field_dims):] if ctx.needs_input_grad[1] else None      # training never asks
        return None, gd, None


class BatchNormFn(torch.autograd.Function):
    """keras BatchNormalization(axis=-1) training forward/backward over the flattened rows."""

    @staticmethod
    def forward(ctx, x, gamma, beta, moving_mean, moving_var):
        x = _f32(x)
        cols = x.shape[-1]
        rows = x.numel() // cols
        y = torch.empty_like(x)
        save_mean = torch.empty(cols, dtype=torch.float32, device=x.device)
        save_var = torch.empty(cols, dtype=torch.float32, device=x.device)
        ws = torch.empty(2 * cols, dtype=torch.float64, device=x.device)
        check(N.lib.dtb_batchnorm_train_fwd(ptr(x), ptr(y), ptr(gamma), ptr(beta), ptr(moving_mean),
                                            ptr(moving_var), ptr(save_mean), ptr(save_var), ptr(ws), rows, cols,
                                            BN_EPS, BN_MOMENTUM, stream_ptr()), 'batchnorm_train_fwd')
        ctx.save_for_backward(x, gamma, save_mean, save_var)
        ctx.ws = ws
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, save_mean, save_var = ctx.saved_tensors
        dy = _f32(dy)
        cols = x.shape[-1]
        rows = x.numel() // cols
        dx = torch.empty_like(x)
        dgamma = torch.zeros_like(gamma)
        dbeta = torch.zeros_like(gamma)
        check(N.lib.dtb_batchnorm_bwd(ptr(x), ptr(dy), ptr(dx), ptr(gamma), ptr(save_mean), ptr(save_var),
                                      ptr(dgamma), ptr(dbeta), ptr(ctx.ws), rows, cols, BN_EPS, stream_ptr()),
              'batchnorm_bwd')
        return dx, dgamma, dbeta, None, None


def batchnorm_infer(x, gamma, beta, moving_mean, moving_var):
    x = _f32(x)
    cols = x.shape[-1]
    rows = x.numel() // cols
    y = torch.empty_like(x)
    check(N.lib.dtb_batchnorm_infer_fwd(ptr(x), ptr(y), ptr(gamma), ptr(beta), ptr(moving_mean),
                                        ptr(moving_var), rows, cols, BN_EPS, stream_ptr()), 'batchnorm_infer_fwd')
    return y


class BatchNormInferFn(torch.autograd.Function):
    """keras BatchNormalization in inference (the moving statistics), differentiated with respect to its input only:
    the input gradient with the parameters and statistics held fixed (explain.gradient_values)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, moving_mean, moving_var):
        ctx.save_for_backward(gamma, moving_var)
        return batchnorm_infer(x, gamma, beta, moving_mean, moving_var)

    @staticmethod
    def backward(ctx, dy):
        gamma, moving_var = ctx.saved_tensors
        dy = _f32(dy)
        cols = dy.shape[-1]
        dx = torch.empty_like(dy)
        check(N.lib.dtb_batchnorm_infer_bwd(ptr(dy), ptr(dx), ptr(gamma), ptr(moving_var), dy.numel() // cols, cols,
                                            BN_EPS, stream_ptr()), 'batchnorm_infer_bwd')
        return dx, None, None, None, None


def _seed_args(seed):
    """(host seed, device seed pointer) of a dropout seed: an integer, or inside the capture of a CUDA graph the
    one-element device slot ``_Scope.next_seed`` hands out."""
    return (0, ptr(seed)) if torch.is_tensor(seed) else (int(seed), None)


def _dropout(x, y, rate, seed, what):
    host, dev = _seed_args(seed)
    if dev is not None:
        check(N.lib.dtb_dropout_dev(ptr(x), ptr(y), x.numel(), rate, dev, stream_ptr()), what)
    else:
        check(N.lib.dtb_dropout(ptr(x), ptr(y), x.numel(), rate, host, stream_ptr()), what)


class DropoutFn(torch.autograd.Function):
    """keras Dropout / SpatialDropout1D on field embeddings: counter-based mask, nothing stored."""

    @staticmethod
    def forward(ctx, x, rate, seed):
        x = _f32(x)
        y = torch.empty_like(x)
        _dropout(x, y, float(rate), seed, 'dropout')
        ctx.cfg = (float(rate), seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _f32(dy)
        dx = torch.empty_like(dy)
        _dropout(dy, dx, ctx.cfg[0], ctx.cfg[1], 'dropout_bwd')
        return dx, None, None


ACT_CODES = {None: 0, 'linear': 0, 'relu': 1, 'tanh': 2}


class DenseFn(torch.autograd.Function):
    """keras Dense: act(x @ kernel + bias) over the last axis."""

    @staticmethod
    def forward(ctx, x, kernel, bias, act, grad_premasked=False):
        """grad_premasked: the consumer's backward already returns the gradient of the PRE-activation (it zeroes it
        where this layer's relu output is zero: AttentionCoreFn with mask_inputs) -- no activation-gradient pass."""
        x = _f32(x)
        in_dim, out_dim = kernel.shape
        rows = x.numel() // in_dim
        y = torch.empty(*x.shape[:-1], out_dim, dtype=torch.float32, device=x.device)
        ws_bytes = N.lib.dtb_dense_workspace_bytes(in_dim, out_dim)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
        check(N.lib.dtb_dense_fwd(ptr(x), ptr(kernel), ptr(bias), ptr(y), ptr(ws), ws_bytes, rows, in_dim, out_dim, act,
                                  stream_ptr()), 'dense_fwd')
        if grad_premasked:
            assert act == ACT_CODES['relu']
            act = 0
        ctx.save_for_backward(x, kernel, y if act else None)
        ctx.has_bias, ctx.act = bias is not None, act
        return y

    @staticmethod
    def backward(ctx, dy):
        x, kernel, y = ctx.saved_tensors
        in_dim, out_dim = kernel.shape
        rows = x.numel() // in_dim
        dz = dy.contiguous().float()
        if ctx.act:
            dz = dz.clone()                             # overwritten with d(pre-activation)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        # input gradients with the weights held fixed (explain.gradient_values) skip the weight-gradient kernels
        want_w = ctx.needs_input_grad[1]
        dw = torch.zeros_like(kernel) if want_w else None
        db = torch.zeros(out_dim, dtype=torch.float32, device=x.device) if ctx.has_bias and want_w else None
        ws_bytes = N.lib.dtb_dense_workspace_bytes(in_dim, out_dim)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device) if ws_bytes else None
        check(N.lib.dtb_dense_bwd(ptr(x), ptr(kernel), ptr(y), ptr(dz), ptr(dx), ptr(dw), ptr(db), ptr(ws), ws_bytes,
                                  rows, in_dim, out_dim, ctx.act, stream_ptr()), 'dense_bwd')
        return dx, dw, db, None, None


class CINFn(torch.autograd.Function):
    """CIN feature maps + sum pooling (layers.py:682-726) with the gather fused."""

    @staticmethod
    def forward(ctx, anchor, weights, bias, block, sizes, direct, act, precision, training):
        t, idx, w, offs = _tabs(block)
        b, f, d = idx.shape[0], t.n_fields, t.dim
        sizes_c = N.int_array(sizes)
        n = len(sizes)
        pooled_w = sum(sizes) if direct else sum(s // 2 for s in sizes[:-1]) + sizes[-1]
        pooled = torch.empty(b, pooled_w, dtype=torch.float32, device=w.device)
        ws_bytes = N.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), int(training))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=w.device)
        saved = None
        if training:
            saved = torch.empty(N.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, int(direct)), dtype=torch.uint8,
                                device=w.device)
        check(N.lib.dtb_cin_fwd(ptr(idx), ptr(w), ptr(offs), ptr(weights), ptr(bias), ptr(pooled), ptr(saved),
                                ptr(ws), ws_bytes, b, f, d, sizes_c, n, int(direct), act, precision,
                                ptr(t.status), stream_ptr()), 'cin_fwd')
        ctx.block, ctx.cfg = block, (b, f, d, tuple(sizes), int(direct), act, precision)
        ctx.saved_buf, ctx.ws, ctx.has_bias = saved, ws, bias is not None
        ctx.save_for_backward(weights)
        _note_consumer(ctx, t)
        return pooled

    @staticmethod
    def backward(ctx, g):
        (weights,) = ctx.saved_tensors
        t, idx, w, offs = _tabs(ctx.block)
        b, f, d, sizes, direct, act, precision = ctx.cfg
        sizes_c = N.int_array(sizes)
        g = _f32(g)
        gt = _grad_target(t)
        want_w = ctx.needs_input_grad[1]       # False for input gradients with the weights held fixed
        dw = torch.zeros_like(weights) if want_w else torch.empty_like(weights)
        db = torch.zeros(sum(sizes), dtype=torch.float32, device=w.device) if ctx.has_bias and want_w else None
        args = (ptr(idx), ptr(w), ptr(offs), ptr(weights), ptr(g), ptr(ctx.saved_buf), ptr(gt), ptr(dw), ptr(db),
                ptr(ctx.ws), ctx.ws.numel(), b, f, d, sizes_c, len(sizes), direct, act, precision)
        # phase 1: everything that adds into the table gradient; then (data parallel) the exchange of the
        # table gradient may start and overlap phase 2, the weight-gradient kernels
        check(N.lib.dtb_cin_bwd_phase(*args, 1, stream_ptr()), 'cin_bwd(dgrad)')
        _table_grad_done(t)
        if want_w:
            check(N.lib.dtb_cin_bwd_phase(*args, 2, stream_ptr()), 'cin_bwd(wgrad)')
        ctx.saved_buf = ctx.ws = None
        return (_TableBackwardMixin.finish_tensor_table(t), dw if want_w else None, db, None, None, None, None, None,
                None)


class CrossFn(torch.autograd.Function):
    """Cross.call (layers.py:428-436)."""

    @staticmethod
    def forward(ctx, x, kernels, biases):
        x = _f32(x)
        b, w = x.shape
        n = kernels.shape[0]
        y = torch.empty_like(x)
        xw = torch.empty(b, n, dtype=torch.float32, device=x.device)
        check(N.lib.dtb_cross_fwd(ptr(x), ptr(kernels), ptr(biases), ptr(y), ptr(xw), b, w, n, stream_ptr()),
              'cross_fwd')
        ctx.save_for_backward(x, kernels, biases, xw)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, kernels, biases, xw = ctx.saved_tensors
        b, w = x.shape
        n = kernels.shape[0]
        dy = _f32(dy)
        dx = torch.empty_like(x)
        dk = torch.zeros_like(kernels)
        db = torch.zeros_like(biases)
        ws_bytes = N.lib.dtb_cross_bwd_workspace_bytes(b, w, n)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
        check(N.lib.dtb_cross_bwd(ptr(x), ptr(kernels), ptr(biases), ptr(xw), ptr(dy), ptr(dx), ptr(dk), ptr(db),
                                  ptr(ws), ws_bytes, b, w, n, stream_ptr()), 'cross_bwd')
        return dx, dk, db


class PNNFn(torch.autograd.Function):
    """InnerProduct / OuterProduct (layers.py:473-487, 541-581) with the gather fused."""

    KT = {'mat': 0, 'vec': 1, 'num': 2}

    @staticmethod
    def forward(ctx, anchor, op_kernel, block, want_ip, want_op, kernel_type):
        t, idx, w, offs = _tabs(block)
        b, f, d = idx.shape[0], t.n_fields, t.dim
        pairs = f * (f - 1) // 2
        ip = torch.empty(b, pairs, dtype=torch.float32, device=w.device) if want_ip else None
        op = torch.empty(b, pairs, dtype=torch.float32, device=w.device) if want_op else None
        check(N.lib.dtb_pnn_fwd(ptr(idx), ptr(w), ptr(offs), ptr(op_kernel), ptr(ip), ptr(op), b, f, d,
                                PNNFn.KT[kernel_type], ptr(t.status), stream_ptr()), 'pnn_fwd')
        ctx.block, ctx.cfg = block, (b, f, d, want_ip, want_op, kernel_type)
        ctx.save_for_backward(op_kernel)
        _note_consumer(ctx, t)
        outs = tuple(o for o in (ip, op) if o is not None)
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *grads):
        (op_kernel,) = ctx.saved_tensors
        t, idx, w, offs = _tabs(ctx.block)
        b, f, d, want_ip, want_op, kernel_type = ctx.cfg
        grads = list(grads)
        d_ip = _f32(grads.pop(0)) if want_ip else None
        d_op = _f32(grads.pop(0)) if want_op else None
        gt = _grad_target(t)
        dk = torch.zeros_like(op_kernel) if want_op else None
        check(N.lib.dtb_pnn_bwd(ptr(idx), ptr(w), ptr(offs), ptr(op_kernel), ptr(d_ip), ptr(d_op), ptr(gt),
                                ptr(dk), b, f, d, PNNFn.KT[kernel_type], stream_ptr()), 'pnn_bwd')
        _table_grad_done(t)
        return _TableBackwardMixin.finish_tensor_table(t), dk, None, None, None, None


class AFMFn(torch.autograd.Function):
    """AFM.call up to the attention-pooled pair product (layers.py:790-804), gather fused: [B, D]."""

    @staticmethod
    def forward(ctx, anchor, att_kernel, att_bias, projection_h, block, act):
        t, idx, w, offs = _tabs(block)
        b, f, d = idx.shape[0], t.n_fields, t.dim
        h = att_kernel.shape[1]
        pooled = torch.empty(b, d, dtype=torch.float32, device=w.device)
        check(N.lib.dtb_afm_fwd(ptr(idx), ptr(w), ptr(offs), ptr(att_kernel), ptr(att_bias), ptr(projection_h), ptr(pooled),
                                b, f, d, h, act, ptr(t.status), stream_ptr()), 'afm_fwd')
        ctx.block, ctx.cfg = block, (b, f, d, h, act)
        ctx.save_for_backward(att_kernel, att_bias, projection_h)
        _note_consumer(ctx, t)
        return pooled

    @staticmethod
    def backward(ctx, g):
        att_kernel, att_bias, projection_h = ctx.saved_tensors
        t, idx, w, offs = _tabs(ctx.block)
        b, f, d, h, act = ctx.cfg
        g = _f32(g)
        gt = _grad_target(t)
        dk, db, dh = torch.zeros_like(att_kernel), torch.zeros_like(att_bias), torch.zeros_like(projection_h)
        # the per-pair scratch (da, dv: (HT + D) floats per row and pair) is 3 GB at 65 536 rows x 26 fields and grows with
        # F^2 (an FGCNN block has ~100 fields): row chunks keep it under 4 GB; every output of the call accumulates
        ws_total = N.lib.dtb_afm_workspace_bytes(b, f, d, h)
        rows_per = max(1, b) if ws_total <= (4 << 30) else max(1, int(b * (4 << 30) // ws_total))
        ws_bytes = N.lib.dtb_afm_workspace_bytes(min(rows_per, b), f, d, h)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=w.device)
        for r0 in range(0, b, rows_per):
            nb = min(rows_per, b - r0)
            check(N.lib.dtb_afm_bwd(ptr(idx[r0:r0 + nb]), ptr(w), ptr(offs), ptr(att_kernel), ptr(att_bias), ptr(projection_h),
                                    ptr(g[r0:r0 + nb]), ptr(gt), ptr(dk), ptr(db), ptr(dh), ptr(ws), ws_bytes, nb, f, d, h, act,
                                    stream_ptr()), 'afm_bwd')
        _table_grad_done(t)
        return _TableBackwardMixin.finish_tensor_table(t), dk, db, dh, None, None


BILINEAR_TYPES = {'field_all': 0, 'field_each': 1, 'field_interaction': 2}


class BilinearFn(torch.autograd.Function):
    """BilinearInteraction.call (layers.py:358-372) on a dense [B, F, D] block; weights stacked [n_w, D, D]."""

    @staticmethod
    def forward(ctx, x, w, bilinear_type):
        x = _f32(x)
        b, f, d = x.shape
        out = torch.empty(b, f * (f - 1) // 2, d, dtype=torch.float32, device=x.device)
        check(N.lib.dtb_bilinear_fwd(ptr(x), ptr(w), ptr(out), b, f, d, BILINEAR_TYPES[bilinear_type], stream_ptr()), 'bilinear_fwd')
        ctx.save_for_backward(x, w)
        ctx.bt = BILINEAR_TYPES[bilinear_type]
        return out

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        b, f, d = x.shape
        g = _f32(g)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.zeros_like(w)
        check(N.lib.dtb_bilinear_bwd(ptr(x), ptr(w), ptr(g), ptr(dx), ptr(dw), b, f, d, ctx.bt, stream_ptr()), 'bilinear_bwd')
        return dx, dw, None


class SenetPoolFn(torch.autograd.Function):
    """SENET squeeze (layers.py:295-298): mean or max over the embedding axis, [B, F, D] -> [B, F]."""

    @staticmethod
    def forward(ctx, x, op):
        x = _f32(x)
        b, f, d = x.shape
        z = torch.empty(b, f, dtype=torch.float32, device=x.device)
        check(N.lib.dtb_senet_pool_fwd(ptr(x), ptr(z), b, f, d, op, stream_ptr()), 'senet_pool_fwd')
        ctx.save_for_backward(x, z)
        ctx.op = op
        return z

    @staticmethod
    def backward(ctx, dz):
        x, z = ctx.saved_tensors
        b, f, d = x.shape
        dx = torch.empty_like(x)
        check(N.lib.dtb_senet_pool_bwd(ptr(x), ptr(z), ptr(_f32(dz)), ptr(dx), b, f, d, ctx.op, stream_ptr()), 'senet_pool_bwd')
        return dx, None


class SenetScaleFn(torch.autograd.Function):
    """SENET re-weighting (layers.py:301): V = X * A[:, :, None]."""

    @staticmethod
    def forward(ctx, x, a):
        x, a = _f32(x), _f32(a)
        b, f, d = x.shape
        v = torch.empty_like(x)
        check(N.lib.dtb_senet_scale_fwd(ptr(x), ptr(a), ptr(v), b, f, d, stream_ptr()), 'senet_scale_fwd')
        ctx.save_for_backward(x, a)
        return v

    @staticmethod
    def backward(ctx, dv):
        x, a = ctx.saved_tensors
        b, f, d = x.shape
        dx, da = torch.empty_like(x), torch.empty_like(a)
        check(N.lib.dtb_senet_scale_bwd(ptr(x), ptr(a), ptr(_f32(dv)), ptr(dx), ptr(da), b, f, d, stream_ptr()), 'senet_scale_bwd')
        return dx, da


class ConvFieldsFn(torch.autograd.Function):
    """FGCNN's Conv2D(filters, (kh, 1), padding='same', activation) along the field axis of [B, H, W, Cin] (layers.py:204-212)."""

    @staticmethod
    def forward(ctx, x, kernel, bias, act):
        x = _f32(x)
        b, h, w, cin = x.shape
        kh, _, _, cout = kernel.shape
        y = torch.empty(b, h, w, cout, dtype=torch.float32, device=x.device)
        check(N.lib.dtb_conv_fields_fwd(ptr(x), ptr(kernel), ptr(bias), ptr(y), b, h, w, cin, cout, kh, act, stream_ptr()),
              'conv_fields_fwd')
        ctx.save_for_backward(x, kernel, y)
        ctx.cfg = (act, bias is not None)
        return y

    @staticmethod
    def backward(ctx, g):
        x, kernel, y = ctx.saved_tensors
        act, has_bias = ctx.cfg
        b, h, w, cin = x.shape
        kh, _, _, cout = kernel.shape
        g = _f32(g)
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dk = torch.zeros_like(kernel)
        db = torch.zeros(cout, dtype=torch.float32, device=x.device) if has_bias else None
        check(N.lib.dtb_conv_fields_bwd(ptr(x), ptr(kernel), ptr(y), ptr(g), ptr(dx), ptr(dk), ptr(db), b, h, w, cin, cout, kh, act,
                                        stream_ptr()), 'conv_fields_bwd')
        return dx, dk, db, None


class MaxPoolFieldsFn(torch.autograd.Function):
    """FGCNN's MaxPooling2D((pool, 1), padding='same') along the field axis (layers.py:214)."""

    @staticmethod
    def forward(ctx, x, pool):
        x = _f32(x)
        b, h, w, c = x.shape
        y = torch.empty(b, -(-h // pool), w, c, dtype=torch.float32, device=x.device)
        check(N.lib.dtb_maxpool_fields_fwd(ptr(x), ptr(y), b, h, w * c, pool, stream_ptr()), 'maxpool_fields_fwd')
        ctx.save_for_backward(x)
        ctx.pool = pool
        return y

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        b, h, w, c = x.shape
        dx = torch.empty_like(x)
        check(N.lib.dtb_maxpool_fields_bwd(ptr(x), ptr(_f32(g)), ptr(dx), b, h, w * c, ctx.pool, stream_ptr()), 'maxpool_fields_bwd')
        return dx, None


class AttentionCoreFn(torch.autograd.Function):
    """MultiheadAttention.call between the projections and the BatchNormalization
    (layers.py:129-150): per-head softmax(QK^T/sqrt(dh))V + residual, relu; with ``rate`` > 0 dropout on the softmax
    weights, its mask regenerated in backward from ``seed``."""

    @staticmethod
    def forward(ctx, qkvr, heads, use_residual, mask_inputs=False, rate=0.0, seed=None):
        """mask_inputs: qkvr are relu outputs and backward returns the gradient of their pre-activations."""
        qkvr = _f32(qkvr)
        b, f, d4 = qkvr.shape
        d = d4 // 4
        y = torch.empty(b, f, d, dtype=torch.float32, device=qkvr.device)
        rate = float(rate)
        if rate > 0:
            check(N.lib.dtb_attention_core_dropout_fwd(ptr(qkvr), ptr(y), b, f, d, heads, int(use_residual), rate,
                                                       *_seed_args(seed), 0, stream_ptr()), 'attention_core_dropout_fwd')
        else:
            check(N.lib.dtb_attention_core_fwd(ptr(qkvr), ptr(y), b, f, d, heads, int(use_residual), stream_ptr()),
                  'attention_core_fwd')
        ctx.save_for_backward(qkvr, y)
        ctx.cfg = (heads, int(use_residual), int(bool(mask_inputs)), rate, seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        qkvr, y = ctx.saved_tensors
        b, f, d4 = qkvr.shape
        heads, use_res, mask, rate, seed = ctx.cfg
        dy = _f32(dy)
        dq = torch.empty_like(qkvr)
        if rate > 0:
            check(N.lib.dtb_attention_core_dropout_bwd(ptr(qkvr), ptr(y), ptr(dy), ptr(dq), b, f, d4 // 4, heads, use_res,
                                                       mask, rate, *_seed_args(seed), 0, stream_ptr()),
                  'attention_core_dropout_bwd')
        else:
            check(N.lib.dtb_attention_core_bwd(ptr(qkvr), ptr(y), ptr(dy), ptr(dq), b, f, d4 // 4, heads, use_res, mask,
                                               stream_ptr()), 'attention_core_bwd')
        return dq, None, None, None, None, None


TASK_CODES = {'binary': 0, 'multilabel': 0, 'regression': 1, 'multiclass': 2}


def loss_forward_backward(z, y_true, task, sample_weight=None, want_grad=True, loss_acc=None, focal=None, loss=None):
    """task_output activation + loss + dLoss/dz in one launch (deepmodel.py:319-346, 436-457).
    Returns (prob, dz or None); adds the sum of per-row losses to ``loss_acc`` (float64[1]).
    ``focal`` = (gamma, alpha): the reference's Binary / CategoricalFocalLoss (layers.py:983-1083) instead of BCE / CCE.
    ``loss``: a ``losses.LossSpec`` (ModelConfig.loss); where it is the task's own BCE / MSE / CCE the task's kernel
    runs it, otherwise ``dtb_keras_loss_fwd_bwd`` (the hinge losses add one launch that checks the labels)."""
    z = _f32(z)
    y_true = _f32(y_true).view(z.shape)
    prob = torch.empty_like(z)
    dz = torch.empty_like(z) if want_grad else None
    rows, cols = z.shape
    if focal is not None:
        if sample_weight is not None:
            raise NotImplementedError('focal losses take no sample weights')
        check(N.lib.dtb_focal_loss_fwd_bwd(ptr(z), ptr(y_true), ptr(prob), ptr(dz), ptr(loss_acc), rows, cols, TASK_CODES[task],
                                           float(focal[0]), float(focal[1]), stream_ptr()), 'focal_loss_fwd_bwd')
        return prob, dz
    if loss is not None and not loss.builtin(task):
        scratch = torch.empty(1, dtype=torch.int32, device=z.device) if loss.hinge else None
        lp = N.LossParams(loss=loss.code, delta=loss.delta, label_smoothing=loss.label_smoothing,
                          scratch=None if scratch is None else scratch.data_ptr())
        check(N.lib.dtb_keras_loss_fwd_bwd(ptr(z), ptr(y_true), ptr(sample_weight), ptr(prob), ptr(dz), ptr(loss_acc),
                                           rows, cols, TASK_CODES[task], lp, stream_ptr()),
              'keras_loss_fwd_bwd')
        return prob, dz
    check(N.lib.dtb_loss_fwd_bwd(ptr(z), ptr(y_true), ptr(sample_weight), ptr(prob), ptr(dz), ptr(loss_acc), rows,
                                 cols, TASK_CODES[task], stream_ptr()), 'loss_fwd_bwd')
    return prob, dz


class MetricsState:
    """Device state of one model's streaming metrics (metrics.Plan): the counters and sums ``dtb_metrics_update`` adds
    each batch to, the threshold lists it reads, and the ``dtb_metric_plan`` that describes both."""

    def __init__(self, plan, device):
        self.plan = plan
        n = N.MetricPlan(cols=plan.cols, n_lists=len(plan.lists), sums=plan.sums, argmax=int(plan.argmax),
                         top_k=plan.top_k)
        for i, lst in enumerate(plan.lists):
            n.list_len[i], n.list_off[i] = len(lst), plan.list_off[i]
        self.native = n
        words = N.lib.dtb_metrics_state_bytes(n) // 8
        if words != plan.words:
            raise RuntimeError(f'metric state layout mismatch: library {words} words, metrics.Plan {plan.words}')
        self.state = torch.zeros(words, dtype=torch.int64, device=device)
        self.thresholds = torch.as_tensor(plan.thresholds()).to(device)

    def reset(self):
        check(N.lib.dtb_metrics_reset(ptr(self.state), self.native, stream_ptr()), 'metrics_reset')

    def update(self, prob, y_true):
        """Add one batch: ``prob`` and ``y_true`` float32 [rows, plan.cols] in device memory."""
        prob, y_true = _f32(prob), _f32(y_true)
        if prob.dim() != 2 or prob.shape[1] != self.plan.cols or y_true.numel() != prob.numel():
            raise ValueError(f'metrics: expected [rows, {self.plan.cols}] predictions and labels, got '
                             f'{tuple(prob.shape)} and {tuple(y_true.shape)}')
        if prob.shape[0] == 0:
            return
        check(N.lib.dtb_metrics_update(ptr(prob), ptr(y_true), ptr(self.state), ptr(self.thresholds), prob.shape[0],
                                       self.native, stream_ptr()), 'metrics_update')

    def read(self):
        """The state as a host uint64 array (one device-to-host copy)."""
        return self.state.cpu().numpy().view('uint64')


def adam_alpha(step, lr=1e-3, b1=ADAM_B1, b2=ADAM_B2):
    """lr * sqrt(1 - b2^t) / (1 - b1^t)  (keras Adam.update_step)."""
    return lr * math.sqrt(1.0 - b2 ** step) / (1.0 - b1 ** step)
