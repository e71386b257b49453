"""Data-parallel gradient exchange (reference: tf.distribute.MirroredStrategy around the model
build, deepmodel.py:88-103 -- gradient all-reduce inside TensorFlow, per-replica BatchNorm).

One process per GPU, ``torch.distributed`` (NCCL between the GPUs of one machine; gloo in the CPU tests).
The path shards by batch rows only, so the exchange is:

  1. the loss gradient is pre-scaled by 1/world_size (``scale_for_mean``), which turns the SUM
     all-reduce into MirroredStrategy's global-batch mean;
  2. ONE all-reduce bucket for every dense weight gradient (the flat gradient buffer);
  3. the embedding-table gradient travels BY ROWS: each rank packs the rows its batch touched
     ([B, F, D], duplicates claimed once) and the ranks all-gather ids and packed rows -- 116 MB per
     rank at the Criteo shape instead of all-reducing the dense 1.66 GB [sum V, D] buffer; every rank
     then adds the ranks' rows in rank order, so the replicas stay bit-identical (TensorFlow exchanges
     embedding gradients as IndexedSlices the same way).  Tables whose width the row kernels do not
     support fall back to one dense all-reduce;
  4. the gathered ids are also the UNION of touched rows every rank's row-wise Adam must visit.

Nothing else crosses GPUs (no embedding sharding, no all-to-all); scoring needs no collective.
"""
import torch
import torch.distributed as dist


def is_distributed():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def world_size():
    return dist.get_world_size() if is_distributed() else 1


def scale_for_mean(dz):
    """dLoss/dz of the local batch mean -> contribution to the global-batch mean."""
    if is_distributed():
        dz.mul_(1.0 / dist.get_world_size())
    return dz


def exchange(flat_grad, table_grad, cat_ids, pack_rows=None, unpack_rows=None):
    """All-reduce the dense gradient bucket in place, exchange the table gradient, and return the
    union of the ranks' id batches ([world*B, F]; ``cat_ids`` itself when single-process / no table).

    pack_rows() -> packed [B,F,D] tensor (moves this rank's touched rows out of ``table_grad``);
    unpack_rows(ids, packed) adds one rank's rows back.  Without them the table gradient is
    all-reduced densely."""
    if not is_distributed():
        return cat_ids
    world = dist.get_world_size()
    dist.all_reduce(flat_grad)
    if table_grad is None or cat_ids is None:
        return cat_ids
    ids = cat_ids.contiguous()
    all_ids = torch.empty((world,) + tuple(ids.shape), dtype=ids.dtype, device=ids.device)
    dist.all_gather_into_tensor(all_ids, ids) if hasattr(dist, 'all_gather_into_tensor') and ids.is_cuda else \
        dist.all_gather(list(all_ids.unbind(0)), ids)
    if pack_rows is None:
        dist.all_reduce(table_grad)
    else:
        packed = pack_rows()
        all_packed = torch.empty((world,) + tuple(packed.shape), dtype=packed.dtype, device=packed.device)
        if packed.is_cuda:
            dist.all_gather_into_tensor(all_packed, packed)
        else:
            dist.all_gather(list(all_packed.unbind(0)), packed)
        for w in range(world):                       # fixed order => identical bits on every replica
            unpack_rows(all_ids[w], all_packed[w])
    return all_ids.reshape(-1, ids.shape[-1])


class TableExchange:
    """The row-wise exchange in two halves so that the all-gathers run under other kernels:
    ``begin`` (pack + asynchronous all-gathers) as soon as the table gradient is final, ``finish``
    (wait + rank-ordered unpack) right before the optimiser."""

    def __init__(self, cat_ids, pack_rows, unpack_rows):
        self.ids = cat_ids.contiguous()
        self.unpack_rows = unpack_rows
        world = dist.get_world_size()
        self.all_ids = torch.empty((world,) + tuple(self.ids.shape), dtype=self.ids.dtype, device=self.ids.device)
        self.packed = pack_rows()
        self.all_packed = torch.empty((world,) + tuple(self.packed.shape), dtype=self.packed.dtype,
                                      device=self.packed.device)
        if self.ids.is_cuda:
            self.works = [dist.all_gather_into_tensor(self.all_ids, self.ids, async_op=True),
                          dist.all_gather_into_tensor(self.all_packed, self.packed, async_op=True)]
        else:
            self.works = [dist.all_gather(list(self.all_ids.unbind(0)), self.ids, async_op=True),
                          dist.all_gather(list(self.all_packed.unbind(0)), self.packed, async_op=True)]

    def finish(self):
        for w in self.works:
            w.wait()
        for r in range(self.all_ids.shape[0]):          # fixed order => identical bits on every replica
            self.unpack_rows(self.all_ids[r], self.all_packed[r])
        return self.all_ids.reshape(-1, self.ids.shape[-1])


def broadcast_parameters(tensors, src=0):
    """Identical replicas at start: rank ``src``'s initial weights win."""
    if is_distributed():
        for t in tensors:
            if t is not None:
                dist.broadcast(t, src)
