"""Data-parallel training on 2 (and, when the box has them, 8) GPUs over NCCL: replicas stay bit-identical -- weights
after 6 optimiser steps and, once averaged (DeepModel.sync_replica_buffers, MirroredStrategy's MEAN aggregation), the
BatchNormalization moving statistics -- and ranks fed the SAME shard reproduce the single-GPU run on that shard (mean
of identical gradients).  With fewer than 2 GPUs the tests skip."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


VOCAB, DIM, N_CONT, B = [50, 40, 30, 20, 60], 8, 3, 64
NETS = ['linear', 'fm_nets', 'cin_nets', 'dnn_nets', 'cross_nets']


def _build(seed=11):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=NETS, embeddings_output_dim=DIM, embedding_dropout=0, metrics=['AUC'],
                                 cin_params={'cross_layer_size': (16, 16), 'activation': 'relu', 'use_residual': False,
                                             'use_bias': False, 'direct': False, 'reduce_D': False})
    cats = [CategoricalColumn(f'c{i}', v, DIM) for i, v in enumerate(VOCAB)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(N_CONT)])]
    m = DeepModel('binary', 2, conf, cats, conts, seed=seed)
    m._build_model()
    return m


def _batch(seed):
    g = np.random.default_rng(seed)
    idx = np.stack([g.integers(0, v, size=B) for v in VOCAB], axis=1).astype(np.int32)
    cont = g.normal(size=(B, N_CONT)).astype(np.float32)
    y = (g.random(B) < 0.4).astype(np.float32)
    return idx, cont, y


def _worker(rank, world, port, out_dir, same_shard, table_mode=None):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m = _build()
        m._table_mode_override = table_mode          # None: adaptive (dense sweep at this size); 'lazy': row-wise Adam on the union
        assert m.world_size == world
        for step in range(6):
            idx, cont, y = _batch(step if same_shard else step * world + rank)
            m.train_on_batch(idx, cont, y)
        m.sync_replica_buffers()                      # BN moving statistics: mean over the replicas (fit() does it per epoch)
        sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}      # state_dict() flushes the lazy state
        np.savez(os.path.join(out_dir, f'rank{rank}_{int(same_shard)}.npz'), **sd)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 8])
@pytest.mark.parametrize('table_mode', [None, 'lazy'])
@pytest.mark.parametrize('same_shard', [True, False])
def test_replicas_stay_bit_identical(tmp_path, same_shard, table_mode, world):
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), same_shard, table_mode), nprocs=world, join=True)
    r0 = np.load(tmp_path / f'rank0_{int(same_shard)}.npz')
    for rank in range(1, world):
        r1 = np.load(tmp_path / f'rank{rank}_{int(same_shard)}.npz')
        for k in r0.files:
            assert np.array_equal(r0[k], r1[k]), f'replica {rank} diverged from replica 0 on {k}'
    if same_shard:
        single = _build()
        for step in range(6):
            single.train_on_batch(*_batch(step))
        sd = single.state_dict()
        for k in r0.files:
            np.testing.assert_allclose(r0[k], sd[k].cpu().numpy(), rtol=1e-4, atol=1e-6, err_msg=k)
    print(f'world {world} same_shard {same_shard} table_mode {table_mode}: {len(r0.files)} tensors bit-identical on '
          f'{world} replicas')
