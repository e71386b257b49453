"""Schedules whose rate grows, on the GPU: a learning-rate range test trains under CUDA-graph replay although its rate
table overflows far ahead, Adam's table rows switch from the lazy replay to the dense sweep where the growing alpha
leaves the replay's bound, a step whose rate overflowed is refused before it runs, and under data parallel ranks whose
ReduceLROnPlateau decisions differ agree on rank 0's rate."""
import os

import numpy as np
import pytest
import torch

from deeptables_b200 import callbacks as C
from deeptables_b200 import optimizers as O
from deeptables_b200 import schedules as S
from test_lr_schedules_gpu import DP_B, DP_CONT, DP_DIM, DP_VOCAB, _free_port, _states_equal, _train, batch, build

pytestmark = pytest.mark.gpu

RANGE_TEST = O.Adam(learning_rate=S.ExponentialDecay(1e-6, decay_steps=10, decay_rate=10.0))


def test_range_test_schedule_trains_under_graph_replay(monkeypatch):
    """The rate grows tenfold every 10 steps; the table the first captured step builds (400 000 entries) holds inf
    from step ~450 on, which no step here reaches."""
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager = _train(RANGE_TEST, 30)
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed = _train(RANGE_TEST, 30)
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    assert not np.isfinite(graphed._rates.host).all(), 'the table reaches the overflow'
    _states_equal(graphed, eager, 'growing schedule: graph replay vs eager')
    assert graphed.optimizer.learning_rate == float(np.float32(1e-6 * 10.0 ** 3))


@pytest.mark.parametrize('graphs', ['0', '1'])
def test_adam_table_leaves_the_lazy_replay_where_alpha_breaks_its_bound(monkeypatch, graphs):
    """With eps = 1e-12 the alpha of step 8 breaks the early-exit bound of the lazy replay: steps 1-7 run the rows
    lazily, later ones the dense sweep, and the weights are those of a run on the dense sweep throughout."""
    opt = O.Adam(learning_rate=S.ExponentialDecay(1e-3, decay_steps=2, decay_rate=10.0), epsilon=1e-12)
    monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
    model, _ = build(['linear', 'fm_nets', 'dnn_nets'], [400, 300, 500], 4, 2, seed=9, optimizer=opt)
    modes = []
    for step in range(10):
        _train(opt, 1, model=model)
        modes.append(model.table.lazy_active)
    assert modes == [True] * 7 + [False] * 3
    dense, _ = build(['linear', 'fm_nets', 'dnn_nets'], [400, 300, 500], 4, 2, seed=9, optimizer=opt)
    dense._table_mode_override = 'dense'
    _train(opt, 10, model=dense)
    assert not dense.table.lazy_active
    _states_equal(model, dense, 'lazy until the bound breaks, then dense, vs dense throughout')


@pytest.mark.parametrize('graphs', ['0', '1'])
def test_step_with_an_overflowed_rate_is_refused_before_it_runs(monkeypatch, graphs):
    """staircase ExponentialDecay: 0.01 for t < 3, then 1e48, which float32 cannot hold."""
    monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
    opt = O.SGD(learning_rate=S.ExponentialDecay(0.01, decay_steps=3, decay_rate=1e50, staircase=True), momentum=0.9)
    model = _train(opt, 3)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(ValueError, match='learning_rate'):
        _train(opt, 1, model=model)
    assert model._step == 3
    after = model.state_dict()
    for k in before:
        assert torch.equal(before[k], after[k]), f'{k} changed in the refused step'


def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m, _ = build(['linear', 'fm_nets', 'dnn_nets'], DP_VOCAB, DP_DIM, DP_CONT, seed=11,
                     optimizer=O.SGD(learning_rate=0.05, momentum=0.9))
        cb = C.ReduceLROnPlateau(monitor='loss', patience=1, factor=0.5, min_delta=0.0)
        cb.set_model(m)
        cb.on_train_begin()
        proposed, agreed = [], []
        for epoch in range(4):
            for step in range(3):
                m.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=(epoch * 3 + step) * world + rank))
            # rank 0's monitor improves every epoch, rank 1's never does: rank 1 alone decides to reduce
            cb.on_epoch_end(epoch, {'loss': 1.0 - epoch if rank == 0 else 1.0})
            proposed.append(m.optimizer.learning_rate)
            m._agree_learning_rate()
            agreed.append(m.optimizer.learning_rate)
        m.sync_replica_buffers()
        sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), __proposed__=np.array(proposed), __agreed__=np.array(agreed),
                 **sd)
    finally:
        dist.destroy_process_group()


def test_data_parallel_ranks_agree_on_rank0_rate_when_their_decisions_differ(tmp_path):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r0 = np.load(tmp_path / 'rank0.npz')
    r1 = np.load(tmp_path / 'rank1.npz')
    lr0 = float(np.float32(0.05))
    assert (r0['__proposed__'] == lr0).all()
    assert (r1['__proposed__'] < lr0).any(), 'rank 1 did not decide differently'
    assert (r0['__agreed__'] == lr0).all() and (r1['__agreed__'] == lr0).all()
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]) or k == '__proposed__', f'replica 1 diverged from replica 0 on {k}'
