"""Benchmark of the denoising auto-encoder (deeptables_b200/dae.py, csrc/dae.cu) on seeded synthetic data in [0, 1].

    python tools/bench_dae.py [--epochs 3] [--out FILE]

Prints one JSON line, with the card's name and power limit from the same nvidia-smi call:
- A, the reference's defaults: encoder_units=(500, 500), feature_units=20, relu, noise_rate=0.15, batch_size=128,
  N = 200 000, M = 200.  ms per epoch with the train step replayed from CUDA graphs and with DTB_CUDA_GRAPH=0, and this
  library's kernel launches per step in each mode;
- B: A with batch_size=4096 and N = 1 000 000;
- C, a wide net: encoder_units=(1500, 1500, 1500), feature_units=1500, M = 221, N = 595 212, batch_size=4096.  Achieved
  TFLOP/s counting 6 * sum(in * out) * rows per step, beside the data sheet's 989 dense BF16 TFLOP/s divided by the
  three bf16 passes of the Dense kernels (a data-sheet bound, not a measurement);
- dtb_dae_swap_batch alone: CUDA events over 100 graph-replayed launches at 4096 x 221, k = 33; GB/s of algorithmic
  bytes (three float32 row images -- the clean read and the two writes -- plus the two int64 permutation reads);
- the CPU baseline for A and C: the same step (swap noise, the Dense stack, MSE, Adam) restated in torch on the host's
  cores, labelled as such: TensorFlow, which the reference needs, is not available.

Epoch times are the gaps between consecutive epoch ends (each ends with the loss read, a device synchronisation); the
first epoch (allocations, the eager first step, the captures) is not counted.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BF16_DENSE_TFLOPS = 989.0          # H100 SXM data sheet, dense
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet

WORKLOADS = {
    'A': dict(units=(500, 500), feat=20, rows=200_000, cols=200, bs=128),
    'B': dict(units=(500, 500), feat=20, rows=1_000_000, cols=200, bs=4096),
    'C': dict(units=(1500, 1500, 1500), feat=1500, rows=595_212, cols=221, bs=4096),
}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:        # the numbers are still printed; the card is then unknown
        return f'unknown ({e})'


def data(rows, cols, seed=0):
    return np.random.default_rng(seed).random((rows, cols), dtype=np.float32)


class _EpochClock:
    def __init__(self):
        self.ends = []

    def set_model(self, model):
        pass

    def on_epoch_end(self, epoch, logs=None):
        self.ends.append(time.perf_counter())


def run_gpu(w, epochs, graphs):
    import torch
    from deeptables_b200 import _native as N, dae
    os.environ['DTB_CUDA_GRAPH'] = graphs
    X = data(w['rows'], w['cols'])
    d = dae.DAE(encoder_units=w['units'], feature_units=w['feat'], noise_rate=0.15, random_state=0)
    ae = d.build_dae(X[:2])
    x = torch.from_numpy(X).cuda()
    clock = _EpochClock()
    l0 = N.lib.dtb_launch_count()
    ae._fit(x, w['bs'], epochs, dae.swap_count(w['cols'], 0.15), True, [clock])
    steps = math.ceil(w['rows'] / w['bs'])
    launches = (N.lib.dtb_launch_count() - l0) / (steps * epochs)
    ms = min(b - a for a, b in zip(clock.ends, clock.ends[1:])) * 1e3
    flops = 6 * sum(i * o for _, i, o, _ in ae.plan) * w['rows']
    return dict(ms_per_epoch=ms, launches_per_step=launches, steps_per_epoch=steps, mse=ae.history.history['mse'],
                tflops=flops / (ms / 1e3) / 1e12)


def swap_kernel(rows=4096, cols=221, k=33):
    import torch
    from deeptables_b200 import _native as N
    from deeptables_b200._native import ptr, stream_ptr
    n = 200_000
    X = torch.from_numpy(data(n, cols)).cuda()
    p1, p2 = torch.randperm(n, device='cuda'), torch.randperm(n, device='cuda')
    step = torch.zeros(1, dtype=torch.int32, device='cuda')
    x_in, x_tgt = torch.empty(rows, cols, device='cuda'), torch.empty(rows, cols, device='cuda')

    def launch():
        N.check(N.lib.dtb_dae_swap_batch(ptr(X), cols, ptr(p1), ptr(p2), ptr(step), ptr(step), rows, rows, k, 1,
                                         ptr(x_in), ptr(x_tgt), stream_ptr()), 'dae_swap_batch')
    launch()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch()
    for _ in range(10):
        graph.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(100):
        graph.replay()
    e.record()
    e.synchronize()
    t = s.elapsed_time(e) / 1e3 / 100
    algo = 3 * rows * cols * 4 + 2 * rows * 8
    return dict(us=t * 1e6, algorithmic_GBps=algo / t / 1e9, hbm_bound_us=algo / HBM_BYTES_PER_S * 1e6)


def cpu_step_ms(w, steps):
    """The same train step in torch on the host: swap noise, the Dense stack, Keras MSE and Adam."""
    import torch
    torch.set_num_threads(os.cpu_count())
    from deeptables_b200 import dae
    plan = dae.layer_plan(w['units'], w['feat'], 'relu', w['cols'])
    g = torch.Generator().manual_seed(0)
    layers = [torch.nn.Linear(i, o) for _, i, o, _ in plan]
    acts = [a for *_, a in plan]
    opt = torch.optim.Adam([p for m in layers for p in m.parameters()], lr=1e-3, eps=1e-7)
    X = torch.from_numpy(data(min(w['rows'], 20 * w['bs']), w['cols']))
    bs, cols, k = w['bs'], w['cols'], dae.swap_count(w['cols'], 0.15)

    def step():
        idx = torch.randint(0, X.shape[0], (bs,), generator=g)
        donor = X[torch.randint(0, X.shape[0], (bs,), generator=g)]
        tgt = X[idx]
        sw = torch.rand(bs, cols, generator=g).argsort(dim=1)[:, :k]
        xin = tgt.clone()
        xin.scatter_(1, sw, donor.gather(1, sw))
        h = xin
        for m, a in zip(layers, acts):
            h = m(h)
            h = torch.relu(h) if a == 'relu' else h
        loss = ((h - tgt) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    ms = (time.perf_counter() - t0) / steps * 1e3
    return dict(ms_per_step=ms, ms_per_epoch=ms * math.ceil(w['rows'] / bs), steps_timed=steps,
                label='CPU restatement — TensorFlow unavailable')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--epochs', type=int, default=3)
    ap.add_argument('--cpu-steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_dae needs a GPU')
    res = {'card': card(), 'cpu_count': os.cpu_count()}
    for name, w in WORKLOADS.items():
        res[name] = {'replayed': run_gpu(w, args.epochs, '1')}
        if name == 'A':
            res[name]['eager'] = run_gpu(w, 2, '0')
    res['C']['datasheet_bound_tflops'] = BF16_DENSE_TFLOPS / 3
    res['swap_kernel_4096x221_k33'] = swap_kernel()
    res['cpu_A'] = cpu_step_ms(WORKLOADS['A'], args.cpu_steps)
    res['cpu_C'] = cpu_step_ms(WORKLOADS['C'], max(2, args.cpu_steps // 10))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
