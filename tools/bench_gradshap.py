"""Throughput of expected gradients (utils.shap.DeepTablesGradientExplainer) on one GPU, against Kernel SHAP on the same
models and against the same expected gradients computed by torch on the CPU over the oracle restatement of the model.

tools/bench_shap.py's two cases, each model fitted for one epoch on 20 000 rows:
- DeepFM on the 16-column bank-shaped frame with 100 background rows;
- xDeepFM on the 39-column Criteo-shaped frame with 50 background rows.
For each case: explained rows per second at nsamples=200 and the time split into dtb_gradshap_compose, the forward,
the backward (output-gradient seed included) and dtb_gradshap_reduce + dtb_gradshap_means (CUDA events); Kernel SHAP's
rows per second (nsamples='auto'); and the CPU baseline's seconds per explained row (oracle/model_ref.py forward in
float32 with torch autograd, the same interpolated inputs, one forward and backward over a row's 200 samples).

    python tools/bench_gradshap.py [--rows 2048] [--shap-rows 32] [--cpu-rows 2] [--rounds 3]

Prints one JSON line per measurement, the card name and power limit first, read in the same run.  Each figure is the
median over rounds.  There is no fallback: without a CUDA device it exits with an error."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_optim import card  # noqa: E402
from bench_shap import bank_frame, criteo_frame, fitted  # noqa: E402

NSAMPLES = 200


def cpu_seconds_per_row(ex, X, rows, seed):
    """The expected gradients of ``rows`` rows by torch on the CPU: the oracle model in float32, the interpolated
    embeddings and continuous values as leaves, one backward of the output per row."""
    import numpy as np
    import torch
    from deeptables_b200 import explain
    from oracle import model_ref as M
    bg = ex._background
    model = bg.model
    state = {k: v.detach().cpu().float() for k, v in model.state_dict().items()}
    table = model.table.weight.detach().cpu()
    offs = model.table.row_offsets_host
    dims = model.table.field_dims
    x_cat, x_cont = bg.encode(X.iloc[:rows])
    xc, bc = x_cat.cpu().numpy(), bg.cat.cpu().numpy()
    xn, bn = x_cont.cpu(), bg.cont.cpu()
    F = xc.shape[1]
    t0 = time.perf_counter()
    for i in range(rows):
        j, alpha = explain.gradient_draws(seed, i, NSAMPLES, bg.rows)
        a = torch.as_tensor(alpha)
        st = dict(state)
        leaves = []
        for f in range(F):
            ei = table[offs[f] + xc[i, f], :dims[f]]
            ej = table[offs[f] + bc[j, f], :dims[f]]
            leaf = (ej + a[:, None] * (ei - ej)).requires_grad_(True)
            st[f'emb_categorical_vars_all/embeddings_{f}'] = leaf
            leaves.append(leaf)
        z = (bn[j] + a[:, None] * (xn[i] - bn[j])).requires_grad_(True)
        idx = torch.arange(NSAMPLES).unsqueeze(1).expand(NSAMPLES, F).contiguous()
        out, _ = M.forward(st, model.config, idx, z, F, False, model.task)
        grads = torch.autograd.grad(out[:, 0].sum(), leaves + [z], allow_unused=True)
        vals = [((g * (table[offs[f] + xc[i, f], :dims[f]] - table[offs[f] + bc[j, f], :dims[f]])).sum(1)).double()
                for f, g in enumerate(grads[:F]) if g is not None]
        vals.append((grads[-1] * (xn[i] - bn[j])).double().sum(0) if grads[-1] is not None else None)
        _ = [v.mean(0) for v in vals if v is not None]
    return (time.perf_counter() - t0) / rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=2048, help='explained rows per expected-gradients call')
    ap.add_argument('--shap-rows', type=int, default=32, help='explained rows per Kernel SHAP call')
    ap.add_argument('--cpu-rows', type=int, default=2, help='explained rows of the CPU baseline')
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    import torch
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesExplainer, DeepTablesGradientExplainer
    if not torch.cuda.is_available():
        sys.exit('bench_gradshap needs a CUDA device')
    print(json.dumps(card()), flush=True)
    cases = [('DeepFM', 'bank', bank_frame, 100, {'embeddings_output_dim': 4}),
             ('xDeepFM', 'criteo', criteo_frame, 50,
              {'embeddings_output_dim': 16, 'categorical_columns': [f'C{i}' for i in range(26)]})]
    for nets, name, make, n_bg, conf in cases:
        X, y = make(20_000 + a.rows + 1000, 0)
        dt = fitted(nets, X.iloc[:20_000], y[:20_000], **conf)
        Xe = X.iloc[20_000:].reset_index(drop=True)
        bg_frame = Xe.iloc[a.rows:]
        ex = DeepTablesGradientExplainer(dt, bg_frame, num_samples=n_bg, random_state=0)
        ex.get_shap_values(Xe.iloc[:a.rows], NSAMPLES)                          # warm-up at the timed shapes
        totals, splits = [], []
        for r in range(a.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            explain.gradient_values(ex._background, Xe.iloc[:a.rows], NSAMPLES, r, ex.batch_size)
            torch.cuda.synchronize()
            totals.append(time.perf_counter() - t0)
            st = {}
            explain.gradient_values(ex._background, Xe.iloc[:a.rows], NSAMPLES, r, ex.batch_size, stages=st)
            splits.append(st)
        total = statistics.median(totals)
        split = {k: round(statistics.median(s[k] for s in splits), 4) for k in splits[0]}
        print(json.dumps({'what': 'expected gradients, device', 'nets': nets, 'frame': name, 'columns': X.shape[1],
                          'background': n_bg, 'nsamples': NSAMPLES, 'explained_rows': a.rows,
                          'call_s': round(total, 3), 'rows_per_s': round(a.rows / total, 1), 'split_s': split,
                          'rounds': a.rounds}), flush=True)

        kex = DeepTablesExplainer(dt, bg_frame, num_samples=n_bg, random_state=0)
        kex.get_shap_values(Xe.iloc[:2])
        times = []
        for r in range(a.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            explain.shap_values(kex._background, Xe.iloc[:a.shap_rows], 'auto', r, kex.batch_size)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        print(json.dumps({'what': 'Kernel SHAP, device', 'nets': nets, 'frame': name, 'explained_rows': a.shap_rows,
                          'rows_per_s': round(a.shap_rows / statistics.median(times), 1)}), flush=True)

        torch.set_num_threads(os.cpu_count() or 1)
        s_row = cpu_seconds_per_row(ex, Xe, a.cpu_rows, 0)
        print(json.dumps({'what': 'expected gradients, torch on the CPU (oracle model, float32)', 'nets': nets,
                          'frame': name, 'explained_rows': a.cpu_rows, 'threads': torch.get_num_threads(),
                          's_per_row': round(s_row, 3), 'rows_per_s': round(1 / s_row, 2)}), flush=True)


if __name__ == '__main__':
    main()
