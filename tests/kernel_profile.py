"""Which of this library's kernels a call launched, with the grid and block of each launch (torch.profiler)."""
import json
import os
import re
import tempfile
import time

import pytest
import torch


def short_name(name):
    """'void dtb::fm_linear_fwd_vec<2>(int const*, ...)' -> 'fm_linear_fwd_vec<2>'"""
    head = name.replace('(anonymous namespace)::', '').split('(', 1)[0]
    if head.startswith('void '):
        head = head[5:]
    return re.sub(r'^(?:\w+::)+', '', head.strip())


def profile_once(fn):
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'trace.json')
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)['traceEvents']
    ks = sorted((e for e in events if e.get('cat') == 'kernel' and 'dtb::' in e['name']), key=lambda e: e['ts'])
    return [(short_name(e['name']), tuple(e['args'].get('grid', ())), tuple(e['args'].get('block', ()))) for e in ks], res


def launches(fn, attempts=6):
    """Run fn() under torch.profiler; returns ([(kernel, grid, block), ...] of this library's kernels (namespace dtb) in
    launch order, fn's result).  Kernels of torch itself (fills of new tensors, copies) are left out.

    Every call profiled here launches at least one kernel of this library, but torch.profiler now and then returns a
    session without any of its device activity (on an H100: 3 of about 320 short sessions, and once several in a
    row for the same call).  Such an empty record says nothing about the dispatch, so the call is profiled again after a
    growing pause; each call allocates its own outputs."""
    for i in range(attempts):
        kernels, res = profile_once(fn)
        if kernels:
            return kernels, res
        time.sleep(0.1 * 2 ** i)
    pytest.fail(f'torch.profiler recorded no kernel of this library in {attempts} sessions of a call that launches one')


def ran(kernels, name):
    """True if `name` ran: an exact kernel name ('fm_linear_fwd_vec<2>') or every instance of a template."""
    return any(k == name or k.startswith(name + '<') for k, _, _ in kernels)
