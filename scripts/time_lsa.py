"""Times fm_lsa on tracker-like and random 200x200 cost matrices (CUDA events, median of 20).
usage: python scripts/time_lsa.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastmot_b200 import _lib  # noqa: E402
from fastmot_b200.devmem import ptr, stream_ptr  # noqa: E402

lib = _lib.require_device()
rng = np.random.default_rng(0)


def bench(C, name):
    nr, nc = C.shape
    c = torch.as_tensor(np.ascontiguousarray(C)).cuda()
    out = torch.zeros(nr, dtype=torch.int32, device="cuda")
    st = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(max(int(lib.fm_lsa_workspace_bytes(nr, nc)), 16), dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(25):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lib.fm_lsa(ptr(c), nr, nc, ptr(out), ptr(st), ptr(ws), stream_ptr())
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts = sorted(ts[5:])
    from scipy.optimize import linear_sum_assignment
    import time
    t0 = time.perf_counter()
    for _ in range(20):
        linear_sum_assignment(C)
    sp = (time.perf_counter() - t0) / 20 * 1e6
    print(f"{name:28s} {nr}x{nc}: gpu median {ts[len(ts) // 2]:8.1f} us  min {ts[0]:8.1f}   scipy (this host) {sp:8.1f} us")


n = 200
C = rng.uniform(0.3, 1.0, (n, n))
C[np.arange(n), rng.permutation(n)] = rng.uniform(0, 0.1, n)
bench(C, "tracker-like (1 good / row)")
G = np.full((n, n), 1e5)
perm = rng.permutation(n)
for i in range(n):
    G[i, perm[i]] = rng.uniform(0, 0.3)
    for jj in rng.choice(n, 3, replace=False):
        G[i, jj] = min(G[i, jj], rng.uniform(0.3, 0.8))
bench(G, "gated (1e5 outside the gate)")
bench(rng.uniform(0, 1, (n, n)), "uniform random")
bench(rng.uniform(0, 1, (200, 177)), "uniform random")
bench(rng.uniform(0, 1, (64, 64)), "uniform random")
