#!/usr/bin/env python
"""Micro-benchmark of the mask top-k path (metric M2): GB/s of algorithmic bytes vs HBM peak."""
import os, sys, statistics
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from turboprune_b200 import ops

def run(n, nseg, density, kind=0, reps=7, flush=True):
    dev = "cuda"
    sizes = [n // nseg] * (nseg - 1); sizes.append(n - sum(sizes))
    ws = [torch.randn(s, device=dev) * (0.01 + 0.002 * i) for i, s in enumerate(sizes)]
    ms = [torch.ones(s, device=dev) for s in sizes]
    gs = [torch.randn(s, device=dev) * 1e-3 for s in sizes] if kind else None
    k = int((1 - density) * n)
    plan = ops.TopKPlan(ws, ms, gs=gs, kind=kind)
    for _ in range(2):
        plan.run(k)
    fl = torch.empty(64 << 20, dtype=torch.float32, device=dev)
    ts = []
    for _ in range(reps):
        if flush: fl.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); plan.enqueue(k); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
        # phase stamps of this call (CTA 0, %globaltimer), read before finish(): its exact fallback reuses the state
        tp = plan.state()["t_phase"]
        _, thr, info = plan.finish(k)
    names = ["P0 sample", "P1 refine", "P2 sweep", "P3 decide", "P4 narrow", "P5 finish"]
    ph = ", ".join(f"{n} {(tp[i + 1] - tp[i]) / 1e3:.1f}" for i, n in enumerate(names) if tp[i + 1] > tp[i] > 0)
    t = statistics.median(ts); bpe = 12 if kind == 0 else 16
    print(f"   phases (us, CTA 0, incl. the barrier that ends each): {ph}")
    print(f"N={n} segs={nseg} density={density} kind={kind}: {t*1e3:.1f} us  {bpe*n/t/1e6:.0f} GB/s  info={info}", flush=True)

if __name__ == "__main__":
    run(25_502_912, 54, 0.2)
    run(25_502_912, 54, 0.8)
    run(134_657_728, 16, 0.05, kind=2)
    run(11_164_352, 21, 0.8)
