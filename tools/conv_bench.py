#!/usr/bin/env python
"""Per-layer micro-benchmark of the masked implicit-GEMM kernels on the ResNet-50 layer shapes
(SURVEY.md Appendix A): time, TFLOP/s and effective GB/s per op, against the per-layer roofline
max(FLOPs / tensor peak, bytes / HBM peak)."""
import os, sys, json, statistics
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from turboprune_b200 import ops, _cabi
from bench import peaks

LAYERS = [  # name, cin, cout, k, stride, pad, hw_in, count
    ("l1.1x1 64->64", 64, 64, 1, 1, 0, 56, 1), ("l1.1x1 256->64", 256, 64, 1, 1, 0, 56, 2), ("l1.3x3 64", 64, 64, 3, 1, 1, 56, 3),
    ("l1.1x1 64->256", 64, 256, 1, 1, 0, 56, 4), ("l2.0.c1 256->128", 256, 128, 1, 1, 0, 56, 1), ("l2.0.c2 3x3 s2", 128, 128, 3, 2, 1, 56, 1),
    ("l2.3x3 128", 128, 128, 3, 1, 1, 28, 3), ("l2.1x1 128->512", 128, 512, 1, 1, 0, 28, 4), ("l2.1x1 512->128", 512, 128, 1, 1, 0, 28, 3),
    ("l2.ds 256->512 s2", 256, 512, 1, 2, 0, 56, 1), ("l3.0.c1 512->256", 512, 256, 1, 1, 0, 28, 1), ("l3.0.c2 3x3 s2", 256, 256, 3, 2, 1, 28, 1),
    ("l3.3x3 256", 256, 256, 3, 1, 1, 14, 5), ("l3.1x1 256->1024", 256, 1024, 1, 1, 0, 14, 6), ("l3.1x1 1024->256", 1024, 256, 1, 1, 0, 14, 5),
    ("l3.ds 512->1024 s2", 512, 1024, 1, 2, 0, 28, 1), ("l4.0.c1 1024->512", 1024, 512, 1, 1, 0, 14, 1), ("l4.0.c2 3x3 s2", 512, 512, 3, 2, 1, 14, 1),
    ("l4.3x3 512", 512, 512, 3, 1, 1, 7, 2), ("l4.1x1 512->2048", 512, 2048, 1, 1, 0, 7, 3), ("l4.1x1 2048->512", 2048, 512, 1, 1, 0, 7, 2),
    ("l4.ds 1024->2048 s2", 1024, 2048, 1, 2, 0, 14, 1),
]

def timeit(fn, reps=5):
    fn(); fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return statistics.median(ts)

def main():
    if os.environ.get("TP_KSKIP", "1") == "0":
        ops.set_kblock_skip(False)
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    only = sys.argv[2] if len(sys.argv) > 2 else None
    pk = peaks()                  # the same peaks as bench.py: MEASURED_PEAKS.json when present, else the H100 data sheet
    dev = "cuda"; tot = {"f": 0, "d": 0, "w": 0, "roof": 0}
    print(f"B={B}  {torch.cuda.get_device_name()}  peak {pk['tf_burst']} TF, {pk['hbm']} GB/s ({pk['src_tf']}; {pk['src_hbm']})")
    print(f"{'layer':22s} {'op':5s} {'ms':>8s} {'TF/s':>7s} {'GB/s':>7s} {'roof_ms':>8s} {'x_roof':>6s}")
    for name, cin, cout, k, s, p, hw, cnt in LAYERS:
        if only and only not in name: continue
        x = torch.randn(B, cin, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = torch.randn(cout, cin, k, k, device=dev) * 0.05; m = (torch.rand_like(w) < 0.3).float()
        desc = ops.make_desc(B, hw, hw, cin, cout, k, k, (s, s), (p, p))
        xn = x.permute(0, 2, 3, 1)
        wf, wd = ops.stage_weights(w, m, cin, True, cout)
        y = ops.conv_fprop(desc, xn, wf)
        dy = torch.randn_like(y)
        flops = 2.0 * B * desc.p * desc.q * cout * cin * k * k
        bytes_io = 2.0 * (x.numel() + y.numel())
        roof = max(flops / (pk["tf_burst"] * 1e12), bytes_io / (pk["hbm"] * 1e9)) * 1e3
        for op, fn in (("fprop", lambda: ops.conv_fprop(desc, xn, wf)), ("dgrad", lambda: ops.conv_dgrad(desc, dy, wd)),
                       ("wgrad", lambda: ops.conv_wgrad(desc, xn, dy, m, cin))):
            t = timeit(fn)
            print(f"{name:22s} {op:5s} {t:8.3f} {flops/t/1e9:7.1f} {bytes_io/t/1e6:7.0f} {roof:8.3f} {t/roof:6.2f}", flush=True)
            tot[op[0]] += t * cnt
        tot["roof"] += roof * cnt
    print(f"totals (x count): fprop {tot['f']:.2f} ms dgrad {tot['d']:.2f} ms wgrad {tot['w']:.2f} ms; per-op roofline sum {tot['roof']:.2f} ms")

if __name__ == "__main__":
    main()
