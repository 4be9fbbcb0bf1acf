"""Times one detector conv-stack forward (CUDA events around the graph replay, L2 flushed between replays).
usage: python scripts/time_yolo.py [model] [--eager]   (FM_CONV_TMA=0 puts every conv on the cp.async kernel)"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastmot_b200 import models  # noqa: E402
from fastmot_b200.engine import build_yolo_engine  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith('-') else 'YOLOv4CSP'
eager = "--eager" in sys.argv
model = models.YOLO.get_model(name)
eng = build_yolo_engine(model, use_graph=not eager)
x = torch.rand(*eng.inp.shape, device='cuda').half()
x[..., 3:] = 0
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for _ in range(2 if eager else 5):
    eng.forward(x)
torch.cuda.synchronize()
ts = []
for _ in range(2 if eager else 20):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.forward(x)
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1))
ts.sort()
med = ts[len(ts) // 2]
print(f"{name} tma={os.environ.get('FM_CONV_TMA', '1')} "
      f"convs tc={eng.n_tc} (tma {eng.n_tma}) simt={eng.n_simt} kernels={eng.kernels_per_replay()}: "
      f"median {med:.3f} ms  min {ts[0]:.3f}  max {ts[-1]:.3f}  {eng.flops / med / 1e9:.1f} TFLOP/s")
