#!/usr/bin/env python
"""Per-kernel time table of one training step (torch profiler, CUDA activities): python tools/profile_step.py [flux_lora|sd3_fullft]"""
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "sd3_fullft"
dev = torch.device("cuda", 0)
from simpletuner_b200.training.optim import AdamWBF16  # noqa: E402
from simpletuner_b200.training.step import TrainStep  # noqa: E402

if cfg == "sd3_fullft":
    w = bench.build_sd3_fullft(dev)
    batches = [bench.synth_batch_sd3(8, dev, hw, seed=i) for i, hw in enumerate(bench.SD3_BUCKETS[:2])]
else:
    w = bench.build_model(dev)
    batches = [bench.synth_batch(1, dev, seed=i) for i in range(2)]   # the bench's flux_lora default batch
params = [p for p in w._denoiser().parameters() if p.requires_grad]
opt = AdamWBF16(params, lr=1e-4, weight_decay=1e-2, eps=1e-6, seed=1)
step = TrainStep(w, opt)
for i in range(3):
    step(dict(batches[i % 2]))
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for i in range(2):
        step(dict(batches[i % 2]))
    torch.cuda.synchronize()
rows = sorted(prof.key_averages(), key=lambda e: -e.device_time_total)
tot = sum(e.device_time_total for e in rows)
print(f"total device time {tot / 2e3:.2f} ms per step, {sum(e.count for e in rows) // 2} kernels per step")
for e in rows[:45]:
    print(f"{e.device_time_total / 2e3:9.3f} ms {100 * e.device_time_total / tot:5.1f}%  n={e.count // 2:5d}  avg {e.device_time_total / e.count:8.1f} us  {e.key[:110]}")
