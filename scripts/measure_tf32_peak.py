"""Measure the dense TF32 peaks of this GPU for mma.sync and wgmma (csrc/peak_tf32.cuh) and write them as JSON."""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from tntorch_b200 import ops

torch.cuda.set_device(0)
best = 0.0
rows = []
for per_commit in (16, 64, 256):
    tf, ms = ops.measure_tf32_peak(reps=2048 // per_commit * 8, per_commit=per_commit, trials=5)
    rows.append({"per_commit": per_commit, "tflops": tf, "ms": ms})
    best = max(best, tf)
best_wg = 0.0
rows_wg = []
for per_commit in (4, 16, 64):
    tf, ms = ops.measure_wgmma_tf32_peak(reps=1024 // per_commit, per_commit=per_commit, trials=5)
    rows_wg.append({"per_commit": per_commit, "tflops": tf, "ms": ms})
    best_wg = max(best_wg, tf)
out = {"tf32_tflops": best, "runs": rows, "wgmma_tf32_tflops": best_wg, "wgmma_runs": rows_wg,
       "gpu": torch.cuda.get_device_name(0),
       "how": "csrc/peak_tf32.cuh: 2 CTAs per SM, every warp issuing mma.sync.m16n8k8 .tf32 on register operands; "
              "and 1 CTA per SM, two warpgroups issuing wgmma m64n256k8 .tf32 (A in registers, B in shared memory); "
              "best of 5, CUDA events"}
dst = sys.argv[1] if len(sys.argv) > 1 else "tf32_peak.json"
json.dump(out, open(dst, "w"), indent=1)
print(json.dumps(out))
