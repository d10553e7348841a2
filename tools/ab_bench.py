"""Developer A/B probe: BASELINE config 4 on the library named by NHD_B200_LIB (relative to nhd_b200/), device-timed,
L2 flushed between solves; prints one JSON line with the per-phase means and a digest of the bindings, so that builds of
different revisions can be compared in one visit to the GPU box.

    python tools/ab_bench.py [4 | 5 | wild | moving]

`wild` and `moving` are bench.py's side workloads on config 4: heterogeneous NICs, and per-pod clocks."""
import hashlib
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import workload
from nhd_b200.solver import Solver

cfg = sys.argv[1] if len(sys.argv) > 1 else '4'
recs, speed, pods, now = workload.make_workload(4 if cfg in ('wild', 'moving') else int(cfg), wild=cfg == 'wild')
if cfg == 'moving':
    now = now + 0.001 * np.arange(len(pods))
s = Solver(speed)
s.load_nodes(recs)
s.snapshot()
s.stage_batch(pods, now)
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
acc = {'filter_ms': [], 'sweep_ms': [], 'total_ms': []}
for it in range(3 + 12):
    s.restore()
    s.sync()
    flush.zero_()
    torch.cuda.synchronize()
    s.solve_staged()
    s.sync()
    t = s.timing()
    if it >= 3:
        for k in acc:
            acc[k].append(t[k])
b = s.fetch_bindings()
h = hashlib.sha256()
for n in b.dtype.names:
    if n != 'pad_':
        h.update(np.ascontiguousarray(b[n]).tobytes())
print(json.dumps({'lib': os.environ.get('NHD_B200_LIB', 'libnhd_b200.so'), 'config': cfg,
                  **{k: round(float(np.mean(v)), 5) for k, v in acc.items()},
                  'min_total_ms': round(float(np.min(acc['total_ms'])), 5),
                  'decisions_per_s': round(len(pods) / (float(np.mean(acc['total_ms'])) / 1e3)),
                  'placed': int((b['status'] == 0).sum()), 'bindings_sha256': h.hexdigest()[:16]}), flush=True)
s.close()
