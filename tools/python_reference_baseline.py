"""The reference's own Python path timed on the BASELINE workloads (BASELINE.md section 3): the unmodified
nhd/Matcher.py + nhd/Node.py, driven like NHDScheduler.AttemptScheduling, one thread, on the first pods of the stream
at full cluster size.  Needs a checkout of the reference named by NHD_REFERENCE_ROOT; bench.py adds the same number
to its line only where that variable is set.

    python tools/python_reference_baseline.py [config] [n_pods]
"""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import workload
from nhd_b200 import packing
from oracle import binding, ref_loader
from tests import pyref

cfg = int(sys.argv[1]) if len(sys.argv) > 1 else 4
n_pods = int(sys.argv[2]) if len(sys.argv) > 2 else 8
recs, speed, pods, now = workload.make_workload(cfg)
ob, _ = binding.solve(recs, speed, pods[:n_pods], now[:n_pods], threads=os.cpu_count() or 1)
# the Node objects rebuilt from labels pack back into the very records the GPU run uses
ref = ref_loader.load()
n_probe = min(64, len(recs))
probe = pyref.nodes_from_records(recs[:n_probe], speed, ref.node)
layout = packing.ClusterLayout()
layout.speed_class(100.0)
back = packing.pack_nodes(list(probe.values()), layout)
assert all(back[i]['used'].tolist() == recs[i]['used'].tolist() and back[i]['nic_inuse'] == recs[i]['nic_inuse']
           and back[i]["gpu_used"] == recs[i]["gpu_used"] for i in range(n_probe)), 'label round trip differs'
out = pyref.time_reference(recs, speed, pods[:n_pods], now[:n_pods], check_against=ob)
out['config'] = f'BASELINE config {cfg}: {len(recs)} nodes'
print(json.dumps(out))
