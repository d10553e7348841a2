"""Node-ingest throughput (host side): labels -> packed records, native parser (nhd_ingest_node) against the
Python object path (ParseLabels + SetHugepages + pack_node) of the mirror and, where NHD_REFERENCE_ROOT names a checkout of it, of
the unmodified reference.  python tools/ingest_bench.py [n_nodes]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np                                               # noqa: E402

from nhd_b200 import Node as mirror_node                         # noqa: E402
from nhd_b200 import packing                                     # noqa: E402
from nhd_b200.ingest import LabelIngest                          # noqa: E402
from tests import scenarios                                      # noqa: E402

n_nodes = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
items = []
seed = 0
while len(items) < n_nodes:
    scn = scenarios.random_scenario(60000 + seed, n_nodes=64, n_pods=1, flavor=('mixed', 'vf', 'big')[seed % 3])
    seed += 1
    for nd in scn['nodes']:
        items.append((nd['labels'], nd.get('active', True), nd['hp_alloc'], nd['hp_free']))
items = items[:n_nodes]
avg_labels = sum(len(i[0]) for i in items) / len(items)


def object_path(node_mod):
    layout = packing.ClusterLayout()
    recs = np.zeros(len(items), dtype=packing.wire.NODE_DTYPE)
    t0 = time.perf_counter()
    for i, (labels, active, alloc, free) in enumerate(items):
        n = node_mod.Node(str(i), active)
        n.ParseLabels(labels)
        n.SetHugepages(alloc, free)
        packing.pack_node(n, layout, out=recs[i])
    return time.perf_counter() - t0, recs


ing = LabelIngest()
t0 = time.perf_counter()
recs, kept = ing.nodes(items)
t_native = time.perf_counter() - t0
t_mirror, recs_m = object_path(mirror_node)
assert recs.tobytes() == recs_m.tobytes()
print(f'{n_nodes} nodes, {avg_labels:.1f} labels/node')
print(f'  native nhd_ingest_node (through ctypes): {n_nodes / t_native:10,.0f} nodes/s')
print(f'  mirror Node.ParseLabels + pack_node    : {n_nodes / t_mirror:10,.0f} nodes/s   ({t_mirror / t_native:.1f}x slower)')
try:
    from oracle import ref_loader
    if ref_loader.available():
        ref = ref_loader.load()
        t_ref, recs_r = object_path(ref.node)
        assert recs.tobytes() == recs_r.tobytes()
        print(f'  reference Node.ParseLabels + pack_node : {n_nodes / t_ref:10,.0f} nodes/s   ({t_ref / t_native:.1f}x slower)')
except ImportError:
    pass
