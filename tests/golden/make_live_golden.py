"""Freeze what the UNMODIFIED reference computes for the differential tests that compare this package with it
(test_oracle_vs_reference, test_scheduler, test_codec, test_ingest, test_rpc) into tests/golden/live/*.json.gz, so
that those tests run anywhere.  Each file holds, in the order the test walks its cases, exactly what the test
compares against.  A scheduler session's end state is large (mostly the Kubernetes event log): it is kept as a
summary — the binds Kubernetes saw and the failed-scheduling count — and a SHA-256 fingerprint of the whole
canonical JSON (``fingerprint``), so a failing comparison still names the first bind that differs.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_live_golden.py [oracle sched codec ingest rpc]
"""
import contextlib
import gzip
import hashlib
import io
import json
import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

LIVE = os.path.join(ROOT, 'tests', 'golden', 'live')


def fingerprint(doc):
    return hashlib.sha256(json.dumps(doc, sort_keys=True).encode()).hexdigest()


def session_summary(doc):
    """The binds and the failed-scheduling count of a scheduler session's end-state document."""
    return json.loads(json.dumps({'binds': doc['k8s']['binds'], 'failed_schedule_count': doc['failed_schedule_count']}))


def load(name):
    with gzip.open(os.path.join(LIVE, name + '.json.gz'), 'rt') as f:
        return json.load(f)


def _save(name, doc):
    os.makedirs(LIVE, exist_ok=True)
    path = os.path.join(LIVE, name + '.json.gz')
    with gzip.GzipFile(path, 'wb', mtime=0) as f:
        f.write(json.dumps(doc, sort_keys=True).encode())
    print(name, os.path.getsize(path) // 1024, 'KiB')


# ---- the case streams, shared by the tests and this generator ---------------------------------------------------
def oracle_scenarios(flavor):
    from tests import scenarios
    off = {'mixed': 1, 'wild': 2, 'vf': 3, 'big': 4}[flavor] * 100003
    return [scenarios.random_scenario(seed * 7 + off, n_nodes=6, n_pods=30, flavor=flavor) for seed in range(30)]


def near_limit_scenarios():
    from tests import scenarios
    out = []
    for seed in range(3):
        scn = scenarios.huge_scenario(81000 + seed, min_busy_secs=30.0 if seed % 3 else 0.0)
        scn['nodes'], scn['pods'], scn['now'] = scn['nodes'][:5], scn['pods'][:14], scn['now'][:14]
        out.append(scn)
    return out


def ingest_node_scenarios():
    from tests import scenarios
    return [scenarios.random_scenario(4242 + seed, n_nodes=5, n_pods=1, flavor='wild' if seed % 2 else 'vf')
            for seed in range(40)]


def node_description(n):
    """What ParseLabels makes of a node's labels, as plain data."""
    return json.loads(json.dumps({
        'cores': [(c.core, c.socket, c.sibling, c.used) for c in n.cores],
        'gpus': [(g.device_id, g.numa_node, g.pciesw, g.gtype.value) for g in n.gpus],
        'nics': [(x.ifname, x.mac, x.speed, x.numa_node, x.pciesw, x.idx, x.card, x.port) for x in n.nics],
        'misc': (n.groups, n.maintenance, n.data_vlan, n.gwip, n.mem.free_hugepages_gb, n.reserved_cores,
                 n.sockets, n.numa_nodes, n.smt_enabled, n.cores_per_proc)}))


def sched_scripts(flavor):
    from tests import sched_harness as H
    return [H.random_script(seed, flavor, codec='triad' if seed % 2 else 'json') for seed in range(100, 112)]


def codec_stream():
    """(seed, text, broken variants or []) of the codec comparison."""
    from tests import triad_cfg as T
    from tests.test_codec import broken_variants
    rng = np.random.default_rng(77)
    out = []
    for seed in range(120):
        pod = T.codec_pod(rng, 'wild' if seed % 2 else 'mixed')
        text = T.pod_to_cfg(pod, rng, gpu_type=[None, 'V100', 'bogus'][seed % 3])
        out.append((seed, text, broken_variants(text, rng) if seed % 4 == 0 else []))
    return out


def stats_scenarios():
    from tests import scenarios
    return [scenarios.random_scenario(45000 + seed, n_nodes=8, n_pods=30, flavor=flavor)
            for seed, flavor in enumerate(['mixed', 'wild', 'vf', 'big', 'mixed', 'big'])]


RPC_NODE_ROWS = [{'name': 'n0', 'freegpu': 3, 'totalgpu': 8, 'freecpu': 40, 'totalcpu': 96, 'freehuge_gb': 20,
                  'totalhuge_gb': 64, 'totalpods': 3, 'active': True, 'nicstats': [[10, 20], [0, 0]]},
                 {'name': 'n1', 'freegpu': 0, 'totalgpu': 0, 'freecpu': 0, 'totalcpu': 64, 'freehuge_gb': 0,
                  'totalhuge_gb': 32, 'totalpods': 0, 'active': False, 'nicstats': []}]
RPC_POD_ROWS = [{'namespace': 'prod', 'podname': 'p0', 'node': 'n0', 'annotations': {'a': 'b', 'sigproc.viasat.io/x': 'y'},
                 'hugepages': 4, 'proc_cores': [3, 4, 5], 'proc_helper_cores': [6], 'misc_cores': [7, 8], 'gpus': [0, 2],
                 'nics': ['0C:42:A1:00:00:01']}]
RPC_ANSWERS = {'TYPE_NODE_INFO': RPC_NODE_ROWS, 'TYPE_SCHEDULER_INFO': 17, 'TYPE_POD_INFO': RPC_POD_ROWS}
RPC_CALLS = ('GetBasicNodeStats', 'GetSchedulerStats', 'GetPodStats')


# ---- generation (needs the reference) ---------------------------------------------------------------------------
def _records(scn):
    from tests import ref_compare
    outs, init, final, _, _ = ref_compare.run_reference(scn)
    return {'outs': outs, 'init': init.tobytes().hex(), 'final': final.tobytes().hex()}


def make_oracle():
    from oracle import ref_loader
    from tests import scenarios
    ref = ref_loader.load()
    doc = {f: [_records(s) for s in oracle_scenarios(f)] for f in ('mixed', 'wild', 'vf', 'big')}
    doc['near_limits'] = [_records(s) for s in near_limit_scenarios()]
    doc['nic_fp64'] = [_records(s) for s in scenarios.nic_bandwidth_scenarios()]
    doc['node_descriptions'] = [{name: node_description(n) for name, n in scenarios.build_nodes(s, ref.node).items()}
                                for s in ingest_node_scenarios()]
    _save('oracle', doc)


def make_sched():
    from tests import helpers, sched_harness as H
    doc = {}
    for flavor in ('mixed', 'vf', 'big', 'wild'):
        doc[flavor] = []
        for script in sched_scripts(flavor):
            want = H.run_reference(script)
            stats = {}
            H.run_mirror(script, solver_factory=helpers.OracleSolver, stats=stats)
            names = sorted(stats['assign_failed_nodes'])
            want = H.drop_speed_residue(want, names)
            doc[flavor].append({'fingerprint': fingerprint(want), 'summary': session_summary(want),
                                'assign_failed_nodes': names})
    _save('sched', doc)


def make_codec():
    from oracle import ref_sched_loader
    from tests.test_codec import run_case
    Ref = ref_sched_loader.load_codec().codec.TriadCfgParser
    doc = []
    for seed, text, broken in codec_stream():
        want = run_case(Ref, text, False, seed)
        want2 = run_case(Ref, want['cfg'], True, seed)
        doc.append({'seed': seed, 'parsed': want, 'reread': want2,
                    'broken': [run_case(Ref, bad, False, seed) for bad in broken]})
    _save('codec', doc)


def make_ingest():
    from nhd_b200 import packing
    from oracle import ref_loader
    from tests import scenarios
    from tests.golden import make_ingest_golden as mk
    from tests.test_ingest import _object_path, _stats_of_objects
    ref = ref_loader.load()
    layout = packing.ClusterLayout()
    fuzz = []
    for case in mk.mutations(random.Random(5), 400):
        kind, rec, n = _object_path(ref.node, case, layout)
        e = {'kind': kind}
        if kind == 'ok':
            e.update(record=rec.tobytes().hex(), data_vlan=n.data_vlan, res_hugepages_gb=n.mem.res_hugepages_gb,
                     n_reserved_cores=len(n.reserved_cores), gpu_device_id=[g.device_id for g in n.gpus],
                     nic_ifname=[x.ifname for x in n.nics])
        fuzz.append(e)
    stats = []
    for scn in stats_scenarios():
        nodes = scenarios.build_nodes(scn, ref.node)
        matcher = ref.matcher.Matcher()
        for pod, t in zip(scn['pods'], scn['now']):
            top = scenarios.build_top(pod, ref.cfg)
            with contextlib.redirect_stdout(io.StringIO()):
                ref_loader.attempt_scheduling(ref, matcher, nodes, top, pod['groups'], t)
        order = list(nodes.values())
        stats.append({'records': packing.pack_nodes(order, packing.ClusterLayout()).tobytes().hex(),
                      'rows': _stats_of_objects(order)})
    _save('ingest', json.loads(json.dumps({'fuzz': fuzz, 'speed_table': layout.speed_table().tolist(),
                                           'stats': stats})))


def make_rpc():
    from queue import Queue
    from nhd_b200 import NHDRpcServer as R
    from oracle import ref_loader
    from tests.test_rpc import _feeder, _proto_fields
    ref_loader.load()
    with open(os.path.join(ref_loader.REFERENCE_ROOT, 'nhd', 'proto', 'nhd_stats.proto')) as f:
        proto = json.loads(json.dumps(_proto_fields(f.read())))
    stub_pb = types.ModuleType('nhd.proto.nhd_stats_pb2')
    for k in dir(R.nhd_stats_pb2):
        if not k.startswith('_'):
            setattr(stub_pb, k, getattr(R.nhd_stats_pb2, k))
    stub_grpc = types.ModuleType('nhd.proto.nhd_stats_pb2_grpc')
    stub_grpc.NHDControlServicer = object
    stub_grpc.add_NHDControlServicer_to_server = R.add_NHDControlServicer_to_server
    pkg = types.ModuleType('nhd.proto')
    pkg.__path__ = []
    pkg.nhd_stats_pb2, pkg.nhd_stats_pb2_grpc = stub_pb, stub_grpc
    sys.modules.update({'nhd.proto': pkg, 'nhd.proto.nhd_stats_pb2': stub_pb, 'nhd.proto.nhd_stats_pb2_grpc': stub_grpc})
    import nhd.NHDRpcServer as ref_rpc
    responses = {}
    for call in RPC_CALLS:
        q = Queue()
        _feeder(q, RPC_ANSWERS, 1)
        responses[call] = getattr(ref_rpc.NHDRpcHandler(q), call)(R.nhd_stats_pb2.Empty(), None) \
            .SerializeToString(deterministic=True).hex()
    q = Queue()
    _feeder(q, {'TYPE_NODE_INFO': [dict(RPC_NODE_ROWS[0], nicstats=[[22.5, 0]])]}, 1)
    try:
        ref_rpc.NHDRpcHandler(q).GetBasicNodeStats(R.nhd_stats_pb2.Empty(), None)
        fractional_gbps = 'answers'
    except (TypeError, ValueError):
        fractional_gbps = 'raises'
    _save('rpc', {'proto': proto, 'responses': responses, 'fractional_gbps': fractional_gbps})


MAKERS = {'oracle': make_oracle, 'sched': make_sched, 'codec': make_codec, 'ingest': make_ingest, 'rpc': make_rpc}


def main(names):
    from oracle import ref_loader
    if not ref_loader.available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    for name in names or MAKERS:
        MAKERS[name]()


if __name__ == '__main__':
    main(sys.argv[1:])
