"""The whole stack on one screen: a synthetic cluster behind a fake Kubernetes manager, pods carrying real Triad
libconfig text, `nhd_b200.NHDScheduler` batching the pending set through the solver, the rewritten config of one pod,
and the gRPC statistics service answering a client.  Developer tool.

    python tools/demo_cluster.py             # on the GPU (CUDA solver)
    python tools/demo_cluster.py --emulated  # anywhere: the same kernels on the CPU emulation of tests/emu
"""
import os
import sys
import threading
import time
from queue import Empty, Queue

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if '--emulated' in sys.argv:
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    import build_emu_cuda
    os.environ['NHD_B200_LIB'] = build_emu_cuda.build()
    os.environ['NHD_B200_ALLOW_EMULATED'] = '1'
    os.environ.setdefault('EMU_LANE_ORDER', 'd')

import grpc                                              # noqa: E402
import numpy as np                                       # noqa: E402

from nhd_b200 import NHDRpcServer as R                   # noqa: E402
from nhd_b200.NHDScheduler import NHDScheduler           # noqa: E402
from nhd_b200.TriadCfgParser import TriadCfgParser       # noqa: E402
from tests import fake_k8s, scenarios         # noqa: E402


def main():
    rng = np.random.default_rng(7)
    nodes = []
    for i in range(64):
        gpu = i % 2 == 0
        nodes.append(scenarios.make_node(
            f'node{i:02d}', 2, 32, True, 2,
            gpus=[(d, d // 4, 0x10 * (d // 2 + 1)) for d in range(8)] if gpu else (),
            nics=[('eth0', 100000, 0, 0x10), ('eth1', 100000, 1, 0x30)], hp_alloc=64))
    k8s = fake_k8s.FakeK8s(nodes, codec='triad')
    for i in range(200):
        gpu = rng.random() < 0.5
        g = scenarios.make_group(pairs=((10, 10), (10, 5)), workers=int(rng.integers(1, 4)), gpus=(1,) if gpu else (),
                                 helpers=int(rng.integers(0, 2)))
        k8s.add_pod('prod', f'pod{i:03d}', scenarios.make_pod([g], misc=1, hugepages=2, map_type='PCI' if gpu else 'NUMA'),
                    uid=f'u{i}')
    rpcq = Queue()
    sched = NHDScheduler(k8s, lambda cfgtype, cfgstr: TriadCfgParser(cfgstr, False), rpcq=rpcq, stats_from_device=True)
    t0 = time.perf_counter()
    sched.Startup()                                      # BuildInitialNodeList + LoadDeployedConfigs + CheckPendingPods
    dt = time.perf_counter() - t0
    c = sched.cluster
    print(f'{len(k8s.binds)} of {len(k8s.pods)} pods bound on {len(nodes)} nodes in {dt * 1e3:.0f} ms '
          f'({c.batches} solver batch(es), {c.full_loads} full upload, {c.delta_nodes} delta records)')
    ns, name, node = k8s.binds[0]
    text = k8s.pods[(ns, name)]['annotations'][fake_k8s.CFG_ANNOTATION]
    print(f'\n{ns}/{name} -> {node}; its rewritten config starts:\n' + '\n'.join(text.splitlines()[:14]) + '\n    ...')

    stop = threading.Event()

    def serve_rpc():
        while not stop.is_set():
            try:
                item = rpcq.get(True, 0.05)
            except Empty:
                continue
            sched.ParseRPCReq(item[0], item[1])
    threading.Thread(target=serve_rpc, daemon=True).start()
    srv = R.NHDRpcServer(rpcq, listen='127.0.0.1:0')
    srv.start()
    srv.ready.wait(10)
    with grpc.insecure_channel(f'127.0.0.1:{srv.port}') as ch:
        stub = R.NHDControlStub(ch)
        st = stub.GetBasicNodeStats(R.nhd_stats_pb2.Empty(), timeout=10)
        print(f'\ngRPC GetBasicNodeStats on 127.0.0.1:{srv.port} (node counters read from the solver\'s records):')
        for n in list(st.info)[:4]:
            print(f'  {n.name}: cpus {n.free_cpus} free / {n.used_cpus} used, gpus {n.free_gpus}/{n.used_gpus}, '
                  f'hugepages {n.free_hugepages}/{n.used_hugepages} GB, pods {n.total_pods}')
        print('  failed_schedule_count =', stub.GetSchedulerStats(R.nhd_stats_pb2.Empty(), timeout=10).failed_schedule_count)
    stop.set()
    srv.stop()
    sched.close()


if __name__ == '__main__':
    main()
