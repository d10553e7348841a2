"""Deterministic clusters and pod streams in which pods find no node for every reason the explanations name
(``NHD_WHY_*``, include/nhd_b200.h): node groups the pod lacks, inactive and maintenance nodes, a hugepage shortage,
GPU pods inside a node's busy window (constant and moving clock), too few GPUs, CPU cores or NIC bandwidth, PCI-switch
pruning, and nodes whose GPU and NIC stages pass on disjoint NUMA nodes so that only the intersection fails.
Scenario format: tests/scenarios.py."""
from tests.scenarios import make_group, make_node, make_pod

G100 = 100000                                     # Mb/s: 90 Gb/s usable per NIC (NIC_BW_AVAIL_PERCENT)


def _cluster(tag):
    nic2 = [('eth0', G100, 0, 0x10), ('eth1', G100, 1, 0x20)]
    gpu4 = [(0, 0, 0x10), (1, 0, 0x10), (2, 1, 0x20), (3, 1, 0x20)]
    return [
        make_node(f'{tag}gpu', gpus=gpu4, nics=nic2),                                   # takes the first GPU pod
        make_node(f'{tag}other', gpus=gpu4, nics=nic2, groups=['grp3']),                # shares no group
        make_node(f'{tag}cordon', gpus=gpu4, nics=nic2, active=False),                  # not active
        make_node(f'{tag}maint', gpus=gpu4, nics=nic2, maintenance=True),               # in maintenance
        make_node(f'{tag}lowhp', gpus=gpu4, nics=nic2, hp_free=2),                      # 2 GB hugepages free
        make_node(f'{tag}cpu', phys_cores=8, smt=False, reserved_per_socket=1, nics=nic2),   # 3 free cores a socket
        make_node(f'{tag}down', gpus=gpu4, nics=[('eth0', 0, 0, 0x10), ('eth1', 0, 1, 0x20)]),   # links down: 0 Gb/s
        make_node(f'{tag}pcisw', gpus=[(0, 0, 0x30), (1, 1, 0x40)], nics=nic2),         # GPUs behind other switches
        make_node(f'{tag}split', gpus=[(0, 0, 0x10), (1, 0, 0x10)], nics=[('eth0', G100, 1, 0x20)]),  # GPUs on 0, NIC on 1
        make_node(f'{tag}onegpu', gpus=[(0, 0, 0x10)], nics=nic2),
    ]


def _pods():
    gpu2 = make_pod([make_group(gpus=(1, 1))], hugepages=1)                # placed on the first GPU node
    gpu2_pci = make_pod([make_group(gpus=(1, 1))], hugepages=4, map_type='PCI')
    gpu1 = make_pod([make_group(gpus=(1,))], hugepages=1)
    cpu_big = make_pod([make_group(workers=20)], misc=1)                   # 22 cores on one socket (14 free)
    nic_big = make_pod([make_group(pairs=((95, 10),))])                    # 95 Gb/s on one NIC
    two_grp = make_pod([make_group(gpus=(1,)), make_group(pairs=((60, 60),))], hugepages=1)
    return [gpu2, gpu2_pci, gpu1, cpu_big, nic_big, two_grp, gpu2_pci, cpu_big, gpu1, nic_big]


def oversized_tail(pods, n):
    """``n`` packed pods made from ``pods`` that no node of the BASELINE clusters (at most 32 cores a socket, 8 GPUs,
    128 GB of hugepages, NICs of at most 100 Gb/s) can take, each for a different stage: 70 cores in one group,
    10 Tb/s on one NIC, 1 TB of hugepages, or 16 GPUs."""
    import numpy as np
    from nhd_b200 import wire
    out = np.array([pods[k % len(pods)] for k in range(n)], dtype=wire.POD_DTYPE)
    for k in range(n):
        p = out[k]
        if k % 4 == 0:
            p['n_groups'], p['n_misc'] = 1, 2
            g = p['groups'][0]
            g['n_gpus'], g['n_proc'], g['n_helpers'], g['flags'] = 0, 70, 0, 0
        elif k % 4 == 1:
            p['groups'][0]['rx_gbps'] = 10000.0
        elif k % 4 == 2:
            p['hugepages_gb'] = 1000
        else:
            p['n_groups'], p['n_misc'] = 2, 1
            for g in (0, 1):
                grp = p['groups'][g]
                grp['n_gpus'], grp['n_proc'], grp['n_helpers'], grp['flags'] = 8, 1, 0, 0
                grp['gpu_feeders'][:] = 0
                grp['rx_gbps'] = grp['tx_gbps'] = 0.0
    return out


def explain_scenarios():
    out = []
    for k, (clock, busy) in enumerate([('const', 30.0), ('moving', 30.0), ('moving', 12.0), ('const', 0.0)]):
        pods = _pods()
        now = [5000.0] * len(pods) if clock == 'const' else [5000.0 + 3.0 * i for i in range(len(pods))]
        out.append({'nodes': _cluster(f's{k}'), 'pods': pods, 'now': now, 'min_busy_secs': busy})
    # several node-group lists in one batch
    pods = _pods()
    for i, p in enumerate(pods):
        p['groups'] = ['grp3'] if i % 3 == 1 else ['default', 'grp5']
    out.append({'nodes': _cluster('g'), 'pods': pods, 'now': [7000.0 + i for i in range(len(pods))],
                'min_busy_secs': 30.0})
    return out
