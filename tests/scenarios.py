"""Synthetic clusters and pod streams as plain data (JSON-able), plus builders that turn
them into reference-shaped objects using EITHER the reference's own classes
(nhd.Node / nhd.CfgTopology, build container only) or this repo's mirrors.

A scenario is
    {'nodes': [{'name', 'labels', 'hp_alloc', 'hp_free', 'active'}...],
     'pods':  [{'groups', 'map_type', 'misc', 'misc_smt', 'hugepages',
                'proc_groups': [{'pairs': [[rx, tx]...], 'workers', 'gpus': [feeders...],
                                 'helpers', 'proc_smt', 'helper_smt'}...]}...],
     'now':   [float per pod],
     'min_busy_secs': float}
Node labels use the NFD formats ``Node.ParseLabels`` reads (nhd/Node.py:327-454); pods
are built the way ``TriadCfgParser.ParseModGroups`` does (nhd/TriadCfgParser.py:134-304).
"""
import zlib

import numpy as np

NFD = 'feature.node.kubernetes.io/'
GROUP_NAMES = ['default'] + [f'grp{i}' for i in range(15)]


# ----------------------------------------------------------------------------------
# node label generation
# ----------------------------------------------------------------------------------
def _ranges(ids):
    """sorted ids -> "a-b,c-d" cpuset string"""
    ids = sorted(ids)
    out, i = [], 0
    while i < len(ids):
        j = i
        while j + 1 < len(ids) and ids[j + 1] == ids[j] + 1:
            j += 1
        out.append(f'{ids[i]}-{ids[j]}' if j > i else f'{ids[i]}')
        i = j + 1
    return ','.join(out)


def make_node(name, sockets=2, phys_cores=32, smt=True, reserved_per_socket=2, gpus=(), nics=(),
              sriov_pfs=(), groups=None, hp_alloc=64, hp_free=None, active=True, maintenance=False,
              isol=True, vlan=100, res_hugepages=None, isolcpus=None):
    """gpus: [(device_id, numa, pciesw)], nics: [(ifname, mbps, numa, pciesw)] in label order."""
    labels = {NFD + 'nfd-extras-cpu.numSockets': str(sockets),
              NFD + 'nfd-extras-cpu.num_cores': str(phys_cores)}
    if smt:
        labels[NFD + 'cpu-hardware_multithreading'] = 'true'
    if isolcpus is not None:
        labels[NFD + 'nfd-extras-cpu.isolcpus'] = isolcpus
    elif isol:
        per = phys_cores // sockets
        iso = []
        for s in range(sockets):
            iso += list(range(s * per + reserved_per_socket, (s + 1) * per))
        if smt:
            iso += [c + phys_cores for c in iso]
        # the reference splits on '_' then parses "a-b,c" (Node.py:356-359)
        labels[NFD + 'nfd-extras-cpu.isolcpus'] = _ranges(iso).replace(',', '_')
    for dev, numa, sw in gpus:
        labels[NFD + f'nfd-extras-gpu.{dev}.V100.{numa}.{sw:x}'] = 'true'
    for pf in sriov_pfs:
        labels[NFD + f'nfd-extras-sriov.x.{pf}'] = 'true'
    for i, (ifname, mbps, numa, sw) in enumerate(nics):
        mac = f'{0x0c42a1000000 + (zlib.crc32(name.encode()) % 65536) * 256 + i:012x}'
        speed = f'{mbps}Mbs' if mbps else 'down'
        labels[NFD + f'nfd-extras-nic.{ifname}.mlx.{mac}.{speed}.{numa}.{sw:x}.{i + 1:x}.0'] = 'true'
    labels['DATA_PLANE_VLAN'] = str(vlan)
    labels['DATA_DEFAULT_GW'] = '10.1.0.1/24'
    if groups is not None:
        labels['NHD_GROUP'] = '.'.join(groups)
    if maintenance:
        labels['sigproc.viasat.io/maintenance'] = 'draining'
    if res_hugepages is not None:
        labels['RES_HUGEPAGES_GB'] = str(res_hugepages)
    return {'name': name, 'labels': labels, 'hp_alloc': hp_alloc,
            'hp_free': hp_alloc if hp_free is None else hp_free, 'active': active}


def make_pod(proc_groups, misc=1, misc_smt=False, map_type='NUMA', hugepages=0, groups=('default',)):
    return {'groups': list(groups), 'map_type': map_type, 'misc': misc, 'misc_smt': misc_smt,
            'hugepages': hugepages, 'proc_groups': proc_groups}


def make_group(pairs=((10, 10),), workers=1, gpus=(), helpers=0, proc_smt=False, helper_smt=False):
    return {'pairs': [list(p) for p in pairs], 'workers': workers, 'gpus': list(gpus),
            'helpers': helpers, 'proc_smt': proc_smt, 'helper_smt': helper_smt}


# ----------------------------------------------------------------------------------
# object builders (cfg_mod / node_mod are the reference's modules or this repo's mirrors)
# ----------------------------------------------------------------------------------
def build_nodes(scn, node_mod):
    nodes = {}
    for nd in scn['nodes']:
        n = node_mod.Node(nd['name'], nd.get('active', True))
        if not n.ParseLabels(nd['labels']):
            raise ValueError(f'labels of {nd["name"]} rejected')
        n.SetHugepages(nd['hp_alloc'], nd['hp_free'])
        nodes[nd['name']] = n
    return nodes


def build_top(pod, cfg_mod):
    C = cfg_mod
    top = C.CfgTopology()
    top.SetTopMapType(pod['map_type'])
    top.SetMiscCoreSmt(C.SMTSetting.SMT_ENABLED if pod['misc_smt'] else C.SMTSetting.SMT_DISABLED)
    top.SetCtrlVlan(C.VLANInfo('ctrl_vlan', 0))
    top.hugepages_gb = pod['hugepages']
    none, rx, tx = (C.NICCoreDirection.NIC_CORE_DIRECTION_NONE, C.NICCoreDirection.NIC_CORE_DIRECTION_RX,
                    C.NICCoreDirection.NIC_CORE_DIRECTION_TX)
    grp = C.NUMASetting.LOGICAL_NUMA_GROUP
    for i in range(pod['misc']):
        top.AddMiscCore(C.Core(f'ext{i}', 0, none, C.NUMASetting.LOGICAL_NUMA_DONT_CARE, -1))
    for gi, g in enumerate(pod['proc_groups']):
        pg = C.ProcGroup()
        pg.SetHelperSmt(C.SMTSetting.SMT_ENABLED if g['helper_smt'] else C.SMTSetting.SMT_DISABLED)
        pg.SetProcSmt(C.SMTSetting.SMT_ENABLED if g['proc_smt'] else C.SMTSetting.SMT_DISABLED)
        for h in range(g['helpers']):
            pg.AddMiscCore(C.Core(f'm{gi}.h{h}', 0, none, grp, -1))
        pg.SetDataVlan(C.VLANInfo(f'm{gi}.vlan', 0))
        for pi, (r, t) in enumerate(g['pairs']):
            rxc = C.Core(f'm{gi}.rx{pi}', r, rx, grp, -1)
            pg.AddGroupCore(rxc)
            txc = C.Core(f'm{gi}.tx{pi}', t, tx, grp, -1)
            pg.AddGroupCore(txc)
            top.AddNicPairing(rxc, txc)
        for w in range(g['workers']):
            pg.AddGroupCore(C.Core(f'm{gi}.w{w}', 0, none, grp, -1))
        for di, feeders in enumerate(g['gpus']):
            clist = [C.Core(f'm{gi}.g{di}.c{k}', 0, none, grp, -1) for k in range(feeders)]
            pg.AddGroupGPU(C.GPU(clist, [f'm{gi}.g{di}.dev'] * feeders, C.GpuType.GPU_TYPE_ALL, -1))
        top.proc_groups.append(pg)
    return top


def extract_result(top):
    """Everything SetPhysicalIdsFromMapping wrote into the topology, canonical order."""
    cores, gpus, macs, vlans = [], [], [], []
    for pg in top.proc_groups:
        for g in pg.group_gpus:
            gpus.append(g.device_id)
            cores += [c.core for c in g.cpu_cores]
        cores += [c.core for c in pg.proc_cores]
        cores += [c.core for c in pg.misc_cores]
        vlans.append(pg.vlan.vlan)
    cores += [c.core for c in top.misc_cores]
    macs = [p.mac for p in top.nic_core_pairing]
    return {'cores': cores, 'gpus': gpus, 'macs': macs, 'vlans': vlans,
            'ctrl_vlan': top.ctrl_vlan.vlan, 'gw': top.data_default_gw}


def node_state(node):
    """Mutable state of a Node object as plain data."""
    return {'used': [i for i, c in enumerate(node.cores) if c.used],
            'gpu_used': [i for i, g in enumerate(node.gpus) if g.used],
            'pods_used': [n.pods_used for n in node.nics],
            'speed_used': [[float(n.speed_used[0]), float(n.speed_used[1])] for n in node.nics],
            'free_hugepages': node.mem.free_hugepages_gb,
            'busy_time': node.busy_time}


# ----------------------------------------------------------------------------------
# random scenarios
# ----------------------------------------------------------------------------------
def random_node(rng, name, flavor='mixed', n_group_names=4):
    sockets = 2
    if flavor == 'wild':
        sockets = int(rng.choice([1, 2, 2, 2, 3, 4]))
    per = int(rng.choice([4, 6, 8, 12, 16])) if flavor != 'big' else int(rng.choice([16, 24, 32]))
    phys = per * sockets
    smt = bool(rng.random() < 0.7)
    reserved = int(rng.integers(0, min(3, per)))
    has_gpu = rng.random() < 0.55
    gpus, nics = [], []
    sw_base = [0x10 * (k + 1) for k in range(sockets)]
    if has_gpu:
        n_gpu = int(rng.choice([2, 4, 4, 8])) if flavor != 'wild' else int(rng.integers(1, 9))
        for d in range(n_gpu):
            numa = d * sockets // n_gpu if flavor != 'wild' or rng.random() < 0.8 else int(rng.integers(0, sockets))
            sw = sw_base[numa] + (d % 2 if n_gpu > 2 * sockets else 0)
            if flavor == 'wild' and rng.random() < 0.15:      # NUMA-inconsistent switch
                sw = sw_base[int(rng.integers(0, sockets))]
            gpus.append((d, numa, sw))
    nic_i = 0
    sriov = []
    for k in range(sockets):
        n_k = int(rng.integers(1, 3)) if flavor != 'vf' else 4
        if flavor == 'wild' and rng.random() < 0.1:
            n_k = 0
        for j in range(n_k):
            mbps = int(rng.choice([100000, 100000, 25000, 40000, 10000, 0]) if flavor == 'wild'
                       else rng.choice([100000, 100000, 25000]))
            sw = sw_base[k] + (j % 2 if has_gpu and len(gpus) > 2 * sockets else 0)
            nics.append((f'eth{nic_i}', mbps, k, sw))
            nic_i += 1
    if flavor == 'wild':
        order = rng.permutation(len(nics))
        nics = [nics[i] for i in order]
        if rng.random() < 0.2 and nics:
            sriov = [nics[0][0]]
    groups = None
    if rng.random() < 0.5:
        k = int(rng.integers(1, 3))
        groups = [GROUP_NAMES[i] for i in rng.choice(n_group_names, size=k, replace=False)]
    hp = int(rng.choice([16, 32, 64]))
    return make_node(name, sockets, phys, smt, reserved, gpus, nics, sriov, groups,
                     hp_alloc=hp, hp_free=hp - int(rng.integers(0, 8)),
                     active=bool(rng.random() < 0.95), maintenance=bool(rng.random() < 0.05),
                     isol=bool(rng.random() < 0.9))


def random_pod(rng, flavor='mixed', n_group_names=4, max_groups=3):
    G = int(rng.integers(1, max_groups + 1))
    gpu_pod = rng.random() < 0.5
    pci = gpu_pod and rng.random() < 0.5
    groups = []
    for _ in range(G):
        n_pairs = int(rng.integers(0, 3))
        if flavor == 'wild':
            speeds = [0, 1, 5, 10, 20, 22.5, 45, 50, 90]
        else:
            speeds = [0, 10, 20, 40]
        pairs = [(float(rng.choice(speeds)) if rng.random() < 0.3 else int(rng.choice([0, 10, 20, 40])),
                  int(rng.choice([0, 10, 20]))) for _ in range(n_pairs)]
        n_g = 0
        if gpu_pod:
            n_g = 1 if (pci and flavor != 'wild') else int(rng.integers(0, 3))
        gpus = [int(rng.integers(0, 3)) for _ in range(n_g)]
        groups.append(make_group(pairs, int(rng.integers(0, 5)), gpus, int(rng.integers(0, 3)),
                                 bool(rng.random() < 0.5), bool(rng.random() < 0.5)))
    pg = ['default'] if rng.random() < 0.6 else [GROUP_NAMES[i] for i in
                                                 rng.choice(n_group_names, size=int(rng.integers(1, 3)), replace=False)]
    return make_pod(groups, int(rng.integers(0, 4)), bool(rng.random() < 0.5),
                    'PCI' if pci else 'NUMA', int(rng.choice([0, 0, 2, 4])), pg)


def random_scenario(seed, n_nodes=8, n_pods=24, flavor='mixed', min_busy_secs=30.0, max_groups=3):
    rng = np.random.default_rng(seed)
    nodes = [random_node(rng, f'n{i}', flavor) for i in range(n_nodes)]
    pods = [random_pod(rng, flavor, max_groups=max_groups) for _ in range(n_pods)]
    t = 1000.0
    now = []
    for _ in range(n_pods):
        r = rng.random()
        t += 0.0 if r < 0.5 else (float(rng.integers(1, 20)) if r < 0.9 else 31.0)
        now.append(t)
    return {'nodes': nodes, 'pods': pods, 'now': now, 'min_busy_secs': min_busy_secs}


# ----------------------------------------------------------------------------------
# objects near the packed layout's limits (include/nhd_b200.h: 256 logical cores, 16 GPUs, 32 NICs per
# node; 72 cores per pod; numa^(groups+1) <= 256 tuples)
# ----------------------------------------------------------------------------------
def huge_node(rng, name):
    sockets = int(rng.choice([1, 2, 4]))
    phys = int(rng.choice([64, 96, 128]))
    smt = bool(rng.random() < 0.7)
    n_gpu = int(rng.choice([0, 8, 16]))
    gpus = [(d, d * sockets // max(1, n_gpu), 0x10 * (d * sockets // max(1, n_gpu) + 1) + (d % 4)) for d in range(n_gpu)]
    n_nic = int(rng.choice([2, 8, 16, 32]))
    nics = [(f'vf{i}', int(rng.choice([25000, 100000, 40000])), i % sockets, 0x10 * ((i % sockets) + 1) + (i % 4))
            for i in range(n_nic)]
    return make_node(name, sockets, phys, smt, int(rng.integers(0, 3)), gpus, nics, (), None, hp_alloc=128)


def huge_pod(rng):
    G = int(rng.integers(1, 4))                      # 4 groups on a 4-NUMA node would exceed the tuple limit
    gpu = rng.random() < 0.5
    pci = gpu and rng.random() < 0.5
    big = rng.random() < 0.3                         # group 0 asks for 40-70 cores: about a whole socket
    groups, budget = [], 72 - 3
    for g in range(G):
        pairs = [(int(rng.choice([0, 5, 10, 20])), int(rng.choice([0, 5, 10]))) for _ in range(int(rng.integers(0, 3)))]
        feeders = [int(rng.integers(0, 3)) for _ in range((1 if pci else int(rng.integers(0, 3))) if gpu else 0)]
        w, h = int(rng.integers(0, 8)), int(rng.integers(0, 4))
        limit = budget // (G - g)
        if big and g == 0:
            w = max(0, int(rng.integers(40, 71)) - 2 * len(pairs) - h - sum(feeders))
            limit = budget - 11 * (G - 1)            # the other groups keep room for their pairs, helpers and feeders
        need = 2 * len(pairs) + w + h + sum(feeders)
        if need > limit:
            w = max(0, w - (need - limit))
            need = 2 * len(pairs) + w + h + sum(feeders)
        budget -= need
        groups.append(make_group(pairs, w, feeders, h, bool(rng.random() < 0.5), bool(rng.random() < 0.5)))
    return make_pod(groups, int(rng.integers(0, 4)), bool(rng.random() < 0.5), 'PCI' if pci else 'NUMA',
                    int(rng.choice([0, 2, 8])))


def huge_scenario(seed, min_busy_secs=30.0):
    rng = np.random.default_rng(seed)
    n_pods = int(rng.integers(20, 120))
    now = [1000.0] * n_pods if seed % 2 else [float(x) for x in 1000.0 + np.cumsum(rng.integers(0, 12, n_pods))]
    return {'nodes': [huge_node(rng, f'n{i}') for i in range(int(rng.integers(3, 20)))],
            'pods': [huge_pod(rng) for _ in range(n_pods)], 'now': now, 'min_busy_secs': min_busy_secs}


# ----------------------------------------------------------------------------------
# the edges of the direct path's tables (nhd_kernels.cuh): free cores per socket around the index clamp of
# TB[type][smt][numa][free cores] (63), NICs per NUMA node around the four the direct path admits, NIC signature
# ids around FAST_NSIG_SMEM (4) and FAST_NSIG (128), more static descriptions than CLASS_SLOTS (4096), and NIC
# bandwidths that are not dyadic.  Each case names its boundary; 'used' (node -> logical cores) and 'nic_inuse'
# (node -> bit mask over Node.nics) are applied to the packed records (apply_preuse) and show what earlier pods
# took, so that one scenario holds many free counts / NIC states at once.
# ----------------------------------------------------------------------------------
def _nic(i, numa, mbps=100000):
    return (f'eth{i}', mbps, numa, 0x10 * (numa + 1))


def _preuse(node_recipe, free):
    """Logical cores to mark as used so that socket k of the node keeps free[k] free physical cores: taken from the
    top of the socket; on an SMT node every other one only through its hyperthread sibling, which makes the
    physical core just as unavailable (Node.GetFreeCpuCores)."""
    phys, smt, res = node_recipe
    per = phys // 2
    out = []
    for k, f in enumerate(free):
        take = per - res - f
        assert 0 <= take, (node_recipe, free)
        for j, c in enumerate(range((k + 1) * per - take, (k + 1) * per)):
            out.append(c + phys if smt and j % 2 else c)
    return out


def _cpu_pod(G, per_socket, flags=(False, False, False), misc=1, pairs=1, helpers=0, rx=10):
    """CPU-only NUMA-mode pod whose groups together ask one socket for `per_socket` physical cores on a node without
    SMT (the misc cores included); flags = (proc_smt, helper_smt, misc_smt)."""
    proc_smt, helper_smt, misc_smt = flags
    rest = per_socket - misc
    groups = []
    for g in range(G):
        share = rest // G + (1 if g < rest % G else 0)
        groups.append(make_group([(rx, rx)] * pairs, share - 2 * pairs - helpers, (), helpers, proc_smt, helper_smt))
    return make_pod(groups, misc=misc, misc_smt=misc_smt)


def _free_core_cases():
    cases = []
    nics2 = [_nic(0, 0), _nic(1, 1)]
    # (physical cores, SMT, reserved per socket), then the free counts per socket of every node built from it
    smt_nodes = [((128, True, 0), f) for f in ((61, 61), (62, 62), (63, 63), (64, 64), (64, 61), (61, 64), (63, 62))]
    flat_nodes = [((256, False, 0), f) for f in ((61, 61), (62, 62), (63, 63), (64, 64), (65, 65), (100, 100),
                                                 (128, 128), (128, 62), (62, 128), (65, 63))]
    gpus4 = [(0, 0, 0x10), (1, 0, 0x10), (2, 1, 0x20), (3, 1, 0x20)]

    def cluster(recipes, gpus=()):
        nodes, used = [], {}
        for i, (rc, free) in enumerate(recipes):
            phys, smt, res = rc
            nodes.append(make_node(f'f{i}', 2, phys, smt, res, gpus, nics2, hp_alloc=64))
            used[i] = _preuse(rc, free)
        return nodes, used

    flag_sets = [(False, False, False), (True, False, False), (False, True, True), (True, True, True)]
    for label, recipes in (('smt', smt_nodes), ('nosmt', flat_nodes)):
        for G in (1, 2):
            nodes, used = cluster(recipes)
            pods = []
            for d in range(60, 73):
                for fi, fl in enumerate(flag_sets):
                    if (d + fi) % 3 == 0:
                        pods.append(_cpu_pod(G, d, fl, misc=1 + (d % 3), helpers=d % 2, pairs=(d + fi) % 2))
            pods = pods[:28]                         # at most FAST_MAX_TYPES (32) distinct types: the tables stay on
            pods += pods[::-1]                       # every node is placed on more than once: it crosses 63 downwards
            cases.append({'id': f'a-free-{label}-G{G}',
                          'name': f'free cores 61-128 per socket around the TB clamp at 63, {label} nodes, G={G}, '
                                  f'demand 60-72 per socket', 'nodes': nodes, 'pods': pods, 'used': used,
                          'now': [2000.0] * len(pods), 'min_busy_secs': 30.0})
    # the reproductions of the clamp bug: 64 free per socket and 71 cores asked; 63 free and 65 asked; 68 free, both
    # groups held on NUMA 0 by its only NIC, 72 asked there
    rows = [('SMT, 64 free per socket, 1 group of 70 workers', [make_node(f'r{i}', 2, 128, True, 0, (), nics2) for i in range(3)],
             make_pod([make_group((), 70)], misc=1)),
            ('SMT, 63 free per socket, 1 group of 64 workers', [make_node(f'r{i}', 2, 128, True, 1, (), nics2) for i in range(3)],
             make_pod([make_group((), 64)], misc=1)),
            ('no SMT, 68 free per socket, NIC on NUMA 0 only, 2 groups of 1 pair + 34 workers',
             [make_node(f'r{i}', 2, 256, False, 60, (), [_nic(0, 0)]) for i in range(3)],
             make_pod([make_group(((10, 10),), 34), make_group(((10, 10),), 34)], misc=0)),
            ('no SMT, 68 free per socket, NIC on NUMA 0 only, 2 groups of 1 pair + 30 workers and 1 misc core (fits: 65 of 68)',
             [make_node(f'r{i}', 2, 256, False, 60, (), [_nic(0, 0)]) for i in range(3)],
             make_pod([make_group(((10, 10),), 30), make_group(((10, 10),), 30)], misc=1))]
    for k, (name, nodes, pod) in enumerate(rows):
        cases.append({'id': f'a-bug-row{k + 1}', 'name': 'clamp bug reproduction: ' + name, 'nodes': nodes, 'pods': [pod] * 4, 'used': {},
                      'now': [2000.0] * 4, 'min_busy_secs': 30.0})
    # a batch that walks one node down through the clamp: 128 -> 88 -> 48 free on a socket, then 64 -> 0 (pods
    # without NICs: a NIC is only ever used by one pod)
    nodes = [make_node(f'w{i}', 2, 256, False, 0, (), nics2) for i in range(2)]
    pods = [_cpu_pod(G, d, pairs=0) for G, d in ((1, 40), (1, 40), (1, 64), (2, 66), (1, 63), (1, 64), (2, 72), (1, 62),
                                                 (1, 40), (2, 70), (1, 65), (1, 63))]
    cases.append({'id': 'a-walk-down', 'name': 'one batch walks 128 free cores per socket down through 63', 'nodes': nodes, 'pods': pods,
                  'used': {}, 'now': [2000.0] * len(pods), 'min_busy_secs': 0.0})
    # the same with GPU pods: the general path's decision memo keys a socket's free cores clamped at 63 as well
    nodes = [make_node(f'v{i}', 2, 256, False, 0, gpus4, nics2) for i in range(2)]
    pods = [make_pod([make_group((), d - 2, gpus=[1])], misc=1, map_type='PCI' if d % 2 else 'NUMA')
            for d in (65, 65, 64, 66, 63, 70, 65, 64, 72, 40, 66)]
    cases.append({'id': 'a-walk-down-gpu', 'name': 'one batch walks 128 free cores per socket down through 63, GPU pods',
                  'nodes': nodes, 'pods': pods, 'used': {}, 'now': [2000.0] * len(pods), 'min_busy_secs': 0.0})
    # GPU and PCI types at the same demands: node_feasible_k2 in the filter, the general path in the sweep
    nodes, used = cluster(smt_nodes[:4] + flat_nodes[:6], gpus=gpus4)
    pods = []
    for d in (60, 62, 63, 64, 65, 68, 72):
        g = make_group(((10, 10),), d - 4 - (d % 2), gpus=[1], helpers=d % 2)
        pods.append(make_pod([g], misc=1, map_type='NUMA' if d % 3 else 'PCI'))
        g2 = [make_group(((10, 10),), (d - 1) // 2 - 3, gpus=[1]), make_group(((10, 10),), (d - 1) - (d - 1) // 2 - 3, gpus=[1])]
        pods.append(make_pod(g2, misc=1, map_type='PCI' if d % 2 else 'NUMA'))
    cases.append({'id': 'a-gpu-pci', 'name': 'GPU and PCI types asking 60-72 cores of a socket with 61-100 free', 'nodes': nodes,
                  'pods': pods + pods[::-1], 'used': used, 'now': [2000.0] * (2 * len(pods)), 'min_busy_secs': 0.0})
    return cases


def _nic_count_cases():
    """3, 4 and 5 NICs on one NUMA node (four is the most the direct path admits), every subset of them in use, NIC
    lists whose order is not NUMA order (ClsFast.li0 / li1 map NodeNic.idx back to Node.nics)."""
    cases = []
    for n in (3, 4, 5):
        for numa in (0, 1):
            other = 1 - numa
            nodes, inuse = [], {}
            for s in range(1 << n):
                # interleaved: the NICs of the two NUMA nodes alternate in the list, one NIC of the other node first
                lst = [_nic(0, other)]
                for j in range(n):
                    lst.append(_nic(len(lst), numa))
                    if j == 1:
                        lst.append(_nic(len(lst), other))
                nodes.append(make_node(f'c{s}', 2, 64, True, 1, (), lst, hp_alloc=64))
                pos = [i for i, x in enumerate(lst) if x[2] == numa]
                inuse[s] = sum(1 << pos[j] for j in range(n) if (s >> j) & 1)
            # pods whose groups all need a NIC of their own on `numa` (the other node's two NICs can take two
            # groups): each one claims the first free NIC, so the batch walks every node through its in-use states
            one = make_pod([make_group(((50, 50),), 2)], misc=1)
            two = make_pod([make_group(((50, 50),), 2), make_group(((50, 50),), 2)], misc=1)
            three = make_pod([make_group(((50, 50),), 1)] * 3, misc=1)
            small = make_pod([make_group(((10, 10),), 1), make_group(((70, 70),), 1)], misc=2, misc_smt=True)
            pods = ([one, two, one, small, two, three] * ((1 << n) // 2))[:3 * (1 << n)]
            cases.append({'id': f'b-nics{n}-numa{numa}',
                          'name': f'{n} NICs on NUMA {numa}, all {1 << n} subsets in use, NIC list not in NUMA order',
                          'nodes': nodes, 'pods': pods, 'used': {}, 'nic_inuse': inuse,
                          'now': [2000.0] * len(pods), 'min_busy_secs': 0.0})
    return cases


def signature_nodes(prefix, sigs, start=0):
    """One node per pair of per-NUMA NIC signatures (a signature: NIC speeds of one NUMA node, in order)."""
    nodes = []
    for i, (s0, s1) in enumerate(sigs):
        lst = [(f'e{j}', m, 0, 0x10) for j, m in enumerate(s0)] + [(f'e{len(s0) + j}', m, 1, 0x20) for j, m in enumerate(s1)]
        nodes.append(make_node(f'{prefix}{start + i}', 2, 16, bool(i % 2), 1, (), lst, hp_alloc=64))
    return nodes


SIG_SPEEDS = (25000, 40000, 100000, 12000)


def signature_list(n):
    """The first n per-NUMA NIC signatures (1-4 NICs over SIG_SPEEDS), fewest NICs first."""
    import itertools
    out = []
    for k in range(1, 5):
        out += list(itertools.product(SIG_SPEEDS, repeat=k))
    return out[:n]


def signature_pods():
    return [make_pod([make_group(((10, 10),), 2)], misc=1), make_pod([make_group(((20, 20),), 1)] * 2, misc=2),
            make_pod([make_group(((30, 5),), 3), make_group((), 2)], misc=0),
            make_pod([make_group(((10, 10),), 2, gpus=(), helpers=1, proc_smt=True)], misc=1, misc_smt=True)]


def _signature_cases():
    cases = []
    sig = signature_list(6)
    # 6 distinct signatures: ids 0-3 have their table rows in shared memory, 4 and 5 only in global memory
    pairs = [(sig[0], sig[1]), (sig[2], sig[3]), (sig[4], sig[5]), (sig[5], sig[0]), (sig[3], sig[4]), (sig[1], sig[1])]
    pods = signature_pods() * 4
    cases.append({'id': 'c-sig-smem', 'name': 'NIC signature ids 0-5 (FAST_NSIG_SMEM = 4 in shared memory, the rest global)',
                  'nodes': signature_nodes('s', pairs * 2), 'pods': pods, 'used': {},
                  'now': [2000.0] * len(pods), 'min_busy_secs': 0.0})
    # 140 distinct signatures: the 128 ids run out during the class scan, the classes after that are not covered
    sig = signature_list(140)
    pairs = [(sig[2 * i], sig[2 * i + 1]) for i in range(70)]
    pods = signature_pods() * 40                          # enough to reach the last nodes
    cases.append({'id': 'c-sig-140', 'name': '140 distinct NIC signatures > FAST_NSIG = 128', 'nodes': signature_nodes('x', pairs), 'pods': pods,
                  'used': {}, 'now': [2000.0] * len(pods), 'min_busy_secs': 0.0})
    return cases


def _class_cases():
    """4 200 nodes, each with its own static description (the PCIe switches of its eight NICs, SMT or not):
    more than the 4 096 slots of the class table, so at least 104 nodes end without a class.  The nodes that claim
    slots last are the likeliest to miss out, so all cores of the first 4 140 are taken and the pods land on the last
    60."""
    def patterns(n):            # switch ids in order of first appearance (the packed records number them so)
        if n == 0:
            yield ()
            return
        for p in patterns(n - 1):
            for s in range(max(p, default=-1) + 2):
                yield p + (s,)

    nodes, used = [], {}
    for i, sw in enumerate(list(patterns(8))[:2100] * 2):
        lst = [(f'e{j}', 100000, j // 4, 0x10 + sw[j]) for j in range(8)]
        nodes.append(make_node(f'k{i}', 2, 16, i >= 2100, 1, (), lst, hp_alloc=64))
        if i < 4140:
            used[i] = list(range(1, 8)) + list(range(9, 16))
    pods = signature_pods() * 20
    return [{'id': 'd-classes-4200', 'name': '4 200 distinct static descriptions > CLASS_SLOTS = 4 096', 'nodes': nodes, 'pods': pods,
             'used': used, 'now': [2000.0] * len(pods), 'min_busy_secs': 0.0}]


# group Gb/s sums that leave a NIC with exactly 0 or within an ulp of it, in one subtraction order and not in the
# other (Matcher.py:261-268 subtracts in group order; CfgTopology.GetTotalNICsRequested sums pairs in core order):
# 25 000 Mb/s -> 22.5 Gb/s: 22.5 - 0.9 - 21.6 == 0 but 22.5 - 21.6 - 0.9 < 0; 36 - 0.8 - 35.2 == 0 but the other
# order < 0; 10.8 - 8.1 - 2.7 > 0 by two ulps
FP64_GROUPS = [((25000,), [(0.2, 0.7), (10.8, 10.8)]),
               ((25000,), [(0.9,), (10.8, 10.8)]),
               ((40000,), [(0.1, 0.7), (12.7, 22.5)]),
               ((12000,), [(8.1,), (2.7,)]),
               ((12000,), [(0.9, 8.1), (0.9, 0.9)]),
               ((25000,), [(0.1, 0.2), (11.1, 11.1)]),
               ((25000,), [(0.3,), (11.1, 11.1)]),
               ((100000,), [(33.3, 33.3), (0.1, 0.2, 0.3), (12.7, 10.1)])]


def nic_bandwidth_scenarios():
    """Non-dyadic NIC demands whose remainders land on 0 or within an ulp of it, both group orders, the groups sharing
    one NIC (NIC on NUMA 0 only) or with a second NIC to move to; CPU-only, GPU and three-group pods."""
    out = []
    for k, ((mbps,), groups) in enumerate(FP64_GROUPS):
        nodes = [make_node('b0', 2, 32, True, 1, (), [('e0', mbps, 0, 0x10)]),
                 make_node('b1', 2, 32, False, 1, (), [('e0', mbps, 0, 0x10), ('e1', mbps, 0, 0x10)]),
                 make_node('b2', 2, 32, True, 1, [(0, 0, 0x10), (1, 1, 0x20)],
                           [('e0', mbps, 0, 0x10), ('e1', mbps, 1, 0x20), ('e2', mbps, 0, 0x10)]),
                 make_node('b3', 2, 32, False, 1, (), [('e0', mbps, 0, 0x10), ('e1', 100000, 1, 0x20)])]
        pods = []
        for order in (groups, groups[::-1]):
            gs = [make_group([(r, r) for r in pr], 1) for pr in order]
            pods.append(make_pod(gs, misc=1))
            pods.append(make_pod([make_group([(r, 0.0) for r in pr], 1, gpus=[1] if j == 0 else ()) for j, pr in enumerate(order)], misc=1))
            pods.append(make_pod(gs + [make_group(((0.1, 0.1),), 1)], misc=0))
        out.append({'id': f'e-fp64-{k}', 'name': f'fp64 NIC bandwidth: {mbps} Mb/s NICs, groups {groups} in both orders', 'nodes': nodes,
                    'pods': pods * 2, 'used': {}, 'now': [2000.0 + (i // 3) * 40 for i in range(2 * len(pods))],
                    'min_busy_secs': 30.0})
    return out


def limit_scenarios():
    """All the cases above, deterministic, in section order."""
    return _free_core_cases() + _nic_count_cases() + _signature_cases() + _class_cases() + nic_bandwidth_scenarios()


# ----------------------------------------------------------------------------------
# full-size streams (tests/test_gpu_full_size.py, tools/emu_full_size.py)
# ----------------------------------------------------------------------------------
def jumping_clocks(n, seed=31, t0=1000.0, step=0.001, p_forward=0.01, p_back=0.004):
    """Per-pod clocks for a 30 s busy window that make nodes leave it inside one batch: steps of ``step`` seconds,
    with some of +31 s (every stamp so far leaves the window) and some of -40 s (the busy set is rebuilt; the stamps
    are then in the future and stay busy until the clock passes them by 30 s, while stamps made after the step expire
    at the next +31 s).  Each clock is the previous one plus its step, in fp64."""
    rng = np.random.default_rng(seed)
    r = rng.random(n)
    steps = np.where(r < p_back, -40.0, np.where(r < p_back + p_forward, 31.0, step))
    steps[0] = 0.0
    out = np.empty(n, dtype='<f8')
    t = t0
    for i in range(n):
        t += steps[i]
        out[i] = t
    return out


def steady_state_update(start, bindings, seed=60, n=1024, moved_every=4):
    """The update a long-lived handle takes between two batches: ``n`` of the nodes the batch bound pods to get
    their start records back (the pods finished), and every ``moved_every``-th of them another node's start record
    instead (the node came back with other hardware, so its hardware class changes).  Returns (idx, new records)."""
    rng = np.random.default_rng(seed)
    bound = np.unique(bindings['node'][bindings['status'] == 0])
    assert len(bound) >= n, len(bound)
    idx = np.sort(rng.choice(bound, size=n, replace=False)).astype(np.int32)
    src = idx.copy()
    src[::moved_every] = rng.integers(0, len(start), size=len(src[::moved_every]))
    return idx, start[src].copy()


def nic_signatures(recs):
    """The distinct per-NUMA NIC signatures of 2-NUMA records (a signature: the NIC count of one NUMA node and the
    speed classes of its NICs in list order), as cls_fast_kernel numbers them."""
    out = set()
    for r in recs:
        if int(r['n_numa']) != 2:
            continue
        spd = int(r['nic_speed'][0]) | int(r['nic_speed'][1]) << 64
        for k in range(2):
            m = int(r['nic_numa_mask'][k])
            out.add(tuple((spd >> (4 * j)) & 0xF for j in range(32) if m >> j & 1))
    return out


def repeated_gpu_nodes(pods, bindings):
    """Nodes that took two or more GPU pods of one batch: with a constant clock the busy window allows one."""
    gpu = pods['groups']['n_gpus'].sum(axis=1) > 0
    placed = bindings['node'][(bindings['status'] == 0) & gpu]
    nodes, counts = np.unique(placed, return_counts=True)
    return nodes[counts >= 2]


def apply_preuse(recs, case):
    """The packed records of a limit case with its pre-used cores and NICs applied."""
    recs = recs.copy()
    for i, cores in case.get('used', {}).items():
        words = [int(w) for w in recs['used'][i]]
        for c in cores:
            assert not (words[c >> 6] >> (c & 63)) & 1, (case['name'], i, c)
            words[c >> 6] |= 1 << (c & 63)
        recs['used'][i] = words
    for i, m in case.get('nic_inuse', {}).items():
        recs['nic_inuse'][i] = m
    return recs
