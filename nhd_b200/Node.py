"""Cluster node model — host-side mirror of the reference's ``nhd/Node.py``.

The classes keep the reference's names and attributes (``Node.py:23-131``) so the
scheduler code that owns ``NHDScheduler.nodes`` keeps working: label ingest
(``ParseLabels``, ``Node.py:312-487``), claim / release of running pods
(``Node.py:530-636``), the busy window (``Node.py:843-850``) and the small
bookkeeping getters.  What is *not* here is the placement arithmetic: the free-core
/ free-GPU / NIC searches and ``GetFreeCpuBatch`` live in the CUDA solver.
``SetPhysicalIdsFromMapping`` therefore only *applies* a binding the solver already
computed (carried inside the mapping returned by ``nhd_b200.Matcher.FindNode``); it
raises if handed a mapping that did not come from the solver — there is no CPU
fallback.
"""
import threading
import time
from typing import Dict, List

from nhd_b200.CfgTopology import GpuType, NICCoreDirection

NIC_BW_AVAIL_PERCENT = 0.9                    # Node.py:18
SCHEDULABLE_NIC_SPEED_THRESH_MBPS = 11000     # Node.py:19
ENABLE_SHARING = False                        # Node.py:20

_NFD = 'feature.node.kubernetes.io/'


class NodeCore:                               # Node.py:23-34
    __slots__ = ('core', 'sibling', 'socket', 'used')

    def __init__(self, core, socket, sib):
        self.core, self.sibling, self.socket, self.used = core, sib, socket, False

    def SetSibling(self, sib):
        self.sibling = sib


class NodeNic:                                # Node.py:37-59
    def __init__(self, ifname, mac, vendor, speed, numa_node, pciesw, card, port):
        self.ifname, self.vendor, self.speed = ifname, vendor, speed
        self.numa_node, self.pciesw, self.card, self.port = numa_node, pciesw, card, port
        self.speed_used = [0, 0]
        self.pods_used = 0
        self.idx = 0
        self.mac = self.FormatMac(mac)

    def SetNodeIndex(self, idx):
        self.idx = idx

    def FormatMac(self, mac):
        return ':'.join(mac[i:i + 2] for i in range(0, len(mac) - 1, 2)).upper()


class NodeMemory:                             # Node.py:62-71
    def __init__(self):
        self.ttl_hugepages_gb = 0
        self.free_hugepages_gb = 0
        self.res_hugepages_gb = 0
        self.ttl_mem_gb = 0
        self.free_mem_gb = 0


class NodeGpu:                                # Node.py:74-97
    _TYPES = (('1080Ti', GpuType.GPU_TYPE_GTX_1080TI), ('1080', GpuType.GPU_TYPE_GTX_1080),
              ('2080Ti', GpuType.GPU_TYPE_GTX_2080TI), ('2080', GpuType.GPU_TYPE_GTX_2080),
              ('V100', GpuType.GPU_TYPE_V100))

    def __init__(self, gtype: str, device_id: int, numa_node: int, pciesw: int):
        self.gtype = self.GetType(gtype)
        self.device_id, self.numa_node, self.pciesw = device_id, numa_node, pciesw
        self.used = False

    def GetType(self, gtype: str):
        for frag, t in self._TYPES:
            if frag in gtype:
                return t
        return GpuType.GPU_TYPE_NOT_SUPPORTED


class Node:
    MIN_BUSY_SECS = float(30)                 # Node.py:107
    NHD_MAINT_LABEL = 'sigproc.viasat.io/maintenance'

    def __init__(self, name, active=True):
        self.name = name
        self.active = active
        self.busy_lock = threading.Lock()
        self.busy_time = float(0)
        self.last_busy_time_seconds = float(0)
        self.cores: List[NodeCore] = []
        self.gpus: List[NodeGpu] = []
        self.nics: List[NodeNic] = []
        self.sockets = 0
        self.numa_nodes = 0
        self.smt_enabled = False
        self.maintenance = False
        self.cores_per_proc = 0
        self.pod_info: Dict = {}
        self.data_vlan = 0
        self.groups: List[str] = ['default']
        self.gwip = '0.0.0.0/32'
        self.mem = NodeMemory()
        self.reserved_cores: List[int] = []

    # ---- label ingest (Node.py:134-142, 298-493) ---------------------------------
    @staticmethod
    def GetMaintenance(labels):
        v = labels.get(Node.NHD_MAINT_LABEL)
        return v is not None and v.lower() != 'not_scheduled'

    @staticmethod
    def ParseRangeList(rl: str):
        """cpuset syntax "a-b,c,d-e" -> sorted unique ints (Node.py:299-306)."""
        out = set()
        for part in rl.split(','):
            ends = part.split('-')
            out.update(range(int(ends[0]), int(ends[-1]) + 1))
        return sorted(out)

    def SetGroups(self, groups: str):
        self.groups = groups.split('.')

    def InitGroups(self, labels):
        self.groups = labels['NHD_GROUP'].split('.') if 'NHD_GROUP' in labels else ['default']
        return True

    def InitMaintenance(self, labels):
        self.maintenance = Node.GetMaintenance(labels)
        return True

    def InitCores(self, labels):
        k_cores, k_sock = _NFD + 'nfd-extras-cpu.num_cores', _NFD + 'nfd-extras-cpu.numSockets'
        if k_cores not in labels or k_sock not in labels:
            return False
        self.sockets = int(labels[k_sock])
        phys = int(labels[k_cores])
        self.smt_enabled = (_NFD + 'cpu-hardware_multithreading') in labels
        self.numa_nodes = self.sockets
        self.cores_per_proc = phys // self.sockets
        n_logical = phys * 2 if self.smt_enabled else phys
        per_socket = phys / self.sockets          # float on purpose (Node.py:344)
        self.cores = []
        for c in range(n_logical):
            sib = (c + phys if c < phys else c - phys) if self.smt_enabled else -1
            self.cores.append(NodeCore(c, int(int(c % phys) // per_socket), sib))
        k_isol = _NFD + 'nfd-extras-cpu.isolcpus'
        if k_isol in labels:
            isolated = set()
            for chunk in labels[k_isol].split('_'):
                isolated.update(Node.ParseRangeList(chunk))
            for c in range(n_logical):
                if c not in isolated:             # OS-owned cores are permanently "used"
                    self.cores[c].used = True
                    self.reserved_cores.append(c)
        return True

    def InitNics(self, labels):
        pfs = [l.split('.')[5] for l in labels if (_NFD + 'nfd-extras-sriov') in l]
        for l in labels:
            if (_NFD + 'nfd-extras-nic') not in l:
                continue
            p = l.split('.')
            ifname, vendor, mac, speed = p[4], p[5], p[6], p[7]
            numa_node, pciesw, card, port = int(p[8]), int(p[9], 16), int(p[10], 16), int(p[11])
            if ifname in pfs:                     # SR-IOV physical functions are not schedulable
                continue
            if 'Mbs' not in speed:                # link down
                continue
            mbps = int(speed[:speed.index('Mbs')])
            if mbps < SCHEDULABLE_NIC_SPEED_THRESH_MBPS:
                continue
            self.nics.append(NodeNic(ifname, mac, vendor, mbps / 1e3, numa_node, pciesw, card, port))
        per_numa: Dict[int, int] = {}
        for n in self.nics:                       # running index inside each NUMA node
            n.SetNodeIndex(per_numa.get(n.numa_node, 0))
            per_numa[n.numa_node] = n.idx + 1
        return True

    def InitGpus(self, labels):
        for l in labels:
            if (_NFD + 'nfd-extras-gpu') in l:
                p = l.split('.')
                self.gpus.append(NodeGpu(p[5], int(p[4]), int(p[6]), int(p[7], 16)))
        return True

    def InitMisc(self, labels):
        if 'DATA_PLANE_VLAN' not in labels or 'DATA_DEFAULT_GW' not in labels:
            return False
        self.data_vlan = int(labels['DATA_PLANE_VLAN'])
        self.gwip = labels['DATA_DEFAULT_GW']
        if 'RES_HUGEPAGES_GB' in labels:
            self.mem.res_hugepages_gb = int(labels['RES_HUGEPAGES_GB'])
        return True

    def ParseLabels(self, labels):
        return all(step(labels) for step in (self.InitGroups, self.InitMaintenance, self.InitCores,
                                             self.InitNics, self.InitGpus, self.InitMisc))

    def SetHugepages(self, alloc: int, free: int) -> bool:
        self.mem.ttl_hugepages_gb = alloc
        self.mem.free_hugepages_gb = free - self.mem.res_hugepages_gb
        return True

    def SetNodeAddr(self, addr):
        self.addr = addr

    # ---- bookkeeping getters (Node.py:163-248) --------------------------------------
    def GetNodeActive(self):
        return self.active

    def GetTotalHugepages(self):
        return self.mem.ttl_hugepages_gb

    def GetFreeHugepages(self):
        return self.mem.free_hugepages_gb

    def GetNIC(self, mac):
        return next((n for n in self.nics if n.mac == mac), None)

    def GetNICUsedSpeeds(self):
        return [n.speed_used for n in self.nics]

    def GetNICFromIfName(self, ifname):
        return next((n for n in self.nics if n.ifname == ifname), None)

    def GetTotalPods(self):
        return len(self.pod_info)

    def PodPresent(self, pod, ns):
        return (pod, ns) in self.pod_info

    def AddScheduledPod(self, pod, ns, top):
        self.pod_info[(pod, ns)] = top

    def RemoveScheduledPod(self, pod, ns):
        self.pod_info.pop((pod, ns), None)

    def GetGPU(self, di):
        return next((g for g in self.gpus if g.device_id == di), None)

    def SMTEnabled(self) -> bool:
        return self.smt_enabled

    def GetFreeCpuCoreCount(self) -> int:
        if self.smt_enabled:
            return sum(1 for x in self.cores if not x.used and not self.cores[x.sibling].used)
        return sum(1 for x in self.cores if not x.used)

    def GetFreeGpuCount(self) -> int:
        return sum(1 for g in self.gpus if not g.used)

    def GetTotalGPUs(self) -> int:
        return len(self.gpus)

    def GetTotalCPUs(self) -> int:
        return len(self.cores)

    # ---- claim / release of already-bound pods (Node.py:144-161, 530-646) ------------
    def ResetResources(self):
        reserved = set(self.reserved_cores)
        for c in self.cores:
            if c.core not in reserved:
                c.used = False
        for g in self.gpus:
            g.used = False
        for n in self.nics:
            n.pods_used = 0
            n.speed_used = [0, 0]
        self.mem.free_hugepages_gb = self.mem.ttl_hugepages_gb
        self.pod_info.clear()

    def _topology_cores(self, top):
        for pv in top.proc_groups:
            yield from pv.misc_cores
            yield from pv.proc_cores
            for g in pv.group_gpus:
                yield from g.cpu_cores
        yield from top.misc_cores

    def _apply_topology(self, top, take: bool) -> bool:
        sign = 1 if take else -1
        for pv in top.proc_groups:
            for c in list(pv.misc_cores) + list(pv.proc_cores):
                if not 0 <= c.core < len(self.cores):
                    return False
                self.cores[c.core].used = take
            for g in pv.group_gpus:
                dev = self.GetGPU(g.device_id)
                if dev is not None:
                    dev.used = take
                for c in g.cpu_cores:
                    self.cores[c.core].used = take
        for c in top.misc_cores:
            self.cores[c.core].used = take
        for pair in top.nic_core_pairing:
            nic = self.GetNIC(pair.mac)
            if nic is None:
                continue
            nic.speed_used[0] += sign * pair.rx_core.nic_speed
            nic.speed_used[1] += sign * pair.tx_core.nic_speed
            nic.pods_used += sign
        if top.hugepages_gb > 0:
            self.mem.free_hugepages_gb -= sign * top.hugepages_gb
        return True

    def RemoveResourcesFromTopology(self, top) -> bool:
        """Take the resources named in an already-filled topology (restart re-claim)."""
        return self._apply_topology(top, True)

    def AddResourcesFromTopology(self, top):
        """Give back the resources named in a filled topology (pod deleted)."""
        self._apply_topology(top, False)

    def GetNADListFromIndices(self, ilist: List[int]):
        return [self.nics[i].ifname for i in ilist]

    def ClaimPodNICResources(self, nidx):
        for ni in nidx:
            self.nics[ni].pods_used += 1

    def GetNicObjFromIndex(self, numa_node, nic_idx):
        return next((n for n in self.nics if n.idx == nic_idx and n.numa_node == numa_node), None)

    # ---- applying a solver binding (replaces Node.py:663-841) ------------------------
    def SetPhysicalIdsFromMapping(self, mapping, top):
        """Write the physical ids the CUDA solver chose into ``top`` and mark them used.

        Same contract as the reference method: returns ``used_nics`` as a list of
        ``(nic_list_index, speed, NICCoreDirection)`` or raises ``IndexError`` when the
        assignment failed (``Node.py:825-837``)."""
        from nhd_b200.packing import apply_binding
        binding = mapping.get('_nhd_binding') if isinstance(mapping, dict) else None
        if binding is None:
            raise RuntimeError('mapping was not produced by nhd_b200.Matcher.FindNode; '
                               'the CUDA solver has no CPU fallback for physical assignment')
        return apply_binding(self, top, binding)

    # ---- busy window (Node.py:843-853) ----------------------------------------------
    def SetBusy(self):
        with self.busy_lock:
            self.busy_time = time.monotonic()

    def IsBusy(self):
        self.last_busy_time_seconds = time.monotonic() - self.busy_time
        return self.last_busy_time_seconds < self.MIN_BUSY_SECS

    def GetBusyTimeSeconds(self):
        return self.last_busy_time_seconds
