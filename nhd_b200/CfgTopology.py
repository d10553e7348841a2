"""Pod request model — host-side mirror of the reference's ``nhd/CfgTopology.py``.

Same class, attribute and method names as the reference (``CfgTopology.py:8-243``)
so that code written against the reference scheduler (``NHDScheduler.py``,
``TriadCfgParser.py:107-304``) can build requests for the CUDA solver unchanged.
These classes only *describe* a request; the solver reads them through
``nhd_b200.packing.pack_pod`` and writes its answer back into ``Core.core``,
``GPU.device_id``, ``NICGroup.mac`` and the VLAN fields, exactly where
``Node.SetPhysicalIdsFromMapping`` (``Node.py:724-818``) leaves them.
"""
from enum import Enum
from typing import List, Optional


class GpuType(Enum):            # CfgTopology.py:8-16
    GPU_TYPE_ALL = 0
    GPU_TYPE_V100 = 1
    GPU_TYPE_GTX_1080 = 2
    GPU_TYPE_GTX_1080TI = 3
    GPU_TYPE_GTX_2080 = 4
    GPU_TYPE_GTX_2080TI = 5
    GPU_TYPE_A100 = 6
    GPU_TYPE_NOT_SUPPORTED = 7


class CpuType(Enum):            # CfgTopology.py:18-24
    CPU_TYPE_ALL = 0
    CPU_TYPE_HASWELL = 1
    CPU_TYPE_BROADWELL = 2
    CPU_TYPE_SKYLAKE = 3
    CPU_TYPE_COOPER_LAKE = 4
    CPU_TYPE_ICE_LAKE = 5


class NICCoreDirection(Enum):   # CfgTopology.py:26-29
    NIC_CORE_DIRECTION_NONE = 0
    NIC_CORE_DIRECTION_RX = 1
    NIC_CORE_DIRECTION_TX = 2


class SMTSetting(Enum):         # CfgTopology.py:31-33
    SMT_DISABLED = 0
    SMT_ENABLED = 1


class NUMASetting(Enum):        # CfgTopology.py:35-39
    LOGICAL_NUMA_DONT_CARE = -1
    LOGICAL_NUMA_0 = 0
    LOGICAL_NUMA_1 = 1
    LOGICAL_NUMA_GROUP = 2


class TopologyMapType(Enum):    # CfgTopology.py:41-45
    TOPOLOGY_MAP_INVALID = 0
    TOPOLOGY_MAP_NUMA = 1
    TOPOLOGY_MAP_PCI = 2
    TOPOLOGY_MAP_NONE = 3


_GPU_NAMES = {'ANY': GpuType.GPU_TYPE_ALL, 'V100': GpuType.GPU_TYPE_V100,
              '1080': GpuType.GPU_TYPE_GTX_1080, '1080Ti': GpuType.GPU_TYPE_GTX_1080TI,
              '2080': GpuType.GPU_TYPE_GTX_2080, '2080Ti': GpuType.GPU_TYPE_GTX_2080TI}
_CPU_NAMES = {'ANY': CpuType.CPU_TYPE_ALL, 'HASWELL': CpuType.CPU_TYPE_HASWELL,
              'BROADWELL': CpuType.CPU_TYPE_BROADWELL, 'SKYLAKE': CpuType.CPU_TYPE_SKYLAKE,
              'COOPER_LAKE': CpuType.CPU_TYPE_COOPER_LAKE, 'ICE_LAKE': CpuType.CPU_TYPE_ICE_LAKE}


class Core:
    """One requested CPU core (CfgTopology.py:48-55); ``core`` is the answer slot."""
    __slots__ = ('name', 'nic_speed', 'nic_dir', 'numa', 'core')

    def __init__(self, name, nic_speed, nic_dir, numa, core):
        self.name, self.nic_speed, self.nic_dir, self.numa, self.core = name, nic_speed, nic_dir, numa, core


class NICGroup:
    """An RX/TX core pair sharing one interface (CfgTopology.py:57-68)."""
    def __init__(self, rx_core: Core, tx_core: Core):
        self.rx_core, self.tx_core = rx_core, tx_core
        self.mac = ""
        self.rx_ring_size = 4096

    def AddInterface(self, mac):
        self.mac = mac

    def SetRxRingSize(self, ring_size: int):
        self.rx_ring_size = ring_size


class GPU:
    """One requested GPU and the cores feeding it (CfgTopology.py:70-75)."""
    def __init__(self, cpu_cores: List[Core], dev_id_names: List[str], gtype: GpuType, dev_id: int):
        self.dev_id_names, self.cpu_cores, self.gtype, self.device_id = dev_id_names, cpu_cores, gtype, dev_id


class VLANInfo:                 # CfgTopology.py:77-80
    def __init__(self, name: str, vlan: int):
        self.name, self.vlan = name, vlan


class ProcGroup:
    """A processing group: cores, helper cores and GPUs that must share a NUMA node
    (CfgTopology.py:82-123)."""
    def __init__(self):
        self.misc_cores: List[Core] = []
        self.proc_cores: List[Core] = []
        self.group_gpus: List[GPU] = []
        self.proc_smt = SMTSetting.SMT_DISABLED
        self.helper_smt = SMTSetting.SMT_DISABLED
        self.vlan: Optional[VLANInfo] = None

    def AddMiscCore(self, c: Core):
        self.misc_cores.append(c)

    def AddGroupCore(self, c: Core):
        self.proc_cores.append(c)

    def AddGroupGPU(self, g: GPU):
        self.group_gpus.append(g)

    def SetGpuType(self, t: GpuType):
        self.gpu_type = t

    def SetProcSmt(self, smt: SMTSetting):
        self.proc_smt = smt

    def SetHelperSmt(self, smt: SMTSetting):
        self.helper_smt = smt

    def SetDataVlan(self, vlan: VLANInfo):
        self.vlan = vlan

    def GetGpuType(self, gpu_type: str):
        return _GPU_NAMES.get(gpu_type)


class CfgTopology:
    """A whole pod request (CfgTopology.py:126-243)."""
    def __init__(self):
        self.arch = CpuType.CPU_TYPE_ALL
        self.misc_cores: List[Core] = []
        self.proc_groups: List[ProcGroup] = []
        self.nic_core_pairing: List[NICGroup] = []
        self.misc_cores_smt = SMTSetting.SMT_DISABLED
        self.map_type = TopologyMapType.TOPOLOGY_MAP_INVALID
        self.ctrl_vlan: Optional[VLANInfo] = None
        self.data_default_gw = ''
        self.hugepages_gb = 0

    def AddPodReservations(self, res):
        if 'hugepages-1Gi' in res:
            self.hugepages_gb = res['hugepages-1Gi']

    def AddNicPairing(self, rx_core: Core, tx_core: Core):
        self.nic_core_pairing.append(NICGroup(rx_core, tx_core))

    def SetCtrlVlan(self, vlan: VLANInfo):
        self.ctrl_vlan = vlan

    def SetDataDefaultGw(self, gw: str):
        self.data_default_gw = gw

    def GetNICGroup(self, coreobj: Core):
        rx, tx = NICCoreDirection.NIC_CORE_DIRECTION_RX, NICCoreDirection.NIC_CORE_DIRECTION_TX
        for pair in self.nic_core_pairing:
            if (coreobj.nic_dir == rx and pair.rx_core is coreobj) or (coreobj.nic_dir == tx and pair.tx_core is coreobj):
                return pair
        return None

    def GetNICGroupFromCoreNumbers(self, rxcore: int, txcore: int):
        for pair in self.nic_core_pairing:
            if pair.rx_core.core == rxcore and pair.tx_core.core == txcore:
                return pair
        return None

    def SetCpuArch(self, arch: str):
        return _CPU_NAMES.get(arch)

    def SetMiscCoreSmt(self, smt: SMTSetting):
        self.misc_cores_smt = smt

    def AddMiscCore(self, core: Core):
        self.misc_cores.append(core)

    def AddProcGroup(self, pg: ProcGroup):
        self.proc_groups.append(pg)

    # Request vectors, CfgTopology.py:199-232
    def GetTotalGpusRequested(self) -> List[int]:
        return [len(p.group_gpus) for p in self.proc_groups]

    def GetTotalCpusRequested(self):
        proc = [[(len(g.proc_cores) + sum(len(gpu.cpu_cores) for gpu in g.group_gpus), g.proc_smt),
                 (len(g.misc_cores), g.helper_smt)] for g in self.proc_groups]
        return {'proc': proc, 'misc': [len(self.misc_cores), self.misc_cores_smt]}

    def GetTotalNICsRequested(self):
        out = []
        for g in self.proc_groups:
            rx = tx = 0
            for c in g.proc_cores:
                if c.nic_dir == NICCoreDirection.NIC_CORE_DIRECTION_RX:
                    rx += c.nic_speed
                elif c.nic_dir == NICCoreDirection.NIC_CORE_DIRECTION_TX:
                    tx += c.nic_speed
            out.append([rx, tx])
        return out

    def SetTopMapType(self, t: str) -> None:
        if t == "NUMA":
            self.map_type = TopologyMapType.TOPOLOGY_MAP_NUMA
        elif t == "PCI":
            self.map_type = TopologyMapType.TOPOLOGY_MAP_PCI
