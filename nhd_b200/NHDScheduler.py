"""``NHDScheduler`` — host-side mirror of the reference's scheduler loop (``nhd/NHDScheduler.py``)
with the pending set solved as ONE batch on the GPU (SURVEY 8f row 1).

What is kept from the reference, method for method and with the same names, arguments, return
values and side effects on ``Node`` / ``pod_state`` / Kubernetes:

* start-up: ``InitNHDNodes`` / ``BuildInitialNodeList`` (``NHDScheduler.py:63-105``),
  ``LoadDeployedConfigs`` / ``ClaimPodResources`` (``:107-144, 161-172``), ``ResetResources`` (``:146-159``);
* ``ReleasePodResources`` (``:174-205``) including its two odd exits — a pod that was never annotated
  triggers a full ``ResetResources``, a pod that was annotated but not bound keeps its resources;
* ``InitialNodeFilter`` (``:235-247``), ``AttemptScheduling`` (``:249-353``), ``CheckPendingPods``
  (``:425-441``), the watch-queue handlers of ``run`` (``:491-577``) as ``HandleWatchItem``;
* ``GetBasicNodeStats`` / ``GetPodStats`` / ``ParseRPCReq`` (``:355-423``).

What is different is *where the placement is computed*.  The reference calls
``Matcher.FindNode`` once per pod (``:277``) against Python ``Node`` objects.  Here the packed
cluster lives on the GPU (``DeviceCluster``): ``CheckPendingPods`` first does the Kubernetes reads
for every pending pod, hands all their ``CfgTopology`` requests to ``nhd_solve_batch`` in one call
(pod *i* sees pods *0..i-1*, exactly like the loop), then walks the bindings in pod order doing what
``AttemptScheduling`` does after ``FindNode``: events, ``SetBusy``, physical ids into the topology,
NIC claim, NAD / GPU-map / config annotations, bind.  Only nodes the host changed outside the
solver (release, re-claim, reset, cordon, maintenance, groups) are re-sent (``nhd_update_nodes``).

A Kubernetes write that fails half way makes the reference call ``ReleasePodResources``, which may
reset the whole cluster; the pods after it in the batch were solved on a state that no longer
exists.  The batch is then cut at that pod: the host objects (always the truth) are pushed to the
device for every node that differs and the rest of the pending set is solved again — the outcome
is the one the sequential loop produces (``tests/test_scheduler.py``, pinned to the unmodified
reference ``NHDScheduler`` driven through the same fake Kubernetes manager).

Kubernetes itself, the kopf controller and the gRPC server are not part of this module: ``k8s`` is
any object with ``K8SMgr``'s method surface, ``cfg_parser(cfgtype, cfgstr)`` returns an object with
``CfgToTopology / TopologyToCfg / TopologyToGpuMap`` (``TriadCfgParser``).  There is no CPU
placement path: without the CUDA library ``DeviceCluster`` raises.
"""
import copy
import re
import threading
import time
from enum import Enum
from queue import Queue
from typing import Callable, Dict, Iterable, List, Optional, Sequence

import numpy as np

from nhd_b200 import packing, wire
from nhd_b200.Node import Node

NHD_SCHED_NAME = "nhd-scheduler"                # NHDScheduler.py:23


class PodStatus(Enum):                          # NHDScheduler.py:29-34
    POD_STATUS_SCHEDULED = 0
    POD_STATUS_FAILED = 1
    POD_STATUS_SUCCEEDED = 2
    POD_STATUS_RUNNING = 3
    POD_STATUS_COMPLETED = 4


class K8SEventType(Enum):                       # K8SMgr.py:16-18
    EVENT_TYPE_NORMAL = 0
    EVENT_TYPE_WARNING = 1


class NHDWatchTypes(Enum):                      # NHDWatchQueue.py:6-15 (the trailing commas make tuples there)
    NHD_WATCH_TYPE_TRIADSET_CREATE = 1
    NHD_WATCH_TYPE_TRIADSET_DELETE = 2
    NHD_WATCH_TYPE_TRIAD_POD_CREATE = 3
    NHD_WATCH_TYPE_TRIAD_POD_DELETE = 4
    NHD_WATCH_TYPE_NODE_UNCORDON = 5
    NHD_WATCH_TYPE_NODE_CORDON = 6
    NHD_WATCH_TYPE_GROUP_UPDATE = 7
    NHD_WATCH_TYPE_NODE_MAINT_START = 8
    NHD_WATCH_TYPE_NODE_MAINT_END = 9


class RpcMsgType(Enum):                         # NHDCommon.py:69-73
    TYPE_NODE_INFO = 1
    TYPE_SCHEDULER_INFO = 2
    TYPE_POD_INFO = 3
    TYPE_NODE_DETAIL = 4


def _type_name(t) -> str:
    """Watch / RPC types may arrive as this module's enums, the reference's, or plain names."""
    return t if isinstance(t, str) else t.name


class DeviceCluster:
    """The packed node records of ``NHDScheduler.nodes`` resident on the GPU.

    The Python ``Node`` objects stay the source of truth (the rest of the reference reads them);
    this class keeps the device copy equal to them: a full ``nhd_load_nodes`` when the node set or
    the solver constants change, ``nhd_update_nodes`` for the nodes named dirty, nothing for nodes
    only the solver itself changed (its own commit already holds what ``apply_binding`` writes
    into the objects — that equality is the parity the GPU tests establish)."""

    def __init__(self, solver_factory: Optional[Callable] = None, device: int = 0):
        self._factory = solver_factory
        self._device = device
        self._solver = None
        self._layout = packing.ClusterLayout()
        self._names: List[str] = []
        self._index: Dict[str, int] = {}
        self._speeds: List[float] = []
        self._min_busy = None
        self.full_loads = 0
        self.delta_nodes = 0
        self.batches = 0
        self.rewinds = 0
        self._last = None
        self.stubs = set()
        self.unsupported_nodes: Dict[str, str] = {}

    @property
    def layout(self):
        return self._layout

    def close(self):
        if self._solver is not None:
            self._solver.close()
            self._solver = None

    def _make_solver(self, min_busy):
        if self._solver is not None:
            self._solver.close()
        factory = self._factory
        if factory is None:
            from nhd_b200.solver import Solver          # raises without the CUDA library / a GPU
            factory = Solver
        self._speeds = list(self._layout.speeds)
        self._min_busy = min_busy
        self._solver = factory(self._layout.speed_table(), nic_bw_avail_percent=0.9,
                               min_busy_secs=min_busy, device=self._device)

    def _pack(self, nodes: Sequence) -> np.ndarray:
        recs = np.zeros(len(nodes), dtype=wire.NODE_DTYPE)
        for i, node in enumerate(nodes):
            try:
                packing.pack_node(node, self._layout, out=recs[i])
            except packing.UnsupportedError as err:
                # a node whose labels were refused stays in NHDScheduler.nodes, deactivated and half
                # initialised (NHDScheduler.py:88-100); it holds its place in the order as an inactive stub.
                # An ACTIVE node beyond the packed limits (> 256 logical cores, > 16 GPUs, ...) cannot be
                # described to the solver either: it is kept out of placement (never approximated) and named in
                # unsupported_nodes for the operator.
                if node.active:
                    if node.name not in self.unsupported_nodes:
                        packing._log.warning('node %s is outside the packed limits and is kept out of placement: %s', node.name, err)
                    self.unsupported_nodes[node.name] = str(err)
                packing.stub_record(recs[i])
                self.stubs.add(node.name)
        return recs

    def sync(self, nodes: Dict[str, object], dirty: Iterable[str]):
        """Make the device copy equal to ``nodes``; ``dirty`` names the nodes the host changed since
        the last call."""
        names = list(nodes)
        min_busy = float(getattr(type(nodes[names[0]]), 'MIN_BUSY_SECS', 30.0)) if names else 30.0
        full = self._solver is None or names != self._names or min_busy != self._min_busy
        recs = idx = None
        if not full:
            dirty = set(dirty)
            todo = [n for n in names if n in dirty]
            if todo:
                recs = self._pack([nodes[n] for n in todo])
                idx = np.asarray([self._index[n] for n in todo], dtype='<i4')
            full = self._layout.speeds != self._speeds      # a NIC speed the solver has no class for yet
        if full:
            recs = self._pack([nodes[n] for n in names])
            if self._solver is None or self._layout.speeds != self._speeds or min_busy != self._min_busy:
                self._make_solver(min_busy)
            self._solver.load_nodes(recs)
            self._names = names
            self._index = {n: i for i, n in enumerate(names)}
            self.full_loads += 1
        elif recs is not None:
            self._solver.update_nodes(idx, recs)
            self.delta_nodes += len(idx)

    def _pods(self, tops: Sequence, pod_groups: Sequence[Iterable[str]], packed: Sequence = None) -> np.ndarray:
        pods = np.zeros(len(tops), dtype=wire.POD_DTYPE)
        for i, top in enumerate(tops):
            if packed is not None and packed[i] is not None:
                pods[i] = packed[i]
                pods[i]['group_mask'] = self._layout.groups_mask(pod_groups[i], create=False)
            else:
                packing.pack_pod(top, pod_groups[i], self._layout, out=pods[i])
        return pods

    def _indices(self, names: Iterable[str], what: str) -> np.ndarray:
        """Indices of the nodes ``names``; a ValueError lists the unknown ones (``what``: what the caller does to them)."""
        names = list(names)
        missing = [n for n in names if n not in self._index]
        if missing:
            raise ValueError(f'cannot {what} unknown node(s) {missing}')
        return np.asarray([self._index[n] for n in names], dtype='<i4')

    @staticmethod
    def _clocks(n: int, now) -> np.ndarray:
        """Per-pod clocks of ``n`` pods from one clock or one per pod."""
        return np.full(n, now, dtype='<f8') if np.isscalar(now) else np.asarray(now, dtype='<f8')

    def solve(self, tops: Sequence, pod_groups: Sequence[Iterable[str]], now: float, packed: Sequence = None):
        """Bindings of ``tops`` scheduled in order on the synced cluster (one GPU call).  ``packed``: records
        ``pack_pod`` already made of them; only the node-group mask is worked out again (``sync`` may have met new
        group names since)."""
        pods = self._pods(tops, pod_groups, packed)
        self.batches += 1
        self._solver.snapshot()                       # so that rewind() can step back inside this batch
        self._last = (pods, np.full(len(tops), now, dtype='<f8'))
        return self._solver.solve_batch(*self._last)

    def explain(self):
        """Per-reason node counts ((pods, wire.WHY_COUNT) array) of the NO_CANDIDATE pods of the last ``solve``,
        each at the state that pod saw; valid right after ``solve`` (before any ``rewind``).  None when the solver
        in use cannot explain (a stand-in without ``explain_batch``)."""
        fn = getattr(self._solver, 'explain_batch', None)
        return fn() if fn is not None else None

    def query(self, tops: Sequence, pod_groups: Sequence[Iterable[str]], now, source: str = 'mirror',
              packed: Sequence = None):
        """Per pod, the binding it would get on its own (one GPU query, nothing placed): on the synced cluster
        (``source='mirror'``) or on the state the last ``solve`` started from (``'snapshot'``, valid until the next
        ``sync`` that uploads records).  ``now``: one clock or one per pod.  None when the solver in use cannot
        answer queries (a stand-in without ``query_batch``)."""
        fn = getattr(self._solver, 'query_batch', None)
        if fn is None:
            return None
        return fn(self._pods(tops, pod_groups, packed), self._clocks(len(tops), now), source=source)

    def plan(self, tops: Sequence, pod_groups: Sequence[Iterable[str]], now, source: str = 'mirror',
             exclude: Iterable[str] = (), packed: Sequence = None, explain: bool = False):
        """The bindings of ``tops`` scheduled in order, each seeing the ones before it, with nothing placed (one GPU
        dry run): on the synced cluster (``source='mirror'``) or on the state the last ``solve`` started from
        (``'snapshot'``), with the nodes named in ``exclude`` taken as in maintenance.  ``explain=True``: also the
        per-reason node counts of the NO_CANDIDATE pods, as ``explain`` gives them after a ``solve``.  None when the
        solver in use cannot plan (a stand-in without ``plan_batch``)."""
        fn = getattr(self._solver, 'plan_batch', None)
        if fn is None:
            return None
        idx = self._indices(exclude, 'exclude')
        return fn(self._pods(tops, pod_groups, packed), self._clocks(len(tops), now), source=source, exclude=idx,
                  explain=explain)

    def plan_scenarios(self, scenarios: Sequence, source: str = 'mirror'):
        """Many independent dry runs in one GPU call, each as ``plan`` would answer it alone.  ``scenarios``: a sequence
        of ``(exclude, tops, pod_groups, now[, packed[, lift[, edits]]])`` with ``exclude`` node names.  ``lift`` (None:
        never): the excluded nodes are back in service from the scenario's pod ``lift`` on.  ``edits`` (None: none):
        ``{node name: Node-like object}``, packed as ``sync`` packs nodes, the records those nodes have for the whole
        scenario.  Returns one ``(code, pod, bindings)`` per scenario (``Solver.plan_scenarios``): ``bindings`` None
        when the scenario is refused, ``code`` and ``pod`` saying why and for which of its pods.  None when the solver
        in use cannot plan scenarios (a stand-in without ``plan_scenarios``)."""
        fn = getattr(self._solver, 'plan_scenarios', None)
        if fn is None:
            return None
        # every scenario's names are checked before any is packed
        self._indices(sorted({n for sc in scenarios for n in list(sc[0]) + list(sc[6] if len(sc) > 6 and sc[6] else ())}),
                      'exclude or edit')
        args = []
        for sc in scenarios:
            exclude, tops, pod_groups, now = sc[:4]
            packed = sc[4] if len(sc) > 4 else None
            lift = sc[5] if len(sc) > 5 else None
            edits = sc[6] if len(sc) > 6 else None
            idx = self._indices(exclude, 'exclude')
            if edits:
                edits = (self._indices(edits, 'edit'), self._pack(list(edits.values())))
            args.append((idx, self._pods(tops, pod_groups, packed), self._clocks(len(tops), now)) +
                        ((lift, edits or None) if lift is not None or edits else ()))
        return fn(args, source=source)

    def rewind(self, k: int):
        """Put the device back to the state right after pod ``k`` of the last batch (restore the
        snapshot taken before it, solve pods ``0..k`` again: the solver is deterministic)."""
        pods, now = self._last
        self._solver.restore()
        self._solver.solve_batch(pods[:k + 1], now[:k + 1])
        self.rewinds += 1

    def read_records(self):
        return self._solver.read_nodes()

    def read_record(self, index: int):
        return self._solver.read_nodes(index, 1)[0]

    def name_of(self, index: int) -> str:
        return self._names[index]


def _copy_node(node):
    """A copy of ``node`` that a planned release may change: ``copy.deepcopy`` with a new ``busy_lock`` (a lock cannot
    be copied) and the pods' topologies shared (a release only reads them)."""
    memo = {id(top): top for top in node.pod_info.values()}
    lock = getattr(node, 'busy_lock', None)
    if lock is not None:
        memo[id(lock)] = threading.Lock()
    return copy.deepcopy(node, memo)


class _Pending:
    """One pending pod between the Kubernetes reads and the Kubernetes writes."""
    __slots__ = ('pos', 'key', 'pobj', 'tcfg', 'top', 'groups', 'ready', 'unsupported', 'rec')

    def __init__(self, pos, key):
        self.pos, self.key = pos, key
        self.pobj = self.tcfg = self.top = self.groups = self.unsupported = self.rec = None
        self.ready = False

    @property
    def solvable(self) -> bool:
        """Read, parsed and within the packed layout: the pod goes to the solver."""
        return self.top is not None and self.unsupported is None


class NHDScheduler:
    def __init__(self, k8s, cfg_parser: Callable, rpcq: Queue = None, solver_factory: Callable = None,
                 device: int = 0, clock: Callable[[], float] = time.monotonic,
                 wall: Callable[[], float] = time.time, node_cls=Node, logger=None,
                 stats_from_device: bool = False, diagnose_contention: bool = False):
        self.nodes: Dict[str, Node] = {}
        self.k8s = k8s
        self.sched_name = NHD_SCHED_NAME
        self.pod_state = {}
        self.rpcq = rpcq
        self.failed_schedule_count = 0
        self.cluster = DeviceCluster(solver_factory, device)
        self._cfg_parser = cfg_parser
        self._clock, self._wall = clock, wall
        self._node_cls = node_cls
        self._dirty = set()
        self._log = logger
        self.pods_solved = 0
        self.assign_failed_nodes = set()
        self.unsupported_pods = []                   # (ns, pod, why): requests beyond the packed layout's limits
        # (ns, pod) -> {reason name: nodes}: why the pod's last attempt found no node (NHD_WHY_*, wire.WHY_NAMES),
        # until the pod is scheduled or deleted
        self.unschedulable_reasons: Dict[tuple, Dict[str, int]] = {}
        self.stats_from_device = stats_from_device
        # opt-in: for a pod that found no node, ask whether it would have fit alone at the start of its batch
        # (nhd_query_batch on the batch-start snapshot); (ns, pod) -> that node, i.e. earlier pods of the same batch
        # took the capacity.  Kept until the pod is scheduled or deleted.
        self.diagnose_contention = diagnose_contention
        self.contended_pods: Dict[tuple, str] = {}

    # ---- small helpers --------------------------------------------------------------------
    def _info(self, msg):
        if self._log is not None:
            self._log.info(msg)

    def _error(self, msg):
        if self._log is not None:
            self._log.error(msg)

    def _touch(self, name):
        """The host changed node ``name`` outside the solver: re-send it before the next batch."""
        self._dirty.add(name)

    def _sync(self):
        """Make the device copy equal to the nodes, re-sending the ones the host changed."""
        self.cluster.sync(self.nodes, self._dirty)
        self._dirty.clear()

    def close(self):
        self.cluster.close()

    # ---- start-up (NHDScheduler.py:63-105) --------------------------------------------------
    def InitNHDNodes(self):
        for node in self.k8s.GetNodes():
            self.nodes[node] = self._node_cls(node, self.k8s.IsNodeActive(node))

    def BuildInitialNodeList(self):
        self.InitNHDNodes()
        for n, v in self.nodes.items():
            try:
                v.SetNodeAddr(self.k8s.GetNodeAddr(n))
                if not v.ParseLabels(self.k8s.GetNodeLabels(n)):
                    self._error(f'Error while parsing labels for node {n}, deactivating node')
                    v.active = False
                    continue
                (alloc, free) = self.k8s.GetNodeHugepageResources(n)
                if alloc == 0 or not v.SetHugepages(alloc, free):
                    self._error(f'Error while parsing allocatable resources for node {n}, deactivating node')
                    v.active = False
            except Exception as e:                   # the reference swallows everything here (:98-100)
                self._error(f'Caught exception while setting up node {n}:\n    {e}')
                v.active = False
        self._dirty.update(self.nodes)

    # ---- claim / release of deployed pods (NHDScheduler.py:107-205) ---------------------------
    def GetCfgParser(self, cfgtype: str, cfgstr: str):
        return self._cfg_parser(cfgtype, cfgstr)

    def ClaimPodResources(self, podname, ns, uid):
        cfgstr = self.k8s.GetCfgAnnotations(podname, ns)
        if cfgstr == False:                          # noqa: E712  (the reference's test, :112)
            self._error(f'Couldn\'t find pod resources for {ns}.{podname}')
            return
        cfgtype = self.k8s.GetCfgType(podname, ns)
        tcfg = self.GetCfgParser(cfgtype, cfgstr)
        top = tcfg.CfgToTopology(True)
        if top is not None:
            n = self.k8s.GetPodNode(podname, ns)
            if not n:
                return
            if n not in self.nodes:
                return
            if self.nodes[n].PodPresent(podname, ns):
                return
            self._touch(n)
            if not self.nodes[n].RemoveResourcesFromTopology(top):
                self._error('Failed removing resources')
                return
            self.nodes[n].AddScheduledPod(podname, ns, top)
            self.pod_state[(ns, podname)] = {'state': PodStatus.POD_STATUS_SCHEDULED, 'time': self._wall(),
                                             'uid': uid}

    def ResetResources(self):
        for name, n in self.nodes.items():
            n.ResetResources()
            self._touch(name)
        self.pod_state.clear()
        self.LoadDeployedConfigs()

    def LoadDeployedConfigs(self):
        for p in self.k8s.GetScheduledPods(self.sched_name):
            if p[3] in ('Running', 'CrashLoopBackOff', 'Pending'):
                self.ClaimPodResources(p[0], p[1], p[2])

    def ReleasePodResources(self, podname, ns):
        target = self._release_target(podname, ns)
        if target is None:                           # never annotated: full re-scan (:178-181)
            self.ResetResources()
            return
        node, top = target
        if node is not None:
            self._touch(node)
            self._give_back(self.nodes[node], podname, ns, top, float(self._clock()))

    def _release_target(self, podname, ns):
        """The Kubernetes reads of ``ReleasePodResources``: ``(node name, topology)`` of what deleting the pod gives
        back, ``(None, None)`` when it gives nothing back, None when the pod was never annotated (the release then
        re-scans every node)."""
        cfgstr = self.k8s.GetCfgAnnotations(podname, ns)
        if cfgstr == False:                          # noqa: E712  (the reference's test)
            return None
        cfgtype = self.k8s.GetCfgType(podname, ns)
        tcfg = self.GetCfgParser(cfgtype, cfgstr)
        top = tcfg.CfgToTopology(True)
        if top is None:
            return None, None
        node = self.k8s.GetPodNode(podname, ns)
        # annotated but not bound (:189-191), an unknown node, a pod the node does not hold: nothing is given back
        if not node or node not in self.nodes or not self.nodes[node].PodPresent(podname, ns):
            return None, None
        return node, top

    @staticmethod
    def _give_back(node, podname, ns, top, now: float):
        """The release proper, on ``node``: the pod's resources back, the pod gone, busy from ``now`` (Node.SetBusy,
        Node.py:843-845, on the scheduler's clock)."""
        node.AddResourcesFromTopology(top)
        node.RemoveScheduledPod(podname, ns)
        node.busy_time = now

    def ParsePodResources(self, pod: str, ns: str) -> Dict[str, int]:      # :214-224
        res = self.k8s.GetRequestedPodResources(pod, ns)
        trimmed = {}
        if 'hugepages-1Gi' in res:
            trimmed['hugepages-1Gi'] = int(res['hugepages-1Gi'][:res['hugepages-1Gi'].find('G')])
        return trimmed

    # ---- placement ------------------------------------------------------------------------------
    def InitialNodeFilter(self, podname: str, ns: str):
        """``NHDScheduler.py:235-247``.  Informational here: the batch path evaluates the same gate
        on the GPU from the pod's group list (group mask AND + active flag)."""
        ngroups = self.k8s.GetPodNodeGroups(podname, ns)
        return {n: v for n, v in self.nodes.items() if len(set(v.groups) & set(ngroups)) > 0 and v.active}

    def _prepare(self, e: _Pending, events: bool = True):
        """The Kubernetes reads of ``AttemptScheduling`` up to ``FindNode`` (``:254-275``); ``events=False`` only
        reads (no pod event is generated)."""
        ns, podname = e.key[0], e.key[1]
        e.ready = True
        e.pobj = self.k8s.GetPodObj(podname, ns)
        if e.pobj is None:
            self._error(f'Could not get pod object for pod {ns}.{podname}')
            return
        if events:
            self.k8s.GeneratePodEvent(e.pobj, podname, ns, 'StartedScheduling', K8SEventType.EVENT_TYPE_NORMAL,
                                      f'Started scheduling {ns}/{podname}')
        _, cfgstr = self.k8s.GetCfgMap(podname, ns)
        cfgtype = self.k8s.GetCfgType(podname, ns)
        e.tcfg = self.GetCfgParser(cfgtype, cfgstr)
        e.top = e.tcfg.CfgToTopology(False)
        if e.top is None:
            if events:
                self.k8s.GeneratePodEvent(e.pobj, podname, ns, 'FailedCfgParse', K8SEventType.EVENT_TYPE_WARNING,
                                          f'Error while processing config for pod {podname}')
            return
        e.groups = self.k8s.GetPodNodeGroups(podname, ns)
        try:                                         # a request beyond the packed layout (include/nhd_b200.h, NHD_MAX_*)
            e.rec = packing.pack_pod(e.top, e.groups, self.cluster.layout)     # kept for the solve (group mask aside)
        except packing.UnsupportedError as err:      # cannot be solved here and is never approximated: the pod fails,
            e.unsupported = str(err)                 # loudly, instead of taking the scheduler thread down

    def _finish(self, e: _Pending, binding, now: float) -> bool:
        """``AttemptScheduling`` from the result of ``FindNode`` on (``:278-353``)."""
        ns, podname = e.key[0], e.key[1]
        if e.pobj is None or e.top is None:
            return False
        k8s, pobj, top, tcfg = self.k8s, e.pobj, e.top, e.tcfg
        if e.unsupported is not None:
            self._error(f'Pod {ns}.{podname} is outside the solver\'s limits: {e.unsupported}')
            k8s.GeneratePodEvent(pobj, podname, ns, 'FailedScheduling', K8SEventType.EVENT_TYPE_WARNING,
                                 f'Pod {podname} cannot be placed by the CUDA solver: {e.unsupported}')
            self.failed_schedule_count += 1
            self.unsupported_pods.append((ns, podname, e.unsupported))
            return False
        if binding is None or int(binding['node']) < 0:
            k8s.GeneratePodEvent(pobj, podname, ns, 'FailedScheduling', K8SEventType.EVENT_TYPE_WARNING,
                                 f'No valid candidate nodes found for scheduling pod {podname}')
            self.failed_schedule_count += 1
            return False
        nodename = self.cluster.name_of(int(binding['node']))
        k8s.GeneratePodEvent(pobj, podname, ns, 'Scheduling', K8SEventType.EVENT_TYPE_NORMAL,
                             f'Node {nodename} selected for scheduling')
        node = self.nodes[nodename]
        node.busy_time = float(now)                                           # SetBusy (:289)
        try:
            packing.apply_binding(node, top, binding)                         # SetPhysicalIdsFromMapping (:292)
        except IndexError:
            self._error('Failed to map physical resources from topology config!')
            # The reference's unwind (Node.py:825-837) gives cores and GPUs back but never the hugepages it
            # took at :794-796 (a failure at the last step, the top-level misc cores); the solver's record
            # holds the node as the reference leaves it.  Its NIC part indexes self.nics with a *speed* and
            # stops at the first entry (IndexError again, or a TypeError that ends the reference's thread:
            # status REF_WOULD_CRASH), leaving the Gb/s it had added in NodeNic.speed_used: that residue of a
            # statistic is not reproduced, the node is remembered in assign_failed_nodes instead.
            rec = self.cluster.read_record(int(binding['node']))
            node.mem.free_hugepages_gb = int(rec['free_hugepages_gb'])
            self.assign_failed_nodes.add(nodename)
            return False
        nidx = [int(x) for x in binding['claimed_nics'][:int(binding['n_claimed'])]]   # list({x[0] ...}) (:302)
        node.ClaimPodNICResources(nidx)
        if any(node.nics[i].pods_used <= 0 for i in nidx):
            # Release counts a NIC down once per RX/TX pairing but the claim counts it up once per pod
            # (Node.py:579,629 vs :644-646), so a counter can sit below zero and a claimed NIC still reads
            # as free (pods_used > 0, Node.py:292).  The device keeps one in-use bit: re-send this node.
            self._touch(nodename)
        nadlist = node.GetNADListFromIndices(nidx)
        csnad = ','.join([f'{x}@{x}' for x in nadlist])
        if not k8s.AddNADToPod(podname, ns, csnad):
            self._error('Failed to set NetworkAttachmentDefinition')
            self.ReleasePodResources(podname, ns)
            return False
        topstr = tcfg.TopologyToCfg()
        gpustr = tcfg.TopologyToGpuMap()
        if gpustr:
            if not k8s.AnnotatePodGpuMap(ns, podname, gpustr):
                k8s.GeneratePodEvent(pobj, podname, ns, 'PodCfgFailed', K8SEventType.EVENT_TYPE_WARNING,
                                     f'Failed to annotate pod\'s GPU configuration')
                self.ReleasePodResources(podname, ns)
                return False
        if not k8s.AnnotatePodConfig(ns, podname, topstr):
            k8s.GeneratePodEvent(pobj, podname, ns, 'PodCfgFailed', K8SEventType.EVENT_TYPE_WARNING,
                                 f'Failed to annotate pod\'s configuration')
            self.ReleasePodResources(podname, ns)
            return False
        else:
            k8s.GeneratePodEvent(pobj, podname, ns, 'PodCfgSuccess', K8SEventType.EVENT_TYPE_NORMAL,
                                 f'Successfully added pod\'s configuration to annotations')
        if not k8s.BindPodToNode(podname, nodename, ns):
            k8s.GeneratePodEvent(pobj, podname, ns, 'FailedScheduling', K8SEventType.EVENT_TYPE_WARNING,
                                 f'Failed to schedule {ns}/{podname} to {nodename}')
            self.ReleasePodResources(podname, ns)
            return False
        else:
            k8s.GeneratePodEvent(pobj, podname, ns, 'Scheduled', K8SEventType.EVENT_TYPE_NORMAL,
                                 f'Successfully assigned {ns}/{podname} to {nodename}')
        node.AddScheduledPod(podname, ns, top)
        return True

    def ScheduleBatch(self, keys: Sequence, wanted: Callable = None) -> Dict:
        """Schedule the pods ``keys`` = ``[(ns, name, uid), ...]`` in order, as if ``AttemptScheduling``
        were called for one after the other.  ``wanted(key)`` is asked again for the pods behind a cut
        (``CheckPendingPods`` re-reads ``pod_state``, which a reset clears).  Returns ``{key: bool}``."""
        results = {}
        entries = [_Pending(i, k) for i, k in enumerate(keys)]
        pos = 0
        while pos < len(entries):
            run = [e for e in entries[pos:] if wanted is None or wanted(e.key)]
            if not run:
                break
            for e in run:
                if not e.ready:
                    self._prepare(e)
            now = float(self._clock())
            solvable = [e for e in run if e.solvable]
            bindings, why, contended = {}, None, None
            if solvable and self.nodes:
                self._sync()
                out, solvable, dropped = self._without_refused(
                    lambda es: self.cluster.solve([e.top for e in es], [e.groups for e in es], now,
                                                  packed=[e.rec for e in es]), solvable)
                for e, err in dropped:                  # the pod fails loudly (_finish), the rest goes on
                    e.unsupported = str(err)
                self.pods_solved += len(solvable)
                if solvable:
                    bindings = {e.pos: b for e, b in zip(solvable, out)}
                    if any(int(b['status']) == wire.NO_CANDIDATE for b in out):
                        # why the NO_CANDIDATE pods found no node: read before a rewind replaces the solved batch
                        why = self.cluster.explain()
                        if why is not None:
                            why = {e.pos: w for e, w in zip(solvable, why)}
                        if self.diagnose_contention:
                            contended = self._contention(solvable, out, now)
            cut = None
            for e in run:
                b = bindings.get(e.pos)
                if b is not None and int(b['status']) == wire.NO_CANDIDATE and why is not None:
                    self._explain(e, why[e.pos])
                if b is not None and int(b['status']) == wire.NO_CANDIDATE and contended is not None:
                    self._contended(e, contended[e.pos])
                rewound = False
                if b is not None and int(b['status']) in (wire.ASSIGN_FAILED, wire.REF_WOULD_CRASH):
                    # what a failed assignment leaves on its node is read back from the solver (see _finish);
                    # for that the device must stand right after this pod, not at the end of the batch
                    self.cluster.rewind(solvable.index(e))
                    rewound = True
                results[e.key] = ok = self._finish(e, b, now)
                self._record(e.key, ok)
                if self._dirty or rewound:            # nodes changed behind the solver's back / device rewound
                    cut = e
                    break
            if cut is None:
                break
            # bindings not yet applied are void: their nodes on the device are ahead of the host objects
            for e in run:
                b = bindings.get(e.pos)
                if e.pos > cut.pos and b is not None and int(b['node']) >= 0:
                    self._touch(self.cluster.name_of(int(b['node'])))
            pos = cut.pos + 1
        return results

    def _explain(self, e: _Pending, counts):
        """Remember and log why pod ``e`` found no node: per reason, the nodes whose first failing stage it was."""
        ns, podname = e.key[0], e.key[1]
        reasons = {name: int(c) for name, c in zip(wire.WHY_NAMES, counts) if int(c)}
        self.unschedulable_reasons[(ns, podname)] = reasons
        total = int(sum(int(c) for c in counts))
        detail = ', '.join(f'{c} {name}' for name, c in sorted(reasons.items(), key=lambda kv: -kv[1]))
        self._info(f'Pod {ns}.{podname}: 0/{total} nodes are available: {detail}')

    def _contention(self, solvable, out, now):
        """{pos: node name or None} for the NO_CANDIDATE pods of the batch just solved: the node each would have been
        placed on alone, at the state the batch started from (a query of the snapshot ``solve`` took).  None when the
        solver in use cannot answer queries."""
        failed = [e for e, b in zip(solvable, out) if int(b['status']) == wire.NO_CANDIDATE]
        q = self.cluster.query([e.top for e in failed], [e.groups for e in failed], now, source='snapshot',
                               packed=[e.rec for e in failed])
        if q is None:
            return None
        placed = self._placements(failed, q)          # a pod listed twice is read and queried the same both times
        return {e.pos: placed[(e.key[0], e.key[1])] for e in failed}

    def _contended(self, e: _Pending, nodename):
        """Remember and log that pod ``e`` found no node although it would have fit alone on ``nodename`` at the start
        of its batch (earlier pods of the batch took the capacity); forget it when it would not have fit either."""
        key = (e.key[0], e.key[1])
        if nodename is None:
            self.contended_pods.pop(key, None)
            return
        self.contended_pods[key] = nodename
        self._info(f'Pod {key[0]}.{key[1]}: would have fit on node {nodename} alone; earlier pods of the same batch '
                   f'took the capacity')

    def _record(self, key, ok: bool):                 # the two branches of CheckPendingPods (:431-436)
        podkey = (key[0], key[1])
        if ok:
            self.contended_pods.pop(podkey, None)
            self.unschedulable_reasons.pop(podkey, None)
            self.pod_state[podkey] = {'state': PodStatus.POD_STATUS_SCHEDULED, 'time': self._wall(), 'uid': key[2]}
        else:
            self._error(f'Failed scheduling pod {key[0]}.{key[1]} [{key[2]}]')
            self.pod_state[podkey] = {'state': PodStatus.POD_STATUS_FAILED, 'time': self._wall(), 'uid': '0'}

    def AttemptScheduling(self, podname, ns) -> bool:
        """Single pod, reference signature (``:249``): a batch of one."""
        saved = self.pod_state.get((ns, podname))
        key = (ns, podname, None)
        ok = self.ScheduleBatch([key])[key]
        if saved is None:                             # the caller owns pod_state for this entry point
            self.pod_state.pop((ns, podname), None)
        else:
            self.pod_state[(ns, podname)] = saved
        return ok

    def PreviewPods(self, keys: Sequence) -> Dict:
        """Where each pod of ``keys`` (``(ns, name[, uid])``) would be placed right now on its own, without scheduling
        anything: ``{(ns, name): node name}``, or None for a pod that would not be placed (no node, a failed
        assignment on the chosen node, a config that does not parse, a request beyond the solver's limits).  The
        pods do not see each other.  Only the Kubernetes reads of a scheduling attempt happen: no event, no write;
        ``pod_state`` and the ``Node`` objects stay as they are.  Nodes the host changed are synced first, as for a
        batch."""
        entries = self._read(keys)
        result = {(e.key[0], e.key[1]): None for e in entries}
        ok = [e for e in entries if e.solvable]
        if not ok or not self.nodes:
            return result
        self._sync()
        now = float(self._clock())
        out, ok, _ = self._without_refused(
            lambda es: self._supported(self.cluster.query([e.top for e in es], [e.groups for e in es], now,
                                                          packed=[e.rec for e in es]),
                                       'answer placement queries (no query_batch)'), ok)
        if ok:
            result.update(self._placements(ok, out))
        return result

    def PlanPods(self, keys: Sequence):
        """Would the pods of ``keys`` (``(ns, name[, uid])``) all be placed if they were scheduled now, in this order?
        A dry run of the batch on the synced cluster: each pod sees the ones before it, nothing is placed.  Returns
        ``(placement, reasons)``: ``placement[(ns, name)]`` is the node the pod would be bound to, or None (no node, a
        failed assignment, a config that does not parse, a request beyond the solver's limits); ``reasons[(ns, name)]``
        is ``{reason name: nodes}`` (``wire.WHY_NAMES``) for each pod that would find no node, as
        ``unschedulable_reasons`` would hold it.  Only the Kubernetes reads of a scheduling attempt happen: no event,
        no write; ``pod_state``, the ``Node`` objects and the counters stay as they are."""
        return self._plan(keys, ())

    def PlanDrain(self, node_names: Sequence[str]):
        """Can these nodes be taken down?  Where the pods now on them (nodes in the given order, pods in
        ``Node.pod_info`` order) would go if they were re-created, read as a scheduling attempt reads them, with those
        nodes in maintenance.  Same dry run and the same ``(placement, reasons)`` as ``PlanPods``."""
        names = list(node_names)
        missing = [n for n in names if n not in self.nodes]
        if missing:
            raise ValueError(f'unknown node(s) {missing}')
        return self._plan(self._pods_on(names), names)

    def PlanDrains(self, node_groups: Sequence[Sequence[str]] = None) -> Dict:
        """Which nodes (or groups of nodes) could be taken down, each group on its own?  ``{tuple(group): placement}``
        with ``placement`` what ``PlanDrain(list(group))[0]`` returns from the same state; by default every node that
        holds pods is its own group, in node order.  All groups are planned side by side in one GPU call; the groups
        do not see each other.  Each pod is read from Kubernetes once, as a scheduling attempt reads it: no event, no
        write; ``pod_state``, the ``Node`` objects and the counters stay as they are.  Reasons are not returned:
        ``PlanDrain(group)`` gives them for the groups that do not drain."""
        groups = self._node_groups(node_groups)
        seen = {}
        group_entries = [self._read(self._pods_on(g), seen) for g in groups]
        result = {}
        todo = []
        for g, entries in zip(groups, group_entries):
            result[g] = {(e.key[0], e.key[1]): None for e in entries}
            ok = [e for e in entries if e.solvable]
            if ok and self.nodes:
                todo.append((g, entries, ok))
        if not todo:
            return result
        self._sync()
        now = float(self._clock())
        res = self._supported(
            self.cluster.plan_scenarios([(g, [e.top for e in ok], [e.groups for e in ok], now, [e.rec for e in ok])
                                         for g, _, ok in todo]), 'plan scenarios (no plan_scenarios)')
        for (g, entries, ok), (code, _, out) in zip(todo, res):
            if out is None:
                # refused (the tuple limits are judged with the group's own nodes counted): the single plan judges
                # them without, and drops a pod beyond them, or raises, as PlanDrain does
                result[g] = self._plan_prepared(entries, list(g), now)[0]
            else:
                result[g].update(self._placements(ok, out))
        return result

    def PlanDefrag(self, keys: Sequence = None, node_groups: Sequence[Sequence[str]] = None,
                   delay: float = None) -> Dict:
        """Which nodes (or groups of nodes), drained and put back in service, would let the pending pods place?  For
        every group, the maintenance workflow planned from the same state, all groups side by side in one GPU call:
          1. ``NODE_MAINT_START`` on the group's nodes;
          2. their pods deleted (each released as ``ReleasePodResources`` releases it: resources back, the node busy
             from now) and re-created, each scheduled at once at the current clock, the group in maintenance;
          3. ``NODE_MAINT_END`` on the group's nodes (back in service, whatever their maintenance flag was);
          4. ``delay`` seconds later, the pods of ``keys`` scheduled in order, as the next ``CheckPendingPods`` would.
        Returns ``{tuple(group): (moved, pending)}``: ``moved[(ns, name)]`` the node each of the group's pods (nodes in
        the given order, pods in ``Node.pod_info`` order, as ``PlanDrain``) goes to, or None; ``pending[(ns, name)]``
        the node each pod of ``keys`` goes to, or None.  ``pending`` is None when some moved pod found no node: the
        next scan would retry that pod too, so the group does not resolve the fragmentation it was planned for.
        ``keys`` (``(ns, name[, uid])``) defaults to the pods the next ``CheckPendingPods`` would attempt, in its
        order; ``node_groups`` to every node holding pods on its own, in node order.  ``delay`` defaults to
        ``MIN_BUSY_SECS``: the first moment the released nodes (busy from the release) take GPU pods again; with less,
        a GPU pod of ``keys`` does not see them.  A group holding a pod that was never annotated is not planned
        (its delete would re-scan every node): its pods map to None and ``pending`` is None.
        Only reads happen, as ``PlanDrains``: each pod is read from Kubernetes once (a scheduling attempt's reads and
        a release's); the releases run on copies of the ``Node`` objects; ``pod_state``, the ``Node`` objects and the
        counters stay as they are."""
        groups = self._node_groups(node_groups)
        if keys is None:
            phase = self._service_pods()
            keys = [k for k in phase if self._wanted(phase)(k)]
        delay = float(self._node_cls.MIN_BUSY_SECS if delay is None else delay)
        seen, targets = {}, {}
        tail = [e for e in self._read([(k[0], k[1]) for k in keys], seen) if e.solvable]
        group_pods = [self._pods_on(g) for g in groups]
        for key in (key for pods in group_pods for key in pods):
            if key not in targets:
                targets[key] = self._release_target(key[1], key[0])
        entries = [self._read(pods, seen) for pods in group_pods]
        result = {g: ({key: None for key in pods}, None) for g, pods in zip(groups, group_pods)}
        if not self.nodes:
            return result
        self._sync()
        now = float(self._clock())
        todo = []
        for g, pods, moved in zip(groups, group_pods, entries):
            if any(targets[key] is None for key in pods):
                continue
            edits = {}
            for n in g:
                edits[n] = _copy_node(self.nodes[n])
                edits[n].maintenance = False                       # NODE_MAINT_END
            for key in pods:
                node, top = targets[key]
                if node is None:
                    continue
                if node not in edits:
                    edits[node] = _copy_node(self.nodes[node])
                self._give_back(edits[node], key[1], key[0], top, now)
            todo.append((g, [e for e in moved if e.solvable], tail, edits))
        while todo:
            res = self._supported(self.cluster.plan_scenarios([self._defrag_scenario(g, ok, tail, edits, now, delay)
                                                               for g, ok, tail, edits in todo]),
                                  'plan scenarios (no plan_scenarios)')
            retry = []
            for (g, ok, tail, edits), (code, pod, out) in zip(todo, res):
                if out is None:
                    # a pod beyond the tuple limits (judged with the group's nodes and the edited records counted):
                    # it gets None, as in PlanDrain, and the group is planned again without it
                    if code != wire.ERR_UNSUPPORTED:
                        raise RuntimeError(f'nhd_plan_scenarios_edited refused group {g}: code {code}, pod {pod}')
                    if pod < len(ok):
                        ok = ok[:pod] + ok[pod + 1:]
                    else:
                        tail = tail[:pod - len(ok)] + tail[pod - len(ok) + 1:]
                    retry.append((g, ok, tail, edits))
                    continue
                moved, _ = result[g]
                moved.update(self._placements(ok, out[:len(ok)]))
                if all(v is not None for v in moved.values()):
                    pending = {(k[0], k[1]): None for k in keys}
                    pending.update(self._placements(tail, out[len(ok):]))
                    result[g] = (moved, pending)
            todo = retry
        return result

    @staticmethod
    def _defrag_scenario(g, moved, tail, edits, now, delay):
        """One ``PlanDefrag`` group as a ``DeviceCluster.plan_scenarios`` scenario."""
        pods = moved + tail
        clock = [now] * len(moved) + [now + delay] * len(tail)
        return (g, [e.top for e in pods], [e.groups for e in pods], clock, [e.rec for e in pods], len(moved), edits)

    def _plan(self, keys: Sequence, exclude: Sequence[str]):
        entries = self._read(keys)
        if not self.nodes or not any(e.solvable for e in entries):
            return {(e.key[0], e.key[1]): None for e in entries}, {}
        self._sync()
        return self._plan_prepared(entries, exclude, float(self._clock()))

    def _plan_prepared(self, entries: Sequence, exclude: Sequence[str], now: float):
        """``_plan`` from pods already read from Kubernetes, on the synced cluster at clock ``now``."""
        placement = {(e.key[0], e.key[1]): None for e in entries}
        res, ok, _ = self._without_refused(
            lambda es: self._supported(self.cluster.plan([e.top for e in es], [e.groups for e in es], now,
                                                         exclude=exclude, packed=[e.rec for e in es], explain=True),
                                       'plan batches (no plan_batch)'), [e for e in entries if e.solvable])
        if not ok:
            return placement, {}
        out, counts = res
        placement.update(self._placements(ok, out))
        reasons = {(e.key[0], e.key[1]): {name: int(n) for name, n in zip(wire.WHY_NAMES, c) if int(n)}
                   for e, b, c in zip(ok, out, counts) if int(b['status']) == wire.NO_CANDIDATE}
        return placement, reasons

    # ---- shared by the batch, the previews and the plans ------------------------------------------------------
    def _read(self, keys: Sequence, seen: Dict = None) -> List[_Pending]:
        """The pods ``keys`` read from Kubernetes as a scheduling attempt reads them, without its events
        (``_prepare(events=False)``).  ``seen``: a dict, shared by calls that read each pod once, from key to entry."""
        entries = []
        for i, k in enumerate(keys):
            e = None if seen is None else seen.get(k)
            if e is None:
                e = _Pending(i, k)
                self._prepare(e, events=False)
                if seen is not None:
                    seen[k] = e
            entries.append(e)
        return entries

    def _pods_on(self, names: Sequence[str]) -> List[tuple]:
        """``(ns, name)`` of the pods on the nodes ``names``: nodes in the given order, pods in ``Node.pod_info``
        order."""
        return [(ns, pod) for n in names for (pod, ns) in self.nodes[n].pod_info]

    def _node_groups(self, node_groups) -> List[tuple]:
        """``node_groups`` as tuples, by default every node that holds pods on its own, in node order."""
        if node_groups is None:
            node_groups = [[n] for n, v in self.nodes.items() if v.pod_info]
        groups = [tuple(g) for g in node_groups]
        missing = sorted({n for g in groups for n in g if n not in self.nodes})
        if missing:
            raise ValueError(f'unknown node(s) {missing}')
        return groups

    @staticmethod
    def _without_refused(call: Callable, entries: Sequence):
        """``call(entries)`` without the pods the library refuses.  A request beyond the limit that depends on the
        cluster as well (numa^(groups+1) tuples, include/nhd_b200.h) makes the library refuse the whole call and name
        the pod; that entry is dropped and ``call`` made again with the rest.  Returns ``(result, kept entries,
        [(dropped entry, error)])``, ``result`` None when every entry was dropped.  Any other error propagates."""
        kept, dropped = list(entries), []
        while kept:
            try:
                return call(kept), kept, dropped
            except Exception as err:
                m = re.search(r'pod (\d+)', str(err)) if getattr(err, 'code', None) == wire.ERR_UNSUPPORTED else None
                if m is None or int(m.group(1)) >= len(kept):
                    raise
                dropped.append((kept.pop(int(m.group(1))), err))
        return None, kept, dropped

    def _placements(self, entries: Sequence, out) -> Dict:
        """``{(ns, name): node name}`` of ``entries`` from their bindings ``out``, None for a pod not placed (a pod
        listed twice keeps the node either entry got)."""
        placement = {(e.key[0], e.key[1]): None for e in entries}
        for e, b in zip(entries, out):
            if int(b['status']) == wire.PLACED:
                placement[(e.key[0], e.key[1])] = self.cluster.name_of(int(b['node']))
        return placement

    @staticmethod
    def _supported(res, what: str):
        """``res``, the answer of a ``DeviceCluster`` call that is None when the solver in use lacks the method."""
        if res is None:
            raise RuntimeError(f'the solver in use cannot {what}')
        return res

    def CheckPendingPods(self):
        """``NHDScheduler.py:425-441`` with the pending set solved as one batch."""
        phase = self._service_pods()
        self.ScheduleBatch(list(phase), self._wanted(phase))
        # The reference's second branch (:437-440) compares the pod_state *dict* with an enum member and
        # therefore never runs; a pod reported 'Failed' keeps its resources until its delete event.

    def _service_pods(self):
        """``{(ns, name, uid): (phase, node)}`` of every pod of this scheduler, in Kubernetes' order."""
        podlist = self.k8s.ServicePods(self.sched_name)
        return {(k[0], k[1], k[2]): p for k, p in podlist.items()}

    def _wanted(self, phase):
        """The pods of ``phase`` (``_service_pods``) that ``CheckPendingPods`` attempts: pending, unbound and not
        scheduled here.  Asked again after a cut, since a reset clears ``pod_state``."""
        def wanted(k):
            p = phase[k]
            podkey = (k[0], k[1])
            return (p[0] == 'Pending' and p[1] == None and                     # noqa: E711
                    ((podkey not in self.pod_state) or
                     self.pod_state[podkey]['state'] != PodStatus.POD_STATUS_SCHEDULED))
        return wanted

    # ---- the thread function (NHDScheduler.py:443-577) ------------------------------------------------
    def Startup(self):
        """What ``run`` does before its loop (``:448-455``)."""
        self.BuildInitialNodeList()
        self.LoadDeployedConfigs()
        self.CheckPendingPods()

    def run(self, nqueue, idle_thresh: int = 60, block_secs: float = 0.5, stop: Callable[[], bool] = None):
        """The reference's loop: watch items first, else one gRPC request, else count idleness and
        re-scan the pending pods every ``idle_thresh`` empty polls (``:468-489``)."""
        from queue import Empty
        self.Startup()
        try:                                           # drop what piled up during start-up (:459-465)
            while True:
                nqueue.get(block=False, timeout=0)
        except Empty:
            pass
        idle_cnt = 0
        while stop is None or not stop():
            try:
                item = nqueue.get(block=False)
            except Empty:
                try:
                    item = self.rpcq.get(True, block_secs)
                    self.ParseRPCReq(item[0], item[1])
                except Empty:
                    idle_cnt += 1
                    if idle_cnt >= idle_thresh:
                        idle_cnt = 0
                        self.CheckPendingPods()
                continue
            self.HandleWatchItem(item)

    # ---- watch queue (NHDScheduler.py:491-577) -----------------------------------------------------
    def HandleWatchItem(self, item):
        t = _type_name(item["type"])
        if t in ('NHD_WATCH_TYPE_TRIAD_POD_DELETE', 'NHD_WATCH_TYPE_TRIAD_POD_CREATE'):
            ns, pn, uid = item["pod"]["ns"], item["pod"]["name"], item["pod"]["uid"]
            if t == 'NHD_WATCH_TYPE_TRIAD_POD_DELETE':
                self.ReleasePodResources(pn, ns)
                self.pod_state.pop((ns, pn), None)
                self.unschedulable_reasons.pop((ns, pn), None)
                self.contended_pods.pop((ns, pn), None)
            else:
                if ((ns, pn) in self.pod_state) and \
                        (self.pod_state[(ns, pn)]['state'] == PodStatus.POD_STATUS_SCHEDULED):
                    if self.pod_state[(ns, pn)]['uid'] == uid:
                        return
                    self.ReleasePodResources(pn, ns)
                    self.pod_state.pop((ns, pn), None)
                key = (ns, pn, uid)
                if self.ScheduleBatch([key])[key]:
                    self.pod_state[(ns, pn)] = {'state': PodStatus.POD_STATUS_SCHEDULED, 'time': self._wall(),
                                                'uid': uid}
                else:
                    self.pod_state[(ns, pn)] = {'state': PodStatus.POD_STATUS_FAILED, 'time': 0, 'uid': '0'}
        elif t in ('NHD_WATCH_TYPE_NODE_CORDON', 'NHD_WATCH_TYPE_NODE_UNCORDON'):
            v = self.nodes.get(item["node"])
            if v is not None:
                want = t == 'NHD_WATCH_TYPE_NODE_UNCORDON'
                if v.active != want:
                    v.active = want
                    self._touch(item["node"])
        elif t in ('NHD_WATCH_TYPE_NODE_MAINT_START', 'NHD_WATCH_TYPE_NODE_MAINT_END'):
            v = self.nodes.get(item["node"])
            if v is not None:
                want = t == 'NHD_WATCH_TYPE_NODE_MAINT_START'
                if v.maintenance != want:
                    v.maintenance = want
                    self._touch(item["node"])
        elif t == 'NHD_WATCH_TYPE_GROUP_UPDATE':
            v = self.nodes.get(item["node"])
            if v is not None:
                v.SetGroups(item["groups"])
                self._touch(item["node"])

    # ---- statistics (NHDScheduler.py:355-423) --------------------------------------------------------
    def GetBasicNodeStats(self):
        nodes = []
        for k, v in self.nodes.items():
            nodes.append({'name': k,
                          'freegpu': v.GetFreeGpuCount(),
                          'totalgpu': v.GetTotalGPUs(),
                          'freecpu': v.GetFreeCpuCoreCount(),
                          'totalcpu': v.GetTotalCPUs(),
                          'freehuge_gb': v.GetFreeHugepages(),
                          'totalhuge_gb': v.GetTotalHugepages(),
                          'totalpods': v.GetTotalPods(),
                          'active': v.GetNodeActive(),
                          'nicstats': v.GetNICUsedSpeeds()})
        return nodes

    def GetBasicNodeStatsFromDevice(self):
        """The same rows with the counters that are placement state taken from the GPU's records
        (``nhd_read_nodes`` + ``nhd_node_stats_from_records``) instead of walking the Python objects;
        ``totalhuge_gb``, ``totalpods`` and ``nicstats`` are not placement state and come from the host."""
        from nhd_b200 import ingest
        self._sync()
        st = ingest.node_stats(self.cluster.read_records())
        rows = []
        by_name = {r['name']: r for r in self.GetBasicNodeStats()} if self.cluster.stubs else {}
        for i, (k, v) in enumerate(self.nodes.items()):
            if k in self.cluster.stubs:              # no usable record: the half-initialised object answers
                rows.append(by_name[k])
                continue
            s = st[i]
            rows.append({'name': k,
                         'freegpu': int(s['freegpu']), 'totalgpu': int(s['totalgpu']),
                         'freecpu': int(s['freecpu']), 'totalcpu': int(s['totalcpu']),
                         'freehuge_gb': int(s['freehuge_gb']), 'totalhuge_gb': v.GetTotalHugepages(),
                         'totalpods': v.GetTotalPods(), 'active': bool(s['active']),
                         'nicstats': v.GetNICUsedSpeeds()})
        return rows

    def GetPodStats(self):
        pinfo = []
        for k, v in self.nodes.items():
            for pname, pval in v.pod_info.items():
                # pod_info is keyed (pod, ns) (Node.py:205-208); the reference passes the two in this order to
                # GetPodAnnotations(podname, ns) (NHDScheduler.py:388), i.e. swapped, so unless a pod's name
                # equals its namespace the lookup fails and the pod is skipped.  Kept as is.
                annots = self.k8s.GetPodAnnotations(pname[1], pname[0])
                if annots == None:                   # noqa: E711
                    continue
                pinfo.append({
                    'namespace': pname[1],
                    'podname': pname[0],
                    'node': k,
                    'annotations': annots,
                    'hugepages': pval.hugepages_gb,
                    'proc_cores': [pc.core for pg in pval.proc_groups for pc in pg.proc_cores],
                    'proc_helper_cores': [pc.core for pg in pval.proc_groups for pc in pg.misc_cores],
                    'misc_cores': [pc.core for pc in pval.misc_cores],
                    'gpus': [g.device_id for pg in pval.proc_groups for g in pg.group_gpus],
                    'nics': [np_.mac for np_ in pval.nic_core_pairing],
                })
        return pinfo

    def ParseRPCReq(self, msgid, q: Queue):
        t = _type_name(msgid)
        if t == 'TYPE_NODE_INFO':
            q.put(self.GetBasicNodeStatsFromDevice() if self.stats_from_device and self.nodes
                  else self.GetBasicNodeStats())
        elif t == 'TYPE_SCHEDULER_INFO':
            q.put(self.failed_schedule_count)
        elif t == 'TYPE_POD_INFO':
            q.put(self.GetPodStats())
