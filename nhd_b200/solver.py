"""``Solver`` — thin object wrapper over the C-ABI handle (include/nhd_b200.h).

Works on packed numpy records (``nhd_b200.wire``); the object-level drop-in lives in
``nhd_b200.Matcher``.  All compute happens in the CUDA library."""
import ctypes
import os
from typing import NamedTuple, Optional, Sequence

import numpy as np

from nhd_b200 import _lib, wire

ERR_NAMES = {-1: 'NHD_ERR_INVALID', -2: 'NHD_ERR_UNSUPPORTED', -3: 'NHD_ERR_CUDA', -4: 'NHD_ERR_NCCL',
             -5: 'NHD_ERR_STATE'}


class SolverError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f'{ERR_NAMES.get(code, code)}: {msg}')
        self.code = code


def nccl_unique_id() -> bytes:
    buf = (ctypes.c_uint8 * 128)()
    rc = _lib.load().nhd_nccl_unique_id(buf)
    if rc != 0:
        raise SolverError(rc, 'nhd_nccl_unique_id')
    return bytes(buf)


def shard_min_pairs() -> int:
    """(nodes x distinct pod types) from which a world_size > 1 handle created now would node-shard its filter
    (``nhd_shard_min_pairs``; ``NHD_SHARD_MIN_PAIRS`` in the environment of every rank overrides the default)."""
    return int(_lib.load().nhd_shard_min_pairs())


def pinned_array(n, dtype):
    """numpy array of n records in page-locked host memory (nhd_alloc_pinned): such buffers go to
    and from the device without a staging copy.  Keep the returned array alive while in use."""
    L = _lib.load()
    dtype = np.dtype(dtype)
    nbytes = max(1, n * dtype.itemsize)
    ptr = ctypes.c_void_p()
    rc = L.nhd_alloc_pinned(nbytes, ctypes.byref(ptr))
    if rc != 0:
        raise SolverError(rc, 'nhd_alloc_pinned')
    buf = (ctypes.c_char * nbytes).from_address(ptr.value)
    arr = np.frombuffer(buf, dtype=dtype, count=n)
    _PINNED[id(arr)] = (ptr, buf)
    return arr


_PINNED = {}


def _source(source):
    """The ``nhd_query_batch`` / ``nhd_plan_*`` source code of ``'mirror'`` or ``'snapshot'``."""
    src = {'mirror': wire.QUERY_MIRROR, 'snapshot': wire.QUERY_SNAPSHOT}.get(source)
    if src is None:
        raise ValueError(f"source must be 'mirror' or 'snapshot', not {source!r}")
    return src


class Scenario(NamedTuple):
    """One dry run of ``Solver.plan_scenarios``.

    ``exclude``: node indices taken as in maintenance; ``pods``, ``now``: the scenario's ``wire.POD_DTYPE`` pods and
    their clocks, planned in order.  ``lift`` (None: never): the excluded nodes are back in service from the scenario's
    pod ``lift`` on.  ``edits`` (None: none): ``(nodes, records)``, node indices and a ``wire.NODE_DTYPE`` array, the
    records those nodes have for the whole scenario.  ``adds`` (None: none): ``(at, records)``, int positions and a
    ``wire.NODE_DTYPE`` array: nodes added for the whole scenario, each right before source node ``at[k]``
    (``n_nodes``: at the end), ``at`` never going down.  ``rounds`` (None: none): the clocks of later pending scans,
    never going down and none before the scenario's pod clocks; at each, the scenario's pods not placed yet are solved
    again in order on the records the previous scan left, and the bindings hold each pod's last attempt.  ``releases``
    (None: none): ``(tracked, pods_used, releases)`` as ``plan_batch_releases`` takes them, node indices of source
    nodes the scenario does not edit, each release applied before its ``round`` (1 .. ``len(rounds)``).  ``arrive``
    (None: every pod pending at the start): per pod the round ``r`` in the gap before which it is created, at its own
    clock, and first attempted then (0: pending at the start); the round-0 pods come first and ``(arrive, now)`` never
    goes down in pod order."""
    exclude: Sequence[int]
    pods: np.ndarray
    now: Sequence[float]
    lift: Optional[int] = None
    edits: Optional[tuple] = None
    adds: Optional[tuple] = None
    rounds: Optional[Sequence[float]] = None
    releases: Optional[tuple] = None
    arrive: Optional[Sequence[int]] = None


class Solver:
    def __init__(self, speed_table, nic_bw_avail_percent=0.9, min_busy_secs=30.0, device=0,
                 rank=0, world_size=1, nccl_id: bytes = None, single_warp: bool = False, cpu_warps: int = 0,
                 sweep_debug: int = 0):
        self._L = _lib.load()
        p = _lib.Params()
        self._L.nhd_default_params(ctypes.byref(p))
        p.nic_bw_avail_percent = nic_bw_avail_percent
        p.min_busy_secs = min_busy_secs
        speeds = [float(x) for x in speed_table]
        nz = max([i + 1 for i, s in enumerate(speeds) if s != 0.0], default=0)
        p.n_speed_classes = nz
        for i, s in enumerate(speeds[:16]):
            p.speed_gbps[i] = s
        p.device, p.rank, p.world_size = device, rank, world_size
        # test knobs (all settings produce identical bindings): single_warp = the general one-warp sweep only;
        # cpu_warps = 1: never sweep the two pod classes side by side; sweep_debug bit 0: no standing decisions,
        # bit 1: same as cpu_warps = 1, bit 2: no direct-path tables in the sweep (warp-wide evaluation everywhere)
        p.reserved_ = (1 if single_warp else (cpu_warps + 1 if cpu_warps else 0)) | \
            ((int(sweep_debug) | int(os.environ.get('NHD_SWEEP_DEBUG', '0'))) << 8)
        if world_size > 1:
            if not nccl_id or len(nccl_id) != 128:
                raise ValueError('world_size > 1 needs the 128-byte NCCL unique id of rank 0')
            ctypes.memmove(p.nccl_unique_id, nccl_id, 128)
        self._h = ctypes.c_void_p()
        rc = self._L.nhd_create(ctypes.byref(p), ctypes.byref(self._h))
        if rc != 0:
            msg = self._L.nhd_last_error(self._h).decode() if self._h else 'no usable CUDA device (no CPU fallback)'
            if self._h:
                self._L.nhd_destroy(self._h)
                self._h = None
            raise SolverError(rc, msg)
        self.n_nodes = 0
        self.n_pods = 0

    def close(self):
        if getattr(self, '_h', None):
            self._L.nhd_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise SolverError(rc, self._L.nhd_last_error(self._h).decode())

    # ---- cluster mirror -------------------------------------------------------------
    def load_nodes(self, recs):
        recs = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE)
        self._ck(self._L.nhd_load_nodes(self._h, len(recs), recs.ctypes.data))
        self.n_nodes = len(recs)

    def update_nodes(self, idx, recs):
        idx = np.ascontiguousarray(idx, dtype='<i4')
        recs = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE)
        assert len(idx) == len(recs)
        self._ck(self._L.nhd_update_nodes(self._h, len(idx), idx.ctypes.data, recs.ctypes.data))

    def read_nodes(self, first=0, n=None):
        n = self.n_nodes - first if n is None else n
        out = np.zeros(n, dtype=wire.NODE_DTYPE)
        self._ck(self._L.nhd_read_nodes(self._h, first, n, out.ctypes.data))
        return out

    def snapshot(self):
        self._ck(self._L.nhd_snapshot(self._h))

    def restore(self):
        self._ck(self._L.nhd_restore(self._h))

    # ---- batches --------------------------------------------------------------------
    def solve_batch(self, pods, now, out=None):
        pods = np.ascontiguousarray(pods, dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(now, dtype='<f8')
        assert len(pods) == len(now)
        if out is None:
            out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        self._ck(self._L.nhd_solve_batch(self._h, len(pods), pods.ctypes.data, now.ctypes.data, out.ctypes.data))
        self.n_pods = len(pods)
        return out

    def stage_batch(self, pods, now):
        pods = np.ascontiguousarray(pods, dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(now, dtype='<f8')
        assert len(pods) == len(now)
        self._ck(self._L.nhd_stage_batch(self._h, len(pods), pods.ctypes.data, now.ctypes.data))
        self.n_pods = len(pods)

    def solve_staged(self):
        self._ck(self._L.nhd_solve_staged(self._h))

    def sync(self):
        self._ck(self._L.nhd_sync(self._h))

    def fetch_bindings(self, out=None):
        if out is None:
            out = np.zeros(self.n_pods, dtype=wire.BINDING_DTYPE)
        self._ck(self._L.nhd_fetch_bindings(self._h, out.ctypes.data))
        return out

    def timing(self):
        t = _lib.Timing()
        self._ck(self._L.nhd_last_timing(self._h, ctypes.byref(t)))
        return {k: getattr(t, k) for k, _ in t._fields_}

    def debug_counters(self):
        out = np.zeros(64, dtype='<u8')
        self._ck(self._L.nhd_debug_counters(self._h, out.ctypes.data))
        return out

    # ---- explanations ---------------------------------------------------------------
    def explain_batch(self):
        """(n_pods, WHY_COUNT) uint32: for every NO_CANDIDATE pod of the last solved batch, how many nodes each
        reference stage (``wire.WHY_NAMES``, first stage that drops the node) ruled out, at the state that pod saw;
        zero rows for the other pods.  Needs ``snapshot()`` right before the batch was staged."""
        out = np.zeros((self.n_pods, wire.WHY_COUNT), dtype='<u4')
        self._ck(self._L.nhd_explain_batch(self._h, out.ctypes.data))
        return out

    def explain_pod(self, i):
        """(n_nodes,) uint8: the reason code of every node for pod ``i`` of the last solved batch
        (``wire.WHY_NONE`` everywhere when that pod is not NO_CANDIDATE)."""
        out = np.zeros(self.n_nodes, dtype=np.uint8)
        self._ck(self._L.nhd_explain_pod(self._h, int(i), out.ctypes.data))
        return out

    # ---- placement queries ----------------------------------------------------------
    def query_batch(self, pods, now, source='mirror', out=None):
        """Where each pod would go on its own (``nhd_query_batch``): per pod the binding ``solve_batch`` would return
        for that pod alone, on the current records (``source='mirror'``) or on those of the last ``snapshot()``
        (``'snapshot'``).  Nothing is placed: records, snapshot, the last batch and its explanations stay as they are."""
        src = _source(source)
        pods = np.ascontiguousarray(pods, dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(now, dtype='<f8')
        assert len(pods) == len(now)
        if out is None:
            out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        self._ck(self._L.nhd_query_batch(self._h, src, len(pods), pods.ctypes.data, now.ctypes.data, out.ctypes.data))
        return out

    def plan_batch(self, pods, now, source='mirror', exclude=(), explain=False, out=None):
        """A dry run of ``solve_batch``: the bindings the pods would get scheduled in order, each seeing the ones before
        it, on the current records (``source='mirror'``) or on those of the last ``snapshot()`` (``'snapshot'``), with
        the node indices ``exclude`` taken as in maintenance.  With ``explain=True`` returns ``(bindings, counts)``,
        counts being what ``explain_batch`` would return after that solve.  Nothing is placed: records, snapshot, the
        last batch and its explanations stay as they are."""
        out, _, counts = self._plan_batch(pods, now, source, exclude, explain, out)
        return (out, counts) if explain else out

    def plan_batch_rounds(self, pods, now, round_clocks, source='mirror', exclude=(), explain=False):
        """``plan_batch`` over several pending scans: after the dry run of the batch, at each clock of ``round_clocks``
        (never going down, none before a pod clock) the pods not placed yet are solved again in order on the records the
        previous scan left, the nodes ``exclude`` in maintenance throughout.  Returns ``(bindings, pod_round)``: each
        pod's last attempt and the round that placed it, or ``len(round_clocks)`` if none did; ``explain=True``:
        ``(bindings, pod_round, counts)``, ``counts`` the per-reason node counts of the pods whose last attempt found no
        node, at that attempt.  The same answer as ``plan_scenarios`` with this one scenario and rounds, from the batch
        path: meant for one large pending set.  Nothing is placed."""
        out, pod_round, counts = self._plan_batch(pods, now, source, exclude, explain, round_clocks=round_clocks)
        return (out, pod_round, counts) if explain else (out, pod_round)

    def plan_batch_releases(self, pods, now, round_clocks, tracked, pods_used, releases, source='mirror', exclude=(),
                            explain=False):
        """``plan_batch_rounds`` with deployed pods ending between the scans.  ``releases``: ``wire.RELEASE_DTYPE``
        records, each applied before its ``round`` (1 .. ``len(round_clocks)``), in array order, clocks never going
        down.  ``tracked``: the node indices whose signed NIC pod counters the plan carries, every released node among
        them; ``pods_used``: ``(len(tracked), MAX_NICS)`` counters at plan start.  Returns what ``plan_batch_rounds``
        returns.  Nothing is placed."""
        out, pod_round, counts = self._plan_batch(pods, now, source, exclude, explain, round_clocks=round_clocks,
                                                  tracked=tracked, pods_used=pods_used, releases=releases)
        return (out, pod_round, counts) if explain else (out, pod_round)

    def plan_batch_arrivals(self, pods, now, round_clocks, tracked, pods_used, releases, arrive_round,
                            source='mirror', exclude=(), explain=False):
        """``plan_batch_releases`` with pods created between the scans, on the batch path: ``arrive_round[i]`` 0 for a
        pod pending at the start, else the round ``r`` (1 .. ``len(round_clocks)``) in whose gap the pod is created, at
        ``now[i]``; the round-0 pods come first and ``(arrive_round, now)`` never goes down.  Each gap plays its
        releases and its arrivals' first attempts merged by clock (a release first at an equal clock), and its scan
        retries every arrived pod not placed yet, the gap's failed arrivals after the older pods.  The exclusions hold
        throughout.  Returns ``(bindings, pod_round, pod_clock)``, ``pod_clock`` the clock of the attempt whose binding
        is given; ``explain=True``: ``(bindings, pod_round, pod_clock, counts)``.  The same answer as ``plan_scenarios``
        with this one timeline as a scenario with ``arrive``, from the batch path: meant for one large timeline.
        Nothing is placed."""
        out, pod_round, counts, pod_clock = self._plan_batch(
            pods, now, source, exclude, explain, round_clocks=round_clocks, tracked=tracked, pods_used=pods_used,
            releases=releases, arrive_round=arrive_round)
        return (out, pod_round, pod_clock, counts) if explain else (out, pod_round, pod_clock)

    def _plan_batch(self, pods, now, source, exclude, explain, out=None, round_clocks=None, tracked=(), pods_used=(),
                    releases=None, arrive_round=None):
        """The three ``plan_batch*`` methods as one ``nhd_plan_batch_releases`` call (no rounds, no tracked nodes and no
        releases are what the two narrower entry points pass): ``(bindings, pod_round, counts or None)``, ``pod_round``
        None without ``round_clocks``.  With ``arrive_round`` the call is ``nhd_plan_batch_arrivals`` and the result
        gains the pod clocks."""
        src = _source(source)
        pods = np.ascontiguousarray(pods, dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(now, dtype='<f8')
        assert len(pods) == len(now)
        ex = np.ascontiguousarray(exclude, dtype='<i4').reshape(-1)
        clocks = np.ascontiguousarray(() if round_clocks is None else round_clocks, dtype='<f8').reshape(-1)
        tr = np.ascontiguousarray(tracked, dtype='<i4').reshape(-1)
        used = np.ascontiguousarray(pods_used, dtype='<i2').reshape(len(tr), wire.MAX_NICS)
        rel = (np.zeros(0, dtype=wire.RELEASE_DTYPE) if releases is None else
               np.ascontiguousarray(releases, dtype=wire.RELEASE_DTYPE).reshape(-1))
        if out is None:
            out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        pod_round = None if round_clocks is None else np.zeros(len(pods), dtype='<i4')
        counts = np.zeros((len(pods), wire.WHY_COUNT), dtype='<u4') if explain else None
        args = [self._h, src, len(ex), ex.ctypes.data if len(ex) else None, len(pods), pods.ctypes.data,
                now.ctypes.data, len(clocks), clocks.ctypes.data if len(clocks) else None, len(tr),
                tr.ctypes.data if len(tr) else None, used.ctypes.data if len(tr) else None, len(rel),
                rel.ctypes.data if len(rel) else None]
        tail = [out.ctypes.data, counts.ctypes.data if explain else None,
                None if pod_round is None else pod_round.ctypes.data]
        if arrive_round is None:            # every existing call goes out as before
            self._ck(self._L.nhd_plan_batch_releases(*args, *tail))
            return out, pod_round, counts
        arrive = np.ascontiguousarray(arrive_round, dtype='<i4').reshape(-1)
        assert len(arrive) == len(pods)
        pod_clock = np.zeros(len(pods), dtype='<f8')
        self._ck(self._L.nhd_plan_batch_arrivals(*args, arrive.ctypes.data, *tail, pod_clock.ctypes.data))
        return out, pod_round, counts, pod_clock

    def plan_scenarios(self, scenarios, source='mirror', explain=False):
        """Many independent dry runs in one call.  ``scenarios``: a sequence of ``Scenario`` records, or plain tuples of
        their fields in order (``(exclude, pods, now[, lift[, edits[, adds[, rounds]]]])``).  Returns one ``(code, pod,
        bindings)`` per scenario: ``code`` 0 and ``bindings`` what ``plan_batch(pods, now, source, exclude)`` returns,
        or the refusal ``plan_batch`` would raise (``wire.ERR_*``), the index of the pod it names and None.
        ``explain=True``: one ``(code, pod, bindings, counts)`` per scenario, ``counts`` a ``(n_s, wire.WHY_COUNT)``
        uint32 array of per-reason node counts for the NO_CANDIDATE pods at the state each saw (zero rows for the
        others), as ``plan_batch(..., explain=True)`` gives them, or None when refused.  Scenarios do not see each
        other.  Unlike ``plan_batch`` the tuple limits are judged with the excluded nodes counted; ``plan_batch`` plans
        a scenario refused for that.  With ``lift``, ``edits`` or ``adds`` the bindings are those of ``solve_batch`` on
        a scratch copy of the records with the edits applied and the additions inserted, the excluded nodes in
        maintenance for the pods before ``lift`` and back after.  A pod placed on an added node gets node
        ``n_nodes + a``, ``a`` its index among the added records of the whole call, in scenario order.  When any
        scenario has ``rounds``, each result gains a last element: the ``(n_s,)`` int32 round that placed each pod, or
        ``len(rounds)`` if none did (None when refused).  When any scenario has ``releases`` the call is
        ``nhd_plan_scenarios_releases``: that scenario's deployed pods end between its rounds, each scenario on its own
        records and NIC counters.  When any scenario has ``arrive`` the call is ``nhd_plan_scenarios_arrivals``: each
        later pod is first attempted alone at its clock, merged with its gap's releases, and retried at every scan from
        then on; each accepted result then also gains a last element, the ``(n_s,)`` float64 clock of the attempt whose
        binding it holds."""
        src = _source(source)
        # (thousands of small scenarios: gathered as bytes, since numpy's per-array checks of the structured pod dtype
        # would cost more than the call itself)
        exs, podb, nowl, lifts, ednodes, edrecs, n_adds, adats, adrecs, rounds = [], [], [], [], [], [], [], [], [], []
        rels, arrs = [], []
        for sc in scenarios:
            sc = Scenario(*sc)
            rounds.append(sc.rounds)
            rels.append(sc.releases)
            arrs.append(sc.arrive)
            pods = np.asarray(sc.pods)
            if pods.dtype != wire.POD_DTYPE:
                pods = pods.astype(wire.POD_DTYPE)
            exs.append(np.asarray(sc.exclude, dtype='<i4').reshape(-1))
            podb.append(np.ascontiguousarray(pods).tobytes())
            nowl.append(np.asarray(sc.now, dtype='<f8').reshape(-1))
            assert pods.size == len(nowl[-1])
            lifts.append(len(nowl[-1]) if sc.lift is None else int(sc.lift))
            if sc.edits is None:
                ednodes.append(np.zeros(0, dtype='<i4'))
            else:
                nodes, recs = sc.edits
                ednodes.append(np.asarray(nodes, dtype='<i4').reshape(-1))
                recs = np.asarray(recs, dtype=wire.NODE_DTYPE).reshape(-1)
                assert len(recs) == len(ednodes[-1])
                edrecs.append(recs.tobytes())
            if sc.adds is None:
                n_adds.append(0)
            else:
                at, recs = sc.adds
                adats.append(np.asarray(at, dtype='<i4').reshape(-1))
                recs = np.asarray(recs, dtype=wire.NODE_DTYPE).reshape(-1)
                assert len(recs) == len(adats[-1])
                adrecs.append(recs.tobytes())
                n_adds.append(len(recs))
        n = len(podb)
        excl_start = np.zeros(n + 1, dtype='<i4')
        pod_start = np.zeros(n + 1, dtype='<i4')
        edit_start = np.zeros(n + 1, dtype='<i4')
        excl_start[1:] = np.cumsum([len(e) for e in exs])
        pod_start[1:] = np.cumsum([len(p) for p in nowl])
        edit_start[1:] = np.cumsum([len(e) for e in ednodes])
        ex = np.ascontiguousarray(np.concatenate(exs) if n else np.zeros(0), dtype='<i4')
        pods = np.frombuffer(b''.join(podb), dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(np.concatenate(nowl) if n else np.zeros(0), dtype='<f8')
        lift = np.asarray(lifts, dtype='<i4')
        ednode = np.ascontiguousarray(np.concatenate(ednodes) if n else np.zeros(0), dtype='<i4')
        edrec = np.frombuffer(b''.join(edrecs), dtype=wire.NODE_DTYPE)
        out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        status = np.zeros(n, dtype='<i4')
        which = np.zeros(n, dtype='<i4')
        counts = np.zeros((len(pods), wire.WHY_COUNT), dtype='<u4') if explain else None
        # NULL addition and round arrays unless some scenario has them: round_start selects the round kernel
        adds, rnds, pod_round = (None, None, None), (None, None), None
        if any(n_adds):
            add_start = np.zeros(n + 1, dtype='<i4')
            add_start[1:] = np.cumsum(n_adds)
            adat = np.ascontiguousarray(np.concatenate(adats), dtype='<i4')
            adrec = np.frombuffer(b''.join(adrecs), dtype=wire.NODE_DTYPE)
            adds = (add_start.ctypes.data, adat.ctypes.data, adrec.ctypes.data)
        if any(r is not None for r in rounds):
            clocks = [np.asarray(() if r is None else r, dtype='<f8').reshape(-1) for r in rounds]
            round_start = np.zeros(n + 1, dtype='<i4')
            round_start[1:] = np.cumsum([len(c) for c in clocks])
            round_clock = np.ascontiguousarray(np.concatenate(clocks), dtype='<f8')
            rnds = (round_start.ctypes.data, round_clock.ctypes.data if len(round_clock) else None)
            pod_round = np.zeros(len(pods), dtype='<i4')
        some = len(pods) > 0
        args = [self._h, src, n, excl_start.ctypes.data, ex.ctypes.data if len(ex) else None,
                lift.ctypes.data if n else None, edit_start.ctypes.data, ednode.ctypes.data if len(ednode) else None,
                edrec.ctypes.data if len(edrec) else None, *adds, pod_start.ctypes.data,
                pods.ctypes.data if some else None, now.ctypes.data if some else None, *rnds]
        tail = [out.ctypes.data if some else None, status.ctypes.data, which.ctypes.data,
                counts.ctypes.data if explain and some else None,
                pod_round.ctypes.data if pod_round is not None and some else None]
        arrivals = any(a is not None for a in arrs)
        pod_clock = np.zeros(len(pods), dtype='<f8') if arrivals else None
        if arrivals and pod_round is None:
            pod_round = np.zeros(len(pods), dtype='<i4')
            tail[-1] = pod_round.ctypes.data if some else None
        if any(r is not None for r in rels) or arrivals:
            # NULL release arrays unless some scenario has that field: existing calls go out as before
            trs, useds, rls = [], [], []
            for r in rels:
                tr, used, rl = ((), (), None) if r is None else r
                trs.append(np.asarray(tr, dtype='<i4').reshape(-1))
                useds.append(np.asarray(used, dtype='<i2').reshape(len(trs[-1]), wire.MAX_NICS))
                rls.append(np.zeros(0, dtype=wire.RELEASE_DTYPE) if rl is None else
                           np.asarray(rl, dtype=wire.RELEASE_DTYPE).reshape(-1))
            track_start = np.zeros(n + 1, dtype='<i4')
            track_start[1:] = np.cumsum([len(t) for t in trs])
            rel_start = np.zeros(n + 1, dtype='<i4')
            rel_start[1:] = np.cumsum([len(x) for x in rls])
            tracked = np.ascontiguousarray(np.concatenate(trs), dtype='<i4')
            used = np.ascontiguousarray(np.concatenate(useds), dtype='<i2')
            rel = np.ascontiguousarray(np.concatenate(rls), dtype=wire.RELEASE_DTYPE)
            rel_args = (track_start.ctypes.data, tracked.ctypes.data if len(tracked) else None,
                        used.ctypes.data if len(tracked) else None, rel_start.ctypes.data,
                        rel.ctypes.data if len(rel) else None)
            if arrivals:
                arrive = np.ascontiguousarray(np.concatenate(
                    [np.zeros(len(t), dtype='<i4') if a is None else np.asarray(a, dtype='<i4').reshape(-1)
                     for a, t in zip(arrs, nowl)]) if n else np.zeros(0), dtype='<i4')
                assert len(arrive) == len(pods)
                self._ck(self._L.nhd_plan_scenarios_arrivals(
                    *args, *rel_args, arrive.ctypes.data if some else None, *tail,
                    pod_clock.ctypes.data if some else None))
            else:
                self._ck(self._L.nhd_plan_scenarios_releases(*args, *rel_args, *tail))
        else:
            self._ck(self._L.nhd_plan_scenarios_rounds(*args, *tail))
        res = self._scenario_results(status, which, pod_start, out, counts)
        if pod_round is None:
            return res
        if pod_clock is None:
            return [r + (pod_round[a:b] if r[0] == 0 else None,)
                    for r, a, b in zip(res, pod_start[:-1].tolist(), pod_start[1:].tolist())]
        return [r + ((pod_round[a:b], pod_clock[a:b]) if r[0] == 0 else (None, None))
                for r, a, b in zip(res, pod_start[:-1].tolist(), pod_start[1:].tolist())]

    @staticmethod
    def _scenario_results(status, which, pod_start, out, counts):
        """``plan_scenarios``' per-scenario tuples: ``(code, pod, bindings[, counts])``."""
        if counts is None:
            return [(code, pod, out[a:b] if code == 0 else None)
                    for code, pod, a, b in zip(status.tolist(), which.tolist(), pod_start[:-1].tolist(),
                                               pod_start[1:].tolist())]
        return [(code, pod, out[a:b], counts[a:b]) if code == 0 else (code, pod, None, None)
                for code, pod, a, b in zip(status.tolist(), which.tolist(), pod_start[:-1].tolist(), pod_start[1:].tolist())]

    def filter_bitmaps(self):
        """Runs only the snapshot predicate kernel on the staged batch; returns
        (feas[type, node] bool, nogpu[node], busy[node], pod_type[pod])."""
        self._ck(self._L.nhd_run_filter_only(self._h))
        nt, wpt = ctypes.c_int32(), ctypes.c_int32()
        self._ck(self._L.nhd_read_filter(self._h, ctypes.byref(nt), ctypes.byref(wpt), None, 0, None, 0))
        words = np.zeros((nt.value + 2) * wpt.value, dtype='<u8')
        pt = np.zeros(self.n_pods, dtype='<i4')
        self._ck(self._L.nhd_read_filter(self._h, ctypes.byref(nt), ctypes.byref(wpt), words.ctypes.data,
                                         len(words), pt.ctypes.data, len(pt)))
        bits = np.unpackbits(words.view(np.uint8), bitorder='little').reshape(nt.value + 2, wpt.value * 64)
        bits = bits[:, :self.n_nodes].astype(bool)
        return bits[:nt.value], bits[nt.value], bits[nt.value + 1], pt
