"""``Solver`` — thin object wrapper over the C-ABI handle (include/nhd_b200.h).

Works on packed numpy records (``nhd_b200.wire``); the object-level drop-in lives in
``nhd_b200.Matcher``.  All compute happens in the CUDA library."""
import ctypes

import os

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
        """A dry run of ``solve_batch`` (``nhd_plan_batch``): the bindings the pods would get scheduled in order, each
        seeing the ones before it, on the current records (``source='mirror'``) or on those of the last ``snapshot()``
        (``'snapshot'``), with the node indices ``exclude`` taken as in maintenance.  With ``explain=True`` returns
        ``(bindings, counts)``, counts being what ``explain_batch`` would return after that solve.  Nothing is placed:
        records, snapshot, the last batch and its explanations stay as they are."""
        src = _source(source)
        pods = np.ascontiguousarray(pods, dtype=wire.POD_DTYPE)
        now = np.ascontiguousarray(now, dtype='<f8')
        assert len(pods) == len(now)
        ex = np.ascontiguousarray(exclude, dtype='<i4').reshape(-1)
        if out is None:
            out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
        counts = np.zeros((len(pods), wire.WHY_COUNT), dtype='<u4') if explain else None
        self._ck(self._L.nhd_plan_batch(self._h, src, len(ex), ex.ctypes.data if len(ex) else None, len(pods),
                                        pods.ctypes.data, now.ctypes.data, out.ctypes.data,
                                        counts.ctypes.data if explain else None))
        return (out, counts) if explain else out

    def plan_scenarios(self, scenarios, source='mirror'):
        """Many independent dry runs in one call (``nhd_plan_scenarios_edited``).  ``scenarios``: a sequence of
        ``(exclude, pods, now[, lift[, edits]])``.  Returns one ``(code, pod, bindings)`` per scenario: ``code`` 0 and
        ``bindings`` what ``plan_batch(pods, now, source, exclude)`` returns, or the refusal ``plan_batch`` would raise
        (``wire.ERR_*``), the index of the pod it names and None.  Scenarios do not see each other.  Unlike
        ``plan_batch`` the tuple limits are judged with the excluded nodes counted; ``plan_batch`` plans a scenario
        refused for that.
        ``lift`` (None: never): the excluded nodes are back in service from the scenario's pod ``lift`` on.  ``edits``
        (None: none): ``(nodes, records)``, node indices and a ``wire.NODE_DTYPE`` array, the records those nodes have
        for the whole scenario.  With either, the bindings are those of ``solve_batch`` on a scratch copy of the records
        with the edits applied, the excluded nodes in maintenance for the pods before ``lift`` and back after."""
        src = _source(source)
        # (thousands of small scenarios: gathered as bytes, since numpy's per-array checks of the structured pod dtype
        # would cost more than the call itself)
        exs, podb, nowl, lifts, ednodes, edrecs = [], [], [], [], [], []
        for sc in scenarios:
            exclude, pods, now = sc[:3]
            lift = sc[3] if len(sc) > 3 else None
            edits = sc[4] if len(sc) > 4 else None
            pods = np.asarray(pods)
            if pods.dtype != wire.POD_DTYPE:
                pods = pods.astype(wire.POD_DTYPE)
            exs.append(np.asarray(exclude, dtype='<i4').reshape(-1))
            podb.append(np.ascontiguousarray(pods).tobytes())
            nowl.append(np.asarray(now, dtype='<f8').reshape(-1))
            assert pods.size == len(nowl[-1])
            lifts.append(len(nowl[-1]) if lift is None else int(lift))
            if edits is None:
                ednodes.append(np.zeros(0, dtype='<i4'))
            else:
                nodes, recs = edits
                ednodes.append(np.asarray(nodes, dtype='<i4').reshape(-1))
                recs = np.asarray(recs, dtype=wire.NODE_DTYPE).reshape(-1)
                assert len(recs) == len(ednodes[-1])
                edrecs.append(recs.tobytes())
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
        self._ck(self._L.nhd_plan_scenarios_edited(self._h, src, n, excl_start.ctypes.data,
                                                   ex.ctypes.data if len(ex) else None,
                                                   lift.ctypes.data if n else None, edit_start.ctypes.data,
                                                   ednode.ctypes.data if len(ednode) else None,
                                                   edrec.ctypes.data if len(edrec) else None, pod_start.ctypes.data,
                                                   pods.ctypes.data if len(pods) else None,
                                                   now.ctypes.data if len(pods) else None,
                                                   out.ctypes.data if len(pods) else None, status.ctypes.data,
                                                   which.ctypes.data))
        return [(code, pod, out[a:b] if code == 0 else None)
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
