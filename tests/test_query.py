"""Where each pod would go on its own (``nhd_query_batch``, ``Solver.query_batch``, ``Matcher.FindNodes``,
``DeviceCluster.query``, ``NHDScheduler.PreviewPods`` and ``diagnose_contention``).

The contract is "equal to a batch of one": pod i of a query gets, byte for byte, the binding a solve of pod i alone
would give on the chosen records.  The chain of evidence:
  * the oracle run as a batch of one on a fresh copy of each state equals the unmodified reference's own
    FindNode + SetPhysicalIdsFromMapping, frozen in tests/golden/live/query.json.gz (no GPU);
  * the query kernels, run on the CPU emulation of the device (tests/emu) in both lane orders, equal the oracle (no GPU);
  * on the GPU the query equals the oracle's batch of one in every sweep mode, equals the GPU's own solve of that pod
    alone, and changes nothing of the handle's state (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from oracle import binding
from tests import helpers, ref_compare, scenarios
from tests.golden import make_live_golden
from tests.golden.make_query_golden import query_states, query_streams
from tests.plan_oracle import OraclePlanner, oracle_alone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'
MODES = (dict(), dict(single_warp=True), dict(cpu_warps=1), dict(cpu_warps=2), dict(sweep_debug=1),
         dict(sweep_debug=5))


def packed(scn):
    recs, pods, now, layout = ref_compare.pack_scenario(scn)
    return scenarios.apply_preuse(recs, scn), pods, now, layout.speed_table(), float(scn.get('min_busy_secs', 30.0))


def oracle_state(recs, speed, pods, now, busy, k):
    """The records after pods 0..k-1 of the stream were scheduled one after the other."""
    return binding.solve(recs, speed, pods[:k], now[:k], min_busy_secs=busy)[1] if k else recs


# ---------------------------------------------------------------------------------------------- CPU: the oracle
def test_oracle_alone_equals_the_reference_queries():
    golden = make_live_golden.load('query')
    n = {}
    for name, scns in query_streams():
        assert len(golden[name]) == len(scns), name
        for j, (scn, want) in enumerate(zip(scns, golden[name])):
            recs, pods, now, speed, busy = packed(scn)
            assert sorted(int(k) for k in want) == query_states(scn), (name, j)
            for k in query_states(scn):
                got = oracle_alone(oracle_state(recs, speed, pods, now, busy, k), speed, pods, now, busy)
                for i, (o, b) in enumerate(zip(want[str(k)], got)):
                    assert ref_compare.diff_outcome(o, b) == [], (name, j, k, i, ref_compare.diff_outcome(o, b))
                    n[o['status']] = n.get(o['status'], 0) + 1
    assert n.get('placed', 0) > 1000 and n.get('none', 0) > 100 and n.get('assign_failed', 0) > 0, n


EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests import helpers
from tests.plan_oracle import oracle_alone
from tests.test_query import emu_cases, oracle_state, packed
n = 0
for scn in emu_cases():
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        for k in (0, len(pods) // 2):
            st = oracle_state(recs, speed, pods, now, busy, k)
            s.load_nodes(st)
            for clock in (now, np.full(len(now), now[0])):
                got, want = s.query_batch(pods, clock), oracle_alone(st, speed, pods, clock, busy)
                assert got.tobytes() == want.tobytes(), (scn.get('name'), k, helpers.first_binding_diff(want, got))
                n += len(pods)
    finally:
        s.close()
print('compared', n)
'''


def emu_cases():
    """Seeded scenarios the emulated-device run compares: random streams of every flavour, the explanation stream
    (busy windows, mixed node-group lists) and the first limit cases."""
    from tests.explain_scenarios import explain_scenarios
    out = []
    for f in ('mixed', 'wild', 'vf', 'big'):
        out += make_live_golden.oracle_scenarios(f)[:4]
    return out + explain_scenarios() + [s for s in scenarios.limit_scenarios() if len(s['nodes']) <= 64][:4]


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_query_kernels_on_the_emulated_device_equal_the_oracle(lane_order):
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    try:
        import build_emu_cuda
    finally:
        sys.path.pop(0)
    lib = build_emu_cuda.build()
    env = dict(os.environ, NHD_B200_LIB=lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=900)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 2000, res.stdout


def test_scheduler_contention_with_the_oracle_stand_in(monkeypatch):
    """The scheduler side of ``diagnose_contention`` without a GPU: the oracle answers the queries."""
    _contention_session(monkeypatch, OraclePlanner, [H_script(10, 'wild'), H_script(101, 'mixed')])


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def _gpu_cases():
    from tests.explain_scenarios import explain_scenarios
    per = 2 if EMULATED else 12
    cases = list(explain_scenarios())
    for f in ('mixed', 'wild', 'vf', 'big'):
        cases += make_live_golden.oracle_scenarios(f)[:per]
    return cases + [s for s in scenarios.limit_scenarios() if len(s['nodes']) <= 512][:3 if EMULATED else None]


@pytest.mark.gpu
def test_query_equals_the_oracle_alone_in_every_sweep_mode():
    """Constant and per-pod clocks (busy windows expiring between pods), mixed node-group lists, NUMA / PCI / bad map
    types and failed assignments, at states the solver itself reached partway along each stream."""
    statuses = np.zeros(5, dtype=np.int64)
    for j, scn in enumerate(_gpu_cases()):
        recs, pods, now, speed, busy = packed(scn)
        for mode in (MODES if not EMULATED else MODES[:1]) if j % 3 == 0 else MODES[:1]:
            s = _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                done = 0
                for k in query_states(scn):
                    if k > done:
                        s.solve_batch(pods[done:k], now[done:k])            # the stream up to the state, on the GPU
                    done = k
                    st = oracle_state(recs, speed, pods, now, busy, k)
                    assert s.read_nodes().tobytes() == st.tobytes(), (j, mode, k)
                    bad = pods.copy()
                    bad['map_type'][::7] = wire.MAP_NONE                     # BAD_MAP_TYPE among the others
                    for q, clock in ((pods, now), (pods, np.full(len(now), now[-1])), (bad, now)):
                        got, want = s.query_batch(q, clock), oracle_alone(st, speed, q, clock, busy)
                        assert got.tobytes() == want.tobytes(), (j, mode, k, helpers.first_binding_diff(want, got))
                        statuses += np.bincount(got['status'], minlength=5)[:5]
            finally:
                s.close()
    assert (statuses > 0).all() if not EMULATED else statuses[[0, 1, 4]].all(), statuses


@pytest.mark.gpu
def test_query_equals_the_gpus_own_solve_of_the_pod_alone():
    for scn in _gpu_cases()[::4]:
        recs, pods, now, speed, busy = packed(scn)
        s = _solver(speed, busy)
        try:
            s.load_nodes(recs)
            s.solve_batch(pods[:len(pods) // 2], now[:len(pods) // 2])
            got = s.query_batch(pods, now)
            for i in range(0, len(pods), 3):
                s.snapshot()
                one = s.solve_batch(pods[i:i + 1], now[i:i + 1])
                s.restore()
                assert one.tobytes() == got[i:i + 1].tobytes(), (i, helpers.first_binding_diff(one, got[i:i + 1]))
        finally:
            s.close()


@pytest.mark.gpu
def test_snapshot_query_after_a_batch_equals_a_mirror_query_after_restore():
    for scn in _gpu_cases()[1::5]:
        recs, pods, now, speed, busy = packed(scn)
        s = _solver(speed, busy)
        try:
            s.load_nodes(recs)
            s.solve_batch(pods[:3], now[:3])
            s.snapshot()
            s.solve_batch(pods, now)
            from_snap = s.query_batch(pods, now, source='snapshot')
            s.restore()
            assert from_snap.tobytes() == s.query_batch(pods, now).tobytes()
            assert from_snap.tobytes() == oracle_alone(s.read_nodes(), speed, pods, now, busy).tobytes()
        finally:
            s.close()


def _filter_words(s):
    import ctypes
    L = s._L
    nt, wpt = ctypes.c_int32(), ctypes.c_int32()
    assert L.nhd_read_filter(s._h, ctypes.byref(nt), ctypes.byref(wpt), None, 0, None, 0) == 0
    words = np.zeros((nt.value + 2) * wpt.value, dtype='<u8')
    pt = np.zeros(s.n_pods, dtype='<i4')
    assert L.nhd_read_filter(s._h, ctypes.byref(nt), ctypes.byref(wpt), words.ctypes.data, len(words),
                             pt.ctypes.data, len(pt)) == 0
    return words, pt


@pytest.mark.gpu
def test_a_query_changes_nothing():
    from tests.explain_scenarios import explain_scenarios
    scn = explain_scenarios()[1]
    recs, pods, now, speed, busy = packed(scn)
    s = _solver(speed, busy)
    try:
        s.load_nodes(recs)
        s.snapshot()
        b = s.solve_batch(pods, now)
        failed = int(np.flatnonzero(b['status'] == wire.NO_CANDIDATE)[0])

        def state():
            words, pt = _filter_words(s)
            return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                    s.explain_batch().tobytes(), s.explain_pod(failed).tobytes())
        before = state()
        for source in ('mirror', 'snapshot'):
            s.query_batch(pods[::-1], now[::-1], source=source)              # other types, other order
            s.query_batch(pods[:1], now[:1], source=source)
            assert state() == before, source
        s.restore()
        assert s.read_nodes().tobytes() == recs.tobytes()                    # the snapshot is untouched too
    finally:
        s.close()


@pytest.mark.gpu
def test_query_refusals():
    from nhd_b200.solver import SolverError
    from tests.explain_scenarios import explain_scenarios
    recs, pods, now, speed, busy = packed(explain_scenarios()[0])
    s = _solver(speed, busy)

    def refused(code, *args, **kw):
        with pytest.raises(SolverError) as e:
            s.query_batch(*args, **kw)
        assert e.value.code == code, str(e.value)
        return str(e.value)
    try:
        refused(wire.ERR_STATE, pods, now)                                   # nothing loaded
        s.load_nodes(recs)
        refused(wire.ERR_STATE, pods, now, source='snapshot')                # no snapshot
        s.snapshot()
        s.solve_batch(pods, now)
        s.stage_batch(pods, now)
        s.restore()
        s.query_batch(pods, now, source='snapshot')                          # solves, stages, restores are fine
        s.update_nodes([0], recs[:1])
        refused(wire.ERR_STATE, pods, now, source='snapshot')                # an update since the snapshot
        s.query_batch(pods, now)
        s.snapshot()
        s.query_batch(pods, now, source='snapshot')
        s.load_nodes(recs)
        refused(wire.ERR_STATE, pods, now, source='snapshot')                # a load since the snapshot
        bad = pods.copy()
        bad[3]['n_groups'] = 0
        assert 'pod 3' in refused(wire.ERR_INVALID, bad, now)
        clock = now.copy()
        clock[2] = np.nan
        assert 'pod 2' in refused(wire.ERR_INVALID, pods, clock)
        with pytest.raises(ValueError):
            s.query_batch(pods, now, source='disk')
        L = s._L
        assert L.nhd_query_batch(s._h, 7, len(pods), pods.ctypes.data, now.ctypes.data, pods.ctypes.data) == wire.ERR_INVALID
        assert L.nhd_query_batch(s._h, 0, 1, None, None, None) == wire.ERR_INVALID
        assert L.nhd_query_batch(None, 0, 0, None, None, None) == wire.ERR_INVALID
        assert len(s.query_batch(pods[:0], now[:0])) == 0
        # a pod beyond the tuple limits: 4 groups on 4-NUMA nodes
        four = recs.copy()
        four['n_numa'], four['phys_cores'] = 4, 32
        four['gpu_numa_mask'], four['nic_numa_mask'] = 0, 0
        four['gpu_numa_mask'][:, 0], four['nic_numa_mask'][:, 0] = recs['gpu_numa_mask'].sum(axis=1), \
            recs['nic_numa_mask'].sum(axis=1)
        four['used'] = 0
        s.load_nodes(four)
        big = pods.copy()
        big[5]['n_groups'] = 4
        for g in range(4):
            big[5]['groups'][g] = big[5]['groups'][0]
        assert 'pod 5' in refused(wire.ERR_UNSUPPORTED, big, now)
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size_against_the_oracle():
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        s.snapshot()
        s.solve_batch(pods, now)                                             # the mirror now holds the whole batch
        got = s.query_batch(pods, now, source='snapshot')                    # the batch-start state
        after = s.query_batch(pods, now)                                     # the state after the whole batch
        final = s.read_nodes()
    finally:
        s.close()
    sample = np.random.default_rng(4).choice(len(pods), 256, replace=False)
    threads = os.cpu_count() or 1
    for state, q in ((recs, got), (final, after)):
        want = oracle_alone(state, speed, pods[sample], now[sample], threads=threads)
        assert q[sample].tobytes() == want.tobytes(), helpers.first_binding_diff(want, q[sample])
    assert (got['status'] == wire.PLACED).all()                              # every pod of the stream fits alone
    assert (after['node'] != got['node']).any()                              # ... not always where it did at the start


@pytest.mark.gpu
def test_matcher_find_nodes_equals_find_node_and_commits_nothing():
    from nhd_b200 import tracking
    from nhd_b200.Matcher import Matcher
    import nhd_b200.CfgTopology as cfg_mod
    import nhd_b200.Node as node_mod
    for scn in _gpu_cases()[:3] + _gpu_cases()[-8:-5]:
        if scn.get('used') or scn.get('nic_inuse'):
            continue
        node_mod.Node.MIN_BUSY_SECS = float(scn.get('min_busy_secs', 30.0))
        try:
            nodes = scenarios.build_nodes(scn, node_mod)
            tops = [scenarios.build_top(p, cfg_mod) for p in scn['pods']]
            groups = [p['groups'] for p in scn['pods']]
            m = Matcher()
            m.FindNodes(nodes, tops[:1], groups[:1], now=scn['now'][0])      # instruments the Node class
            vers = {n: vars(v).get(tracking.VERSION, 0) for n, v in nodes.items()}
            before = m._solver.read_nodes().tobytes()
            got = m.FindNodes(nodes, tops, groups, now=scn['now'])
            assert {n: vars(v).get(tracking.VERSION, 0) for n, v in nodes.items()} == vers
            assert m._solver.read_nodes().tobytes() == before and not m._cl.force
            for i, top in enumerate(tops):
                one = Matcher().FindNode(nodes, top, groups[i], now=scn['now'][i])
                assert got[i][0] == one[0], i
                if one[0] is not None:
                    assert got[i][1]['_nhd_binding'].tobytes() == one[1]['_nhd_binding'].tobytes(), i
        finally:
            node_mod.Node.MIN_BUSY_SECS = 30.0


def H_script(seed, flavor):
    from tests import sched_harness as H
    return H.random_script(seed, flavor)


@pytest.mark.gpu
def test_preview_pods_makes_no_kubernetes_traffic():
    from nhd_b200 import NHDScheduler as S
    from tests import fake_k8s, sched_harness as H
    import nhd_b200.CfgTopology as cfg_mod
    import nhd_b200.Node as node_mod
    script = H_script(101, 'mixed')
    node_mod.Node.MIN_BUSY_SECS = float(script['min_busy_secs'])
    try:
        clock = H.Clock(script['clock0'])
        k8s = fake_k8s.FakeK8s(script['nodes'])
        for st in script['init']:
            H.apply_k8s_op(k8s, clock, st)
        for st in script['steps']:
            if st['op'] in H.K8S_OPS:
                H.apply_k8s_op(k8s, clock, st)
        sched = S.NHDScheduler(k8s, lambda t, c: fake_k8s.JsonCfgParser(c, cfg_mod), clock=clock)
        sched.Startup()
        keys = [k for k, p in k8s.ServicePods(sched.sched_name).items() if p[0] == 'Pending']
        assert keys
        traffic, batches = k8s.transcript(), sched.cluster.batches
        state = dict(sched.pod_state)
        objs = {n: scenarios.node_state(v) for n, v in sched.nodes.items()}
        got = sched.PreviewPods(keys)
        assert k8s.transcript() == traffic and sched.pod_state == state
        assert {n: scenarios.node_state(v) for n, v in sched.nodes.items()} == objs
        assert sched.cluster.batches == batches
        recs = sched.cluster.read_records()
        for key in keys:
            e = S._Pending(0, key)
            sched._prepare(e, events=False)
            if e.top is None or e.unsupported is not None:
                assert got[(key[0], key[1])] is None
                continue
            pod = sched.cluster._pods([e.top], [e.groups], [e.rec])
            want = oracle_alone(recs, sched.cluster.layout.speed_table(), pod, np.array([clock()]),
                                float(script['min_busy_secs']))[0]
            name = sched.cluster.name_of(int(want['node'])) if int(want['status']) == wire.PLACED else None
            assert got[(key[0], key[1])] == name, key
        assert any(v is not None for v in got.values())
        sched.close()
    finally:
        node_mod.Node.MIN_BUSY_SECS = 30.0


def _contention_session(monkeypatch, factory, scripts):
    """Each script with ``diagnose_contention`` on and off: identical end state (events, binds, nodes), and every
    diagnosis equal to the oracle's batch of one at that batch's snapshot."""
    from nhd_b200 import NHDScheduler as S
    from tests import sched_harness as H

    class Recording(factory):
        def snapshot(self):
            super().snapshot()
            self.snap_recs = self.read_nodes()

    checked, finals = [], []
    real = S.NHDScheduler._contention

    def spy(self, solvable, out, now):
        got = real(self, solvable, out, now)
        sv = self.cluster._solver
        failed = [i for i, b in enumerate(out) if int(b['status']) == wire.NO_CANDIDATE]
        pods = self.cluster._pods([solvable[i].top for i in failed], [solvable[i].groups for i in failed],
                                  [solvable[i].rec for i in failed])
        want = oracle_alone(sv.snap_recs, self.cluster.layout.speed_table(), pods, np.full(len(failed), now),
                            float(sv._min_busy) if hasattr(sv, '_min_busy') else 30.0)
        for i, w in zip(failed, want):
            name = self.cluster.name_of(int(w['node'])) if int(w['status']) == wire.PLACED else None
            assert got[solvable[i].pos] == name
            checked.append(name)
        return got

    real_close = S.NHDScheduler.close

    def close(self):
        finals.append((self.diagnose_contention, dict(self.contended_pods), dict(self.pod_state)))
        real_close(self)
    monkeypatch.setattr(S.NHDScheduler, '_contention', spy)
    monkeypatch.setattr(S.NHDScheduler, 'close', close)
    base_init = S.NHDScheduler.__init__
    for script in scripts:
        docs = []
        for flag in (False, True):
            monkeypatch.setattr(S.NHDScheduler, '__init__',
                                lambda self, *a, _f=flag, **kw: base_init(self, *a, diagnose_contention=_f, **kw))
            docs.append(H.run_mirror(script, solver_factory=Recording))
        assert docs[0] == docs[1]
    monkeypatch.setattr(S.NHDScheduler, '__init__', base_init)
    assert checked and any(c is not None for c in checked), checked
    for flag, contended, pod_state in finals:
        if not flag:
            assert not contended
        for key in contended:
            assert pod_state.get(key, {}).get('state') != S.PodStatus.POD_STATUS_SCHEDULED, key


@pytest.mark.gpu
def test_scheduler_contention_diagnosis_matches_the_oracle(monkeypatch):
    from nhd_b200.solver import Solver

    class GpuSolver(Solver):
        def __init__(self, speed_table, nic_bw_avail_percent=0.9, min_busy_secs=30.0, device=0):
            super().__init__(speed_table, nic_bw_avail_percent=nic_bw_avail_percent, min_busy_secs=min_busy_secs,
                             device=device)
            self._min_busy = min_busy_secs
    # seeds 10 and 17 (wild) include failed assignments (a rewind, a batch cut)
    scripts = [H_script(10, 'wild'), H_script(17, 'wild'), H_script(101, 'mixed')]
    _contention_session(monkeypatch, GpuSolver, scripts[:2] if EMULATED else scripts)
