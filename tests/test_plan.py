"""Dry runs of a batch (``nhd_plan_batch``, ``Solver.plan_batch``, ``DeviceCluster.plan``, ``NHDScheduler.PlanPods`` /
``PlanDrain``).

The contract is "equal to the solve, with nothing committed": a plan returns, byte for byte, the bindings
``nhd_solve_batch`` would return on the chosen records with the excluded nodes in maintenance, and the counts
``nhd_explain_batch`` would return after it.  The chain of evidence:
  * the scheduler's ``PlanDrain``, answered by the oracle on a copy of the records with the maintenance flags set,
    equals where the unmodified reference re-schedules the pods of drained nodes, frozen in
    tests/golden/live/plan.json.gz (no GPU);
  * the plan's launch path, run on the CPU emulation of the device (tests/emu) in both lane orders, equals the oracle
    and the explanation oracle on those records (no GPU);
  * on the GPU the plan equals the oracle in every sweep mode, equals the GPU's own commit path with the nodes put in
    maintenance, and changes nothing of the handle's state (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from tests import helpers, scenarios
from tests.golden import make_live_golden
from tests.golden.make_plan_golden import drain_sessions, mirror_session
from tests.plan_oracle import OraclePlanner, excluded, oracle_scenario
from tests.test_query import MODES, _filter_words, _gpu_cases, emu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def exclusion_sets(recs):
    """No exclusion, every third node, and every node with GPUs."""
    n = len(recs)
    return [(), tuple(range(0, n, 3)), tuple(int(i) for i in np.flatnonzero(recs['n_gpus'] > 0))]


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _drain_against_the_reference(factory):
    golden = make_live_golden.load('plan')['sessions']
    sessions = drain_sessions()
    assert [g['name'] for g in golden] == [name for name, _, _ in sessions]
    n, none, busy_gpu = 0, 0, 0
    for (name, script, _), want in zip(sessions, golden):
        sched, k8s, clock = mirror_session(script, factory)
        try:
            assert [(ns, pod) for nd in want['drain'] for (pod, ns) in sched.nodes[nd].pod_info] == \
                [tuple(p) for p in want['pods']], name
            state, traffic = dict(sched.pod_state), k8s.transcript()
            objs = {nd: (scenarios.node_state(v), v.maintenance) for nd, v in sched.nodes.items()}
            placement, reasons = sched.PlanDrain(want['drain'])
            assert k8s.transcript() == traffic and sched.pod_state == state, name
            assert {nd: (scenarios.node_state(v), v.maintenance) for nd, v in sched.nodes.items()} == objs, name
            assert list(placement) == [tuple(p) for p in want['pods']], name
            assert list(placement.values()) == want['outcome'], (name, list(placement.values()), want['outcome'])
            for key, node in placement.items():
                assert (key in reasons) == (node is None) or node is None, (name, key)
            # GPU pods re-created while some GPU node is inside its busy window
            recs = sched.cluster.read_records()
            hot = ((clock() - recs['busy_time'] < script['min_busy_secs']) & (recs['n_gpus'] > 0)).any()
            spec = {(st['ns'], st['name']): st['pod'] for st in script['init'] + script['steps'] if st['op'] == 'add_pod'}
            busy_gpu += sum(1 for key in placement if hot and any(g['gpus'] for g in spec[key]['proc_groups']))
            n += len(placement)
            none += sum(v is None for v in placement.values())
        finally:
            sched.close()
    assert n > 100 and none > 20 and busy_gpu >= 3, (n, none, busy_gpu)


def test_plan_drain_equals_the_reference_drain():
    """Where the reference re-schedules the pods of drained nodes, answered before the drain by ``PlanDrain`` with
    the oracle standing in for the GPU."""
    _drain_against_the_reference(OraclePlanner)


def test_plan_pods_equals_the_batch_with_the_oracle_stand_in():
    _plan_pods_equals_the_batch(OraclePlanner, _plain_scripts()[:3])


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200.solver import Solver
from tests import helpers
from tests.plan_oracle import oracle_scenario
from tests.test_plan import exclusion_sets
from tests.test_query import emu_cases, oracle_state, packed
n = 0
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        s.load_nodes(recs)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        s.solve_batch(pods[:k], now[:k])
        source = 'mirror'
        if j %% 2:                                      # a snapshot plan, with the mirror moved on since
            s.snapshot()
            s.solve_batch(pods[k:2 * k], now[k:2 * k])
            source = 'snapshot'
        clock = now[k:] if j %% 3 else np.full(len(now) - k, now[k])
        for ex in exclusion_sets(recs):
            got, counts = s.plan_batch(pods[k:], clock, source=source, exclude=ex, explain=True)
            want, _, wcounts, _ = oracle_scenario(st, speed, (ex, pods[k:], clock), busy=busy, explain=True)
            assert got.tobytes() == want.tobytes(), (j, ex, helpers.first_binding_diff(want, got))
            assert counts.tobytes() == wcounts.tobytes(), (j, ex)
            n += len(got)
    finally:
        s.close()
print('compared', n)
'''


def _emu_lib():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    try:
        import build_emu_cuda
    finally:
        sys.path.pop(0)
    return build_emu_cuda.build()


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_plan_on_the_emulated_device_equals_the_oracle(lane_order):
    """Mirror and snapshot sources; no, some and all-GPU-node exclusions; constant and per-pod clocks; mixed node-group
    lists (the explanation stream); the ``emu_cases()`` family."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 1000, res.stdout


RANK_CODE = r'''
import ctypes, os, sys, time
import numpy as np
sys.path.insert(0, %(root)r)
ctypes.CDLL(%(nccl)r, mode=ctypes.RTLD_GLOBAL)
import workload
from nhd_b200.solver import Solver, nccl_unique_id
rank, tmp = int(sys.argv[1]), sys.argv[2]
idf, done = os.path.join(tmp, 'nccl_id'), os.path.join(tmp, 'done')
if rank == 0:
    nid = nccl_unique_id()
    open(idf + '.tmp', 'wb').write(nid); os.rename(idf + '.tmp', idf)
else:
    t0 = time.time()
    while not os.path.exists(idf):
        time.sleep(0.02)
        assert time.time() - t0 < 60
    nid = open(idf, 'rb').read()
recs, speed, pods, now = workload.make_workload(3, n_nodes=1800, n_pods=300)
s = Solver(speed, rank=rank, world_size=2, nccl_id=nid)
s.load_nodes(recs)
if rank == 0:                                     # rank 0 plans alone; rank 1 only holds its handle open
    ex = np.arange(0, len(recs), 5)
    got, counts = s.plan_batch(pods, now, exclude=ex, explain=True)
    one = Solver(speed)
    one.load_nodes(recs)
    want, wcounts = one.plan_batch(pods, now, exclude=ex, explain=True)
    one.close()
    assert got.tobytes() == want.tobytes() and counts.tobytes() == wcounts.tobytes()
    assert (got['status'] == 0).sum() > 100
    open(done, 'w').write('ok')
else:
    t0 = time.time()
    while not os.path.exists(done):
        time.sleep(0.05)
        assert time.time() - t0 < 600
s.close()
print('rank', rank, 'ok')
'''


def test_a_two_rank_handle_plans_alone_as_one_rank(tmp_path):
    """A ``world_size`` 2 handle (node-sharded batches forced with NHD_SHARD_MIN_PAIRS=1): rank 0 plans on its own,
    entering no collective, and gets the single-rank answer."""
    nccl_dir = os.path.join(ROOT, 'tests', 'emu', 'fake_nccl')
    nccl = os.path.join(nccl_dir, 'libnccl.so.2')
    src = os.path.join(nccl_dir, 'fake_nccl.c')
    if not os.path.exists(nccl) or os.path.getmtime(nccl) < os.path.getmtime(src):
        subprocess.run(['gcc', '-O2', '-fPIC', '-shared', '-w', '-Wl,-soname,libnccl.so.2', '-o', nccl, src, '-lrt'], check=True)
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='d',
               NHD_SHARD_MIN_PAIRS='1')
    code = RANK_CODE % dict(root=ROOT, nccl=nccl)
    procs = [subprocess.Popen([sys.executable, '-c', code, str(r), str(tmp_path)], cwd=ROOT, env=env,
                              stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=900) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0, (o + e)[-2000:]


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


@pytest.mark.gpu
def test_plan_equals_the_oracle_in_every_sweep_mode():
    """The query tests' case families, with and without exclusions, bindings and counts, from a state the solver itself
    reached partway along each stream; constant and per-pod clocks."""
    statuses = np.zeros(5, dtype=np.int64)
    for j, scn in enumerate(_gpu_cases()):
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        sets = exclusion_sets(recs)
        for mode in (MODES if not EMULATED else MODES[:1]) if j % 3 == 0 else MODES[:1]:
            s = _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                s.solve_batch(pods[:k], now[:k])
                for ex in sets:
                    for clock in (now[k:], np.full(len(pods) - k, now[k])):
                        got, counts = s.plan_batch(pods[k:], clock, exclude=ex, explain=True)
                        want, _, wcounts, _ = oracle_scenario(st, speed, (ex, pods[k:], clock), busy=busy, explain=True)
                        assert got.tobytes() == want.tobytes(), (j, mode, ex, helpers.first_binding_diff(want, got))
                        assert counts.tobytes() == wcounts.tobytes(), (j, mode, ex)
                        statuses += np.bincount(got['status'], minlength=5)[:5]
            finally:
                s.close()
    assert statuses[[0, 1]].all(), statuses


def _commit_path(s, pods, now, exclude, recs_now):
    """The plan's equivalent on the GPU's own commit path: put the nodes in maintenance, snapshot, solve, explain,
    restore, put them back (``recs_now``: the records as they are before)."""
    ex = np.asarray(sorted(set(int(i) for i in exclude)), dtype='<i4')
    if len(ex):
        s.update_nodes(ex, excluded(recs_now[ex], range(len(ex))))
    try:
        s.snapshot()
        out = s.solve_batch(pods, now)
        counts = s.explain_batch()
        s.restore()
    finally:
        if len(ex):
            s.update_nodes(ex, recs_now[ex])
    return out, counts


@pytest.mark.gpu
def test_plan_equals_the_gpus_own_commit_path():
    for scn in _gpu_cases()[::3]:
        recs, pods, now, speed, busy = packed(scn)
        s = _solver(speed, busy)
        try:
            s.load_nodes(recs)
            s.solve_batch(pods[:len(pods) // 4], now[:len(pods) // 4])
            cur = s.read_nodes()
            for ex in exclusion_sets(recs):
                got, counts = s.plan_batch(pods, now, exclude=ex, explain=True)
                want, wcounts = _commit_path(s, pods, now, ex, cur)
                assert got.tobytes() == want.tobytes(), (ex, helpers.first_binding_diff(want, got))
                assert counts.tobytes() == wcounts.tobytes(), ex
                assert s.read_nodes().tobytes() == cur.tobytes()
        finally:
            s.close()


@pytest.mark.gpu
def test_a_plan_changes_nothing():
    from tests.explain_scenarios import explain_scenarios
    scn = explain_scenarios()[1]
    recs, pods, now, speed, busy = packed(scn)
    s = _solver(speed, busy)
    try:
        s.load_nodes(recs)
        s.snapshot()
        b = s.solve_batch(pods, now)
        failed = int(np.flatnonzero(b['status'] == wire.NO_CANDIDATE)[0])
        timing = s.timing()
        counters = s.debug_counters()

        def state():
            words, pt = _filter_words(s)
            return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                    s.explain_batch().tobytes(), s.explain_pod(failed).tobytes())
        before = state()
        for source in ('mirror', 'snapshot'):
            for ex in exclusion_sets(recs):
                s.plan_batch(pods[::-1], now[::-1], source=source, exclude=ex, explain=True)   # other types, other order
                s.plan_batch(pods[:1], now[:1], source=source, exclude=ex)
            assert state() == before, source
            assert s.timing() == timing and (s.debug_counters() == counters).all(), source
        s.restore()
        assert s.read_nodes().tobytes() == recs.tobytes()                        # the snapshot is untouched too
        # the staged batch: solving it again (from the snapshot) gives what it gave before
        s.snapshot()
        s.solve_batch(pods, now)
        s.restore()
        s.plan_batch(pods[::-1], now[::-1], exclude=exclusion_sets(recs)[1], explain=True)
        s.solve_staged()
        assert s.fetch_bindings().tobytes() == b.tobytes()
    finally:
        s.close()


@pytest.mark.gpu
def test_a_batch_after_plans_equals_one_on_a_fresh_handle():
    """What a plan leaves behind (the shared mapping memo included) changes no later batch."""
    for scn in _gpu_cases()[2::5]:
        recs, pods, now, speed, busy = packed(scn)
        s, fresh = _solver(speed, busy), _solver(speed, busy)
        try:
            s.load_nodes(recs)
            fresh.load_nodes(recs)
            for ex in exclusion_sets(recs):
                s.plan_batch(pods[::-1], now, exclude=ex, explain=True)
            assert s.solve_batch(pods, now).tobytes() == fresh.solve_batch(pods, now).tobytes()
            assert s.read_nodes().tobytes() == fresh.read_nodes().tobytes()
        finally:
            s.close()
            fresh.close()


def _four_numa(recs):
    four = recs.copy()
    four['n_numa'], four['phys_cores'] = 4, 32
    four['gpu_numa_mask'], four['nic_numa_mask'] = 0, 0
    four['gpu_numa_mask'][:, 0], four['nic_numa_mask'][:, 0] = recs['gpu_numa_mask'].sum(axis=1), \
        recs['nic_numa_mask'].sum(axis=1)
    four['used'] = 0
    return four


@pytest.mark.gpu
def test_plan_refusals():
    from nhd_b200.solver import SolverError
    from tests.explain_scenarios import explain_scenarios
    recs, pods, now, speed, busy = packed(explain_scenarios()[0])
    s = _solver(speed, busy)

    def refused(code, *args, **kw):
        with pytest.raises(SolverError) as e:
            s.plan_batch(*args, **kw)
        assert e.value.code == code, str(e.value)
        return str(e.value)
    try:
        refused(wire.ERR_STATE, pods, now)                                   # nothing loaded
        s.load_nodes(recs)
        refused(wire.ERR_STATE, pods, now, source='snapshot')                # no snapshot
        s.snapshot()
        s.solve_batch(pods, now)
        s.plan_batch(pods, now, source='snapshot')
        s.update_nodes([0], recs[:1])
        refused(wire.ERR_STATE, pods, now, source='snapshot')                # an update since the snapshot
        assert f'{len(recs)}' in refused(wire.ERR_INVALID, pods, now, exclude=[len(recs)])
        assert '-1' in refused(wire.ERR_INVALID, pods, now, exclude=[2, -1])
        dup = s.plan_batch(pods, now, exclude=[1, 1, 3], explain=True)       # a duplicate counts once
        one = s.plan_batch(pods, now, exclude=[3, 1], explain=True)
        assert dup[0].tobytes() == one[0].tobytes() and dup[1].tobytes() == one[1].tobytes()
        bad = pods.copy()
        bad[3]['n_groups'] = 0
        assert 'pod 3' in refused(wire.ERR_INVALID, bad, now)
        clock = now.copy()
        clock[2] = np.nan
        assert 'pod 2' in refused(wire.ERR_INVALID, pods, clock)
        with pytest.raises(ValueError):
            s.plan_batch(pods, now, source='disk')
        L = s._L
        assert L.nhd_plan_batch(s._h, 7, 0, None, len(pods), pods.ctypes.data, now.ctypes.data, pods.ctypes.data,
                                None) == wire.ERR_INVALID
        assert L.nhd_plan_batch(s._h, 0, 1, None, 0, None, None, None, None) == wire.ERR_INVALID
        assert L.nhd_plan_batch(s._h, 0, 0, None, 1, None, None, None, None) == wire.ERR_INVALID
        assert L.nhd_plan_batch(None, 0, 0, None, 0, None, None, None, None) == wire.ERR_INVALID
        assert len(s.plan_batch(pods[:0], now[:0])) == 0

        # the tuple limit: 4 groups on 4-NUMA nodes.  Accepted once the 4-NUMA nodes are excluded, refused exactly
        # when the equivalent solve (the same nodes put in maintenance) refuses
        mixed = recs.copy()
        four_idx = np.arange(0, len(recs), 2)
        mixed[four_idx] = _four_numa(recs)[four_idx]
        s.load_nodes(mixed)
        big = pods.copy()
        big[5]['n_groups'] = 4
        for g in range(4):
            big[5]['groups'][g] = big[5]['groups'][0]
        for ex in (four_idx, four_idx[1:], ()):
            try:
                got = s.plan_batch(big, now, exclude=ex)
                plan_err = None
            except SolverError as e:
                got, plan_err = None, e
            try:
                want, _ = _commit_path(s, big, now, ex, mixed)
                solve_err = None
            except SolverError as e:
                solve_err = e
            assert (plan_err is None) == (solve_err is None), (len(ex), plan_err, solve_err)
            if plan_err is None:
                assert got.tobytes() == want.tobytes()
            else:
                assert plan_err.code == solve_err.code == wire.ERR_UNSUPPORTED and 'pod 5' in str(plan_err)
            assert (plan_err is None) == (len(ex) == len(four_idx)), len(ex)
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    ex = np.random.default_rng(4).choice(len(recs), 1024, replace=False)
    try:
        s.load_nodes(recs)
        s.snapshot()
        bench = s.solve_batch(pods, now)                                     # the bench's solve: the mirror moves on
        snap = s.plan_batch(pods, now, source='snapshot')
        assert snap.tobytes() == bench.tobytes(), helpers.first_binding_diff(bench, snap)
        s.restore()
        got, counts = s.plan_batch(pods, now, exclude=ex, explain=True)
        want, wcounts = _commit_path(s, pods, now, ex, recs)
        assert got.tobytes() == want.tobytes(), helpers.first_binding_diff(want, got)
        assert counts.tobytes() == wcounts.tobytes()
        head = s.plan_batch(pods[:256], now[:256], exclude=ex)
    finally:
        s.close()
    want = oracle_scenario(recs, speed, (ex, pods[:256], now[:256]), threads=os.cpu_count() or 1, explain=True)[0]
    assert head.tobytes() == want.tobytes(), helpers.first_binding_diff(want, head)
    assert head.tobytes() == got[:256].tobytes()


# ---------------------------------------------------------------------------------------------- scheduler
def _plain_scripts():
    """Sessions without Kubernetes write failures (a failed write cuts a batch, which a plan does not foresee)."""
    from tests import sched_harness as H
    return [H.random_script(seed, flavor, fail_rate=0.0) for seed, flavor in
            ((41, 'mixed'), (42, 'wild'), (43, 'vf'), (44, 'big'), (45, 'wild'), (46, 'mixed'))]


def _plan_pods_equals_the_batch(factory, scripts):
    """At every pending scan of each session: ``PlanPods`` of the pending pods, then the scan itself.  The plan names
    the nodes the scan binds the pods to and the pods it fails, with the reasons it records; the plan itself makes no
    Kubernetes traffic and leaves ``pod_state``, the ``Node`` objects and the device records as they were."""
    from nhd_b200 import NHDScheduler as S
    checked = placed = failed = 0
    real = S.NHDScheduler.CheckPendingPods

    def check(self):
        phase = {(k[0], k[1], k[2]): p for k, p in self.k8s.ServicePods(self.sched_name).items()}
        keys = [k for k, p in phase.items() if p[0] == 'Pending' and p[1] is None and
                self.pod_state.get((k[0], k[1]), {}).get('state') != S.PodStatus.POD_STATUS_SCHEDULED]
        nonlocal checked, placed, failed
        if keys and self.nodes:
            traffic, state = self.k8s.transcript(), dict(self.pod_state)
            objs = {n: scenarios.node_state(v) for n, v in self.nodes.items()}
            counters = (self.failed_schedule_count, self.pods_solved, self.cluster.batches)
            placement, reasons = self.PlanPods(keys)
            assert self.k8s.transcript() == traffic and self.pod_state == state
            assert {n: scenarios.node_state(v) for n, v in self.nodes.items()} == objs
            assert (self.failed_schedule_count, self.pods_solved, self.cluster.batches) == counters
            real(self)
            for (ns, name), node in placement.items():
                st = self.pod_state.get((ns, name), {}).get('state')
                where = [n for n, v in self.nodes.items() if (name, ns) in v.pod_info]
                if node is None:
                    assert st != S.PodStatus.POD_STATUS_SCHEDULED, (ns, name)
                else:
                    assert st == S.PodStatus.POD_STATUS_SCHEDULED and where == [node], (ns, name, node, where)
                if (ns, name) in reasons:
                    assert self.unschedulable_reasons.get((ns, name)) == reasons[(ns, name)], (ns, name)
                    failed += 1
                placed += node is not None
            checked += 1
        else:
            real(self)
    from tests import sched_harness as H
    S.NHDScheduler.CheckPendingPods = check
    try:
        for script in scripts:
            H.run_mirror(script, solver_factory=factory)
    finally:
        S.NHDScheduler.CheckPendingPods = real
    assert checked > 5 and placed > 20 and failed > 0, (checked, placed, failed)


def _gpu_factory():
    from nhd_b200.solver import Solver

    class GpuSolver(Solver):
        def __init__(self, speed_table, nic_bw_avail_percent=0.9, min_busy_secs=30.0, device=0):
            super().__init__(speed_table, nic_bw_avail_percent=nic_bw_avail_percent, min_busy_secs=min_busy_secs,
                             device=device)
    return GpuSolver


@pytest.mark.gpu
def test_plan_pods_equals_the_batch_on_the_gpu():
    _plan_pods_equals_the_batch(_gpu_factory(), _plain_scripts()[:2] if EMULATED else _plain_scripts())


@pytest.mark.gpu
def test_plan_drain_equals_the_reference_drain_on_the_gpu():
    _drain_against_the_reference(_gpu_factory())
