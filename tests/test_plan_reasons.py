"""Why planned pods find no node: per-reason node counts of the scenario calls (``nhd_plan_scenarios_explained``,
``Solver.plan_scenarios(explain=True)``, ``NHDScheduler.PlanDrains(reasons=True)`` / ``PlanDefrag(reasons=True)``).

The contract is "a row is what ``nhd_explain_batch`` returns for that pod after the five steps": the records at the
start of the pod's own phase (before or after the lift) with the phase's earlier pods bound.  The chain of evidence:
  * ``PlanDrains`` / ``PlanDefrag`` with reasons, answered by the explanation oracle on the two-phase state, equal the
    unmodified reference's own drop decisions, frozen in tests/golden/live/plan_reasons.json.gz, and ``PlanDrains``
    equals ``PlanDrain`` group by group (no GPU);
  * the scenario kernel's correction rows and the base pass, run on the CPU emulation of the device (tests/emu) in both
    lane orders, equal the oracle per pod over the drain and defrag scenario families (no GPU);
  * on the GPU the bindings equal ``nhd_plan_scenarios_edited``, the rows equal ``nhd_plan_batch`` in every sweep mode
    and the GPU's own commit path, the call changes nothing, and so at config 4's full size (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import wire
from nhd_b200.solver import Scenario
from tests import helpers
from tests.golden import make_live_golden
from tests.golden.make_defrag_golden import defrag_sessions
from tests.golden.make_plan_golden import drain_sessions, mirror_session
from tests.plan_oracle import OraclePlanner, excluded, oracle_scenario
from tests.test_defrag import defrag_scenarios
from tests.test_drains import _each_plan, drain_scenarios
from tests.test_plan import _emu_lib, _gpu_factory
from tests.test_query import MODES, _filter_words, _gpu_cases, oracle_state, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def check_explained(got, plain, scens, refused, st, speed, busy, where=''):
    """Every accepted scenario: the bindings of the plain call and the oracle's bindings and rows on ``st``; the refused
    ones name the pod and have neither.  Returns the number of NO_CANDIDATE rows compared."""
    n = 0
    for j, (sc, g, p) in enumerate(zip(scens, got, plain)):
        sc = Scenario(*sc)
        if j in refused:
            assert g == refused[j] + (None, None) and p[:2] == refused[j], (where, j, g[:2])
            continue
        assert g[:2] == (0, -1) and g[2].tobytes() == p[2].tobytes(), (where, j, g[:2])
        if len(sc.pods):
            want, _, wc, _ = oracle_scenario(st, speed, sc, busy=busy, explain=True)
            assert g[2].tobytes() == want.tobytes(), (where, j, helpers.first_binding_diff(want, g[2]))
            assert (g[3] == wc).all(), (where, j, np.flatnonzero((g[3] != wc).any(1)), g[3][(g[3] != wc).any(1)][:2],
                                        wc[(g[3] != wc).any(1)][:2])
            n += int((g[2]['status'] == wire.NO_CANDIDATE).sum())
    return n


def raw_explained(s, scens, fill=0xA5A5A5A5):
    """``nhd_plan_scenarios_explained`` of scenarios ``(exclude, pods, now)`` with the counts pre-filled with ``fill``:
    ``(status, counts)``."""
    pods = np.concatenate([sc[1] for sc in scens]).astype(wire.POD_DTYPE)
    now = np.concatenate([np.asarray(sc[2], dtype='<f8') for sc in scens])
    ex = np.concatenate([np.asarray(sc[0], dtype='<i4').reshape(-1) for sc in scens] + [np.zeros(1, dtype='<i4')])
    excl_start = np.concatenate([[0], np.cumsum([len(sc[0]) for sc in scens])]).astype('<i4')
    pod_start = np.concatenate([[0], np.cumsum([len(sc[1]) for sc in scens])]).astype('<i4')
    out = np.zeros(len(pods), dtype=wire.BINDING_DTYPE)
    status = np.zeros(len(scens), dtype='<i4')
    which = np.zeros(len(scens), dtype='<i4')
    counts = np.full((len(pods), wire.WHY_COUNT), fill, dtype='<u4')
    assert s._L.nhd_plan_scenarios_explained(s._h, 0, len(scens), excl_start.ctypes.data, ex.ctypes.data, None, None,
                                             None, None, pod_start.ctypes.data, pods.ctypes.data, now.ctypes.data,
                                             out.ctypes.data, status.ctypes.data, which.ctypes.data,
                                             counts.ctypes.data) == 0
    return status, [counts[a:b] for a, b in zip(pod_start[:-1], pod_start[1:])]


# ---------------------------------------------------------------------------------------------- CPU: the reference
def _reasons_against_the_reference(factory):
    golden = make_live_golden.load('plan_reasons')
    drains, defrag = golden['drains'], golden['defrag']
    want_drains = make_live_golden.load('drains')['sessions']
    want_defrag = make_live_golden.load('defrag')['sessions']
    assert [g['name'] for g in drains] == [name for name, _, _ in drain_sessions()] == [g['name'] for g in want_drains]
    assert [g['name'] for g in defrag] == [name for name, _ in defrag_sessions()] == [g['name'] for g in want_defrag]
    n = 0
    for (name, script, _), why, want in zip(drain_sessions(), drains, want_drains):
        sched, _, _ = mirror_session(script, factory)
        try:
            names = list(sched.nodes)
            got = sched.PlanDrains([[d['node']] for d in want['drains']], reasons=True)
            for d, rows in zip(want['drains'], why['drains']):
                placement, reasons = got[(d['node'],)]
                assert list(placement.values()) == d['outcome'], (name, d['node'])
                assert rows['node'] == d['node'] and reasons == _counted(rows['moved'], names), (name, d['node'])
                n += len(reasons)
        finally:
            sched.close()
    for (name, script), why, want in zip(defrag_sessions(), defrag, want_defrag):
        sched, _, _ = mirror_session(script, factory)
        try:
            names = list(sched.nodes)
            for d, wd in zip(want['delays'], why['delays']):
                got = sched.PlanDefrag(node_groups=[[c['node']] for c in d['drains']], delay=d['delay'], reasons=True)
                for c, rows in zip(d['drains'], wd['drains']):
                    moved, pending, reasons = got[(c['node'],)]
                    assert list(moved.values()) == c['moved_to'] and rows['node'] == c['node'], (name, c['node'])
                    want_rows = dict(rows['moved'], **(rows['pending'] if pending is not None else {}))
                    assert reasons == _counted(want_rows, names), (name, d['delay'], c['node'])
                    n += len(reasons)
        finally:
            sched.close()
    assert n > 200, n


def _counted(rows, names):
    """{(ns, name): one digit per node} -> {(ns, name): {reason name: nodes}}"""
    assert all(len(codes) == len(names) for codes in rows.values())
    out = {}
    for key, codes in rows.items():
        ns, pod = key.split('/', 1)
        c = np.bincount([int(ch) for ch in codes], minlength=wire.WHY_COUNT)
        out[(ns, pod)] = {name: int(v) for name, v in zip(wire.WHY_NAMES, c) if v}
    return out


def test_plan_drains_and_defrag_reasons_equal_the_reference():
    """The reference's own drop decisions for every re-created or pending pod it leaves without a node, answered
    before any drain by ``PlanDrains`` / ``PlanDefrag`` with ``reasons=True`` and the oracle standing in for the GPU."""
    _reasons_against_the_reference(OraclePlanner)


def _drains_reasons_equal_plan_drain(factory, sessions):
    n = 0
    for name, script, _ in sessions:
        sched, _, _ = mirror_session(script, factory)
        try:
            holding = [nd for nd, v in sched.nodes.items() if v.pod_info]
            groups = [[nd] for nd in holding] + [holding[i:i + 2] for i in range(0, len(holding) - 1, 2)]
            got = sched.PlanDrains(groups, reasons=True)
            assert list(got) == [tuple(g) for g in groups], name
            assert {g: v[0] for g, v in got.items()} == sched.PlanDrains(groups), name
            for g in groups:
                assert got[tuple(g)] == sched.PlanDrain(g), (name, g)
                n += len(got[tuple(g)][1])
        finally:
            sched.close()
    assert n > 10, n


def test_plan_drains_reasons_equal_plan_drain_per_group():
    """``PlanDrains(groups, reasons=True)[g]`` is ``PlanDrain(g)`` from the same state, for single nodes and pairs."""
    _drains_reasons_equal_plan_drain(OraclePlanner, drain_sessions()[:6])


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
from nhd_b200 import wire
from nhd_b200.solver import Solver
from tests.test_defrag import defrag_scenarios
from tests.test_drains import drain_scenarios
from tests.test_plan_reasons import check_explained, raw_explained
from tests.test_query import emu_cases, oracle_state, packed
n = 0
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        s.load_nodes(recs)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        first = s.solve_batch(pods[:k], now[:k])
        source = 'mirror'
        if j %% 2:                                      # a snapshot source, with the mirror moved on since
            s.snapshot()
            s.solve_batch(pods[k:2 * k], now[k:2 * k])
            source = 'snapshot'
        clock = now[k:] if j %% 3 else np.full(len(now) - k, now[k])
        again = clock[:k] if len(clock) >= k else np.full(k, clock[0] if len(clock) else now[0])
        drains, refused = drain_scenarios(recs, pods[:k], again, first['node'], rest=(pods[k:], clock))
        scens = drains + defrag_scenarios(recs, pods[:k], np.resize(clock, k), first['node'], (pods[k:], clock), busy)
        got = s.plan_scenarios(scens, source=source, explain=True)
        n += check_explained(got, s.plan_scenarios(scens, source=source), scens, refused, st, speed, busy, j)
        if source == 'mirror' and refused:              # rows of refused scenarios are not written
            status, rows = raw_explained(s, drains)
            for r, (code, c, g) in enumerate(zip(status, rows, got)):
                assert code == (refused[r][0] if r in refused else 0), r
                assert (c == 0xA5A5A5A5).all() if r in refused else (c == g[3]).all(), r
    finally:
        s.close()
print('compared', n)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_explained_scenarios_on_the_emulated_device_equal_the_oracle(lane_order):
    """The ``test_drains`` and ``test_defrag`` families: mirror and snapshot sources, edits, lift 0 / part-way / none,
    held and lifted exclusions, duplicate exclusions, constant and per-pod clocks, mixed node-group lists, failed
    assignments, bad map types, refused scenarios with their rows left untouched."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1500)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    assert int(res.stdout.split()[-1]) > 100, res.stdout


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
    keep = lambda r: np.arange(r, len(recs), 100)                        # 18 nodes left in service: pods fail
    scens = [(np.setdiff1d(np.arange(len(recs)), keep(r)), pods[r * 30:(r + 1) * 30], now[r * 30:(r + 1) * 30])
             for r in range(10)]
    got = s.plan_scenarios(scens, explain=True)
    one = Solver(speed)
    one.load_nodes(recs)
    want = one.plan_scenarios(scens, explain=True)
    one.close()
    assert all(g[0] == 0 and g[2].tobytes() == w[2].tobytes() and (g[3] == w[3]).all() for g, w in zip(got, want))
    assert sum(int((g[3].sum(1) > 0).sum()) for g in got) > 0
    open(done, 'w').write('ok')
else:
    t0 = time.time()
    while not os.path.exists(done):
        time.sleep(0.05)
        assert time.time() - t0 < 600
s.close()
print('rank', rank, 'ok')
'''


def test_a_two_rank_handle_explains_scenarios_alone_as_one_rank(tmp_path):
    """A ``world_size`` 2 handle (node-sharded batches forced with NHD_SHARD_MIN_PAIRS=1): rank 0 explains scenarios
    on its own, entering no collective, and gets the single-rank answer."""
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


def commit_path(scratch, base, scens):
    """Each scenario on the GPU's own commit path, ``scratch`` loaded with ``base`` first: the edited records with the
    excluded nodes in maintenance, snapshot, the pods before the lift, ``explain_batch``; the flags back, snapshot, the
    rest, ``explain_batch``.  ``[(bindings, counts)]``."""
    out = []
    for sc in scens:
        sc = Scenario(*sc)
        ex, p, c, lift, edits = sc.exclude, sc.pods, sc.now, sc.lift, sc.edits
        scratch.load_nodes(base)
        if edits is not None and len(edits[0]):
            scratch.update_nodes(np.asarray(edits[0], dtype='<i4'), edits[1])
        ex = np.unique(np.asarray(list(ex), dtype='<i4'))
        lift = len(p) if lift is None else lift
        held = scratch.read_nodes()[ex] if len(ex) else None
        if len(ex):
            scratch.update_nodes(ex, excluded(held, range(len(ex))))
        b, w = [], []
        if lift:
            scratch.snapshot()
            b.append(scratch.solve_batch(p[:lift], c[:lift]))
            w.append(scratch.explain_batch())
        if len(ex):
            back = scratch.read_nodes()[ex]
            back['flags'] = held['flags']
            scratch.update_nodes(ex, back)
        if lift < len(p):
            scratch.snapshot()
            b.append(scratch.solve_batch(p[lift:], c[lift:]))
            w.append(scratch.explain_batch())
        out.append((np.concatenate(b) if b else np.zeros(0, dtype=wire.BINDING_DTYPE),
                    np.concatenate(w) if w else np.zeros((0, wire.WHY_COUNT), dtype='<u4')))
    return out


@pytest.mark.gpu
def test_explained_scenarios_equal_plan_batch_the_commit_path_and_the_oracle():
    """The query tests' case families at a state the solver itself reached partway along each stream.  Drain
    scenarios: bindings equal ``nhd_plan_scenarios_edited``, rows equal ``nhd_plan_batch(..., why_counts)`` of each
    scenario alone in every sweep mode.  Defrag scenarios (edits, lifts): rows equal the commit path on a scratch
    handle.  Both equal the oracle."""
    n = 0
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::4] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        k = len(pods) // 3
        st = oracle_state(recs, speed, pods, now, busy, k)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s, scratch = _solver(speed, busy, **mode), _solver(speed, busy, **mode)
            try:
                s.load_nodes(recs)
                first = s.solve_batch(pods[:k], now[:k])
                base = s.read_nodes()
                for clock in (now[k:], np.full(len(pods) - k, now[k])):
                    again = np.resize(clock, k) if len(clock) else now[:k]
                    drains, refused = drain_scenarios(recs, pods[:k], again, first['node'], rest=(pods[k:], clock))
                    got = s.plan_scenarios(drains, explain=True)
                    for g, w, sc in zip(got, _each_plan(s, [(ex, p, c) for ex, p, c in drains]), drains):
                        assert g[:2] == w[:2], (j, mode)
                        if w[2] is not None:
                            wb, wc = s.plan_batch(sc[1], sc[2], exclude=sc[0], explain=True)
                            assert g[2].tobytes() == wb.tobytes() and (g[3] == wc).all(), (j, mode)
                    defrag = defrag_scenarios(recs, pods[:k], again, first['node'], (pods[k:], clock), busy)
                    got_d = s.plan_scenarios(defrag, explain=True)
                    plain = s.plan_scenarios(defrag)
                    for g, p, (wb, wc) in zip(got_d, plain, commit_path(scratch, base, defrag)):
                        assert g[2].tobytes() == p[2].tobytes() == wb.tobytes() and (g[3] == wc).all(), (j, mode)
                    if not mode:
                        n += check_explained(got, s.plan_scenarios(drains), drains, refused, st, speed, busy, j)
                        n += check_explained(got_d, plain, defrag, {}, st, speed, busy, j)
            finally:
                s.close()
                scratch.close()
    assert n > (20 if EMULATED else 200), n


@pytest.mark.gpu
def test_an_explained_scenario_call_changes_nothing():
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
        scens = drain_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1])[0] + \
            defrag_scenarios(recs, pods[::-1], now[::-1], b['node'][::-1], (pods, now), busy)
        for source in ('mirror', 'snapshot'):
            got = s.plan_scenarios(scens, source=source, explain=True)
            assert any(g[3] is not None and g[3].any() for g in got)
            s.plan_scenarios(scens[:1], source=source, explain=True)
            assert state() == before, source
            assert s.timing() == timing and (s.debug_counters() == counters).all(), source
        s.query_batch(pods[:4], now[:4], source='snapshot')                           # the snapshot is still valid
        s.restore()
        assert s.read_nodes().tobytes() == recs.tobytes()
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After the 4 096-pod solve: the 2 560 single-node drains and the 64 racks of 32 nodes with reasons; every
    scenario's bindings and rows equal ``nhd_plan_batch`` with counts, a sample of 32 equals the oracle.  (Config 4's
    cluster is large enough that every drained pod places: this pins the reasons call at full size, not its rows.)"""
    import workload
    recs, speed, pods, now = workload.make_workload(4)
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        first = s.solve_batch(pods, now)
        after = s.read_nodes()
        clock = float(now.max()) + 5.0
        node = first['node']
        order = np.argsort(node, kind='stable')
        holding, starts = np.unique(node[order], return_index=True)
        bounds = list(starts) + [len(order)]
        scens = [([int(n)], pods[order[bounds[i]:bounds[i + 1]]], np.full(bounds[i + 1] - bounds[i], clock))
                 for i, n in enumerate(holding) if n >= 0]
        racks = []
        for r in range(64):
            rack = np.arange(r * 1024, r * 1024 + 32)
            rows = np.sort(np.flatnonzero(np.isin(node, rack)))
            racks.append((rack, pods[rows], np.full(len(rows), clock)))
        assert len(scens) > 1000, len(scens)
        for group in (scens, racks):
            got = s.plan_scenarios(group, explain=True)
            for (ex, p, c), g in zip(group, got):
                wb, wc = s.plan_batch(p, c, exclude=ex, explain=True)
                assert g[0] == 0 and g[2].tobytes() == wb.tobytes() and (g[3] == wc).all(), ex
        sample = [scens[i] for i in np.random.default_rng(4).choice(len(scens), 32, replace=False)]
        got = s.plan_scenarios(sample, explain=True)
    finally:
        s.close()
    for (ex, p, c), (code, _, b, counts) in zip(sample, got):
        want, _, wc, _ = oracle_scenario(after, speed, (ex, p, c), threads=os.cpu_count() or 1, explain=True)
        assert code == 0 and b.tobytes() == want.tobytes() and (counts == wc).all(), ex


@pytest.mark.gpu
def test_plan_drains_and_defrag_reasons_equal_the_reference_on_the_gpu():
    _reasons_against_the_reference(_gpu_factory())


@pytest.mark.gpu
def test_plan_drains_reasons_equal_plan_drain_per_group_on_the_gpu():
    _drains_reasons_equal_plan_drain(_gpu_factory(), drain_sessions()[:2] if EMULATED else drain_sessions())
