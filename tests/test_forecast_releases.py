"""Forecasts with running pods finishing between the scans (``nhd_plan_batch_releases``,
``Solver.plan_batch_releases``).

The contract is "the reference's scheduler, every round solved one pod at a time on the records and the signed NIC pod
counters, the releases played between rounds": byte for byte each pod's last attempt, the round that placed it, and
the reasons of the pods whose last attempt found no node.  ``oracle_releases`` is that loop: one oracle solve per pod,
``ClaimPodNICResources`` on the counters after each placement, ``AddResourcesFromTopology`` + ``SetBusy`` for each
release, and every tracked NIC's bit re-derived from its counter.  The chain of evidence:
  * on the CPU emulation of the device (tests/emu), both lane orders, the call equals that loop on every field, with
    and without reasons, including rounds cut several times and cuts in round 0 from negative starting counters; with
    no releases and no tracking it is ``nhd_plan_batch_rounds`` byte for byte; every malformed argument is refused and
    nothing of the handle moves (no GPU);
  * on the GPU the same in every sweep mode, the same loop run on a scratch handle (one ``solve_batch`` per pod, the
    releases and counter bits written with ``update_nodes``), and config 4 at full size against a scratch handle that
    commits each round and applies the releases with ``update_nodes`` (``-m gpu``)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from nhd_b200 import _lib, wire
from tests import helpers
from tests.plan_oracle import OraclePlanner, _nic_bits, oracle_releases
from tests.test_forecast import _steps
from tests.test_plan import _emu_lib
from tests.test_query import MODES, _filter_words, _gpu_cases, emu_cases, packed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'


def test_the_symbol_is_declared_and_exported():
    from nhd_b200 import build
    build.build()
    text = open(os.path.join(ROOT, 'include', 'nhd_b200.h')).read()
    assert 'int32_t nhd_plan_batch_releases(nhd_handle* h, int32_t source, int32_t n_excluded' in text
    assert 'typedef struct nhd_release {' in text and wire.RELEASE_DTYPE.itemsize == 88
    assert 'nhd_plan_batch_releases' in _lib.EXPORTS and hasattr(_lib.load(), 'nhd_plan_batch_releases')


# ---------------------------------------------------------------------------------------------- the cases
def release_of(b, pod, node, rnd, clock, pairings):
    """The release record of the deployed pod ``pod`` bound by ``b``: its cores, GPUs, hugepages, and ``pairings``
    nic_core_pairing entries on each NIC it claimed."""
    rl = np.zeros((), dtype=wire.RELEASE_DTYPE)
    rl['node'], rl['round'], rl['clock'] = node, rnd, clock
    for c in b['cores'][:b['n_cores']]:
        rl['cores'][c >> 6] |= np.uint64(1) << np.uint64(c & 63)
    rl['gpus'] = sum(1 << int(g) for g in b['gpu_index'][:b['n_gpus']])
    rl['hugepages_gb'] = pod['hugepages_gb']
    for j in range(int(b['n_claimed'])):
        rl['nic_pairings'][b['claimed_nics'][j]] = pairings
    return rl


def release_cases(recs, speed, pods, now, busy, seed):
    """``(state, pending pods, clocks, rounds, tracked, pods_used, releases)`` cases on one stream: the first half of
    the stream deployed (the oracle's bindings), the rest pending at one clock or at their own.  Releases of deployed
    pods with one or two pairings per NIC (two drive the counter to -1), landing mid-gap, exactly at a scan's clock, a
    third of the busy window before a scan, or at the start of the gap; some free NICs of untouched nodes start at -1
    or -2 (cuts in round 0); no releases but tracking; releases on tracked nodes only."""
    from oracle import binding
    rng = np.random.default_rng(seed)
    k = len(pods) // 2
    b0, st = binding.solve(recs, speed, pods[:k], now[:k], min_busy_secs=busy)
    placed = np.flatnonzero(b0['status'] == wire.PLACED)
    tail, tclock = pods[k:], now[k:]
    t0 = float(tclock.max()) if len(tclock) else 1000.0
    out = []
    for v in range(4):
        clock = tclock if v % 2 else np.full(len(tail), t0)
        period = (busy, busy / 3.0, busy + 1.0, busy)[v] or 10.0
        rounds = _steps(t0, period, 1 + (seed + v) % 4)
        pick = rng.permutation(placed)[:(0, 4, 12, len(placed))[v]] if len(placed) else placed
        rels = []
        for i in pick:
            rnd = int(rng.integers(1, len(rounds) + 1))
            lo, hi = (t0 if rnd == 1 else rounds[rnd - 2]), rounds[rnd - 1]
            at = (0.5 * (lo + hi), hi, max(lo, hi - busy / 3.0), lo)[int(rng.integers(4))]
            rels.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd, at, 1 + int(rng.integers(2))))
        rels = np.array(sorted(rels, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
        tracked = sorted({int(x['node']) for x in rels})
        free = [int(n) for n in np.flatnonzero(st['n_nics'] > 0) if int(n) not in tracked]
        extra = list(rng.permutation(free)[:(1, 3, 0, 6)[v]]) if free else []
        tracked = tracked + [int(x) for x in extra]
        used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
        for t, node in enumerate(tracked):
            nn = int(st['n_nics'][node])
            bits = int(st['nic_inuse'][node])
            for i in range(nn):
                used[t, i] = 1 if bits >> i & 1 else 0
            if node in extra:
                for i in range(nn):
                    if not bits >> i & 1 and rng.integers(2):
                        used[t, i] = -1 - int(rng.integers(2))
        out.append((st, tail, clock, rounds, tracked, used, rels))
    return out


def check_cases(s, cases, speed, busy, where=''):
    """Every case equals the oracle loop, with reasons and without.  Returns (pods compared, pods placed at a round
    >= 1, cuts, rounds with several cuts, cuts in round 0)."""
    n = later = cuts = several = zero = 0
    for j, (st, p, c, rounds, tracked, used, rels) in enumerate(cases):
        s.load_nodes(st)
        got, rnd, rows = s.plan_batch_releases(p, c, rounds, tracked, used, rels, explain=True)
        b, wrnd, wrows, cut = oracle_releases(st, speed, p, c, rounds, tracked, used, rels, busy=busy, explain=True)
        assert got.tobytes() == b.tobytes(), (where, j, helpers.first_binding_diff(b, got))
        assert (rnd == wrnd).all(), (where, j, rnd, wrnd)
        assert (rows == wrows).all(), (where, j, np.flatnonzero((rows != wrows).any(1)))
        plain, prnd = s.plan_batch_releases(p, c, rounds, tracked, used, rels)
        assert plain.tobytes() == got.tobytes() and (prnd == rnd).all(), (where, j)
        n += len(p)
        later += int(((got['status'] == wire.PLACED) & (rnd >= 1)).sum())
        cuts += sum(cut)
        several += sum(x > 1 for x in cut)
        zero += cut[0]
    return n, later, cuts, several, zero


def check_identity(s, cases):
    """No releases and no tracking: ``nhd_plan_batch_rounds`` byte for byte."""
    for st, p, c, rounds, _, _, _ in cases:
        s.load_nodes(st)
        a = s.plan_batch_releases(p, c, rounds, [], np.zeros((0, wire.MAX_NICS)), [], explain=True)
        b = s.plan_batch_rounds(p, c, rounds, explain=True)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def check_refusals(s, case):
    """Every malformed argument is NHD_ERR_INVALID and leaves records, snapshot, staged batch, bindings, bitmaps,
    explanations, timing and counters as they were."""
    from nhd_b200.solver import SolverError
    st, p, c, rounds, tracked, used, rels = case
    assert len(rels) and len(rounds) >= 1
    s.load_nodes(st)
    s.snapshot()
    b = s.solve_batch(p, c)
    timing, counters = s.timing(), s.debug_counters()

    def state():
        words, pt = _filter_words(s)
        return (s.read_nodes().tobytes(), s.fetch_bindings().tobytes(), words.tobytes(), pt.tobytes(),
                s.explain_batch().tobytes())
    before = state()

    def refused(what, tr=tracked, u=used, r=rels, rd=rounds):
        with pytest.raises(SolverError) as e:
            s.plan_batch_releases(p, c, rd, tr, u, r, source='snapshot')
        assert e.value.code == wire.ERR_INVALID and what in str(e.value), (what, str(e.value))

    def edit(f):
        r = rels.copy()
        f(r)
        return r
    last = len(rounds)
    refused('outside [1,', r=edit(lambda r: r['round'].__setitem__(0, 0)))
    refused('outside [1,', r=edit(lambda r: r['round'].__setitem__(0, last + 1)))
    refused('not finite', r=edit(lambda r: r['clock'].__setitem__(0, np.nan)))
    if len(rels) > 1:
        refused('go down', r=edit(lambda r: r['clock'].__setitem__(1, r['clock'][0] - 1e-3)))
    refused('outside the gap', r=edit(lambda r: (r['round'].__setitem__(0, 1), r['clock'].__setitem__(0, float(np.max(c)) - 1.0))))
    refused('outside the gap', r=edit(lambda r: (r['round'].__setitem__(0, 1), r['clock'].__setitem__(0, rounds[0] + 1.0))))
    refused('not tracked', tr=tracked[1:], u=used[1:])
    refused('tracked twice', tr=tracked + tracked[:1], u=np.concatenate([used, used[:1]]))
    refused('outside the', tr=[len(st)] + tracked[1:], u=used)
    node = tracked[0]
    flip = used.copy()
    flip[0, 0] = 0 if st['nic_inuse'][node] & 1 else 1
    if st['n_nics'][node]:
        refused('disagrees', u=flip)
    beyond = used.copy()
    beyond[0, wire.MAX_NICS - 1] = 1 if st['n_nics'][node] < wire.MAX_NICS else beyond[0, wire.MAX_NICS - 1]
    if st['n_nics'][node] < wire.MAX_NICS:
        refused('disagrees', u=beyond)
    lc = int(st['phys_cores'][rels[0]['node']]) * (2 if st['flags'][rels[0]['node']] & wire.NODE_SMT else 1)
    if lc < 256:
        refused('beyond node', r=edit(lambda r: r['cores'][0].__setitem__(lc >> 6, r['cores'][0][lc >> 6] | np.uint64(1) << np.uint64(lc & 63))))
    ng = int(st['n_gpus'][rels[0]['node']])
    if ng < 16:
        refused('beyond node', r=edit(lambda r: r['gpus'].__setitem__(0, r['gpus'][0] | (1 << ng))))
    nn = int(st['n_nics'][rels[0]['node']])
    if nn < wire.MAX_NICS:
        refused('beyond node', r=edit(lambda r: r['nic_pairings'][0].__setitem__(nn, 1)))
    L, h = s._L, s._h
    out = np.zeros(len(p), dtype=wire.BINDING_DTYPE)
    clk = np.asarray(rounds, dtype='<f8')
    args = (0, 0, None, len(p), p.ctypes.data, c.ctypes.data, len(clk), clk.ctypes.data)
    assert L.nhd_plan_batch_releases(h, *args, -1, None, None, 0, None, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_releases(h, *args, 1, None, None, 0, None, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert L.nhd_plan_batch_releases(h, *args, 0, None, None, 1, None, out.ctypes.data, None, None) == wire.ERR_INVALID
    assert state() == before
    assert s.timing() == timing and (s.debug_counters() == counters).all()
    # a forecast between a solve and its explanations moves nothing either
    s.plan_batch_releases(p, c, rounds, tracked, used, rels, source='snapshot', explain=True)
    assert state() == before
    s.restore()
    s.solve_staged()
    assert s.fetch_bindings().tobytes() == b.tobytes()


# ---------------------------------------------------------------------------------------------- CPU: emulated device
EMU_CODE = r'''
import sys
sys.path.insert(0, %(root)r)
from nhd_b200.solver import Solver
from tests.test_forecast_releases import check_cases, check_identity, check_refusals, release_cases
from tests.test_query import emu_cases, packed
tot = [0] * 5
for j, scn in enumerate(emu_cases()):
    recs, pods, now, speed, busy = packed(scn)
    s = Solver(speed, min_busy_secs=busy)
    try:
        cases = release_cases(recs, speed, pods, now, busy, j)
        tot = [a + b for a, b in zip(tot, check_cases(s, cases, speed, busy, j))]
        if j %% 4 == 0:
            check_identity(s, cases)
        if j == 1:
            check_refusals(s, cases[3])
    finally:
        s.close()
print('compared', *tot)
'''


@pytest.mark.parametrize('lane_order', ['d', 'a'], ids=['descending', 'ascending'])
def test_releases_on_the_emulated_device_equal_the_oracle_loop(lane_order):
    """``emu_cases()`` streams half deployed, releases of their pods over 1 to 4 later scans, negative starting
    counters; with reasons and without; the identity with ``nhd_plan_batch_rounds``; the refusals."""
    env = dict(os.environ, NHD_B200_LIB=_emu_lib(), NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER=lane_order)
    res = subprocess.run([sys.executable, '-c', EMU_CODE % dict(root=ROOT)], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=2400)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    n, later, cuts, several, zero = (int(x) for x in res.stdout.split()[-5:])
    assert n > 300 and later > 10 and cuts > 5 and several >= 1 and zero >= 1, res.stdout


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def _scratch_one(scratch):
    """``solve_one`` of ``oracle_releases`` on a device handle: load the records, solve the one pod, read them back."""
    def solve_one(r, pod, clock):
        scratch.load_nodes(r)
        b = scratch.solve_batch(pod[None], np.array([clock]))
        return b[0], scratch.read_nodes()
    return solve_one


@pytest.mark.gpu
def test_releases_equal_the_oracle_loop_and_a_scratch_handle_in_every_sweep_mode():
    tot = [0] * 5
    cases = _gpu_cases()
    for j, scn in enumerate(cases[::6] if EMULATED else cases):
        recs, pods, now, speed, busy = packed(scn)
        rc = release_cases(recs, speed, pods, now, busy, 100 + j)
        for mode in (MODES[:1] if EMULATED or j % 3 else MODES):
            s = _solver(speed, busy, **mode)
            try:
                tot = [a + b for a, b in zip(tot, check_cases(s, rc, speed, busy, (j, mode)))]
                if j % 4 == 0:
                    check_identity(s, rc)
            finally:
                s.close()
        if j % 3 == 0:
            scratch, s = _solver(speed, busy), _solver(speed, busy)
            try:
                for st, p, c, rounds, tracked, used, rels in rc[2:]:
                    s.load_nodes(st)
                    got, rnd = s.plan_batch_releases(p, c, rounds, tracked, used, rels)
                    b, wrnd, _, _ = oracle_releases(st, speed, p, c, rounds, tracked, used, rels, busy=busy,
                                                    solve_one=_scratch_one(scratch))
                    assert got.tobytes() == b.tobytes() and (rnd == wrnd).all(), (j, helpers.first_binding_diff(b, got))
            finally:
                scratch.close()
                s.close()
    n, later, cuts, several, zero = tot
    assert n > (100 if EMULATED else 2000) and later > 0 and cuts > 0, tot


@pytest.mark.gpu
def test_a_release_forecast_changes_nothing_and_refuses_as_documented():
    scn = emu_cases()[1]
    recs, pods, now, speed, busy = packed(scn)
    s = _solver(speed, busy)
    try:
        check_refusals(s, release_cases(recs, speed, pods, now, busy, 1)[3])
    finally:
        s.close()


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_config4_full_size():
    """After config 4's solve, 4 096 pending one-GPU pods over 8 scans with 1 024 of the placed pods released over the
    gaps (one pairing per claimed NIC: no counter goes negative, so no cut) equal a scratch handle that solves each
    round as one batch and applies each gap's releases with ``update_nodes``; 32 sampled pending pods with two pairings
    per NIC (cuts) equal the oracle loop."""
    import workload
    from oracle import binding
    from tests.test_forecast_batch import config4_pending
    recs, speed, pods, now = workload.make_workload(4)
    recs, tail = config4_pending(recs, pods, 4096, 64)
    s, scratch = _solver(speed, 30.0), _solver(speed, 30.0)
    try:
        s.load_nodes(recs)
        b0 = s.solve_batch(pods, now)
        after = s.read_nodes()
        t = float(now.max()) + 5.0
        clock, rounds = np.full(len(tail), t), _steps(t, 30.0, 8)
        placed = np.flatnonzero(b0['status'] == wire.PLACED)
        pick = np.random.default_rng(4).choice(placed, 1024, replace=False)
        rels = []
        for k, i in enumerate(pick):
            rnd = 1 + k % 8
            lo = t if rnd == 1 else rounds[rnd - 2]
            rels.append(release_of(b0[i], pods[i], int(b0[i]['node']), rnd, lo + 0.5 * (rounds[rnd - 1] - lo), 1))
        rels = np.array(sorted(rels, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
        tracked = sorted({int(x['node']) for x in rels})
        used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
        for q, node in enumerate(tracked):
            used[q, :after['n_nics'][node]] = [after['nic_inuse'][node] >> i & 1 for i in range(after['n_nics'][node])]
        # every claimed NIC of a released pod is held by that pod alone: one pairing brings its counter to 0
        got, rnd = s.plan_batch_releases(tail, clock, rounds, tracked, used, rels)
        scratch.load_nodes(after)
        want = np.zeros(len(tail), dtype=wire.BINDING_DTYPE)
        want[:] = scratch.solve_batch(tail, clock)
        wrnd = np.where(want['status'] == wire.PLACED, 0, len(rounds)).astype('<i4')
        count = {n: used[q].astype(np.int64) for q, n in enumerate(tracked)}
        for k, c in enumerate(rounds, 1):
            idx = np.flatnonzero(want['status'] != wire.PLACED)
            if not len(idx):
                break
            cur = scratch.read_nodes()
            mine = rels[rels['round'] == k]
            for rl in mine:
                node = int(rl['node'])
                cur['used'][node] &= ~rl['cores']
                cur['gpu_used'][node] &= ~rl['gpus']
                if rl['hugepages_gb'] > 0:
                    cur['free_hugepages_gb'][node] += rl['hugepages_gb']
                count[node] -= rl['nic_pairings']
                cur['nic_inuse'][node] = _nic_bits(count[node], int(cur['n_nics'][node]))
                cur['busy_time'][node] = rl['clock']
            nodes = np.unique(mine['node']).astype('<i4')
            if len(nodes):
                scratch.update_nodes(nodes, cur[nodes])
            want[idx] = scratch.solve_batch(tail[idx], np.full(len(idx), c))
            for i in idx:
                node = int(want[i]['node'])
                if want[i]['status'] == wire.PLACED and node in count:
                    for j in range(int(want[i]['n_claimed'])):
                        count[node][want[i]['claimed_nics'][j]] += 1
            wrnd[idx[want['status'][idx] == wire.PLACED]] = k
        assert got.tobytes() == want.tobytes() and (rnd == wrnd).all(), helpers.first_binding_diff(want, got)
        placed = got['status'] == wire.PLACED
        assert placed.any() and not placed.all() and rnd[placed].max() >= 2
        base, brnd = s.plan_batch_rounds(tail, clock, rounds)
        assert int((got['status'] == wire.PLACED).sum()) >= int((base['status'] == wire.PLACED).sum())
    finally:
        s.close()
        scratch.close()
    # cuts on a sample: the 32 pods planned alone, releases with two pairings per NIC, and every free NIC of the nodes
    # the pods can take starting at -1
    sample = np.sort(np.random.default_rng(5).choice(len(tail), 32, replace=False))
    rels2 = rels[:64].copy()
    for rl in rels2:
        rl['nic_pairings'] = np.where(rl['nic_pairings'] > 0, 2, 0)
    group = [int(n) for n in np.flatnonzero(after['group_mask'] & tail['group_mask'][0])]
    tr2 = sorted({int(x['node']) for x in rels2} | set(group))
    used2 = np.zeros((len(tr2), wire.MAX_NICS), dtype='<i2')
    for q, node in enumerate(tr2):
        for i in range(int(after['n_nics'][node])):
            used2[q, i] = 1 if int(after['nic_inuse'][node]) >> i & 1 else (-1 if node in group else 0)
    s = _solver(speed, 30.0)
    try:
        s.load_nodes(after)
        got, rnd = s.plan_batch_releases(tail[sample], clock[sample], rounds, tr2, used2, rels2)
    finally:
        s.close()
    b, wrnd, _, cuts = oracle_releases(after, speed, tail[sample], clock[sample], rounds, tr2, used2, rels2, busy=30.0)
    assert got.tobytes() == b.tobytes() and (rnd == wrnd).all(), helpers.first_binding_diff(b, got)
    assert sum(cuts) > 0, cuts


# ---------------------------------------------------------------------------------------------- the scheduler
def _releases_against_the_reference(factory, limit=None):
    """``ForecastPending(departures=...)`` equals the reference's scans with the deletes played between them, frozen in
    tests/golden/live/releases.json.gz: the scan and node of every pending pod, and the reasons at the last scan of
    those no scan placed; nothing is written."""
    from tests.golden import make_live_golden
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import SCANS, evidence, release_sessions
    from tests.test_plan_reasons import _counted
    golden = make_live_golden.load('releases')['sessions']
    sessions = release_sessions()
    assert [g['name'] for g in golden] == [name for name, _ in sessions]
    assert all(evidence(golden))
    n = 0
    for (name, script), want in list(zip(sessions, golden))[:limit]:
        keys = [tuple(k) for k in want['pending']]
        for case in want['cases']:
            sched, k8s, _ = mirror_session(script, factory)
            try:
                state, traffic = dict(sched.pod_state), k8s.transcript()
                before = {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics]) for nd, v in sched.nodes.items()}
                deps = {(ns, pod): off for ns, pod, off in case['departures']}
                placement, reasons = sched.ForecastPending(SCANS, keys=keys, period=case['period'], reasons=True,
                                                           departures=deps)
                want_p = [None if p is None else (p[0], p[1]) for p in case['placed']]
                assert list(placement) == keys and list(placement.values()) == want_p, \
                    (name, case['departures'], list(placement.values()), want_p)
                assert reasons == _counted(case['reasons'], list(sched.nodes)), (name, case['departures'])
                assert k8s.transcript() == traffic and sched.pod_state == state, name
                assert {nd: (v.busy_time, list(v.pod_info), [x.pods_used for x in v.nics])
                        for nd, v in sched.nodes.items()} == before, name
                n += 1
            finally:
                sched.close()
    assert limit is not None or n >= 100, n


def test_forecast_pending_with_departures_equals_the_reference():
    """Deletes mid-gap, exactly at a scan's clock and inside the busy window before a scan, periods of 30 and 10 s;
    pods placed only after a release, held a scan by its busy stamp, and pods sharing a NIC a release drove negative."""
    _releases_against_the_reference(OraclePlanner)


def test_forecast_pending_checks_its_departures():
    from tests.golden.make_plan_golden import mirror_session
    from tests.golden.make_release_golden import release_sessions
    name, script = release_sessions()[-1]
    sched, _, _ = mirror_session(script, OraclePlanner)
    try:
        pending = list(sched.ForecastPending(3))
        deployed = [(ns, pod) for n in sched.nodes.values() for (pod, ns) in n.pod_info]
        with pytest.raises(ValueError):
            sched.ForecastPending(3, departures={deployed[0]: 10.0}, additions=[[]])
        with pytest.raises(ValueError):
            sched.ForecastPending(3, departures={pending[0]: 10.0})
        with pytest.raises(ValueError):
            sched.ForecastPending(3, departures={deployed[0]: 0.0})
        with pytest.raises(ValueError):
            sched.ForecastPending(3, departures={('ns0', 'never-annotated'): 10.0})
        plain = sched.ForecastPending(3, reasons=True)
        assert sched.ForecastPending(3, reasons=True, departures={}) == plain
        assert sched.ForecastPending(3, reasons=True, departures={deployed[0]: 1000.0}) == plain   # after the last scan
        assert sched.ForecastPending(3, departures={deployed[0]: 15.0}) != sched.ForecastPending(3)
    finally:
        sched.close()


@pytest.mark.gpu
def test_forecast_pending_with_departures_on_the_gpu():
    from tests.test_plan import _gpu_factory
    _releases_against_the_reference(_gpu_factory(), limit=6 if EMULATED else None)
