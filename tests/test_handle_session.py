"""One long-lived solver handle against a fresh handle and the oracle, call after call.

In production one handle lives as long as the process: it is loaded once and then takes updates, batches, previews,
plans, scenario calls, snapshots and restores by the thousand.  What it carries from one call to the next (node
arrays reused at the same super-tile count, hardware classes and NIC signatures that only grow, the tuple-limit
bookkeeping, the generations behind the explanation and snapshot rules, workspaces and scratch that only grow) is
pinned here: a seeded session generator and a runner that drives one ``Solver`` through the session and, after every
call, compares it

  * with the oracle (``oracle.binding.solve``, ``test_query.oracle_alone``, ``test_plan.oracle_plan``,
    ``test_defrag.oracle_defrag``, ``tests/explain_oracle.py``), byte for byte;
  * with a fresh handle in the same sweep mode, loaded with the records the call reads (a snapshot source is asked of
    the fresh handle as its mirror), refusals included: the same code, naming the same pod;
  * with the runner's own model of the records, the snapshot and the legality rules (DESIGN §8.6 - §8.10).

A session is plain data, a list of ``(op, args)``; ``make_session(seed, ...)`` rebuilds it from its seed, so a failure
names ``seed / step / op`` and replays alone.  ``tools/session_fuzz.py`` runs the same generator over many seeds."""
import os
import re

import numpy as np
import pytest

from nhd_b200 import packing, wire
from tests import scenarios

EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'
MODES = (dict(), dict(single_warp=True), dict(cpu_warps=1), dict(cpu_warps=2), dict(sweep_debug=1),
         dict(sweep_debug=5))                                             # as tests/test_query.py
BUSY = 30.0
# the speed table every session's handle is created with: workload.make_cluster's wild table first (100 / 40 / 25 G),
# then the other speeds scenarios.random_node and scenarios.signature_nodes use
SPEEDS = (100.0, 40.0, 25.0, 10.0, 12.0)
# one node, both sides of the 256-node super tile, more than 32 bitmap words (2 049 and 4 100 nodes)
SIZES = (1, 255, 256, 257, 700, 2049, 4100)
EMU_SIZES = (1, 255, 256, 257, 300)


def new_layout():
    """The packed layout every record and pod of a session goes through: fixed speed classes and group names."""
    lay = packing.ClusterLayout()
    for s in SPEEDS:
        lay.speed_class(s)
    for g in scenarios.GROUP_NAMES[:5]:
        lay.group_bit(g)
    return lay


def speed_table():
    return new_layout().speed_table()


def tuple_ok(k, g):
    """The mapping stage's enumeration limits (numa^(groups+1) tuples, numa^groups per group pick)."""
    return k ** (g + 1) <= wire.MAX_TUPLES and k ** g <= 64


def max_numa(recs, exclude=()):
    """The largest NUMA count among the nodes the filter could accept (active, not in maintenance, not excluded)."""
    ok = ((recs['flags'] & wire.NODE_ACTIVE) != 0) & ((recs['flags'] & wire.NODE_MAINTENANCE) == 0)
    if len(exclude):
        ok[np.asarray(list(exclude), dtype=np.int64)] = False
    return max(1, int(recs['n_numa'][ok].max())) if ok.any() else 1


def pod_refusal(pods, now, k):
    """(code, pod) of the first pod ``nhd_stage_batch`` refuses at tuple-limit NUMA count k, or None."""
    for i in range(len(pods)):
        if not np.isfinite(now[i]):
            return wire.ERR_INVALID, i
        if not tuple_ok(k, int(pods[i]['n_groups'])):
            return wire.ERR_UNSUPPORTED, i
    return None


def static_key(r):
    """What makes a node's hardware class: the static half of the record, the counts and the SMT flag."""
    b = np.ascontiguousarray(r).tobytes()
    return b[64:] + bytes([int(r['n_gpus']), int(r['n_nics']), int(r['n_numa']), int(r['flags']) & wire.NODE_SMT])


# ---------------------------------------------------------------------------------------------- records and pods
def pack(layout, nodes):
    import nhd_b200.Node as node_mod
    built = scenarios.build_nodes({'nodes': nodes}, node_mod)
    recs = packing.pack_nodes(list(built.values()), layout)
    assert layout.speeds == list(SPEEDS), layout.speeds                  # the handle's speed table still holds
    return recs


def special_nodes(rng, layout, k, tag):
    """k records from the scenario generators: random_node of every flavour, huge_node (1 / 2 / 4 NUMA nodes, up to
    256 logical cores) and NIC signature nodes."""
    nodes, sigs = [], scenarios.signature_list(400)
    for j in range(k):
        kind = int(rng.integers(0, 6))
        name = f'{tag}{j}'
        if kind < 4:
            nodes.append(scenarios.random_node(rng, name, ('mixed', 'wild', 'vf', 'big')[kind]))
        elif kind == 4:
            nodes.append(scenarios.huge_node(rng, name))
        else:
            a, b = rng.integers(0, len(sigs), 2)
            nodes.append(scenarios.signature_nodes(f'{name}s', [(sigs[a], sigs[b])])[0])
    return pack(layout, nodes)


def cluster_records(rng, layout, n):
    """n records: workload.make_cluster (regular or wild) with up to 24 of them replaced by scenario nodes."""
    import workload
    recs = workload.make_cluster(3, n_nodes=n, seed=int(rng.integers(1 << 30)), wild=bool(rng.random() < 0.5))[0]
    k = int(rng.integers(0, min(n, 24) + 1))
    if k:
        at = rng.choice(n, k, replace=False)
        recs[at] = special_nodes(rng, layout, k, 'x')
    return recs


def pod_pool(rng, layout):
    """Packed pod descriptors: random_pod of every flavour (up to four groups), huge_pod, the workload's types."""
    import nhd_b200.CfgTopology as cfg_mod
    import workload
    out = []
    for j in range(28):
        flavor = ('mixed', 'wild', 'vf', 'big')[j % 4]
        p = scenarios.random_pod(rng, flavor, max_groups=4 if j % 3 == 0 else 3)
        out.append(packing.pack_pod(scenarios.build_top(p, cfg_mod), p['groups'], layout))
    for _ in range(6):
        p = scenarios.huge_pod(rng)
        out.append(packing.pack_pod(scenarios.build_top(p, cfg_mod), p['groups'], layout))
    pods = np.concatenate([np.stack(out), workload.make_pod_types(3, seed=int(rng.integers(1 << 30)))])
    four = pods[pods['n_groups'] == 4]
    if not len(four):                                                      # at least one four-group pod
        four = pods[:1].copy()
        four['n_groups'] = 4
        for g in range(1, 4):
            four[0]['groups'][g] = four[0]['groups'][0]
        pods = np.concatenate([pods, four])
    return pods


class Draw:
    """The random parts of a session that need no handle state: pods with their clocks, node records."""

    def __init__(self, rng, layout):
        self.rng, self.layout = rng, layout
        self.pool = pod_pool(rng, layout)
        self.t = 1000.0

    def pods(self, lo, hi, four=None):
        rng = self.rng
        n = int(rng.integers(lo, hi + 1))
        four = rng.random() < 0.3 if four is None else four
        pool = self.pool if four else self.pool[self.pool['n_groups'] < 4]
        pods = pool[rng.integers(0, len(pool), n)].copy()
        if n and rng.random() < 0.5:                                       # one group list for the whole set
            pods['group_mask'] = pods[0]['group_mask']
        if rng.random() < 0.3:
            pods['map_type'][rng.random(n) < 0.15] = wire.MAP_NONE          # BAD_MAP_TYPE among the others
        if rng.random() < 0.5:                                             # standing decisions: one clock
            now = np.full(n, self.t)
        else:                                                              # busy windows that expire between pods
            steps = rng.choice([0.0, 0.0, 1.0, 5.0, 17.0, 31.0], n)
            now = self.t + np.cumsum(steps)
        if rng.random() < 0.06 and n:
            now[int(rng.integers(0, n))] = np.nan                          # refused, naming the pod
        self.t = float(np.nanmax(now, initial=self.t)) + float(rng.choice([0.0, 3.0, 40.0]))
        return pods, now

    def nodes(self, n):
        return cluster_records(self.rng, self.layout, n)


def make_session(seed, n_steps=30, sizes=SIZES):
    """A random session: ``{'seed', 'steps': [(op, args), ...]}``.  Ops and arguments only depend on the seed (node
    counts are tracked here so that indices stay in range); what they do to the records is the runner's business."""
    rng = np.random.default_rng(seed)
    d = Draw(rng, new_layout())
    steps = []
    weights = {'load_nodes': 2, 'update_nodes': 5, 'snapshot': 2, 'restore': 1.5, 'solve_batch': 6, 'query_batch': 3,
               'plan_batch': 3, 'plan_scenarios': 3, 'explain_batch': 1, 'explain_pod': 1, 'explain_macro': 2}
    names = list(weights)
    p = np.array([weights[k] for k in names])
    p = p / p.sum()
    n = int(rng.choice(sizes))
    steps.append(('load_nodes', {'recs': d.nodes(n)}))

    def src():
        return 'snapshot' if rng.random() < 0.4 else 'mirror'

    def some(k):
        return np.sort(rng.choice(n, min(n, k), replace=False)).astype(np.int32)

    def query():
        pods, now = d.pods(1, 12)
        return ('query_batch', {'pods': pods, 'now': now, 'source': src()})

    def plan():
        pods, now = d.pods(1, 32)
        ex = some(int(rng.integers(0, 6))) if rng.random() < 0.7 else np.zeros(0, np.int32)
        return ('plan_batch', {'pods': pods, 'now': now, 'source': src(), 'exclude': ex,
                               'explain': bool(rng.random() < 0.3)})

    def scen():
        out = []
        for _ in range(int(rng.integers(1, 6))):
            pods, now = d.pods(0, 14)
            ex = some(int(rng.integers(0, 4)))
            kind = rng.random()
            if kind < 0.4:
                out.append((ex, pods, now))                                # a plain drain
            else:
                lift = int(rng.integers(0, len(pods) + 1)) if kind < 0.8 else None
                edits = None
                if rng.random() < 0.6:
                    at = some(int(rng.integers(1, 3)))
                    edits = (at, d.nodes(len(at)))
                out.append((ex, pods, now, lift, edits))
        return ('plan_scenarios', {'scenarios': out, 'source': src()})

    while len(steps) < n_steps:
        op = names[int(rng.choice(len(names), p=p))]
        if op == 'load_nodes':
            n = int(rng.choice(sizes))
            steps.append((op, {'recs': d.nodes(n)}))
        elif op == 'update_nodes':
            idx = some(int(rng.integers(1, 17)))
            kind = ('hardware', 'flags', 'groups', 'release')[int(rng.integers(0, 4))]
            args = {'idx': idx, 'kind': kind}
            if kind == 'hardware':
                args['recs'] = d.nodes(len(idx))
            elif kind == 'flags':                                          # ACTIVE = 2, MAINTENANCE = 4
                args['set'] = rng.choice([0, wire.NODE_ACTIVE, wire.NODE_MAINTENANCE], len(idx)).astype(np.uint8)
                args['clear'] = rng.choice([0, wire.NODE_ACTIVE, wire.NODE_MAINTENANCE], len(idx)).astype(np.uint8)
            elif kind == 'groups':
                args['masks'] = rng.integers(1, 32, len(idx)).astype(np.uint64)
            else:
                args['back'] = int(rng.integers(1, 4))                     # the record from that many batches ago
            steps.append((op, args))
        elif op == 'solve_batch':
            pods, now = d.pods(1, 64)
            steps.append((op, {'pods': pods, 'now': now}))
        elif op == 'query_batch':
            steps.append(query())
        elif op == 'plan_batch':
            steps.append(plan())
        elif op == 'plan_scenarios':
            steps.append(scen())
        elif op in ('explain_batch', 'explain_pod'):
            steps.append((op, {'which': float(rng.random())}))
        elif op == 'explain_macro':                                         # the sequence explanations need
            steps.append(('snapshot', {}))
            pods, now = d.pods(8, 64, four=False)
            steps.append(('solve_batch', {'pods': pods, 'now': now}))
            for _ in range(int(rng.integers(0, 3))):
                steps.append((query, plan, scen)[int(rng.integers(0, 3))]())
            steps.append(('explain_batch', {'which': 0.0}))
            steps.append(('explain_pod', {'which': float(rng.random())}))
        else:
            steps.append((op, {}))
    return {'seed': seed, 'steps': steps}


# ---------------------------------------------------------------------------------------------- the runner
class Mismatch(AssertionError):
    pass


def _refusal(e):
    """(code, pod named or None) of a SolverError."""
    m = re.search(r'pod (\d+)', str(e))
    return e.code, (int(m.group(1)) if m else None)


class Runner:
    """Drives one handle through sessions, keeping the model: the current records, the snapshot's, and what the
    legality rules depend on.  ``stats`` counts what was compared."""

    def __init__(self, mode, speed=None, stats=None, fresh=True):
        from nhd_b200.solver import Solver
        self.Solver, self.mode = Solver, dict(mode)
        self.speed = speed_table() if speed is None else speed
        self.s = Solver(self.speed, min_busy_secs=BUSY, **self.mode)
        self.stats = stats if stats is not None else new_stats()
        self.check_fresh = fresh
        self.recs = None              # the mirror's records
        self.snap = None              # the snapshot's records (None: no snapshot since the last load)
        self.snap_fresh = False       # no load or update since the snapshot: the snapshot may be a source
        self.after_snap = False       # the last call that moved the generation was nhd_snapshot
        self.expl = None              # (pods, now, batch-start records, bindings) of an explainable batch
        self.history = []             # the records at the start of every batch

    def close(self):
        self.s.close()

    # -- helpers
    def fresh(self, recs):
        f = self.Solver(self.speed, min_busy_secs=BUSY, **self.mode)
        f.load_nodes(recs)
        return f

    def call(self, fn):
        from nhd_b200.solver import SolverError
        try:
            return fn(), None
        except SolverError as e:
            return None, _refusal(e)

    def expect(self, where, got_ref, want_ref):
        if got_ref is not None:
            self.stats['refusals'][got_ref[0]] = self.stats['refusals'].get(got_ref[0], 0) + 1
        if (got_ref is None) != (want_ref is None) or (want_ref is not None and
                                                       (got_ref[0], got_ref[1]) != tuple(want_ref)):
            raise Mismatch(f'{where}: refusal {got_ref}, expected {want_ref}')

    def same(self, where, got, want):
        if got.tobytes() != want.tobytes():
            from tests import helpers
            raise Mismatch(f'{where}: {helpers.first_binding_diff(want, got)}')
        if len(got) and got['node'].max() >= len(self.recs):
            raise Mismatch(f'{where}: a node outside the {len(self.recs)} loaded nodes (padding) was chosen')
        self.stats['bindings'] += len(got)
        st = self.stats['status']
        for k, v in zip(*np.unique(got['status'], return_counts=True)):
            st[int(k)] = st.get(int(k), 0) + int(v)

    def source(self, source):
        """(records the call reads, the refusal the model expects of the source)."""
        if source == 'snapshot' and (self.snap is None or not self.snap_fresh):
            return None, (wire.ERR_STATE, None)
        return (self.snap if source == 'snapshot' else self.recs), None

    def moved(self):
        self.after_snap = False
        self.expl = None

    # -- the operations
    def load_nodes(self, recs):
        self.s.load_nodes(recs)
        self.recs = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE).copy()
        self.snap, self.snap_fresh = None, False
        self.history = []
        self.moved()

    def update_nodes(self, idx, kind, recs=None, set=None, clear=None, masks=None, back=None):
        idx = np.asarray(idx, dtype=np.int64)
        new = self.recs[idx].copy()
        if kind == 'hardware':
            new = np.asarray(recs, dtype=wire.NODE_DTYPE).copy()
        elif kind == 'flags':
            new['flags'] = (new['flags'] & ~np.asarray(clear, dtype=np.uint8)) | np.asarray(set, dtype=np.uint8)
        elif kind == 'groups':
            new['group_mask'] = masks
        elif kind == 'release':
            if len(self.history) >= back:
                new = self.history[-back][idx].copy()
        self.s.update_nodes(idx, new)
        self.recs[idx] = new
        self.snap_fresh = False
        self.moved()

    def snapshot(self):
        self.s.snapshot()
        self.snap, self.snap_fresh = self.recs.copy(), True
        self.moved()
        self.after_snap = True

    def restore(self):
        _, ref = self.call(self.s.restore)
        self.expect('restore', ref, None if self.snap is not None else (wire.ERR_STATE, None))
        if self.snap is not None:
            self.recs = self.snap.copy()
            self.moved()

    def solve_batch(self, pods, now):
        from oracle import binding
        start, on_snap = self.recs.copy(), self.after_snap
        want_ref = pod_refusal(pods, now, max_numa(start))
        got, ref = self.call(lambda: self.s.solve_batch(pods, now))
        self.expect('solve_batch', ref, want_ref)
        self.moved()
        if self.check_fresh:
            f = self.fresh(start)
            try:
                fgot, fref = self.call(lambda: f.solve_batch(pods, now))
            finally:
                f.close()
            self.expect('solve_batch on a fresh handle', fref, want_ref)
        if want_ref is not None:
            return
        want, final = binding.solve(start, self.speed, pods, now, min_busy_secs=BUSY)
        self.same('solve_batch against the oracle', got, want)
        if self.check_fresh:
            self.same('solve_batch against a fresh handle', got, fgot)
        self.history.append(start)
        self.recs = final
        if on_snap:
            self.expl = (pods.copy(), now.copy(), start, got.copy())

    def query_batch(self, pods, now, source):
        from tests.test_query import oracle_alone
        recs, want_ref = self.source(source)
        want_ref = want_ref or pod_refusal(pods, now, max_numa(self.recs))
        got, ref = self.call(lambda: self.s.query_batch(pods, now, source=source))
        self.expect(f'query_batch ({source})', ref, want_ref)
        if recs is None:
            return
        if self.check_fresh:
            f = self.fresh(recs)
            try:
                fgot, fref = self.call(lambda: f.query_batch(pods, now))
            finally:
                f.close()
            self.expect('query_batch on a fresh handle', fref, want_ref)
        if want_ref is None:
            self.same(f'query_batch ({source}) against the oracle', got, oracle_alone(recs, self.speed, pods, now, BUSY))
            if self.check_fresh:
                self.same(f'query_batch ({source}) against a fresh handle', got, fgot)

    def plan_batch(self, pods, now, source, exclude, explain):
        from tests.test_plan import oracle_plan
        recs, want_ref = self.source(source)
        ex = [int(i) for i in exclude]
        want_ref = want_ref or pod_refusal(pods, now, max_numa(self.recs, ex))
        got, ref = self.call(lambda: self.s.plan_batch(pods, now, source=source, exclude=ex, explain=explain))
        self.expect(f'plan_batch ({source})', ref, want_ref)
        if recs is None:
            return
        if self.check_fresh:
            f = self.fresh(recs)
            try:
                fgot, fref = self.call(lambda: f.plan_batch(pods, now, exclude=ex, explain=explain))
            finally:
                f.close()
            self.expect('plan_batch on a fresh handle', fref, want_ref)
        if want_ref is not None:
            return
        want, counts = oracle_plan(recs, self.speed, pods, now, ex, BUSY)
        b = got[0] if explain else got
        self.same(f'plan_batch ({source}) against the oracle', b, want)
        if explain and got[1].tobytes() != counts.tobytes():
            raise Mismatch(f'plan_batch ({source}): explanation counts differ from the oracle')
        if self.check_fresh:
            self.same(f'plan_batch ({source}) against a fresh handle', b, fgot[0] if explain else fgot)

    def plan_scenarios(self, scenarios, source):
        from tests.test_defrag import oracle_defrag
        from tests.test_plan import oracle_plan
        recs, want_ref = self.source(source)
        got, ref = self.call(lambda: self.s.plan_scenarios(scenarios, source=source))
        self.expect(f'plan_scenarios ({source})', ref, want_ref)
        if recs is None:
            return
        fgot = None
        if self.check_fresh:
            f = self.fresh(recs)
            try:
                fgot = f.plan_scenarios(scenarios)
            finally:
                f.close()
        k = max_numa(self.recs)
        for sc in scenarios:
            if len(sc) > 4 and sc[4] is not None:
                k = max(k, int(np.asarray(sc[4][1])['n_numa'].max()))
        for j, sc in enumerate(scenarios):
            ex, pods, now = sc[:3]
            lift = sc[3] if len(sc) > 3 else None
            edits = sc[4] if len(sc) > 4 else None
            code, pod, b = got[j]
            want_ref = pod_refusal(pods, now, k)
            self.expect(f'plan_scenarios ({source}) scenario {j}', None if code == 0 else (code, pod), want_ref)
            if fgot is not None:
                self.expect(f'plan_scenarios scenario {j} on a fresh handle',
                            None if fgot[j][0] == 0 else fgot[j][:2], want_ref)
            if want_ref is not None:
                continue
            exl = [int(i) for i in ex]
            if lift is None and edits is None:
                want = oracle_plan(recs, self.speed, pods, now, exl, BUSY)[0] if len(pods) else b
            else:
                want = oracle_defrag(recs, self.speed, pods, now, exl, lift, edits, busy=BUSY)
            self.same(f'plan_scenarios ({source}) scenario {j} against the oracle', b, want)
            if fgot is not None:
                self.same(f'plan_scenarios ({source}) scenario {j} against a fresh handle', b, fgot[j][2])

    def _explained(self, what, fn, fresh_fn, want_fn):
        got, ref = self.call(fn)
        self.expect(what, ref, None if self.expl is not None else (wire.ERR_STATE, None))
        if self.expl is None:
            return
        pods, now, start, bindings = self.expl
        want = want_fn(pods, now, start)
        if got.tobytes() != want.tobytes():
            raise Mismatch(f'{what}: differs from the oracle')
        if self.check_fresh:
            f = self.fresh(start)
            try:
                f.snapshot()
                f.solve_batch(pods, now)
                if fresh_fn(f).tobytes() != got.tobytes():
                    raise Mismatch(f'{what}: differs from a fresh handle')
            finally:
                f.close()
        if self.s.fetch_bindings().tobytes() != bindings.tobytes():
            raise Mismatch(f'{what}: the batch\'s bindings changed')
        self.stats['explained'] += 1

    def explain_batch(self, which):
        from tests import explain_oracle
        self._explained('explain_batch', self.s.explain_batch, lambda f: f.explain_batch(),
                        lambda pods, now, start: explain_oracle.counts(
                            explain_oracle.batch(start, self.speed, pods, now, min_busy_secs=BUSY)[1], len(pods)))

    def explain_pod(self, which):
        from tests import explain_oracle
        i = 0
        if self.expl is not None:
            failed = np.flatnonzero(self.expl[3]['status'] == wire.NO_CANDIDATE)
            n = len(self.expl[3])
            i = int(failed[int(which * len(failed))]) if len(failed) and which < 0.8 else int(which * n)

        def want(pods, now, start):
            r = explain_oracle.batch(start, self.speed, pods, now, which=[i], min_busy_secs=BUSY)[1]
            return r[i] if i in r else np.full(len(start), wire.WHY_NONE, dtype=np.uint8)
        self._explained(f'explain_pod({i})', lambda: self.s.explain_pod(i), lambda f: f.explain_pod(i), want)

    # -- one step, then the records
    def step(self, op, args):
        self.stats['ops'][op] = self.stats['ops'].get(op, 0) + 1
        getattr(self, op)(**args)
        self.stats['calls'] += 1
        if self.recs is not None and self.s.read_nodes().tobytes() != self.recs.tobytes():
            from tests import ref_compare
            raise Mismatch(f'records after {op}: {ref_compare.diff_records(self.recs, self.s.read_nodes())[:3]}')

    def run(self, session):
        for k, (op, args) in enumerate(session['steps']):
            try:
                self.step(op, args)
            except Mismatch as e:
                raise Mismatch(f"seed {session['seed']} / step {k} / op {op} / mode {self.mode}: {e}") from None


def new_stats():
    return {'ops': {}, 'refusals': {}, 'status': {}, 'bindings': 0, 'calls': 0, 'explained': 0}


def run_session(session, mode, stats=None):
    r = Runner(mode, stats=stats)
    try:
        r.run(session)
    finally:
        r.close()
    return r.stats


# ---------------------------------------------------------------------------------------------- random sessions
N_SESSIONS, N_STEPS = (12, 20) if EMULATED else (48, 30)


@pytest.mark.gpu
def test_random_sessions_equal_a_fresh_handle_and_the_oracle():
    stats = new_stats()
    for seed in range(N_SESSIONS):
        run_session(make_session(seed, N_STEPS, EMU_SIZES if EMULATED else SIZES), MODES[seed % len(MODES)], stats)
    print('session stats:', stats)
    ops = set(stats['ops'])
    assert ops >= {'load_nodes', 'update_nodes', 'snapshot', 'restore', 'solve_batch', 'query_batch', 'plan_batch',
                   'plan_scenarios', 'explain_batch', 'explain_pod'}, stats['ops']
    assert set(stats['refusals']) >= {wire.ERR_STATE, wire.ERR_UNSUPPORTED, wire.ERR_INVALID}, stats['refusals']
    assert all(stats['status'].get(s, 0) > 0 for s in (wire.PLACED, wire.NO_CANDIDATE, wire.ASSIGN_FAILED,
                                                       wire.BAD_MAP_TYPE)), stats['status']
    assert stats['explained'] >= (3 if EMULATED else 20), stats
    assert stats['bindings'] > (2000 if EMULATED else 15000), stats


# ---------------------------------------------------------------------------------------------- named sessions
def _mode_params():
    return [pytest.param(m, id='-'.join(f'{k}{v}' for k, v in m.items()) or 'default')
            for m in (MODES[:1] if EMULATED else MODES)]


def _pods(layout, pods):
    import nhd_b200.CfgTopology as cfg_mod
    return np.stack([packing.pack_pod(scenarios.build_top(p, cfg_mod), p['groups'], layout) for p in pods])


def _restricted_growth(n):
    """Switch ids of n NICs in order of first appearance (as the packed records number them): 4 140 for n = 8."""
    if n == 0:
        yield ()
        return
    for p in _restricted_growth(n - 1):
        for s in range(max(p, default=-1) + 2):
            yield p + (s,)


def class_records(layout, patterns, smt):
    """One 2-NUMA node with eight 100 G NICs per switch pattern: a distinct static description each."""
    base = pack(layout, [scenarios.make_node('k', 2, 16, smt, 1, (), [(f'e{j}', 100000, j // 4, 0x10 + j)
                                                                      for j in range(8)], hp_alloc=64)])[0]
    recs = np.repeat(base[None], len(patterns))
    for i, sw in enumerate(patterns):
        recs[i]['nic_sw'][0] = sum(int(s) << (4 * j) for j, s in enumerate(sw))
    return recs


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_class_slots_run_out_through_updates_and_loads(mode):
    """More than 4 096 distinct static descriptions through updates and loads of one handle: its later nodes have
    no class and take the general path, while a fresh handle loaded with the same records classifies them all."""
    lay = new_layout()
    pats = list(_restricted_growth(8))
    n = 300 if EMULATED else 2049
    a, b = class_records(lay, pats, False), class_records(lay, pats, True)
    pods = _pods(lay, scenarios.signature_pods() * 6)
    now = np.full(len(pods), 2000.0)
    seen = set()
    steps = []
    for k in range(0, len(pats) if not EMULATED else 2 * n, n):           # loads and updates in turn
        recs = np.concatenate([a, b])[k:k + n]
        if len(recs) < n:
            break
        if not steps or (k // n) % 2 == 0:
            steps.append(('load_nodes', {'recs': recs}))
        else:
            steps.append(('update_nodes', {'idx': np.arange(n, dtype=np.int32), 'kind': 'hardware', 'recs': recs}))
        seen.update(static_key(r) for r in recs)
    tail = np.concatenate([b[-n:]])
    seen.update(static_key(r) for r in tail)
    steps += [('load_nodes', {'recs': tail}), ('solve_batch', {'pods': pods, 'now': now}),
              ('query_batch', {'pods': pods[:8], 'now': now[:8], 'source': 'mirror'}),
              ('snapshot', {}), ('solve_batch', {'pods': pods, 'now': now + 1}),
              ('plan_batch', {'pods': pods, 'now': now, 'source': 'snapshot', 'exclude': np.arange(0, n, 7),
                              'explain': False}),
              ('update_nodes', {'idx': np.arange(0, n, 3, dtype=np.int32), 'kind': 'hardware', 'recs': a[:n][::3]}),
              ('solve_batch', {'pods': pods, 'now': now + 40})]
    if not EMULATED:
        assert len(seen) > 4096, len(seen)                                 # the slots really ran out
    stats = run_session({'seed': 'class-slots', 'steps': steps}, mode)
    assert stats['status'].get(wire.PLACED, 0) > 20, stats


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_signature_ids_past_128_through_loads(mode):
    """Two loads of 100 distinct per-NUMA NIC signatures each: the handle's signature table (128 ids) runs out on the
    second load, a fresh handle's does not."""
    lay = new_layout()
    sigs = scenarios.signature_list(200)
    first = pack(lay, scenarios.signature_nodes('s', [(sigs[2 * i], sigs[2 * i + 1]) for i in range(50)]))
    second = pack(lay, scenarios.signature_nodes('t', [(sigs[100 + 2 * i], sigs[101 + 2 * i]) for i in range(50)]))
    pods = _pods(lay, scenarios.signature_pods() * 10)
    now = np.full(len(pods), 2000.0)
    steps = [('load_nodes', {'recs': first}), ('solve_batch', {'pods': pods, 'now': now}),
             ('load_nodes', {'recs': second}), ('solve_batch', {'pods': pods, 'now': now}),
             ('query_batch', {'pods': pods[:12], 'now': now[:12], 'source': 'mirror'}),
             ('plan_batch', {'pods': pods, 'now': now, 'source': 'mirror', 'exclude': np.arange(0, 50, 4),
                             'explain': True}),
             ('load_nodes', {'recs': np.concatenate([second, first])}), ('solve_batch', {'pods': pods, 'now': now})]
    run_session({'seed': 'signatures', 'steps': steps}, mode)


def _four_numa_cluster(lay, n=300, seed=3):
    """A regular cluster with node 5 a 4-NUMA node (huge_node), in maintenance at first."""
    rng = np.random.default_rng(seed)
    while True:
        four = special_nodes(rng, lay, 1, 'q')
        if four['n_numa'][0] == 4:
            break
    four['flags'] |= wire.NODE_ACTIVE | wire.NODE_MAINTENANCE
    recs = cluster_records(rng, lay, n)
    recs = recs[recs['n_numa'] <= 2].copy()                                # no other node decides the limit
    recs[5] = four[0]
    return recs


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_the_tuple_limit_follows_updates(mode):
    """A 4-NUMA node into and out of maintenance, inactive and active again, through updates (and back through a
    restore): 4-group pods are refused exactly while it is schedulable, by batch, query, plan and scenario calls."""
    lay = new_layout()
    recs = _four_numa_cluster(lay)
    d = Draw(np.random.default_rng(11), lay)
    pods, now = d.pods(10, 10, four=False)
    four = d.pool[d.pool['n_groups'] == 4][:1]
    pods = np.concatenate([pods[:3], four, pods[3:]])
    now = np.full(len(pods), 5000.0)

    def whatif(t):
        return [('solve_batch', {'pods': pods, 'now': now + t}),
                ('query_batch', {'pods': pods, 'now': now + t, 'source': 'mirror'}),
                ('plan_batch', {'pods': pods, 'now': now + t, 'source': 'mirror', 'exclude': np.array([5]),
                                'explain': False}),
                ('plan_batch', {'pods': pods, 'now': now + t, 'source': 'mirror', 'exclude': np.array([6]),
                                'explain': False}),
                ('plan_scenarios', {'scenarios': [([5], pods, now + t), ([], pods, now + t, 2, None)],
                                    'source': 'mirror'})]

    def flags(set_, clear):
        return ('update_nodes', {'idx': np.array([5], np.int32), 'kind': 'flags',
                                 'set': np.array([set_], np.uint8), 'clear': np.array([clear], np.uint8)})
    steps = [('load_nodes', {'recs': recs})] + whatif(0)
    steps += [flags(0, wire.NODE_MAINTENANCE)] + whatif(100)               # schedulable: refused
    steps += [flags(0, wire.NODE_ACTIVE)] + whatif(200)                    # inactive: accepted
    steps += [flags(wire.NODE_ACTIVE, 0), ('snapshot', {})] + whatif(300)  # schedulable again
    steps += [flags(wire.NODE_MAINTENANCE, 0)] + whatif(400)               # in maintenance
    steps += [('restore', {})] + whatif(500)                               # back to the snapshot: schedulable
    steps += [flags(wire.NODE_MAINTENANCE, 0), ('snapshot', {}), flags(0, wire.NODE_MAINTENANCE), ('restore', {})]
    steps += whatif(600)                                                   # back to maintenance by the restore
    stats = run_session({'seed': 'tuple-limit', 'steps': steps}, mode)
    assert stats['refusals'].get(wire.ERR_UNSUPPORTED, 0) >= 3 * 4, stats['refusals']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_a_restore_after_hardware_updates_equals_a_fresh_handle(mode):
    """snapshot -> updates that change the nodes' hardware -> restore: the restored records are classified again,
    and the batch after the restore equals a fresh handle's and the oracle's (the mirror once kept the updated nodes'
    hardware classes, and the tuple-limit bookkeeping of the updated records, across the restore)."""
    lay = new_layout()
    rng = np.random.default_rng(21)
    recs = cluster_records(rng, lay, 257)
    other = cluster_records(rng, lay, 257)
    d = Draw(rng, lay)
    pods, now = d.pods(40, 40, four=False)
    half = np.arange(0, 257, 2, dtype=np.int32)
    steps = [('load_nodes', {'recs': recs}), ('snapshot', {}),
             ('update_nodes', {'idx': half, 'kind': 'hardware', 'recs': other[half]}),
             ('restore', {}), ('solve_batch', {'pods': pods, 'now': now}),
             ('query_batch', {'pods': pods[:10], 'now': now[:10], 'source': 'mirror'}),
             ('plan_scenarios', {'scenarios': [([1, 2], pods, now), ([3], pods, now, 5, ([4], other[[4]]))],
                                 'source': 'mirror'})]
    run_session({'seed': 'restore-after-update', 'steps': steps}, mode)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_shrink_and_grow_across_a_super_tile_around_a_snapshot(mode):
    """257 -> 255 -> 700 nodes with snapshots in between: after a load the snapshot source and restore are refused,
    no padding node is ever chosen, and the first batch on the grown cluster equals a fresh handle's."""
    lay = new_layout()
    rng = np.random.default_rng(31)
    d = Draw(rng, lay)
    big, small, grown = d.nodes(257), d.nodes(255), d.nodes(700)
    pods, now = d.pods(48, 48, four=False)
    steps = [('load_nodes', {'recs': big}), ('snapshot', {}), ('solve_batch', {'pods': pods, 'now': now}),
             ('load_nodes', {'recs': small}),
             ('query_batch', {'pods': pods[:6], 'now': now[:6], 'source': 'snapshot'}),
             ('plan_batch', {'pods': pods, 'now': now, 'source': 'snapshot', 'exclude': np.zeros(0), 'explain': False}),
             ('plan_scenarios', {'scenarios': [([], pods, now)], 'source': 'snapshot'}),
             ('restore', {}), ('solve_batch', {'pods': pods, 'now': now + 50}),
             ('snapshot', {}), ('load_nodes', {'recs': grown}), ('restore', {}),
             ('solve_batch', {'pods': pods, 'now': now + 100}),
             ('query_batch', {'pods': pods, 'now': now + 100, 'source': 'mirror'}),
             ('load_nodes', {'recs': small}), ('solve_batch', {'pods': pods, 'now': now + 200}),
             ('snapshot', {}), ('load_nodes', {'recs': small[:250]}),        # the same super-tile count
             ('query_batch', {'pods': pods[:6], 'now': now[:6], 'source': 'snapshot'}), ('restore', {}),
             ('solve_batch', {'pods': pods, 'now': now + 300})]
    stats = run_session({'seed': 'shrink-grow', 'steps': steps}, mode)
    assert stats['refusals'].get(wire.ERR_STATE, 0) == 7, stats['refusals']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_explanations_after_interleaved_whatif_calls(mode):
    """snapshot -> batch -> queries, plans and scenarios on both sources -> explanations: equal to the oracle's and a
    fresh handle's, and the batch's bindings unchanged; a restore then makes them refuse."""
    from tests.explain_scenarios import explain_scenarios
    from tests.test_query import packed
    recs, pods, now, speed, busy = packed(explain_scenarios()[1])
    assert busy == BUSY
    r = Runner(mode, speed=speed)
    try:
        r.run({'seed': 'explain', 'steps': [
            ('load_nodes', {'recs': recs}), ('snapshot', {}), ('solve_batch', {'pods': pods, 'now': now}),
            ('query_batch', {'pods': pods, 'now': now, 'source': 'mirror'}),
            ('query_batch', {'pods': pods[::-1], 'now': now[::-1], 'source': 'snapshot'}),
            ('plan_batch', {'pods': pods, 'now': now, 'source': 'snapshot', 'exclude': [0, 2], 'explain': True}),
            ('plan_batch', {'pods': pods[:5], 'now': now[:5], 'source': 'mirror', 'exclude': [], 'explain': False}),
            ('plan_scenarios', {'scenarios': [([1], pods, now), ([0], pods, now, 3, ([2], recs[[1]]))],
                                'source': 'snapshot'}),
            ('plan_scenarios', {'scenarios': [([], pods[:4], now[:4])], 'source': 'mirror'}),
            ('explain_batch', {'which': 0.0}), ('explain_pod', {'which': 0.0}), ('explain_pod', {'which': 0.5}),
            ('explain_pod', {'which': 0.9}), ('restore', {}), ('explain_batch', {'which': 0.0})]})
        assert r.stats['explained'] == 4 and r.stats['refusals'] == {wire.ERR_STATE: 1}, r.stats
    finally:
        r.close()
