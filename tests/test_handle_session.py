"""One long-lived solver handle against a fresh handle and the oracle, call after call.

In production one handle lives as long as the process: it is loaded once and then takes updates, batches, previews,
plans, scenario calls, snapshots and restores by the thousand.  What it carries from one call to the next (node
arrays reused at the same super-tile count, hardware classes and NIC signatures that only grow, the tuple-limit
bookkeeping, the generations behind the explanation and snapshot rules, workspaces and scratch that only grow) is
pinned here: a seeded session generator and a runner that drives one ``Solver`` through the session and, after every
call, compares it

  * with the oracle (``oracle.binding.solve``, ``test_query.oracle_alone``, ``test_plan.oracle_plan``,
    ``test_defrag.oracle_defrag``, ``tests/explain_oracle.py``; for the forecasts ``test_plan_reasons.oracle_explained``,
    ``test_expand.oracle_grown``, ``test_forecast.oracle_rounds``, ``test_forecast_releases.oracle_releases``), byte
    for byte;
  * with a fresh handle in the same sweep mode, loaded with the records the call reads (a snapshot source is asked of
    the fresh handle as its mirror), refusals included: the same code, naming the same pod;
  * with the runner's own model of the records, the snapshot, the deployed pods and the legality rules (DESIGN §8.6 -
    §8.15), refusals in the order the library checks them.

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


def scenario_call_refusal(scs, src_ref, n_classes):
    """(code, pod, rule) refusing a whole scenario call, in the order nhd_api.cu's plan_scenarios checks: every
    scenario's first round clock against its pods' clocks (before the source is read), the source, then the added
    records (a NIC speed class the handle lacks).  ``scs``: 7-tuples."""
    for ex, pods, now, lift, edits, adds, rounds in scs:
        if rounds is not None and len(rounds):
            late = np.flatnonzero(np.asarray(now) > rounds[0])
            if len(late):
                return wire.ERR_INVALID, int(late[0]), 'round clock'
    if src_ref is not None:
        return src_ref + ('source',)
    for sc in scs:
        if sc[5] is not None:
            for r in np.asarray(sc[5][1], dtype=wire.NODE_DTYPE):
                spd = int(r['nic_speed'][0]) | int(r['nic_speed'][1]) << 64
                if any((spd >> (4 * i)) & 0xF >= n_classes for i in range(int(r['n_nics']))):
                    return wire.ERR_INVALID, None, 'speed class'
    return None


def batch_refusal(pods, now, rounds, rel, src_ref, recs, k):
    """(code, pod, rule) of plan_batch_rounds (``rel`` None) or plan_batch_releases (``rel``: tracked, pods_used,
    releases), in the order nhd_api.cu's plan_batch checks: round clocks and the releases' rounds and clocks, the
    source, tracked nodes and untracked releases, the device check of pods_used against the NIC bits, then the pods
    (non-finite clocks, the tuple limit at NUMA count k)."""
    if len(rounds):
        late = np.flatnonzero(np.asarray(now) > rounds[0])
        if len(late):
            return wire.ERR_INVALID, int(late[0]), 'round clock'
    if rel is not None:
        fin = now[np.isfinite(now)]
        t0 = float(fin.max()) if len(fin) else -np.inf
        for j, rl in enumerate(rel[2]):
            r, c = int(rl['round']), float(rl['clock'])
            if not (1 <= r <= len(rounds)) or not np.isfinite(c) or (j and c < rel[2][j - 1]['clock']) or \
                    c < (t0 if r == 1 else rounds[r - 2]) or c > rounds[r - 1]:
                return wire.ERR_INVALID, None, 'release gap'
    if src_ref is not None:
        return src_ref + ('source',)
    if rel is not None:
        tracked, used, rels = rel
        if len(set(tracked)) != len(tracked) or any(t < 0 or t >= len(recs) for t in tracked):
            return wire.ERR_INVALID, None, 'tracked'
        if any(int(n) not in tracked for n in rels['node']):
            return wire.ERR_INVALID, None, 'untracked'
        for t, node in enumerate(tracked):
            nn, inuse = int(recs['n_nics'][node]), int(recs['nic_inuse'][node])
            if any(((used[t, i] > 0) != bool(inuse >> i & 1)) if i < nn else used[t, i] != 0
                   for i in range(wire.MAX_NICS)):
                return wire.ERR_INVALID, None, 'pods_used sign'
    ref = pod_refusal(pods, now, k)
    return None if ref is None else ref + ('pod',)


def _result_bytes(res):
    """A call's result, arrays as bytes, to compare two handles' answers."""
    return None if res is None else tuple(x.tobytes() if isinstance(x, np.ndarray) else x for x in res)


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


    def added(self, k):
        """k records for a grown scenario: the cluster's kinds, some replaced by a 4-NUMA huge_node, made GPU-less, put
        in maintenance or given a node-group bit no loaded node has."""
        rng = self.rng
        recs = self.nodes(k)
        for j in range(k):
            kind = int(rng.integers(0, 7))
            if kind == 0:
                recs[j] = self.four_numa()
            elif kind == 1:
                for f in ('n_gpus', 'gpu_used', 'gpu_numa_mask', 'gpu_sw'):
                    recs[j][f] = 0
            elif kind == 2:
                recs[j]['flags'] |= wire.NODE_ACTIVE | wire.NODE_MAINTENANCE
            elif kind == 3:
                recs[j]['group_mask'] = np.uint64(1) << np.uint64(62)
        return recs

    def four_numa(self):
        if not hasattr(self, '_four'):
            while True:
                r = special_nodes(self.rng, self.layout, 1, 'h')
                if r['n_numa'][0] == 4:
                    break
            r['flags'] |= wire.NODE_ACTIVE
            r['flags'] &= np.uint8(0xFF ^ wire.NODE_MAINTENANCE)
            self._four = r[0]
        return self._four

    def rounds(self, now, lo=1, hi=6, early=False):
        """Later scan clocks from the pods' last clock, periods around the busy window; ``early``: the first is before
        the clock of one of the pods (a malformed call)."""
        rng = self.rng
        fin = now[np.isfinite(now)]
        t = float(fin.max()) if len(fin) else self.t
        k = int(rng.integers(lo, hi + 1))
        out = list(t + np.cumsum(rng.choice([0.0, BUSY / 3.0, BUSY, BUSY + 1.0, 7.0], k)))
        if early and k and len(fin):
            out[0] = float(fin[int(rng.integers(0, len(fin)))]) - 1.0
        return out


# the ops of the sessions before the forecast calls, with their weights: the default of make_session, so that every
# seed still generates the session it always did
BASIC_WEIGHTS = {'load_nodes': 2, 'update_nodes': 5, 'snapshot': 2, 'restore': 1.5, 'solve_batch': 6, 'query_batch': 3,
                 'plan_batch': 3, 'plan_scenarios': 3, 'explain_batch': 1, 'explain_pod': 1, 'explain_macro': 2}
BASIC = tuple(BASIC_WEIGHTS)
# the scenario and batch forecasts: explained, grown and round scenario calls, plan_batch_rounds, plan_batch_releases
FORECAST_WEIGHTS = {'plan_explained': 2, 'plan_grown': 2, 'plan_rounds': 2, 'batch_rounds': 2, 'batch_releases': 3}
FORECASTS = tuple(FORECAST_WEIGHTS)
# the share of scenario forecasts and plan_batch_rounds calls malformed on purpose (with every fourth
# plan_batch_releases call: some 3 % of the calls of a session with the forecasts)
MALFORMED = 0.22


def make_session(seed, n_steps=30, sizes=SIZES, kinds=BASIC):
    """A random session: ``{'seed', 'steps': [(op, args), ...]}``.  Ops and arguments only depend on the seed (node
    counts are tracked here so that indices stay in range); what they do to the records is the runner's business.
    ``kinds``: the ops drawn (``BASIC``, the default, or with ``FORECASTS``); the explanation sequence also mixes in
    the forecast ops drawn."""
    rng = np.random.default_rng(seed)
    d = Draw(rng, new_layout())
    steps = []
    weights = {k: v for k, v in {**BASIC_WEIGHTS, **FORECAST_WEIGHTS}.items() if k in kinds}
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

    def bad():
        return rng.random() < MALFORMED
    made = []

    def forecast_scen(op):
        """Scenarios of 0 to 8 pods (32 at most per call) with lifts and edits; grown: added records, an unknown speed
        class on one of them now and then; rounds: mixed with scenarios of no rounds (None) and empty ones."""
        out = []
        wrong = bad()
        for _ in range(int(rng.integers(1, 5))):
            pods, now = d.pods(0, 8)
            ex = some(int(rng.integers(0, 4)))
            lift = int(rng.integers(0, len(pods) + 1)) if rng.random() < 0.5 else None
            edits = None
            if rng.random() < 0.4:
                at = some(int(rng.integers(1, 3)))
                edits = (at, d.nodes(len(at)))
            adds = None
            if op != 'plan_explained' and (op == 'plan_grown' or rng.random() < 0.4) and rng.random() < 0.85:
                k = int(rng.integers(1, 4))
                adds = (np.sort(rng.integers(0, n + 1, k)).astype(np.int32), d.added(k))
                if op == 'plan_grown' and wrong and (adds[1]['n_nics'] > 0).any():
                    j = int(np.flatnonzero(adds[1]['n_nics'] > 0)[0])
                    adds[1][j]['nic_speed'][0] = (int(adds[1][j]['nic_speed'][0]) & ~0xF) | 0xF
                    wrong = False
            rounds = None
            if op == 'plan_rounds':
                kind = rng.random()
                rounds = d.rounds(now, early=wrong) if kind < 0.7 else ([] if kind < 0.85 else None)
                wrong = wrong and not rounds
            out.append((ex, pods, now, lift, edits, adds, rounds))
        return (op, {'scenarios': out, 'source': src()})

    def batch_forecast(op):
        """plan_batch_rounds / plan_batch_releases of up to 32 pods over up to 6 rounds; the releases and the tracked
        free-NIC nodes as fractions of the deployed pods and nodes the runner knows of."""
        pods, now = d.pods(1, 32)
        if rng.random() < 0.4 and np.isfinite(now).any():                 # one descriptor at one clock: the nodes
            pods[:] = pods[int(rng.integers(0, len(pods)))]               # that fit it are stamped busy in turn, and
            now[:] = now[np.isfinite(now)].max()                          # the rest wait for a later round
        wrong = bad()
        ex = some(int(rng.integers(0, 6))) if rng.random() < 0.7 else np.zeros(0, np.int32)
        args = {'pods': pods, 'now': now, 'source': src(), 'exclude': ex, 'explain': bool(rng.random() < 0.5)}
        if op == 'batch_rounds':
            args['rounds'] = d.rounds(now, 0 if rng.random() < 0.1 else 1, early=wrong)
            return (op, args)
        made.append(op)                                                    # every fourth one broken, the ways in turn
        k = made.count(op)
        how = ('gap', 'untracked', 'sign')[(seed + k // 4) % 3] if k % 4 == 0 else None
        args['rounds'] = d.rounds(now)
        r = len(args['rounds'])
        args['ends'] = [(float(rng.random()), int(rng.integers(1, r + 1)), float(rng.choice([0.0, 0.5, 1.0, rng.random()])),
                         int(rng.integers(1, 3))) for _ in range(int(rng.integers(0, 9)))]
        args['extra'] = [(float(rng.random()), int(rng.integers(1, 1 << 32)), -1 - int(rng.integers(0, 2)))
                         for _ in range(int(rng.integers(0, 4)))]
        args['bad'] = how
        return (op, args)

    def forecast(op):
        return forecast_scen(op) if op.startswith('plan_') else batch_forecast(op)
    mix = [query, plan, scen] + [lambda op=op: forecast(op) for op in FORECASTS if op in kinds]

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
        elif op in FORECASTS:
            steps.append(forecast(op))
        elif op in ('explain_batch', 'explain_pod'):
            steps.append((op, {'which': float(rng.random())}))
        elif op == 'explain_macro':                                         # the sequence explanations need
            steps.append(('snapshot', {}))
            pods, now = d.pods(8, 64, four=False)
            steps.append(('solve_batch', {'pods': pods, 'now': now}))
            for _ in range(int(rng.integers(0, 3))):
                steps.append(mix[int(rng.integers(0, len(mix)))]())
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
        self.deployed = []            # (binding, pod) of every pod a batch placed on the records as they are
        self.snap_deployed = []       # the same list at the snapshot

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
        """The refusal (code, pod named) the model expects, or none; a third element of ``want_ref`` names the rule
        for the stats."""
        if got_ref is not None:
            self.stats['refusals'][got_ref[0]] = self.stats['refusals'].get(got_ref[0], 0) + 1
        if (got_ref is None) != (want_ref is None) or (want_ref is not None and
                                                       (got_ref[0], got_ref[1]) != tuple(want_ref[:2])):
            raise Mismatch(f'{where}: refusal {got_ref}, expected {want_ref}')
        if want_ref is not None and len(want_ref) > 2:
            self.stats['rules'][want_ref[2]] = self.stats['rules'].get(want_ref[2], 0) + 1

    def same(self, where, got, want, n_nodes=None):
        """Bindings equal byte for byte, none on a node past ``n_nodes`` (the loaded nodes and the call's added ones)."""
        n_nodes = len(self.recs) if n_nodes is None else n_nodes
        if got.tobytes() != want.tobytes():
            from tests import helpers
            raise Mismatch(f'{where}: {helpers.first_binding_diff(want, got)}')
        if len(got) and got['node'].max() >= n_nodes:
            raise Mismatch(f'{where}: a node outside the {n_nodes} loaded and added nodes (padding) was chosen')
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
        self.deployed, self.snap_deployed = [], []
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
        if kind in ('hardware', 'release'):                               # those pods are gone with the record
            gone = {int(i) for i in idx}
            self.deployed = [(b, p) for b, p in self.deployed if int(b['node']) not in gone]
        self.snap_fresh = False
        self.moved()

    def snapshot(self):
        self.s.snapshot()
        self.snap, self.snap_fresh = self.recs.copy(), True
        self.snap_deployed = list(self.deployed)
        self.moved()
        self.after_snap = True

    def restore(self):
        _, ref = self.call(self.s.restore)
        self.expect('restore', ref, None if self.snap is not None else (wire.ERR_STATE, None))
        if self.snap is not None:
            self.recs = self.snap.copy()
            self.deployed = list(self.snap_deployed)
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
        self.deployed += [(got[i].copy(), pods[i].copy()) for i in np.flatnonzero(got['status'] == wire.PLACED)]
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

    def plan_scenarios(self, scenarios, source, explain=False, what='plan_scenarios'):
        """Any scenario call: plain, edited, explained, grown (sixth element) and with rounds (seventh), each scenario
        against the oracle of its entry point, added nodes numbered call-wide."""
        from tests.test_defrag import oracle_defrag
        from tests.test_expand import oracle_grown
        from tests.test_forecast import _sc, oracle_rounds
        from tests.test_plan import oracle_plan
        from tests.test_plan_reasons import oracle_explained
        scs = [_sc(sc) for sc in scenarios]
        recs, want_ref = self.source(source)
        want_ref = scenario_call_refusal(scs, want_ref, self.n_classes())
        got, ref = self.call(lambda: self.s.plan_scenarios(scenarios, source=source, explain=explain))
        self.expect(f'{what} ({source})', ref, want_ref)
        if recs is None:
            return
        fgot, fref = None, None
        if self.check_fresh:
            f = self.fresh(recs)
            try:
                fgot, fref = self.call(lambda: f.plan_scenarios(scenarios, explain=explain))
            finally:
                f.close()
            self.expect(f'{what} on a fresh handle', fref, want_ref)
        if want_ref is not None:
            return
        rounds = any(sc[6] is not None for sc in scs)
        grown_call = any(sc[5] is not None for sc in scs)
        k = max_numa(self.recs)
        for sc in scs:
            for change in (sc[4], sc[5]):                                  # edits and additions count, held or not
                if change is not None and len(change[1]):
                    k = max(k, int(np.asarray(change[1])['n_numa'].max()))
        base, st = 0, self.stats
        for j, (ex, pods, now, lift, edits, adds, clocks) in enumerate(scs):
            res, where = got[j], f'{what} ({source}) scenario {j}'
            n_add = 0 if adds is None else len(adds[0])
            want_ref = pod_refusal(pods, now, k)
            self.expect(where, None if res[0] == 0 else tuple(res[:2]), want_ref)
            if fgot is not None and _result_bytes(fgot[j]) != _result_bytes(res):
                raise Mismatch(f'{where}: differs from a fresh handle')
            if want_ref is not None or not len(pods):
                base += n_add
                continue
            b, exl, wrows, wrnd = res[2], [int(i) for i in ex], None, None
            if rounds:
                want, wrnd, wrows, _ = oracle_rounds(recs, self.speed, pods, now, exl, lift, edits, adds, clocks, base,
                                                     BUSY, explain=explain)
            elif grown_call:
                want = oracle_grown(recs, self.speed, pods, now, exl, lift, edits, adds, base, BUSY, explain=explain)
                want, wrows = want if explain else (want, None)
            elif explain:
                want, wrows = oracle_explained(recs, self.speed, pods, now, exl, lift, edits, BUSY)
            elif lift is None and edits is None:
                want = oracle_plan(recs, self.speed, pods, now, exl, BUSY)[0]
            else:
                want = oracle_defrag(recs, self.speed, pods, now, exl, lift, edits, busy=BUSY)
            self.same(f'{where} against the oracle', b, want, len(recs) + base + n_add)
            if explain:
                self.same_rows(where, res[3], wrows, b, len(recs) + n_add)
            if rounds:
                self.same_rounds(where, res[-1], wrnd, b)
            placed = b['status'] == wire.PLACED
            st['on_added'] += int((placed & (b['node'] >= len(recs))).sum())
            base += n_add

    def plan_explained(self, scenarios, source):
        self.plan_scenarios(scenarios, source, explain=True, what='plan_explained')

    def plan_grown(self, scenarios, source):
        self.plan_scenarios(scenarios, source, explain=bool(len(scenarios) % 2), what='plan_grown')

    def plan_rounds(self, scenarios, source):
        self.plan_scenarios(scenarios, source, explain=bool(len(scenarios) % 2), what='plan_rounds')

    def same_rows(self, where, rows, want, b, n_nodes):
        """Reason rows equal the oracle's; every NO_CANDIDATE row counts each loaded and added node once."""
        if rows.tobytes() != want.tobytes():
            raise Mismatch(f'{where}: reason rows {np.flatnonzero((rows != want).any(1))} differ from the oracle')
        none = b['status'] == wire.NO_CANDIDATE
        if (rows[none].sum(1) != n_nodes).any():
            raise Mismatch(f'{where}: a NO_CANDIDATE row does not sum to {n_nodes} nodes')
        self.stats['rows'] += int(none.sum())

    def same_rounds(self, where, rnd, want, b):
        if rnd.tobytes() != np.asarray(want, dtype='<i4').tobytes():
            raise Mismatch(f'{where}: pod rounds {rnd} differ from the oracle\'s {want}')
        self.stats['later'] += int(((b['status'] == wire.PLACED) & (rnd >= 1)).sum())

    def n_classes(self):
        return max([i + 1 for i, s in enumerate(self.speed) if s != 0.0], default=0)

    def batch_rounds(self, pods, now, rounds, source, exclude, explain):
        self._batch_forecast('batch_rounds', pods, now, rounds, source, exclude, explain, None)

    def batch_releases(self, pods, now, rounds, source, exclude, explain, ends, extra, bad):
        """The releases are pods a batch of this session deployed on the source records (``ends``: fractions of that
        list, a round, a place in the round's gap and the pairings per NIC); the tracked nodes are theirs plus free-NIC
        nodes (``extra``) whose free NICs start at -1 or -2; ``pods_used`` from the source records' NIC bits.  ``bad``
        breaks one argument: a release out of its gap, a release on an untracked node, a flipped pods_used sign."""
        from tests.test_forecast_releases import release_of
        snap = source == 'snapshot' and self.snap is not None
        recs, dep = (self.snap, self.snap_deployed) if snap else (self.recs, self.deployed)
        fin = now[np.isfinite(now)]
        t0 = float(fin.max()) if len(fin) else -np.inf

        def gap(rnd):
            return (t0 if rnd == 1 else rounds[rnd - 2]), rounds[rnd - 1]
        rels, taken = [], set()
        for which, rnd, at, pairings in ends:
            i = int(which * len(dep))
            if not dep or i in taken:
                continue
            taken.add(i)
            b, pod = dep[i]
            lo, hi = gap(rnd)
            clock = hi if at == 1.0 or not np.isfinite(lo) else min(hi, lo + at * (hi - lo))
            rels.append(release_of(b, pod, int(b['node']), rnd, clock, pairings))
        rels = np.array(sorted(rels, key=lambda x: (int(x['round']), float(x['clock']))), dtype=wire.RELEASE_DTYPE)
        tracked = sorted({int(x['node']) for x in rels})
        # free-NIC nodes the pods take when nothing ends (where a negative counter cuts), else any with NICs
        from oracle import binding
        from tests.test_plan import excluded
        ok = np.isfinite(now)
        first = binding.solve(excluded(recs, [int(i) for i in exclude]), self.speed, pods[ok], now[ok],
                              min_busy_secs=BUSY)[0]
        free = sorted({int(v) for v in first['node'][first['n_claimed'] > 0]} - set(tracked)) or \
            [int(v) for v in np.flatnonzero(recs['n_nics'] > 0) if int(v) not in tracked]
        negs = {}
        for which, bits, neg in extra:
            if free:
                negs[free[int(which * len(free))]] = (bits, neg)
        tracked += sorted(negs)
        used = np.zeros((len(tracked), wire.MAX_NICS), dtype='<i2')
        for t, node in enumerate(tracked):
            inuse, bits, neg = int(recs['nic_inuse'][node]), *negs.get(node, (0, 0))
            for i in range(int(recs['n_nics'][node])):
                used[t, i] = 1 if inuse >> i & 1 else (neg if bits >> i & 1 else 0)
        if bad == 'gap' and len(rels):
            rels[0]['clock'] = gap(int(rels[0]['round']))[0] - 1.0
        elif bad == 'untracked' and len(rels):
            t = tracked.index(int(rels[0]['node']))
            tracked, used = tracked[:t] + tracked[t + 1:], np.delete(used, t, axis=0)
        elif bad == 'sign' and tracked:
            node = tracked[0]
            used[0, 0] = 0 if recs['n_nics'][node] and recs['nic_inuse'][node] & 1 else 1
        self._batch_forecast('batch_releases', pods, now, rounds, source, exclude, explain, (tracked, used, rels))

    def _batch_forecast(self, what, pods, now, rounds, source, exclude, explain, rel):
        """plan_batch_rounds (``rel`` None) or plan_batch_releases (``rel``: tracked, pods_used, releases) against the
        refusal model, a fresh handle and the oracle loop; a rounds forecast also against the scenario call of that
        one scenario on this handle."""
        from tests.test_forecast import oracle_rounds
        from tests.test_forecast_releases import oracle_releases
        recs, src_ref = self.source(source)
        ex = [int(i) for i in exclude]
        want_ref = batch_refusal(pods, now, rounds, rel, src_ref, recs, max_numa(self.recs, ex))

        def run(s, src):
            if rel is None:
                return s.plan_batch_rounds(pods, now, rounds, source=src, exclude=ex, explain=explain)
            return s.plan_batch_releases(pods, now, rounds, *rel, source=src, exclude=ex, explain=explain)
        got, ref = self.call(lambda: run(self.s, source))
        self.expect(f'{what} ({source})', ref, want_ref)
        if recs is None:
            return
        if self.check_fresh:
            f = self.fresh(recs)
            try:
                fgot, fref = self.call(lambda: run(f, 'mirror'))
            finally:
                f.close()
            self.expect(f'{what} on a fresh handle', fref, want_ref)
            if want_ref is None and _result_bytes(fgot) != _result_bytes(got):
                raise Mismatch(f'{what} ({source}): differs from a fresh handle')
        if want_ref is not None:
            return
        if rel is None:
            want, wrnd, wrows, _ = oracle_rounds(recs, self.speed, pods, now, ex, rounds=rounds, busy=BUSY,
                                                 explain=explain)
        else:
            want, wrnd, wrows, cuts = oracle_releases(recs, self.speed, pods, now, rounds, *rel, exclude=ex, busy=BUSY,
                                                      explain=explain)
            self.stats['cuts'] += sum(cuts)
        b, rnd = got[:2]
        self.same(f'{what} ({source}) against the oracle', b, want)
        self.same_rounds(f'{what} ({source})', rnd, wrnd, b)
        if explain:
            self.same_rows(f'{what} ({source})', got[2], wrows, b, len(recs))
        if rel is None:                        # the scenario call of this one scenario, on this handle
            sres = self.s.plan_scenarios([(ex, pods, now, None, None, None, rounds)], source=source, explain=explain)[0]
            if sres[0] == 0:
                mine = (sres[2], sres[-1]) + ((sres[3],) if explain else ())
                if _result_bytes(mine) != _result_bytes(got):
                    raise Mismatch(f'{what} ({source}): differs from the scenario call')
            elif sres[0] != wire.ERR_UNSUPPORTED or not ex:
                raise Mismatch(f'{what} ({source}): the scenario call refused with {sres[:2]}')

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
    """``rules``: refusals by the model's rule; ``rows``: NO_CANDIDATE reason rows compared; ``later``: pods placed at a
    round >= 1; ``on_added``: pods placed on added nodes; ``cuts``: the oracle loop's cuts in release forecasts."""
    return {'ops': {}, 'refusals': {}, 'status': {}, 'bindings': 0, 'calls': 0, 'explained': 0, 'rules': {}, 'rows': 0,
            'later': 0, 'on_added': 0, 'cuts': 0}


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
                                    'source': 'mirror'}),
                ('plan_explained', {'scenarios': [([5], pods, now + t), ([], pods, now + t, 2, None)],
                                    'source': 'mirror'}),
                ('plan_grown', {'scenarios': [([], pods, now + t, None, None, ([0], recs[[1]]))], 'source': 'mirror'}),
                ('plan_rounds', {'scenarios': [([6], pods, now + t, None, None, None, [5100.0 + t])],
                                 'source': 'mirror'}),
                ('batch_rounds', {'pods': pods, 'now': now + t, 'rounds': [5100.0 + t], 'source': 'mirror',
                                  'exclude': np.array([5]), 'explain': False}),
                ('batch_releases', {'pods': pods, 'now': now + t, 'rounds': [5100.0 + t], 'source': 'mirror',
                                    'exclude': np.array([6]), 'explain': True, 'ends': [(0.5, 1, 0.5, 2)],
                                    'extra': [], 'bad': None})]

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
    t = float(np.max(now))
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
            ('plan_explained', {'scenarios': [([1], pods, now), ([0], pods, now, 3, ([2], recs[[1]]))],
                                'source': 'snapshot'}),
            ('plan_grown', {'scenarios': [([], pods, now, None, None, ([0, len(recs)], recs[[1, 2]]))],
                            'source': 'mirror'}),
            ('plan_rounds', {'scenarios': [([1], pods, now, None, None, ([1], recs[[0]]), [t + 10.0, t + 40.0]),
                                           ([], pods[:3], now[:3], None, None, None, None)], 'source': 'snapshot'}),
            ('batch_rounds', {'pods': pods, 'now': now, 'rounds': [t + 30.0], 'source': 'snapshot', 'exclude': [0],
                              'explain': True}),
            ('batch_releases', {'pods': pods, 'now': now, 'rounds': [t + 30.0, t + 60.0], 'source': 'mirror',
                                'exclude': [], 'explain': True, 'ends': [(0.1, 1, 0.5, 2), (0.6, 2, 1.0, 1)],
                                'extra': [(0.5, 0xFF, -1)], 'bad': None}),
            ('explain_batch', {'which': 0.0}), ('explain_pod', {'which': 0.0}), ('explain_pod', {'which': 0.5}),
            ('explain_pod', {'which': 0.9}), ('restore', {}), ('explain_batch', {'which': 0.0})]})
        assert r.stats['explained'] == 4 and r.stats['refusals'] == {wire.ERR_STATE: 1}, r.stats
    finally:
        r.close()
