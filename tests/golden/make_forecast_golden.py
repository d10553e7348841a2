"""Freeze the UNMODIFIED reference's answer to "which pending pods get in at a later scan, and which never do?" into
tests/golden/live/forecast.json.gz.

The sessions are ``defrag_sessions()`` (make_defrag_golden.py) and ``queue_script`` sessions, in which more one-GPU pods
arrive at once than there are GPU nodes (``min_busy_secs`` 30): a scan places at most one GPU pod per node, so the rest
wait for later scans.  Each session is played to its end state in the reference; then, per case, the candidate nodes
of the case (none, or a subset of make_expand_golden.py's ``expand_cases``) are inserted into the reference scheduler's
node dict (``_AddNodes``), optionally the clock is moved by a fraction of a second, and ``SCANS`` pending scans run
with the clock stepped by ``period`` between them (the steps ``idle``, ``clock``, ``idle``, ...).  Periods: 30.0 (equal to
``MIN_BUSY_SECS``), 31.0 and 10.0, and 30.0 from a start clock moved by 0.1 s (the busy test is ``now - busy_time <
MIN_BUSY_SECS`` in fp64: from a fractional clock, ``t + 30.0 - t`` need not be 30.0).
The file records, per case, the pods the scans attempt (in the first scan's order, read from this repository's
scheduler replaying the session with the oracle stand-in), for each the scan that bound it and its node, or None, and
the reference's own reasons at its last scan for every pod no scan placed (make_plan_reasons_golden.py's
``_Attempts``).  A pod bound by some scan was attempted once by every scan up to that one, so its scan is its number of
attempts minus one.  Cases with a failing Kubernetes write, or in which the reference itself raises, are left out, as
in make_expand_golden.py.  ``NHDScheduler.ForecastPending`` answers all of one session's cases of one clock variant in
one call.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_forecast_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402
from tests.golden.make_defrag_golden import _WriteFailures, defrag_sessions, pending_keys   # noqa: E402
from tests.golden.make_expand_golden import _AddNodes, expand_cases, grown_names   # noqa: E402
from tests.golden.make_plan_golden import mirror_session   # noqa: E402

SCANS = 4
VARIANTS = ((30.0, 0.0), (31.0, 0.0), (10.0, 0.0), (30.0, 0.1))       # (period, start clock moved by)
LABELS = ('shape0-end', 'shape0-front', 'copies2', 'gpuless-front')  # the expand cases kept, besides no addition


def queue_script(seed):
    """More pending one-GPU pods than GPU nodes: two or three GPU nodes (maybe a CPU-only node first), then 6 to 11 pods
    arriving together and one scan, which places one per GPU node; the clock then moves 5 s, inside the busy window."""
    from tests import scenarios as S
    rng = np.random.default_rng(seed)
    per_numa = int(rng.choice([1, 2]))
    nodes = []
    if rng.random() < 0.5:
        nodes.append(S.make_node('cpu0', 2, 32, False, 1, (), [('eth0', 100000, 0, 0x10)], hp_alloc=64, hp_free=64))
    for i in range(int(rng.integers(2, 4))):
        gpus = [(d, d // per_numa, 0x10 * (d // per_numa + 1)) for d in range(2 * per_numa)]
        nics = [(f'eth{k}', 100000, k, 0x10 * (k + 1)) for k in range(2)]
        nodes.append(S.make_node(f'n{i}', 2, 32, bool(rng.random() < 0.5), 1, gpus, nics, hp_alloc=64, hp_free=64))
    steps = []
    for k in range(int(rng.integers(6, 12))):
        n_gpus = 2 if rng.random() < 0.15 else 1
        spec = S.make_pod([S.make_group([], int(rng.integers(1, 3)), [int(rng.integers(0, 2))] * n_gpus, 0)],
                          int(rng.integers(0, 2)), False, 'NUMA', int(rng.choice([0, 2])))
        steps.append({'op': 'add_pod', 'ns': 'ns0', 'name': f'q{k}', 'uid': f'uq{k}', 'fail': [], 'pod': spec})
    steps += [{'op': 'idle'}, {'op': 'clock', 'dt': 5.0}]
    return {'nodes': nodes, 'min_busy_secs': 30.0, 'clock0': 1000.0, 'init': [], 'steps': steps, 'codec': 'json'}


def forecast_sessions():
    """``defrag_sessions()`` and the ``queue_script`` sessions: ``(name, script)``."""
    return defrag_sessions() + [(f'json{seed}_queue', queue_script(seed)) for seed in range(51, 59)]


def scan_steps(nodes, period, frac):
    """The steps after a session: the start clock moved by ``frac``, the candidate nodes, ``SCANS`` scans ``period``
    apart.  (The clock step comes first: the reference driver plays clock steps from its watch queue only, and the
    added nodes right before the scan that sees them.)"""
    steps = ([{'op': 'clock', 'dt': frac}] if frac else []) + ([{'op': 'add_nodes', 'nodes': nodes}] if nodes else [])
    for k in range(SCANS):
        steps += ([{'op': 'clock', 'dt': period}] if k else []) + [{'op': 'idle'}]
    return steps


def forecast_session(item):
    from tests import helpers
    from tests import sched_harness as H
    from tests.golden.make_plan_reasons_golden import _Attempts, _last, _run
    name, script = item
    sched, k8s, _ = mirror_session(script, helpers.OracleSolver)
    try:
        names = list(sched.nodes)
        pending = pending_keys(sched)
        requested = sorted({g for ns, pod in pending for g in k8s.GetPodNodeGroups(pod, ns)} - {'default'})
    finally:
        sched.close()
    cases = [{'label': 'none', 'nodes': []}] + [c for c in expand_cases(script, names, requested) if c['label'] in LABELS]
    out, left_out, crashed, later, unplaced = [], 0, 0, 0, 0
    with _Attempts() as att, _WriteFailures() as failures, _AddNodes():
        start = len(_run(att, script))
        prefix_failures = failures.n
        for case in cases:
            for period, frac in VARIANTS:
                failures.n = 0
                att.log = []
                try:
                    doc = H.run_reference(dict(script, steps=script['steps'] + scan_steps(case['nodes'], period, frac)))
                except TypeError:               # the reference's own crash in SetPhysicalIdsFromMapping (Node.py:833)
                    crashed += 1
                    continue
                log = list(att.log)
                if failures.n != prefix_failures:
                    left_out += 1
                    continue
                assert list(doc['nodes']) == grown_names(names, case['nodes']), (name, case['label'])
                where = {p: nd for nd, st in doc['nodes'].items() for p in st['pods']}
                tries = {}
                for ns, pod, _ in log[start:]:
                    tries[(ns, pod)] = tries.get((ns, pod), 0) + 1
                placed = [None if where.get(f'{ns}/{pod}') is None else [tries[(ns, pod)] - 1, where[f'{ns}/{pod}']]
                          for ns, pod in pending]
                later += any(p is not None and p[0] >= 1 for p in placed)
                unplaced += any(p is None for p in placed)
                never = {k for k, p in zip(pending, placed) if p is None}
                out.append(dict(case, period=period, frac=frac, placed=placed, reasons=_last(log, start, never)))
    print(name, len(pending), 'pending,', len(out), 'cases kept,', left_out, 'left out,', crashed, 'crashed,', later,
          'placing at a later scan,', unplaced, 'leaving a pod unplaced', flush=True)
    return {'name': name, 'pending': [list(p) for p in pending], 'cases': out}, len(out), later, unplaced


def main():
    import multiprocessing
    with multiprocessing.get_context('fork').Pool(os.cpu_count() or 1) as pool:
        res = pool.map(forecast_session, forecast_sessions(), chunksize=1)
    cases, later, unplaced = (sum(r[i] for r in res) for i in (1, 2, 3))
    print(cases, 'cases,', later, 'placing a pod at scan >= 1,', unplaced, 'leaving a pod unplaced')
    assert later > 0 and unplaced > 0, (later, unplaced)
    live._save('forecast', {'sessions': [r[0] for r in res]})


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    main()
