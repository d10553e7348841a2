"""Why a pod found no node (``nhd_explain_batch`` / ``nhd_explain_pod``, ``Solver.explain_batch`` / ``explain_pod``).

For a NO_CANDIDATE pod every node gets the first reference stage that drops it (NHD_WHY_*, include/nhd_b200.h), at
the state that pod saw.  The chain of evidence:
  * the explanation oracle (tests/explain_oracle.c: the oracle's own stage restatements, run stage by stage) equals
    the reference's own drop decisions, frozen from its log in tests/golden/live/explain.json.gz (no GPU);
  * the CUDA kernels equal the oracle node by node, in every sweep mode, and the counts equal the per-node codes
    (``-m gpu``; on a machine without a GPU test_emulated_device.py runs them on the CPU emulation)."""
import ctypes
import os

import numpy as np
import pytest

from nhd_b200 import wire
from tests import explain_oracle, helpers, ref_compare
from tests.explain_scenarios import explain_scenarios
from tests.golden import make_live_golden

EMULATED = os.environ.get('NHD_B200_ALLOW_EMULATED') == '1'
MODES = (dict(), dict(single_warp=True), dict(cpu_warps=1), dict(cpu_warps=2), dict(sweep_debug=1),
         dict(sweep_debug=5))


def _streams():
    """(name, scenarios) of the frozen comparison: the four random oracle streams and the explanation stream."""
    out = [(f, make_live_golden.oracle_scenarios(f)) for f in ('mixed', 'wild', 'vf', 'big')]
    out.append(('explain', explain_scenarios()))
    return out


def _packed(scn):
    recs, pods, now, layout = ref_compare.pack_scenario(scn)
    return recs, pods, now, layout.speed_table(), float(scn.get('min_busy_secs', 30.0))


# ---------------------------------------------------------------------------------------------- CPU: the oracle
def test_oracle_explanations_equal_the_reference_drop_decisions():
    golden = make_live_golden.load('explain')
    seen = np.zeros(wire.WHY_COUNT, dtype=np.int64)
    n_pods = 0
    for name, scns in _streams():
        assert len(golden[name]) == len(scns), name
        for k, (scn, want) in enumerate(zip(scns, golden[name])):
            recs, pods, now, speed, busy = _packed(scn)
            out, got = explain_oracle.batch(recs, speed, pods, now, min_busy_secs=busy)
            assert sorted(got) == sorted(int(i) for i in want), (name, k)
            for i, codes in want.items():
                r = got[int(i)]
                assert ''.join(map(str, r)) == codes, (name, k, i, ''.join(map(str, r)), codes)
                seen += np.bincount(r, minlength=wire.WHY_COUNT + 1)[:wire.WHY_COUNT]
                n_pods += 1
    assert n_pods > 100 and (seen >= 5).all(), seen


def test_explanation_stream_reaches_every_reason():
    seen = np.zeros(wire.WHY_COUNT + 1, dtype=np.int64)
    for scn in explain_scenarios():
        recs, pods, now, speed, busy = _packed(scn)
        _, got = explain_oracle.batch(recs, speed, pods, now, min_busy_secs=busy)
        for r in got.values():
            seen += np.bincount(r, minlength=wire.WHY_COUNT + 1)
    assert (seen[:wire.WHY_COUNT] >= 5).all() and seen[wire.WHY_COUNT] == 0, seen


# ---------------------------------------------------------------------------------------------- GPU
def _solver(speed, busy, **mode):
    from nhd_b200.solver import Solver
    return Solver(speed, min_busy_secs=busy, **mode)


def _run(s, recs, pods, now):
    s.load_nodes(recs)
    s.snapshot()
    return s.solve_batch(pods, now)


def _gpu_cases():
    cases = [('explain', scn) for scn in explain_scenarios()]
    per = 2 if EMULATED else 30
    for f in ('mixed', 'wild', 'vf', 'big'):
        cases += [(f, scn) for scn in make_live_golden.oracle_scenarios(f)[:per]]
    return cases


@pytest.mark.gpu
def test_explain_pod_equals_the_oracle_node_by_node_in_every_sweep_mode():
    n_failed = 0
    for name, scn in _gpu_cases():
        recs, pods, now, speed, busy = _packed(scn)
        ob, want = explain_oracle.batch(recs, speed, pods, now, min_busy_secs=busy)
        for mode in (MODES if name == 'explain' or not EMULATED else MODES[:2]):
            s = _solver(speed, busy, **mode)
            try:
                b = _run(s, recs, pods, now)
                assert helpers.binding_bytes_equal(ob, b), (name, mode, helpers.first_binding_diff(ob, b))
                for i in range(len(pods)):
                    got = s.explain_pod(i)
                    if i in want:
                        assert np.array_equal(got, want[i]), (name, mode, i, got, want[i])
                    else:
                        assert (got == wire.WHY_NONE).all(), (name, mode, i)
                counts = s.explain_batch()
                assert np.array_equal(counts, explain_oracle.counts(want, len(pods))), (name, mode)
            finally:
                s.close()
        n_failed += len(want)
    assert n_failed > 50


@pytest.mark.gpu
def test_counts_are_the_histogram_of_the_node_codes():
    for scn in explain_scenarios()[:2] + make_live_golden.oracle_scenarios('big')[:2]:
        recs, pods, now, speed, busy = _packed(scn)
        s = _solver(speed, busy)
        try:
            b = _run(s, recs, pods, now)
            counts = s.explain_batch()
            assert counts.shape == (len(pods), wire.WHY_COUNT) and counts.dtype == np.uint32
            for i in range(len(pods)):
                codes = s.explain_pod(i)
                if b[i]['status'] == wire.NO_CANDIDATE:
                    assert codes.max() < wire.WHY_COUNT
                    assert np.array_equal(counts[i], np.bincount(codes, minlength=wire.WHY_COUNT))
                    assert int(counts[i].sum()) == len(recs)
                else:
                    assert not counts[i].any() and (codes == wire.WHY_NONE).all()
            assert (b['status'] == wire.NO_CANDIDATE).any()
        finally:
            s.close()


def _filter_words(s):
    L = s._L
    nt, wpt = ctypes.c_int32(), ctypes.c_int32()
    assert L.nhd_read_filter(s._h, ctypes.byref(nt), ctypes.byref(wpt), None, 0, None, 0) == 0
    words = np.zeros((nt.value + 2) * wpt.value, dtype='<u8')
    assert L.nhd_read_filter(s._h, ctypes.byref(nt), ctypes.byref(wpt), words.ctypes.data, len(words), None, 0) == 0
    return words


@pytest.mark.gpu
def test_explaining_changes_nothing():
    scn = explain_scenarios()[1]
    recs, pods, now, speed, busy = _packed(scn)
    s = _solver(speed, busy)
    try:
        b = _run(s, recs, pods, now)
        before = (s.read_nodes(), s.fetch_bindings(), _filter_words(s))
        first = s.explain_batch()
        s.explain_pod(int(np.flatnonzero(b['status'] == wire.NO_CANDIDATE)[0]))
        after = (s.read_nodes(), s.fetch_bindings(), _filter_words(s))
        assert before[0].tobytes() == after[0].tobytes()
        assert before[1].tobytes() == after[1].tobytes() and helpers.binding_bytes_equal(b, after[1])
        assert np.array_equal(before[2], after[2])
        assert np.array_equal(first, s.explain_batch())            # and asking again gives the same answer
    finally:
        s.close()


@pytest.mark.gpu
def test_explanations_need_the_snapshot_the_batch_started_from():
    from nhd_b200.solver import SolverError
    scn = explain_scenarios()[0]
    recs, pods, now, speed, busy = _packed(scn)

    def refused(s):
        for call in (s.explain_batch, lambda: s.explain_pod(0)):
            with pytest.raises(SolverError) as e:
                call()
            assert e.value.code == wire.ERR_STATE

    s = _solver(speed, busy)
    try:
        s.load_nodes(recs)
        s.solve_batch(pods, now)
        refused(s)                                                  # no snapshot
        s.snapshot()
        s.update_nodes([0], recs[:1])
        s.solve_batch(pods, now)
        refused(s)                                                  # update between snapshot and stage
        s.snapshot()
        s.solve_batch(pods, now)
        s.explain_batch()                                           # the valid sequence
        s.update_nodes([0], recs[:1])
        refused(s)                                                  # update after the solve
        s.snapshot()
        s.solve_batch(pods, now)
        s.restore()
        refused(s)                                                  # restore after the solve
        s.snapshot()
        s.solve_batch(pods, now)
        s.stage_batch(pods, now)
        refused(s)                                                  # a second stage
        s.solve_staged()
        s.sync()
        refused(s)                                                  # ... and its solve: not on the snapshot
        s.snapshot()
        s.stage_batch(pods, now)
        s.filter_bitmaps()
        refused(s)                                                  # filter-only run: no bindings
    finally:
        s.close()


class _RecordingSolver:
    """The CUDA Solver, with every explanation checked against the oracle at the batch's own snapshot."""
    checked = []

    def __init__(self, speed_table, nic_bw_avail_percent=0.9, min_busy_secs=30.0, device=0):
        from nhd_b200.solver import Solver
        self._s = Solver(speed_table, nic_bw_avail_percent=nic_bw_avail_percent, min_busy_secs=min_busy_secs,
                         device=device)
        self._speed, self._busy, self._snap, self._last = speed_table, min_busy_secs, None, None

    def __getattr__(self, name):
        return getattr(self._s, name)

    def snapshot(self):
        self._s.snapshot()
        self._snap = self._s.read_nodes()

    def solve_batch(self, pods, now):
        self._last = (self._snap, np.array(pods), np.array(now))
        self._snap = None
        return self._s.solve_batch(pods, now)

    def explain_batch(self):
        got = self._s.explain_batch()
        snap, pods, now = self._last
        _, want = explain_oracle.batch(snap, self._speed, pods, now, min_busy_secs=self._busy)
        assert np.array_equal(got, explain_oracle.counts(want, len(pods)))
        _RecordingSolver.checked.append(len(want))
        return got


@pytest.mark.gpu
def test_scheduler_keeps_the_reasons_of_unschedulable_pods(monkeypatch):
    from nhd_b200 import NHDScheduler as S
    from tests import sched_harness as H
    import itertools
    sessions = itertools.count()                # not id(): a closed scheduler's id can be reused by the next one

    def sid_of(sched):
        return sched.__dict__.setdefault('_explain_test_session', next(sessions))
    stored = []
    real = S.NHDScheduler._explain

    def spy(self, e, counts):
        stored.append((sid_of(self), (e.key[0], e.key[1]), {n: int(c) for n, c in zip(wire.WHY_NAMES, counts) if int(c)}))
        real(self, e, counts)
    monkeypatch.setattr(S.NHDScheduler, '_explain', spy)
    finals = []
    real_close = S.NHDScheduler.close

    def close(self):
        finals.append((sid_of(self), dict(self.unschedulable_reasons), dict(self.pod_state), self.cluster.rewinds))
        real_close(self)
    monkeypatch.setattr(S.NHDScheduler, 'close', close)
    _RecordingSolver.checked = []
    # seeds 10 and 17 (wild) include failed assignments (a rewind), every script includes failed Kubernetes writes
    scripts = [H.random_script(10, 'wild'), H.random_script(17, 'wild'), H.random_script(101, 'mixed')]
    for script in scripts[:2 if EMULATED else 3]:
        H.run_mirror(script, solver_factory=_RecordingSolver)
    assert stored and sum(_RecordingSolver.checked) > 0
    assert any(rw for _, _, _, rw in finals), 'no rewind after a failed assignment'
    for sid, reasons, pod_state, _ in finals:
        for key, r in reasons.items():
            assert pod_state.get(key, {}).get('state') != S.PodStatus.POD_STATUS_SCHEDULED, key
            assert r == [v for i, k, v in stored if i == sid and k == key][-1], key
            assert sum(r.values()) > 0


@pytest.mark.gpu
@pytest.mark.skipif(EMULATED, reason='65 536 nodes on the CPU emulation take too long for the suite')
def test_full_size_with_an_oversized_tail():
    import workload
    from tests.explain_scenarios import oversized_tail
    recs, speed, pods, now = workload.make_workload(4)
    tail = oversized_tail(pods, 256)                                # pods no node can take, after the 4 096
    pods, now = np.concatenate([pods, tail]), np.concatenate([now, np.full(len(tail), now[-1])])
    s = _solver(speed, 30.0)
    try:
        b = _run(s, recs, pods, now)
        failed = np.flatnonzero(b['status'] == wire.NO_CANDIDATE)
        assert len(failed) >= 64
        counts = s.explain_batch()
        assert (counts[failed].sum(axis=1) == len(recs)).all()
        assert not np.delete(counts, failed, axis=0).any()
        sample = set(int(i) for i in failed[np.linspace(0, len(failed) - 1, 32).astype(int)])
        ob, want = explain_oracle.batch(recs, speed, pods, now, which=sample, threads=os.cpu_count() or 1)
        assert helpers.binding_bytes_equal(ob, b)
        for i in sorted(sample):
            got = s.explain_pod(i)
            assert np.array_equal(got, want[i]), i
            assert np.array_equal(counts[i], np.bincount(got, minlength=wire.WHY_COUNT))
    finally:
        s.close()
