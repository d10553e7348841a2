"""The forecasts on one long-lived handle: explained, grown and round scenario calls, ``plan_batch_rounds`` and
``plan_batch_releases`` among loads, updates, snapshots, restores, batches and the other what-if calls.

These calls keep the most per-handle state of all (DESIGN §8.11 - §8.15): the round buffers that only grow, the pod
arrays ``plan_batch`` swaps with the round buffer every round, the release area whose offsets move with the node count,
the index buffer shared by the tracked nodes and the exclusions, the scenario scratch in two layouts, the reason
buffers shared with the batch explanations.  The runner of tests/test_handle_session.py compares every call with the
oracle (``oracle_scenario`` and ``oracle_releases`` of tests/plan_oracle.py), with a fresh handle and with its refusal
model; the releases are pods the session itself deployed.  The named sessions each aim at one way the carried state
could go wrong; the random ones assert that they reached what they are meant to test."""
import numpy as np
import pytest

from nhd_b200 import wire
from tests import scenarios
from tests.test_handle_session import (BASIC, EMU_SIZES, EMULATED, FORECASTS, MODES, SIZES, Draw, _four_numa_cluster,
                                       _mode_params, _pods, _restricted_growth, class_records, make_session, new_layout,
                                       new_stats, pack, run_session)


def _rounds(t, k, period=30.0):
    return [t + period * (j + 1) for j in range(k)]


def _bf(op, pods, now, rounds, source='mirror', exclude=(), explain=False, **rel):
    """A batch forecast step; ``rel`` (plan_batch_releases): ends, extra, bad."""
    args = {'pods': pods, 'now': now, 'rounds': rounds, 'source': source,
            'exclude': np.asarray(exclude, dtype=np.int32), 'explain': explain}
    if op == 'batch_releases':
        args.update({'ends': [], 'extra': [], 'bad': None}, **rel)
    return (op, args)


def _ends(k, r, pairings=2):
    """k releases spread over the deployed pods and over r rounds, mid-gap, two pairings a NIC (counters to -1)."""
    return [((j + 0.5) / k, 1 + j % r, 0.5, pairings) for j in range(k)]


# ---------------------------------------------------------------------------------------------- random sessions
N_SESSIONS, N_STEPS = (20, 24) if EMULATED else (48, 30)


@pytest.mark.gpu
def test_random_forecast_sessions_equal_a_fresh_handle_and_the_oracle():
    stats = new_stats()
    for seed in range(N_SESSIONS):
        run_session(make_session(seed, N_STEPS, EMU_SIZES if EMULATED else SIZES, BASIC + FORECASTS),
                    MODES[seed % len(MODES)], stats)
    print('session stats:', stats)
    assert set(stats['ops']) >= set(BASIC) - {'explain_macro'} | set(FORECASTS), stats['ops']
    assert stats['later'] > 0 and stats['on_added'] > 0 and stats['cuts'] > 0 and stats['rows'] > 0, stats
    assert set(stats['rules']) >= {'round clock', 'speed class', 'source', 'pod'}, stats['rules']
    assert set(stats['rules']) & {'release gap', 'untracked', 'pods_used sign'}, stats['rules']
    assert stats['bindings'] > (5000 if EMULATED else 20000), stats


# ---------------------------------------------------------------------------------------------- named sessions
@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_the_round_workspace_shrinks_after_a_large_forecast(mode):
    """A large rounds forecast (mixed node-group lists: the pod-groups area exists; 8 rounds), then on the same handle
    a one-pod forecast, a query, an explained plan, a rounds scenario call (slots from slot_start), a batch and its
    explanations; then all of it again with one node-group list for every pod."""
    lay = new_layout()
    d = Draw(np.random.default_rng(41), lay)
    n, big = (300, 96) if EMULATED else (4100, 600)
    recs = d.nodes(n)
    steps = [('load_nodes', {'recs': recs})]
    for one_list in (False, True):
        pods = d.pool[d.pool['n_groups'] < 4][d.rng.integers(0, int((d.pool['n_groups'] < 4).sum()), big)].copy()
        if one_list:
            pods['group_mask'] = pods[0]['group_mask']
        else:
            assert len(np.unique(pods['group_mask'])) > 1
        now = np.full(big, d.t)
        small, snow = d.pods(6, 6, four=False)
        t = float(max(now.max(), snow.max()))
        steps += [_bf('batch_rounds', pods, now, _rounds(t, 8, 10.0), exclude=np.arange(0, n, 97)),
                  _bf('batch_rounds', small[:1], snow[:1], _rounds(t, 2), explain=True),
                  ('query_batch', {'pods': small, 'now': snow, 'source': 'mirror'}),
                  ('plan_batch', {'pods': small, 'now': snow, 'source': 'mirror', 'exclude': np.array([1, 2]),
                                  'explain': True}),
                  ('plan_rounds', {'scenarios': [([0], small, snow, None, None, None, _rounds(t, 3)),
                                                 ([], small[:2], snow[:2], None, None, None, None),
                                                 ([3], small[2:], snow[2:], 1, None, None, _rounds(t, 1))],
                                   'source': 'mirror'}),
                  ('snapshot', {}), ('solve_batch', {'pods': pods[:64], 'now': now[:64]}),
                  ('explain_batch', {'which': 0.0}), ('explain_pod', {'which': 0.3})]
        d.t = t + 400.0
    stats = run_session({'seed': 'round-workspace', 'steps': steps}, mode)
    assert stats['ops']['batch_rounds'] == 4, stats


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_releases_next_to_exclusions_and_a_smaller_cluster(mode):
    """Release forecasts with few tracked nodes and many exclusions, many tracked nodes and few exclusions, then after
    a load of a smaller cluster: the index buffer holds the tracked nodes and then the exclusions, and the release
    area's offsets move with the node count."""
    lay = new_layout()
    d = Draw(np.random.default_rng(43), lay)
    n, m = (300, 257) if EMULATED else (2049, 700)
    pods, now = d.pods(64, 64, four=False)
    late, lnow = d.pods(24, 24, four=False)
    t = float(lnow.max())
    steps = [('load_nodes', {'recs': d.nodes(n)}), ('solve_batch', {'pods': pods, 'now': now}),
             _bf('batch_releases', late, lnow, _rounds(t, 3), exclude=np.arange(0, n, 3), explain=True,
                 ends=_ends(2, 3), extra=[(0.5, 0xFFFFFFFF, -1)]),
             _bf('batch_releases', late, lnow, _rounds(t, 4, 10.0), exclude=[7],
                 ends=_ends(30, 4), extra=[(j / 6, 0x55555555, -2) for j in range(6)]),
             ('snapshot', {}), ('solve_batch', {'pods': late, 'now': lnow}),
             _bf('batch_releases', late, lnow + 100.0, _rounds(t + 100.0, 2), source='snapshot', explain=True,
                 ends=_ends(8, 2, 1), extra=[(0.2, 0xF, -1)]),
             ('load_nodes', {'recs': d.nodes(m)}), ('solve_batch', {'pods': pods, 'now': now + 200.0}),
             _bf('batch_releases', late, lnow + 200.0, _rounds(t + 200.0, 3), exclude=np.arange(0, m, 5),
                 explain=True, ends=_ends(12, 3), extra=[(0.9, 0xFFFF, -1)]),
             _bf('batch_releases', late, lnow + 200.0, _rounds(t + 200.0, 3), ends=_ends(4, 3), bad='sign'),
             _bf('batch_releases', late, lnow + 200.0, _rounds(t + 200.0, 3), ends=_ends(4, 3), bad='untracked'),
             _bf('batch_releases', late, lnow + 200.0, _rounds(t + 200.0, 3), ends=_ends(4, 3), bad='gap')]
    stats = run_session({'seed': 'releases-exclusions', 'steps': steps}, mode)
    assert stats['ops']['batch_releases'] == 7 and stats['cuts'] > 0, stats
    assert {'pods_used sign', 'untracked', 'release gap'} <= set(stats['rules']), stats['rules']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_growth_after_the_class_and_signature_tables_ran_out(mode):
    """More than 4 096 static descriptions through loads and 128 signature ids through two loads, then grown and
    explained scenarios whose added and edited records carry descriptions and signatures the handle has no slot for,
    next to untouched nodes without a class."""
    lay = new_layout()
    pats = list(_restricted_growth(8))
    n = 300 if EMULATED else 2049
    a, b = class_records(lay, pats, False), class_records(lay, pats, True)
    both = np.concatenate([a, b])
    steps = [('load_nodes', {'recs': both[k:k + n]}) for k in range(0, len(both) - n + 1, n)][:2 if EMULATED else None]
    sigs = scenarios.signature_list(300)
    first = pack(lay, scenarios.signature_nodes('s', [(sigs[2 * i], sigs[2 * i + 1]) for i in range(70)]))
    second = pack(lay, scenarios.signature_nodes('t', [(sigs[140 + 2 * i], sigs[141 + 2 * i]) for i in range(70)]))
    fresh = pack(lay, scenarios.signature_nodes('u', [(sigs[280 + i], sigs[299 - i]) for i in range(4)]))
    recs = np.concatenate([b[-n // 2:], second])
    steps += [('load_nodes', {'recs': first}), ('load_nodes', {'recs': recs})]
    pods = _pods(lay, scenarios.signature_pods() * 2)
    now = np.full(len(pods), 2000.0)
    new = np.concatenate([a[:3], fresh[:2]])                               # descriptions and signatures not seen yet
    scens = [([1], pods, now, None, ([2, 5], new[:2]), (np.array([0, 9, len(recs)], np.int32), new[2:])),
             ([], pods[:6], now[:6], 3, ([len(recs) - 1], fresh[2:3]), None),
             ([], pods, now + 1.0, None, None, (np.array([len(recs)], np.int32), fresh[3:4]))]
    steps += [('plan_grown', {'scenarios': scens, 'source': 'mirror'}),
              ('plan_explained', {'scenarios': [sc[:5] for sc in scens], 'source': 'mirror'}),
              ('plan_rounds', {'scenarios': [sc + (_rounds(2001.0, 2),) for sc in scens] + [scens[0][:6] + (None,)],
                               'source': 'mirror'}),
              ('solve_batch', {'pods': pods, 'now': now})]
    stats = run_session({'seed': 'tables-ran-out', 'steps': steps}, mode)
    assert stats['on_added'] > 0 and stats['status'].get(wire.PLACED, 0) > 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_an_added_four_numa_node_refuses_its_own_call_only(mode):
    """An added 4-NUMA record refuses the 4-group pods of its own call (the scenario with it and the one without);
    the forecasts, batch and scenario calls after it, without it, accept them."""
    lay = new_layout()
    recs = _four_numa_cluster(lay)
    d = Draw(np.random.default_rng(47), lay)
    pods, now = d.pods(8, 8, four=False)
    four = d.pool[d.pool['n_groups'] == 4][:1]
    pods = np.concatenate([pods[:2], four, pods[2:]])
    now = np.full(len(pods), 5000.0)
    big = recs[[5]].copy()                                                # the 4-NUMA record, schedulable
    big['flags'] = (big['flags'] | wire.NODE_ACTIVE) & (0xFF ^ wire.NODE_MAINTENANCE)
    at = np.array([7], np.int32)
    steps = [('load_nodes', {'recs': recs}),
             ('plan_grown', {'scenarios': [([], pods, now, None, None, (at, big)), ([], pods, now)],
                             'source': 'mirror'}),
             ('plan_rounds', {'scenarios': [([], pods, now, None, None, (at, big), _rounds(5000.0, 2))],
                              'source': 'mirror'}),
             _bf('batch_rounds', pods, now, _rounds(5000.0, 2)),
             ('solve_batch', {'pods': pods, 'now': now}),
             ('plan_rounds', {'scenarios': [([], pods, now + 1, None, None, None, _rounds(5001.0, 2))],
                              'source': 'mirror'}),
             ('plan_grown', {'scenarios': [([], pods, now + 2, None, None, (at, recs[[0]]))], 'source': 'mirror'})]
    stats = run_session({'seed': 'four-numa-added', 'steps': steps}, mode)
    assert stats['refusals'].get(wire.ERR_UNSUPPORTED, 0) == 3, stats['refusals']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', _mode_params())
def test_forecasts_on_the_snapshot_source(mode):
    """Forecasts and growth plans with ``source='snapshot'``: answered right after the snapshot, refused after an
    update and after the restore that follows it (no snapshot since the update), answered after snapshot -> batch,
    where the mirror has moved on and the snapshot is still the source."""
    lay = new_layout()
    d = Draw(np.random.default_rng(53), lay)
    n = 257
    recs, other = d.nodes(n), d.nodes(n)
    pods, now = d.pods(40, 40, four=False)
    late, lnow = d.pods(12, 12, four=False)
    t = float(lnow.max())
    add = (np.array([0, n], np.int32), d.added(2))

    def whatif(dt, src='snapshot'):
        return [_bf('batch_rounds', late, lnow + dt, _rounds(t + dt, 3), src, [4], True),
                _bf('batch_releases', late, lnow + dt, _rounds(t + dt, 3), src, [], True, ends=_ends(6, 3),
                    extra=[(0.4, 0xFF, -1)]),
                ('plan_explained', {'scenarios': [([1], late, lnow + dt), ([], late, lnow + dt, 2, ([3], other[[3]]))],
                                    'source': src}),
                ('plan_grown', {'scenarios': [([], late, lnow + dt, None, None, add)], 'source': src}),
                ('plan_rounds', {'scenarios': [([2], late, lnow + dt, None, None, add, _rounds(t + dt, 2)),
                                               ([], late, lnow + dt, None, None, None, [])], 'source': src})]
    steps = [('load_nodes', {'recs': recs}), ('solve_batch', {'pods': pods, 'now': now}), ('snapshot', {})]
    steps += whatif(0)                                                     # no change since the snapshot
    steps += [('update_nodes', {'idx': np.arange(0, n, 4, dtype=np.int32), 'kind': 'hardware',
                                'recs': other[::4]})] + whatif(100)        # refused
    steps += [('restore', {})] + whatif(200)                               # refused, answered on the mirror
    steps += whatif(200, 'mirror') + [('snapshot', {}), ('solve_batch', {'pods': pods, 'now': now + 300})]
    steps += whatif(300) + whatif(300, 'mirror')                           # the snapshot is still the source
    stats = run_session({'seed': 'snapshot-forecasts', 'steps': steps}, mode)
    assert stats['rules'].get('source', 0) == 10, stats
