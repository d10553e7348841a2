"""Hardware parity at the sizes BASELINE.json names: every binding and every final node record of the CUDA
solver against the C oracle (all host threads, ``nhd_oracle_solve_mt``), not just invariants.

  config 3   16 384 nodes x 1 024 pods   (+GPU / NIC PCI-switch affinity)            in full
  config 4   65 536 nodes x 4 096 pods   (the metric's configuration)                in full, every sweep mode
  config 5  262 144 nodes x 8 192 pods   (SR-IOV VFs + node groups N:N)              all nodes, the first 1 024 pods
                                          (the host needs minutes for all 8 192; NHD_FULL_CONFIG5=1 does them),
                                          and windows of 256 pods deep in the stream

and the side workloads bench.py times on one GPU at the size it times them:

  config 4 `wild` (heterogeneous: more hardware classes than class slots, 120 NIC signatures), then a second batch on
  the same handle after an update; config 4 with per-pod clocks: bench.py's 1 ms steps, and a stream whose +31 s and
  -40 s steps make nodes leave the busy window and the busy set be rebuilt inside the batch (scenarios.jumping_clocks)

The oracle walks every node for every pod like the reference does (nhd/Matcher.py:86-391), so these cost tens of
seconds of host time each; they are `-m gpu` tests.  A multi-rank run (sharded filter + exchange + replicated
sweep) is compared with the oracle in tests/test_gpu_multirank.py."""
import os

import numpy as np
import pytest

import workload
from tests import helpers, ref_compare, scenarios
from tests.test_handle_session import static_key

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get('NHD_B200_ALLOW_EMULATED') == '1',
                                 reason='full sizes on the CPU-emulated device take too long for the suite '
                                        '(tools/emu_full_size.py does them)')]

THREADS = max(1, os.cpu_count() or 1)
CLASS_SLOTS = 4096                # nhd_kernels.cuh: the claim table of the hardware classes
FAST_NSIG_SMEM = 4                # nhd_kernels.cuh: NIC signatures whose direct-path rows the sweep keeps in shared memory
MODES = (dict(), dict(single_warp=True), dict(cpu_warps=1), dict(sweep_debug=1), dict(sweep_debug=5))


def _cuda(recs, speed, pods, now, **mode):
    from nhd_b200 import solver
    s = solver.Solver(speed, **mode)
    try:
        s.load_nodes(recs)
        b = s.solve_batch(pods, now)
        return b, s.read_nodes()
    finally:
        s.close()


def _check(ob, orecs, cb, crecs, tag):
    assert helpers.binding_bytes_equal(ob, cb), (tag, helpers.first_binding_diff(ob, cb))
    assert orecs.tobytes() == crecs.tobytes(), (tag, ref_compare.diff_records(orecs, crecs)[:3])


def test_config3_full_size_equals_oracle(oracle_lib):
    recs, speed, pods, now = workload.make_workload(3)
    assert len(recs) == 16384 and len(pods) == 1024
    ob, orecs = oracle_lib.solve(recs, speed, pods, now, threads=THREADS)
    for mode in MODES[:3]:
        cb, crecs = _cuda(recs, speed, pods, now, **mode)
        _check(ob, orecs, cb, crecs, mode)
    assert int((ob['status'] == 0).sum()) > 900


def test_config4_full_size_equals_oracle_in_every_sweep_mode(oracle_lib):
    recs, speed, pods, now = workload.make_workload(4)
    assert len(recs) == 65536 and len(pods) == 4096
    ob, orecs = oracle_lib.solve(recs, speed, pods, now, threads=THREADS)
    for mode in MODES:
        cb, crecs = _cuda(recs, speed, pods, now, **mode)
        _check(ob, orecs, cb, crecs, mode)
    assert int((ob['status'] == 0).sum()) > 3000


def test_config5_full_cluster_equals_oracle(oracle_lib):
    recs, speed, pods, now = workload.make_workload(5)
    assert len(recs) == 262144 and len(pods) == 8192
    n = len(pods) if os.environ.get('NHD_FULL_CONFIG5') == '1' else 1024
    ob, orecs = oracle_lib.solve(recs, speed, pods[:n], now[:n], threads=THREADS)
    for mode in MODES[:2]:
        cb, crecs = _cuda(recs, speed, pods[:n], now[:n], **mode)
        _check(ob, orecs, cb, crecs, mode)
    # and the whole stream is at least self-consistent across sweep modes
    full = [_cuda(recs, speed, pods, now, **mode) for mode in MODES[:2]]
    assert helpers.binding_bytes_equal(full[0][0], full[1][0])
    assert full[0][1].tobytes() == full[1][1].tobytes()
    assert helpers.binding_bytes_equal(full[0][0][:n], ob)


def test_config4_wild_full_size_then_a_second_batch_in_every_sweep_mode(oracle_lib):
    """bench.py's `heterogeneous_65536x4096`: the class table is full before the sweep starts (nodes whose class
    missed it bypass the memos), NIC signature ids run past the four whose rows sit in shared memory, and most
    decisions take the general path.  Then the scheduler's steady state on the same handle: an update gives 1 024
    nodes of the batch their start records back (a quarter of them another node's, so their hardware class changes)
    and a second batch a minute later meets the full class table, the warm mapping memo and the NIC signatures carried
    over; it is compared with the oracle run on the oracle's own records after the same update."""
    from nhd_b200 import solver
    recs, speed, pods, now = workload.make_workload(4, wild=True)
    assert len(recs) == 65536 and len(pods) == 4096
    classes, sigs = len({static_key(r) for r in recs}), len(scenarios.nic_signatures(recs))
    print(f'static descriptions {classes} for {CLASS_SLOTS} class slots, {sigs} NIC signatures')
    assert classes > CLASS_SLOTS and sigs > FAST_NSIG_SMEM
    ob, orecs = oracle_lib.solve(recs, speed, pods, now, threads=THREADS)
    idx, upd = scenarios.steady_state_update(recs, ob)
    assert sum(static_key(a) != static_key(b) for a, b in zip(orecs[idx], upd)) > 200
    pods2, now2 = workload.make_pods(4, n_pods=1024, seed=61)
    now2 = now2 + 60.0
    after = orecs.copy()
    after[idx] = upd
    ob2, orecs2 = oracle_lib.solve(after, speed, pods2, now2, threads=THREADS)
    for mode in MODES:
        s = solver.Solver(speed, **mode)
        try:
            s.load_nodes(recs)
            _check(ob, orecs, s.solve_batch(pods, now), s.read_nodes(), mode)
            s.update_nodes(idx, upd)
            _check(ob2, orecs2, s.solve_batch(pods2, now2), s.read_nodes(), (mode, 'second batch'))
        finally:
            s.close()
    assert int((ob['status'] == 0).sum()) > 3000 and int((ob2['status'] == 0).sum()) > 900
    assert np.isin(ob2['node'], idx).sum() > 100                    # the second batch lands on the updated nodes


@pytest.mark.parametrize('stream', ['moving', 'jumps'])
def test_config4_per_pod_clocks_full_size_equals_oracle_in_every_sweep_mode(oracle_lib, stream):
    """Config 4 with a clock per pod: the one-warp general path and its busy list.  `moving` is bench.py's
    `moving_clock_65536x4096` stream (1 ms steps: nothing leaves the 30 s window, so the forward shortcut holds
    throughout); `jumps` (scenarios.jumping_clocks) adds +31 s steps, after which stamps expire and GPU nodes take
    GPU pods again, and -40 s steps, which rebuild the busy set over all nodes with thousands of stamps on it."""
    recs, speed, pods, now = workload.make_workload(4)
    now = now + 0.001 * np.arange(len(pods)) if stream == 'moving' else scenarios.jumping_clocks(len(pods))
    ob, orecs = oracle_lib.solve(recs, speed, pods, now, threads=THREADS)
    back, repeated = int((np.diff(now) < 0).sum()), len(scenarios.repeated_gpu_nodes(pods, ob))
    print(f'{stream}: {back} backwards steps, {repeated} GPU nodes with two or more GPU pods')
    if stream == 'jumps':
        assert back >= 5 and repeated >= 50
    for mode in MODES:
        cb, crecs = _cuda(recs, speed, pods, now, **mode)
        _check(ob, orecs, cb, crecs, mode)
    assert int((ob['status'] == 0).sum()) > 3000


def test_config5_windows_deep_in_the_stream(oracle_lib):
    """Config 5 beyond the first 1 024 pods: a handle solves pods[:k] (k = 2 048, 4 096, 7 936), the oracle and a
    fresh handle then solve pods[k:k + 256] from the records it read back, and both must equal bindings [k:k + 256]
    of the whole stream solved at once; the first handle's second batch pods[k:] must reproduce the rest of the whole
    run's bindings and its final records byte for byte (the prefix property at 262 144 nodes).

    What this does not prove: each window starts from the GPU's own state at k, which is pinned to the oracle only
    through the first 1 024 pods (test_config5_full_cluster_equals_oracle) and the prefix property.  A difference
    before k that left the records wrong would go unseen here; NHD_FULL_CONFIG5=1 runs the whole stream against the
    oracle."""
    from nhd_b200 import solver
    recs, speed, pods, now = workload.make_workload(5)
    fb, frecs = _cuda(recs, speed, pods, now)
    for k in (2048, 4096, 7936):
        s = solver.Solver(speed)
        try:
            s.load_nodes(recs)
            head = s.solve_batch(pods[:k], now[:k])
            mid = s.read_nodes()
            rest = s.solve_batch(pods[k:], now[k:])
            final = s.read_nodes()
        finally:
            s.close()
        assert helpers.binding_bytes_equal(head, fb[:k]), (k, helpers.first_binding_diff(fb[:k], head))
        assert helpers.binding_bytes_equal(rest, fb[k:]), (k, helpers.first_binding_diff(fb[k:], rest))
        assert final.tobytes() == frecs.tobytes(), (k, ref_compare.diff_records(frecs, final)[:3])
        win = slice(k, k + 256)
        ob, orecs = oracle_lib.solve(mid, speed, pods[win], now[win], threads=THREADS)
        cb, crecs = _cuda(mid, speed, pods[win], now[win])
        _check(ob, orecs, cb, crecs, k)
        assert helpers.binding_bytes_equal(ob, fb[win]), (k, helpers.first_binding_diff(ob, fb[win]))
        print(f'config 5 window at {k}: {int((ob["status"] == 0).sum())} of 256 placed')
        assert int((ob['status'] == 0).sum()) > 128
