"""The CUDA solver against the oracle at the edges of the direct path's tables (tests/scenarios.py, limit_scenarios):
free cores per socket around the index clamp of TB at 63, 3 / 4 / 5 NICs per NUMA node, NIC signature ids on both
sides of FAST_NSIG_SMEM (4) and FAST_NSIG (128), more static descriptions than CLASS_SLOTS (4096), and NIC bandwidths
whose remainders land on 0 or within an ulp of it.  Every case compares every binding byte and every final record in
every sweep mode, and the filter's candidate bitmaps with the oracle's candidates."""
import numpy as np
import pytest

from tests import helpers, ref_compare, scenarios
from tests.test_gpu_parity import ALL_CPU_WARPS, _run_cuda

pytestmark = pytest.mark.gpu

CASES = scenarios.limit_scenarios()


@pytest.fixture(scope='module')
def solver_mod():
    from nhd_b200 import solver
    return solver


def _cases(prefix):
    out = [c for c in CASES if c['name'].startswith(prefix)]
    assert out, prefix
    return out


def _check_filter(oracle_lib, solver_mod, recs, speed, pods, now, case):
    """F[type][node] of the filter kernel == the oracle's candidates, for every pod type of the batch."""
    s = solver_mod.Solver(speed, min_busy_secs=case['min_busy_secs'])
    try:
        s.load_nodes(recs)
        s.stage_batch(pods, now)
        feas, _, _, pt = s.filter_bitmaps()
    finally:
        s.close()
    seen = set()
    for i, pod in enumerate(pods):
        if pt[i] in seen:
            continue
        seen.add(pt[i])
        cand = oracle_lib.candidates(recs, speed, pod, now=1e9).astype(bool)
        elig = (recs['group_mask'] & pod['group_mask']) != 0
        assert np.array_equal(feas[pt[i]] & elig, cand), (case['name'], i, np.flatnonzero(feas[pt[i]] != cand)[:8])


def _check(oracle_lib, solver_mod, case):
    """-> the oracle's bindings, after checking the CUDA solver's against them."""
    recs, pods, now, layout = ref_compare.pack_scenario(case)
    recs = scenarios.apply_preuse(recs, case)
    speed = layout.speed_table()
    busy = case['min_busy_secs']
    ob, orecs = oracle_lib.solve(recs, speed, pods, now, min_busy_secs=busy)
    cb, crecs, _ = _run_cuda(solver_mod, recs, speed, pods, now, min_busy=busy, extra_cpu_warps=ALL_CPU_WARPS)
    assert helpers.binding_bytes_equal(ob, cb), (case['name'], helpers.first_binding_diff(ob, cb))
    assert orecs.tobytes() == crecs.tobytes(), (case['name'], ref_compare.diff_records(orecs, crecs)[:3])
    _check_filter(oracle_lib, solver_mod, recs, speed, pods, now, case)
    return ob, recs


def _free_phys(recs):
    """free physical cores per socket of 2-NUMA records (Node.GetFreeCpuCores)."""
    used = np.unpackbits(recs['used'].view(np.uint8).reshape(len(recs), 32), axis=1, bitorder='little').astype(bool)
    out = []
    for r, u in zip(recs, used):
        phys, per = int(r['phys_cores']), int(r['phys_cores']) // 2
        busy = u[:phys] | (u[phys:2 * phys] if r['flags'] & 1 else False)
        out.append((int((~busy[:per]).sum()), int((~busy[per:phys]).sum())))
    return out


def _signatures(recs):
    """distinct per-NUMA NIC signatures (NIC count and speed classes in list order) of 2-NUMA records."""
    sigs = set()
    for r in recs:
        for k in range(2):
            m = int(r['nic_numa_mask'][k])
            sigs.add(tuple((int(r['nic_speed'][l >> 4]) >> (4 * (l & 15))) & 15 for l in range(32) if (m >> l) & 1))
    return sigs


def _reaches_its_side(case, ob, recs):
    """The case sits where its name says: the free counts, NIC counts, signatures and descriptions it claims."""
    cid, placed = case['id'], int((ob['status'] == 0).sum())
    if cid.startswith('a-free'):
        want = {61, 62, 63, 64} | ({65, 100, 128} if 'nosmt' in cid else set())
        assert want <= {f for fr in _free_phys(recs) for f in fr}
        assert placed >= 6 and (ob['status'] == 1).sum() >= 6, placed
    elif cid.startswith('a-bug'):
        # NO_CANDIDATE, but in row 4 the two groups and the misc core take 65 of the 68 free cores (and the only NIC)
        assert ob['status'][0] == 0 if cid == 'a-bug-row4' else (ob['status'] == 1).all()
    elif cid.startswith('a-walk-down'):
        assert placed >= 6 and (ob['status'] == 1).sum() >= 2
    elif cid == 'a-gpu-pci':
        assert placed >= 4 and (ob['n_gpus'][ob['status'] == 0] > 0).all()
    elif cid.startswith('b-nics'):
        n, numa = int(cid[6]), int(cid[-1])
        assert all(bin(int(m)).count('1') == n for m in recs['nic_numa_mask'][:, numa])
        assert len(set(int(m) for m in recs['nic_inuse'])) == 1 << n      # every subset in use on some node
        assert placed > len(ob) // 2
    elif cid == 'c-sig-smem':
        assert len(_signatures(recs)) == 6              # ids 0-3 in shared memory, 4 and 5 in global memory only
        assert placed >= 12
    elif cid == 'c-sig-140':
        assert len(_signatures(recs)) == 140            # 12 more than the 128 ids the tables hold
        assert len(set(ob['node'][ob['status'] == 0].tolist())) >= 60      # the pods reach the nodes past the limit
    elif cid == 'd-classes-4200':
        static = {(r['nic_sw'].tobytes(), r['nic_speed'].tobytes(), r['flags'] & 1) for r in recs}
        assert len(static) == 4200                      # 104 more than the class table has slots
        assert (ob['node'][ob['status'] == 0] >= 4140).all() and placed > 40
    elif cid.startswith('e-fp64'):
        assert placed >= 2 and (ob['status'] != 0).sum() >= 2
    else:
        raise AssertionError(f'no check for {cid}')


@pytest.mark.parametrize('case', CASES, ids=[c['id'] for c in CASES])
def test_limit_case_matches_oracle(oracle_lib, solver_mod, case):
    """a: TB[type][smt][numa][free cores] clamps the free count at 63 (sockets with 61-65, 100 and 128 free physical
    cores, CPU-only types asking 60-72 of one socket with misc cores and the SMT flags, G = 1 and 2, both groups held on
    one socket by its only NIC, batches that take a node down through 63, GPU / PCI types at the same demands).
    b: 3, 4 and 5 NICs on NUMA 0 or 1 (the direct path admits at most 4: fast_node_aux's unrolled gather, the filter's
    loop), every subset of them in use on some node, NIC lists that interleave the two NUMA nodes.
    c, d: routing limits, where either side must give the same answer: signature ids below FAST_NSIG_SMEM read their
    table rows from shared memory, the others from global memory (the general path's direct_single); past FAST_NSIG
    a class has no direct-path entry; past CLASS_SLOTS a node has no class.
    e: group Gb/s that are not dyadic, so that a NIC's remainder lands on 0, or an ulp either side of it, in one group
    order and not in the other, with NICs shared by the groups of a pod (nic_sub_solve, nic_first_fit); the
    reference's outcomes on the same scenarios are frozen in golden/live (test_oracle_vs_reference.py)."""
    ob, recs = _check(oracle_lib, solver_mod, case)
    _reaches_its_side(case, ob, recs)


def test_signature_ids_run_out_across_updates(oracle_lib, solver_mod):
    """Signatures are only ever added: one handle, 60 signatures at load, 100 after one update_nodes, 140 (past
    FAST_NSIG = 128) after a second; each stage against the oracle on the same records."""
    sig = scenarios.signature_list(140)
    stages = []
    for hi in (60, 100, 140):
        # nodes 0 .. hi/2 - 1 bring new signatures, the rest repeat the first 60
        pairs = [(sig[2 * i], sig[2 * i + 1]) if 2 * i < hi else (sig[2 * i % 60], sig[2 * i % 60 + 1]) for i in range(70)]
        stages.append({'nodes': scenarios.signature_nodes('u', pairs), 'pods': scenarios.signature_pods() * 12,
                       'now': [2000.0] * 48, 'min_busy_secs': 0.0})
    packed = [ref_compare.pack_scenario(st) for st in stages]
    speed = packed[0][3].speed_table()
    assert all(np.array_equal(p[3].speed_table(), speed) for p in packed)
    assert [len(_signatures(p[0])) for p in packed] == [60, 100, 140]
    pods, now = packed[0][1], packed[0][2]
    for dbg in (0, 5):
        s = solver_mod.Solver(speed, min_busy_secs=0.0, sweep_debug=dbg)
        try:
            state = packed[0][0].copy()
            s.load_nodes(state)
            for k, (recs, _, _, _) in enumerate(packed):
                if k:
                    idx = np.flatnonzero([a.tobytes() != b.tobytes() for a, b in zip(recs, packed[k - 1][0])])
                    assert len(idx) > 0
                    state[idx] = recs[idx]
                    s.update_nodes(idx.astype(np.int32), recs[idx])
                ob, orecs = oracle_lib.solve(state, speed, pods, now, min_busy_secs=0.0)
                cb = s.solve_batch(pods, now)
                assert helpers.binding_bytes_equal(ob, cb), (dbg, k, helpers.first_binding_diff(ob, cb))
                assert s.read_nodes().tobytes() == orecs.tobytes(), (dbg, k)
                assert (ob['status'] == 0).sum() > 20
                state = orecs.copy()
        finally:
            s.close()
