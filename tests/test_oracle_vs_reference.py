"""Differential test: the C oracle against the UNMODIFIED reference, whose outcomes on these scenarios are frozen in
tests/golden/live/oracle.json.gz (tests/golden/make_live_golden.py).  This is the pin that makes the oracle
trustworthy; tests/golden/*.json are further frozen runs of the same kind."""
import numpy as np
import pytest

from nhd_b200 import wire
from tests import ref_compare, scenarios
from tests.golden import make_live_golden as live


def _records(hexstr):
    return np.frombuffer(bytes.fromhex(hexstr), dtype=wire.NODE_DTYPE)


def _compare(oracle_lib, scn, want, tag):
    """-> (attempts, placed) after checking the oracle's run of scn against the reference's frozen one."""
    init, final = _records(want['init']), _records(want['final'])
    recs, pods, now, layout2 = ref_compare.pack_scenario(scn)
    # the packer gives identical records from the reference's Node objects and from the mirrors
    assert ref_compare.records_equal(recs, init), ref_compare.diff_records(recs, init)[:3]
    b, orecs = oracle_lib.solve(recs, layout2.speed_table(), pods, now, min_busy_secs=scn['min_busy_secs'])
    assert len(want['outs']) == len(b)
    placed = 0
    for i, (o, bb) in enumerate(zip(want['outs'], b)):
        errs = ref_compare.diff_outcome(o, bb)
        assert not errs, (tag, i, errs)
        placed += o['status'] == 'placed'
    assert not ref_compare.diff_records(orecs, final), tag
    return len(b), placed


@pytest.mark.parametrize('flavor', ['mixed', 'wild', 'vf', 'big'])
def test_oracle_matches_live_reference(oracle_lib, flavor):
    attempts = placed = 0
    golden = live.load('oracle')[flavor]
    for seed, (scn, want) in enumerate(zip(live.oracle_scenarios(flavor), golden, strict=True)):
        a, p = _compare(oracle_lib, scn, want, (flavor, seed))
        attempts += a
        placed += p
    assert attempts == 900 and placed > 150


def test_mirror_node_ingest_matches_reference_labels():
    """nhd_b200.Node.ParseLabels builds the same node as nhd.Node.ParseLabels (Node.py:312-487)."""
    import nhd_b200.Node as mirror
    golden = live.load('oracle')['node_descriptions']
    for seed, (scn, want) in enumerate(zip(live.ingest_node_scenarios(), golden, strict=True)):
        got = {name: live.node_description(n) for name, n in scenarios.build_nodes(scn, mirror).items()}
        assert list(got) == list(want), seed
        for name in want:
            assert got[name] == want[name], (seed, name)


def test_oracle_matches_live_reference_near_the_limits(oracle_lib):
    """Nodes with up to 256 logical cores / 16 GPUs / 32 NICs / 4 NUMA nodes and pods with up to 72 cores: the
    reference itself is slow here (seconds per pod), so a few short streams."""
    attempts = placed = 0
    golden = live.load('oracle')['near_limits']
    for seed, (scn, want) in enumerate(zip(live.near_limit_scenarios(), golden, strict=True)):
        a, p = _compare(oracle_lib, scn, want, seed)
        attempts += a
        placed += p
    assert attempts == 42 and placed > 20


def test_oracle_matches_live_reference_on_non_dyadic_nic_bandwidth(oracle_lib):
    """Group Gb/s such as 0.1, 0.3, 12.7 and 33.3, summed per group in core order and taken off a NIC in group order,
    leave remainders of exactly 0 or an ulp either side of it (tests/scenarios.py, nic_bandwidth_scenarios): the
    per-group sums of the packing and the oracle's subtraction order against the reference's."""
    attempts = placed = 0
    golden = live.load('oracle')['nic_fp64']
    for seed, (scn, want) in enumerate(zip(scenarios.nic_bandwidth_scenarios(), golden, strict=True)):
        a, p = _compare(oracle_lib, scn, want, scn['id'])
        attempts += a
        placed += p
    assert attempts == 96 and placed > 40
