"""Freeze the UNMODIFIED reference's own reasons for dropping nodes into tests/golden/live/explain.json.gz.

Every pod of the streams (the four ``oracle_scenarios`` flavours of make_live_golden.py and
``tests.explain_scenarios.explain_scenarios()``) is scheduled by the reference (``ref_loader.attempt_scheduling``),
with a ``logging.Handler`` on the reference Matcher's logger.  For each pod that gets ``(None,)`` every node is given
the code (NHD_WHY_*, include/nhd_b200.h) of the record that dropped it:
    NHDScheduler.InitialNodeFilter (:240 groups, :241 active)   -> 0 / 1, from the restatement in ref_loader
    "Node ... in maintenance. Removing node"          Matcher.py:74   -> 2
    "Node ... only has ... hugepages ... Removing"             :79    -> 3
    "Dropping node ... last deploy was only ..."               :109   -> 4
    "Dropping node ... not enough free GPUs"                   :133   -> 5
    "Dropping node ... not enough free CPU cores"              :215   -> 6
    "Dropping node ... not enough free NIC resources"          :271   -> 7
    "Node ... has no valid intersection candidates" / "Not enough resources of at least one type" :353/:386 -> 8
The file holds, per stream and scenario, {pod index: one digit per node}.  Every code must occur at least 5 times.

    NHD_REFERENCE_ROOT=<checkout of the reference> python tests/golden/make_explain_golden.py
"""
import contextlib
import io
import logging
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden import make_live_golden as live       # noqa: E402

DROPS = [(re.compile(r'^Node (\S+) in maintenance\. Removing node'), 2),
         (re.compile(r'^Node (\S+) only has .* Removing node'), 3),
         (re.compile(r'^Dropping node (\S+) from candidate list beacause last deploy'), 4),
         (re.compile(r'^Dropping node (\S+) from candidate list since not enough free GPUs'), 5),
         (re.compile(r'^Dropping node (\S+) from candidate list since not enough free CPU cores'), 6),
         (re.compile(r'^Dropping node (\S+) from candidate list since not enough free NIC resources'), 7),
         (re.compile(r'^Node (\S+) has no valid intersection candidates'), 8),
         (re.compile(r'^Not enough resources of at least one type for node (\S+)\.'), 8)]


class _Records(logging.Handler):
    def __init__(self):
        super().__init__(logging.DEBUG)
        self.msgs = []

    def emit(self, record):
        self.msgs.append(record.getMessage())


def reference_reasons(scn, ref, handler):
    """{pod index: codes string} for the pods of scn the reference cannot place."""
    from oracle import ref_loader
    from tests import scenarios
    ref.node.Node.MIN_BUSY_SECS = float(scn.get('min_busy_secs', 30.0))
    nodes = scenarios.build_nodes(scn, ref.node)
    names = list(nodes)
    matcher = ref.matcher.Matcher()
    out = {}
    for i, (pod, now) in enumerate(zip(scn['pods'], scn['now'])):
        top = scenarios.build_top(pod, ref.cfg)
        handler.msgs = []
        with contextlib.redirect_stdout(io.StringIO()):
            r = ref_loader.attempt_scheduling(ref, matcher, nodes, top, pod['groups'], now)
        if r['status'] != 'none' or pod['map_type'] not in ('NUMA', 'PCI'):
            continue
        codes = {}
        for n, v in nodes.items():                            # InitialNodeFilter, NHDScheduler.py:240-241
            if not set(v.groups) & set(pod['groups']):
                codes[n] = 0
            elif not v.active:
                codes[n] = 1
        for msg in handler.msgs:
            for rx, code in DROPS:
                m = rx.match(msg)
                if m:
                    assert m.group(1) not in codes, (msg, codes)
                    codes[m.group(1)] = code
        assert sorted(codes) == sorted(names), (i, codes, handler.msgs)
        out[str(i)] = ''.join(str(codes[n]) for n in names)
    ref.node.Node.MIN_BUSY_SECS = 30.0
    return out


def make_explain():
    from oracle import ref_loader
    from tests.explain_scenarios import explain_scenarios
    ref = ref_loader.load()
    logging.disable(logging.NOTSET)
    handler = _Records()
    logger = logging.getLogger(ref.matcher.__name__)
    logger.addHandler(handler)
    logger.setLevel(logging.DEBUG)
    try:
        doc = {f: [reference_reasons(s, ref, handler) for s in live.oracle_scenarios(f)]
               for f in ('mixed', 'wild', 'vf', 'big')}
        doc['explain'] = [reference_reasons(s, ref, handler) for s in explain_scenarios()]
    finally:
        logger.removeHandler(handler)
        logging.disable(logging.CRITICAL)
    seen = [0] * 9
    for rows in doc.values():
        for per_pod in rows:
            for codes in per_pod.values():
                for c in codes:
                    seen[int(c)] += 1
    assert min(seen) >= 5, seen
    print('codes', seen)
    live._save('explain', doc)


if __name__ == '__main__':
    if not __import__('oracle.ref_loader', fromlist=['x']).available():
        raise SystemExit('set NHD_REFERENCE_ROOT to a checkout of the reference')
    make_explain()
