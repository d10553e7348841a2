"""Load the UNMODIFIED reference hot-path modules from the checkout named by
NHD_REFERENCE_ROOT.

TEST INFRASTRUCTURE ONLY (oracle).  The reference is not part of this
repository, so no test or smoke() imports this module.  It is used by the
generators under tests/golden/ (make_golden.py, make_live_golden.py, ...) to
freeze golden vectors, and by the optional Python-reference leg of bench.py
(through tests/pyref.py), which runs only when NHD_REFERENCE_ROOT is set.

Recipe follows SURVEY.md appendix D: a `colorlog` stub on sys.path, logging
disabled, and a fake clock patched into nhd.Node.time.monotonic so the 30 s
busy window (nhd/Node.py:843-850) is deterministic.
"""
import logging
import os
import sys
import types

REFERENCE_ROOT = os.environ.get('NHD_REFERENCE_ROOT', '')
_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_shim')


def available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, 'nhd', 'Matcher.py'))


class FakeClock:
    """Replacement for time.monotonic inside nhd.Node."""
    def __init__(self, t=1000.0):
        self.t = float(t)

    def __call__(self):
        return self.t


_loaded = None


def load(silent=True):
    """Returns a namespace with the reference modules and the fake clock."""
    global _loaded
    if _loaded is not None:
        return _loaded
    if not available():
        raise RuntimeError(f'reference not found under {REFERENCE_ROOT}')
    if _SHIM not in sys.path:
        sys.path.insert(0, _SHIM)
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(1, REFERENCE_ROOT)
    if silent:
        logging.disable(logging.CRITICAL)
    import nhd.CfgTopology as ref_cfg
    import nhd.Node as ref_node
    import nhd.Matcher as ref_matcher
    clock = FakeClock()
    fake_time = types.SimpleNamespace(monotonic=clock)
    ref_node.time = fake_time          # only time.monotonic is used (Node.py:845,848)
    ns = types.SimpleNamespace(cfg=ref_cfg, node=ref_node, matcher=ref_matcher, clock=clock)
    _loaded = ns
    return ns


def attempt_scheduling(ref, matcher, nodes, top, pod_groups, now):
    """The compute lines of NHDScheduler.AttemptScheduling (NHDScheduler.py:274-304)
    and InitialNodeFilter (:235-247), with all Kubernetes I/O removed.

    Returns a dict describing the outcome; mutates `nodes` and `top` exactly as
    the reference scheduler thread would."""
    ref.clock.t = float(now)
    # InitialNodeFilter, NHDScheduler.py:239-245
    nl = {}
    for n, v in nodes.items():
        if len(set(v.groups) & set(pod_groups)) > 0:
            if v.active:
                nl[n] = v
    match = matcher.FindNode(nl, top)                       # :277
    nodename = match[0]                                     # :278
    if nodename is None:
        return {'status': 'none'}
    nodes[nodename].SetBusy()                               # :289
    out = {'node': nodename, 'mapping': match[1]}
    try:
        nic_list = nodes[nodename].SetPhysicalIdsFromMapping(match[1], top)   # :292
    except IndexError:
        out['status'] = 'assign_failed'                     # :296-299
        return out
    except TypeError:
        out['status'] = 'crash'                             # Node.py:833-835 (would kill the thread)
        return out
    nidx = list({x[0] for x in nic_list})                   # :302
    nodes[nodename].ClaimPodNICResources(nidx)              # :304
    out['status'] = 'placed'
    out['nic_list'] = nic_list
    out['nidx'] = nidx
    return out
