"""nhd_b200/tracking.py: the change counter Matcher.FindNode relies on moves on every mutation of a Node — attribute
writes and every method that is not a plain getter — on this package's mirror of the reference's class."""
from nhd_b200 import tracking
from tests import scenarios


def _exercise(node_mod, cfg_mod):
    scn = scenarios.random_scenario(515, n_nodes=2, n_pods=6, flavor='mixed')
    assert tracking.track_changes(node_mod.Node) and tracking.track_changes(node_mod.Node)      # idempotent
    nodes = scenarios.build_nodes(scn, node_mod)
    n = next(iter(nodes.values()))
    ver = lambda: n.__dict__.get(tracking.VERSION, 0)
    v = ver()
    for getter in ('GetFreeCpuCores', 'GetTotalGPUs', 'GetFreeNumaGPUs', 'IsBusy', 'SMTEnabled', 'GetFreeGpuCount'):
        if hasattr(n, getter):
            getattr(n, getter)()
    assert ver() == v                                          # getters do not count
    n.active = not n.active; assert ver() > v; v = ver()       # attribute writes (NHDScheduler.py:541-549)
    n.maintenance = True; assert ver() > v; v = ver()
    n.SetBusy(); assert ver() > v; v = ver()                   # Node.py:843-845
    n.SetGroups('default.a'); assert ver() > v; v = ver()
    n.ClaimPodNICResources([0] if n.nics else []); assert ver() > v; v = ver()
    n.SetHugepages(64, 32); assert ver() > v; v = ver()
    top = scenarios.build_top(scn['pods'][0], cfg_mod)
    try:
        n.RemoveResourcesFromTopology(top)                      # counts whether or not it succeeds / raises
    except Exception:
        pass
    assert ver() > v; v = ver()
    n.ResetResources(); assert ver() > v
    other = list(nodes.values())[1]
    w = other.__dict__.get(tracking.VERSION, 0)
    n.active = True
    assert other.__dict__.get(tracking.VERSION, 0) == w        # per instance
    tracking.bump(other)
    assert other.__dict__[tracking.VERSION] == w + 1


def test_counter_on_the_mirror_node():
    import nhd_b200.CfgTopology as cfg_mod
    import nhd_b200.Node as node_mod
    _exercise(node_mod, cfg_mod)


def test_classes_that_cannot_carry_a_counter_are_reported():
    class Slotted:
        __slots__ = ('x',)
    assert tracking.track_changes(Slotted) is False and not tracking.is_tracked(Slotted)
    tracking.bump(Slotted())                                    # harmless
