"""Load the UNMODIFIED reference scheduler (nhd/NHDScheduler.py) from NHD_REFERENCE_ROOT.

TEST INFRASTRUCTURE ONLY (oracle), golden-vector generators only — same rules as ref_loader.py.

``nhd.NHDScheduler`` imports ``kubernetes`` (through ``nhd.K8SMgr``), ``libconf`` and
``magicattr`` (through ``nhd.TriadCfgParser``), none of which exist here (SURVEY 8c).  The last two
are restated under ``oracle/_shim`` so that the reference's codec runs (``load_codec``); ``kubernetes``
is only *imported* on the path we drive — ``CheckPendingPods`` / ``AttemptScheduling`` /
``ReleasePodResources`` / ``ResetResources`` / ``GetBasicNodeStats`` / ``GetPodStats``
(``NHDScheduler.py:107-205, 235-441``) talk to ``self.k8s`` and ``self.GetCfgParser`` — so empty
stub modules are enough: the scheduler object is created without running its constructor
(which would open a cluster connection, ``NHDScheduler.py:43-60``) and is handed a fake
Kubernetes manager and a fake config parser (tests/fake_k8s.py).
"""
import logging
import sys
import types
import warnings

from oracle import ref_loader

_loaded = None


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def load():
    """Returns ref_loader's namespace extended with ``sched`` (the reference module)."""
    global _loaded
    if _loaded is not None:
        return _loaded
    ref = ref_loader.load()
    if 'kubernetes' in sys.modules:
        raise RuntimeError('kubernetes unexpectedly importable; review this loader')
    k = _stub('kubernetes')
    k.client = _stub('kubernetes.client')
    k.config = _stub('kubernetes.config')
    k.watch = _stub('kubernetes.watch')
    k.client.rest = _stub('kubernetes.client.rest', ApiException=type('ApiException', (Exception,), {}))
    # libconf / magicattr: the stand-ins under oracle/_shim (already on sys.path) are imported by
    # nhd.TriadCfgParser itself
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import nhd.NHDScheduler as ref_sched
    ref.sched = ref_sched
    _loaded = ref
    return ref


def load_codec():
    """The UNMODIFIED ``nhd.TriadCfgParser`` running on the libconf / magicattr stand-ins."""
    ref = ref_loader.load()
    if not hasattr(ref, 'codec'):
        import nhd.TriadCfgParser as ref_codec
        ref.codec = ref_codec
    return ref


def make_scheduler(ref, k8s, cfg_parser=None):
    """A reference ``NHDScheduler`` wired to fakes; ``cfg_parser(cfgtype, cfgstr)`` replaces
    ``GetCfgParser`` (``NHDScheduler.py:226-232``)."""
    S = ref.sched.NHDScheduler
    s = S.__new__(S)                                   # fields of NHDScheduler.__init__ (:43-60) minus the I/O
    s.logger = logging.getLogger('nhd.ref_sched')
    s.nodes = {}
    s.k8s = k8s
    s.sched_name = ref.sched.NHD_SCHED_NAME
    s.matcher = ref.matcher.Matcher()
    s.pod_state = {}
    s.rpcq = None
    s.failed_schedule_count = 0
    if cfg_parser is not None:                         # else the reference's own GetCfgParser -> TriadCfgParser
        s.GetCfgParser = cfg_parser
    return s
