"""ctypes binding of the explanation oracle (tests/explain_oracle.c).  ORACLE — tests only.

The library is compiled on first use into the temporary directory (keyed by the sources' contents), so that the
repository tree is never written."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from nhd_b200 import wire

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SOURCES = [os.path.join(_HERE, 'explain_oracle.c'), os.path.join(_ROOT, 'oracle', 'nhd_oracle.c'),
            os.path.join(_ROOT, 'oracle', 'pyset_model.c'), os.path.join(_ROOT, 'oracle', 'nhd_oracle.h'),
            os.path.join(_ROOT, 'oracle', 'pyset_model.h'), os.path.join(_ROOT, 'include', 'nhd_b200.h')]
_lib = None


def build():
    """Compile (once per content) with the oracle's own flags (oracle/Makefile); returns the library path."""
    h = hashlib.sha256()
    for s in _SOURCES:
        with open(s, 'rb') as f:
            h.update(f.read())
    so = os.path.join(tempfile.gettempdir(), f'nhd_explain_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so')
    if not os.path.exists(so):
        tmp = f'{so}.{os.getpid()}.tmp'
        subprocess.run(['gcc', '-O2', '-fPIC', '-Wall', '-std=gnu11', '-ffp-contract=off', '-pthread', '-shared',
                        '-o', tmp, _SOURCES[0], _SOURCES[2], '-lm'], check=True, capture_output=True)
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        from oracle.binding import OracleParams
        L = ctypes.CDLL(build())
        L.nhd_oracle_explain.restype = ctypes.c_int
        L.nhd_oracle_explain.argtypes = [ctypes.POINTER(OracleParams), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_double, ctypes.c_void_p]
        _lib = L
    return _lib


def explain(recs, speed_table, pod, now, nic_bw_avail_percent=0.9, min_busy_secs=30.0):
    """Reason code (wire.WHY_*) of every node for one pod on the given state; wire.WHY_COUNT = the node fits."""
    from oracle.binding import OracleParams
    recs = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE)
    pod = np.ascontiguousarray(pod, dtype=wire.POD_DTYPE).reshape(1)
    speed = np.ascontiguousarray(speed_table, dtype='<f8')
    out = np.zeros(len(recs), dtype=np.uint8)
    p = OracleParams(nic_bw_avail_percent, min_busy_secs)
    rc = lib().nhd_oracle_explain(ctypes.byref(p), speed.ctypes.data, len(recs), recs.ctypes.data, pod.ctypes.data,
                                  float(now), out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f'nhd_oracle_explain failed: {rc}')
    return out


def batch(recs, speed_table, pods, now, which=None, nic_bw_avail_percent=0.9, min_busy_secs=30.0, threads=1):
    """The oracle's bindings of the batch and {pod index: node reasons} for its NO_CANDIDATE pods (only those in
    ``which`` when given), each on the state after ``nhd_oracle_solve`` of the pods before it."""
    from oracle import binding
    kw = dict(nic_bw_avail_percent=nic_bw_avail_percent, min_busy_secs=min_busy_secs, threads=threads)
    out, _ = binding.solve(recs, speed_table, pods, now, **kw)
    targets = [i for i in range(len(pods)) if out[i]['status'] == wire.NO_CANDIDATE and (which is None or i in which)]
    cur = np.ascontiguousarray(recs, dtype=wire.NODE_DTYPE).copy()
    reasons, prev = {}, 0
    for i in targets:
        if i > prev:
            _, cur = binding.solve(cur, speed_table, pods[prev:i], now[prev:i], **kw)
            prev = i
        reasons[i] = explain(cur, speed_table, pods[i], now[i], nic_bw_avail_percent, min_busy_secs)
    return out, reasons


def counts(reasons, n_pods):
    """{pod: node reasons} -> (n_pods, WHY_COUNT) histogram rows, as nhd_explain_batch returns them."""
    rows = np.zeros((n_pods, wire.WHY_COUNT), dtype='<u4')
    for i, r in reasons.items():
        rows[i] = np.bincount(r, minlength=wire.WHY_COUNT + 1)[:wire.WHY_COUNT]
    return rows
