"""nhd_b200 — H100-native batched placement solver for the NHD scheduler's hot path.

Layout:
  csrc/            CUDA kernels (sm_90a) and the C-ABI library (include/nhd_b200.h)
  _lib, solver     ctypes binding and handle wrapper
  wire, packing    packed record formats and object <-> record conversion
  CfgTopology, Node, Matcher, NHDScheduler   host-side mirrors of the reference interface
  ingest           native node-label ingest and node statistics
  TriadCfgParser, libconfig   the request codec (libconfig text <-> CfgTopology)
  NHDRpcServer     the gRPC statistics service
"""
__all__ = ['CfgTopology', 'Node', 'Matcher', 'NHDScheduler', 'packing', 'wire', 'solver', 'ingest']
