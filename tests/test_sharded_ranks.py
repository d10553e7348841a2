"""Node-sharded ranks on the emulated device, every rank against the oracle.

With ``world_size > 1`` every rank filters its shard of the super-tiles into a slot, one all-gather hands every rank
all slots, and every rank runs the sweep on its own replica.  A node's summary carries its hardware class id, and the
id is rank-private: it is the slot the class won in that rank's claim table, so it depends on the order the claims
arrived in and on what the rank loaded before.  These runs give the ranks different claim orders (lane order,
warp schedule) and different load histories, and check that every rank still returns the oracle's bindings and final
records, across the shapes of the exchange (uneven and empty shards, three ranks, partial super-tiles, group-name
rows, many pod types) and across one long-lived handle (updates, snapshot / restore, staged re-solves, reloads at
other sizes, the sharding threshold).

One worker script (``WORKER``) runs a list of operations on every rank, in a process of its own with the emulated
library and ``tests/emu/fake_nccl``; a rank-restricted operation runs on the named ranks only.  The parent replays
the common operations through the oracle, and the rank-local calls (explanations, queries, plans) are compared with
one single-rank handle that runs the common operations."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import workload  # noqa: E402
from nhd_b200 import wire  # noqa: E402
from tests import helpers  # noqa: E402

CLASS_SLOTS = 4096                       # nhd_kernels.cuh: the claim table of the hardware classes
SUPER_NODES = 256
SMEM_OPTIN = 227 * 1024                  # shared memory per block of an H100 (and of the emulated device)

WORKER = r'''
import ctypes, json, os, sys, time
import numpy as np
root, tmp, rank, world = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
sys.path.insert(0, root)
if world > 1:
    ctypes.CDLL(os.path.join(root, 'tests', 'emu', 'fake_nccl', 'libnccl.so.2'), mode=ctypes.RTLD_GLOBAL)
from nhd_b200 import wire
from nhd_b200.solver import Solver, nccl_unique_id
ops = json.load(open(os.path.join(tmp, 'ops.json')))
arr = lambda name: np.load(os.path.join(tmp, name + '.npy'))
nid = None
if world > 1:
    idf = os.path.join(tmp, 'nccl_id')
    if rank == 0:
        nid = nccl_unique_id()
        open(idf + '.tmp', 'wb').write(nid); os.rename(idf + '.tmp', idf)
    else:
        t0 = time.time()
        while not os.path.exists(idf):
            time.sleep(0.02)
            assert time.time() - t0 < 120
        nid = open(idf, 'rb').read()
out = os.path.join(tmp, 'rank%d' % rank if world > 1 else 'single')
os.makedirs(out, exist_ok=True)
save = lambda tag, what, a: np.save(os.path.join(out, '%s.%s.npy' % (tag, what)), np.asarray(a))
s = Solver(arr('speed'), rank=rank, world_size=world, nccl_id=nid)
for op in ops:
    if 'ranks' in op and (world == 1 or rank not in op['ranks']):
        continue
    k = op['op']
    if k == 'load':
        s.load_nodes(arr(op['recs']))
    elif k == 'update':
        s.update_nodes(arr(op['idx']), arr(op['recs']))
    elif k == 'snapshot':
        s.snapshot()
    elif k == 'restore':
        s.restore()
    elif k == 'stage':
        s.stage_batch(arr(op['pods']), arr(op['now']))
    elif k in ('solve', 'staged'):
        if k == 'solve':
            b = s.solve_batch(arr(op['pods']), arr(op['now']))
        else:
            s.solve_staged(); s.sync(); b = s.fetch_bindings()
        t = s.timing()
        save(op['tag'], 'bind', b); save(op['tag'], 'final', s.read_nodes())
        save(op['tag'], 'launches', [t['n_launches'], t['n_types']])
    elif k == 'explain':
        counts = s.explain_batch()
        save(op['tag'], 'counts', counts)
        none = np.flatnonzero(counts.any(axis=1))[:3]
        save(op['tag'], 'why', np.stack([s.explain_pod(int(i)) for i in none]) if len(none) else np.zeros((0, s.n_nodes), np.uint8))
    elif k == 'query':
        save(op['tag'], 'query', s.query_batch(arr(op['pods']), arr(op['now'])))
    elif k == 'plan':
        b, c = s.plan_batch(arr(op['pods']), arr(op['now']), exclude=op.get('exclude', ()), explain=True)
        save(op['tag'], 'plan', b); save(op['tag'], 'plan_counts', c)
    else:
        raise ValueError(k)
s.close()
print('rank', rank, 'done')
'''


# ---------------------------------------------------------------- the hash of a hardware class, as the device computes it

def class_hash(rec):
    """``static_key`` of nhd_kernels.cuh on one wire record: the 64-bit hash of a node's static hardware description
    (bytes 64..127 of the record, then n_gpus, n_nics, n_numa and the SMT flag) and the 17-word key itself."""
    raw = np.ascontiguousarray(rec).tobytes()
    words = np.frombuffer(raw[64:128], dtype='<u4').tolist()
    c2 = np.frombuffer(raw[32:48], dtype='<u4').tolist()
    key = words + [(c2[0] >> 16) | ((c2[3] & 0xFF) << 16) | (((c2[3] >> 8) & wire.NODE_SMT) << 24)]
    h, m = 0x9E3779B97F4A7C15, (1 << 64) - 1
    for x in key:
        h ^= x
        h = (h * 0xff51afd7ed558ccd) & m
        h ^= h >> 29
    return h | 1, tuple(key)


def colliding_pair(recs):
    """Two nodes of different hardware classes whose hashes claim the same probe-0 slot of the class table, picked
    so that their classes differ in the NICs (the part of a class the sweep reads through its id)."""
    first = {}
    for i in range(len(recs)):
        h, key = class_hash(recs[i])
        first.setdefault(key, (i, h))
    by_slot = {}
    for key, (i, h) in first.items():
        by_slot.setdefault(h % CLASS_SLOTS, []).append(i)
    for nodes in by_slot.values():
        for a in nodes:
            for b in nodes:
                if a < b and recs[a]['n_nics'] != recs[b]['n_nics']:
                    return a, b
    return None


def test_class_hash_reproduces_the_class_count_of_a_cluster():
    """The helper is the device's hash: the classes it tells apart are exactly the distinct static descriptions."""
    recs, _ = workload.make_cluster(3, n_nodes=1800, wild=True)
    keys = {class_hash(r)[1] for r in recs}
    hashes = {class_hash(r)[0] for r in recs}
    assert len(keys) == len(hashes) > 200
    a, b = colliding_pair(recs)
    assert class_hash(recs[a])[0] % CLASS_SLOTS == class_hash(recs[b])[0] % CLASS_SLOTS
    assert class_hash(recs[a])[1] != class_hash(recs[b])[1]


# ---------------------------------------------------------------- runs

@pytest.fixture(scope='module')
def emu_env():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    try:
        import build_emu_cuda
    finally:
        sys.path.pop(0)
    lib = build_emu_cuda.build()
    nccl_dir = os.path.join(ROOT, 'tests', 'emu', 'fake_nccl')
    nccl, src = os.path.join(nccl_dir, 'libnccl.so.2'), os.path.join(nccl_dir, 'fake_nccl.c')
    if not os.path.exists(nccl) or os.path.getmtime(nccl) < os.path.getmtime(src):
        subprocess.run(['gcc', '-O2', '-fPIC', '-shared', '-w', '-Wl,-soname,libnccl.so.2', '-o', nccl, src, '-lrt'],
                       check=True)
    env = dict(os.environ, NHD_B200_LIB=lib, NHD_B200_ALLOW_EMULATED='1', EMU_LANE_ORDER='a')
    for k in ('NHD_SHARD_MIN_PAIRS', 'EMU_SCHED_SEED'):
        env.pop(k, None)
    return env


class Run:
    """One list of operations: arrays by name, the operations, and what the ranks and the oracle made of them."""

    def __init__(self, tmp, speed):
        self.tmp, self.ops, self.arrays, self.n_nodes = str(tmp), [], {}, 0
        self.put('speed', speed)

    def put(self, name, a):
        self.arrays[name] = a
        np.save(os.path.join(self.tmp, name + '.npy'), a)
        return name

    def op(self, op, **kw):
        self.ops.append(dict(op=op, n_nodes=self.n_nodes, **kw))

    def load(self, name, recs, **kw):
        self.op('load', recs=self.put(name, recs), **kw)
        if 'ranks' not in kw:
            self.n_nodes = len(recs)

    def update(self, name, idx, recs, **kw):
        self.op('update', idx=self.put(name + '_idx', np.asarray(idx, dtype='<i4')), recs=self.put(name, recs), **kw)

    def pods(self, name, pods, now=None):
        now = np.full(len(pods), workload.NOW0) if now is None else now
        return dict(pods=self.put(name, pods), now=self.put(name + '_now', np.asarray(now, dtype='<f8')))

    def solve(self, tag, pods, now=None, launches=None):
        self.op('solve', tag=tag, launches=launches, **self.pods(tag + '_pods', pods, now))

    def launch(self, env, ranks):
        """``ranks``: one environment overlay per rank (lane order, schedule seed)."""
        json.dump(self.ops, open(os.path.join(self.tmp, 'ops.json'), 'w'))
        world = len(ranks)
        procs = [subprocess.Popen([sys.executable, '-c', WORKER, ROOT, self.tmp, str(r), str(world)], cwd=ROOT,
                                  env=dict(env, **ranks[r]), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
                 for r in range(world)]
        outs = [p.communicate(timeout=900)[0] for p in procs]
        for r, (p, o) in enumerate(zip(procs, outs)):
            assert p.returncode == 0, (r, o[-3000:])

    def result(self, who, tag, what):
        return np.load(os.path.join(self.tmp, who, '%s.%s.npy' % (tag, what)))

    def oracle(self, oracle_lib):
        """The common operations through the oracle: {tag: (bindings, final records)}."""
        speed, state, snap, staged, want = self.arrays['speed'], None, None, None, {}
        for op in self.ops:
            if 'ranks' in op:
                continue
            k = op['op']
            if k == 'load':
                state = self.arrays[op['recs']].copy()
            elif k == 'update':
                state = state.copy()
                state[self.arrays[op['idx']]] = self.arrays[op['recs']]
            elif k == 'snapshot':
                snap = state.copy()
            elif k == 'restore':
                state = snap.copy()
            elif k == 'stage':
                staged = (op['pods'], op['now'])
            elif k in ('solve', 'staged'):
                pods, now = (op['pods'], op['now']) if k == 'solve' else staged
                ob, state = oracle_lib.solve(state, speed, self.arrays[pods], self.arrays[now])
                want[op['tag']] = (ob, state)
        return want

    def check(self, oracle_lib, world, min_placed=1):
        """Every rank's bindings and final records against the oracle after every batch; every rank the same type
        count, and the expected launch count where the operation names one: 8 sharded (7 without direct-path
        tables, more than 32 pod types), 6 filtered whole (5); a sharded rank whose shard is empty (more ranks than
        super-tiles, or a last slot past the end) launches no filter."""
        placed = 0
        for tag, (ob, orecs) in self.oracle(oracle_lib).items():
            op = next(o for o in self.ops if o.get('tag') == tag)
            n_super = max(1, -(-op.get('n_nodes', 0) // SUPER_NODES))
            S = -(-n_super // world)
            types = set()
            for r in range(world):
                b = self.result('rank%d' % r, tag, 'bind')
                assert helpers.binding_bytes_equal(ob, b), (tag, 'rank', r, helpers.first_binding_diff(ob, b))
                assert self.result('rank%d' % r, tag, 'final').tobytes() == orecs.tobytes(), (tag, 'rank', r)
                launches, n_types = self.result('rank%d' % r, tag, 'launches').tolist()
                types.add(n_types)
                if op.get('launches') is not None:
                    assert launches == op['launches'] - (op['launches'] in (7, 8) and r * S >= n_super), (tag, r, launches)
            assert len(types) == 1, (tag, types)
            placed += int((ob['status'] == wire.PLACED).sum())
        assert placed >= min_placed


def _ranks(*orders, seeds=None):
    return [dict(EMU_LANE_ORDER=o, **({'EMU_SCHED_SEED': str(seeds[i])} if seeds else {})) for i, o in enumerate(orders)]


def many_types(n, seed=5):
    """``n`` pod records of pairwise different descriptors (so ``n`` pod types), drawn around config 3's catalogue."""
    base = workload.make_pod_types(3)
    rng = np.random.default_rng(seed)
    cand = base[rng.integers(0, len(base), size=8 * n)].copy()
    cand['hugepages_gb'] = rng.integers(0, 9, size=len(cand))
    cand['n_misc'] = rng.integers(1, 4, size=len(cand))
    cand['groups'][:, 0]['n_proc'] = rng.integers(1, 7, size=len(cand))
    _, first = np.unique(cand.view(np.uint8).reshape(len(cand), -1), axis=0, return_index=True)
    pods = cand[np.sort(first)[:n]]
    assert len(pods) == n
    return pods


# ---------------------------------------------------------------- a. rank-private numbering

@pytest.mark.parametrize('ranks', [
    _ranks('a', 'd'),
    _ranks('a', 'd', 'a'),
    _ranks('a', 'a', 'd', 'd', seeds=[1, 2, 3, 4]),
], ids=['2-opposite-lanes', '3-lanes-a-d-a', '4-schedule-seeds'])
def test_numbering_wild_cluster(emu_env, oracle_lib, tmp_path, ranks):
    """A heterogeneous cluster (hundreds of classes, many sharing a probe-0 slot) whose ranks claim the class slots
    in different orders: the ids differ between ranks, the bindings and records may not."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=300, wild=True)
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('b1', pods[:150], launches=8)
    run.solve('b2', pods[150:], launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), ranks)
    run.check(oracle_lib, len(ranks), min_placed=250)


def test_numbering_two_colliding_classes(emu_env, oracle_lib, tmp_path):
    """Two hardware classes whose hashes share a probe-0 slot, alternating node by node over both shards: with the
    lanes ascending on rank 0 the first class wins the slot, descending on rank 1 the second one does."""
    wild, speed = workload.make_cluster(3, n_nodes=1800, wild=True)
    pair = colliding_pair(wild)
    assert pair is not None, 'no two classes of the cluster share a probe-0 slot'
    a, b = pair
    recs = wild[np.where(np.arange(600) % 2 == 0, a, b)].copy()       # 3 super-tiles: shards of 2 and 1
    pods, now = workload.make_pods(3, 200)
    run = Run(tmp_path, speed)
    run.load('pair', recs)
    run.solve('b1', pods, launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd'))
    run.check(oracle_lib, 2, min_placed=100)


# ---------------------------------------------------------------- b. rank-private history

@pytest.mark.parametrize('history', ['other-cluster', 'update-and-back'])
def test_history_of_one_rank(emu_env, oracle_lib, tmp_path, history):
    """Rank 0 has seen hardware the others never did, so its class slots are taken differently: after a load of
    another heterogeneous cluster, or after updating nodes to other hardware and back before a common update brings
    new classes.  Two sharded batches, every rank equal to the oracle after each."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=300, wild=True)
    other, _ = workload.make_cluster(4, n_nodes=1800, seed=7, wild=True)
    run = Run(tmp_path, speed)
    if history == 'other-cluster':
        run.load('other', other, ranks=[0])
        run.load('c', recs)
    else:
        run.load('c', recs)
        idx = np.arange(0, 1800, 2)
        run.update('away', idx, other[idx], ranks=[0])
        run.update('back', idx, recs[idx], ranks=[0])
        newhw, _ = workload.make_cluster(3, n_nodes=1800, seed=11, wild=True)
        run.update('new', idx, newhw[idx])
    run.solve('b1', pods[:150], launches=8)
    run.solve('b2', pods[150:], launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'a'))
    run.check(oracle_lib, 2, min_placed=250)


# ---------------------------------------------------------------- c. shapes of the exchange

@pytest.mark.parametrize('world', [2, 3, 4])
def test_uneven_shards_and_many_types(emu_env, oracle_lib, tmp_path, world):
    """5 super-tiles (the last one partial) over 2, 3 and 4 ranks: shards that do not divide, and one empty shard
    on 4 ranks; one batch of 16 pod types, then one of 40 (no direct-path tables: one launch fewer)."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1100, n_pods=160, wild=True)
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('b16', pods, launches=8)
    run.solve('b40', many_types(40), launches=7)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks(*'adad'[:world]))
    run.check(oracle_lib, world, min_placed=150)


def test_tiny_clusters_and_batches(emu_env, oracle_lib, tmp_path):
    """One handle on 4 ranks, reloaded: 1 node, 63 nodes, 300 nodes (2 super-tiles: ranks 2 and 3 hold empty
    shards); a batch of no pods (no exchange) and one of a single pod."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=300, n_pods=120, wild=True)
    run = Run(tmp_path, speed)
    run.load('n1', recs[:1])
    run.solve('t1', pods[:20], launches=8)
    run.load('n63', recs[:63])
    run.solve('t63', pods[:60], launches=8)
    run.load('n300', recs)
    run.solve('t300', pods[:100], launches=8)
    run.solve('t0', pods[:0])
    run.solve('tone', pods[100:101], launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd', 'a', 'd'))
    run.check(oracle_lib, 4, min_placed=100)


def test_node_group_lists(emu_env, oracle_lib, tmp_path):
    """Config 5's pods name node groups: the group-name rows travel in the exchange with the type rows."""
    recs, speed, pods, now = workload.make_workload(5, n_nodes=1100, n_pods=200)
    assert len(np.unique(pods['group_mask'])) > 10
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('b1', pods, launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd', 'a'))
    run.check(oracle_lib, 3, min_placed=100)


def test_bitmaps_outside_shared_memory(emu_env, oracle_lib, tmp_path):
    """Enough pod types that the bitmap rows do not fit the sweep's shared memory (its ``sweep_kernel<false>``
    instance reads them from global memory)."""
    n_nodes, n_types = 8192, 240
    recs, speed = workload.make_cluster(4, n_nodes=n_nodes, wild=True)
    pods = many_types(n_types, seed=9)
    assert (n_types + 2) * (n_nodes // 64) * 8 > SMEM_OPTIN
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('b1', pods, launches=7)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd'))
    run.check(oracle_lib, 2, min_placed=100)


# ---------------------------------------------------------------- d. one long-lived sharded handle

def test_long_lived_handle(emu_env, oracle_lib, tmp_path):
    """Load, batch; an update that brings new hardware classes, batch; snapshot, batch, restore (the classes are
    taken again); one staged batch solved three times from the snapshot, as the benchmark repeats it; a reload at a
    smaller and then a larger size (other super-tile counts and slot sizes).  Ranks with opposite lane orders."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=400, wild=True)
    other, _ = workload.make_cluster(4, n_nodes=2000, seed=7, wild=True)
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('d1', pods[:80], launches=8)
    idx = np.arange(5, 1800, 3)
    run.update('newhw', idx, other[idx])
    run.solve('d2', pods[80:160], launches=8)
    run.op('snapshot')
    run.solve('d3', pods[160:240], launches=8)
    run.op('restore')
    run.op('stage', **run.pods('staged_pods', pods[240:400]))
    for i in range(3):
        run.op('restore')
        run.op('staged', tag='s%d' % i, launches=8)
    run.load('small', other[:700])
    run.solve('d5', pods[:120], launches=8)
    run.load('large', other)
    run.solve('d6', pods[120:300], launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd'))
    run.check(oracle_lib, 2, min_placed=500)
    for i in (1, 2):
        assert run.result('rank0', 's%d' % i, 'bind').tobytes() == run.result('rank0', 's0', 'bind').tobytes()


def test_sharding_threshold_on_one_handle(emu_env, oracle_lib, tmp_path):
    """``NHD_SHARD_MIN_PAIRS`` between the (node, type) pair counts of two batches: the batch with more pod types is
    filtered in shards and exchanged (8 launches), the one with fewer is filtered whole on every rank (6)."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=300, wild=True)
    few = workload.make_pod_types(4)[np.arange(60) % 3]                 # 3 pod types: 5 400 pairs
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('many', pods[:150], launches=8)                            # 16 pod types: 28 800 pairs
    run.solve('few', few, launches=6)
    run.solve('many2', pods[150:], launches=8)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS=str(1800 * 8)), _ranks('a', 'd'))
    run.check(oracle_lib, 2, min_placed=200)


# ---------------------------------------------------------------- e. rank-local calls after a sharded batch

def test_rank_local_calls_after_a_sharded_batch(emu_env, oracle_lib, tmp_path):
    """Explanations, placement queries and plans run on each rank alone, on that rank's replica: after a sharded
    batch (different claim orders on the two ranks) every rank answers what a single-rank handle given the same
    records and batch answers."""
    recs, speed, pods, now = workload.make_workload(4, n_nodes=1800, n_pods=500, wild=True)
    run = Run(tmp_path, speed)
    run.load('c', recs)
    run.solve('b0', pods[:300], launches=8)
    run.op('snapshot')
    second = pods[300:500].copy()
    second['hugepages_gb'][::10] = 256                                    # more than any node has: no node for these
    run.solve('b1', second, launches=8)
    run.op('explain', tag='e')
    q = run.pods('qpods', pods[:64])
    run.op('query', tag='q', **q)
    run.op('plan', tag='p', exclude=list(range(0, 1800, 7)), **q)
    run.launch(dict(emu_env, NHD_SHARD_MIN_PAIRS='1'), _ranks('a', 'd'))
    run.check(oracle_lib, 2, min_placed=200)
    run.launch(emu_env, [dict(EMU_LANE_ORDER='a')])                  # the same operations on one rank
    assert run.result('single', 'e', 'counts').any(), 'no pod of the second batch went unplaced'
    for what in (('e', 'counts'), ('e', 'why'), ('q', 'query'), ('p', 'plan'), ('p', 'plan_counts')):
        want = run.result('single', *what)
        for r in range(2):
            assert run.result('rank%d' % r, *what).tobytes() == want.tobytes(), (what, r)
