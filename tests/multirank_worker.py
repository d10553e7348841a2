"""One rank of the multi-GPU parity check (launched by tests/test_gpu_multirank.py with torch.distributed.run).

Every rank holds a replica of the cluster, filters its shard of the nodes, takes part in the one exchange of the
batch and runs the replicated sweep (nhd_api.cu: world_size > 1).  Rank 0 computes the C oracle's bindings and final
records and hands their digest to every rank; every rank compares the digest of its own results with it, and rank 0
names the first difference of its own."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _digest(bindings, final):
    h = hashlib.sha256()
    for n in bindings.dtype.names:
        if n != 'pad_':
            h.update(np.ascontiguousarray(bindings[n]).tobytes())
    h.update(final.tobytes())
    return h.digest()


def main():
    import torch
    import torch.distributed as dist
    import workload
    from nhd_b200.solver import Solver, nccl_unique_id
    from tests import helpers

    rank, local, world = int(os.environ['RANK']), int(os.environ['LOCAL_RANK']), int(os.environ['WORLD_SIZE'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    failures = []
    threads = max(1, os.cpu_count() or 1)

    def oracle(recs, speed, pods, now):
        from oracle import binding
        return binding.solve(recs, speed, pods, now, threads=threads)

    def compare(label, got, final, want):
        """got / final: this rank's; want: the oracle's (bindings, records) on rank 0, None elsewhere."""
        ref = torch.zeros(32, dtype=torch.uint8, device='cuda')
        if rank == 0:
            ref.copy_(torch.frombuffer(bytearray(_digest(*want)), dtype=torch.uint8))
        dist.broadcast(ref, 0)                                              # the oracle's digest, from rank 0
        mine = torch.frombuffer(bytearray(_digest(got, final)), dtype=torch.uint8).cuda()
        ok = bool((mine == ref).all())
        if not ok:
            failures.append(f'{label}: rank {rank} differs from the oracle')
        if rank == 0:
            ob, orecs = want
            if not helpers.binding_bytes_equal(ob, got):
                failures.append(f'{label}: bindings differ from the oracle: {helpers.first_binding_diff(ob, got)}')
        bad = torch.tensor([0 if ok else 1], device='cuda')
        dist.all_reduce(bad)
        if rank == 0:
            print(f'{label} on {world} ranks: '
                  f'{"equal to the oracle" if int(bad.item()) == 0 else "%d ranks differ" % int(bad.item())}', flush=True)

    def solver(speed):
        # one communicator per solver handle: a fresh NCCL unique id each time (they are single-use)
        idt = torch.zeros(128, dtype=torch.uint8, device='cuda')
        if rank == 0:
            idt.copy_(torch.frombuffer(bytearray(nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(idt, 0)
        return Solver(speed, device=local, rank=rank, world_size=world, nccl_id=bytes(idt.cpu().numpy().tobytes()))

    def threshold(min_pairs):
        os.environ.pop('NHD_SHARD_MIN_PAIRS', None)
        if min_pairs is not None:
            os.environ['NHD_SHARD_MIN_PAIRS'] = min_pairs          # read by nhd_create; the same on every rank

    # (config, nodes, pods, wild, NHD_SHARD_MIN_PAIRS, rank 0's history): the small clusters and the full config 4
    # (also its heterogeneous variant, whose ranks number thousands of colliding hardware classes each in their own
    # order) are forced onto the node-sharded path (filter shards + all-gather); config 4 also runs at the default
    # threshold, where every rank filters the whole cluster and no collective is entered.  'other cluster': rank 0
    # alone loads another heterogeneous cluster first, so its class ids differ from the other ranks' for certain.
    legs = ((3, 4096, 384, False, '1', None), (5, 8192, 512, False, '1', None), (4, None, None, False, '1', None),
            (4, None, None, False, None, None), (4, None, None, True, '1', None), (3, None, None, True, '1', 'other cluster'))
    for cfg, n_nodes, n_pods, wild, min_pairs, history in legs:
        threshold(min_pairs)
        recs, speed, pods, now = workload.make_workload(cfg, n_nodes, n_pods, wild=wild)
        s = solver(speed)
        try:
            if history and rank == 0:
                s.load_nodes(workload.make_cluster(cfg, seed=7, wild=True)[0])
            s.load_nodes(recs)
            b1 = s.solve_batch(pods[:len(pods) // 2], now[:len(pods) // 2])      # two batches: the second starts from
            b2 = s.solve_batch(pods[len(pods) // 2:], now[len(pods) // 2:])      # the state the first one committed
            final = s.read_nodes()
        finally:
            s.close()
        want = oracle(recs, speed, pods, now) if rank == 0 else None
        label = (f'config {cfg}{" wild" if wild else ""} ({"node-sharded" if min_pairs else "default threshold"}'
                 f'{", " + history + " on rank 0" if history else ""}): {len(recs)} nodes x {len(pods)} pods')
        compare(label, np.concatenate([b1, b2]), final, want)

    # staged re-solves, as the benchmark repeats them: one staged batch, then restore + solve_staged three times, each
    # from the snapshot
    threshold('1')
    recs, speed, pods, now = workload.make_workload(3, wild=True)
    s = solver(speed)
    try:
        s.load_nodes(recs)
        s.snapshot()
        s.stage_batch(pods, now)
        want = oracle(recs, speed, pods, now) if rank == 0 else None
        for i in range(3):
            s.restore()
            s.solve_staged()
            s.sync()
            compare(f'config 3 wild staged re-solve {i}: {len(recs)} nodes x {len(pods)} pods', s.fetch_bindings(),
                    s.read_nodes(), want)
    finally:
        s.close()
    threshold(None)

    bad = torch.tensor([len(failures)], device='cuda')
    dist.all_reduce(bad)
    dist.destroy_process_group()
    if failures:
        print('\n'.join(failures), flush=True)
    sys.exit(1 if int(bad.item()) else 0)


if __name__ == '__main__':
    main()
