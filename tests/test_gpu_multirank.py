"""Multi-GPU parity on hardware: the world_size > 1 path of the C-ABI (node-sharded filter, one exchange per
batch, replicated sweep; NHDScheduler.py:235-247,277-304 semantics unchanged) against the C oracle.
Skipped on a one-GPU box; `gpurun --gpus 2 -- python -m pytest tests/test_gpu_multirank.py -m gpu` runs it."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize('world', [2, 4, 8])
def test_sharded_ranks_equal_the_oracle(oracle_lib, world):
    if os.environ.get('NHD_B200_ALLOW_EMULATED') == '1':
        pytest.skip('emulated device: tests/test_emulated_device.py::test_node_sharded_ranks_match_the_oracle covers it')
    if _n_gpus() < world:
        pytest.skip(f'needs {world} GPUs')
    port = 29500 + world
    res = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={world}',
                          '--master-addr', '127.0.0.1', '--master-port', str(port),
                          os.path.join(ROOT, 'tests', 'multirank_worker.py')],
                         cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    # six two-batch legs (tests/multirank_worker.py) and three staged re-solves
    assert res.stdout.count('equal to the oracle') == 9, res.stdout[-2000:]
