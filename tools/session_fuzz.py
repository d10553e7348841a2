"""Long-lived handle sessions over many seeds (tests/test_handle_session.py's generator and runner): one handle
through loads, updates, snapshots, restores, batches, queries, plans, scenario calls and explanations, every call
compared with a fresh handle and the oracle.  Developer tool.

    python tools/session_fuzz.py [first_seed] [n_seeds] [n_steps] [kinds]

``kinds``: ``all`` (the default: every op, the forecasts included), ``basic`` (the ops of the sessions before the
forecasts, as ``make_session``'s default) or a comma-separated list of ops.

Runs on the CPU-emulated device (tests/emu) unless NHD_B200_LIB is unset and a CUDA device exists, in which case it
runs on the GPU.  Environment: EMU_SCHED_SEED=<n> shuffles the emulated warp schedule, EMU_LANE_ORDER=a|d sets the
emulated lane order (default d).  Prints seed / step / op of every mismatch.
"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _on_gpu():
    if os.environ.get('NHD_B200_LIB'):
        return False
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


if not _on_gpu():
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'emu'))
    import build_emu_cuda                                                 # noqa: E402
    os.environ['NHD_B200_LIB'] = os.environ.get('NHD_B200_LIB') or build_emu_cuda.build()
    os.environ['NHD_B200_ALLOW_EMULATED'] = '1'
    os.environ.setdefault('EMU_LANE_ORDER', 'd')

from tests.test_handle_session import (BASIC, EMU_SIZES, FORECASTS, MODES, SIZES, Mismatch,  # noqa: E402
                                       make_session, new_stats, run_session)


def main():
    first = int(sys.argv[1]) if len(sys.argv) > 1 else 0
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 200
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 30
    arg = sys.argv[4] if len(sys.argv) > 4 else 'all'
    kinds = {'all': BASIC + FORECASTS, 'basic': BASIC}.get(arg) or tuple(arg.split(','))
    sizes = EMU_SIZES if os.environ.get('NHD_B200_ALLOW_EMULATED') == '1' else SIZES
    bad = 0
    stats = new_stats()
    t0 = time.time()
    for seed in range(first, first + n):
        try:
            run_session(make_session(seed, steps, sizes, kinds), MODES[seed % len(MODES)], stats)
        except Mismatch as e:
            bad += 1
            print('MISMATCH', e, flush=True)
    print(f"{n} sessions, {stats['calls']} calls, {stats['bindings']} bindings compared, {bad} mismatches, "
          f'{time.time() - t0:.0f} s')
    print('ops', stats['ops'])
    print('refused by rule', stats['rules'], '/ reason rows', stats['rows'], '/ placed at a later round', stats['later'],
          '/ on added nodes', stats['on_added'], '/ cuts', stats['cuts'])


if __name__ == '__main__':
    main()
