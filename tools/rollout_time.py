"""Time promp_rollout in isolation and, with a -DPROMP_EXP_CLOCKS build (PROMP_B200_LIB=...), print the per-phase clock
breakdown of one warp.  usage: python tools/rollout_time.py [point|cheetah]"""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402
import bench  # noqa: E402


def main():
    wl_name = sys.argv[1] if len(sys.argv) > 1 else 'point'
    wl = bench.WORKLOADS[wl_name]
    np.random.seed(1)
    tr = bench.build_stack(wl, 'device', None)
    sampler = tr.sampler
    sampler.update_tasks()
    tr.policy.switch_to_pre_update()
    from promp_b200.samplers.device_data import PhaseData
    ph = PhaseData(sampler.meta_batch_size, sampler.envs_per_task, sampler.max_path_length, tr.policy.obs_dim, tr.policy.action_dim,
                   sampler.device)

    def run():
        sampler.rollout_into(ph)
    for _ in range(5):
        run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        run()
    b.record()
    torch.cuda.synchronize()
    print('%s rollout (+counter_add) %.1f us per phase' % (wl_name, a.elapsed_time(b) / 20 * 1e3))
    lib = _lib.load()
    if hasattr(lib, 'promp_debug_rollout_clocks'):
        buf = (ctypes.c_ulonglong * 16)()
        lib.promp_debug_rollout_clocks(buf, 1)
        n = 10
        for _ in range(n):
            run()
        lib.promp_debug_rollout_clocks(buf, 1)
        names = ['prologue (weights -> registers, reset)', 'noise chunk + flush chunk', 'layer 0 + tanh + stage obs + syncwarp', 'layer 1 (64x64, registers)',
                 'tanh + layer 2 + warp_sum', 'sample + stage act/mean', 'env step', 'syncwarp + observe + syncwarp']
        H = sampler.max_path_length
        tot = sum(buf[i] for i in range(8))
        print('  warp 0 clocks per launch %.0f (%.0f per env step):' % (tot / n, tot / n / H))
        for i, nm in enumerate(names):
            print('    %-44s %9.0f clk  %5.1f %%  (%.0f / step)' % (nm, buf[i] / n, 100.0 * buf[i] / max(tot, 1), buf[i] / n / H))


if __name__ == '__main__':
    main()
