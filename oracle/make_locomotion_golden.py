"""Generate tests/golden/locomotion_tasks.npz: the task draws of the UNMODIFIED reference Walker2d / Swimmer envs.

Like oracle/make_golden.py this imports the reference modules from where they lie (PROMP_REFERENCE_DIR, by default
../reference next to this repository) with the stub packages of oracle/stubs standing in for gym.  Only
`sample_tasks` is called (the MuJoCo constructor is never run), under fixed seeds, followed by a probe of the global
numpy stream so that the number of draws is pinned too.  Nothing from the reference is copied.

    python oracle/make_locomotion_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get('PROMP_REFERENCE_DIR', os.path.join(os.path.dirname(ROOT), 'reference'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'locomotion_tasks.npz')

CASES = (('walker2d_rand_vel', 'Walker2DRandVelEnv'), ('walker2d_rand_direc', 'Walker2DRandDirecEnv'),
         ('swimmer_rand_vel', 'SwimmerRandVelEnv'))
SEEDS = (0, 7, 123)
N_TASKS = (1, 5, 40)


def main():
    if not os.path.isdir(REF):
        raise SystemExit("reference tree %s not present (set PROMP_REFERENCE_DIR)" % REF)
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'stubs'))
    sys.path.insert(0, REF)
    import importlib
    out = {}
    for mod, cls in CASES:
        klass = getattr(importlib.import_module('meta_policy_search.envs.mujoco_envs.' + mod), cls)
        for seed in SEEDS:
            for n in N_TASKS:
                np.random.seed(seed)
                out['%s_s%d_n%d' % (cls, seed, n)] = np.asarray(klass.sample_tasks(None, n), dtype=np.float64)
                out['%s_s%d_n%d_probe' % (cls, seed, n)] = np.random.uniform(size=3)
    np.savez(OUT, **out)
    print("wrote %s (%d arrays)" % (OUT, len(out)))


if __name__ == '__main__':
    main()
