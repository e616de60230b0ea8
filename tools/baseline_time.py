"""Sample-processing time per phase for each kind of baseline, on one real sampling phase of each configuration:
  point    normalize(MetaPointEnvCorner), M x E x H = 40 x 20 x 100, obs_dim 2
  cheetah  normalize(HalfCheetahRandDirecEnv) surrogate, 40 x 20 x 200, obs_dim 17
  kernel   promp_process_samples with LinearFeatureBaseline (kind 1) and LinearTimeBaseline (kind 2): --iters launches
           captured in one CUDA graph (so no host launch overhead enters the number), CUDA events around its replay
           after --warmup eager launches, the two kinds alternated --reps times
  host     MetaSampleProcessor.process_phase with a baseline object that has no device kind (a numpy LinearTimeBaseline):
           ZERO pass, host copy, M host fits and E*M predicts, one upload, GIVEN pass; host clock around --host-iters
           synchronised phases
Prints the card name and power limit with the numbers.
usage: python tools/baseline_time.py [--iters 200] [--warmup 20] [--reps 3] [--host-iters 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CONFIGS = (('point', 'MetaPointEnvCorner', 40, 20, 100), ('cheetah', 'HalfCheetahRandDirecEnv', 40, 20, 200))


class NumpyTimeBaseline(object):
    """LinearTimeBaseline (baselines/linear_baseline.py:109-126) in numpy, without a device kind: runs on the host."""

    def __init__(self, reg_coeff=1e-5):
        self._coeffs, self._reg_coeff = None, reg_coeff

    @staticmethod
    def _features(path):
        t = np.arange(len(path['observations'])).reshape(-1, 1) / 100.0
        return np.concatenate([t, t ** 2, t ** 3, np.ones_like(t)], axis=1)

    def fit(self, paths, target_key='returns'):
        f = np.concatenate([self._features(p) for p in paths])
        y = np.concatenate([p[target_key] for p in paths])
        self._coeffs = np.linalg.lstsq(f.T.dot(f) + self._reg_coeff * np.identity(4), f.T.dot(y), rcond=-1)[0]

    def predict(self, path):
        return self._features(path).dot(self._coeffs)


def _phase(env_name, M, E, H):
    import torch
    from promp_b200 import envs
    from promp_b200.policies import MetaGaussianMLPPolicy
    from promp_b200.samplers import MetaSampler
    np.random.seed(1)
    torch.manual_seed(1)
    env = envs.normalize(getattr(envs, env_name)())
    policy = MetaGaussianMLPPolicy(name="p", obs_dim=int(np.prod(env.observation_space.shape)),
                                   action_dim=int(np.prod(env.action_space.shape)), meta_batch_size=M, hidden_sizes=(64, 64))
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=E, meta_batch_size=M, max_path_length=H)
    sampler.update_tasks()
    policy.switch_to_pre_update()
    return sampler.obtain_samples().phase


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--host-iters', type=int, default=5)
    args = ap.parse_args()
    import torch
    from promp_b200 import _lib
    from promp_b200.samplers import MetaSampleProcessor
    from promp_b200.samplers.meta_sample_processor import run_process_kernel
    _lib.require_cuda()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print('card: %s' % (card[0] if card else 'unknown'))
    for name, env_name, M, E, H in CONFIGS:
        phase = _phase(env_name, M, E, H)

        def launch(kind):
            run_process_kernel(phase, 0.99, 1.0, 1e-5, kind, True, False)

        times = {1: [], 2: []}
        for _ in range(args.reps):
            for kind in (1, 2):
                for _ in range(args.warmup):
                    launch(kind)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    for _ in range(args.iters):
                        launch(kind)
                graph.replay()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                graph.replay()
                b.record()
                torch.cuda.synchronize()
                times[kind].append(a.elapsed_time(b) / args.iters * 1e3)
                del graph
        for kind, label in ((1, 'linear-feature'), (2, 'linear-time')):
            print('%-8s %dx%dx%d kernel %-15s %s us per phase' % (name, M, E, H, label,
                                                                  ' '.join('%.1f' % t for t in times[kind])))
        proc = MetaSampleProcessor(NumpyTimeBaseline(), 0.99, 1.0, True, False)
        proc.process_phase(phase)
        torch.cuda.synchronize()
        wall = []
        for _ in range(args.host_iters):
            t0 = time.perf_counter()
            proc.process_phase(phase)
            torch.cuda.synchronize()
            wall.append((time.perf_counter() - t0) * 1e3)
        print('%-8s %dx%dx%d host baseline phase (wall) %s ms' % (name, M, E, H, ' '.join('%.2f' % t for t in wall)))


if __name__ == '__main__':
    main()
