"""ProMP on the 2-D point mass, H100-native path.  Same config keys / defaults as the reference's
run_scripts/pro-mp_run_point_mass.py:95-127; `--config_file` takes the same JSON.  `--graph` replays the device part
of every meta-iteration as one CUDA graph."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200.baselines import LinearFeatureBaseline, LinearTimeBaseline  # noqa: E402,F401
from promp_b200.envs import MetaPointEnvCorner, HalfCheetahRandDirecEnv, normalize  # noqa: E402,F401
from promp_b200.meta_algos import ProMP  # noqa: E402
from promp_b200.meta_trainer import Trainer  # noqa: E402
from promp_b200.policies import MetaGaussianMLPPolicy  # noqa: E402
from promp_b200.samplers import MetaSampler, MetaSampleProcessor  # noqa: E402
from promp_b200.utils import set_seed  # noqa: E402

DEFAULTS = {
    'seed': 1, 'baseline': 'LinearFeatureBaseline', 'env': 'MetaPointEnvCorner',
    'rollouts_per_meta_task': 20, 'max_path_length': 100, 'parallel': True,
    'discount': 0.99, 'gae_lambda': 1, 'normalize_adv': True,
    'hidden_sizes': (64, 64), 'learn_std': True,
    'inner_lr': 0.1, 'learning_rate': 1e-3, 'num_promp_steps': 5, 'clip_eps': 0.3, 'target_inner_step': 0.01,
    'init_inner_kl_penalty': 5e-4, 'adaptive_inner_kl_penalty': False, 'n_itr': 1001, 'meta_batch_size': 40,
    'num_inner_grad_steps': 1,
}


def main(config, use_cuda_graph=False):
    set_seed(config['seed'])
    baseline = globals()[config['baseline']]()
    env = normalize(globals()[config['env']]())
    policy = MetaGaussianMLPPolicy(name="meta-policy", obs_dim=np.prod(env.observation_space.shape),
                                   action_dim=np.prod(env.action_space.shape), meta_batch_size=config['meta_batch_size'],
                                   hidden_sizes=config['hidden_sizes'])
    sampler = MetaSampler(env=env, policy=policy, rollouts_per_meta_task=config['rollouts_per_meta_task'],
                          meta_batch_size=config['meta_batch_size'], max_path_length=config['max_path_length'],
                          parallel=config['parallel'])
    sample_processor = MetaSampleProcessor(baseline=baseline, discount=config['discount'], gae_lambda=config['gae_lambda'],
                                           normalize_adv=config['normalize_adv'])
    algo = ProMP(policy=policy, inner_lr=config['inner_lr'], meta_batch_size=config['meta_batch_size'],
                 num_inner_grad_steps=config['num_inner_grad_steps'], learning_rate=config['learning_rate'],
                 num_ppo_steps=config['num_promp_steps'], clip_eps=config['clip_eps'],
                 target_inner_step=config['target_inner_step'], init_inner_kl_penalty=config['init_inner_kl_penalty'],
                 adaptive_inner_kl_penalty=config['adaptive_inner_kl_penalty'])
    Trainer(algo=algo, policy=policy, env=env, sampler=sampler, sample_processor=sample_processor, n_itr=config['n_itr'],
            num_inner_grad_steps=config['num_inner_grad_steps'], use_cuda_graph=use_cuda_graph).train()


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description='ProMP: Proximal Meta-Policy Search (promp_b200)')
    ap.add_argument('--config_file', type=str, default='')
    ap.add_argument('--n_itr', type=int, default=None)
    ap.add_argument('--env', type=str, default=None, help='MetaPointEnvCorner | HalfCheetahRandDirecEnv (surrogate)')
    ap.add_argument('--graph', action='store_true')
    args = ap.parse_args()
    cfg = dict(DEFAULTS)
    if args.config_file:
        with open(args.config_file) as f:
            cfg.update(json.load(f))
    if args.n_itr is not None:
        cfg['n_itr'] = args.n_itr
    if args.env is not None:
        cfg['env'] = args.env
    main(cfg, use_cuda_graph=args.graph)
