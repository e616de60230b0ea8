"""Write tests/golden/tf_half_depth.npz: what the reference's UNMODIFIED graph code computes for policies with one and three
hidden layers (MetaGaussianMLPPolicy(hidden_sizes=(64,)), (32,), (64, 64, 64), (32, 16, 8))).

Runs policies/*, meta_algos/{base,pro_mp,trpo_maml}.py and optimizers/* from the reference checkout on the torch-backed
`tensorflow` stand-in of oracle/stubs_tf, as tools/make_otanh_golden.py does.  The cases are made here (seeded, not
stored): theta with Xavier-uniform kernels in the reference's variable order, two sampling phases of M tasks x N samples
each, old means from a numpy forward of a drifted theta.  The graph is evaluated in float64.  Stored per case under
'<case>/': the inputs (theta, obs, act, adv, mean, log_std per phase), the inner adapt step (theta' - theta for every task),
and for ProMP the meta objective, inner / outer KL, the second-order meta-gradient and theta after ONE step of the
reference's Adam train op; for TRPO-MAML the objective gradient and the KL gradient.  Vectors are stored as float32.

Needs a checkout of jonasrothfuss/ProMP (commit 93ae339): PROMP_REFERENCE_DIR, by default ../reference next to this
repository.

    python tools/make_depth_golden.py
"""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402

# name: (algo, M, N, Do, Da, hidden_sizes)
CASES = {
    'promp_d1_h64': ('promp', 3, 150, 2, 2, (64,)),
    'promp_d1_h32': ('promp', 3, 130, 17, 6, (32,)),
    'promp_d3_h64': ('promp', 3, 140, 2, 2, (64, 64, 64)),
    'promp_d3_uneven': ('promp', 3, 120, 5, 3, (32, 16, 8)),
    'trpo_d1_h64': ('trpo', 3, 150, 2, 2, (64,)),
    'trpo_d3_uneven': ('trpo', 3, 120, 5, 3, (32, 16, 8)),
}
HYPER = dict(inner_lr=0.1, learning_rate=1e-3, num_ppo_steps=1, clip_eps=0.3, init_inner_kl_penalty=5e-4, step_size=0.01)
OUT = os.path.join(ROOT, 'tests', 'golden', 'tf_half_depth.npz')


def shapes(Do, Da, sizes):
    ins = (Do,) + tuple(sizes)
    out = []
    for i in range(len(sizes)):
        out += [('mean_network/hidden_%d/kernel' % i, (ins[i], ins[i + 1])), ('mean_network/hidden_%d/bias' % i, (ins[i + 1],))]
    return out + [('mean_network/output/kernel', (sizes[-1], Da)), ('mean_network/output/bias', (Da,)),
                  ('log_std_network/log_std_var', (1, Da))]


def unflatten(theta, Do, Da, sizes):
    from collections import OrderedDict
    out, off = OrderedDict(), 0
    for k, shp in shapes(Do, Da, sizes):
        n = int(np.prod(shp))
        out[k] = theta[off:off + n].reshape(shp)
        off += n
    return out


def make_case(name):
    algo, M, N, Do, Da, sizes = CASES[name]
    rng = np.random.RandomState(sum(map(ord, name)) * 7 + 1)
    theta = []
    for k, shp in shapes(Do, Da, sizes):
        if k.endswith('kernel'):
            lim = math.sqrt(6.0 / (shp[0] + shp[1]))
            theta.append(rng.uniform(-lim, lim, size=shp).reshape(-1))
        elif k.endswith('bias'):
            theta.append(0.1 * rng.randn(*shp).reshape(-1))
        else:
            theta.append(-0.3 + 0.2 * rng.randn(*shp).reshape(-1))
    theta = np.concatenate(theta).astype(np.float32)
    phases = []
    for s in range(2):
        obs = (rng.randn(M, N, Do) * 1.2).astype(np.float32)
        mean = np.zeros((M, N, Da), np.float32)
        log_std = np.zeros((M, Da), np.float32)
        for m in range(M):
            p = list(unflatten(theta + (0.01 * rng.randn(theta.size)).astype(np.float32), Do, Da, sizes).values())
            h = obs[m]
            for i in range(len(sizes)):
                h = np.tanh(h @ p[2 * i] + p[2 * i + 1])
            mean[m], log_std[m] = h @ p[-3] + p[-2], p[-1].reshape(-1)
        act = (mean + np.exp(log_std)[:, None, :] * rng.randn(M, N, Da)).astype(np.float32)
        adv = rng.randn(M, N)
        adv = ((adv - adv.mean(1, keepdims=True)) / (adv.std(1, keepdims=True) + 1e-8)).astype(np.float32)
        phases.append(dict(obs=obs, act=act, adv=adv, mean=mean, log_std=log_std))
    return dict(name=name, algo=algo, M=M, N=N, Do=Do, Da=Da, sizes=sizes, theta=theta, phases=phases)


def reference_samples(case):
    out = []
    for ph in case['phases']:
        N = ph['obs'].shape[1]
        out.append([dict(observations=ph['obs'][m], actions=ph['act'][m], advantages=ph['adv'][m],
                         adj_avg_rewards=np.zeros(N, np.float32),
                         agent_infos=dict(mean=ph['mean'][m], log_std=np.tile(ph['log_std'][m][None], (N, 1))))
                    for m in range(case['M'])])
    return out


def _build(case, torch_dtype):
    import tensorflow as tf
    from meta_policy_search.policies.meta_gaussian_mlp_policy import MetaGaussianMLPPolicy
    from meta_policy_search.meta_algos.pro_mp import ProMP
    from meta_policy_search.meta_algos.trpo_maml import TRPOMAML
    H = HYPER
    tf.reset_default_graph()
    tf.set_compute_dtype(torch_dtype)
    M = case['M']
    policy = MetaGaussianMLPPolicy(name='meta-policy', obs_dim=case['Do'], action_dim=case['Da'], meta_batch_size=M,
                                   hidden_sizes=case['sizes'])
    if case['algo'] == 'promp':
        algo = ProMP(policy=policy, inner_lr=H['inner_lr'], meta_batch_size=M, num_inner_grad_steps=1,
                     learning_rate=H['learning_rate'], num_ppo_steps=H['num_ppo_steps'], clip_eps=H['clip_eps'],
                     target_inner_step=0.01, init_inner_kl_penalty=H['init_inner_kl_penalty'], adaptive_inner_kl_penalty=False)
    else:
        algo = TRPOMAML(policy=policy, step_size=H['step_size'], inner_type='likelihood_ratio', inner_lr=H['inner_lr'],
                        meta_batch_size=M, num_inner_grad_steps=1)
    sess = tf.Session()
    sess.__enter__()
    uninit = [v for v in tf.global_variables() if not sess.run(tf.is_variable_initialized(v))]
    sess.run(tf.variables_initializer(uninit))
    policy.set_params(unflatten(case['theta'], case['Do'], case['Da'], case['sizes']))
    return tf, sess, policy, algo


def main():
    import torch
    torch.set_num_threads(1)
    make_golden._import_reference()
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'stubs_tf'))
    make_golden._np_cast_shim()
    out = {}
    flat = lambda od: np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in od.values()])    # noqa: E731
    for name in CASES:
        case = make_case(name)
        pre = name + '/'
        out[pre + 'theta'] = case['theta']
        for s, ph in enumerate(case['phases']):
            for k, v in ph.items():
                out[pre + 'phase%d_%s' % (s, k)] = v
        samples = reference_samples(case)
        tf, sess, policy, algo = _build(case, torch.float64)
        try:
            policy.switch_to_pre_update()
            algo._adapt(samples[0])
            out[pre + 'adapt_delta'] = (np.stack([flat(od) for od in policy.policies_params_vals])
                                        - case['theta'].astype(np.float64))
            inp = algo._extract_input_dict_meta_op(samples, algo._optimization_keys)
            params = list(policy.get_params().values())
            opt = algo.optimizer
            if case['algo'] == 'promp':
                inp['inner_kl_coeff'] = algo.inner_kl_coeff
                inp['clip_eps'] = algo.clip_eps
                feed = opt.create_feed_dict(inp)
                loss, ikl, okl, grads = sess.run([opt._loss, opt._inner_kl, opt._outer_kl, tf.gradients(opt._loss, params)], feed)
                out[pre + 'loss'], out[pre + 'inner_kl'], out[pre + 'outer_kl'] = (np.float64(loss), np.asarray(ikl, np.float64),
                                                                                  np.float64(okl))
                out[pre + 'grad'] = np.concatenate([np.asarray(g, np.float64).reshape(-1) for g in grads])
                sess.run(opt._train_op, feed)          # one Adam step of the reference's optimizer
                out[pre + 'adam_theta'] = flat(policy.get_param_values())
            else:
                out[pre + 'loss'] = np.float64(opt.loss(inp))
                out[pre + 'outer_kl'] = np.float64(opt.constraint_val(inp))
                out[pre + 'grad'] = np.asarray(opt.gradient(inp), np.float64)
                out[pre + 'kl_grad'] = np.asarray(opt._hvp_approach.constraint_gradient(inp), np.float64)
        finally:
            sess.__exit__(None, None, None)
        print('tf_half_depth', name, 'done', flush=True)
    out = {k: (np.asarray(v, np.float32) if np.ndim(v) >= 1 and np.asarray(v).dtype == np.float64 and np.size(v) > 8 else v)
           for k, v in out.items()}
    np.savez_compressed(OUT, **out)
    print(OUT)


if __name__ == '__main__':
    main()
