"""Write tests/golden/tf_half_meta_sgd.npz: what the reference's UNMODIFIED graph code computes with trainable inner step sizes.

Runs policies/*, meta_algos/{base,pro_mp,vpg_maml}.py and optimizers/* from the reference checkout on the torch-backed
`tensorflow` stand-in of oracle/stubs_tf, as tools/make_relu_golden.py does, with trainable_inner_step_size=True.  The
step-size variables of `_create_step_size_vars` are set to a seeded non-uniform alpha = inner_lr * exp(U(-1/2, 1/2)) (one
value per parameter) and the meta objective is differentiated with respect to the policy variables and the step-size
variables (the var_list the first-order optimizer would take with the reference's TODO fixed).  Inputs are the seeded cases
of oracle/tf_cases.py (not stored).  The graph is evaluated in float64.  Stored per case: alpha (flat, the policy's key
order), the meta objective, and the theta- and alpha-gradients; vectors as float32.

Needs a checkout of jonasrothfuss/ProMP (commit 93ae339): PROMP_REFERENCE_DIR, by default ../reference next to this
repository.

    python tools/make_meta_sgd_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402

CASES = ('promp_small', 'promp_s3', 'vpg_small')
OUT = os.path.join(ROOT, 'tests', 'golden', 'tf_half_meta_sgd.npz')


def alpha_of(case, inner_lr):
    """The case's non-uniform step sizes, flat in the policy's key order (float32, as the reference's variables)."""
    from oracle import tf_half as th
    n = th.num_params(case['Do'], case['Da'], (case['hidden'],) * 2)
    rng = np.random.RandomState(4242 + case['M'] * 7 + case['S'])
    return (inner_lr * np.exp(rng.uniform(-0.5, 0.5, n))).astype(np.float32)


def main():
    import torch
    torch.set_num_threads(1)
    make_golden._import_reference()
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'stubs_tf'))
    make_golden._np_cast_shim()
    import tensorflow as tf
    from oracle import tf_cases
    from meta_policy_search.policies.meta_gaussian_mlp_policy import MetaGaussianMLPPolicy
    from meta_policy_search.meta_algos.pro_mp import ProMP
    from meta_policy_search.meta_algos.vpg_maml import VPGMAML
    H = tf_cases.HYPER
    out = {}
    flat = lambda vals: np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in vals])
    for name in CASES:
        case = tf_cases.make_case(name)
        samples = tf_cases.reference_samples(case)
        pre = name + '/f64/'
        tf.reset_default_graph()
        tf.set_compute_dtype(torch.float64)
        M, S1 = case['M'], case['S'] - 1
        policy = MetaGaussianMLPPolicy(name='meta-policy', obs_dim=case['Do'], action_dim=case['Da'], meta_batch_size=M,
                                       hidden_sizes=(case['hidden'], case['hidden']))
        if case['algo'] == 'promp':
            algo = ProMP(policy=policy, inner_lr=H['inner_lr'], meta_batch_size=M, num_inner_grad_steps=S1,
                         learning_rate=H['learning_rate'], num_ppo_steps=H['num_ppo_steps'], clip_eps=H['clip_eps'],
                         target_inner_step=0.01, init_inner_kl_penalty=H['init_inner_kl_penalty'],
                         adaptive_inner_kl_penalty=False, trainable_inner_step_size=True)
        else:
            algo = VPGMAML(policy=policy, learning_rate=H['learning_rate'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                           meta_batch_size=M, num_inner_grad_steps=S1, trainable_inner_step_size=True)
        sess = tf.Session()
        sess.__enter__()
        try:
            uninit = [v for v in tf.global_variables() if not sess.run(tf.is_variable_initialized(v))]
            sess.run(tf.variables_initializer(uninit))
            policy.set_params(tf_cases.unflatten(case['theta'], case['Do'], case['Da'], case['hidden']))
            keys = list(policy.get_params().keys())
            steps = [algo.step_sizes[k] for k in keys]
            alpha = alpha_of(case, H['inner_lr'])
            off = 0
            for v in steps:
                n = int(np.prod(v.shape))
                sess.run(tf.assign(v, alpha[off:off + n].reshape(tuple(v.shape))))
                off += n
            assert off == alpha.size
            inp = algo._extract_input_dict_meta_op(samples, algo._optimization_keys)
            params = [policy.get_params()[k] for k in keys]
            opt = algo.optimizer
            if case['algo'] == 'promp':
                inp['inner_kl_coeff'] = algo.inner_kl_coeff
                inp['clip_eps'] = algo.clip_eps
            feed = opt.create_feed_dict(inp)
            loss, g_theta, g_alpha = sess.run([opt._loss, tf.gradients(opt._loss, params), tf.gradients(opt._loss, steps)], feed)
            out[pre + 'alpha'] = alpha
            out[pre + 'loss'] = np.float64(loss)
            out[pre + 'grad'] = flat(g_theta)
            out[pre + 'grad_alpha'] = flat(g_alpha)
        finally:
            sess.__exit__(None, None, None)
        print('tf_half_meta_sgd', name, 'done', flush=True)
    out = {k: (np.asarray(v, np.float32) if np.ndim(v) >= 1 and np.asarray(v).dtype == np.float64 and np.size(v) > 8 else v)
           for k, v in out.items()}
    np.savez_compressed(OUT, **out)
    print(OUT)


if __name__ == '__main__':
    main()
