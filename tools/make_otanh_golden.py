"""Write tests/golden/tf_half_otanh.npz: what the reference's UNMODIFIED graph code computes for a policy with a tanh output
layer (MetaGaussianMLPPolicy(output_nonlinearity=tf.tanh)), with tanh and with ReLU hidden layers.

Runs policies/*, meta_algos/{base,pro_mp,trpo_maml,vpg_maml}.py and optimizers/* from the reference checkout on the
torch-backed `tensorflow` stand-in of oracle/stubs_tf, as tools/make_relu_golden.py does, but builds the policy with
output_nonlinearity=tf.tanh.  Inputs are the seeded cases of oracle/tf_cases.py (not stored).  The graph is evaluated in
float64.  Stored per (case, hidden activation), under '<case>/<activation>/f64/': the inner adapt step (the update
theta' - theta of the first and last task, and its norm for every task), the meta objective, inner / outer KL and the
second-order meta-gradient (ProMP, VPG-MAML), and for TRPO-MAML the objective gradient, the KL gradient and the
finite-difference Hessian-vector product of the KL along the normalised objective gradient.  Vectors are stored as float32.

Needs a checkout of jonasrothfuss/ProMP (commit 93ae339): PROMP_REFERENCE_DIR, by default ../reference next to this
repository.

    python tools/make_otanh_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402

# (hidden activation, case)
CASES = (('tanh', 'promp_small'), ('tanh', 'promp_cheetah'), ('tanh', 'promp_s3'), ('tanh', 'promp_h32'),
         ('tanh', 'trpo_small'), ('tanh', 'vpg_small'), ('relu', 'promp_small'), ('relu', 'vpg_small'))
OUT = os.path.join(ROOT, 'tests', 'golden', 'tf_half_otanh.npz')


def _build(case, act, torch_dtype):
    """The reference policy with a tanh output layer + the case's algorithm, parameters set to the case's theta."""
    import tensorflow as tf
    from oracle import tf_cases
    from meta_policy_search.policies.meta_gaussian_mlp_policy import MetaGaussianMLPPolicy
    from meta_policy_search.meta_algos.pro_mp import ProMP
    from meta_policy_search.meta_algos.trpo_maml import TRPOMAML
    from meta_policy_search.meta_algos.vpg_maml import VPGMAML
    H = tf_cases.HYPER
    tf.reset_default_graph()
    tf.set_compute_dtype(torch_dtype)
    M, S1 = case['M'], case['S'] - 1
    policy = MetaGaussianMLPPolicy(name='meta-policy', obs_dim=case['Do'], action_dim=case['Da'], meta_batch_size=M,
                                   hidden_sizes=(case['hidden'], case['hidden']),
                                   hidden_nonlinearity=tf.nn.relu if act == 'relu' else tf.tanh, output_nonlinearity=tf.tanh)
    if case['algo'] == 'promp':
        algo = ProMP(policy=policy, inner_lr=H['inner_lr'], meta_batch_size=M, num_inner_grad_steps=S1,
                     learning_rate=H['learning_rate'], num_ppo_steps=H['num_ppo_steps'], clip_eps=H['clip_eps'],
                     target_inner_step=0.01, init_inner_kl_penalty=H['init_inner_kl_penalty'], adaptive_inner_kl_penalty=False)
    elif case['algo'] == 'trpo':
        algo = TRPOMAML(policy=policy, step_size=H['step_size'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                        meta_batch_size=M, num_inner_grad_steps=S1, exploration=case.get('exploration', False))
    else:
        algo = VPGMAML(policy=policy, learning_rate=H['learning_rate'], inner_type=case['inner_type'], inner_lr=H['inner_lr'],
                       meta_batch_size=M, num_inner_grad_steps=S1, exploration=case.get('exploration', False))
    sess = tf.Session()
    sess.__enter__()
    uninit = [v for v in tf.global_variables() if not sess.run(tf.is_variable_initialized(v))]
    sess.run(tf.variables_initializer(uninit))
    policy.set_params(tf_cases.unflatten(case['theta'], case['Do'], case['Da'], case['hidden']))
    return tf, sess, policy, algo


def main():
    import torch
    torch.set_num_threads(1)
    make_golden._import_reference()
    sys.path.insert(0, os.path.join(ROOT, 'oracle', 'stubs_tf'))
    make_golden._np_cast_shim()
    from oracle import tf_cases
    out = {}
    flat = lambda od: np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in od.values()])
    for act, name in CASES:
        case = tf_cases.make_case(name)
        samples = tf_cases.reference_samples(case)
        keep = [0, case['M'] - 1]
        out[name + '/keep_tasks'] = np.asarray(keep)
        pre = '%s/%s/f64/' % (name, act)
        tf, sess, policy, algo = _build(case, act, torch.float64)
        try:
            policy.switch_to_pre_update()
            for s in range(case['S'] - 1):
                algo._adapt(samples[s])
                delta = np.stack([flat(od) for od in policy.policies_params_vals]) - case['theta'].astype(np.float64)
                out[pre + 'adapt%d_delta' % s] = delta[keep]
                out[pre + 'adapt%d_delta_norm' % s] = np.sqrt((delta ** 2).sum(1))
            inp = algo._extract_input_dict_meta_op(samples, algo._optimization_keys)
            params = list(policy.get_params().values())
            opt = algo.optimizer
            if case['algo'] == 'promp':
                inp['inner_kl_coeff'] = algo.inner_kl_coeff
                inp['clip_eps'] = algo.clip_eps
                feed = opt.create_feed_dict(inp)
                loss, ikl, okl, grads = sess.run([opt._loss, opt._inner_kl, opt._outer_kl, tf.gradients(opt._loss, params)], feed)
                out[pre + 'loss'], out[pre + 'inner_kl'], out[pre + 'outer_kl'] = np.float64(loss), np.asarray(ikl, np.float64), np.float64(okl)
                out[pre + 'grad'] = np.concatenate([np.asarray(g, np.float64).reshape(-1) for g in grads])
            elif case['algo'] == 'trpo':
                out[pre + 'loss'] = np.float64(opt.loss(inp))
                out[pre + 'outer_kl'] = np.float64(opt.constraint_val(inp))
                g = opt.gradient(inp)
                out[pre + 'grad'] = np.asarray(g, np.float64)
                out[pre + 'kl_grad'] = np.asarray(opt._hvp_approach.constraint_gradient(inp), np.float64)
                x = (g / (np.linalg.norm(g) + 1e-12)).astype(g.dtype)
                out[pre + 'hx'] = np.asarray(opt._hvp_approach.Hx(inp, x), np.float64)
            else:
                feed = opt.create_feed_dict(inp)
                loss, grads = sess.run([opt._loss, tf.gradients(opt._loss, params)], feed)
                out[pre + 'loss'] = np.float64(loss)
                out[pre + 'grad'] = np.concatenate([np.asarray(g, np.float64).reshape(-1) for g in grads])
        finally:
            sess.__exit__(None, None, None)
        print('tf_half_otanh', name, act, 'done', flush=True)
    out = {k: (np.asarray(v, np.float32) if np.ndim(v) >= 1 and np.asarray(v).dtype == np.float64 and np.size(v) > 8 else v)
           for k, v in out.items()}
    np.savez_compressed(OUT, **out)
    print(OUT)


if __name__ == '__main__':
    main()
