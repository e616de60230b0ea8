"""Run a fixed, seeded matrix of calls to the env entry points of the library PROMP_B200_LIB selects and write every output
buffer to an .npz; or compare two such dumps byte for byte (uint8 views, so NaN payloads and untouched sentinel bytes
compare too).  A change to the env or rollout kernels that must not change results leaves every array identical.

    PROMP_B200_LIB=path/to/lib.so python tools/env_kernels_dump.py OUT.npz
    python tools/env_kernels_dump.py --compare A.npz B.npz

The matrix: promp_rollout for every kind it accepts with each valid reward_type (walker: task mode 0 / 1), hidden 32 / 64,
normalize_actions 0 / 1, init_state + noise fed or drawn in-kernel, param_stride 0 (with a device stream counter) or P,
M x E x H = 2 x 5 x 70 (a partial 4-warp CTA and a partial 32-step chunk); promp_rollout_early_term for the point env and
the walker with timeline_len = 2 * horizon - 1; promp_env_step chained over several steps (n_env = 300, H = 3: horizon
resets, the point env's done, fallen walkers); promp_env_observe; the argument errors of each entry point.
"""
import argparse
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from promp_b200 import _lib  # noqa: E402

L = _lib
KINDS = (L.ENV_POINT_CORNER, L.ENV_POINT, L.ENV_CHEETAH_DIR, L.ENV_POINT_WALLS, L.ENV_POINT_MOMENTUM, L.ENV_WALKER, L.ENV_SWIMMER)
DIMS = {L.ENV_POINT_CORNER: (2, 2), L.ENV_POINT: (2, 2), L.ENV_CHEETAH_DIR: (17, 6), L.ENV_POINT_WALLS: (2, 2),
        L.ENV_POINT_MOMENTUM: (4, 2), L.ENV_WALKER: (17, 6), L.ENV_SWIMMER: (8, 2)}       # (obs, action) size
ROLLOUT_REWARDS = {L.ENV_POINT_CORNER: (0, 1, 2), L.ENV_CHEETAH_DIR: (0, 1), L.ENV_POINT_WALLS: (1, 2),
                   L.ENV_POINT_MOMENTUM: (0, 1), L.ENV_WALKER: (0, 1), L.ENV_SWIMMER: (0,)}   # walker: the task's mode
STEP_REWARDS = {**ROLLOUT_REWARDS, L.ENV_POINT: (0,)}
M, E, H, RADIUS = 2, 5, 70, 0.8


def tasks(kind, n, rt, rng):
    if kind == L.ENV_POINT_CORNER:
        t = rng.uniform(-2, 2, (n, 2))
        t[::2] = (2.0, -2.0)                                   # corner goals take the sparse reward's exact-corner path
    elif kind == L.ENV_POINT_WALLS:
        t = np.concatenate([rng.uniform(-2, 2, (n, 2)), np.tile([[0.0, 1.0, 0.0, -2.0]], (n, 1))], 1)
    elif kind == L.ENV_POINT_MOMENTUM:
        t = rng.uniform(-0.5, 0.5, (n, 2))
    elif kind == L.ENV_WALKER:
        t = np.stack([rng.uniform(-1.5, 1.5, n), np.full(n, float(rt))], 1)
    elif kind == L.ENV_POINT:
        t = np.zeros((n, 1))
    else:
        t = rng.uniform(-2, 2, (n, 1))
    return t


def states(kind, n, rng):
    sd = L.load().promp_env_state_dim(kind)
    s = rng.normal(0, 0.1 if sd > 4 else 0.5, (n, sd))
    if kind == L.ENV_WALKER:
        s[:, 1] += 1.25
        s[: n // 8, 1] = 0.5                                   # fallen: done after the step
    if kind == L.ENV_POINT:
        s[: n // 8] = 0.004                                    # at the goal: done after a small step
    return s


class Runner:
    def __init__(self):
        import torch
        self.torch = torch
        self.lib = L.load()
        self.stream = torch.cuda.current_stream().cuda_stream
        self.out = {}

    def dev(self, a, dtype=None):
        t = self.torch
        return t.as_tensor(np.ascontiguousarray(a), dtype=dtype or t.float32, device='cuda')

    def buf(self, shape, dtype=None):
        t = self.torch
        if dtype == t.uint8:
            return t.full(shape, 0xAB, dtype=t.uint8, device='cuda')
        return t.full(shape, float('nan'), dtype=dtype or t.float32, device='cuda')   # sentinel for untouched elements

    def check(self, rc, what):
        if rc != 0:
            raise RuntimeError('%s: rc %d: %s' % (what, rc, L.last_error()))

    def save(self, name, **bufs):
        self.torch.cuda.synchronize()
        for k, v in bufs.items():
            self.out['%s/%s' % (name, k)] = v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)

    def params(self, kind, hidden, rng, log_std):
        do, da = DIMS[kind]
        P = self.lib.promp_num_params(do, da, hidden)
        th = rng.normal(0, 0.4, (M, P)).astype(np.float32)
        th[:, P - da:] = log_std + rng.uniform(-0.2, 0.2, (M, da))
        return self.dev(th), P

    def rollout(self, kind, rt, hidden, norm, fed, shared, early):
        rng = np.random.default_rng([kind, rt, hidden, norm, fed, shared, early])
        do, da = DIMS[kind]
        sd = self.lib.promp_env_state_dim(kind)
        hz = 36
        T = 2 * hz - 1 if early else H
        th, P = self.params(kind, hidden, rng, 0.3 if early else -0.5)
        task = self.dev(tasks(kind, M, rt, rng))
        init = self.dev(states(kind, M * E, rng)[rng.permutation(M * E)]) if fed else None
        noise = self.dev(rng.normal(0, 1, (M, E, T, da))) if fed else None
        ctr = self.dev(np.array([7], np.int64), self.torch.int64) if shared else None
        obs, act, mean = self.buf((M, E, T, do)), self.buf((M, E, T, da)), self.buf((M, E, T, da))
        rew, done, info = self.buf((M, E, T)), self.buf((M, E, T), self.torch.uint8), self.buf((3, M, E, T))
        ls, fs = self.buf((M, da)), self.buf((M, E, sd))
        p = lambda x: x.data_ptr() if x is not None else None   # noqa: E731
        seed, sid, stride = 1234 + kind, (5 << 32) + 11, 0 if shared else P
        if early:
            name = 'early_term/k%d_h%d_n%d_f%d_s%d' % (kind, hidden, norm, fed, shared)
            self.check(self.lib.promp_rollout_early_term(kind, norm, M, E, T, hz, hidden, p(th), stride, p(task), p(init), p(noise),
                                                         seed, sid, p(ctr), 1, -1.0, p(obs), p(act), p(mean), p(rew), p(done),
                                                         p(ls), self.stream), name)
            self.save(name, obs=obs, act=act, mean=mean, rew=rew, done=done, log_std=ls)
        else:
            name = 'rollout/k%d_r%d_h%d_n%d_f%d_s%d' % (kind, rt, hidden, norm, fed, shared)
            self.check(self.lib.promp_rollout(kind, 0 if kind == L.ENV_WALKER else rt, RADIUS, norm, M, E, T, hidden, p(th), stride,
                                              p(task), p(init), p(noise), seed, sid, p(ctr), 1, -1.0, p(obs), p(act), p(mean),
                                              p(rew), p(done), p(info), p(ls), p(fs), self.stream), name)
            self.save(name, obs=obs, act=act, mean=mean, rew=rew, done=done, info=info, log_std=ls, final_state=fs)
        return done

    def env_step(self, kind, rt, norm, n=300, steps=5):
        rng = np.random.default_rng([kind, rt, norm, 99])
        do, da = DIMS[kind]
        state = self.dev(states(kind, n, rng))
        ts = self.dev(rng.integers(0, 3, n), self.torch.int32)
        task = self.dev(tasks(kind, n, rt, rng))
        for s in range(steps):
            a = rng.normal(0, 1.5, (n, da))
            if kind == L.ENV_POINT:
                a[: n // 8] = 0.0
            reset = self.dev(states(kind, n, rng))
            nobs, rew, done = self.buf((n, do)), self.buf((n,)), self.buf((n,), self.torch.uint8)
            info = self.buf((3, n)) if norm == 0 else None    # both the info and the NULL-info path
            name = 'env_step/k%d_r%d_n%d/%d' % (kind, rt, norm, s)
            self.check(self.lib.promp_env_step(kind, rt, RADIUS, norm, n, 3, state.data_ptr(), ts.data_ptr(), self.dev(a).data_ptr(),
                                               task.data_ptr(), reset.data_ptr(), nobs.data_ptr(), rew.data_ptr(), done.data_ptr(),
                                               info.data_ptr() if info is not None else None, self.stream), name)
            self.save(name, next_obs=nobs, rew=rew, done=done, state=state.clone(), ts=ts.clone(),
                      **({'info': info} if info is not None else {}))

    def observe(self, kind, n=300):
        rng = np.random.default_rng([kind, 7])
        do = DIMS[kind][0]
        st, obs = self.dev(states(kind, n, rng) * 30.0), self.buf((n, do))     # * 30: the walker's velocity clip
        self.check(self.lib.promp_env_observe(kind, n, st.data_ptr(), obs.data_ptr(), self.stream), 'observe')
        self.save('observe/k%d' % kind, obs=obs)


def errors(lib):
    """Return codes and messages of rejected calls (host-side argument checks; no device work)."""
    x = ctypes.c_void_p(16)     # non-null placeholder; every call below is rejected before any launch
    rows = []
    for kind in (-1,) + KINDS + (7,):
        rows.append('dims %d: %d %d' % (kind, lib.promp_env_state_dim(kind), lib.promp_env_task_dim(kind)))
    rejected = [(-1, 0, x), (7, 0, x), (L.ENV_POINT, 0, x), (L.ENV_CHEETAH_DIR, 0, None), (L.ENV_CHEETAH_DIR, 2, x),
                (L.ENV_POINT_WALLS, 0, x), (L.ENV_SWIMMER, 0, None), (L.ENV_SWIMMER, 1, x), (L.ENV_POINT_CORNER, 3, x)]
    for kind, rt, info in rejected:
        rc = lib.promp_rollout(kind, rt, 0.5, 0, 1, 1, 1, 32, x, 0, x, None, None, 0, 0, None, 0, 0.0, x, x, x, x, x, info, x, None,
                               None)
        rows.append('rollout k%d r%d info%d: %d %s' % (kind, rt, info is not None, rc, L.last_error()))
    for kind in (-1, 0, 2, 3, 4, 6, 7):
        rc = lib.promp_rollout_early_term(kind, 0, 1, 1, 1, 1, 32, x, 0, x, None, None, 0, 0, None, 0, 0.0, x, x, x, x, x, x, None)
        rows.append('early_term k%d: %d %s' % (kind, rc, L.last_error()))
    for kind in (-1, 7):
        rc = lib.promp_env_step(kind, 0, 0.5, 0, 4, 3, x, x, x, x, x, x, x, x, None, None)
        rows.append('env_step k%d: %d %s' % (kind, rc, L.last_error()))
        rc = lib.promp_env_observe(kind, 4, x, x, None)
        rows.append('observe k%d: %d %s' % (kind, rc, L.last_error()))
    return np.array(rows)


def dump(path):
    lib = L.load()
    out = {'errors': errors(lib)}
    r = Runner()
    n_early = {}
    for kind, rts in ROLLOUT_REWARDS.items():
        for rt in rts:
            for hidden in (32, 64):
                for norm in (0, 1):
                    for fed in (0, 1):
                        for shared in (0, 1):
                            r.rollout(kind, rt, hidden, norm, fed, shared, early=False)
    for kind in L.EARLY_TERM_ENVS:
        for hidden in (32, 64):
            for norm in (0, 1):
                for fed in (0, 1):
                    done = r.rollout(kind, 0, hidden, norm, fed, fed, early=True)
                    n_early[kind] = n_early.get(kind, 0) + int(done.sum().item())
    for kind, rts in STEP_REWARDS.items():
        for rt in rts:
            for norm in (0, 1):
                r.env_step(kind, rt, norm)
    for kind in KINDS:
        r.observe(kind)
    out.update(r.out)
    np.savez(path, **out)
    print('%s: %d arrays, %d bytes from %s; path ends per early-term kind %s' % (
        path, len(out), sum(v.nbytes for v in out.values()), L.LIB_PATH, n_early))


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    bad = sorted(set(a.files) ^ set(b.files))
    for k in sorted(set(a.files) & set(b.files)):
        x, y = a[k], b[k]
        if x.dtype != y.dtype or x.shape != y.shape or not np.array_equal(x.view(np.uint8), y.view(np.uint8)):
            bad.append(k)
    print('%d arrays compared, %d differ%s' % (len(set(a.files) | set(b.files)), len(bad), ''.join('\n  ' + k for k in bad[:50])))
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out', nargs='?')
    ap.add_argument('--compare', nargs=2, metavar=('A', 'B'))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    dump(args.out)


if __name__ == '__main__':
    main()
