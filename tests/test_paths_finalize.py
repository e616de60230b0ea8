"""promp_paths_finalize (promp_b200/csrc/paths.cu): the device path table of early-terminating rollouts against a plain
statement of the reference's collect-until-enough rule (meta_sampler.py:87-137).

CPU part: `collect_until`, the rule applied to recorded `done` timelines, against the reference loop
(oracle.numpy_half.Sampler driven by a scripted env); the premise that 2H-1 recorded steps always reach M*E*H samples;
the entry point's argument checks.
GPU part (pytest -m gpu): the four kernels on seeded synthetic timelines at the edges of their index arithmetic (one warp
or many, one 1024-step scan chunk or several, a table filled to max_paths or not), one workspace reused across calls,
tables truncated at max_paths, and two consecutive long-horizon phases through MetaSampler(reset_mode='device').
"""
import itertools
from collections import namedtuple

import numpy as np
import pytest

Rule = namedtuple('Rule', 'paths t_star reached')

POISON_I = -123456789               # int32 outputs
POISON_F = 0x7FC0DEAD               # float32 outputs: a NaN bit pattern no copied sample can have
POISON_U8 = 0xA5                    # the compacted done flags


def collect_until(done, target, max_paths=None):
    """The reference's sampling rule on recorded timelines done [M, E, T]: step every env; at the step a path completes,
    append it to its task's list (env index order within a step, meta_sampler.py:116-125); stop after the first step at
    which the completed paths hold >= target samples; drop unfinished paths.

    Returns Rule(paths, t_star, reached): paths[m] is an int64 array [n, 3] of (slot, start, length) rows in the rule's
    order; t_star is the step the rule stopped at (T-1 if the target is never reached, with every completed path kept).
    With max_paths, a task keeps only its first max_paths paths (promp_paths_finalize's truncation); t_star and reached
    still describe where the rule stopped."""
    done = np.asarray(done, dtype=bool)
    M, E, T = done.shape
    start = np.zeros((M, E), dtype=np.int64)
    rows, n, t_star, reached = [], 0, T - 1, False
    for t in range(T):
        m, e = np.nonzero(done[:, :, t])            # row-major: task, then env index
        if len(m):
            s = start[m, e]
            rows.append(np.stack([m, e, s, t + 1 - s], 1))
            n += int((t + 1 - s).sum())
            start[m, e] = t + 1
        if n >= target:
            t_star, reached = t, True
            break
    allr = np.concatenate(rows) if rows else np.zeros((0, 4), dtype=np.int64)
    allr = allr[np.argsort(allr[:, 0], kind='stable')]          # per task, keeping the (step, env) order
    bounds = np.searchsorted(allr[:, 0], np.arange(M + 1))
    paths = [allr[bounds[m]:bounds[m + 1], 1:][:max_paths] for m in range(M)]
    return Rule(paths, t_star, reached)


def horizon_timeline(rng, M, E, T, H, p):
    """done [M, E, T] whose paths all end at the horizon H or earlier: each step ends the running path with probability p,
    and a path that reaches H steps ends there."""
    done = rng.random_sample((M, E, T)) < p
    run = np.zeros((M, E), dtype=np.int64)
    for t in range(T):
        run += 1
        d = done[:, :, t] | (run >= H)
        done[:, :, t] = d
        run[d] = 0
    return done


def ragged_rows(paths_m, T):
    """Path offsets of one task's rule result and, for every kept sample, its row (slot*T + step) in the task's timeline."""
    lens = paths_m[:, 2]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    k = np.repeat(np.arange(len(lens)), lens)
    src = paths_m[k, 0] * T + paths_m[k, 1] + (np.arange(off[-1]) - off[k])
    return off, src


# ================================================================================================================ CPU
class _ScriptedEnv(object):
    """Replays a done timeline [M*E, T] for one env slot; the observation is (slot, step), so every sampled path names
    where it came from.  The iterative executor deep-copies the env once per slot, in slot order."""

    def __init__(self, done, counter):
        self.done, self.counter, self.slot, self.t = done, counter, None, 0

    def __deepcopy__(self, memo):
        env = _ScriptedEnv(self.done, self.counter)
        env.slot = next(self.counter)
        return env

    def sample_tasks(self, n):
        return list(range(n))

    def set_task(self, task):
        self.task = task

    def reset(self):
        return np.array([self.slot, self.t], dtype=np.float64)

    def step(self, action):
        d = bool(self.done[self.slot, self.t])
        self.t += 1
        return np.array([self.slot, self.t], dtype=np.float64), float(self.t), d, {}


class _ZeroPolicy(object):
    def get_actions(self, obs_per_task):
        return [np.zeros((len(o), 1)) for o in obs_per_task], [[{} for _ in o] for o in obs_per_task]


@pytest.mark.parametrize('M,E,H,p,seed', [(1, 1, 4, 0.3, 0), (2, 3, 5, 0.0, 1), (2, 3, 5, 1.0, 2), (3, 4, 7, 0.1, 3),
                                          (2, 5, 6, 0.3, 4), (4, 2, 9, 0.5, 5)])
def test_collect_until_matches_reference_loop(M, E, H, p, seed):
    """collect_until(done, M*E*H) lists the same paths, in the same order, as the reference loop (oracle.numpy_half.Sampler,
    iterative executor) stepping envs that replay `done`; p = 0: every path runs to the horizon, p = 1: one-step paths."""
    from oracle import numpy_half as nh
    T = 2 * H - 1
    done = horizon_timeline(np.random.RandomState(seed), M, E, T, H, p)
    sampler = nh.Sampler(_ScriptedEnv(done.reshape(M * E, T), itertools.count()), _ZeroPolicy(), E, M, H)
    sampler.update_tasks()
    got = sampler.obtain_samples()
    rule = collect_until(done, M * E * H)
    assert rule.reached
    for m in range(M):
        have = []
        for path in got[m]:
            o = path['observations']
            slot, s0, L = int(o[0, 0]), int(o[0, 1]), len(path['rewards'])
            np.testing.assert_array_equal(o[:, 0], slot)
            np.testing.assert_array_equal(o[:, 1], np.arange(s0, s0 + L))
            have.append((slot - m * E, s0, L))
        assert have == [tuple(r) for r in rule.paths[m].tolist()], m
    # the loop stopped after step t*: the last path of some task completes there
    assert max(int(r[1] + r[2] - 1) for m in range(M) for r in rule.paths[m]) == rule.t_star
    # truncation keeps each task's first max_paths paths and does not move the cut
    for k in (1, 2, 5):
        tr = collect_until(done, M * E * H, max_paths=k)
        assert tr.t_star == rule.t_star and tr.reached
        for m in range(M):
            np.testing.assert_array_equal(tr.paths[m], rule.paths[m][:k])


def test_timeline_of_2h_minus_1_steps_reaches_the_target():
    """paths.cu records T = 2H-1 steps: at step t every slot has at most H-1 samples in an unfinished path, so at step 2H-2
    every slot has completed >= H samples.  Random horizon-respecting timelines and the worst case, where every slot starts
    a path at step H-1, all reach M*E*H; in the worst case only at the last step."""
    rng = np.random.RandomState(7)
    M, E = 2, 5
    for H in (1, 2, 3, 7, 50, 600):
        T = 2 * H - 1
        for p in (0.0, 0.01, 0.2, 0.9):
            for _ in range(3):
                r = collect_until(horizon_timeline(rng, M, E, T, H, p), M * E * H)
                assert r.reached and r.t_star <= T - 1
        worst = np.zeros((M, E, T), dtype=bool)
        if H > 1:
            worst[:, :, H - 2] = True
        worst[:, :, 2 * H - 2] = True
        r = collect_until(worst, M * E * H)
        assert r.reached and r.t_star == T - 1
        if H > 1:
            assert not collect_until(worst[:, :, :T - 1], M * E * H).reached


def test_paths_finalize_argument_checks():
    """Bad sizes, a short workspace, a null timeline and a non-positive target are rejected before anything is launched
    (every pointer is a non-null dummy address that must never be dereferenced)."""
    from promp_b200 import _lib
    lib = _lib.load()
    dummy = 16
    M, E, T = 2, 4, 9
    ws = lib.promp_paths_workspace_bytes(M, E, T)

    def call(E=E, max_samples=E * T, target=M * E * 5, t_done=dummy, ws_bytes=ws):
        return lib.promp_paths_finalize(M, E, T, E * T, max_samples, 2, 2, target, t_done, *([dummy] * 16), ws_bytes, None)

    for kw, msg in ((dict(E=0), 'bad sizes'), (dict(E=1025, max_samples=1025 * T), 'bad sizes'),
                    (dict(max_samples=E * T - 1), 'max_samples must cover'), (dict(ws_bytes=ws - 1), 'workspace too small'),
                    (dict(t_done=None), 'null pointer'), (dict(target=0), 'target_samples must be positive'),
                    (dict(target=-5), 'target_samples must be positive')):
        assert call(**kw) == -1, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())


# ================================================================================================================ GPU
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _outputs(torch, M, P, N, Do, Da):
    i32 = lambda *s: torch.full(s, POISON_I, dtype=torch.int32, device='cuda')
    f32 = lambda *s: torch.full(s, POISON_F, dtype=torch.int32, device='cuda').view(torch.float32)
    return dict(path_off=i32(M, P + 1), n_paths=i32(M), n_valid=i32(M), src_slot=i32(M, P), src_start=i32(M, P),
                obs=f32(M, N, Do), act=f32(M, N, Da), mean=f32(M, N, Da), rew=f32(M, N),
                done=torch.full((M, N), POISON_U8, dtype=torch.uint8, device='cuda'), cut=i32(2))


def _finalize(torch, done, target, Do, Da, max_paths=None, ws=None, seed=0):
    """One promp_paths_finalize call on `done` and seeded float32 timelines, every output poisoned beforehand.  Returns the
    host timelines, the host outputs and the (device) workspace."""
    from promp_b200 import _lib
    M, E, T = done.shape
    rng = np.random.default_rng(seed)
    tl = dict(obs=rng.standard_normal((M, E, T, Do), dtype=np.float32), act=rng.standard_normal((M, E, T, Da), dtype=np.float32),
              mean=rng.standard_normal((M, E, T, Da), dtype=np.float32), rew=rng.standard_normal((M, E, T), dtype=np.float32))
    d = {k: torch.from_numpy(v).cuda() for k, v in tl.items()}
    d_done = torch.from_numpy(done.astype(np.uint8)).cuda()
    P = E * T if max_paths is None else max_paths
    N = (E * T + 3) // 4 * 4
    out = _outputs(torch, M, P, N, Do, Da)
    if ws is None:
        ws = torch.zeros(_lib.load().promp_paths_workspace_bytes(M, E, T) // 4, dtype=torch.int32, device='cuda')
    p = _lib.ptr
    _lib.call('promp_paths_finalize', M, E, T, P, N, Do, Da, int(target), p(d_done), p(d['obs']), p(d['act']), p(d['mean']),
              p(d['rew']), p(out['path_off']), p(out['n_paths']), p(out['n_valid']), p(out['src_slot']), p(out['src_start']),
              p(out['obs']), p(out['act']), p(out['mean']), p(out['rew']), p(out['done']), p(out['cut']), p(ws), ws.numel() * 4,
              _lib.stream())
    return tl, {k: v.cpu().numpy() for k, v in out.items()}, ws


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _check_against_rule(out, tl, done, target, ws, max_paths=None, poisoned=True):
    """Exact comparison of promp_paths_finalize's outputs with collect_until on the same timelines; ws (unless None) must
    be all zero."""
    M, E, T = done.shape
    rule = collect_until(done, target, max_paths)
    assert list(out['cut']) == [rule.t_star, int(rule.reached)], ('cut', list(out['cut']), rule.t_star, rule.reached)
    P =out['path_off'].shape[1] - 1
    for m in range(M):
        paths = rule.paths[m]
        n = len(paths)
        off, src = ragged_rows(paths, T)
        nv = int(off[-1])
        assert out['n_paths'][m] == n and out['n_valid'][m] == nv, (m, out['n_paths'][m], n, out['n_valid'][m], nv)
        np.testing.assert_array_equal(out['path_off'][m, :n + 1], off)
        np.testing.assert_array_equal(out['path_off'][m, n + 1:P + 1], nv)        # padding entries = closing offset
        np.testing.assert_array_equal(out['src_slot'][m, :n], paths[:, 0])
        np.testing.assert_array_equal(out['src_start'][m, :n], paths[:, 1])
        for key in ('obs', 'act', 'mean', 'rew'):
            got = out[key][m].reshape(out[key].shape[1], -1)
            want = tl[key][m].reshape(E * T, -1)[src]
            assert np.array_equal(_bits(got[:nv]), _bits(want)), (m, key)          # bit for bit
            if poisoned:
                assert (_bits(got[nv:]) == POISON_F).all(), (m, key)
        want_done = np.zeros(nv, dtype=np.uint8)
        want_done[off[1:] - 1] = 1
        np.testing.assert_array_equal(out['done'][m, :nv], want_done)
        if poisoned:
            assert (out['src_slot'][m, n:] == POISON_I).all() and (out['src_start'][m, n:] == POISON_I).all()
            assert (out['done'][m, nv:] == POISON_U8).all()
    if ws is not None:
        assert not ws.cpu().numpy().any(), "workspace not left zero"
    return rule


def _timeline(rng, M, E, T, kind, arg=None, never=0.0, quiet=()):
    if kind == 'rand':
        done = rng.random_sample((M, E, T)) < arg
    elif kind == 'horizon':
        done = horizon_timeline(rng, M, E, T, *arg)
    else:
        done = np.full((M, E, T), kind == 'every')
    flat = done.reshape(M * E, T)
    if never:
        flat[rng.random_sample(M * E) < never] = False            # slots that never finish
    for t in quiet:
        done[:, :, t] = False                                     # steps at which no path completes
    return done


def _target(done, cut):
    """Target that puts the rule's crossing exactly at step t0: 'eq' (the cumulative count there equals the target),
    'over' (it overshoots), 'never' (not reached), or ('natural', H) = M*E*H.  Forces a path to complete at t0."""
    kind, t0 = cut
    M, E, T = done.shape
    flat = done.reshape(M * E, T)
    if kind == 'natural':
        return M * E * t0, None
    if kind == 'eq':
        flat[0, t0] = True
    elif kind == 'over':                                           # a completing path of >= 2 samples, or two at step 0
        if t0 == 0:
            flat[:2, 0] = True
        else:
            flat[0, t0 - 1], flat[0, t0] = False, True
    every = np.concatenate(collect_until(done, np.inf).paths)      # all completed paths
    hist = np.bincount(every[:, 1] + every[:, 2] - 1, weights=every[:, 2], minlength=T).astype(np.int64)
    cum = np.cumsum(hist)                                          # completed samples up to each step
    if kind == 'never':
        return int(cum[-1]) + 1, None
    before = cum[t0 - 1] if t0 > 0 else 0
    target = cum[t0] if kind == 'eq' else before + 1
    assert before < target <= cum[t0] and (kind == 'eq') == (target == cum[t0])
    return int(target), t0


# (M, E, T, Do, Da, timeline, cut): E covers one lane, the warp boundary, a partial last warp and the full 1024-thread
# block; T and the cut cover one scan chunk and several, cuts on the first and last step of a chunk, a chunk whose last
# step completes no path, and a target never reached
CASES = {
    'E1_T1_eq0':              (1, 1, 1, 1, 1, ('every',), ('eq', 0)),
    'E1_T1_nopath':           (1, 1, 1, 1, 1, ('none',), ('never', None)),
    'E31_T33_over20':         (3, 31, 33, 2, 2, ('rand', 0.3), ('over', 20)),
    'E32_T33_over0':          (2, 32, 33, 2, 2, ('rand', 0.2), ('over', 0)),
    'E32_T1023_eq0':          (2, 32, 1023, 2, 2, ('rand', 0.05), ('eq', 0)),
    'E33_T1024_eq1023':       (2, 33, 1024, 17, 6, ('horizon', (512, 0.02)), ('eq', 1023)),
    'E40_T1025_over1024':     (4, 40, 1025, 2, 2, ('rand', 0.02, 0.0, (1023,)), ('over', 1024)),
    'E1000_T2047_over1023':   (1, 1000, 2047, 1, 1, ('rand', 0.01), ('over', 1023)),
    'E1024_T2049_eq2047':     (1, 1024, 2049, 1, 1, ('rand', 0.01, 0.0, (1023,)), ('eq', 2047)),
    'E1024_T2049_over2048':   (1, 1024, 2049, 1, 1, ('rand', 0.002, 0.25, (1023, 2047)), ('over', 2048)),
    'E1024_T2049_eq1024':     (1, 1024, 2049, 2, 2, ('horizon', (1025, 0.001)), ('eq', 1024)),
    'E1024_T2049_never':      (1, 1024, 2049, 1, 1, ('rand', 0.003, 0.25), ('never', None)),
    'E1024_T33_d19':          (2, 1024, 33, 19, 8, ('rand', 0.5), ('eq', 16)),
    'E32_T1024_every':        (2, 32, 1024, 1, 1, ('every',), ('eq', 1023)),
    'E31_T33_every_never':    (3, 31, 33, 2, 2, ('every',), ('never', None)),
    'E1_T2049_horizon':       (3, 1, 2049, 2, 2, ('horizon', (1025, 0.001)), ('natural', 1025)),
    'E8_T33_M300_d17':        (300, 8, 33, 17, 6, ('horizon', (17, 0.1)), ('natural', 17)),
    'E40_T65_M64_d19':        (64, 40, 65, 19, 8, ('horizon', (33, 0.05), 0.1), ('natural', 33)),
    'E33_T199_M100_d2':       (100, 33, 199, 2, 2, ('horizon', (100, 0.03)), ('natural', 100)),
}


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(CASES))
def test_paths_finalize_matches_rule(name):
    """promp_paths_finalize on a seeded synthetic timeline: cut, path table, offsets and padding, source slots, compacted
    rows (bit for bit) and done flags equal collect_until; rows past n_valid keep their poison; the workspace is left zero."""
    torch = _cuda()
    M, E, T, Do, Da, tl_spec, cut = CASES[name]
    rng = np.random.RandomState(sorted(CASES).index(name))
    done = _timeline(rng, M, E, T, tl_spec[0], *tl_spec[1:])
    target, t0 = _target(done, cut)
    tl, out, ws = _finalize(torch, done, target, Do, Da, seed=sorted(CASES).index(name))
    rule = _check_against_rule(out, tl, done, target, ws)
    if t0 is not None:
        assert rule.t_star == t0 and rule.reached
    if cut[0] == 'never':
        assert not rule.reached
    if tl_spec[0] == 'every':
        assert all(len(p) == E * T for p in rule.paths)                              # fills max_paths = E*T exactly
    if E >= 1000 and T > 1024:
        assert max(len(p) for p in rule.paths) > 256                                   # the compact kernel's grid-stride loop


def _two_phase_done():
    """8 slots, H = 600, T = 1199.  Phase 1: 150-step paths, cut at 599, 1200 samples completing at step 1049.  Phase 2:
    every slot finishes at steps 549 and 1100, so the cut is 1100; a stale hist[1049] = 1200 would move it to 1049."""
    T = 1199
    d1 = np.zeros((1, 8, T), dtype=bool)
    d1[:, :, 149::150] = True
    d2 = np.zeros((1, 8, T), dtype=bool)
    d2[:, :, [549, 1100]] = True
    return d1, d2


@pytest.mark.gpu
def test_workspace_reuse_across_calls():
    """One zero-filled workspace through a sequence of calls: a cut before step 1024 followed by a true cut past it, then
    seeded timelines at T = 1199 and 1999 with cuts on both sides of step 1024.  Every call matches the rule, and the
    workspace is zero after every call (the histogram past the cut's scan chunk included; checked last, so that counts
    left behind show up first as the wrong cut they cause)."""
    torch = _cuda()
    from promp_b200 import _lib
    ws = torch.zeros(_lib.load().promp_paths_workspace_bytes(2, 40, 1999) // 4, dtype=torch.int32, device='cuda')
    left = []                                               # nonzero workspace words after each call
    d1, d2 = _two_phase_done()
    tl, out, _ = _finalize(torch, d1, 4800, 2, 2, ws=ws, seed=1)
    assert _check_against_rule(out, tl, d1, 4800, None).t_star == 599
    left.append(int(torch.count_nonzero(ws)))
    tl, out, _ = _finalize(torch, d2, 4800, 2, 2, ws=ws, seed=2)
    rule = _check_against_rule(out, tl, d2, 4800, None)
    assert rule.t_star == 1100 and out['n_valid'][0] == 8 * 550 + 8 * 551
    left.append(int(torch.count_nonzero(ws)))
    rng = np.random.RandomState(11)
    for i, (T, t0) in enumerate([(1999, 700), (1999, 1500), (1199, 900), (1199, 1100), (1999, 300), (1999, 1998)]):
        done = horizon_timeline(rng, 2, 40, T, (T + 1) // 2, 0.003)
        target, _ = _target(done, ('eq', t0))
        tl, out, _ = _finalize(torch, done, target, 2, 2, ws=ws, seed=10 + i)
        assert _check_against_rule(out, tl, done, target, None).t_star == t0
        left.append(int(torch.count_nonzero(ws)))
    assert left == [0] * 8, left


@pytest.mark.gpu
def test_max_paths_truncation():
    """max_paths below some tasks' path counts and above others': each task keeps its first max_paths paths in the rule's
    order, n_valid and the closing / padding offsets count only their samples, and the cut still says where the rule
    stopped."""
    torch = _cuda()
    M, E, T = 4, 33, 100
    rng = np.random.RandomState(5)
    done = np.stack([rng.random_sample((E, T)) < p for p in (0.02, 0.1, 0.3, 0.6)])
    target, _ = _target(done, ('eq', 70))
    counts = sorted(len(p) for p in collect_until(done, target).paths)
    assert counts[0] < 257 < counts[-1]
    for k, max_paths in enumerate([1, counts[1], (counts[1] + counts[2]) // 2, 257, counts[-1] - 1]):
        tl, out, ws = _finalize(torch, done, target, 3, 2, max_paths=max_paths, seed=k)
        rule = _check_against_rule(out, tl, done, target, ws, max_paths=max_paths)
        assert rule.t_star == 70 and max(len(p) for p in rule.paths) == max_paths


@pytest.mark.gpu
def test_rejected_calls_leave_outputs_untouched():
    """A rejected call on real buffers returns an error and launches nothing: outputs keep their poison, the workspace
    keeps its contents."""
    torch = _cuda()
    from promp_b200 import _lib
    M, E, T, Do, Da = 2, 4, 9, 2, 2
    done = torch.ones(M, E, T, dtype=torch.uint8, device='cuda')
    tlf = torch.zeros(M, E, T, 8, dtype=torch.float32, device='cuda')
    out = _outputs(torch, M, E * T, E * T, Do, Da)
    wsb = _lib.load().promp_paths_workspace_bytes(M, E, T)
    ws = torch.full((wsb // 4 + 1,), 7, dtype=torch.int32, device='cuda')
    p = _lib.ptr
    for max_samples, target, ws_bytes in ((E * T, 0, wsb), (E * T, -1, wsb), (E * T - 1, 40, wsb), (E * T, 40, wsb - 1)):
        with pytest.raises(_lib.PrompLibraryError):
            _lib.call('promp_paths_finalize', M, E, T, E * T, max_samples, Do, Da, target, p(done), p(tlf), p(tlf), p(tlf),
                      p(tlf), *[p(out[k]) for k in ('path_off', 'n_paths', 'n_valid', 'src_slot', 'src_start', 'obs', 'act',
                                                     'mean', 'rew', 'done', 'cut')], p(ws), ws_bytes, _lib.stream())
    torch.cuda.synchronize()
    for k, v in out.items():
        want = POISON_U8 if k == 'done' else POISON_I if v.dtype == torch.int32 else None
        if want is None:
            assert (v.view(torch.int32) == POISON_F).all(), k
        else:
            assert (v == want).all(), k
    assert (ws == 7).all()


@pytest.mark.gpu
@pytest.mark.parametrize('env_name', ['walker_vel', 'point'])
def test_sampler_long_horizon_phases(env_name):
    """MetaSampler(reset_mode='device') at H = 600 (T = 1199, two scan chunks), two consecutive obtain_samples() calls on
    one sampler: after each, the path table and compacted tensors equal collect_until(timeline.done, M*E*H), the sampler's
    workspace is zero and the kept paths hold >= M*E*H samples."""
    torch = _cuda()
    H = 600
    if env_name == 'point':
        from test_gpu_parity import _origin_seeking_policy
        from promp_b200.envs import normalize, MetaPointEnv
        from promp_b200.samplers import MetaSampler
        M, E = 2, 40
        policy = _origin_seeking_policy(torch, M)
        sampler = MetaSampler(env=normalize(MetaPointEnv()), policy=policy, rollouts_per_meta_task=E, meta_batch_size=M,
                              max_path_length=H, reset_mode='device', seed=5)
    else:
        from test_locomotion_envs import _stack
        from oracle import locomotion_surrogates as ls
        M, E = 2, 8
        _, policy, sampler = _stack(env_name, M, E, H, reset_mode='device', seed=4)
        theta = policy.theta.cpu().numpy().copy()
        theta[-6:] = np.log(10.0)                          # the falling policy of test_walker_fused_early_termination
        theta[-12:-6] = 2.0 * np.sign(ls.Walker.P)
        policy.set_params(theta)
    assert sampler._fused_early_ok()
    sampler.update_tasks()
    policy.switch_to_pre_update()
    for _ in range(2):
        ph = sampler.obtain_samples().phase
        tl = {k: v.cpu().numpy() for k, v in ph.timeline.items() if k != 'ws'}
        done = tl['done'].astype(bool)
        assert done.shape == (M, E, 2 * H - 1)
        out = dict(cut=ph.cut, n_paths=ph.n_paths, n_valid=ph.n_valid, path_off=ph.path_off, src_slot=ph.src_slot,
                   src_start=ph.src_start, obs=ph.obs, act=ph.act, mean=ph.mean, rew=ph.rew, done=ph.done)
        out = {k: v.cpu().numpy() for k, v in out.items()}
        rule = _check_against_rule(out, tl, done, M * E * H, sampler._timeline['ws'], poisoned=False)
        assert rule.reached and int(out['n_valid'].sum()) >= M * E * H
        assert max(len(p) for p in rule.paths) > 1
