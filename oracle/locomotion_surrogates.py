"""Specification + CPU restatement of the MuJoCo-free Walker2d and Swimmer surrogates.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

What follows the reference (meta_policy_search/envs/mujoco_envs/):
  Walker2d (walker2d_rand_vel.py, walker2d_rand_direc.py)
  * qpos = (x, z, pitch, 6 joints), qvel likewise: 9 + 9; action = 6 torques, ctrlrange [-1, 1]
  * obs = qpos[1:] (8) ++ clip(qvel, -10, 10) (9) = 17 floats                               (_get_obs)
  * frame_skip = 8 with walker2d.xml's timestep 0.002 => dt = 0.016
  * reset: qpos = init_qpos + U(-.005,.005)^9, qvel = U(-.005,.005)^9, init_qpos = (0, 1.25, 0, ...)  (reset_model)
  * RandVel:   reward = -|dx/dt - goal| + 15 - 1e-3*|a|^2,  goal ~ U(0, 10)
    RandDirec: reward = dir*dx/dt + 1 - 1e-3*|a|^2,         dir ~ {-1, +1}
  * done = not (0.8 < z < 2.0 and -1 < pitch < 1); env_infos = {}
  Swimmer (swimmer_rand_vel.py)
  * qpos = (x, y, rot, 2 joints), qvel likewise: 5 + 5; action = 2 torques, ctrlrange [-1, 1]
  * obs = qpos[2:] (3) ++ qvel (5) = 8 floats
  * frame_skip = 4 with swimmer.xml's timestep 0.01 => dt = 0.04
  * reset: qpos = U(-.1,.1)^5, qvel = U(-.1,.1)^5 (init state zero)
  * reward_fwd = |dx/dt - goal| (the reference's sign: deviating from the goal is rewarded),
    reward_ctrl = -1e-4*|a|^2, reward = reward_fwd + reward_ctrl, goal ~ U(0.1, 0.2); done = False
  * env_infos = {reward_fwd, reward_ctrl}

What is NEW (MuJoCo is absent): the dynamics, semi-implicit Euler with the sub-step h = timestep.

Walker2d, per sub-step (joint j = 0..5; the root terms use the joint state after this sub-step's joint
update and the pitch of the start of the sub-step):
    acc = G[j]*u[j] - K[j]*q[j] - D[j]*qd[j];   qd[j] += h*acc;   q[j] += h*qd[j]
    thrust += C[j]*qd[j]*sin(q[j] + pitch + PH[j]);   lift += C[j]*qd[j]*cos(q[j] + pitch + PH[j])
    xd    += h*(thrust - BX*xd);                                   x     += h*xd
    zd    += h*(KZ*(Z0*cos(pitch) - z) - DZ*zd + LZ*lift);         z     += h*zd
    pd    += h*(AP*sin(pitch) + sum_j P[j]*u[j] - DP*pd);          pitch += h*pd
The torso is an inverted pendulum (AP > 0): left alone it tips over, the height follows Z0*cos(pitch),
and the done rule ends the path once it has fallen (z < 0.8 near |pitch| = 0.88, or |pitch| >= 1).

Swimmer, per sub-step:
    acc = G[j]*u[j] - K[j]*q[j] - D[j]*qd[j];   qd[j] += h*acc;   q[j] += h*qd[j]      (j = 0, 1)
    thrust = CS*(q[0]*qd[1] - q[1]*qd[0])        (swept area of the two-joint stroke: a phase-lagged
                                                    stroke swims, a reciprocal one does not)
    rd += h*(P[0]*u[0] + P[1]*u[1] - DR*rd);     (rotation of the start of the sub-step below)
    xd += h*(thrust*cos(rot) - BV*xd);  x += h*xd
    yd += h*(thrust*sin(rot) - BV*yd);  y += h*yd
    rot += h*rd

All arithmetic is float32 in the CUDA kernels; this restatement runs in the dtype of its inputs so tests can
evaluate it in float32 (same rounding model) or float64.
"""
import numpy as np


class Walker(object):
    NQ = 9
    OBS_DIM = 17
    ACT_DIM = 6
    FRAME_SKIP = 8
    H_SIM = 0.002
    DT = FRAME_SKIP * H_SIM
    INIT_QPOS = (0.0, 1.25, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    RESET_NOISE = 0.005
    G = (6.0, 5.0, 3.0, 6.0, 5.0, 3.0)               # torque gain
    K = (20.0, 16.0, 10.0, 20.0, 16.0, 10.0)          # joint spring
    D = (3.0, 2.5, 1.5, 3.0, 2.5, 1.5)                # joint damping
    C = (0.8, 0.6, 0.3, 0.8, 0.6, 0.3)                # thrust / lift coupling
    PH = (0.4, -0.3, 0.9, -0.4, 0.3, -0.9)            # leg phase offsets
    P = (1.2, -0.8, 0.5, -1.0, 0.9, -0.6)             # pitch torque coupling
    BX, Z0, KZ, DZ, LZ = 1.0, 1.25, 60.0, 12.0, 0.5
    AP, DP = 5.0, 0.5                                  # inverted-pendulum gain, pitch damping


class Swimmer(object):
    NQ = 5
    OBS_DIM = 8
    ACT_DIM = 2
    FRAME_SKIP = 4
    H_SIM = 0.01
    DT = FRAME_SKIP * H_SIM
    RESET_NOISE = 0.1
    G = (10.0, 10.0)
    K = (4.0, 4.0)
    D = (1.0, 1.0)
    P = (0.5, -0.5)
    CS, DR, BV = 0.02, 2.0, 1.0


# ------------------------------------------------------------------------------------------------ walker
def walker_reset_state(rng, n, dtype=np.float64):
    """reset_model: qpos noise for every env, then qvel noise (the cheetah's vectorised convention)."""
    out = np.empty((n, 2 * Walker.NQ))
    out[:, :Walker.NQ] = np.asarray(Walker.INIT_QPOS) + rng.uniform(low=-.005, high=.005, size=(n, Walker.NQ))
    out[:, Walker.NQ:] = rng.uniform(low=-.005, high=.005, size=(n, Walker.NQ))
    return out.astype(dtype)


def walker_obs(qpos, qvel):
    return np.concatenate([qpos[..., 1:], np.clip(qvel, -10, 10)], axis=-1)


def walker_done(qpos):
    z, ang = qpos[..., 1], qpos[..., 2]
    return ~((z > 0.8) & (z < 2.0) & (ang > -1.0) & (ang < 1.0))


def walker_step(qpos, qvel, u, task, mode):
    """One env step on (..., 9) state arrays; `u` is the clipped torque (..., 6).  mode 0: RandDirec (task = direction),
    mode 1: RandVel (task = goal velocity).  Returns (qpos', qvel', reward, done, forward_vel)."""
    W = Walker
    f = qpos.dtype.type
    qpos, qvel = qpos.copy(), qvel.copy()
    u = u.astype(qpos.dtype)
    h = f(W.H_SIM)
    x0 = qpos[..., 0].copy()
    twist = np.zeros_like(x0)
    for j in range(6):
        twist = twist + f(W.P[j]) * u[..., j]
    for _ in range(W.FRAME_SKIP):
        thrust = np.zeros_like(x0)
        lift = np.zeros_like(x0)
        pitch = qpos[..., 2].copy()
        for j in range(6):
            q, qd = qpos[..., 3 + j], qvel[..., 3 + j]
            acc = f(W.G[j]) * u[..., j] - f(W.K[j]) * q - f(W.D[j]) * qd
            qd = qd + h * acc
            q = q + h * qd
            qpos[..., 3 + j], qvel[..., 3 + j] = q, qd
            ang = q + pitch + f(W.PH[j])
            thrust = thrust + f(W.C[j]) * qd * np.sin(ang)
            lift = lift + f(W.C[j]) * qd * np.cos(ang)
        xd = qvel[..., 0] + h * (thrust - f(W.BX) * qvel[..., 0])
        qvel[..., 0] = xd
        qpos[..., 0] = qpos[..., 0] + h * xd
        zd = qvel[..., 1] + h * (f(W.KZ) * (f(W.Z0) * np.cos(pitch) - qpos[..., 1]) - f(W.DZ) * qvel[..., 1] + f(W.LZ) * lift)
        qvel[..., 1] = zd
        qpos[..., 1] = qpos[..., 1] + h * zd
        pd = qvel[..., 2] + h * (f(W.AP) * np.sin(pitch) + twist - f(W.DP) * qvel[..., 2])
        qvel[..., 2] = pd
        qpos[..., 2] = pitch + h * pd
    fwd = (qpos[..., 0] - x0) / f(W.DT)
    ctrl = f(1e-3) * np.sum(np.square(u), axis=-1)
    task = np.asarray(task, dtype=qpos.dtype)
    if mode == 1:
        reward = -np.abs(fwd - task) + f(15.0) - ctrl
    else:
        reward = task * fwd + f(1.0) - ctrl
    return qpos, qvel, reward, walker_done(qpos), fwd


# ------------------------------------------------------------------------------------------------ swimmer
def swimmer_reset_state(rng, n, dtype=np.float64):
    out = np.empty((n, 2 * Swimmer.NQ))
    out[:, :Swimmer.NQ] = rng.uniform(low=-.1, high=.1, size=(n, Swimmer.NQ))
    out[:, Swimmer.NQ:] = rng.uniform(low=-.1, high=.1, size=(n, Swimmer.NQ))
    return out.astype(dtype)


def swimmer_obs(qpos, qvel):
    return np.concatenate([qpos[..., 2:], qvel], axis=-1)


def swimmer_step(qpos, qvel, u, goal_vel):
    """Returns (qpos', qvel', reward, reward_fwd, reward_ctrl)."""
    S = Swimmer
    f = qpos.dtype.type
    qpos, qvel = qpos.copy(), qvel.copy()
    u = u.astype(qpos.dtype)
    h = f(S.H_SIM)
    x0 = qpos[..., 0].copy()
    twist = f(S.P[0]) * u[..., 0] + f(S.P[1]) * u[..., 1]
    for _ in range(S.FRAME_SKIP):
        for j in range(2):
            q, qd = qpos[..., 3 + j], qvel[..., 3 + j]
            acc = f(S.G[j]) * u[..., j] - f(S.K[j]) * q - f(S.D[j]) * qd
            qd = qd + h * acc
            qpos[..., 3 + j], qvel[..., 3 + j] = q + h * qd, qd
        thrust = f(S.CS) * (qpos[..., 3] * qvel[..., 4] - qpos[..., 4] * qvel[..., 3])
        rot = qpos[..., 2].copy()
        rd = qvel[..., 2] + h * (twist - f(S.DR) * qvel[..., 2])
        c, s = np.cos(rot), np.sin(rot)
        xd = qvel[..., 0] + h * (thrust * c - f(S.BV) * qvel[..., 0])
        yd = qvel[..., 1] + h * (thrust * s - f(S.BV) * qvel[..., 1])
        qvel[..., 0], qvel[..., 1], qvel[..., 2] = xd, yd, rd
        qpos[..., 0] = qpos[..., 0] + h * xd
        qpos[..., 1] = qpos[..., 1] + h * yd
        qpos[..., 2] = rot + h * rd
    fwd = (qpos[..., 0] - x0) / f(S.DT)
    reward_fwd = np.abs(fwd - np.asarray(goal_vel, dtype=qpos.dtype))
    reward_ctrl = -f(1e-4) * np.sum(np.square(u), axis=-1)
    return qpos, qvel, reward_fwd + reward_ctrl, reward_fwd, reward_ctrl
