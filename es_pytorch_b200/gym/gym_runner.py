"""Rollout runner (mirror of src/gym/gym_runner.py:33-67).

``run_model`` keeps the reference signature.  When the env is the synthetic open-loop env
and the model is a tanh ``FeedForward`` or a tanh ``FFBinned`` (``BaseNet.head``), the whole episode is ONE launch of the fused rollout
kernel (per-policy compatibility path: theta' is the module's current weights, sigma = 0;
action noise, nn.py:47-48, is drawn from ``rs`` for the whole episode at once and added on
the device); any other env is stepped in the reference's python loop with the module's own
forward.
"""
from __future__ import annotations

import time
from typing import Callable, List, Tuple

import numpy as np
import torch


def pybullet_envs_pos(env):
    return env.robot.body_real_xyz


def pybullet_gym_pos(env):
    return env.robot.robot_body.pose().xyz()


def mujoco_pos(env):
    """Centre of mass of a mujoco model (gym_runner.py:25-30)."""
    mass = np.reshape(env.model.body_mass, (-1, 1))
    centre = np.sum(mass * env.data.xipos, 0) / np.sum(mass)
    return centre[0], centre[1], centre[2]


def hbaselines_pos(env):
    return tuple(env.wrapped_env.get_body_com('torso')[:3])


def _device_episode(model, env, max_steps: int, rs=None, episodes: int = 1, activation=None):
    """One evaluation on the open- or closed-loop synthetic env as one launch (sigma = 0).  With ``rs`` and a tanh model's
    ac_std != 0: the action noise of ``episodes`` episodes drawn back to back from ``rs``, the per-step mean over the episodes
    (obj.py:54-63).  ``activation``: the model's ``nn.Activation`` when it is not a tanh one (its outputs are the actions, as
    a tanh model's).  Returns (fitness, the last episode's final position, steps), steps the number of steps the last episode
    ran: T, or t_d + 1 on a closed-loop env whose episode ended at step t_d (``ClosedLoopEnv(fall_height=h)``).  There the
    noise of ``episodes`` x T steps is drawn from a copy of ``rs``, and ``rs`` then advances by exactly the gaussians the
    executed steps consumed, as the reference's per-step ``rs.randn(act)`` calls leave it."""
    from ..engine import get_engine
    from ..core.policy import Policy
    eng = get_engine()
    sizes, head = model.layer_sizes(), ('tanh' if activation is not None else model.head())
    T = min(int(max_steps), env.T)
    obs_dev, rew_dev = env.device_arrays(eng)
    theta = eng.to_device(Policy.get_flat(model), torch.float32)
    mean = eng.to_device(np.ascontiguousarray(model._obmean, dtype=np.float64).reshape(-1), torch.float64)
    std = eng.to_device(np.ascontiguousarray(model._obstd, dtype=np.float64).reshape(-1), torch.float64)
    table = torch.zeros(theta.numel() + 1, dtype=torch.float32, device=eng.device)      # sigma = 0: the slice is irrelevant
    idx = torch.zeros(1, dtype=torch.int64, device=eng.device)
    fit = torch.zeros(2, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, 3, dtype=torch.float32, device=eng.device)
    noise = None
    ac_std = float(getattr(model, '_action_std', 0) or 0)
    closed = getattr(env, 'is_synthetic_closedloop', False)
    term = closed and getattr(env, 'terminates', False)
    if rs is not None and ac_std != 0 and head == 'tanh':
        # nn.py:47-48: T calls of rs.randn(act) * ac_std per episode; one call of rs.randn(episodes * T * act) consumes the stream
        # identically (legacy gaussians are produced one by one, cached second value included; neither env's noise depends on
        # its state).  [pair 0][+ | -][episodes][T][act]: both evaluations of the sigma = 0 "pair" see it, only + is used.
        src = rs
        if term:                                        # how many are consumed is known after the rollout
            src = np.random.RandomState()
            src.set_state(rs.get_state())
        nz = (src.randn(episodes * T * sizes[-1]) * ac_std).astype(np.float32)
        noise = eng.to_device(np.stack([nz, nz]).reshape(1, 2, -1))
    else:
        episodes = 1
    out = (fit[0:1], fit[1:2], 1, behv[0:1].view(-1), behv[1:2].view(-1))
    if term:
        steps, used = eng.rollout_closed_terminal(
            table, idx, theta, 0.0, sizes, mean, std, float(model.ob_clip), *env.device_closed(eng), rew_dev[:T].contiguous(),
            env.pos_scale, *out, head=head, act_noise=noise, episodes=episodes, activation=activation,
            fall_height=env.fall_height, steps=torch.zeros(2, 1, dtype=torch.int32, device=eng.device),
            noise_used=torch.zeros(2, 1, dtype=torch.int64, device=eng.device))
        t_d, n_used = int(steps[0, 0].item()), int(used[0, 0].item())
        if noise is not None:
            rs.randn(n_used)
        return float(fit[0].item()), behv[0].cpu().numpy().astype(np.float64), t_d + 1
    if closed:
        eng.rollout_closed_mlp(table, idx, theta, 0.0, sizes, mean, std, float(model.ob_clip), *env.device_closed(eng),
                               rew_dev[:T].contiguous(), env.pos_scale, *out, head=head, act_noise=noise, episodes=episodes,
                               activation=activation)
    else:
        obsn = eng.normalise_obs(obs_dev[:T], mean, std, float(model.ob_clip))
        eng.rollout(table, idx, theta, 0.0, sizes, obsn, rew_dev[:T].contiguous(), env.pos_scale, *out, act_noise=noise,
                    episodes=episodes, head=head, activation=activation)
    return float(fit[0].item()), behv[0].cpu().numpy().astype(np.float64), T


def run_model(model: torch.nn.Module, env, max_steps: int, rs: np.random.RandomState = None, render: bool = False,
              get_pos_fn: Callable = pybullet_gym_pos) -> Tuple[List[float], List[float], np.ndarray, int]:
    """(rewards, positions padded to max_steps triples, post-step observations, last loop index)."""
    fused = (getattr(env, 'is_synthetic_openloop', False) and hasattr(model, 'head') and model.head() is not None
             and not render)
    if fused:
        total, pos, T = _device_episode(model, env, max_steps, rs)
        # the episode total is exact; it is reported as a one-element reward list so that
        # sum(rews) (training_result.py:28) reproduces it bit for bit
        rews = [total]
        behv = [float(pos[0]), float(pos[1]), float(pos[2])] * int(max_steps)
        return rews, behv, env.obs_stream[1:T + 1], T - 1

    behv, rews, obs = [], [], []
    with torch.no_grad():
        ob = env.reset()
        for step in range(max_steps):
            ob = torch.from_numpy(np.asarray(ob)).float()
            action = model(ob, rs=rs)
            ob, rew, done, _ = env.step(action.cpu().numpy() if torch.is_tensor(action) else np.asarray(action))
            rews += [rew]
            obs.append(ob)
            behv.extend(get_pos_fn(env.unwrapped))
            if render:
                env.render('human')
                time.sleep(1 / 60)
            if done:
                break
    behv += behv[-3:] * (max_steps - int(len(behv) / 3))
    return rews, behv, np.array(obs), step


def multi_agent_gym_runner(policies, env, max_steps: int, rs: np.random.RandomState = None, save_obs: bool = False,
                           render: bool = False):
    """gym_runner.py:70-110 drives a Unity ML-Agents environment (src/gym/unity.py); that simulator and its wrapper are
    outside this package's scope."""
    raise NotImplementedError('multi_agent_gym_runner needs the Unity ML-Agents wrapper (src.gym.unity), which is not part of '
                              'es_pytorch_b200: the device path covers single-agent rollouts on the synthetic env')
