"""Synthetic open-loop vector environment (SURVEY.md section 8d).

Observations are a fixed stream shared by every policy (``obs_stream[t]`` is what the
policy sees at step ``t``; ``obs_stream[t+1]`` is what ``step`` returns), the reward is
``r_t = <a_t, rew_vec[t]>`` in float32 and the 'robot position' integrates the first
three action components.  It offers the classic gym single-env API (``reset``/``step``,
used by the per-perturbation compatibility path of ``gym_runner.run_model``) and, through
``device_arrays``, the resident HBM copy that the batched rollout kernels read.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

# name fragments -> (obs_dim, act_dim) of the gym/pybullet tasks the reference's configs name
KNOWN_SHAPES = {
    'HalfCheetah': (17, 6),          # BASELINE.json config 2 ("HalfCheetah-shaped")
    'Humanoid': (376, 17),           # BASELINE.json configs 3-5 ("Humanoid-shaped")
    'Hopper': (15, 3),               # configs/simple_conf.json (HopperBulletEnv-v0)
    'Walker2D': (22, 6),
    'Ant': (28, 8),
}


class Box:
    """Stand-in for gym.spaces.Box: shape/low/high/seed/sample are all the reference reads."""

    def __init__(self, low, high, shape, dtype=np.float32):
        self.shape = tuple(shape)
        self.low = np.full(self.shape, low, dtype=dtype)
        self.high = np.full(self.shape, high, dtype=dtype)
        self.dtype = dtype
        self._rs = np.random.RandomState()

    def seed(self, seed=None):
        self._rs = np.random.RandomState(seed)
        return [seed]

    def sample(self):
        return self._rs.uniform(-1, 1, self.shape).astype(self.dtype)


class _Robot:
    """pybullet-gym style handle so position getters like ``env.robot.robot_body.pose().xyz()``
    (src/gym/gym_runner.py:17-18) keep working on the synthetic env."""

    def __init__(self, env):
        self._env = env
        self.robot_body = self

    def pose(self):
        return self

    def xyz(self):
        return tuple(float(x) for x in self._env.pos)

    @property
    def body_real_xyz(self):
        return self.xyz()


class SyntheticEnv:
    is_synthetic_openloop = True

    def __init__(self, obs_dim: int, act_dim: int, max_episode_steps: int = 1000, obs_seed: int = 11,
                 rew_seed: int = 13, pos_scale: float = 0.05, name: str = 'Synthetic-v0'):
        self.name = name
        self.obs_dim, self.act_dim, self.T = int(obs_dim), int(act_dim), int(max_episode_steps)
        self.pos_scale = float(pos_scale)
        self.observation_space = Box(-np.inf, np.inf, (self.obs_dim,))
        self.action_space = Box(-1.0, 1.0, (self.act_dim,))
        self.obs_stream = self._host(np.random.RandomState(obs_seed).randn(self.T + 1, self.obs_dim).astype(np.float32))
        self.rew_vec = self._host(np.random.RandomState(rew_seed).randn(self.T, self.act_dim).astype(np.float32))
        self.host_pinned = bool(SyntheticEnv._pinned_keepalive) and SyntheticEnv._last_pinned
        self.robot = _Robot(self)
        self.unwrapped = self
        self.t = 0
        self.pos = np.zeros(3, dtype=np.float32)
        self._dev = None

    @staticmethod
    def _host(a: np.ndarray) -> np.ndarray:
        """Keep the env's host arrays in pinned memory when a GPU is present, so the per-generation upload of the
        observation / reward streams is a direct asynchronous copy (the ndarray is a view of the pinned tensor)."""
        try:
            import torch
            if torch.cuda.is_available():
                t = torch.from_numpy(a).pin_memory()
                v = t.numpy()
                v.setflags(write=True)
                SyntheticEnv._pinned_keepalive.append(t)
                SyntheticEnv._last_pinned = True
                return v
        except Exception:
            pass
        SyntheticEnv._last_pinned = False
        return a

    _pinned_keepalive = []
    _last_pinned = False

    # ---- gym API -------------------------------------------------------------------------
    def seed(self, seed=None):
        return [seed]

    def reset(self):
        self.t = 0
        self.pos = np.zeros(3, dtype=np.float32)
        return self.obs_stream[0].copy()

    def step(self, action) -> Tuple[np.ndarray, float, bool, dict]:
        if self.t >= self.T:
            raise RuntimeError('step() called on a finished episode; call reset()')
        a = np.asarray(action, dtype=np.float32).reshape(-1)
        c = self.rew_vec[self.t]
        acc = np.float32(0.0)
        for j in range(self.act_dim):
            acc = np.float32(acc + np.float32(a[j] * c[j]))
        ps = np.float32(self.pos_scale)
        for j in range(3):
            self.pos[j] = np.float32(self.pos[j] + np.float32(ps * a[j % self.act_dim]))
        self.t += 1
        return self.obs_stream[self.t].copy(), float(acc), self.t >= self.T, {}

    def render(self, *args, **kwargs):
        return None

    def close(self):
        pass

    # ---- device residency ----------------------------------------------------------------------
    def device_arrays(self, engine):
        """(obs_stream[T+1,obs] , rew_vec[T,act]) as float32 tensors in HBM (uploaded once)."""
        if self._dev is None or self._dev[0].device != engine.device:
            self._dev = (engine.to_device(self.obs_stream), engine.to_device(self.rew_vec))
        return self._dev


class ClosedLoopEnv(SyntheticEnv):
    """The closed-loop variant of the synthetic env (SURVEY.md section 8d, optional; reported separately from the open-loop
    headline): ``obs_{t+1} = tanh(A obs_t + B a_t)`` -- what the policy sees depends on what it did, so the episode cannot
    be batched over time.  A is banded with wrap-around (``band`` diagonals centred on the main one, gain ``a_gain`` keeps
    the map contractive), B dense; obs_0 is row 0 of the open-loop stream; reward and position as in the open-loop env.
    float32 throughout, pre-activation accumulated in index order (A's diagonals, then B's columns).

    ``fall_height``: None (the default), every episode runs ``max_episode_steps`` steps.  A float h > 0: the episode also ends
    (``step`` returns ``done``) at the first step after which the third position component leaves [-h, h], evaluated in
    float32 after that step's position update -- a torso height that drifts out of its healthy range, as the pybullet Hopper
    and Ant envs end an episode when the robot falls.  A NaN position ends the episode too."""
    is_synthetic_openloop = False
    is_synthetic_closedloop = True

    def __init__(self, obs_dim: int, act_dim: int, max_episode_steps: int = 1000, band: int = 8, a_seed: int = 17,
                 b_seed: int = 19, a_gain: float = 0.5, b_gain: float = 0.5, name: str = 'SyntheticClosedLoop-v0',
                 fall_height: Optional[float] = None, **kwargs):
        if fall_height is not None:
            if isinstance(fall_height, bool) or not isinstance(fall_height, (int, float, np.integer, np.floating)):
                raise TypeError(f'fall_height must be a number or None, got {fall_height!r}')
            with np.errstate(over='ignore'):
                h = np.float32(fall_height)
            if not (np.isfinite(h) and h > 0):
                raise ValueError(f'fall_height must be finite and > 0 as a float32, got {fall_height!r}')
            fall_height = h
        self.fall_height = fall_height
        super().__init__(obs_dim, act_dim, max_episode_steps, name=name, **kwargs)
        self.band = int(band)
        self.env_a = (np.random.RandomState(a_seed).randn(self.obs_dim, self.band) * (a_gain / np.sqrt(self.band))).astype(np.float32)
        self.env_b = (np.random.RandomState(b_seed).randn(self.obs_dim, self.act_dim) * (b_gain / np.sqrt(self.act_dim))).astype(np.float32)
        self.ob = self.obs_stream[0].copy()
        self._dev_closed = None

    def reset(self):
        super().reset()
        self.ob = self.obs_stream[0].copy()
        return self.ob.copy()

    def step(self, action) -> Tuple[np.ndarray, float, bool, dict]:
        a = np.asarray(action, dtype=np.float32).reshape(-1)
        _, rew, done, info = super().step(a)
        f32, half = np.float32, self.band // 2
        acc = np.zeros(self.obs_dim, dtype=f32)
        for d in range(self.band):
            acc = (acc + (self.env_a[:, d] * np.roll(self.ob, half - d)).astype(f32)).astype(f32)
        for j in range(self.act_dim):
            acc = (acc + (self.env_b[:, j] * a[j]).astype(f32)).astype(f32)
        self.ob = np.tanh(acc).astype(f32)
        if self.fall_height is not None:
            done = bool(done or not (abs(self.pos[2]) <= self.fall_height))      # float32 |z| against float32 h; NaN falls
        return self.ob.copy(), rew, done, info

    @property
    def terminates(self) -> bool:
        """Whether an episode can end before ``max_episode_steps`` (a ``fall_height`` is set)."""
        return self.fall_height is not None

    def device_closed(self, engine):
        """(obs_0 [obs], A transposed [band][obs], B transposed [act][obs]) as float32 tensors in HBM."""
        if self._dev_closed is None or self._dev_closed[0].device != engine.device:
            self._dev_closed = (engine.to_device(self.obs_stream[0].copy()),
                                engine.to_device(np.ascontiguousarray(self.env_a.T)),
                                engine.to_device(np.ascontiguousarray(self.env_b.T)))
        return self._dev_closed


def make(name: str, **kwargs) -> SyntheticEnv:
    """``gym.make`` replacement: any task name maps to a synthetic env of the matching shape."""
    for frag, (o, a) in KNOWN_SHAPES.items():
        if frag.lower() in name.lower():
            if 'closedloop' in name.lower().replace('-', '').replace('_', ''):
                return ClosedLoopEnv(o, a, name=name, **kwargs)
            return SyntheticEnv(o, a, name=name, **kwargs)
    raise ValueError(f'no synthetic shape registered for env {name!r}; known: {sorted(KNOWN_SHAPES)}')
