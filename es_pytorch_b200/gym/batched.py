"""``BatchedRollout``: the fit_fn that lets ``es.test_params`` / ``es.step`` evaluate ALL of a
rank's antithetic pairs in one fused launch.

The reference's ``fit_fn`` is an opaque per-policy python callback (src/core/es.py:28,71-72),
which forces one rollout per call.  A ``BatchedRollout`` is still callable like that (it is
what ``es.step`` uses for the noiseless evaluation, es.py:48) but it also *describes* the
evaluation -- env, episode length, how many ``rs.random()`` coins the script's fit_fn draws
per evaluation, how many episodes it averages, which TrainingResult adaptor it builds -- so
the generation can run on the device with the same RNG consumption and the same results layout.

``episodes`` is obj.py's ``eps_per_policy`` (obj.py:54-63): the fit_fn draws its coin, runs
``max(1, episodes)`` episodes and returns the per-step mean of their rewards (float64, episodes
in order), with the last episode's behaviour.  With action noise every episode draws its own
T x act gaussians from the stream; without it the episodes are identical and the mean is
exactly the single episode (E copies of a float32 sum exactly in float64, and (E r) / E == r).

``fuse_activations``: FeedForward policies whose activation is not tanh (ReLU, LeakyReLU, ELU, Sigmoid: ``BaseNet.activation``)
run the fused device rollouts too (es_rollout_*_activation) -- in ``es.step``, ``es.test_params`` and this object's own
call.  Off by default: such a policy then runs run_model's python loop with the module's own forward, as the reference does.

``fuse_noisy_terminal``: a policy with action noise on an env whose episodes end early (``ClosedLoopEnv(fall_height=h)``) runs
the whole generation in one launch that walks each stream's index, coin and noise draws inside the rollout
(es_rollout_closedloop_terminal_streams), in ``es.step`` and ``es.test_params``.  Off by default: such a generation then runs
one evaluation per launch with numpy's own gaussians.  The fused route's gaussians use CUDA's log (<= 1 ulp of float64), so a
float32 noise value can differ from numpy's where it lies next to a rounding midpoint; this object's own call is unchanged.

``result`` is the TrainingResult adaptor the script's fit_fn builds (training_result.py:62-97): RewardResult (the default
without an archive), MeanRewardResult, DistResult, XDistResult, NSResult (novelty alone) or NSRResult (reward and novelty,
the default with an archive).  The fused generation computes the same column(s) on the device.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from .. import _lib
from .gym_runner import run_model
from .training_result import DistResult, MeanRewardResult, NSResult, NSRResult, RewardResult, TrainingResult, XDistResult

# adaptor -> DeviceGeneration's objective (NSRResult is the reward column plus the novelty column of an archive)
_OBJECTIVES = {RewardResult: 'reward', MeanRewardResult: 'mean_reward', DistResult: 'dist', XDistResult: 'xdist',
               NSResult: 'novelty', NSRResult: 'reward'}


class BatchedRollout:
    is_batched_rollout = True

    def __init__(self, env, max_steps: int, coins_per_eval: int = 1, save_obs_chance: float = 0.0,
                 archive: Optional[np.ndarray] = None, nov_k: int = 10,
                 rank_streams: Optional[Sequence[np.random.RandomState]] = None,
                 rollout_mode: int = _lib.ES_ROLLOUT_F32, episodes: int = 1, result: Optional[type] = None,
                 fuse_activations: bool = False, fuse_noisy_terminal: bool = False):
        if not (getattr(env, 'is_synthetic_openloop', False) or getattr(env, 'is_synthetic_closedloop', False)):
            raise TypeError('BatchedRollout needs a synthetic env (es_pytorch_b200.gym.synthetic_env: open- or closed-loop)')
        self.env = env
        self.max_steps = min(int(max_steps), env.T)
        self.coins_per_eval = int(coins_per_eval)
        self.save_obs_chance = float(save_obs_chance)
        self.archive = None if archive is None else np.asarray(archive, dtype=np.float64)
        self.nov_k = int(nov_k)
        self.rank_streams = list(rank_streams) if rank_streams is not None else None
        self.rollout_mode = rollout_mode
        self.fuse_activations = bool(fuse_activations)
        self.fuse_noisy_terminal = bool(fuse_noisy_terminal)
        if isinstance(episodes, bool) or not isinstance(episodes, (int, np.integer)):
            raise TypeError(f'episodes must be an integer, got {episodes!r}')
        if episodes < 0:
            raise ValueError(f'episodes must be >= 0 (0 means 1, as max(1, eps_per_policy) in obj.py), got {episodes}')
        self.episodes = max(1, int(episodes))
        if result is None:
            result = RewardResult if self.archive is None else NSRResult
        if not any(result is c for c in _OBJECTIVES):
            raise ValueError(f'result must be one of {", ".join(c.__name__ for c in _OBJECTIVES)}, got {result!r}')
        novelty = result in (NSResult, NSRResult)
        if novelty and self.archive is None:
            raise ValueError(f'{result.__name__} scores the novelty of the final position: it needs an archive')
        if self.archive is not None and not novelty:
            raise ValueError(f'an archive is the novelty search\'s: {result.__name__} does not read it (use NSResult or NSRResult)')
        self.result = result
        self.objective = _OBJECTIVES[result]
        if self.episodes > 1 and self.archive is not None:
            raise ValueError('episodes > 1 with a novelty archive: no reference script averages episodes for novelty search')
        self._gen = None            # cached DeviceGeneration (see core.es)
        self._streams_in_use = None  # the RandomState streams of the last batched evaluation (set by core.es)
        self.stream_env_from_host = False   # True: re-upload the env's obs/reward streams every generation

    @property
    def n_obj(self) -> int:
        return 2 if self.result is NSRResult else 1

    def _result(self, rews, behv, obs, steps) -> TrainingResult:
        """The adaptor as the scripts build it (nsra.py:93 hands the novelty adaptors the last position only)."""
        if self.result in (NSResult, NSRResult):
            return self.result(rews, behv[-3:], obs, steps, self.archive, self.nov_k)
        return self.result(rews, behv, obs, steps)

    def result_from_device(self, total: float, pos, steps: Optional[int] = None) -> TrainingResult:
        """The TrainingResult ``__call__`` would build, from an episode total and final position computed on the device.
        ``steps``: the step t_d at which the episode ended on an env whose episodes end early; None, the episode ran
        ``max_steps`` steps."""
        rews = [float(total)]
        behv = [float(pos[0]), float(pos[1]), float(pos[2])] * int(self.max_steps)
        no_obs = np.array([np.zeros(self.env.observation_space.shape)])
        if steps is None:
            steps = self.max_steps - 1                          # run_model returns the last loop index (gym_runner.py:50,67)
        return self._result(rews, behv, no_obs, int(steps))

    @property
    def terminates(self) -> bool:
        """Whether the env's episodes can end before ``max_steps`` (``ClosedLoopEnv(fall_height=h)``)."""
        return bool(getattr(self.env, 'is_synthetic_closedloop', False) and getattr(self.env, 'terminates', False))

    def __call__(self, model, use_ac_noise=True) -> TrainingResult:
        """Single-policy evaluation with the reference's fit_fn contract.  Like the scripts' fit_fn (simple_example.py:38,
        obj.py:54) it first draws the save_obs coin(s) -- from every stream this process carries: each stream is one
        reference rank, and every rank runs its own noiseless evaluation (es.py:48).  ``use_ac_noise`` (obj.py:53-55): the
        rollout draws the policy's action noise from the first stream; es.step's noiseless call passes False."""
        streams = self.rank_streams if self.rank_streams is not None else self._streams_in_use
        if streams is not None:
            for rs in streams:
                for _ in range(self.coins_per_eval):
                    rs.random()
        noise_rs = streams[0] if (use_ac_noise and streams is not None and len(streams)) else None
        head = model.head() if hasattr(model, 'head') else None
        activation = self.fused_activation(model) if head is None else None
        if activation is not None:
            head = 'tanh'                                   # the outputs are the actions
        noisy = noise_rs is not None and float(getattr(model, '_action_std', 0) or 0) != 0
        episodes = self.episodes if noisy else 1
        if head is not None and (getattr(self.env, 'is_synthetic_openloop', False)
                                 or self._closed_on_device(model.layer_sizes(), head, activation)):
            # the evaluation, all its episodes, as one launch (the observations are not returned: this result never carries them)
            from .gym_runner import _device_episode
            total, pos, ran = _device_episode(model, self.env, self.max_steps, noise_rs if noisy else None, episodes, activation)
            return self.result_from_device(total, pos, ran - 1 if self.terminates else None)
        if episodes > 1:
            rews, behv, steps = self._run_episodes(model, noise_rs, episodes)
        else:
            rews, behv, obs, steps = run_model(model, self.env, self.max_steps, noise_rs)
        no_obs = np.array([np.zeros(self.env.observation_space.shape)])
        return self._result(rews, behv, no_obs, steps)

    def fused_activation(self, model):
        """The ``nn.Activation`` (not tanh) this object rolls ``model`` out with on the device, or None: only with
        ``fuse_activations`` and a network whose ``BaseNet.activation`` is one."""
        if not self.fuse_activations or not hasattr(model, 'activation'):
            return None
        act = model.activation()
        return None if act is None or act.kind == _lib.ES_ACT_TANH else act

    def _closed_on_device(self, sizes, head='tanh', activation=None) -> bool:
        """Whether a closed-loop episode of a tanh MLP runs as one launch (es_rollout_closedloop_mlp): two hidden layers always
        do (a shape outside the kernels' coverage raises there); three or four when the kernels cover the shape; anything else
        runs run_model's python loop.  A binned head (es_rollout_closedloop_mlp_binned) runs as one launch when the cluster
        kernel covers the shape, and so does a policy with another activation (es_rollout_closedloop_mlp_activation).  On an env
        whose episodes end early every policy runs the cluster kernel (es_rollout_closedloop_terminal) when it covers the
        shape."""
        n_hidden = len(sizes) - 2
        if n_hidden == 2 and head == 'tanh' and activation is None and not self.terminates:
            return True
        if n_hidden not in (2, 3, 4):
            return False
        from ..engine import get_engine
        try:
            get_engine().closed_mlp_plan(sizes, self.env.band, head, activation)
        except _lib.EsLibraryError:
            return False
        return True

    def _run_episodes(self, model, rs, episodes: int):
        """obj.py:57-60 with action noise for a policy ``__call__`` does not run on the device: ``episodes`` runs of run_model
        drawing from ``rs``, rewards summed per step in float64 in episode order and divided by the count."""
        rews = np.zeros(self.max_steps)
        for _ in range(episodes):
            rew, behv, _, steps = run_model(model, self.env, self.max_steps, rs)
            rews[:len(rew)] += np.array(rew)
        rews /= episodes
        return rews.tolist(), behv, steps
