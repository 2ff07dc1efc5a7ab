"""Policy networks (mirror of src/nn/nn.py:9-50): ``BaseNet`` and ``FeedForward``.

The modules are the *description* of the policy (layer sizes, activation, observation
statistics, action noise); the batched evaluation of perturbed copies happens in
``es_rollout_openloop`` which reads the same flat parameter layout
(state_dict order: weight[out,in] row-major then bias, policy.py:33-35).
``forward`` keeps the reference contract (``model(ob, rs=rs)``) for user code that steps
an arbitrary gym env itself.
"""
from __future__ import annotations

from abc import ABC
from typing import List, NamedTuple, Optional, Union

import numpy as np
import torch
from torch import nn, Tensor


_BINNED_MAX_OUT = 256          # adim * bins the binned kernels take (es_rollout_openloop_binned, es_rollout_closedloop_mlp_binned)


class BinnedHead(NamedTuple):
    """FFBinned's head as the fused rollouts take it: ``bins`` outputs per action dimension, the action
    ``1 / (bins - 1) * argmax * (high - low) + low`` in float32 (nn.py:114-117)."""
    bins: int
    low: np.ndarray                 # float32 [adim]
    high: np.ndarray                # float32 [adim]

    @property
    def adim(self) -> int:
        return int(self.low.shape[0])

    def key(self) -> tuple:
        """What identifies the head's arithmetic (a cache key)."""
        return ('binned', self.bins, self.low.tobytes(), self.high.tobytes())

    def device_arrays(self, engine):
        """(low, high - low) as float32 device tensors; ``high - low`` is rounded to float32 as FFBinned.forward's ac_range."""
        low = np.ascontiguousarray(self.low, dtype=np.float32)
        rng = np.ascontiguousarray(np.asarray(self.high, dtype=np.float32) - low, dtype=np.float32)
        return engine.to_device(low), engine.to_device(rng)


class Activation(NamedTuple):
    """The activation a FeedForward applies after every layer, as the fused rollouts take it (es_rollout_*_activation):
    ``kind`` one of the ``_lib.ES_ACT_*`` constants, ``param`` LeakyReLU's negative slope or ELU's alpha rounded to float32
    (torch's CPU kernels compute with the float32 value; 0 for the other kinds)."""
    kind: int
    param: float

    def key(self) -> tuple:
        """What identifies the activation's arithmetic (a cache key)."""
        return ('activation', int(self.kind), float(self.param))


def _activation_of(m: nn.Module) -> Optional[Activation]:
    """The Activation of one torch module, None for a module the kernels do not evaluate (subclasses included: they may
    override forward)."""
    from .._lib import ES_ACT_ELU, ES_ACT_LEAKY_RELU, ES_ACT_RELU, ES_ACT_SIGMOID, ES_ACT_TANH
    kind = {nn.Tanh: ES_ACT_TANH, nn.ReLU: ES_ACT_RELU, nn.LeakyReLU: ES_ACT_LEAKY_RELU, nn.ELU: ES_ACT_ELU,
            nn.Sigmoid: ES_ACT_SIGMOID}.get(type(m))
    if kind is None:
        return None
    param = 0.0
    if kind == ES_ACT_LEAKY_RELU:
        param = float(np.float32(m.negative_slope))
    elif kind == ES_ACT_ELU:
        param = float(np.float32(m.alpha))
    if not np.isfinite(param):
        return None
    return Activation(kind, param)


class BaseNet(nn.Module, ABC):
    def __init__(self, layers: List[nn.Module], ob_shape: tuple, ob_clip: float = 5):
        super().__init__()
        self.model = nn.Sequential(*layers)
        self._obmean: np.ndarray = np.zeros(ob_shape)
        self._obstd: np.ndarray = np.ones(ob_shape)
        self.ob_clip = ob_clip

    def set_ob_mean_std(self, mean: np.ndarray, std: np.ndarray):
        self._obmean = mean
        self._obstd = std

    def layer_sizes(self) -> List[int]:
        """[in, h1, ..., out] of the Linear stack (what the rollout kernel needs)."""
        lin = [m for m in self.model if isinstance(m, nn.Linear)]
        return [lin[0].in_features] + [m.out_features for m in lin]

    def is_tanh_mlp(self) -> bool:
        """True for the networks the fused rollout kernels evaluate: Linear + Tanh after every layer with the plain
        FeedForward forward (subclasses that post-process the outputs -- integrated gaussian actions, binned actions --
        are stepped through their own forward)."""
        if type(self).forward is not FeedForward.forward:
            return False
        return self._tanh_stack()

    def _tanh_stack(self) -> bool:
        mods = list(self.model)
        return (len(mods) % 2 == 0 and all(isinstance(m, nn.Linear) for m in mods[0::2])
                and all(isinstance(m, nn.Tanh) for m in mods[1::2]))

    def activation(self) -> Optional[Activation]:
        """The activation the fused rollouts evaluate for this network (es_rollout_*_activation): a plain-forward FeedForward
        whose stack is Linear layers each followed by the same kind of supported module (Tanh, ReLU, LeakyReLU, ELU, Sigmoid)
        with the same float32 parameter.  None for anything else: mixed activations, other modules, FFBinned,
        FFIntegGausAction* and subclasses with their own forward.  Tanh networks give ``Activation(ES_ACT_TANH, 0.0)``; they
        are fused by default (``head``), the other kinds only where a ``BatchedRollout(fuse_activations=True)`` asks for it."""
        if type(self).forward is not FeedForward.forward:
            return None
        mods = list(self.model)
        if len(mods) == 0 or len(mods) % 2 or not all(type(m) is nn.Linear for m in mods[0::2]):
            return None
        acts = {_activation_of(m) for m in mods[1::2]}
        if len(acts) != 1 or None in acts:
            return None
        return acts.pop()

    def head(self) -> Optional[Union[str, BinnedHead]]:
        """How the fused rollout kernels turn this network's outputs into actions: ``'tanh'`` for the tanh MLPs of
        ``is_tanh_mlp`` (the outputs are the actions), a ``BinnedHead`` for an FFBinned the kernels evaluate exactly as its
        forward does, None for anything else (stepped through the module's own forward, as the reference does).

        An FFBinned is fused when it is a Linear + Tanh stack, its action bounds are float32 arrays of shape [adim] (with
        float64 bounds FFBinned.forward computes the action in float64 and rounds once; the kernels round every operation
        to float32), ``bins >= 2`` (the reference divides by ``bins - 1``), ``adim * bins <= 256`` outputs and every layer
        fits the float32 kernel's activation tiles (the limit ``es_rollout_openloop_binned`` refuses beyond)."""
        if self.is_tanh_mlp():
            return 'tanh'
        if type(self).forward is not FFBinned.forward or not self._tanh_stack():
            return None
        low, high = np.asarray(self.alow), np.asarray(self.ahigh)
        adim, bins = int(self.adim), int(self.bins)
        if low.dtype != np.float32 or high.dtype != np.float32 or low.shape != (adim,) or high.shape != (adim,):
            return None
        sizes = self.layer_sizes()
        if bins < 2 or sizes[-1] != adim * bins or sizes[-1] > _BINNED_MAX_OUT:
            return None
        if 2 * 32 * max((s + 3) & ~3 for s in sizes) * 4 + 32 * 8 > 227 * 1024:       # rollout_f32.cu's activation tiles
            return None
        return BinnedHead(bins, low.copy(), high.copy())


class FeedForward(BaseNet):
    def __init__(self, layer_sizes: List[int], activation: nn.Module, env, ac_std: float, ob_clip: float = 5):
        """layer_sizes are the hidden sizes; input/output come from the env spaces (nn.py:32)."""
        sizes = [int(np.prod(env.observation_space.shape))] + list(layer_sizes) + \
                [int(np.prod(env.action_space.shape))]
        stack = []
        for fan_in, fan_out in zip(sizes, sizes[1:]):
            stack.append(nn.Linear(fan_in, fan_out))
            stack.append(activation)            # activation after every layer, output included (nn.py:35-36)
        super().__init__(stack, env.observation_space.shape, ob_clip)
        self._action_std = ac_std

    def forward(self, inp: Tensor, **kwargs) -> Tensor:
        rs = kwargs['rs']
        mean = torch.as_tensor(self._obmean, dtype=torch.float64, device=inp.device)
        std = torch.as_tensor(self._obstd, dtype=torch.float64, device=inp.device)
        x = torch.clamp((inp.double() - mean) / std, min=-self.ob_clip, max=self.ob_clip)   # float64, nn.py:45
        a = self.model(x.float())
        if self._action_std != 0 and rs is not None:
            noise = torch.as_tensor(rs.randn(*a.shape) * self._action_std, device=a.device)   # nn.py:47-48
            a = (a.double() + noise).float()
        return a


def _normalised(net: BaseNet, inp: Tensor) -> Tensor:
    mean = torch.as_tensor(net._obmean, dtype=torch.float64, device=inp.device)
    std = torch.as_tensor(net._obstd, dtype=torch.float64, device=inp.device)
    return torch.clamp((inp.double() - mean) / std, min=-net.ob_clip, max=net.ob_clip).float()      # nn.py:45


class FFIntegGausAction(FeedForward):
    """The network's FIRST output is the std of the gaussian noise added to the remaining outputs (nn.py:53-75):
    ``act, std = out[1:], out[0]; act += rs.standard_normal(act.shape) * std``.  Returns an ndarray like the reference.
    Evaluated through its own forward in run_model's step loop: the noise scale is a network output, so the stream
    consumption is as in the reference but the rollout is not one of the fused kernels (SURVEY 8f.4)."""

    def forward(self, inp: Tensor, **kwargs) -> np.ndarray:
        rs = kwargs.get('rs')
        out = self.model(_normalised(self, inp)).detach().cpu().numpy()
        action, action_std = out[1:], out[0]
        if action_std != 0 and rs is not None:
            action = action + rs.standard_normal(*action.shape) * action_std
        return action


class FFIntegGausActionMulti(FeedForward):
    """First half of the outputs = action means, second half = their stds (absolute value) (nn.py:78-97)."""

    def forward(self, inp: Tensor, **kwargs) -> np.ndarray:
        rs = kwargs.get('rs')
        out = self.model(_normalised(self, inp)).detach().cpu().numpy()
        mid = len(out) // 2
        action, action_std = out[:mid], np.abs(out[mid:])
        if rs is not None:
            action = action + rs.standard_normal(*action.shape) * action_std
        return action


class FFBinned(BaseNet):
    """``n_bins`` outputs per action dimension; the action is the centre of the arg-max bin, spread evenly over the action
    space's [low, high] (nn.py:100-117)."""

    def __init__(self, layer_sizes: List[int], activation: nn.Module, env, n_bins: int, ob_clip=5):
        self.bins = n_bins
        self.adim, self.ahigh, self.alow = env.action_space.shape[0], env.action_space.high, env.action_space.low
        sizes = [int(np.prod(env.observation_space.shape))] + list(layer_sizes) + [self.adim * self.bins]
        stack = []
        for fan_in, fan_out in zip(sizes, sizes[1:]):
            stack += [nn.Linear(fan_in, fan_out), activation]
        super().__init__(stack, env.observation_space.shape, ob_clip)

    def forward(self, inp: Tensor, **kwargs) -> Tensor:
        a = self.model(_normalised(self, inp))
        ac_range = torch.as_tensor(self.ahigh - self.alow)[None, :]
        binned = a.reshape((-1, self.adim, self.bins)).argmax(2)
        return (1. / (self.bins - 1.) * binned * ac_range + torch.as_tensor(self.alow)[None, :]).squeeze()
