"""Shared noise table (mirror of src/core/noisetable.py:27-91), resident in HBM.

The reference keeps one float32 table per node in an MPI-3 shared-memory window
(noisetable.py:13-24); here every GPU holds a full replica in its own HBM (1 GB of 180 GB
for the shipped 250 M-float configs), drawn there by ``create_shared``, and a host copy backs
the numpy-facing API (``get`` returns views, ``noise`` is an ndarray -- both part of the
reference contract), downloaded the first time it is read.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import numpy as np
import torch


class NoiseTable:
    def __init__(self, n_params: int, noise):
        self.n_params: int = n_params
        self._host: Optional[np.ndarray] = None
        self._dev: Optional[torch.Tensor] = None
        if isinstance(noise, torch.Tensor):
            if noise.is_cuda:
                self._dev = noise.contiguous()
            else:
                self._host = noise.numpy()
        else:
            self._host = noise
        self._size = int(noise.numel() if isinstance(noise, torch.Tensor) else len(noise))

    # -- the two residencies -------------------------------------------------------------------
    @property
    def noise(self) -> np.ndarray:
        if self._host is None:
            self._host = self._dev.cpu().numpy()
        return self._host

    def device_table(self, engine) -> torch.Tensor:
        """float32 table in this GPU's HBM (uploaded on first use)."""
        if self._dev is None or self._dev.device != engine.device:
            self._dev = engine.to_device(np.ascontiguousarray(self.noise), torch.float32)
        return self._dev

    # -- reference API ---------------------------------------------------------------------------
    def get(self, i, size) -> np.ndarray:
        assert len(self) > i + size, 'trying to index outside the range of the noise table'
        return self.noise[i:i + size]

    def sample_idx(self, rs: np.random.RandomState, size: int):
        upper_bound = len(self) - size
        if upper_bound <= 0:
            raise ValueError(f'Network (size:{size}) is too large for noise table (size:{len(self)})')
        return rs.randint(0, upper_bound)

    def sample(self, rs: np.random.RandomState = None, size=None) -> Tuple[int, np.ndarray]:
        size = self.n_params if size is None else size
        rs = np.random.RandomState() if rs is None else rs
        idx = self.sample_idx(rs, size)
        return idx, self.get(idx, size)

    def __getitem__(self, item) -> np.ndarray:
        return self.get(item, self.n_params)

    def __len__(self):
        return self._size

    def __call__(self, *args, **kwargs) -> Tuple[int, np.ndarray]:
        return self.sample()

    @staticmethod
    def _random_state(seed, gym_seeding: bool) -> np.random.RandomState:
        if gym_seeding:
            from gym.utils import seeding
            try:
                rs, _ = seeding.np_random(seed, hashed=True)          # the shim's restatement of gym 0.17.1's seed hashing
            except TypeError:
                rs, _ = seeding.np_random(seed)                       # a real gym installation
            return rs
        return np.random.RandomState(seed)

    @staticmethod
    def make_noise(size: int, seed=None, gym_seeding: bool = False) -> np.ndarray:
        """Table content.  Default = what the reference's own test asserts
        (test/es/noisetable_test.py:26): ``RandomState(seed).randn(size)`` as float32.
        ``gym_seeding=True`` routes the seed through ``gym.utils.seeding.np_random`` like
        noisetable.py:61-64 (needs a gym that provides it; the two disagree in gym 0.17)."""
        return NoiseTable._random_state(seed, gym_seeding).randn(size).astype(np.float32)

    @staticmethod
    def make_noise_device(size: int, seed=None, gym_seeding: bool = False, engine=None) -> torch.Tensor:
        """``make_noise`` drawn on the GPU (es_randn): the RandomState is seeded on the host exactly as ``make_noise``
        seeds it, its 624-word key and position go to the device, and the ``size`` gaussians are drawn there in numpy's
        stream order.  Equal to ``make_noise`` except that a value can be one float32 ulp off when its float64 value lies
        next to a float32 rounding midpoint (CUDA's log is not glibc's; about one value in 2^28)."""
        from ..engine import get_engine
        eng = engine or get_engine()
        _, key, pos, has_gauss, gauss = NoiseTable._random_state(seed, gym_seeding).get_state()
        st = [eng.to_device(np.asarray(key, dtype=np.uint32).view(np.int32)),
              eng.to_device(np.array([pos], dtype=np.int32)), eng.to_device(np.array([has_gauss], dtype=np.int32)),
              eng.to_device(np.array([gauss], dtype=np.float64))]
        return eng.randn(*st, size)

    @staticmethod
    def create_shared(global_comm, size: int, n_params: int, reporter=None, seed=None) -> 'NoiseTable':
        """noisetable.py:66-91 without the MPI window: rank 0 picks the seed, every process
        builds the identical table.  With a CUDA device and the library, every process draws
        its own replica on its GPU (``make_noise_device``: no host table until ``noise`` is
        read); ``ES_NOISE_TABLE_HOST=1``, or no device, builds it with numpy and uploads it on
        first device use."""
        from .. import _lib, dist
        if getattr(global_comm, 'rank', 0) == 0:
            seed = seed if seed is not None else np.random.randint(0, 1000000)
            if reporter is not None:
                reporter.print(f'nt seed:{seed}')
        if getattr(global_comm, 'size', 1) > 1:
            seed = dist.world().broadcast_object(seed, 0)
        if hasattr(seed, '__len__'):          # simple_example.py:34 passes cfg.general.seed (a list or None)
            seed = int(seed[0])
        if os.environ.get('ES_NOISE_TABLE_HOST') != '1' and torch.cuda.is_available() and os.path.exists(_lib.LIB_PATH):
            return NoiseTable(n_params, NoiseTable.make_noise_device(size, seed))
        return NoiseTable(n_params, NoiseTable.make_noise(size, seed))
