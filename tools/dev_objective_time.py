"""Dev tool: what the single-objective adaptors cost in a fused generation at BASELINE config 3 (376-64-64-17 tanh, T = 1000,
K = 10 000 pairs, sigma 0.02, ES_ROLLOUT_TC3, 8 virtual-rank streams, one save_obs coin per evaluation).

One DeviceGeneration per objective -- 'reward' (RewardResult), 'dist' (DistResult), 'novelty' (NSResult: k = 10 of a 64-entry
archive, as bench.py's NSRA workload) -- run in turns in one process, REPS rounds of one generation each after a warm-up
generation: CUDA-event ms per generation (evaluate + rank + reconstruction + Adam) and of the objective step alone
(es_fitness_objective or es_novelty on the 2K evaluations, after the rollout).  Then es_fitness_objective alone over 2K values,
LAUNCHES back-to-back launches per kind.  The card's name, power limit and max SM clock head the output."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from es_pytorch_b200 import _lib  # noqa: E402
from es_pytorch_b200.engine import get_engine  # noqa: E402
from es_pytorch_b200.generation import DeviceGeneration  # noqa: E402
from es_pytorch_b200.gym.synthetic_env import SyntheticEnv  # noqa: E402
from es_pytorch_b200.nn.optimizers import Adam  # noqa: E402

K = int(os.environ.get('K', 10000))
REPS = int(os.environ.get('REPS', 5))
LAUNCHES = int(os.environ.get('LAUNCHES', 2000))
STREAMS = 8
obs, act, T = 376, 17, 1000
sizes = [obs, 64, 64, act]
P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}; K={K}, {"-".join(map(str, sizes))}, T={T}, ES_ROLLOUT_TC3, {STREAMS} streams, REPS={REPS}', flush=True)

table = torch.randn(50_000_000, generator=torch.Generator(device=eng.device).manual_seed(1), device=eng.device)
env = SyntheticEnv(obs, act, T)
obs_dev, rew_dev = env.device_arrays(eng)
theta0 = (np.random.RandomState(7).randn(P) * 0.1).astype(np.float32)
archive = eng.to_device(np.random.RandomState(3).randn(64, 2) * 0.5, torch.float64)
gens = {}
for objective in ('reward', 'dist', 'novelty'):
    gens[objective] = DeviceGeneration(table, eng.to_device(theta0.copy()), sizes, obs_dev, rew_dev,
                                       [np.random.RandomState(1000 + r) for r in range(STREAMS)], 0.02, 0.005, Adam(P, 0.01),
                                       coins_per_eval=1, save_obs_chance=0.01, rollout_mode=_lib.ES_ROLLOUT_TC3, engine=eng,
                                       archive=archive if objective == 'novelty' else None, objective=objective)


class _TimedScore:
    """Brackets DeviceGeneration._score (the objective step) with CUDA events."""

    def __init__(self, gen):
        self.gen, self.inner, self.events = gen, gen._score, []

    def __call__(self):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self.inner()
        b.record()
        self.events.append((a, b))


for gen in gens.values():
    gen.run(K // STREAMS)                                  # warm-up: buffers, modules, float16 shadows
    gen._score = _TimedScore(gen)
torch.cuda.synchronize()
times = {k: [] for k in gens}
for _ in range(REPS):
    for name, gen in gens.items():                         # in turns: a drift of the clock hits every objective alike
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        gen.run(K // STREAMS)
        b.record()
        torch.cuda.synchronize()
        times[name].append(a.elapsed_time(b))
for name, gen in gens.items():
    t = np.array(times[name])
    sc = np.array([a.elapsed_time(b) for a, b in gen._score.events[-REPS:]])
    print(f'{name:8s}: generation median {np.median(t):8.2f} ms (min {t.min():8.2f}, max {t.max():8.2f}); objective step median '
          f'{np.median(sc) * 1e3:7.1f} us', flush=True)

fit = torch.randn(2 * K, dtype=torch.float64, device=eng.device)
behv = torch.randn(2 * K, 3, dtype=torch.float32, device=eng.device)
for kind, name in ((_lib.ES_OBJ_MEAN_REWARD, 'MEAN_REWARD'), (_lib.ES_OBJ_DIST, 'DIST'), (_lib.ES_OBJ_XDIST, 'XDIST')):
    for _ in range(10):
        eng.fitness_objective(kind, fit, 1, behv, 2 * K, T - 1)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(LAUNCHES):
        eng.fitness_objective(kind, fit, 1, behv, 2 * K, T - 1)
    b.record()
    torch.cuda.synchronize()
    print(f'es_fitness_objective {name:11s} over {2 * K} values: {a.elapsed_time(b) / LAUNCHES * 1e3:6.2f} us per launch '
          f'({LAUNCHES} back-to-back launches)', flush=True)
