"""Dev tool: one generation with E episodes per evaluation (obj.py's eps_per_policy) and action noise (ac_std = 0.01) at the
bench size (K = 10 000 pairs, 376-64-64-17, T = 1000): es_draw_noisy and rollout time separately, pairs/s, and the
action-noise buffer.  RUNS = 'E:streams,...' (default 1:8,2:8,5:8,10:64), MODE = rollout mode (default 2 = TC3)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.generation import DeviceGeneration
from es_pytorch_b200.gym.synthetic_env import SyntheticEnv
from es_pytorch_b200.nn.optimizers import Adam

K = int(os.environ.get('K', 10000))
MODE = int(os.environ.get('MODE', 2))
RUNS = [tuple(int(v) for v in r.split(':')) for r in os.environ.get('RUNS', '1:8,2:8,5:8,10:64').split(',')]
eng = get_engine(0)
obs, act, T = 376, 17, 1000
sizes = [obs, 64, 64, act]; P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
g = torch.Generator(device=eng.device).manual_seed(1)
table = torch.randn(50_000_000, generator=g, device=eng.device)
env = SyntheticEnv(obs, act, T)
obs_dev, rew_dev = env.device_arrays(eng)
theta0 = (np.random.RandomState(7).randn(P) * 0.1).astype(np.float32)
print(f'{torch.cuda.get_device_name(eng.device)}, K={K}, {"-".join(map(str, sizes))}, T={T}, ac_std=0.01, mode={MODE}', flush=True)
for E, R in RUNS:
    gen = DeviceGeneration(table, eng.to_device(theta0.copy()), sizes, obs_dev, rew_dev,
                           [np.random.RandomState(1000 + r) for r in range(R)], 0.02, 0.005, Adam(P, 0.01), coins_per_eval=1,
                           save_obs_chance=0.01, rollout_mode=MODE, engine=eng, ac_std=0.01, episodes=E)
    gen.run(K // R); torch.cuda.synchronize()
    gen.enable_timers(True)
    n0 = eng.launches
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(3):
        gen.run(K // R)
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 3
    kern = {k: float(np.mean([x.elapsed_time(y) for x, y in v])) for k, v in gen.timers.items()}
    noise_gb = gen.act_noise.numel() * 4 / 1e9
    print(f'E={E:2d} R={R:2d}: {ms:8.2f} ms/generation ({K / ms * 1e3 / 1e6:.3f} M pairs/s); draw {kern["draw_indices"]:8.2f} ms, '
          f'rollout {kern["rollout"]:7.2f} ms; noise buffer {noise_gb:.2f} GB; {(eng.launches - n0) / 3:.0f} launches/generation; '
          f'peak allocated by torch {torch.cuda.max_memory_allocated(eng.device) / 1e9:.1f} GB', flush=True)
    del gen
    torch.cuda.empty_cache()
