"""Dev tool: closed-loop generations with action noise (es_draw_noisy + es_rollout_closedloop_mlp_episodes) at each shipped
config's policy, population K, episode length T, ac_std and episodes E (flagrun: E = 10) on a ClosedLoopEnv of the policy's
obs / act (band 8), plus bench.py's closed-loop shape 376-64-64-17 on the one-CTA kernel.  Per row, alternating in one process
a DeviceGeneration with the config's ac_std and one with ac_std = 0 (same K, T, E, 8 virtual-rank streams): CUDA-event ms of
the draw and of the rollout (the kernel groups DeviceGeneration.enable_timers brackets), pairs/s of the rollout, and the noise
buffer's size.  The card's name, power limit and max SM clock head the output.  ROWS=name,... picks rows; REPS (ns: NS_REPS)."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.generation import DeviceGeneration
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
from es_pytorch_b200.nn.optimizers import Adam

ROWS = [  # (name, sizes, pairs K, T, ac_std, E)
    ('simple_conf', [15, 256, 256, 3], 2400, 1000, 0.01, 1),
    ('nsra', [15, 256, 256, 3], 4800, 2000, 0.01, 1),
    ('obj', [17, 256, 256, 256, 6], 320, 1000, 0.01, 1),
    ('ns', [28, 256, 256, 256, 8], 2400, 10000, 0.05, 1),
    ('flagrun', [28, 128, 256, 256, 128, 8], 600, 500, 0.01, 10),
    ('control', [376, 64, 64, 17], 2400, 1000, 0.01, 1),
]
REPS = int(os.environ.get('REPS', 3))
NS_REPS = int(os.environ.get('NS_REPS', 1))
STREAMS = 8
want = os.environ.get('ROWS')
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}', flush=True)

L = 20_000_000
table = torch.randn(L, generator=torch.Generator(device=eng.device).manual_seed(1), device=eng.device)


def ms(gen, name):
    return sum(a.elapsed_time(b) for a, b in gen.timers[name])


for name, sizes, K, T, ac_std, E in ROWS:
    if want and name not in want.split(','):
        continue
    obs, act = sizes[0], sizes[-1]
    P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
    env = ClosedLoopEnv(obs, act, T)
    obs_dev, rew = env.device_arrays(eng)
    closed = env.device_closed(eng)
    theta = eng.to_device((np.random.RandomState(len(name)).randn(P) * 0.03).astype(np.float32))
    n = K // STREAMS
    gens = {}
    for s in (ac_std, 0.0):
        gens[s] = DeviceGeneration(table, theta, sizes, obs_dev[:T + 1].contiguous(), rew[:T].contiguous(),
                                   [np.random.RandomState(100 + r) for r in range(STREAMS)], 0.02, 0.0, Adam(P, 0.01),
                                   coins_per_eval=1, save_obs_chance=0.01, engine=eng, ac_std=s, closed=closed, episodes=E,
                                   closed_act_noise=True)
        gens[s].evaluate(n)                            # warm-up (buffers, modules)
    eng.sync()
    t = {s: ([], []) for s in gens}
    for _ in range(NS_REPS if name == 'ns' else REPS):
        for s, gen in gens.items():                    # noisy and noise-free alternate
            gen.enable_timers()
            gen.evaluate(n)
            eng.sync()
            t[s][0].append(ms(gen, 'draw_indices'))
            t[s][1].append(ms(gen, 'rollout'))
    (dn, rn), (d0, r0) = (np.array(v) for v in t[ac_std]), (np.array(v) for v in t[0.0])
    C = eng.closed_mlp_plan(sizes, env.band)[0]
    print(f'{name:12s} {"-".join(map(str, sizes)):22s} K={K:5d} T={T:6d} E={E:2d} ac_std={ac_std}: '
          f'noisy draw {dn.mean():8.2f} ms rollout {rn.mean():10.2f} ms (min {rn.min():.2f}, max {rn.max():.2f})  |  '
          f'ac_std=0 draw {d0.mean():6.2f} ms rollout {r0.mean():10.2f} ms (min {r0.min():.2f}, max {r0.max():.2f})  |  '
          f'rollout noisy / clean {rn.mean() / r0.mean():.3f}, {K / rn.mean() * 1e3:8.0f} pairs/s noisy, '
          f'{K / r0.mean() * 1e3:8.0f} clean  |  noise buffer {K * 2 * E * T * act * 4 / 2 ** 20:.0f} MiB  |  '
          f'{"one CTA per pair" if C == 0 else f"C = {C}"}  ({len(rn)} reps)', flush=True)
    del gens
    torch.cuda.empty_cache()
