"""Dev tool: the closed-loop rollout (es_rollout_closedloop_mlp) at the shipped configs' policies, populations and episode lengths,
on a ClosedLoopEnv of each policy's obs / act (band 8), E = 1 and ac_std = 0; plus a Humanoid-shaped wide policy and, as a control,
376-64-64-17 (bench.py's closed-loop workload, which runs rollout_closed.cu).  Per row: CUDA-event ms per rollout after a
warm-up (REPS repetitions, ns: NS_REPS), pairs/s, the cluster size C and the clusters resident at once.  ROWS=name,... picks rows."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv

ROWS = [  # (name, sizes, pairs K, T)
    ('simple_conf', [15, 256, 256, 3], 2400, 1000),
    ('nsra', [15, 256, 256, 3], 4800, 2000),
    ('obj', [17, 256, 256, 256, 6], 320, 1000),
    ('ns', [28, 256, 256, 256, 8], 2400, 10000),
    ('flagrun', [28, 128, 256, 256, 128, 8], 600, 500),
    ('humanoid_wide', [376, 256, 256, 17], 2400, 1000),
    ('control', [376, 64, 64, 17], 2400, 1000),
]
REPS = int(os.environ.get('REPS', 3))
NS_REPS = int(os.environ.get('NS_REPS', 1))
want = os.environ.get('ROWS')
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}', flush=True)

L = 20_000_000
g = torch.Generator(device=eng.device).manual_seed(1)
table = torch.randn(L, generator=g, device=eng.device)
for name, sizes, K, T in ROWS:
    if want and name not in want.split(','):
        continue
    obs, act = sizes[0], sizes[-1]
    P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
    env = ClosedLoopEnv(obs, act, T)
    _, rew = env.device_arrays(eng)
    obs0, env_a, env_b = env.device_closed(eng)
    rs = np.random.RandomState(len(name))
    theta = eng.to_device((rs.randn(P) * 0.03).astype(np.float32))
    idx = eng.to_device(rs.randint(0, L - P, size=K).astype(np.int64))
    mean, std = eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs))
    fit = torch.zeros(2, K, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, K, 3, dtype=torch.float32, device=eng.device)
    C, clusters, smem = eng.closed_mlp_plan(sizes, env.band)

    def run(n):
        eng.rollout_closed_mlp(table, idx[:n], theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew[:T].contiguous(), 0.05,
                               fit[0, :n], fit[1, :n], 1, behv[0, :n].reshape(-1), behv[1, :n].reshape(-1))

    run(min(K, 64))                                    # warm-up
    eng.sync()
    times = []
    for _ in range(NS_REPS if name == 'ns' else REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); run(K); b.record()
        eng.sync()
        times.append(a.elapsed_time(b))
    t = np.array(times)
    kernel = 'rollout_closed.cu (one CTA per pair)' if C == 0 else f'C = {C} CTAs per evaluation, {smem / 1024:.1f} KiB each'
    print(f'{name:14s} {"-".join(map(str, sizes)):22s} K={K:5d} T={T:6d}: {t.mean():10.2f} ms (min {t.min():.2f}, max {t.max():.2f}, '
          f'{len(t)} reps)  {K / t.mean() * 1e3:9.0f} pairs/s  {kernel}, {clusters} resident {"CTAs" if C == 0 else "clusters"}',
          flush=True)
    del fit, behv
