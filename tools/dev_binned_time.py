"""Dev tool: binned-action policies (FFBinned) on the device at the shipped configs' trunks, with bins 5 and 11.
Open loop: es_rollout_openloop_binned in ES_ROLLOUT_F32 (the float32 kernel of rollout_f32.cu) and ES_ROLLOUT_TC3 (rollout_tcw.cu),
next to the same trunk with a tanh head of adim outputs in the same mode (ES_F32_GENERAL=1 is set, so obs-64-64-act trunks would
not take the packed-FMA kernel either).
Closed loop: es_rollout_closedloop_mlp_binned (rollout_closedw.cu's cluster kernel).  Per row: CUDA-event ms per rollout after a
warm-up (REPS repetitions), pairs/s, and for the closed loop the cluster size and the clusters resident at once.  The card, its
power limit and its max SM clock are printed first.  ROWS=name,... picks rows."""
import os, subprocess, sys
os.environ.setdefault('ES_F32_GENERAL', '1')
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200._lib import ES_ROLLOUT_F32, ES_ROLLOUT_TC3
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv, SyntheticEnv
from es_pytorch_b200.nn.nn import BinnedHead

OPEN = [  # (name, obs, hidden, adim, pairs K, T)
    ('simple_conf', 15, [256, 256], 3, 2400, 1000),
    ('obj', 17, [256, 256, 256], 6, 320, 1000),
    ('flagrun', 28, [128, 256, 256, 128], 8, 600, 500),
]
CLOSED = [
    ('simple_conf', 15, [256, 256], 3, 2400, 1000),
    ('obj', 17, [256, 256, 256], 6, 320, 1000),
]
BINS = (5, 11)
REPS = int(os.environ.get('REPS', 3))
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


def timed(run, K):
    run(min(K, 64))                                    # warm-up
    eng.sync()
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); run(K); b.record()
        eng.sync()
        times.append(a.elapsed_time(b))
    return np.array(times)


def line(kind, name, sizes, K, T, t, extra=''):
    print(f'{kind:6s} {name:12s} {"-".join(map(str, sizes)):24s} K={K:5d} T={T:5d}: {t.mean():9.2f} ms (min {t.min():.2f}, '
          f'max {t.max():.2f}, {len(t)} reps) {K / t.mean() * 1e3:9.0f} pairs/s {extra}', flush=True)


for name, obs, hidden, adim, K, T in OPEN:
    if want and name not in want.split(','):
        continue
    env = SyntheticEnv(obs, adim, T)
    obs_dev, rew = env.device_arrays(eng)
    obsn = eng.normalise_obs(obs_dev[:T].contiguous(), eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs)), 5.0)
    rew = rew[:T].contiguous()
    fit = torch.zeros(2, K, dtype=torch.float64, device=eng.device)
    for mode, mname in ((ES_ROLLOUT_F32, 'F32'), (ES_ROLLOUT_TC3, 'TC3')):
        for bins in (None,) + BINS:
            head = None if bins is None else BinnedHead(bins, env.action_space.low, env.action_space.high)
            sizes = [obs, *hidden, adim * (bins or 1)]
            P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
            rs = np.random.RandomState(len(name))
            theta = eng.to_device((rs.randn(P) * 0.05).astype(np.float32))
            idx = eng.to_device(rs.randint(0, L - P, size=K).astype(np.int64))

            def run(n):
                eng.rollout(table, idx[:n], theta, 0.02, sizes, obsn, rew, 0.05, fit[0, :n], fit[1, :n], mode=mode, head=head)

            line('open', name, sizes, K, T, timed(run, K), f'{mname}, ' + ('tanh head' if bins is None else f'bins {bins}'))

for name, obs, hidden, adim, K, T in CLOSED:
    if want and name not in want.split(','):
        continue
    env = ClosedLoopEnv(obs, adim, T)
    _, rew = env.device_arrays(eng)
    rew = rew[:T].contiguous()
    obs0, env_a, env_b = env.device_closed(eng)
    mean, std = eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs))
    fit = torch.zeros(2, K, dtype=torch.float64, device=eng.device)
    for bins in BINS:
        head = BinnedHead(bins, env.action_space.low, env.action_space.high)
        sizes = [obs, *hidden, adim * bins]
        P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
        rs = np.random.RandomState(len(name))
        theta = eng.to_device((rs.randn(P) * 0.03).astype(np.float32))
        idx = eng.to_device(rs.randint(0, L - P, size=K).astype(np.int64))
        C, clusters, smem = eng.closed_mlp_plan(sizes, env.band, head)

        def run(n):
            eng.rollout_closed_mlp(table, idx[:n], theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew, 0.05, fit[0, :n],
                                   fit[1, :n], head=head)

        line('closed', name, sizes, K, T, timed(run, K), f'bins {bins}, C = {C}, {clusters} resident clusters')
