"""Dev tool: policies with ReLU, leaky-ReLU, ELU and sigmoid activations (es_rollout_*_activation) timed against tanh, the kinds
alternating within each row.  Open loop: ES_ROLLOUT_F32 and ES_ROLLOUT_TC3 at config 3 (376-64-64-17, K = 10 000, T = 1000:
tanh runs the headline kernels, rollout_f32x.cu and rollout_tc2.cu, the other kinds the general float32 kernel and, where
obs <= 256, the wide tensor-core kernel's code) and at the shipped shapes (simple_conf, obj, flagrun).  Closed loop: the cluster
kernel (rollout_closedw.cu) at simple_conf and obj.  Per row and kind: CUDA-event ms per rollout after a
warm-up (REPS rounds, kinds interleaved) and pairs/s; a kind a mode refuses prints the refusal.  The card, its power limit and
its max SM clock are printed first.  ROWS=name,... picks rows."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200 import _lib
from es_pytorch_b200._lib import ES_ROLLOUT_F32, ES_ROLLOUT_TC3
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
from es_pytorch_b200.nn.nn import Activation

OPEN = [  # (name, sizes, pairs K, T)
    ('config3', [376, 64, 64, 17], 10_000, 1000),
    ('simple_conf', [15, 256, 256, 3], 2400, 1000),
    ('obj', [17, 256, 256, 256, 6], 320, 1000),
    ('flagrun', [28, 128, 256, 256, 128, 8], 600, 500),
]
CLOSED = [('simple_conf', [15, 256, 256, 3], 2400, 1000), ('obj', [17, 256, 256, 256, 6], 320, 1000)]
KINDS = [('tanh', Activation(_lib.ES_ACT_TANH, 0.0)), ('relu', Activation(_lib.ES_ACT_RELU, 0.0)),
         ('leaky', Activation(_lib.ES_ACT_LEAKY_RELU, float(np.float32(0.01)))), ('elu', Activation(_lib.ES_ACT_ELU, 1.0)),
         ('sigmoid', Activation(_lib.ES_ACT_SIGMOID, 0.0))]
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


def theta_for(sizes, seed=0):
    """Weights of scale 1 / sqrt(fan_in): hidden values of order 1 for every kind (TC3's float16 operands hold them)."""
    rs = np.random.RandomState(seed)
    parts = [rs.randn(fi * fo + fo) / np.sqrt(fi) for fi, fo in zip(sizes[:-1], sizes[1:])]
    return eng.to_device(np.concatenate(parts).astype(np.float32))


def rounds(runs, K):
    """runs: {kind: callable(K)}; the kinds alternate within every round.  Returns {kind: ms array} or the refusal text."""
    out = {}
    for k, run in runs.items():
        try:
            run(min(K, 64))                                # warm-up
            eng.sync()
            out[k] = []
        except _lib.EsLibraryError as e:
            out[k] = str(e).split(': ', 2)[-1][:90]
    for _ in range(REPS):
        for k, run in runs.items():
            if isinstance(out[k], str):
                continue
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); run(K); b.record()
            eng.sync()
            out[k].append(a.elapsed_time(b))
    return {k: (np.array(v) if isinstance(v, list) else v) for k, v in out.items()}


def report(kind, name, sizes, K, T, res):
    for k, t in res.items():
        if isinstance(t, str):
            print(f'{kind:10s} {name:12s} {"-".join(map(str, sizes)):24s} {k:8s} refused: {t}', flush=True)
        else:
            print(f'{kind:10s} {name:12s} {"-".join(map(str, sizes)):24s} {k:8s} K={K:5d} T={T:5d}: {t.mean():9.2f} ms '
                  f'(min {t.min():.2f}, max {t.max():.2f}) {K / t.mean() * 1e3:9.0f} pairs/s', flush=True)


for name, sizes, K, T in OPEN:
    if want and name not in want.split(','):
        continue
    rs = np.random.RandomState(2)
    obsn = eng.to_device(np.clip(rs.randn(T, sizes[0]), -5, 5).astype(np.float32))
    rew = eng.to_device(rs.randn(T, sizes[-1]).astype(np.float32))
    idx = eng.to_device(rs.randint(0, L - 2_000_000, size=K).astype(np.int64))
    theta = theta_for(sizes)
    fit = torch.zeros((2, K), dtype=torch.float64, device=eng.device)
    for mode, mname in ((ES_ROLLOUT_F32, 'open F32'), (ES_ROLLOUT_TC3, 'open TC3')):
        runs = {k: (lambda n, a=a, m=mode: eng.rollout(table, idx[:n], theta, 0.02, sizes, obsn, rew, 0.05, fit[0, :n],
                                                        fit[1, :n], 1, None, None, m, activation=None if a.kind == 0 else a))
                for k, a in KINDS}
        report(mname, name, sizes, K, T, rounds(runs, K))

for name, sizes, K, T in CLOSED:
    if want and name not in want.split(','):
        continue
    env = ClosedLoopEnv(sizes[0], sizes[-1], T)
    obs0, env_a, env_b = env.device_closed(eng)
    _, rew_dev = env.device_arrays(eng)
    rew = rew_dev[:T].contiguous()
    rs = np.random.RandomState(3)
    idx = eng.to_device(rs.randint(0, L - 2_000_000, size=K).astype(np.int64))
    theta = theta_for(sizes)
    mean = torch.zeros(sizes[0], dtype=torch.float64, device=eng.device)
    std = torch.ones(sizes[0], dtype=torch.float64, device=eng.device)
    fit = torch.zeros((2, K), dtype=torch.float64, device=eng.device)
    runs = {k: (lambda n, a=a: eng.rollout_closed_mlp(table, idx[:n], theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew,
                                                       0.05, fit[0, :n], fit[1, :n], 1, activation=None if a.kind == 0 else a))
            for k, a in KINDS}
    plans = {k: eng.closed_mlp_plan(sizes, env.band, activation=None if a.kind == 0 else a) for k, a in KINDS}
    report('closed', name, sizes, K, T, rounds(runs, K))
    print(f'           (cluster size, resident clusters, smem bytes): {plans}', flush=True)
