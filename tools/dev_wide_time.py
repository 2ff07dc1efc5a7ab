"""Dev tool: the rollout at the shipped configs' policies, population and episode lengths (ac_std = 0.01), for
ES_ROLLOUT_F32 (staged weights), ES_ROLLOUT_TC3 and ES_ROLLOUT_TC (rollout_tcw.cu).  The modes alternate in one process,
REPS times each after a warm-up (ns: NS_REPS); CUDA-event time per rollout, pairs/s, and the achieved rate in TFLOP/s from
the policy's MACs per step (2 FLOP per MAC; an evaluation's E episodes share one forward pass).  Then the float64-truth error
(tests/f64_rollout.py) of SAMPLE pairs per mode: max |f - truth| / reward mass and rms(f - truth) / spread.
ROWS=simple_conf,nsra,... picks rows."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np, torch
import f64_rollout as f64
from es_pytorch_b200 import _lib
from es_pytorch_b200.engine import get_engine

F32, TC, TC3 = _lib.ES_ROLLOUT_F32, _lib.ES_ROLLOUT_TC, _lib.ES_ROLLOUT_TC3
NAMES = {F32: 'f32', TC3: 'tc3', TC: 'tc'}
ROWS = [  # (config, sizes, pairs K, T, E)
    ('simple_conf', [15, 256, 256, 3], 2400, 1000, 1),
    ('nsra', [15, 256, 256, 3], 4800, 2000, 1),
    ('obj', [17, 256, 256, 256, 6], 320, 1000, 1),
    ('ns', [28, 256, 256, 256, 8], 2400, 10000, 1),
    ('flagrun', [28, 128, 256, 256, 128, 8], 600, 500, 10),
]
REPS = int(os.environ.get('REPS', 3))
NS_REPS = int(os.environ.get('NS_REPS', 1))
SAMPLE = int(os.environ.get('SAMPLE', 4))
want = os.environ.get('ROWS')
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}', flush=True)

L = 40_000_000
rs = np.random.RandomState(0)
table = rs.randn(L).astype(np.float32)
d_table = eng.to_device(table)
for name, sizes, K, T, E in ROWS:
    if want and name not in want.split(','):
        continue
    P = f64.n_params(sizes)
    macs = sum(a * b for a, b in zip(sizes[:-1], sizes[1:]))
    flop = 2.0 * macs * T * 2 * K
    rs = np.random.RandomState(len(name))
    theta = (rs.randn(P) * 0.1).astype(np.float32)
    idx = rs.randint(0, L - P, size=K).astype(np.int64)
    obsn = np.clip(rs.randn(T, sizes[0]), -5, 5).astype(np.float32)
    rew = rs.randn(T, sizes[-1]).astype(np.float32)
    g = torch.Generator(device=eng.device).manual_seed(1)
    noise = torch.randn((K, 2, E, T, sizes[-1]), generator=g, device=eng.device, dtype=torch.float32) * 0.01
    d_theta, d_idx, d_obsn, d_rew = (eng.to_device(x) for x in (theta, idx, obsn, rew))
    fit = {m: torch.zeros(2, K, dtype=torch.float64, device=eng.device) for m in NAMES}
    behv = {m: torch.zeros(2, K, 3, dtype=torch.float32, device=eng.device) for m in NAMES}

    def run(m):
        eng.rollout(d_table, d_idx, d_theta, 0.02, sizes, d_obsn, d_rew, 0.05, fit[m][0], fit[m][1], 1, behv[m][0], behv[m][1],
                    m, act_noise=noise, episodes=E)

    for m in NAMES:                                    # warm-up
        run(m)
    eng.sync()
    times = {m: [] for m in NAMES}
    for _ in range(NS_REPS if name == 'ns' else REPS):
        for m in NAMES:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); run(m); b.record()
            eng.sync()
            times[m].append(a.elapsed_time(b))
    print(f'\n{name} {"-".join(map(str, sizes))}: K={K} T={T} E={E}, {flop / 1e12:.2f} TFLOP per rollout', flush=True)
    for m in NAMES:
        t = np.array(times[m])
        print(f'  {NAMES[m]:4s} {t.mean():9.2f} ms (min {t.min():.2f}, max {t.max():.2f})  {K / t.mean() * 1e3:10.0f} pairs/s  '
              f'{flop / t.mean() / 1e9:7.1f} TFLOP/s', flush=True)
    pairs = sorted(set([0, K - 1] + list(np.random.RandomState(2).choice(K, SAMPLE, replace=False))))
    nz = noise[pairs].cpu().numpy()
    tf, tb, mass, _ = f64.rollout_f64(table, idx[pairs], theta, 0.02, sizes, obsn, rew, 0.05, nz, E)
    spread = max(tf.std(), 1e-3 * np.sqrt(T))
    for m in NAMES:
        f = fit[m].cpu().numpy()[:, pairs]
        err = np.abs(f - tf)
        print(f'  {NAMES[m]:4s} error vs float64 on {len(pairs)} pairs: max err/mass {(err / mass).max():.3g}, '
              f'rms/spread {np.sqrt((err ** 2).mean()) / spread:.3g}', flush=True)
    del noise, fit, behv
    torch.cuda.empty_cache()
