"""Dev tool: action noise on an env whose episodes end early, fused (es_rollout_closedloop_terminal_streams,
BatchedRollout(fuse_noisy_terminal=True)), at simple_conf's and obj's policy, population and T (ac_std = 0.01, E = 1) and one
flagrun row at E = 10.  Fall heights giving mean episodes of about T/10, T/2 and T are found by bisection on the noise-free
terminal call (256 pairs), as dev_closed_terminal_time.py does.  Per height and stream count (8, and the resident clusters):
the jump-ahead fill's ms (torch.profiler, one call), the call's CUDA-event ms (median of REPS after a warm-up) and the rollout's
share of it, executed evaluation-steps and us per executed evaluation-step; alternated in the same process, the noise-free
terminal call at the same height over the same pairs, and the per-evaluation route's wall time (es.test_params without the
flag) on a NOISY_PAIRS-pair sample.  The card's name, power limit and max SM clock head the output."""
import os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200 import dist
from es_pytorch_b200.core import es
from es_pytorch_b200.core.noisetable import NoiseTable
from es_pytorch_b200.core.policy import Policy
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.batched import BatchedRollout
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv
from es_pytorch_b200.nn.nn import FeedForward
from es_pytorch_b200.nn.obstat import ObStat
from es_pytorch_b200.nn.optimizers import Adam

ROWS = [('simple_conf', [15, 256, 256, 3], 2400, 1000, 1), ('obj', [17, 256, 256, 256, 6], 320, 1000, 1),
        ('flagrun', [28, 128, 256, 256, 128, 8], 256, 1000, 10)]
ROWS = [r for r in ROWS if r[0] in os.environ.get('ROWS', 'simple_conf,obj,flagrun').split(',')]
REPS = int(os.environ.get('REPS', 3))
NOISY_PAIRS = int(os.environ.get('NOISY_PAIRS', 16))
AC_STD = 0.01
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}', flush=True)


def timed(fn, reset=None):
    if reset: reset()
    fn()
    eng.sync()
    ms = []
    for _ in range(REPS):
        if reset: reset()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        eng.sync()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def fill_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        eng.sync()
    return sum(e.device_time_total for e in prof.key_averages() if e.key.startswith(('mt_fill', 'mj_order', 'mj_lists')) or
               'mt_fill_kernel' in e.key) / 1e3


for name, sizes, K, T, E in ROWS:
    obs, act = sizes[0], sizes[-1]
    env = ClosedLoopEnv(obs, act, T)
    net = FeedForward(sizes[1:-1], torch.nn.Tanh(), env, AC_STD, 5)
    P = sum(p.numel() for p in net.parameters())
    rs = np.random.RandomState(len(name))
    table_np = rs.randn(P + 2_000_000).astype(np.float32)
    table = eng.to_device(table_np)
    theta = eng.to_device((rs.randn(P) * 0.03).astype(np.float32))
    _, rew = env.device_arrays(eng)
    rew = rew[:T].contiguous()
    obs0, env_a, env_b = env.device_closed(eng)
    mean, std = eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs))
    fit = torch.zeros(2, K, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, K, 3, dtype=torch.float32, device=eng.device)
    idx = eng.to_device(rs.randint(0, table.numel() - P, size=K).astype(np.int64))
    sample = torch.zeros(2, 256, dtype=torch.int32, device=eng.device)
    C, resident, _ = eng.closed_mlp_plan(sizes, env_a.shape[0])

    def args(n):
        return (table, idx[:n], theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew, 0.05, fit[0, :n], fit[1, :n], 1,
                behv[0, :n].reshape(-1), behv[1, :n].reshape(-1))

    def mean_len(h):
        eng.rollout_closed_terminal(*args(256), fall_height=h, steps=sample)
        eng.sync()
        return float((sample.double() + 1).mean())

    def height(target):
        lo, hi = 1e-6, 1e3
        for _ in range(40):
            mid = (lo * hi) ** 0.5
            lo, hi = (mid, hi) if mean_len(mid) < target else (lo, mid)
        return hi

    for label, h in (('T/10', height(T / 10)), ('T/2', height(T / 2)), ('T', 1e30)):
        h = float(np.float32(h))
        for R in (8, resident):
            n = K // R
            k = R * n
            seeds = [np.random.RandomState(1000 + s).get_state() for s in range(R)]
            key0 = eng.to_device(np.stack([s[1] for s in seeds]).astype(np.uint32).view(np.int32))
            key, pos = key0.clone(), torch.zeros(R, dtype=torch.int32, device=eng.device)
            has, gv = torch.zeros(R, dtype=torch.int32, device=eng.device), torch.zeros(R, dtype=torch.float64, device=eng.device)

            st_k = torch.zeros(2, k, dtype=torch.int32, device=eng.device)
            used = torch.zeros(2, k, dtype=torch.int64, device=eng.device)

            def reset():
                key.copy_(key0); pos.fill_(624); has.zero_(); gv.zero_()

            def walk():
                eng.rollout_closed_terminal_streams(key, pos, has, gv, n, table.numel() - P, 0, AC_STD, table, theta, 0.02, sizes,
                                                    mean, std, 5.0, obs0, env_a, env_b, rew, 0.05, fit[0, :k], fit[1, :k], 1,
                                                    behv[0, :k].reshape(-1), behv[1, :k].reshape(-1), episodes=E, fall_height=h,
                                                    idx_out=idx[:k], steps=st_k, noise_used=used)

            def plain():
                eng.rollout_closed_terminal(*args(k), fall_height=h, steps=st_k)

            t_walk = timed(walk, reset)
            executed = int(used.sum()) // act                  # every episode's executed steps
            reset()
            f = fill_ms(walk)
            t_plain = timed(plain)
            executed_plain = int((st_k.long() + 1).sum())
            t_walk2 = timed(walk, reset)
            ex = executed
            print(f'{name:11s} K={k} T={T} E={E} C={C} h={h:.4g} ({label:4s}) streams={R:3d}: call {t_walk:9.2f} / {t_walk2:9.2f} ms '
                  f'(fill {f:7.2f} ms, rollout {min(t_walk, t_walk2) - f:9.2f} ms)'
                  + f', executed eval-steps {ex} ({ex / (2 * k * T * E):.3f}) = {min(t_walk, t_walk2) * 1e3 / ex:.4f} us/eval-step'
                  + f'; noise-free terminal {t_plain:9.2f} ms ({executed_plain} eval-steps = '
                  f'{t_plain * 1e3 / executed_plain:.4f} us/eval-step)', flush=True)
        # the per-evaluation route (es.test_params without the flag) on a NOISY_PAIRS-pair sample at this height
        if E == 1:
            envh = ClosedLoopEnv(obs, act, T, fall_height=h)
            pol = Policy(FeedForward(sizes[1:-1], torch.nn.Tanh(), envh, AC_STD, 5), 0.02, Adam(P, 0.01))
            nt = NoiseTable(P, table_np)
            fb = BatchedRollout(envh, T, coins_per_eval=0)
            srs = np.random.RandomState(3)
            es.test_params(dist.world(), 2, pol, nt, ObStat((obs,), 0), fb, srs)      # warm-up
            t0 = time.perf_counter()
            _, _, _, st = es.test_params(dist.world(), NOISY_PAIRS, pol, nt, ObStat((obs,), 0), fb, srs)
            dt = time.perf_counter() - t0
            ex = st + 2 * NOISY_PAIRS
            print(f'{name:11s} per-evaluation route, {NOISY_PAIRS} pairs, h={h:.4g} ({label}): {dt * 1e3:.1f} ms wall, {ex} executed '
                  f'eval-steps = {dt * 1e6 / ex:.3f} us/eval-step', flush=True)
