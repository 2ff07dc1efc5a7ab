"""Dev tool: the closed-loop rollout on an env whose episodes end early (es_rollout_closedloop_terminal) at simple_conf's and
obj's policies, populations and episode lengths (ac_std = 0, E = 1), at fall heights giving mean episode lengths of about T/10,
T/2 and T (nothing falls), each alternated in one process with the same call at fall_height=None (es_rollout_closedloop_mlp).
Per row: executed evaluation-steps, CUDA-event ms per rollout (median of REPS after a warm-up) and us per executed
evaluation-step.  The heights are found by bisection on a 256-pair sample.  Then one generation of es.step with ac_std = 0.01 at
simple_conf's shape, which runs one evaluation per launch (NOISY_PAIRS pairs): wall time, executed evaluation-steps and
wall time per executed evaluation-step.  The card's name, power limit and max SM clock head the output."""
import os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200.engine import get_engine
from es_pytorch_b200.gym.synthetic_env import ClosedLoopEnv

ROWS = [('simple_conf', [15, 256, 256, 3], 2400, 1000), ('obj', [17, 256, 256, 256, 6], 320, 1000)]
REPS = int(os.environ.get('REPS', 3))
NOISY_PAIRS = int(os.environ.get('NOISY_PAIRS', 16))
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


def timed(fn):
    fn()
    eng.sync()
    ms = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        eng.sync()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


for name, sizes, K, T in ROWS:
    obs, act = sizes[0], sizes[-1]
    P = sum(i * o + o for i, o in zip(sizes[:-1], sizes[1:]))
    env = ClosedLoopEnv(obs, act, T)
    _, rew = env.device_arrays(eng)
    rew = rew[:T].contiguous()
    obs0, env_a, env_b = env.device_closed(eng)
    rs = np.random.RandomState(len(name))
    theta = eng.to_device((rs.randn(P) * 0.03).astype(np.float32))
    idx = eng.to_device(rs.randint(0, L - P, size=K).astype(np.int64))
    mean, std = eng.to_device(np.zeros(obs)), eng.to_device(np.ones(obs))
    fit = torch.zeros(2, K, dtype=torch.float64, device=eng.device)
    behv = torch.zeros(2, K, 3, dtype=torch.float32, device=eng.device)
    steps = torch.zeros(2, K, dtype=torch.int32, device=eng.device)

    def args(n):
        return (table, idx[:n], theta, 0.02, sizes, mean, std, 5.0, obs0, env_a, env_b, rew, 0.05, fit[0, :n], fit[1, :n], 1,
                behv[0, :n].reshape(-1), behv[1, :n].reshape(-1))

    sample = torch.zeros(2, min(K, 256), dtype=torch.int32, device=eng.device)

    def term(h, n=K):
        eng.rollout_closed_terminal(*args(n), fall_height=h, steps=steps if n == K else sample)

    def mean_len(h):
        term(h, sample.shape[1])
        eng.sync()
        return float((sample.double() + 1).mean())

    def height(target):
        lo, hi = 1e-6, 1e3
        for _ in range(40):
            mid = (lo * hi) ** 0.5
            lo, hi = (mid, hi) if mean_len(mid) < target else (lo, mid)
        return hi

    for label, h in (('T/10', height(T / 10)), ('T/2', height(T / 2)), ('T', 1e30)):
        t_none = timed(lambda: eng.rollout_closed_mlp(*args(K)))
        t_term = timed(lambda: term(h))
        t_none2 = timed(lambda: eng.rollout_closed_mlp(*args(K)))
        executed = int((steps.long() + 1).sum())
        print(f'{name:12s} K={K} T={T} h={h:.4g} ({label:4s}): executed evaluation-steps {executed} of {2 * K * T} '
              f'({executed / (2 * K * T):.3f}); terminal {t_term:8.2f} ms = {t_term * 1e3 / executed:.4f} us/eval-step; '
              f'fall_height=None {t_none:8.2f} / {t_none2:8.2f} ms = {min(t_none, t_none2) * 1e3 / (2 * K * T):.4f} us/eval-step',
              flush=True)

# one generation of es.step with action noise at simple_conf's shape: the per-evaluation route
from es_pytorch_b200 import dist
from es_pytorch_b200.core import es
from es_pytorch_b200.core.noisetable import NoiseTable
from es_pytorch_b200.core.policy import Policy
from es_pytorch_b200.gym.batched import BatchedRollout
from es_pytorch_b200.nn.nn import FeedForward
from es_pytorch_b200.nn.optimizers import Adam
from es_pytorch_b200.utils.rankers import CenteredRanker
from es_pytorch_b200.utils.reporters import Reporter


class _Cfg(dict):
    __getattr__ = dict.__getitem__


T = 1000
env = ClosedLoopEnv(15, 3, T, fall_height=0.5)
net = FeedForward([256, 256], torch.nn.Tanh(), env, 0.01, 5)
P = sum(p.numel() for p in net.parameters())
policy = Policy(net, 0.02, Adam(P, 0.01))
nt = NoiseTable(P, np.random.RandomState(0).randn(P + 1_000_000).astype(np.float32))
fit_fn = BatchedRollout(env, T, coins_per_eval=1, save_obs_chance=0.01)
cfg = _Cfg(general=_Cfg(policies_per_gen=2 * NOISY_PAIRS, batch_size=500), policy=_Cfg(l2coeff=0.005))
class _Steps(Reporter):
    def log_gen(self, fits, noiseless_tr, policy, steps):
        self.steps = steps


rs = np.random.RandomState(1)
es.step(cfg, dist.world(), policy, nt, env, fit_fn, rs, CenteredRanker(), Reporter())      # warm-up
eng.sync()
rep = _Steps()
t0 = time.perf_counter()
es.step(cfg, dist.world(), policy, nt, env, fit_fn, rs, CenteredRanker(), rep)
eng.sync()
dt = time.perf_counter() - t0
n_evals = 2 * NOISY_PAIRS
executed = rep.steps + n_evals                          # steps sums t_d; an evaluation executes t_d + 1 steps
print(f'noisy per-evaluation route, simple_conf shape, {NOISY_PAIRS} pairs, T={T}, h=0.5: {dt * 1e3:.1f} ms per generation '
      f'({dt * 1e3 / n_evals:.2f} ms per evaluation), executed evaluation-steps {executed} ({executed / n_evals:.0f} per '
      f'evaluation), {dt * 1e6 / executed:.2f} us of wall time per executed evaluation-step', flush=True)
