"""Dev tool: the cost of building the shipped noise table (SIZE = 250 000 000 float32 values) on the GPU with
NoiseTable.make_noise_device: CUDA-event time of the draw (first call, which allocates the scratch, and the mean of REPS
calls after it), wall time of the whole call including the host seeding and the state upload, es_randn's scratch size and
number of windows.  HOST=1 also times numpy's make_noise (+ the upload it needs) and counts the values that differ."""
import os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from es_pytorch_b200.core.noisetable import NoiseTable
from es_pytorch_b200.engine import get_engine

SIZE = int(os.environ.get('SIZE', 250_000_000))
SEED = int(os.environ.get('SEED', 123))
REPS = int(os.environ.get('REPS', 5))
eng = get_engine(0)
try:
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:                                 # (the timing does not depend on it)
    card = f'unknown ({e})'
print(f'device: {card}', flush=True)
nbytes, windows = eng.randn_plan(SIZE)
print(f'es_randn({SIZE}): {windows} windows, scratch {nbytes / 2 ** 20:.1f} MiB', flush=True)


def timed():
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    a.record()
    t = NoiseTable.make_noise_device(SIZE, SEED, engine=eng)
    b.record()
    eng.sync()
    return t, a.elapsed_time(b), (time.perf_counter() - t0) * 1e3


dev, first_ms, first_wall = timed()
print(f'first call: {first_ms:.2f} ms on the device, {first_wall:.2f} ms wall (scratch allocation included)', flush=True)
runs = []
for _ in range(REPS):
    t, ms, wall = timed()
    assert torch.equal(t, dev), 'make_noise_device is not deterministic'
    runs.append((ms, wall))
    del t
ms = np.array([r[0] for r in runs]); wall = np.array([r[1] for r in runs])
print(f'steady state ({REPS} calls): {ms.mean():.2f} ms on the device (min {ms.min():.2f}, max {ms.max():.2f}), '
      f'{wall.mean():.2f} ms wall; {SIZE / ms.mean() / 1e6:.2f} G values/s', flush=True)
if os.environ.get('HOST') == '1':
    t0 = time.perf_counter()
    host = NoiseTable.make_noise(SIZE, SEED)
    t1 = time.perf_counter()
    up = eng.to_device(host)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    print(f'numpy make_noise: {t1 - t0:.2f} s, upload {(t2 - t1) * 1e3:.1f} ms', flush=True)
    diff = int((up != dev).sum())
    print(f'values that differ from numpy: {diff} of {SIZE}', flush=True)
