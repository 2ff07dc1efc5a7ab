"""CPU (no GPU): ptxas keeps the tensor-core rollout's wgmmas asynchronous.

When ptxas cannot prove that the code between a wgmma and its wait is safe for registers in flight, it makes every wgmma
of the kernel wait for the previous one (C7520: divergent path, C7512: not enough registers), and when a warpgroup's
setmaxnreg cannot be honoured it drops the register split (C7507).  Each of these only prints an info line and costs the
kernel its overlap, so the compile log is checked here."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from es_pytorch_b200 import build

SRC = os.path.join(build.CSRC, 'rollout_tc2.cu')


def _nvcc():
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_rollout_tc2_wgmma_not_serialized():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
               '-o', os.path.join(tmp, 'rollout_tc2.o'), SRC]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    bad = [l for l in log.splitlines() if re.search(r'\((C7520|C7512|C7507)\)', l)]
    assert not bad, '\n'.join(bad)
    # the four rollout_tc2_kernel instantiations (SPLIT x NOISE) were compiled, with no spills
    props = re.findall(r'Function properties for (\S*rollout_tc2_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill '
                       r'stores, (\d+) bytes spill loads', log)
    assert len(props) == 4, log
    for name, _, st, ld in props:
        assert st == '0' and ld == '0', f'{name}: {st} bytes spill stores, {ld} bytes spill loads'
