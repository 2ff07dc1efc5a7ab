"""CPU (no GPU): ptxas keeps the wide tensor-core rollout's wgmmas asynchronous (rollout_tcw.cu).

C7520 (divergent path), C7512 / C7511 (not enough registers for the wgmma pipeline) make every wgmma of a kernel wait for the
previous one, and C7507 means a warpgroup's setmaxnreg was dropped; each only prints an info line, so the compile log is
checked here, and every rollout_tcw_kernel instantiation must compile without spills."""
import os
import re
import subprocess
import tempfile

import pytest

from es_pytorch_b200 import build

SRC = os.path.join(build.CSRC, 'rollout_tcw.cu')


def _nvcc():
    import shutil
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_rollout_tcw_wgmma_not_serialized():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
               '-o', os.path.join(tmp, 'rollout_tcw.o'), SRC]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    bad = [l for l in log.splitlines() if re.search(r'\((C7520|C7512|C7511|C7507)\)', l)]
    assert not bad, '\n'.join(bad)
    # the four rollout_tcw_kernel instantiations (SPLIT x NOISE) were compiled, with no spills
    props = re.findall(r'Function properties for (\S*rollout_tcw_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill '
                       r'stores, (\d+) bytes spill loads', log)
    assert len(props) == 4, log
    for name, _, st, ld in props:
        assert st == '0' and ld == '0', f'{name}: {st} bytes spill stores, {ld} bytes spill loads'
