"""CPU (no GPU): the kernels of es_randn -- its own two and the jump-ahead kernels it runs per window -- compile for sm_90a
without spilling registers to local memory."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

from es_pytorch_b200 import build

SRC = os.path.join(build.CSRC, 'mt_gauss.cu')
KERNELS = ['mr_window_kernel', 'mr_emit_kernel', 'mt_fill_kernel', 'mt_flags_kernel', 'mt_scan_kernel', 'mj_order_kernel',
           'mj_lists_kernel']


def _nvcc():
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.mark.skipif(_nvcc() is None, reason='needs nvcc')
def test_randn_kernels_do_not_spill():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
               '-o', os.path.join(tmp, 'mt_gauss.o'), SRC]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    props = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill '
                       r'loads', log)
    for k in KERNELS:
        found = [p for p in props if k in p[0]]
        assert len(found) == 1, (k, log)
        name, _, st, ld = found[0]
        assert st == '0' and ld == '0', f'{k}: {st} bytes spill stores, {ld} bytes spill loads'
