"""CPU (no GPU): the closed-loop cluster rollout (rollout_closedw.cu) compiles for sm_90a to one kernel per depth and variant
(tanh, binned head, action noise, another activation, another activation with action noise), none with a stack frame or
spills, and the shared memory it requests fits an H100 CTA (227 KiB, static included) for every shape it accepts.

The plan (es_closedw_plan: coverage, cluster size, dynamic shared memory per CTA) is host code, so a small host program that
includes the source runs it here over the shipped shapes and a grid of covered shapes up to every limit."""
import os
import re
import subprocess
import tempfile

import pytest

from es_pytorch_b200 import build

SRC = os.path.join(build.CSRC, 'rollout_closedw.cu')
SMEM_PER_CTA = 227 * 1024


def _nvcc():
    import shutil
    cand = build.nvcc_path()
    return cand if (os.path.isabs(cand) and os.path.exists(cand)) or shutil.which(cand) else None


@pytest.fixture(scope='module')
def ptxas_log():
    if _nvcc() is None:
        pytest.skip('needs nvcc')
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
               '-o', os.path.join(tmp, 'rollout_closedw.o'), SRC]
        res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    return log


def _props(log):
    """(name, stack, spill stores, spill loads) of every cluster-kernel instantiation in the ptxas log."""
    return re.findall(r'Function properties for (\S*rollout_closedw_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill '
                      r'stores, (\d+) bytes spill loads', log)


def test_cluster_kernel_variants_compile_without_spills(ptxas_log):
    props = _props(ptxas_log)
    assert len(props) == 15, ptxas_log
    for name, stack, st, ld in props:
        assert stack == '0' and st == '0' and ld == '0', f'{name}: {stack} bytes stack, {st} bytes spill stores, {ld} loads'


def test_cluster_kernel_has_three_depths_of_each_variant(ptxas_log):
    assert 'rollout_closedw.cu' in build.SOURCES and 'rollout_closedw.cuh' in build.HEADERS
    # (depth, binned, noisy, activation) from the mangled template arguments <NL, BINNED, NOISY, ACT>
    variants = []
    for name, _, _, _ in _props(ptxas_log):
        m = re.search(r'rollout_closedw_kernelILi(\d)ELb([01])ELb([01])ELb([01])E', name)
        assert m, name
        variants.append(tuple(int(g) for g in m.groups()))
    # 2, 3 and 4 hidden layers x (tanh, binned, tanh + noise, activation, activation + noise): binned heads draw no noise
    want = {(nl, b, n, a) for nl in (3, 4, 5) for b, n, a in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 1, 1))}
    assert len(variants) == 15 and set(variants) == want, ptxas_log


HARNESS = r'''
#include <stdarg.h>
#include <stdio.h>
#include "%s"
static char g_msg[512];
void es_set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_msg, sizeof g_msg, fmt, ap); va_end(ap); }
static void one(const char* name, const int* d, int nl, int band) {
    int C = 0; size_t smem = 0;
    const int rc = es_closedw_plan(d, nl, band, &C, &smem);
    printf("%%s rc %%d C %%d smem %%zu\n", name, rc, C, smem);
}
int main() {
    const int s1[] = {15, 256, 256, 3}, s2[] = {17, 256, 256, 256, 6}, s3[] = {26, 256, 256, 256, 6}, s4[] = {28, 256, 256, 256, 8},
              s5[] = {28, 128, 256, 256, 128, 8}, s6[] = {376, 256, 256, 17};
    one("simple_conf", s1, 3, 8); one("obj", s2, 4, 8); one("obj26", s3, 4, 8); one("ns", s4, 4, 8); one("flagrun", s5, 5, 8);
    one("humanoid_wide", s6, 3, 8);
    const int obs_[] = {1, 2, 8, 15, 28, 100, 376, 384}, act_[] = {1, 17, 64}, band_[] = {2, 8, 16}, w_[] = {1, 64, 129, 200, 256};
    size_t worst = 0; long covered = 0, total = 0;
    for (int nh = 2; nh <= 4; ++nh) {
        int n = 1;
        for (int i = 0; i < nh; ++i) n *= 5;
        for (int c = 0; c < n; ++c)
            for (int o : obs_) for (int a : act_) for (int b : band_) {
                if (b > o) continue;
                int d[6], k = c;
                d[0] = o;
                for (int i = 1; i <= nh; ++i) { d[i] = w_[k %% 5]; k /= 5; }
                d[nh + 1] = a;
                int C = 0; size_t smem = 0;
                ++total;
                if (es_closedw_plan(d, nh + 1, b, &C, &smem) == 0) { ++covered; if (smem > worst) worst = smem; }
            }
    }
    printf("grid covered %%ld of %%ld worst %%zu\n", covered, total, worst);
    return 0;
}
'''


def test_rollout_closedw_shared_memory_fits_every_covered_shape(ptxas_log):
    # (the source's only kernels are the rollout_closedw_kernel instantiations)
    static = [int(x) for x in re.findall(r'Used \d+ registers, used \d+ barriers, (\d+) bytes smem', ptxas_log)]
    assert len(static) == 15, ptxas_log
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, 'plan.cu')
        with open(src, 'w') as f:
            f.write(HARNESS % SRC.replace('\\', '/'))
        exe = os.path.join(tmp, 'plan')
        res = subprocess.run([_nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-std=c++17', '-o', exe, src],
                             capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120).stdout
    static_max = max(static)
    assert static_max <= 1024, ptxas_log                     # the 1 KiB the plan leaves for the kernel's static shared memory
    plans = {m.group(1): (int(m.group(2)), int(m.group(3)), int(m.group(4)))
             for m in re.finditer(r'^(\w+) rc (-?\d+) C (\d+) smem (\d+)$', out, re.M)}
    # every shipped policy is covered, with the cluster size the README states
    want_c = {'simple_conf': 2, 'obj': 4, 'obj26': 4, 'ns': 4, 'flagrun': 4, 'humanoid_wide': 4}
    for name, c in want_c.items():
        rc, got_c, smem = plans[name]
        assert rc == 0 and got_c == c, (name, plans[name])
        assert smem + static_max <= SMEM_PER_CTA, (name, smem)
    m = re.search(r'grid covered (\d+) of (\d+) worst (\d+)', out)
    assert m and int(m.group(1)) > 0 and int(m.group(1)) < int(m.group(2)), out
    assert int(m.group(3)) + static_max <= SMEM_PER_CTA, out
