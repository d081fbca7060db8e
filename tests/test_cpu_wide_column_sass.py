"""What ptxas made of the CTA-per-column kernels for codebooks above K = 1055 (posterior_sample_wide_kernel in csrc/sampler.cu,
train_loss_wide_kernel in csrc/train.cu), read from the sm_90a build: no GPU needed, only nvcc and cuobjdump.

Every CAP instantiation must have no stack frame, no spills and no local-memory instruction (the CALLs in the SASS are the fp64
slow-path subroutines of exp / log / division, which use registers only), and a register count that fits the CTAs per SM
DESIGN.md states (256 threads per CTA, 64 K registers per SM, allocated per warp in units of 8 registers per thread):
  sampler   CAP 2, 4, 9 (K + 1 <= 2304, so the 2048-code codebook): 3 CTAs / SM;  CAP 16 (K + 1 <= 4096): 2 CTAs / SM
  train     CAP 9: 2 CTAs / SM;  CAP 16: 1 CTA / SM"""
import os
import re
import shutil
import subprocess

import pytest

from tests.helpers import ROOT

CSRC = os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc")
NT = 256
SAMPLER_CTAS = {2: 3, 4: 3, 9: 3, 16: 2}
TRAIN_CTAS = {9: 2, 16: 1}


def _tool(name):
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return cand if os.access(cand, os.X_OK) else shutil.which(name)


def _compile(tmp_path_factory, src):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("nvcc / cuobjdump not installed")
    out = str(tmp_path_factory.mktemp("wide_sass") / (src + ".cubin"))
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-Xptxas", "-v", "-cubin", os.path.join(CSRC, src + ".cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


@pytest.fixture(scope="module")
def sampler(tmp_path_factory):
    return _compile(tmp_path_factory, "sampler")


@pytest.fixture(scope="module")
def train(tmp_path_factory):
    return _compile(tmp_path_factory, "train")


def _props(log, kernel):
    """{CAP: (stack, spill stores, spill loads, registers)} of every instantiation of `kernel`."""
    pat = (r"Function properties for (_ZN3dsb\d+" + kernel + r"ILi(\d+)E\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
           r"(\d+) bytes spill loads\n[^\n]*Used (\d+) registers")
    return {int(m[1]): tuple(int(v) for v in m[2:]) for m in re.findall(pat, log)}


def _sass_of(sass, kernel):
    out, on = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            on = m.group(1) if kernel in m.group(1) else None
            if on:
                out[on] = []
        elif on:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                out[on].append(m.group(1))
    return out


def _ctas_per_sm(regs):
    return 65536 // (NT * ((regs + 7) // 8 * 8))


@pytest.mark.parametrize("which,kernel,want", [("sampler", "posterior_sample_wide_kernel", SAMPLER_CTAS),
                                               ("train", "train_loss_wide_kernel", TRAIN_CTAS)])
def test_wide_kernels_do_not_spill_and_fit_their_occupancy(request, which, kernel, want):
    log, sass = request.getfixturevalue(which)
    props = _props(log, kernel)
    assert sorted(props) == sorted(want), props
    for cap, (stack, st, ld, regs) in props.items():
        assert (stack, st, ld) == (0, 0, 0), (kernel, cap, stack, st, ld)
        assert _ctas_per_sm(regs) >= want[cap], (kernel, cap, regs)
        print(f"{kernel}<{cap}>: {regs} registers, {_ctas_per_sm(regs)} CTAs / SM")
    fns = _sass_of(sass, kernel)
    assert len(fns) == len(want)
    for name, ins in fns.items():
        bad = [i for i in ins if re.match(r"(@!?U?P\w+\s+)?(LDL|STL)\b", i)]
        assert not bad, (name, bad[:3])
