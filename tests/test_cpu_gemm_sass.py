"""What ptxas made of the wgmma GEMM (csrc/gemm_wgmma.cu), read from its sm_90a SASS: no GPU needed, only nvcc and cuobjdump.

* no C7510 / C7519 advisories: nothing makes ptxas serialise the wgmma pipeline or inject warpgroup.arrive around the MMAs;
* no spills in any gemm_wgmma_kernel instantiation;
* no CALL anywhere in a gemm_wgmma_kernel, so the mainloop cannot cross a function boundary;
* the HGMMAs of one commit group issue back to back: a WARPGROUP.DEPBAR only follows the group's last HGMMA (the one that carries gsb0);
* the split-fp16 form issues the 12 HGMMAs of a k-block as one group: ptxas used to split it into 12 groups of one."""
import os
import re
import shutil
import subprocess

import pytest

from tests.helpers import ROOT

CSRC = os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc")


def _tool(name):
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return cand if os.access(cand, os.X_OK) else shutil.which(name)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("nvcc / cuobjdump not installed")
    out = str(tmp_path_factory.mktemp("gemm_sass") / "gemm_wgmma.cubin")
    # the Makefile's flags for this translation unit
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-Xptxas", "-v", "-cubin", os.path.join(CSRC, "gemm_wgmma.cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    kernels = {}
    name = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "gemm_wgmma_kernel" in m.group(1) else None
            if name:
                kernels[name] = []
        elif name:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                kernels[name].append(m.group(1))
    return r.stderr, kernels


def _split_form(kernels):
    # gemm_wgmma_kernel<128, DSB_DTYPE_F16, true>
    (name,) = [k for k in kernels if k.startswith("_ZN3dsb17gemm_wgmma_kernelILi128ELi2ELb1E")]
    return kernels[name]


def test_ptxas_keeps_the_wgmma_pipeline_and_does_not_spill(compiled):
    log, kernels = compiled
    assert len(kernels) == 7
    assert "C7510" not in log, [l for l in log.splitlines() if "C7510" in l][:3]
    assert "C7519" not in log, [l for l in log.splitlines() if "C7519" in l][:3]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    gemm = [p for p in props if "gemm_wgmma_kernel" in p[0]]
    assert len(gemm) == 7
    for fn, _, st, ld in gemm:
        assert (st, ld) == ("0", "0"), f"{fn} spills {st} / {ld} bytes"


def test_no_call_in_gemm_kernels(compiled):
    _, kernels = compiled
    for name, ins in kernels.items():
        calls = [i for i in ins if re.match(r"(@!?U?P\w+\s+)?CALL", i)]
        assert not calls, f"{name}: {calls[:3]}"


def test_hgmma_groups_issue_back_to_back(compiled):
    _, kernels = compiled
    for name, ins in kernels.items():
        open_group = 0
        for i in ins:
            if "HGMMA" in i:
                open_group = 0 if "gsb0" in i else open_group + 1
            elif "WARPGROUP.DEPBAR" in i:
                assert open_group == 0, f"{name}: wgmma wait inside a commit group ({open_group} HGMMAs issued without gsb0)"
        assert any("HGMMA" in i for i in ins), name


def test_split_form_issues_a_kblock_as_one_group(compiled):
    _, kernels = compiled
    groups, n = [], 0
    for i in _split_form(kernels):
        if "HGMMA" in i:
            n += 1
            if "gsb0" in i:
                groups.append(n)
                n = 0
    # lo*hi, hi*lo, hi*hi over 4 K slices of 16 per 64-deep k-block
    assert groups and all(g == 12 for g in groups), groups
