"""What ptxas made of the split-fp16 attention kernel (csrc/attention_tc_split.cu), read from its sm_90a SASS: no GPU needed, only nvcc
and cuobjdump.

* no C7510 / C7514 / C7519 advisories: nothing makes ptxas serialise the wgmma pipeline or inject warpgroup.arrive around the MMAs;
* no spills, no local memory and no CALL in the kernel;
* S = Q K^T and O += P V each issue as one group of 12 back-to-back HGMMAs (3 split passes x 4 k-steps of 16): the first from shared
  memory on both sides, the second with P from registers and V read transposed (MN-major)."""
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
    out = str(tmp_path_factory.mktemp("attn_sass") / "attention_tc_split.cubin")
    # the Makefile's flags for this translation unit
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr",
                        "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-Xptxas", "-v", "-cubin", os.path.join(CSRC, "attention_tc_split.cu"),
                        "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    ins, on = [], False
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            on = "attention_tc_split_kernel" in m.group(1)
        elif on:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                ins.append(m.group(1))
    assert ins, "attention_tc_split_kernel not found in the SASS"
    return r.stderr, ins


def test_ptxas_keeps_the_wgmma_pipeline_and_does_not_spill(compiled):
    log, _ = compiled
    for code in ("C7510", "C7514", "C7519"):
        assert code not in log, [l for l in log.splitlines() if code in l][:3]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    attn = [p for p in props if "attention_tc_split_kernel" in p[0]]
    assert len(attn) == 1
    assert attn[0][1:] == ("0", "0", "0"), f"stack / spills: {attn[0][1:]}"


def test_no_call_and_no_local_memory(compiled):
    _, ins = compiled
    bad = [i for i in ins if re.match(r"(@!?U?P\w+\s+)?(CALL|LDL|STL)\b", i)]
    assert not bad, bad[:3]


def test_s_and_pv_issue_as_two_groups_of_twelve(compiled):
    _, ins = compiled
    groups, cur = [], []
    for i in ins:
        if "HGMMA" in i:
            cur.append(i)
            if "gsb0" in i:
                groups.append(cur)
                cur = []
        elif "WARPGROUP.DEPBAR" in i:
            assert not cur, f"wgmma wait inside a commit group ({len(cur)} HGMMAs issued without gsb0)"
    assert not cur
    assert [len(g) for g in groups] == [12, 12], [len(g) for g in groups]
    s, pv = groups
    assert all(i.startswith("HGMMA.64x64x16.F32 ") and "gdesc" in i and "tnspB" not in i and not re.search(r", R\d+, gdesc", i) for i in s), s
    assert all("tnspB" in i and re.search(r"F32 R\d+, R\d+, gdesc", i) for i in pv), pv
