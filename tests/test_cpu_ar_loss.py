"""Scoring the autoregressive SpecVQGAN transformer, on the CPU: the fp32 oracle's loss against the unmodified reference
(tests/golden/ar_loss.npz, oracle/gen_golden_ar_loss.py), what ptxas made of the causal split attention (csrc/attention_tc_split_causal.cu),
refusals raised before any launch, and tools/ar_val_loss.py's dry run."""
import json
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import _pkg

_pkg.load()
from diffsound_b200 import ops  # noqa: E402
from diffsound_b200.modeling.models.cond_transformer import Net2NetTransformer  # noqa: E402
from diffsound_b200.modeling.transformers.mingpt import GPT, GPTFeats  # noqa: E402
from diffsound_b200.utils.builders import AR_CONFIGS, ar_transformer_config, build_ar_transformer  # noqa: E402
from oracle import ar_oracle as A  # noqa: E402
from oracle import ar_loss_oracle as AL  # noqa: E402
from tests.helpers import ROOT  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CSRC = os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc")
CASES = ["v32_tc1", "v32_tc3", "v2048_tc1", "v2048_tc3", "full"]


def _golden():
    with np.load(os.path.join(GOLDEN, "ar_loss.npz")) as z:
        return {k: z[k] for k in z.files}


def _gpt(meta):
    V, Tc, seed, D, NL, NH, Cf = (int(v) for v in meta)
    fe, gc = A.gpt_config(V, D, NL, NH, Cf)
    torch.manual_seed(seed)
    g = GPTFeats(fe, gc).eval()
    A.perturb_(g.state_dict(), seed)
    return g, Tc, NL, NH


@pytest.mark.parametrize("case", CASES)
def test_oracle_loss_matches_reference(case):
    gd = _golden()
    g, Tc, NL, NH = _gpt(gd[case + "/meta"])
    sd = g.state_dict()
    z, feats = torch.from_numpy(gd[case + "/z"]), torch.from_numpy(gd[case + "/feats"])
    gpt = AL.loss(sd, z[:, :-1], feats, torch.from_numpy(gd[case + "/gpt_targets"]), first_row=0, n_layer=NL, n_head=NH)
    step = AL.loss(sd, z[:, :-1], feats, z, first_row=Tc - 1, n_layer=NL, n_head=NH)
    for mine, key in ((gpt, "gpt_loss"), (step, "step_loss")):
        ref = float(gd[f"{case}/{key}"])
        assert abs(float(mine) - ref) <= 1e-6 * abs(ref), (key, float(mine), ref)
    assert int((torch.from_numpy(gd[case + "/gpt_targets"]) == -100).sum()) > 0


# ---------------------------------------------------------------- SASS of the causal kernels
def _tool(name):
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return cand if os.access(cand, os.X_OK) else shutil.which(name)


def _nvcc_flags():
    """The Makefile's flags for a translation unit."""
    return ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"),
            "-I" + CSRC, "--expt-relaxed-constexpr"]


def _hd(mangled):
    m = re.search(r"attention_tc_split_kernelILi(\d+)ELb1EE", mangled)
    return int(m.group(1)) if m else None


@pytest.fixture(scope="module")
def causal_build(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    obj = str(tmp_path_factory.mktemp("causal_sass") / "unit.o")
    r = subprocess.run([nvcc, *_nvcc_flags(), "-Xptxas", "-v", "-c", os.path.join(CSRC, "attention_tc_split_causal.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    ins, hd = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            hd = _hd(m.group(1))
            if hd:
                ins[hd] = []
        elif hd:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                ins[hd].append(m.group(1))
    assert sorted(ins) == [32, 64], sorted(ins)
    return r.stderr, ins, obj, cuobjdump, nvcc


def test_causal_kernels_keep_the_wgmma_pipeline_and_do_not_spill(causal_build):
    log, ins, _, _, _ = causal_build
    for code in ("C7510", "C7514", "C7519"):
        assert code not in log, [l for l in log.splitlines() if code in l][:3]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    attn = {_hd(p[0]): p[1:] for p in props if _hd(p[0])}
    assert attn == {64: ("0", "0", "0"), 32: ("0", "0", "0")}, attn
    for hd, seq in ins.items():
        bad = [i for i in seq if re.match(r"(@!?U?P\w+\s+)?(CALL|LDL|STL)\b", i)]
        assert not bad, (hd, bad[:3])


@pytest.mark.parametrize("hd,groups", [(64, [12, 12]), (32, [6, 12])])
def test_causal_s_and_pv_hgmma_groups(causal_build, hd, groups):
    """Per 64-key chunk: S as one back-to-back group from shared memory, P V as one group with P from registers and V read transposed."""
    _, ins, _, _, _ = causal_build
    found, cur = [], []
    for i in ins[hd]:
        if "HGMMA" in i:
            cur.append(i)
            if "gsb0" in i:
                found.append(cur)
                cur = []
        elif "WARPGROUP.DEPBAR" in i:
            assert not cur, f"wgmma wait inside a commit group ({len(cur)} HGMMAs issued without gsb0)"
    assert not cur and [len(g) for g in found] == groups, [len(g) for g in found]
    s, pv = found
    assert all(i.startswith("HGMMA.64x64x16.F32 ") and "tnspB" not in i and not re.search(r", R\d+, gdesc", i) for i in s), s
    assert all(i.startswith(f"HGMMA.64x{hd}x16.F32 ") and "tnspB" in i and re.search(r"F32 R\d+, R\d+, gdesc", i) for i in pv), pv


def test_causal_kernels_sass_digests(causal_build):
    """The causal instantiations' instruction sequences (tests/golden/attention_causal_sass.json, addresses and encodings ignored)."""
    _, _, obj, cuobjdump, nvcc = causal_build
    from tests.sass_digest import sass_digests
    with open(os.path.join(GOLDEN, "attention_causal_sass.json")) as f:
        ref = json.load(f)
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != ref["nvcc"]:
        pytest.skip(f"digests were recorded with {ref['nvcc']}, this is {ver}")
    mine = {f"attention_tc_split_kernel<{_hd(k)},causal>": v for k, v in sass_digests(obj, cuobjdump).items() if _hd(k)}
    assert mine == ref["functions"]["attention_tc_split_causal.cu"]


# ---------------------------------------------------------------- refusals before launch
def test_training_mode_and_shape_refusals_before_launch():
    g = _gpt([32, 1, 0, 128, 2, 2, 16])[0]
    feats = torch.randn(1, 16, 1)
    emb = torch.zeros(1, 1, 128)
    idx = torch.zeros(1, 4, dtype=torch.long)
    g.train()
    with pytest.raises(NotImplementedError, match="only the forward .* is implemented; training"):
        GPT.forward(g, idx, embeddings=emb, targets=torch.zeros(1, 5, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="training"):
        g.forward_loss(idx, feats, torch.zeros(1, 5, dtype=torch.long), 0)
    g.eval()
    with pytest.raises(ValueError, match="targets"):
        GPT.forward(g, idx, embeddings=emb, targets=torch.zeros(1, 4, dtype=torch.long))
    with pytest.raises(ValueError, match="targets"):
        g.forward_loss(idx, feats, torch.zeros(1, 4, dtype=torch.long), 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        GPT.forward(g, idx, embeddings=emb, targets=torch.zeros(1, 5, dtype=torch.long))
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS["caps_transformer_small"]), device="cpu").train()
    assert isinstance(m, Net2NetTransformer)
    with pytest.raises(NotImplementedError, match="only the forward .* is implemented; training"):
        m.shared_step({"image": torch.zeros(1, 80, 848), "feature": torch.zeros(1, 1, 512)}, 0)
    with pytest.raises(ValueError, match="head_dim"):
        ops.attention_tc_split_causal(*(torch.zeros(4, 8, dtype=torch.float16),) * 4, q_lo=0, k_lo=0, v_lo=0, o_lo=0, B=1, H=1, L=4, scale=1.0,
                                      head_dim=48)


def test_get_xc_follows_the_reference_layouts():
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS["caps_transformer_small"]), device="cpu")
    batch = {"image": torch.randn(3, 80, 848, dtype=torch.float64), "feature": torch.randn(3, 1, 512)}
    x, c = m.get_xc(batch)
    assert x.shape == (3, 1, 80, 848) and x.dtype == torch.float32 and torch.equal(x[:, 0], batch["image"].float())
    assert c.shape == (3, 512, 1) and torch.equal(c[:, :, 0], batch["feature"][:, 0])
    x2, c2 = m.get_xc(batch, N=2)
    assert x2.shape[0] == c2.shape[0] == 2


def _val_loss_inputs(tmp_path, monkeypatch):
    """A caps_transformer_small YAML, mels in [0, 1] in the nested layout tools/extract_mel.py writes (one 860 frames wide, one 848), and three
    captions of two clips."""
    import yaml
    from tests.helpers import bpe_vocab_file
    monkeypatch.setenv("DIFFSOUND_BPE_VOCAB", bpe_vocab_file(tmp_path))
    cfg = tmp_path / "caps_transformer_small.yaml"
    cfg.write_text(yaml.safe_dump({"model": ar_transformer_config(**AR_CONFIGS["caps_transformer_small"])}))
    mels = tmp_path / "mels"
    (mels / "a").mkdir(parents=True)
    (mels / "b" / "c").mkdir(parents=True)
    mel = np.random.default_rng(0).random((80, 860), dtype=np.float32)
    np.save(mels / "a" / "Y1_mel.npy", mel)
    np.save(mels / "b" / "c" / "Y2_mel.npy", mel[:, 3:851])
    caps = tmp_path / "captions.csv"
    caps.write_text("file_name,caption\nY1.wav,a dog barks\nY1.wav,a dog barks twice\nY2.wav,rain on a roof\n")
    return cfg, mels, caps, mel


def test_ar_val_loss_dry_run(tmp_path, monkeypatch):
    """tools/ar_val_loss.py builds the model, reads the captions, pairs each with its <name>_mel.npy found anywhere under --mels, prepares the mel
    as caps.py's validation data does (center crop 80 x 848, then 2 * crop - 1) and stops before the first kernel; a caption without a mel and a
    name found twice are refused, naming the file."""
    from tools import ar_val_loss as V
    cfg, mels, caps, mel = _val_loss_inputs(tmp_path, monkeypatch)
    model, text, _, jobs = V.main(["--config", str(cfg), "--captions", str(caps), "--mels", str(mels), "--batch-size", "2", "--dry-run"])
    assert isinstance(model, Net2NetTransformer) and text.pick_last_embedding
    y1, y2 = str(mels / "a" / "Y1_mel.npy"), str(mels / "b" / "c" / "Y2_mel.npy")
    assert jobs == [(y1, "a dog barks"), (y1, "a dog barks twice"), (y2, "rain on a roof")]
    x = V.load_mel(y1)
    assert torch.equal(x, 2 * torch.from_numpy(mel[:, 6:854]) - 1)
    assert x.shape == (80, 848) and float(x.min()) >= -1 and float(x.max()) <= 1 and float(x.min()) < -0.9 and float(x.max()) > 0.9
    assert torch.equal(V.load_mel(y2), 2 * torch.from_numpy(mel[:, 3:851]) - 1)
    np.save(mels / "Y2_mel.npy", mel)
    with pytest.raises(ValueError, match="Y2_mel.npy is under --mels more than once"):
        V.main(["--config", str(cfg), "--captions", str(caps), "--mels", str(mels), "--dry-run"])
    caps.write_text("file_name,caption\nY1.wav,a dog barks\n")  # a duplicate the captions do not need is ignored
    assert len(V.main(["--config", str(cfg), "--captions", str(caps), "--mels", str(mels), "--dry-run"])[3]) == 1
    caps.write_text("file_name,caption\nY3.wav,silence\n")
    with pytest.raises(FileNotFoundError, match="Y3"):
        V.main(["--config", str(cfg), "--captions", str(caps), "--mels", str(mels), "--dry-run"])
