"""Diffsound's small denoiser (caps_small_transformer.yaml: 18 layers, n_embd 512, 16 heads of 32) on the CPU: the oracle against the reference's
head_dim-32 fixtures (made by oracle/gen_golden_small.py from the unmodified reference), the drop-in DALLE built from the YAML, argument
refusals, what ptxas made of the head_dim-32 split attention kernel, and the head_dim-64 attention kernels unchanged by the templating."""
import json
import os
import re
import shutil
import subprocess
import tempfile

import pytest
import torch

from oracle import diffsound_oracle as O
from oracle.gen_golden_small import portable_params
from tests.helpers import ROOT, bpe_vocab_file, load_golden

GOLDEN = os.path.join(ROOT, "tests", "golden")
CFG = os.path.join(GOLDEN, "ref_configs", "caps_small_transformer.yaml")
CSRC = os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc")


def _cfg():
    """The fixture's schedule buffers plus its parameters, regenerated from their shapes exactly as oracle/gen_golden_small.py loaded them into
    the reference."""
    sd, g = load_golden("xf_small_tiny.npz")
    sd.update(portable_params(json.loads(str(g["__param_shapes"]))))
    K, D, NL, NH, CD, B, L = [int(v) for v in g["__cfg"]]
    assert D // NH == 32
    return sd, g, K, NL, NH


def test_oracle_logits_match_reference():
    sd, g, K, NL, NH = _cfg()
    cond, x_t, t = torch.from_numpy(g["in_cond"]), torch.from_numpy(g["in_x_t"]).long(), torch.from_numpy(g["in_t"])
    logits = O.transformer_forward(sd, x_t, cond, t, n_layer=NL, n_head=NH, spatial=(5, 53))
    ref = torch.from_numpy(g["out_logits"])
    assert logits.shape == ref.shape
    assert float((logits - ref).abs().max() / ref.abs().max()) <= 1e-5


def test_oracle_staged_methods_match_reference():
    """The truncating predict_start and q_posterior on the reference's logits, bit for bit."""
    sd, g, K, NL, NH = _cfg()
    x_t, t = torch.from_numpy(g["in_x_t"]).long(), torch.from_numpy(g["in_t"])
    ref = torch.from_numpy(g["out_logits"])
    sched = {k: sd[k] for k in sd if k.startswith("log_")}
    lp = O.nucleus_filter(O.predict_start_tail(ref), 0.85)
    assert torch.equal(lp, torch.from_numpy(g["out_lp"]))
    post = O.q_posterior(sched, lp, O.index_to_log_onehot(x_t, K + 1), t, 100)
    assert torch.equal(post, torch.from_numpy(g["out_post"]))


def test_oracle_100_step_sample_matches_reference_tokens():
    sd, g, K, NL, NH = _cfg()
    gen = torch.Generator().manual_seed(int(g["__seed"][0]))  # the MT19937 stream the reference's rand_like consumed
    tok = O.sample(sd, torch.from_numpy(g["in_cond"]), gen, n_layer=NL, n_head=NH, spatial=(5, 53))
    assert torch.equal(tok, torch.from_numpy(g["out_sample_tokens"]).long())


@pytest.fixture
def bpe_vocab(tmp_path, monkeypatch):
    path = bpe_vocab_file(tmp_path)
    monkeypatch.setenv("DIFFSOUND_BPE_VOCAB", path)
    return path


def test_dropin_from_yaml_has_reference_state_dict_keys_and_shapes(bpe_vocab):
    """Every key of the reference DALLE built with caps_small_transformer.yaml's codec and diffusion model exists in the drop-in built from the
    same YAML, with the same shape; the drop-in's other keys are the CLIP condition embedding (left out of the fixture) and attention masks."""
    import _pkg
    _pkg.load()
    import yaml
    from diffsound_b200.utils.misc import instantiate_from_config, retarget_config
    with open(CFG) as f:
        cfg = yaml.full_load(f)["model"]
    cfg["params"]["content_codec_config"]["params"]["ckpt_path"] = None
    new = retarget_config(cfg)
    new["params"]["content_codec_config"]["params"]["lossconfig"] = None
    new["params"]["condition_codec_config"]["params"]["tokenizer_config"]["params"]["bpe_path"] = bpe_vocab
    model = instantiate_from_config(new)
    with open(os.path.join(GOLDEN, "caps_small_transformer_state_dict.json")) as f:
        ref = json.load(f)
    mine = {k: list(v.shape) for k, v in model.state_dict().items()}
    missing = sorted(k for k in ref if k not in mine)
    assert not missing, missing[:5]
    wrong = sorted(k for k in ref if mine[k] != ref[k])
    assert not wrong, [(k, mine[k], ref[k]) for k in wrong[:5]]
    extra = [k for k in mine if k not in ref and not k.startswith("transformer.condition_emb.") and "attn2.mask" not in k]
    assert not extra, extra[:5]
    tr = model.transformer.transformer
    assert (tr.n_embd, tr.n_head, len(tr.blocks)) == (512, 16, 18)


def test_builder_config_matches_yaml():
    import _pkg
    _pkg.load()
    import yaml
    from diffsound_b200.utils.builders import DALLE_CONFIGS, dalle_config
    with open(CFG) as f:
        tp = yaml.full_load(f)["model"]["params"]["diffusion_config"]["params"]
    c = DALLE_CONFIGS["caps_small_transformer"]
    mine = dalle_config(CD=512, **c)["params"]["diffusion_config"]["params"]
    for key in ("n_layer", "n_embd", "n_head", "condition_dim", "mlp_hidden_times"):
        assert mine["transformer_config"]["params"][key] == tp["transformer_config"]["params"][key], key
    assert mine["content_emb_config"]["params"]["embed_dim"] == tp["content_emb_config"]["params"]["embed_dim"] == 512


def test_generate_samples_cli_dry_run(tmp_path, bpe_vocab):
    import importlib.util
    spec = importlib.util.spec_from_file_location("generate_samples", os.path.join(ROOT, "tools", "generate_samples.py"))
    gs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gs)
    csvp = tmp_path / "val.csv"
    csvp.write_text("file_name,caption\nY1.wav,a dog barks\nY2.wav,rain\n")
    model, vocoder, caps, st = gs.main(["--config", CFG, "--captions", str(csvp), "--out", str(tmp_path / "o"), "--dry-run"])
    assert caps == {"Y1.wav": ["a dog barks"], "Y2.wav": ["rain"]}
    assert type(model).__module__.startswith("diffsound_b200.") and model.transformer.transformer.n_embd == 512
    assert not (tmp_path / "o").exists()


def test_head_dim_refusals_before_launch():
    """On CPU tensors (nothing launched): a head dimension other than 32 / 64, and fp16 operands at 32, are refused before the CUDA check."""
    import _pkg
    _pkg.load()
    from diffsound_b200 import ops
    x = torch.zeros(4, 96)
    for hd in (16, 48, 128):
        with pytest.raises(ValueError, match="head_dim"):
            ops.attention(x, x, x, x, B=1, H=1, Lq=4, Lk=4, scale=1.0, head_dim=hd)
        with pytest.raises(ValueError, match="head_dim"):
            ops.attention_tc_split(x.half(), x.half(), x.half(), x.half(), q_lo=48, k_lo=48, v_lo=48, o_lo=48, B=1, H=1, Lq=4, Lk=4, scale=1.0,
                                   head_dim=hd)


# ------------------------------------------------------------------ SASS
def _tool(name):
    for p in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name), shutil.which(name)):
        if p and os.access(p, os.X_OK):
            return p
    return None


def _nvcc_flags():
    # the Makefile's flags for one translation unit
    return ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"),
            "-I" + CSRC, "--expt-relaxed-constexpr"]


@pytest.fixture(scope="module")
def hd32_sass(tmp_path_factory):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("nvcc / cuobjdump not installed")
    out = str(tmp_path_factory.mktemp("attn32_sass") / "attention_tc_split_hd32.o")
    r = subprocess.run([nvcc, *_nvcc_flags(), "-Xptxas", "-v", "-c", os.path.join(CSRC, "attention_tc_split_hd32.cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    ins, on, names = [], False, []
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            on = "attention_tc_split_kernel" in m.group(1)
            names.append(m.group(1))
        elif on:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
            if m:
                ins.append(m.group(1))
    assert [n for n in names if "attention_tc_split_kernel" in n] and len(names) == 1, names
    return r.stderr, ins


def test_hd32_kernel_keeps_the_wgmma_pipeline_and_does_not_spill(hd32_sass):
    log, ins = hd32_sass
    for code in ("C7510", "C7514", "C7519"):
        assert code not in log, [l for l in log.splitlines() if code in l][:3]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    attn = [p for p in props if "attention_tc_split_kernel" in p[0]]
    assert len(attn) == 1 and attn[0][1:] == ("0", "0", "0"), attn
    bad = [i for i in ins if re.match(r"(@!?U?P\w+\s+)?(CALL|LDL|STL)\b", i)]
    assert not bad, bad[:3]


def test_hd32_s_issues_as_6_and_pv_as_12(hd32_sass):
    """S: one back-to-back group of 6 HGMMA.64x64x16 from shared memory (3 split passes x 2 k-steps); P V: one group of 12 HGMMA.64x32x16 with P
    from registers and V read transposed (3 passes x 4 k-steps of 16 keys)."""
    _, ins = hd32_sass
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
    assert [len(g) for g in groups] == [6, 12], [len(g) for g in groups]
    s, pv = groups
    assert all(i.startswith("HGMMA.64x64x16.F32 ") and "gdesc" in i and "tnspB" not in i and not re.search(r", R\d+, gdesc", i) for i in s), s
    assert all(i.startswith("HGMMA.64x32x16.F32 ") and "tnspB" in i and re.search(r"F32 R\d+, R\d+, gdesc", i) for i in pv), pv


def _kernel_key(mangled):
    """A kernel's name without the anonymous-namespace tag and with the head-dimension template argument dropped when it is 64, so the
    head_dim-64 instantiation of a templated kernel keys like the plain kernel it replaced; other head dims get a '<hd>' suffix."""
    assert mangled.startswith("_ZN"), mangled
    pos, parts = 3, []
    while (m := re.match(r"\d+", mangled[pos:])):  # <length><identifier> nested-name components
        n, pos = int(m.group()), pos + len(m.group())
        parts.append(mangled[pos:pos + n])
        pos += n
    name = [c for c in parts if c != "dsb" and not c.startswith("_GLOBAL__N")][-1]
    t = re.match(r"ILi(\d+)EE", mangled[pos:])
    return name if not t or t.group(1) == "64" else f"{name}<{t.group(1)}>"


@pytest.mark.parametrize("unit", ["attention.cu", "attention_tc_split.cu"])
def test_head_dim_64_attention_kernels_unchanged(unit):
    """The head_dim-64 fp32 and split-fp16 attention kernels compile to the same instruction sequences as before they were templated on the head
    dimension (digests in tests/golden/attention_sass.json, addresses and encodings ignored)."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    from tests.sass_digest import sass_digests
    with open(os.path.join(GOLDEN, "attention_sass.json")) as f:
        ref = json.load(f)
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != ref["nvcc"]:
        pytest.skip(f"digests were recorded with {ref['nvcc']}, this is {ver}")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "unit.o")
        subprocess.run([nvcc, *_nvcc_flags(), "-c", os.path.join(CSRC, unit), "-o", obj], check=True)
        mine = {_kernel_key(k): v for k, v in sass_digests(obj, cuobjdump).items()}
    for name, digest in ref["functions"][unit].items():
        assert mine.get(name) == digest, (name, sorted(mine))
