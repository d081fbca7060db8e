"""The autoregressive SpecVQGAN transformer on the CPU: the fp32 oracle against the reference fixtures (oracle/gen_golden_ar.py ran the unmodified
reference), the drop-in's state_dict against the reference's for the three caps_transformer configs, argument refusals before anything is
launched, and the diffusion sampler's SASS unchanged by the shared Philox header."""
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import _pkg

_pkg.load()
from diffsound_b200.modeling.models.cond_transformer import Net2NetTransformer  # noqa: E402
from diffsound_b200.modeling.transformers.mingpt import GPTFeats  # noqa: E402
from diffsound_b200.utils.builders import AR_CONFIGS, ar_transformer_config, build_ar_transformer  # noqa: E402
from oracle import ar_oracle as A  # noqa: E402
from tests.helpers import ROOT  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _golden(name):
    with np.load(os.path.join(GOLDEN, name)) as z:
        return {k: z[k] for k in z.files}


def tiny_gpt(V, seed, **over):
    """The fixtures' weights: the reference init order under torch.manual_seed(seed), then ar_oracle.perturb_."""
    c = dict(A.TINY, **over)
    fe, gc = A.gpt_config(V, c["n_embd"], c["n_layer"], c["n_head"], c["Cf"])
    torch.manual_seed(seed)
    g = GPTFeats(fe, gc).eval()
    A.perturb_(g.state_dict(), seed)
    return g


@pytest.mark.parametrize("case", ["v32_tc1", "v32_tc3", "v2048_tc1", "v2048_tc3", "full"])
def test_oracle_forward_matches_reference(case):
    g = _golden("ar_forward.npz")
    V, Tc, seed = (int(v) for v in g[case + "/meta"])
    m = tiny_gpt(V, seed) if case != "full" else tiny_gpt(V, seed, n_embd=1024, n_layer=19, n_head=16, Cf=512)
    nl, nh = (A.TINY["n_layer"], A.TINY["n_head"]) if case != "full" else (19, 16)
    out = A.forward(m.state_dict(), torch.from_numpy(g[case + "/idx"]), torch.from_numpy(g[case + "/feats"]), n_layer=nl, n_head=nh)
    ref = torch.from_numpy(g[case + "/logits"])
    assert out.shape == ref.shape and out.shape[1] == Tc + g[case + "/idx"].shape[1]
    err = float((out - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err


def test_oracle_sample_matches_reference():
    g = _golden("ar_sample.npz")
    V, seed, steps = (int(v) for v in g["meta"])
    m = tiny_gpt(V, seed)
    sd, feats, gt = m.state_dict(), torch.from_numpy(g["feats"]), torch.from_numpy(g["gt"])
    n = 0
    while f"c{n}/ids" in g:
        mode, top_k, temperature, do_sample, rseed = g[f"c{n}/args"].tolist()
        x0 = gt[:, :0] if mode == 0 else gt[:, :steps // 2]
        torch.manual_seed(int(rseed))
        out = A.sample(sd, x0, feats, steps - x0.shape[1], n_layer=A.TINY["n_layer"], n_head=A.TINY["n_head"], temperature=temperature,
                       sample=bool(do_sample), top_k=None if top_k < 0 else int(top_k))
        assert torch.equal(out, torch.from_numpy(g[f"c{n}/ids"])), (n, g[f"c{n}/args"])
        n += 1
    assert n == 32


@pytest.mark.parametrize("name", list(AR_CONFIGS))
def test_dropin_state_dict_matches_reference(name):
    with open(os.path.join(GOLDEN, "ar_state_dict_keys.json")) as f:
        ref = json.load(f)[name]
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS[name]), device="cpu")
    mine = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert mine == ref
    assert isinstance(m, Net2NetTransformer)


def test_refusals_before_launch():
    """On the CPU (no device, nothing launched): every refusal is raised before the CUDA check."""
    feats = torch.randn(1, 16, 1)
    with pytest.raises(ValueError, match="vocab_size"):
        tiny_gpt(5000, 0)(torch.zeros(1, 3, dtype=torch.long), feats)
    with pytest.raises(ValueError, match="head_dim"):
        tiny_gpt(32, 0, n_head=1)(torch.zeros(1, 3, dtype=torch.long), feats)
    with pytest.raises(AssertionError, match="block size"):
        tiny_gpt(32, 0)(torch.zeros(1, 266, dtype=torch.long), feats)
    g = tiny_gpt(32, 0)
    with pytest.raises(AssertionError, match="block size"):
        g.sample_tokens(torch.zeros(1, 0, dtype=torch.long), feats, 267)
    with pytest.raises(ValueError, match="top_k"):
        g.sample_tokens(torch.zeros(1, 0, dtype=torch.long), feats, 4, top_k=33)
    with pytest.raises(ValueError, match="top_k"):
        g.sample_tokens(torch.zeros(1, 0, dtype=torch.long), feats, 4, top_k=0)
    with pytest.raises(NotImplementedError, match="Conv1d"):
        fe, gc = A.gpt_config(32, 128, 1, 2, 16)
        fe["params"]["kernel_size"] = 3
        GPTFeats(fe, gc)(torch.zeros(1, 3, dtype=torch.long), feats)
    with pytest.raises(RuntimeError, match="CUDA"):
        g(torch.zeros(1, 3, dtype=torch.long), feats)


def _tool(name):
    for p in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name), shutil.which(name)):
        if p and os.access(p, os.X_OK):
            return p
    return None


def test_diffusion_sampler_sass_unchanged():
    """csrc/sampler.cu takes its Philox replay from philox.cuh (shared with ar_decode.cu): every function of sampler.cu compiles to the same
    instruction sequence as before the move (digests in tests/golden/sampler_sass.json, addresses and encodings ignored)."""
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    from tests.sass_digest import sass_digests
    with open(os.path.join(GOLDEN, "sampler_sass.json")) as f:
        ref = json.load(f)
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1]
    if ver != ref["nvcc"]:
        pytest.skip(f"digests were recorded with {ref['nvcc']}, this is {ver}")
    pkg = os.path.join(ROOT, "text-to-sound-synthesis_b200")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "sampler.o")
        subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
                        "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(pkg, "csrc"), "--expt-relaxed-constexpr", "-c",
                        os.path.join(pkg, "csrc", "sampler.cu"), "-o", obj], check=True)
        assert sass_digests(obj, cuobjdump) == ref["functions"]


def test_generate_samples_ar_dry_run(tmp_path, monkeypatch):
    """tools/generate_samples_ar.py builds the reference's caps_transformer-style YAML on the drop-ins, the CLIP text tower and the tokenizer,
    pairs every caption with its output name and stops before the first kernel."""
    import yaml
    from tests.helpers import bpe_vocab_file
    from tools import generate_samples_ar as G
    monkeypatch.setenv("DIFFSOUND_BPE_VOCAB", bpe_vocab_file(tmp_path))
    cfg = tmp_path / "caps_transformer_small.yaml"
    cfg.write_text(yaml.safe_dump({"model": ar_transformer_config(**AR_CONFIGS["caps_transformer_small"])}))
    caps = tmp_path / "captions.csv"
    caps.write_text("file_name,caption\nY1.wav,a dog barks\nY1.wav,a dog barks twice\nY2.wav,rain on a roof\n")
    model, text, vocoder, jobs = G.main(["--config", str(cfg), "--captions", str(caps), "--out", str(tmp_path / "out"), "--dry-run"])
    assert isinstance(model, Net2NetTransformer) and vocoder is None and text.pick_last_embedding
    assert jobs == [("Y1", 0, "a dog barks"), ("Y1", 1, "a dog barks twice"), ("Y2", 0, "rain on a roof")]
    assert not (tmp_path / "out").exists()
