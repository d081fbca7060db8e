"""The 2048-code AudioSet codebook (Diffsound caps_2048.yaml) on the CPU: the oracle against the reference's K = 2048 fixtures (made by
oracle/gen_golden_k2048.py from the unmodified reference), and the drop-in DALLE built from caps_2048.yaml (tests/golden/ref_configs)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import diffsound_oracle as O
from tests.helpers import ROOT, bpe_vocab_file, load_golden, sampler_case_inputs

K = 2048
CFG = os.path.join(ROOT, "tests", "golden", "ref_configs", "caps_2048.yaml")


def test_schedule_k2048_matches_reference_buffers():
    _, ref = load_golden("schedule_k2048.npz")
    mine = O.schedule_buffers(100, K + 1)
    for k, v in ref.items():
        assert np.array_equal(mine[k].numpy(), v), k


@pytest.mark.parametrize("case", [0, 1, 2])
@pytest.mark.parametrize("trunc", ["top0.85r", None, "top20p"])
def test_sampler_cases_k2048_match_reference(case, trunc):
    _, g = load_golden("sampler_cases_k2048.npz")
    logits, x_t, t, u = sampler_case_inputs(case, K=K)
    sched = O.schedule_buffers(100, K + 1)
    nxt, post, lp = O.posterior_sample_step(sched, logits, x_t, t, u, T=100, truncation=trunc, first_step_carrier=(case == 0))
    tag = f"c{case}_{ {'top0.85r': 'nuc', None: 'raw', 'top20p': 'topk'}[trunc] }"
    assert torch.equal(lp[:, :, :6], torch.from_numpy(g[tag + "_lp_head"]))
    assert torch.equal(post[:, :, :6], torch.from_numpy(g[tag + "_post_head"]))
    same = nxt == torch.from_numpy(g[tag + "_next"]).long()
    # the reference leaves equal log-probs in no defined order; a different id is allowed only where its top-2 margin is a tie
    assert bool((same | (torch.from_numpy(g[tag + "_margin"]) == 0)).all()), int((~same).sum())


@pytest.fixture
def bpe_vocab(tmp_path, monkeypatch):
    """Points the tokenizer at the stored CLIP BPE merge table."""
    path = bpe_vocab_file(tmp_path)
    monkeypatch.setenv("DIFFSOUND_BPE_VOCAB", path)
    return path


def _build_dropin(bpe_path):
    import _pkg
    _pkg.load()
    import yaml
    from diffsound_b200.utils.misc import instantiate_from_config, retarget_config
    with open(CFG) as f:
        cfg = yaml.full_load(f)["model"]
    cfg["params"]["content_codec_config"]["params"]["ckpt_path"] = None
    new = retarget_config(cfg)
    new["params"]["content_codec_config"]["params"]["lossconfig"] = None
    new["params"]["condition_codec_config"]["params"]["tokenizer_config"]["params"]["bpe_path"] = bpe_path
    return instantiate_from_config(new)


def test_caps_2048_dropin_has_reference_state_dict_keys_and_shapes(bpe_vocab):
    """Every key of the reference DALLE built with caps_2048.yaml's codec and diffusion model exists in the drop-in with the same shape; the
    drop-in's other keys are the CLIP condition embedding (left out of the fixture) and the attention masks."""
    with open(os.path.join(ROOT, "tests", "golden", "caps_2048_state_dict.json")) as f:
        ref = json.load(f)
    model = _build_dropin(bpe_vocab)
    mine = {k: list(v.shape) for k, v in model.state_dict().items()}
    missing = sorted(k for k in ref if k not in mine)
    assert not missing, missing[:5]
    wrong = sorted(k for k in ref if mine[k] != ref[k])
    assert not wrong, [(k, mine[k], ref[k]) for k in wrong[:5]]
    extra = [k for k in mine if k not in ref and not k.startswith("transformer.condition_emb.") and "attn2.mask" not in k]
    assert not extra, extra[:5]
    assert ref["content_codec.quantize.embedding.weight"] == [K, 256]
    assert model.transformer.num_classes == K + 1 and model.transformer.transformer.content_emb.num_embed == K + 1


def test_generate_samples_cli_dry_run_on_caps_2048(tmp_path, bpe_vocab):
    import importlib.util
    spec = importlib.util.spec_from_file_location("generate_samples", os.path.join(ROOT, "tools", "generate_samples.py"))
    gs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gs)
    csvp = tmp_path / "val.csv"
    csvp.write_text("file_name,caption\nY1.wav,a dog barks\nY2.wav,rain\n")
    model, vocoder, caps, st = gs.main(["--config", CFG, "--captions", str(csvp), "--out", str(tmp_path / "o"), "--fast", "3", "--dry-run"])
    assert caps == {"Y1.wav": ["a dog barks"], "Y2.wav": ["rain"]} and st == "top0.85r,fast2"
    assert type(model).__module__.startswith("diffsound_b200.") and model.transformer.num_classes == K + 1
