"""Every drop-in module's engine follows the module's weights: after an in-place update, after a round trip through the CPU and in a deep copy,
each call must equal a fresh module built from the same state_dict, bit for bit."""
import copy
import os
import tempfile

import pytest
import torch

from tests import gpu_common  # noqa: F401  (loads the package)

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _denoiser():
    from diffsound_b200.utils.builders import build_diffusion_transformer
    torch.manual_seed(0)
    return build_diffusion_transformer(32, 128, 2, 2, 64)


def _run_denoiser(m):
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(2, 77, 64, generator=g)
    cond = (cond / cond.norm(dim=-1, keepdim=True)).to(DEV)
    x = torch.randint(0, 33, (2, 265), generator=g).to(DEV)
    t = torch.tensor([99, 40]).to(DEV)
    torch.manual_seed(3)
    tok = m.sample(None, None, cond, filter_ratio=0, batch_size=2)["content_token"]  # captures the sampling graph
    return tok, m.transformer(x, cond, t)


def _vq():
    from tests.test_gpu_decoder import build_vq
    torch.manual_seed(0)
    return build_vq(32, 64, 32, (1, 1, 1, 1, 2))


def _run_decoder(m):
    ids = torch.randint(0, 32, (2, 265), generator=torch.Generator().manual_seed(2)).to(DEV)
    return (m.decode_tokens(ids, (5, 53)),)  # captures a graph


def _run_encoder(m):
    mel = torch.rand(2, 1, 80, 96, generator=torch.Generator().manual_seed(3)).to(DEV)
    quant, _, (_, _, ids) = m.encode(mel)
    return quant, ids, m.last_latent


def _melgan():
    from diffsound_b200.vocoder.modules import Generator
    torch.manual_seed(0)
    with torch.no_grad():  # torch's weight_norm caches `weight` as a non-leaf tensor under autograd, which copy.deepcopy refuses
        return Generator(80, 4, 3).to(DEV).eval()


def _run_melgan(m):
    return (m(torch.rand(2, 80, 16, generator=torch.Generator().manual_seed(4)).to(DEV)),)


def _clip():
    from diffsound_b200.modeling.embeddings.clip_text_embedding import CLIPTextEmbedding
    torch.manual_seed(0)
    return CLIPTextEmbedding(num_embed=1000, text_layers=2, pick_last_embedding=False, embed_dim=512).to(DEV)


def _run_clip(m):
    return (m(torch.randint(0, 1000, (2, 77), generator=torch.Generator().manual_seed(5)).to(DEV)),)


def _gpt():
    from diffsound_b200.modeling.transformers.mingpt import GPTFeats
    torch.manual_seed(0)
    emb = {"target": "torch.nn.Conv1d", "params": dict(in_channels=64, out_channels=256, kernel_size=1, padding=0)}
    return GPTFeats(emb, dict(vocab_size=256, block_size=266, n_layer=2, n_head=4, n_embd=256)).to(DEV).eval()


def _run_gpt(m):
    g = torch.Generator().manual_seed(6)
    idx = torch.randint(0, 256, (2, 40), generator=g).to(DEV)
    feats = torch.randn(2, 64, 1, generator=g).to(DEV)
    targets = torch.randint(0, 256, (2, 41), generator=g).to(DEV)
    return m(idx, feats)[0], m.forward_loss(idx, feats, targets, 0)[1]  # the KV-cached decode's and the prefill's captured graphs


def _act():
    from diffsound_b200.evaluation.audiocaption import ACT
    from oracle import act_oracle as O
    from tests.test_cpu_audiocaption import CASES, EOS, V, config
    c = CASES["cap"]
    m = ACT(config(c), V)
    m.load_state_dict(O.seeded_state_dict(m.state_dict(), c["seed"], EOS, c["eos_bias"]))
    return m.to(DEV).eval()


def _act_inputs():
    g = torch.Generator().manual_seed(7)
    return torch.rand(2, 64, 80, generator=g).to(DEV), torch.randint(0, 5000, (2, 6), generator=g).to(DEV)


def _run_act(m):
    from tests.test_cpu_audiocaption import SOS
    spec, tgt = _act_inputs()
    mem = m.encode(spec)  # captures the encoder graph
    return mem, m.decode(mem, tgt), m.engine.greedy(mem.transpose(0, 1), SOS, max_len=5)


def _melception():
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    from oracle import melception_oracle as MO
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "w.pt")
        torch.save({"model": MO.make_melception_state_dict(21, "he")}, path)
        return Melception(309, ["2048", "logits"], path).to(DEV).eval()


def _run_melception(m):
    return m(torch.rand(2, 80, 96, generator=torch.Generator().manual_seed(8)).to(DEV) * 4 - 2)


CASES = {"denoiser": (_denoiser, _run_denoiser), "decoder": (_vq, _run_decoder), "encoder": (_vq, _run_encoder), "melgan": (_melgan, _run_melgan),
         "clip_text": (_clip, _run_clip), "gpt": (_gpt, _run_gpt), "act": (_act, _run_act), "melception": (_melception, _run_melception)}


def _fresh(build, m):
    f = build()
    f.load_state_dict(m.state_dict())
    return f


def _assert_same(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b), float((a.double() - b.double()).abs().max())


def _scale_parameters(m):
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(1.01)


@pytest.mark.parametrize("name", list(CASES))
def test_inplace_update_repacks(name):
    build, run = CASES[name]
    m = build()
    before = run(m)
    _scale_parameters(m)
    after = run(m)
    _assert_same(after, run(_fresh(build, m)))
    assert any(not torch.equal(a, b) for a, b in zip(before, after))


@pytest.mark.parametrize("name", list(CASES))
def test_update_on_the_cpu_then_back(name):
    build, run = CASES[name]
    m = build()
    run(m)
    m.cpu()
    _scale_parameters(m)
    m.cuda()
    _assert_same(run(m), run(_fresh(build, m)))


@pytest.mark.parametrize("name", list(CASES))
def test_deepcopy_after_a_first_call(name):
    build, run = CASES[name]
    m = build()
    run(m)
    cp = copy.deepcopy(m)
    _assert_same(run(cp), run(m))


def test_act_decode_after_an_update_projects_the_memory_again():
    """decode() on the memory of the last encode() reuses that encode's cross-attention K / V only while the weights are unchanged."""
    m = _act()
    spec, tgt = _act_inputs()
    mem = m.encode(spec)
    _scale_parameters(m)
    _assert_same((m.decode(mem, tgt),), (_fresh(_act, m).decode(mem, tgt),))
