"""The 2048-code AudioSet codebook (Diffsound caps_2048.yaml: K = 2048, 2049 sampler classes) end to end on the H100: the denoiser chain
against the fp32 oracle, the public sample(), the training loss and step, and the codec at 2048 codes.  The sampler runs on the CTA-per-column
kernel here (dsb_posterior_sample_wide), chosen by DiffusionTransformer._sampler_ops; test_gpu_sampler_wide.py checks that kernel per element."""
import pytest
import torch

from oracle import diffsound_oracle as O
from tests.helpers import build_dt, rel_err
from tests.test_gpu_decoder import build_vq
from tests.test_gpu_train import _oracle_step
from tests.test_gpu_train import test_q_sample_and_fused_loss_match_oracle as _loss_vs_oracle

pytestmark = pytest.mark.gpu

K = 2048
D, NL, NH, CD, L = 1024, 19, 16, 512, 265


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


@pytest.fixture(scope="module")
def TO():
    from tests import gpu_common  # noqa: F401  (loads the package)
    from diffsound_b200 import train_ops
    return train_ops


def _run_chain(m, cond, us, steps):
    """Fused step on supplied uniforms (no torch RNG), through the model's own sampler choice: the token grid after `steps` steps."""
    eng = m.transformer.engine
    B = cond.shape[0]
    kv = eng.encode_condition(cond)
    x = torch.full((B, L), m.num_classes - 1, dtype=torch.long, device="cuda")
    mode, r, k = m._trunc()
    sample = m._sampler_ops()[0]
    for i, ti in enumerate(range(99, 99 - steps, -1)):
        t = torch.full((B,), ti, dtype=torch.long, device="cuda")
        x = sample(eng.forward(x, kv, t, cond.shape[1]), x, t, us[i], m._sched(), T=100, trunc_mode=mode, trunc_r=r, trunc_k=k)
    return x


def _cond(B, g):
    c = torch.randn(B, 77, CD, generator=g)
    return c / c.norm(dim=-1, keepdim=True)


def test_sampler_choice_follows_the_codebook(G):
    ops = G.ops
    for k, wide in ((256, False), (1055, False), (1056, True), (2048, True)):
        m = build_dt(k, 128, 1, 2, 64)
        assert m._sampler_ops() == ((ops.posterior_sample_wide, ops.posterior_sample_wide_loop) if wide else
                                    (ops.posterior_sample, ops.posterior_sample_loop)), k


def test_k2048_codebook_19_layers_token_ids_equal_oracle(G):
    """19 layers, D = 1024, K = 2048, B = 4: 10 free-running top0.85r steps from all-[MASK]; every token id equals the fp32 oracle's."""
    B, steps = 4, 10
    torch.set_num_threads(min(16, torch.get_num_threads()))
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)
    g = torch.Generator().manual_seed(8)
    cond = _cond(B, g)
    us = [torch.rand(B, K + 1, L, generator=g) for _ in range(steps)]
    ref = O.sample(sd, cond, lambda i: us[i], n_layer=NL, n_head=NH, spatial=(5, 53), steps=list(range(99, 99 - steps, -1)))
    m = build_dt(K, D, NL, NH, CD, sd, precision="f16x3")
    m.truncation = "top0.85r"
    got = _run_chain(m, cond.cuda(), [u.cuda() for u in us], steps).cpu()
    assert int((ref != K).sum()) > 0
    assert torch.equal(got, ref), f"{int((got != ref).sum())} of {ref.numel()} token ids differ"


def test_k2048_public_sample_batch16(G):
    """Full-size denoiser, K = 2048, B = 16.  sample() (CUDA graph, torch RNG): ids in [0, K) with no [MASK] left after 100 steps, two runs
    identical, and the fused graph loop, the eager loop and the stage-by-stage reference-named methods give the same tokens.  On supplied
    uniforms, clip j gets the same tokens alone as inside the batch."""
    torch.manual_seed(0)
    m = build_dt(K, D, NL, NH, CD)
    m.truncation = "top0.85r"
    g = torch.Generator().manual_seed(9)
    B = 16
    cond = _cond(B, g).cuda()
    toks = []
    for mode in ("graph", "graph", "eager", "unfused"):
        m.use_cuda_graph = mode == "graph"
        if mode == "unfused":
            m.p_sample = m.p_sample
        torch.manual_seed(1234)
        toks.append(m.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"].cpu())
    del m.__dict__["p_sample"]
    m.use_cuda_graph = True
    tok = toks[0]
    assert tok.shape == (B, L) and int(tok.min()) >= 0 and int(tok.max()) < K
    assert torch.equal(toks[0], toks[1]), "two sample() runs differ"
    assert torch.equal(toks[1], toks[2]), "CUDA-graph replay changed the sampled tokens"
    assert torch.equal(toks[2], toks[3]), "fused and stage-by-stage paths disagree"
    steps = 12
    us = [torch.rand(B, K + 1, L, generator=g).cuda() for _ in range(steps)]
    full = _run_chain(m, cond, us, steps)
    for j in (0, 7, 15):
        solo = _run_chain(m, cond[j:j + 1], [u[j:j + 1].contiguous() for u in us], steps)
        assert torch.equal(solo[0], full[j]), f"clip {j} depends on its batch neighbours"


@pytest.mark.parametrize("k", [1056, 1087, 2047, 2048, 4095])
def test_train_loss_wide_matches_oracle(G, TO, k):
    """The CTA-per-column training loss (K above 1055, up to the ceiling 4095) against the oracle's autograd, with the assertions and
    tolerances of the warp kernel's test in test_gpu_train.py."""
    _loss_vs_oracle(G, TO, k)


def test_k2048_training_step_matches_oracle_autograd(G, TO):
    """D = 128 / 2 heads / 2 layers / K = 2048, tf32, B = 4: loss and every parameter gradient vs torch autograd through the oracle, at the
    tolerances of the midsize tf32 step (loss 1.5e-5, gradient 1.25e-2)."""
    _oracle_step(G, TO, "k2048", K, 128, 2, 2, 96, torch.tensor([3, 0, 77, 99]), torch.tensor([0.01, 0.02, 0.005, 0.01]), "tf32", 1.5e-5, 1.25e-2)


def test_k2048_decode_and_gather_flag(G):
    """decode_to_img of ids up to 2047 on a 2048-code codebook vs the oracle (the decoder test's 1.2e-4); id 2048 sets the gather's err_flag."""
    sd = O.make_decoder_state_dict(n_embed=K, seed=2)
    m = build_vq(K, 256, 128, (1, 1, 2, 2, 4), sd)
    ids = torch.randint(0, K, (2, 265), generator=torch.Generator().manual_seed(9))
    ids[0, 0], ids[1, 264] = K - 1, 0
    ref = O.decode_to_img(sd, ids)
    mel = m.decode_tokens(ids.cuda(), (5, 53)).cpu()
    err = rel_err(mel, ref)
    print("decoder K=2048 rel err", err)
    assert mel.shape == (2, 1, 80, 848) and err < 1.2e-4
    cb = sd["content_codec.quantize.embedding.weight"].cuda()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    G.ops.codebook_gather_padded(ids.cuda(), cb, 5, 53, split_f16=True, err_flag=flag)
    assert int(flag) == 0
    bad = ids.clone()
    bad[1, 17] = K
    G.ops.codebook_gather_padded(bad.cuda(), cb, 5, 53, split_f16=True, err_flag=flag)
    assert int(flag) == 1


def test_k2048_encoder_matches_oracle(G):
    """Real ddconfig encoder with a 2048-code codebook: latents within 1e-3, >= 99 % of the 265 codes equal the oracle's."""
    torch.manual_seed(5)
    m = build_vq(K, 256, 128, (1, 1, 2, 2, 4))
    g = torch.Generator().manual_seed(6)
    mel = torch.rand(1, 1, 80, 848, generator=g) * 2 - 1
    sd = {"content_codec." + k: v.detach().cpu() for k, v in m.state_dict().items()}
    z_ref = O._conv(sd, "content_codec.quant_conv.", O.encoder_forward(sd, mel), 0)
    zf = z_ref.permute(0, 2, 3, 1).reshape(-1, 256)
    cb = zf.mean(0, keepdim=True) + torch.randn(K, 256, generator=g) * zf.std(0, keepdim=True)
    sd["content_codec.quantize.embedding.weight"] = cb
    m.quantize.embedding.weight.data.copy_(cb.cuda())
    m.enc_engine.repack()
    _, tok_ref = O.encode_to_tokens(sd, mel)
    quant, _, info = m.encode(mel.cuda())
    e_z = rel_err(m.last_latent.cpu(), z_ref)
    ids = info[2].view(1, 265).cpu()
    col_major = torch.arange(265).reshape(5, 53).t().reshape(-1)
    agree = float((ids[:, col_major] == tok_ref).float().mean())
    print("encoder K=2048: z rel err", e_z, "token agreement", agree)
    assert quant.shape == (1, 256, 5, 53) and e_z < 1e-3 and agree >= 0.99 and int(ids.max()) < K
