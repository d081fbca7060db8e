"""Scoring the autoregressive SpecVQGAN transformer on the GPU: causal split-fp16 attention (attention_tc_split_causal.cu) against fp64, the
cross-entropy kernel (dsb_ar_cross_entropy) against fp64 log_softmax, and the full-sequence forward (AREngine.prefill) behind GPT.forward(targets),
GPTFeats.forward_loss and Net2NetTransformer.shared_step / validation_step against the fp32 oracle, the reference fixture and the KV-cached
forward."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _pkg

_pkg.load()
from diffsound_b200 import _lib, ops  # noqa: E402
from diffsound_b200.modeling.transformers.mingpt import GPT, GPTFeats  # noqa: E402
from diffsound_b200.utils.builders import AR_CONFIGS, ar_transformer_config, build_ar_transformer  # noqa: E402
from oracle import ar_oracle as A  # noqa: E402
from tests.helpers import ROOT  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = 7.0


@pytest.fixture(autouse=True)
def _fp32_oracle():
    """The oracle runs in fp32 on the GPU here: no TF32 in its matmuls or its Conv1d."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# ---------------------------------------------------------------- causal split attention
def _causal_case(B, H, L, hd, seed):
    """qkv (B*L, 6D) = the split pair [Qh Kh Vh | Ql Kl Vl] of random fp32 Q / K / V, and the fp64 causal attention of the pair's values."""
    D = H * hd
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B * L, 3 * D, generator=g) * 2).to(DEV)
    qkv = ops.split_f16(x)
    val = (qkv[:, :3 * D].double() + qkv[:, 3 * D:].double()).view(B, L, 3, H, hd).permute(2, 0, 3, 1, 4)  # (3, B, H, L, hd)
    s = val[0] @ val[1].transpose(-1, -2) / math.sqrt(hd)
    s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=DEV).triu(1), float("-inf"))
    ref = (torch.softmax(s, -1) @ val[2]).permute(0, 2, 1, 3).reshape(B * L, D)
    return qkv, ref


def _run_causal(qkv, B, H, L, hd, extra_rows=5):
    D = H * hd
    out = torch.full((B * L + extra_rows, 2 * D), SENTINEL, dtype=torch.float16, device=DEV)
    ops.attention_tc_split_causal(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], out[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D, B=B, H=H,
                                  L=L, scale=1.0 / math.sqrt(hd), head_dim=hd)
    return out


@pytest.mark.parametrize("hd", [64, 32])
@pytest.mark.parametrize("L", [1, 63, 64, 65, 128, 265, 266])
def test_causal_split_attention_vs_fp64(hd, L):
    B, H = 3, 16
    qkv, ref = _causal_case(B, H, L, hd, seed=L * 100 + hd)
    out = _run_causal(qkv, B, H, L, hd)
    D = H * hd
    o = out[:B * L, :D].double() + out[:B * L, D:].double()
    err = float((o - ref).abs().max() / ref.abs().max())
    assert err < 3e-6, (hd, L, err)
    assert bool((out[B * L:] == SENTINEL).all())  # rows past the last sequence are untouched
    assert torch.equal(_run_causal(qkv, B, H, L, hd), out)  # the same bits on a second run


@pytest.mark.parametrize("hd", [64, 32])
def test_causal_split_attention_graph_replay(hd):
    B, H, L = 16, 16, 266
    D = H * hd
    qkv, _ = _causal_case(B, H, L, hd, seed=5)
    eager = _run_causal(qkv, B, H, L, hd, extra_rows=0)
    out = torch.zeros_like(eager)
    call = lambda: ops.attention_tc_split_causal(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], out[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D,
                                                 o_lo=D, B=B, H=H, L=L, scale=1.0 / math.sqrt(hd), head_dim=hd)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    for _ in range(3):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)


def test_causal_split_attention_refusals():
    B, H, L, hd = 1, 2, 64, 64
    D = H * hd
    qkv, _ = _causal_case(B, H, L, hd, seed=1)
    out = torch.zeros(B * L, 2 * D, dtype=torch.float16, device=DEV)
    fn = _lib.lib().dsb_attention_tc_split_causal
    args = lambda Lq, Lk, head_dim: (qkv.data_ptr(), qkv.stride(0), 3 * D, qkv[:, D:].data_ptr(), qkv.stride(0), 3 * D, qkv[:, 2 * D:].data_ptr(),
                                     qkv.stride(0), 3 * D, out.data_ptr(), out.stride(0), D, B, H, Lq, Lk, 0.125, head_dim, ops._stream())
    with pytest.raises(RuntimeError, match="Lq == Lk"):
        _lib.check(fn(*args(64, 63, 64)), "dsb_attention_tc_split_causal")
    with pytest.raises(RuntimeError, match="head_dim=48"):
        _lib.check(fn(*args(64, 64, 48)), "dsb_attention_tc_split_causal")
    with pytest.raises(ValueError, match="head_dim"):
        ops.attention_tc_split_causal(qkv[:, :D], qkv[:, D:], qkv[:, 2 * D:], out, q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D, B=B, H=H, L=L,
                                      scale=0.125, head_dim=16)
    assert bool((out == 0).all())


# ---------------------------------------------------------------- cross-entropy
def _xent_ref(logits, targets, r0):
    """fp64 log_softmax / gather over rows r0 ... r0 + n - 1: (per-row NLL with 0 at -100, mean over the non-ignored rows)."""
    n = targets.shape[1]
    lp = torch.log_softmax(logits[:, r0:r0 + n].double(), -1)
    keep = targets != -100
    nll = -lp.gather(-1, targets.clamp(min=0)[..., None])[..., 0] * keep
    return nll, nll.sum() / keep.sum()


@pytest.mark.parametrize("V", [32, 256, 2048, 4096])
def test_cross_entropy_vs_fp64(V):
    B, T, r0, n = 5, 12, 3, 8
    g = torch.Generator().manual_seed(V)
    logits = (torch.randn(B, T, V, generator=g) * 4).to(DEV)
    targets = torch.randint(0, V, (B, n), generator=g)
    targets[0, 1] = targets[3, 0] = targets[4, 7] = -100
    targets = targets.to(DEV)
    loss, nll = ops.ar_cross_entropy(logits, targets, first_row=r0)
    ref_nll, ref_loss = _xent_ref(logits, targets, r0)
    assert float((nll.double() - ref_nll).abs().max()) < 2e-6 * max(1.0, float(ref_nll.abs().max()))
    assert bool((nll[targets == -100] == 0).all())
    assert abs(float(loss) - float(ref_loss)) < 1e-6 * float(ref_loss), (float(loss), float(ref_loss))
    torch_loss = F.cross_entropy(logits[:, r0:r0 + n].reshape(-1, V), targets.reshape(-1))
    assert abs(float(loss) - float(torch_loss)) < 2e-6 * float(ref_loss)


def test_cross_entropy_all_ignored_is_nan_and_bad_target_raises():
    logits = torch.randn(2, 4, 32, device=DEV)
    loss, nll = ops.ar_cross_entropy(logits, torch.full((2, 4), -100, dtype=torch.int64, device=DEV))
    assert math.isnan(float(loss)) and bool((nll == 0).all())
    assert math.isnan(float(F.cross_entropy(logits.reshape(-1, 32), torch.full((8,), -100, device=DEV))))
    for bad in (32, -1, 1 << 40):
        t = torch.zeros(2, 4, dtype=torch.int64, device=DEV)
        t[1, 2] = bad
        with pytest.raises(IndexError, match="Target"):
            ops.ar_cross_entropy(logits, t)
    ops.ar_cross_entropy(logits, torch.zeros(2, 4, dtype=torch.int64, device=DEV))  # a fresh flag per call


def test_cross_entropy_rows_do_not_depend_on_the_batch():
    B, T, V = 16, 266, 256
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(B, T, V, generator=g) * 3).to(DEV)
    targets = torch.randint(0, V, (B, 265), generator=g).to(DEV)
    _, nll16 = ops.ar_cross_entropy(logits, targets, first_row=0)
    for b in (0, 7, 15):
        _, nll1 = ops.ar_cross_entropy(logits[b:b + 1].contiguous(), targets[b:b + 1].contiguous(), first_row=0)
        assert torch.equal(nll1[0], nll16[b])


# ---------------------------------------------------------------- prefill behind the drop-ins
def _model(name, seed):
    """A drop-in Net2NetTransformer (config `name`): reference init, then perturb_ (tests/test_gpu_ar.py's weights)."""
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS[name]), seed=seed, device="cpu")
    A.perturb_(m.transformer.state_dict(), seed)
    return m.to(DEV).eval()


def _feats(B, seed, Tc=1):
    f = torch.randn(B, 512, Tc, generator=torch.Generator().manual_seed(seed))
    return (f / f.norm(dim=1, keepdim=True)).to(DEV)


def _loss_bound(ref_logits):
    """A row's NLL moves by at most twice the largest logit error; logits are held to 3e-5 of their largest magnitude."""
    return 2 * 3e-5 * float(ref_logits.abs().max())


@pytest.mark.parametrize("name", list(AR_CONFIGS))
def test_prefill_logits_and_loss(name):
    c = AR_CONFIGS[name]
    m = _model(name, 1)
    tr = m.transformer
    B = 2
    g = torch.Generator().manual_seed(2)
    idx = torch.randint(0, c["V"], (B, 265), generator=g).to(DEV)
    feats = _feats(B, 3)
    targets = torch.randint(0, c["V"], (B, 266), generator=g)
    targets[0, :3] = -100
    targets = targets.to(DEV)
    logits, loss, att = GPT.forward(tr, idx, embeddings=tr.engine.embed_condition(feats), targets=targets)
    ref = A.forward(tr.state_dict(), idx, feats, n_layer=c["NL"], n_head=c["NH"])
    err = float((logits - ref).abs().max() / ref.abs().max())
    assert att is None and logits.shape == (B, 266, c["V"]) and err < 3e-5, err
    ref_loss = F.cross_entropy(ref.reshape(-1, c["V"]), targets.reshape(-1))
    assert abs(float(loss) - float(ref_loss)) < _loss_bound(ref), (float(loss), float(ref_loss))
    kv, _, _ = tr(idx, feats)  # the KV-cached teacher-forced forward
    kv_loss = F.cross_entropy(kv.reshape(-1, c["V"]), targets.reshape(-1))
    assert abs(float(loss) - float(kv_loss)) < _loss_bound(ref), (float(loss), float(kv_loss))
    again, loss2, _ = GPT.forward(tr, idx, embeddings=tr.engine.embed_condition(feats), targets=targets)  # graph replay
    assert torch.equal(again, logits) and torch.equal(loss2, loss)
    l1, _, _ = GPT.forward(tr, idx[1:], embeddings=tr.engine.embed_condition(feats[1:]), targets=targets[1:])
    assert float((l1 - logits[1:]).abs().max() / ref.abs().max()) < 3e-5


def _golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "ar_loss.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("case", ["v32_tc1", "v32_tc3", "v2048_tc1", "v2048_tc3", "full"])
def test_loss_vs_reference_fixture(case):
    """GPT.forward(idx, embeddings, targets) and shared_step's sliced loss against the unmodified reference (oracle/gen_golden_ar_loss.py)."""
    gd = _golden()
    V, Tc, seed, D, NL, NH, Cf = (int(v) for v in gd[case + "/meta"])
    fe, gc = A.gpt_config(V, D, NL, NH, Cf)
    torch.manual_seed(seed)
    tr = GPTFeats(fe, gc).eval()
    A.perturb_(tr.state_dict(), seed)
    tr = tr.to(DEV)
    z, feats = torch.from_numpy(gd[case + "/z"]).to(DEV), torch.from_numpy(gd[case + "/feats"]).to(DEV)
    ref_logits = A.forward(tr.state_dict(), z[:, :-1], feats, n_layer=NL, n_head=NH)
    bound = _loss_bound(ref_logits)
    _, gpt_loss, _ = GPT.forward(tr, z[:, :-1], embeddings=tr.engine.embed_condition(feats), targets=torch.from_numpy(gd[case + "/gpt_targets"]).to(DEV))
    assert abs(float(gpt_loss) - float(gd[case + "/gpt_loss"])) < bound, (float(gpt_loss), float(gd[case + "/gpt_loss"]))
    logits, step_loss, nll = tr.forward_loss(z[:, :-1], feats, z, Tc - 1)
    assert logits.shape == (z.shape[0], z.shape[1], V) and nll.shape == z.shape
    assert abs(float(step_loss) - float(gd[case + "/step_loss"])) < bound, (float(step_loss), float(gd[case + "/step_loss"]))
    if case == "full":
        ref = torch.from_numpy(gd["full/logits"]).to(DEV)[:, Tc - 1:]
        assert float((logits - ref).abs().max() / ref.abs().max()) < 3e-5


@pytest.mark.parametrize("name", list(AR_CONFIGS))
def test_shared_step_and_validation_step_vs_oracle(name):
    c = AR_CONFIGS[name]
    m = _model(name, 4)
    B = 2
    g = torch.Generator().manual_seed(5)
    mel = (torch.rand(B, 80, 848, generator=g) * 2 - 1).to(DEV)
    feature = _feats(B, 6).permute(0, 2, 1).contiguous()  # the dataset's (B, Tc, 512) layout
    batch = {"image": mel, "feature": feature}
    loss = m.shared_step(batch, 0)
    x, cfeat = m.get_xc(batch)
    assert x.shape == (B, 1, 80, 848) and cfeat.shape == (B, 512, 1)
    _, z = m.encode_to_z(x)
    ref_logits = A.forward(m.transformer.state_dict(), z[:, :-1], cfeat, n_layer=c["NL"], n_head=c["NH"])
    ref = F.cross_entropy(ref_logits[:, cfeat.size(-1) - 1:].reshape(-1, c["V"]), z.reshape(-1))
    assert loss.shape == () and abs(float(loss) - float(ref)) < _loss_bound(ref_logits), (float(loss), float(ref))
    assert torch.equal(m.validation_step(batch, 0), loss)


def test_prefill_out_of_range_token_raises():
    m = _model("caps_transformer_small", 7)
    tr = m.transformer
    idx = torch.zeros(1, 5, dtype=torch.long, device=DEV)
    idx[0, 2] = 999
    tg = torch.zeros(1, 6, dtype=torch.long, device=DEV)
    with pytest.raises(IndexError, match="tok_emb"):
        GPT.forward(tr, idx, embeddings=tr.engine.embed_condition(_feats(1, 8)), targets=tg)
    tg[0, 1] = 256
    with pytest.raises(IndexError, match="Target"):
        GPT.forward(tr, idx.clamp(max=10), embeddings=tr.engine.embed_condition(_feats(1, 8)), targets=tg)
    _, loss, _ = GPT.forward(tr, idx.clamp(max=10), embeddings=tr.engine.embed_condition(_feats(1, 8)), targets=tg.clamp(max=10))
    assert math.isfinite(float(loss))  # the flags were cleared


def test_ar_val_loss_scores_the_datasets_mel_input(tmp_path, monkeypatch):
    """tools/ar_val_loss.py's scoring path: [0, 1] log-mels from files, center-cropped and mapped to 2 * crop - 1 (caps.py VASSpecs), CLIP
    features of each caption, validation_step per batch (a ragged last batch), token-weighted.  Equal to shared_step on batches the test
    prepares itself from the same arrays."""
    from tests.test_cpu_ar_loss import _val_loss_inputs
    from tools import ar_val_loss as V
    from tools import generate_samples_ar as G
    cfg, mels, caps, mel = _val_loss_inputs(tmp_path, monkeypatch)
    model, text, tok, jobs = V.main(["--config", str(cfg), "--captions", str(caps), "--mels", str(mels), "--dry-run"])
    model, text = model.cuda().eval(), text.cuda()
    mean, count = V.score(model, text, tok, jobs, 2)
    imgs = [2 * torch.from_numpy(mel[:, 6:854]) - 1] * 2 + [2 * torch.from_numpy(mel[:, 3:851]) - 1]
    total = 0.0
    for i in (0, 2):
        chunk = jobs[i:i + 2]
        feats = G.caption_features(text, tok, [t for _, t in chunk])
        batch = {"image": torch.stack(imgs[i:i + 2]).to(DEV), "feature": feats.permute(0, 2, 1)}
        total += float(model.shared_step(batch, 0)) * len(chunk) * 265
    assert count == 3 * 265 and math.isfinite(mean)
    assert abs(mean - total / count) <= 1e-12 * abs(mean), (mean, total / count)
