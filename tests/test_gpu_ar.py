"""The autoregressive SpecVQGAN transformer's decode kernels and drop-ins on the GPU (ar_decode.cu, ar_engine.py, mingpt.py / cond_transformer.py):
the exponential replay bit for bit against torch, the sampler step against a restatement and against torch.multinomial under the same generator
state, decode attention and GELU against fp64, teacher-forced logits and free-running ids against the fp32 oracle."""
import math

import numpy as np
import pytest
import torch

import _pkg

_pkg.load()
from diffsound_b200 import ops  # noqa: E402
from diffsound_b200.utils.builders import AR_CONFIGS, ar_transformer_config, build_ar_transformer  # noqa: E402
from oracle import ar_oracle as A  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _fp32_oracle():
    """The oracle runs in fp32 on the GPU here: no TF32 in its matmuls or its Conv1d."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _gen():
    torch.cuda.init()  # the default generators exist once CUDA is initialised
    return torch.cuda.default_generators[torch.cuda.current_device()]


def _ctrl(B, V, p=0, n_pos=1, first=0):
    gen = _gen()
    nthreads, inc = ops.aten_rand_geometry(B * V)
    seed = gen.initial_seed()
    s = np.array([seed & (2 ** 64 - 1)], dtype=np.uint64).view(np.int64)[0].item()
    return torch.tensor([s, gen.get_offset(), inc, nthreads, p, n_pos, first, 0], dtype=torch.int64, device=DEV)


@pytest.mark.parametrize("numel", [256, 16 * 256, 96 * 256, 96 * 2048, 4096])
def test_aten_exponential_bitwise(numel):
    for seed, skip in ((0, 0), (123, 1), (2 ** 40 + 7, 3)):
        torch.cuda.manual_seed(seed)
        for _ in range(skip):
            torch.empty(1000, device=DEV).exponential_()
        s, off = _gen().initial_seed(), _gen().get_offset()
        ref = torch.empty(numel, device=DEV).exponential_()
        mine = ops.aten_exponential(numel, s, off)
        assert torch.equal(mine, ref), (numel, seed, skip)


def _restate_probs(logits, temperature, top_k):
    """The reference's step on the CPU (true fp32 division by the temperature, as the kernel does)."""
    return A.step_probs(logits.cpu(), temperature, top_k).to(DEV)


@pytest.mark.parametrize("V", [1, 255, 256, 2048, 4096])
@pytest.mark.parametrize("temperature", [1.0, 0.7])
@pytest.mark.parametrize("top_k", [None, 1, 100, "V-1", "V"])
@pytest.mark.parametrize("integer", [False, True])
def test_sampler_step(V, temperature, top_k, integer):
    k = {"V-1": V - 1, "V": V}.get(top_k, top_k)
    if k is not None and not 1 <= k <= V:
        pytest.skip("top_k outside 1 ... V")
    B = 16
    g = torch.Generator().manual_seed(V * 7 + (k or 0))
    logits = (torch.randint(-3, 4, (B, V), generator=g).float() if integer else torch.randn(B, V, generator=g) * 3).to(DEV)
    ref = _restate_probs(logits, temperature, k)
    for do_sample in (False, True):
        torch.cuda.manual_seed(V + 11)
        off0 = _gen().get_offset()
        ctrl = _ctrl(B, V)
        ids = torch.full((B, 2), -1, dtype=torch.int64, device=DEV)
        probs = torch.empty(B, V, device=DEV)
        ops.ar_sample(logits, ids, ctrl, Tc=1, temperature=temperature, top_k=k, sample=do_sample, probs_out=probs)
        assert torch.equal(probs == 0, ref == 0)  # the same kept set (ties at the k-th value kept)
        assert torch.allclose(probs, ref, rtol=1e-5, atol=1e-9), float((probs - ref).abs().max())
        assert int(ctrl[4]) == 1
        if do_sample:
            _gen().set_offset(off0)
            want = torch.multinomial(probs, 1)
            assert int(ctrl[1]) == _gen().get_offset()
        else:
            want = torch.argmax(probs, dim=-1, keepdim=True)
            assert int(ctrl[1]) == off0
        assert torch.equal(ids[:, :1], want), (do_sample, (ids[:, :1] != want).sum())
        assert bool((ids[:, 1] == -1).all())


def test_sampler_nan_sets_flag():
    B, V = 2, 64
    logits = torch.randn(B, V, device=DEV)
    logits[1, 5] = float("nan")
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    ops.ar_sample(logits, torch.zeros(B, 2, dtype=torch.int64, device=DEV), _ctrl(B, V), Tc=1, err_flag=err)
    assert int(err) == 1


@pytest.mark.parametrize("hd", [32, 64])
@pytest.mark.parametrize("B", [1, 3, 96])
def test_decode_attention_vs_fp64(hd, B):
    H, P = 4 if B == 96 else 16, 266
    D = H * hd
    g = torch.Generator().manual_seed(hd + B)
    for Lk in ((1, 2, 63, 64, 65, 129, 200, 255, 256, 257, 266) if B != 96 else (1, 133, 266)):
        kc = (torch.randn(B, P, D, generator=g) * 2).to(DEV)
        vc = torch.randn(B, P, D, generator=g).to(DEV)
        qkv = (torch.randn(B, 3 * D, generator=g) * 2).to(DEV)
        kc0, vc0 = kc.clone(), vc.clone()
        out = torch.zeros(B, 2 * D, dtype=torch.float16, device=DEV)
        ctrl = _ctrl(B, 1, p=Lk - 1, n_pos=P)
        ops.ar_attention(qkv, kc, vc, out, ctrl, H=H, scale=1.0 / math.sqrt(hd))
        p = Lk - 1
        assert torch.equal(kc[:, p], qkv[:, D:2 * D]) and torch.equal(vc[:, p], qkv[:, 2 * D:])  # bit-exact cache rows
        keep = torch.ones(P, dtype=torch.bool)
        keep[p] = False
        assert torch.equal(kc[:, keep], kc0[:, keep]) and torch.equal(vc[:, keep], vc0[:, keep])
        q = qkv[:, :D].double().view(B, H, hd)
        K = kc[:, :Lk].double().view(B, Lk, H, hd).permute(0, 2, 1, 3)
        Vv = vc[:, :Lk].double().view(B, Lk, H, hd).permute(0, 2, 1, 3)
        s = torch.einsum("bhd,bhjd->bhj", q, K) / math.sqrt(hd)
        ref = torch.einsum("bhj,bhjd->bhd", torch.softmax(s, -1), Vv).reshape(B, D)
        o = out[:, :D].double() + out[:, D:].double()
        err = float((o - ref).abs().max() / ref.abs().max())
        assert err < 3e-6, (Lk, err)


def test_gelu_erf_split_vs_fp64():
    x = torch.linspace(-60, 60, 1 << 20, dtype=torch.float32, device=DEV).view(1024, 1024)
    out = ops.gelu_erf_split(x)
    y = out[:, :1024].double() + out[:, 1024:].double()
    xd = x.double()
    ref = xd * 0.5 * (1.0 + torch.special.erf(xd / math.sqrt(2.0)))
    # the fp16 (hi | lo) pair holds 22 significant bits (2^-22 relative), fp16's subnormal step bounds tiny values, erff is within 2 ulp of
    # erf and enters scaled by |x| / 2, and the fp32 output rounds to half an ulp
    bound = 2.0 ** -22 * ref.abs() + 2.0 ** -24 * ref.abs() + 2 * 2.0 ** -24 * 0.5 * xd.abs() + 2.0 ** -24
    assert bool(((y - ref).abs() <= bound).all()), float(((y - ref).abs() - bound).max())


def _model(name, seed):
    """A drop-in Net2NetTransformer (config `name`) whose transformer carries the fixtures' weights: reference init, then perturb_."""
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS[name]), seed=seed, device="cpu")
    A.perturb_(m.transformer.state_dict(), seed)
    return m.to(DEV).eval()


def _feats(B, seed, Tc=1):
    f = torch.randn(B, 512, Tc, generator=torch.Generator().manual_seed(seed))
    return (f / f.norm(dim=1, keepdim=True)).to(DEV)


@pytest.mark.parametrize("name", list(AR_CONFIGS))
def test_teacher_forced_logits_vs_oracle(name):
    m = _model(name, 1)
    c = AR_CONFIGS[name]
    B = 2
    idx = torch.randint(0, c["V"], (B, 265), generator=torch.Generator().manual_seed(2)).to(DEV)
    feats = _feats(B, 3)
    logits, _, _ = m.transformer(idx, feats)
    ref = A.forward(m.transformer.state_dict(), idx, feats, n_layer=c["NL"], n_head=c["NH"])
    err = float((logits - ref).abs().max() / ref.abs().max())
    assert logits.shape == (B, 266, c["V"]) and err < 3e-5, err


def test_batch_invariance_loop_consistency_and_graph_replay():
    m = _model("caps_transformer_small", 4)
    tr = m.transformer
    V = AR_CONFIGS["caps_transformer_small"]["V"]
    feats = _feats(16, 5)
    idx = torch.randint(0, V, (16, 60), generator=torch.Generator().manual_seed(6)).to(DEV)
    l16, _, _ = tr(idx, feats)
    l1, _, _ = tr(idx[3:4], feats[3:4])
    assert torch.equal(l16[3:4], l1)  # a row's logits do not depend on the batch
    torch.cuda.manual_seed(7)
    ids, seen = tr.sample_tokens(idx[:, :0], feats, 40, sample=True, top_k=100, record_logits=True)
    lf, _, _ = tr(ids[:, :-1], feats)
    assert torch.equal(lf, seen)  # forward() sees exactly the logits sample() saw at every step
    tr.engine.use_cuda_graph = False
    torch.cuda.manual_seed(7)
    ids_eager, seen_eager = tr.sample_tokens(idx[:, :0], feats, 40, sample=True, top_k=100, record_logits=True)
    tr.engine.use_cuda_graph = True
    assert torch.equal(ids, ids_eager) and torch.equal(seen, seen_eager)


@pytest.mark.parametrize("name,mode,steps", [("caps_transformer", "nopix", 265), ("caps_transformer", "half", 133),
                                             ("caps_transformer_2048", "nopix", 40), ("caps_transformer_small", "nopix", 48)])
def test_free_running_sample_vs_oracle_same_q(name, mode, steps):
    c = AR_CONFIGS[name]
    m = _model(name, 8)
    B = 2
    feats = _feats(B, 9)
    gt = torch.randint(0, c["V"], (B, 265), generator=torch.Generator().manual_seed(10)).to(DEV)
    x0 = gt[:, :0] if mode == "nopix" else gt[:, :265 - steps]
    torch.cuda.manual_seed(11)
    calls = []
    out, att = m.sample(x0, feats, steps, temperature=1.0, sample=True, top_k=100, callback=calls.append)
    off_after = _gen().get_offset()
    assert att is None and calls == list(range(steps)) and out.shape == (B, x0.shape[1] + steps)
    assert torch.equal(out[:, :x0.shape[1]], x0)  # prefix untouched
    torch.cuda.manual_seed(11)
    q = [torch.empty(B, c["V"], device=DEV).exponential_() for _ in range(steps)]
    assert _gen().get_offset() == off_after
    sd = {k: v for k, v in m.transformer.state_dict().items()}
    ref = A.sample(sd, x0, feats, steps, n_layer=c["NL"], n_head=c["NH"], sample=True, top_k=100, q_fn=lambda k: q[k])
    bad = int((ref != out).sum())
    assert bad == 0, f"{bad} ids differ from the oracle"


def test_greedy_sample_and_decode_to_img():
    m = _model("caps_transformer", 12)
    feats = _feats(2, 13)
    out, _ = m.sample(torch.zeros(2, 0, dtype=torch.long, device=DEV), feats, 265, sample=False, top_k=None)
    ref = A.sample(m.transformer.state_dict(), out[:, :0], feats, 8, n_layer=19, n_head=16, sample=False)
    assert torch.equal(out[:, :8], ref)
    mel = m.decode_to_img(out, (2, 256, 5, 53))
    assert mel.shape == (2, 1, 80, 848) and bool(torch.isfinite(mel).all())


def test_out_of_range_token_raises():
    m = _model("caps_transformer_small", 14)
    idx = torch.zeros(1, 5, dtype=torch.long, device=DEV)
    idx[0, 2] = 999
    with pytest.raises(IndexError):
        m.transformer(idx, _feats(1, 15))
    m.transformer(idx.clamp(max=10), _feats(1, 15))  # the flag was cleared


def test_decode_attention_past_the_cache_writes_nothing():
    """A control block armed past max_pos (the cache capacity the caller declares) is a no-op: nothing is written, here into rows that do exist."""
    from diffsound_b200 import _lib
    B, H, hd, P = 2, 4, 64, 266
    D = H * hd
    kc, vc = torch.randn(B, P, D, device=DEV), torch.randn(B, P, D, device=DEV)
    kc0, vc0 = kc.clone(), vc.clone()
    qkv = torch.randn(B, 3 * D, device=DEV)
    out = torch.full((B, 2 * D), 7.0, dtype=torch.float16, device=DEV)
    max_pos = 10
    ctrl = _ctrl(B, 1, p=max_pos, n_pos=P)
    _lib.check(_lib.lib().dsb_ar_attention(qkv.data_ptr(), qkv.stride(0), kc.data_ptr(), vc.data_ptr(), P * D, max_pos, out.data_ptr(), out.stride(0), D,
                                           ctrl.data_ptr(), B, H, hd, 0.125, ops._stream()), "dsb_ar_attention")
    torch.cuda.synchronize()
    assert torch.equal(kc, kc0) and torch.equal(vc, vc0) and bool((out == 7.0).all())


def test_unconditioned_forward_after_an_index_error():
    """GPT.forward without embeddings (no condition rows: position 0 is a token) right after a call that raised IndexError: the step captured
    for it embeds the new tokens, not the rejected ones still in the workspace."""
    from diffsound_b200.modeling.transformers.mingpt import GPT
    m = _model("caps_transformer_small", 19)
    tr = m.transformer
    bad = torch.zeros(1, 4, dtype=torch.long, device=DEV)
    bad[0, 0] = 999
    with pytest.raises(IndexError):
        tr(bad, _feats(1, 20))
    idx = torch.randint(0, 256, (1, 6), generator=torch.Generator().manual_seed(21)).to(DEV)
    logits, _, _ = GPT.forward(tr, idx)
    assert logits.shape == (1, 6, 256) and bool(torch.isfinite(logits).all())


def test_caption_to_wav_through_generate_samples_ar(tmp_path):
    """captions -> CLIP pooled feature -> Net2NetTransformer.sample -> decode_to_img -> MelGAN -> save_clip, through tools/generate_samples_ar.py's
    functions.  Every token equals the oracle's fed the same exponential draws; the mel is within the decoder's full-config bound of the oracle
    decode of those tokens (1.2e-4, tests/test_gpu_decoder.py); the waveform is finite."""
    import os
    from diffsound_b200 import pipeline
    from diffsound_b200.modeling.embeddings.clip_text_embedding import CLIPTextEmbedding
    from diffsound_b200.modeling.modules.clip.simple_tokenizer import SimpleTokenizer
    from diffsound_b200.utils.builders import build_vocoder
    from oracle import diffsound_oracle as O
    from tests.helpers import ROOT, bpe_vocab_file, rel_err
    from tools import generate_samples_ar as G
    m = _model("caps_transformer", 16)
    dec = O.make_decoder_state_dict(seed=2)
    _, unexpected = m.first_stage_model.load_state_dict({k[len("content_codec."):]: v for k, v in dec.items()}, strict=False)
    assert not unexpected
    torch.manual_seed(17)
    text = CLIPTextEmbedding(pick_last_embedding=True, normalize=False).cuda()
    feats = G.caption_features(text, SimpleTokenizer(bpe_path=bpe_vocab_file(tmp_path)), ["a dog barks in the distance", "rain falls on a tin roof"])
    assert feats.shape == (2, 512, 1) and bool(torch.isfinite(feats).all())
    voc = build_vocoder(os.path.join(ROOT, "oracle", "_ref", "best_netG.pt"))
    torch.cuda.manual_seed(18)
    out = G.synthesize(m, voc, feats, top_k=100)
    ids, mel, wav = out["tokens"], out["mel"], out["wav"]
    torch.cuda.manual_seed(18)
    q = [torch.empty(2, 256, device=DEV).exponential_() for _ in range(265)]
    ref_ids = A.sample(m.transformer.state_dict(), ids[:, :0], feats, 265, n_layer=19, n_head=16, sample=True, top_k=100, q_fn=lambda k: q[k])
    assert torch.equal(ids, ref_ids), int((ids != ref_ids).sum())
    ref_mel = O.decode_to_img(dec, ids.cpu())
    err = rel_err(mel.cpu(), ref_mel)
    assert mel.shape == (2, 1, 80, 848) and err < 1.2e-4, err
    assert wav.shape[0] == 2 and wav.shape[-1] > 0 and bool(torch.isfinite(wav).all())
    stem = pipeline.save_clip(str(tmp_path / "out"), "Y1", 0, mel[0], wav[0])
    assert os.path.getsize(stem + ".wav") > 0 and os.path.exists(stem + ".npy")
