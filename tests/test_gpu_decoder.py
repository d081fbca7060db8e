"""SpecVQGAN decoder + MelGAN vocoder parity on the H100 (reference-generated goldens + the CPU oracle)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import diffsound_oracle as O  # noqa: E402
from tests.helpers import ROOT, load_golden, rel_err  # noqa: E402


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def build_vq(K, E, ch, ch_mult, sd=None, z_channels=None, prefix="content_codec.", precision="f16x3"):
    from diffsound_b200.modeling.codecs.spec_codec.vqgan import VQModel
    dd = dict(double_z=False, z_channels=z_channels or E, resolution=848, in_channels=1, out_ch=1, ch=ch, ch_mult=list(ch_mult), num_res_blocks=2,
              attn_resolutions=[53], dropout=0.0)
    m = VQModel(dd, None, n_embed=K, embed_dim=E, precision=precision)
    if sd is not None:
        missing, unexpected = m.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}, strict=False)
        assert not unexpected, unexpected
        # a golden carries either the decode side or the encode side of the codec; the other half keeps its random init
        halves = ("encoder.", "quant_conv.") if any(k.startswith(prefix + "decoder.") for k in sd) else ("decoder.", "post_quant_conv.")
        assert all(k.startswith(halves) for k in missing), missing
    return m.cuda().eval()


# f16x3 (the default) is held to 4x the 5.0e-6 measured on an H100, far inside its north-star 1e-3
_MEASURED_BOUND = {"f16x3": 2e-5}


@pytest.mark.parametrize("precision,tol", [("f16x3", 1e-3), ("tf32x3", 1e-3), ("tf32", 1.5e-2)])
def test_decoder_tiny_matches_reference_golden(G, precision, tol):
    """tol is the north-star tolerance (1e-3 relative) of the split modes; single-pass TF32 is the fast, looser mode."""
    sd, g = load_golden("decoder_tiny.npz")
    K, E, ch, H, W = [int(v) for v in g["__cfg"]]
    m = build_vq(K, E, ch, (1, 1, 1, 1, 2), sd, precision=precision)
    mel = m.decode_tokens(torch.from_numpy(g["in_ids"]).long().cuda(), (H, W)).cpu()
    ref = torch.from_numpy(g["out_mel"])
    assert mel.shape == ref.shape
    err = rel_err(mel, ref)
    print(f"decoder tiny [{precision}] rel err", err)
    assert err < min(tol, _MEASURED_BOUND.get(precision, tol))
    # the reference-shaped entry point (NCHW latents) agrees with the token fast path
    ids_rm = O.column_major_reverse(torch.from_numpy(g["in_ids"]).long(), H, W)
    z = O.codebook_lookup(sd, ids_rm, (ids_rm.shape[0], H, W, E))
    mel2 = m.decode(z.cuda()).cpu()
    assert rel_err(mel2, mel) < 1e-5


def test_decoder_full_config_matches_oracle(G):
    """The shipped ddconfig (ch=128, ch_mult 1,1,2,2,4, 256-d codebook) on the 5x53 grid, B=1: mel (1,1,80,848)."""
    sd = O.make_decoder_state_dict(seed=2)
    m = build_vq(256, 256, 128, (1, 1, 2, 2, 4), sd)
    ids = torch.randint(0, 256, (1, 265), generator=torch.Generator().manual_seed(9))
    ref = O.decode_to_img(sd, ids)
    mel = m.decode_tokens(ids.cuda(), (5, 53)).cpu()
    assert mel.shape == (1, 1, 80, 848)
    err = rel_err(mel, ref)
    mse = float(((mel - ref) ** 2).mean())
    print("decoder full [default precision] rel err", err, "mel MSE", mse, "ref rms", float(ref.pow(2).mean().sqrt()))
    assert err < 1.2e-4  # 4x the 3.1e-5 measured on an H100 in the default f16x3 mode; the north-star bound for the decoder is 1e-3


def test_melgan_tiny_matches_reference_golden(G):
    from diffsound_b200.vocoder.modules import Generator
    sd, g = load_golden("melgan_tiny.npz")
    m = Generator(80, 4, 3)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    wav = m(torch.from_numpy(g["in_mel"]).cuda()).cpu()
    ref = torch.from_numpy(g["out_wav"])
    assert wav.shape == ref.shape
    err = rel_err(wav, ref)
    print("melgan tiny [default precision] rel err", err)
    assert err < 1e-3


def test_melgan_real_checkpoint(G):
    """The reference's shipped generator weights (staged in oracle/_ref by build()): reference-generated I/O golden, then a
    full 848-frame clip against the oracle."""
    from diffsound_b200.vocoder.modules import Generator
    ck = os.path.join(ROOT, "oracle", "_ref", "best_netG.pt")
    if not os.path.exists(ck):
        pytest.skip("oracle/_ref/best_netG.pt not staged")
    sd = torch.load(ck, map_location="cpu")
    m = Generator(80, 32, 3)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    _, g = load_golden("melgan_real_io.npz")
    wav = m(torch.from_numpy(g["in_mel"]).cuda()).cpu()
    ref = torch.from_numpy(g["out_wav"])
    err = rel_err(wav, ref)
    print("melgan real (40 frames) [default precision] rel err", err)
    assert err < 1e-3
    mel = torch.rand(2, 80, 848, generator=torch.Generator().manual_seed(21))
    ref = O.melgan_forward(sd, mel)
    wav = m(mel.cuda()).cpu()
    assert wav.shape == (2, 1, 217088)
    err = rel_err(wav, ref)
    print("melgan real (848 frames, B=2) [default precision] rel err", err, "rms ref", float(ref.pow(2).mean().sqrt()))
    assert err < 1e-3


# ------------------------------------------------------------------------------------------------ encoder / tokeniser (N4)
def test_space_to_depth_and_row_argmin_kernels(G):
    B, H, W, C = 2, 6, 10, 8
    g = torch.Generator().manual_seed(0)
    img = torch.randn(B, H, W, C, generator=g)
    xp = torch.nn.functional.pad(img, (0, 0, 1, 1, 1, 1)).cuda()
    out = G.ops.space_to_depth_padded(xp).cpu()
    assert out.shape == (B, H // 2 + 2, W // 2 + 2, 4 * C)
    padded = torch.nn.functional.pad(img, (0, 0, 0, 2, 0, 2))            # zero right / bottom, as Downsample's F.pad (+1 spare)
    for p in range(2):
        for q in range(2):
            ref = padded[:, p::2, q::2, :][:, :H // 2 + 1, :W // 2 + 1, :]
            assert torch.equal(out[:, 1:, 1:, (2 * p + q) * C:(2 * p + q + 1) * C], ref), (p, q)
    assert float(out[:, 0].abs().max()) == 0.0 and float(out[:, :, 0].abs().max()) == 0.0
    sp = G.ops.space_to_depth_padded(xp, split=True).cpu()
    assert torch.equal(sp[..., :4 * C], G.tf32_round_ref(out)) and float((sp[..., :4 * C] + sp[..., 4 * C:] - out).abs().max()) < 1e-6
    x = torch.randn(300, 40, generator=g)
    x[5, 7] = x[5, 3] = x[5].min() - 1.0                                 # a tie: the first index wins
    ids = G.ops.row_argmin(x.cuda()[:, :33], 33).cpu()
    assert torch.equal(ids, x[:, :33].argmin(1)) and int(ids[5]) == 3


def test_encoder_tokeniser_matches_reference_golden(G):
    """DALLE.get_tokens' compute (encoder + quant_conv + nearest code + ColumnMajor) vs the unmodified reference (tests/golden/encoder_tiny.npz)."""
    sd, g = load_golden("encoder_tiny.npz")
    K, E, ch, H, W = [int(v) for v in g["__cfg"]]
    m = build_vq(K, E, ch, (1, 1, 1, 1, 2), sd)
    quant, _, info = m.encode(torch.from_numpy(g["in_mel"]).cuda())
    ref_z = torch.from_numpy(g["out_z"])
    e_z = rel_err(m.last_latent.cpu(), ref_z)
    ids = info[2].view(-1, H * W).cpu()
    col_major = torch.arange(H * W).reshape(H, W).t().reshape(-1)
    ref_tok = torch.from_numpy(g["out_tokens"]).long()
    print("encoder tiny: z rel err", e_z, "token mismatches", int((ids[:, col_major] != ref_tok).sum()))
    assert e_z < 1e-3
    assert torch.equal(ids[:, col_major], ref_tok)
    assert torch.allclose(quant.cpu(), torch.from_numpy(g["out_quant"]), rtol=1e-5, atol=1e-6)  # z_q = the chosen codebook rows (the reference returns z + (z_q - z))


def test_encoder_full_config_matches_oracle(G):
    """Real ddconfig (80 x 848 mel, ch 128, ch_mult 1-1-2-2-4, attention at 5 x 53), random init: latents within 1e-3, >= 99 % of the 265 codes equal."""
    import _pkg
    _pkg.load()
    from diffsound_b200.modeling.models.dalle_spec import DALLE  # noqa: F401  (import check of the training-side entry)
    torch.manual_seed(5)
    m = build_vq(256, 256, 128, (1, 1, 2, 2, 4))
    g = torch.Generator().manual_seed(6)
    mel = torch.rand(1, 1, 80, 848, generator=g) * 2 - 1
    sd = {"content_codec." + k: v.detach().cpu() for k, v in m.state_dict().items()}
    z_ref = O._conv(sd, "content_codec.quant_conv.", O.encoder_forward(sd, mel), 0)
    zf = z_ref.permute(0, 2, 3, 1).reshape(-1, 256)
    cb = zf.mean(0, keepdim=True) + torch.randn(256, 256, generator=g) * zf.std(0, keepdim=True)   # codes with the latents' statistics
    sd["content_codec.quantize.embedding.weight"] = cb
    m.quantize.embedding.weight.data.copy_(cb.cuda())
    m.enc_engine.repack()
    _, tok_ref = O.encode_to_tokens(sd, mel)
    quant, _, info = m.encode(mel.cuda())
    e_z = rel_err(m.last_latent.cpu(), z_ref)
    ids = info[2].view(1, 265).cpu()
    col_major = torch.arange(265).reshape(5, 53).t().reshape(-1)
    agree = float((ids[:, col_major] == tok_ref).float().mean())
    print("encoder full: z rel err", e_z, "token agreement", agree, "launches", m.enc_engine.launches)
    assert quant.shape == (1, 256, 5, 53) and e_z < 1e-3 and agree >= 0.99
