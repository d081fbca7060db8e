"""Model builders shared by bench.py, __graft_entry__.smoke(), tools/ and the tests: reference-style `{target, params}` configs
(the layout of Diffsound/configs/caps.yaml:2-87) instantiated through this package's drop-in classes.  Weights are the modules'
own seeded random initialisation (the reference ships no Diffsound / SpecVQGAN checkpoint, SURVEY.md section 0 fact 7)."""
from __future__ import annotations

import os

import torch

from .misc import instantiate_from_config, retarget_config

DDCONFIG = dict(double_z=False, z_channels=256, resolution=848, in_channels=1, out_ch=1, ch=128, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=2,
                attn_resolutions=[53], dropout=0.0)  # Diffsound/configs/caps.yaml:13-23


def diffusion_config(K, D, NL, NH, CD, spatial=(5, 53), T=100, precision=None, train_precision=None):
    """`diffusion_config` block of caps.yaml (reference class paths; retarget_config maps them to the drop-ins)."""
    tp = dict(attn_type="selfcross", n_layer=NL, condition_seq_len=77, content_seq_len=spatial[0] * spatial[1], content_spatial_size=list(spatial),
              n_embd=D, condition_dim=CD, n_head=NH, attn_pdrop=0.0, resid_pdrop=0.0, block_activate="GELU2", timestep_type="adalayernorm",
              mlp_hidden_times=4)
    if precision is not None:
        tp["precision"] = precision
    if train_precision is not None:
        tp["train_precision"] = train_precision
    return {"target": "sound_synthesis.modeling.transformers.diffusion_transformer.DiffusionTransformer", "params": {
        "diffusion_step": T, "alpha_init_type": "alpha1", "auxiliary_loss_weight": 5.0e-4, "adaptive_auxiliary_loss": True, "mask_weight": [1, 1],
        "condition_emb_config": None,
        "transformer_config": {"target": "sound_synthesis.modeling.transformers.transformer_utils.Text2ImageTransformer", "params": tp},
        "content_emb_config": {"target": "sound_synthesis.modeling.embeddings.dalle_mask_image_embedding.DalleMaskImageEmbedding", "params": dict(
            num_embed=K, spatial_size=tuple(spatial), embed_dim=D, trainable=True, pos_emb_type="embedding")}}}


def dalle_config(K, D, NL, NH, CD, precision=None, train_precision=None, ddconfig=None):
    """`model` block of caps.yaml with synthetic-embedding conditioning (condition_codec_config None, the reference's own bypass)."""
    return {"target": "sound_synthesis.modeling.models.dalle_spec.DALLE", "params": {
        "content_info": {"key": "image"}, "condition_info": {"key": "text"},
        "content_codec_config": {"target": "sound_synthesis.modeling.codecs.spec_codec.vqgan.VQModel", "params": {
            "ckpt_path": None, "embed_dim": 256, "n_embed": K, "lossconfig": {"target": "specvqgan.modules.losses.DummyLoss"},
            "ddconfig": dict(ddconfig or DDCONFIG)}},
        "condition_codec_config": None,
        "first_stage_permuter_config": {"target": "specvqgan.modules.transformer.permuter.ColumnMajor", "params": {"H": 5, "W": 53}},
        "diffusion_config": diffusion_config(K, D, NL, NH, CD, precision=precision, train_precision=train_precision)}}


def build_diffusion_transformer(K, D, NL, NH, CD, sd=None, spatial=(5, 53), T=100, precision=None):
    """DiffusionTransformer drop-in on cuda:current, eval mode; `sd` (reference key names) is loaded with strict=False."""
    m = instantiate_from_config(retarget_config(diffusion_config(K, D, NL, NH, CD, spatial=spatial, T=T, precision=precision)))
    if sd is not None:
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected, unexpected
        assert all("attn2.mask" in k for k in missing), missing  # reference goldens drop the dead causal-mask buffers
    return m.cuda().eval()


# Diffsound/configs/ denoisers by (num_embed, n_embd, n_layer, n_head): caps_small_transformer.yaml differs from caps.yaml in n_layer, n_embd and
# the position embed_dim (= n_embd here), so its heads are 32 wide; build_dalle(**DALLE_CONFIGS[name]) builds one
DALLE_CONFIGS = {"caps": dict(K=256, D=1024, NL=19, NH=16), "caps_2048": dict(K=2048, D=1024, NL=19, NH=16),
                 "caps_small_transformer": dict(K=256, D=512, NL=18, NH=16)}


def build_dalle(K=256, D=1024, NL=19, NH=16, CD=512, precision=None, seed=0):
    """The full caps.yaml model (DALLE = SpecVQGAN codec + ColumnMajor + DiffusionTransformer), seeded random init, on the GPU."""
    torch.manual_seed(seed)
    return instantiate_from_config(retarget_config(dalle_config(K, D, NL, NH, CD, precision=precision))).cuda().eval()


def build_vocoder(ckpt=None):
    """MelGAN Generator(80, 32, 3) (vocoder/modules.py:88-130) with the reference's shipped weights when `ckpt` exists."""
    from ..vocoder.modules import Generator
    voc = Generator(80, 32, 3)
    if ckpt and os.path.exists(ckpt):
        voc.load_state_dict(torch.load(ckpt, map_location="cpu"), strict=True)
    return voc.cuda().eval()


# the three autoregressive-transformer configs of Codebook/configs/ (caps_transformer.yaml, caps_transformer_2048.yaml,
# caps_transformer_small.yaml): they differ only in vocab_size / n_layer / n_embd / n_head
AR_CONFIGS = {"caps_transformer": dict(V=256, NL=19, D=1024, NH=16), "caps_transformer_2048": dict(V=2048, NL=19, D=1024, NH=16),
              "caps_transformer_small": dict(V=256, NL=18, D=512, NH=16)}


def ar_transformer_config(V=256, NL=19, D=1024, NH=16, Cf=512, block_size=266, ddconfig=None):
    """`model` block of Codebook/configs/caps_transformer.yaml (reference class paths; retarget_config maps them to the drop-ins), without the
    codebook checkpoint path."""
    return {"target": "specvqgan.models.cond_transformer.Net2NetTransformer", "params": {
        "cond_stage_key": "feature",
        "transformer_config": {"target": "specvqgan.modules.transformer.mingpt.GPTFeats", "params": {
            "feat_embedding_config": {"target": "torch.nn.Conv1d", "params": dict(in_channels=Cf, out_channels=D, kernel_size=1, padding=0)},
            "GPT_config": dict(vocab_size=V, block_size=block_size, n_layer=NL, n_head=NH, n_embd=D)}},
        "first_stage_permuter_config": {"target": "specvqgan.modules.transformer.permuter.ColumnMajor", "params": {"H": 5, "W": 53}},
        "first_stage_config": {"target": "specvqgan.models.vqgan.VQModel", "params": {
            "ckpt_path": None, "embed_dim": 256, "n_embed": V, "ddconfig": dict(ddconfig or DDCONFIG),
            "lossconfig": {"target": "specvqgan.modules.losses.DummyLoss"}}},
        "cond_stage_config": {"target": "specvqgan.modules.misc.raw_feats.RawFeatsStage"}}}


def build_ar_transformer(config, seed=0, device="cuda"):
    """Net2NetTransformer drop-in from a reference-style `model` config (e.g. ar_transformer_config(**AR_CONFIGS[name])), seeded random init
    (the reference's own init order), eval mode, on `device`."""
    torch.manual_seed(seed)
    return instantiate_from_config(retarget_config(config)).to(device).eval()
