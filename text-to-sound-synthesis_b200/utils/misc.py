"""{target, params} factory -- same contract as the reference's sound_synthesis/utils/misc.py:125-132."""
import importlib


def instantiate_from_config(config):
    if config is None:
        return None
    if "target" not in config:
        raise KeyError("Expected key `target` to instantiate.")
    module, cls = config["target"].rsplit(".", 1)
    cls = getattr(importlib.import_module(module, package=None), cls)
    return cls(**config.get("params", dict()))


# reference class path -> drop-in class path of this package (see INTEGRATION.md)
TARGET_MAP = {
    "sound_synthesis.modeling.transformers.diffusion_transformer.DiffusionTransformer":
        "diffsound_b200.modeling.transformers.diffusion_transformer.DiffusionTransformer",
    "sound_synthesis.modeling.transformers.transformer_utils.Text2ImageTransformer":
        "diffsound_b200.modeling.transformers.transformer_utils.Text2ImageTransformer",
    "sound_synthesis.modeling.embeddings.dalle_mask_image_embedding.DalleMaskImageEmbedding":
        "diffsound_b200.modeling.embeddings.dalle_mask_image_embedding.DalleMaskImageEmbedding",
    "sound_synthesis.modeling.codecs.spec_codec.vqgan.VQModel":
        "diffsound_b200.modeling.codecs.spec_codec.vqgan.VQModel",
    "sound_synthesis.modeling.models.dalle_spec.DALLE":
        "diffsound_b200.modeling.models.dalle_spec.DALLE",
    "specvqgan.modules.transformer.permuter.ColumnMajor":
        "diffsound_b200.modeling.codecs.spec_codec.vqgan.ColumnMajor",
    "sound_synthesis.modeling.codecs.text_codec.tokenize.Tokenize":
        "diffsound_b200.modeling.codecs.text_codec.tokenize.Tokenize",
    "sound_synthesis.modeling.modules.clip.simple_tokenizer.SimpleTokenizer":
        "diffsound_b200.modeling.modules.clip.simple_tokenizer.SimpleTokenizer",
    "sound_synthesis.modeling.embeddings.clip_text_embedding.CLIPTextEmbedding":
        "diffsound_b200.modeling.embeddings.clip_text_embedding.CLIPTextEmbedding",
    "sound_synthesis.engine.ema.EMA":
        "diffsound_b200.engine_utils.ema.EMA",
    # the autoregressive SpecVQGAN baseline (Codebook/configs/caps_transformer*.yaml)
    "specvqgan.models.cond_transformer.Net2NetTransformer":
        "diffsound_b200.modeling.models.cond_transformer.Net2NetTransformer",
    "specvqgan.modules.transformer.mingpt.GPTFeats":
        "diffsound_b200.modeling.transformers.mingpt.GPTFeats",
    "specvqgan.models.vqgan.VQModel":
        "diffsound_b200.modeling.codecs.spec_codec.vqgan.VQModel",
    "specvqgan.modules.misc.raw_feats.RawFeatsStage":
        "diffsound_b200.modeling.modules.raw_feats.RawFeatsStage",
    "specvqgan.modules.transformer.permuter.Identity":
        "diffsound_b200.modeling.codecs.spec_codec.vqgan.Identity",
}


def retarget_config(config):
    """Recursively rewrite reference `target:` strings of a loaded YAML config to this package's drop-in classes."""
    if isinstance(config, dict):
        out = {k: retarget_config(v) for k, v in config.items()}
        if isinstance(out.get("target"), str):
            out["target"] = TARGET_MAP.get(out["target"], out["target"])
        return out
    if isinstance(config, (list, tuple)):
        return type(config)(retarget_config(v) for v in config)
    return config
