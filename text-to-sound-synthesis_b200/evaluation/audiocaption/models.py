"""ACT (Codebook/AudiocaptionLoss/models/TransModel.py) and its encoder AudioTransformer_80 (models/AudioTransformer.py) with the reference's
module tree, so state_dicts (ACTm.pth's 'model') load unchanged.  Inference only: the forward passes run on caption_engine.CaptionEngine; train
mode, SpecAugment and dropout are not implemented."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn as nn

from ...caption_engine import CaptionEngine
from ...engine_base import EngineModule

NUM_CLASSES, PATCH, EMBED_DIM, DEPTH, HEADS, MLP_DIM = 527, (4, 80), 768, 12, 12, 3072


def _refuse_training(module: nn.Module) -> None:
    if module.training:
        raise NotImplementedError(f"{type(module).__name__} runs inference only: call .eval() (training, dropout and SpecAugment are not implemented)")


class _PatchRows(nn.Module):
    """Rearrange('b c (h p1) (w p2) -> b (h w) (p1 p2 c)', p1=4, p2=80) of a (B, 1, T, 80) input: each clip's (T, 80) rows as (T / 4, 320)."""

    def forward(self, x):
        return x.reshape(x.shape[0], x.shape[2] // PATCH[0], PATCH[0] * PATCH[1])


class _Attention(nn.Module):
    def __init__(self, dim, heads, dim_head):
        super().__init__()
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.qkv = nn.Linear(dim, dim_head * heads * 3)
        self.proj = nn.Sequential(nn.Linear(dim_head * heads, dim), nn.Dropout(0.0))


class _FeedForward(nn.Module):
    def __init__(self, dim, hidden_dim):
        super().__init__()
        self.mlp = nn.Sequential(OrderedDict([("fc1", nn.Linear(dim, hidden_dim)), ("ac1", nn.GELU()), ("dropout1", nn.Dropout(0.0)),
                                              ("fc2", nn.Linear(hidden_dim, dim)), ("dropout2", nn.Dropout(0.0))]))


class _PreNorm(nn.Module):
    def __init__(self, dim, fn):
        super().__init__()
        self.norm = nn.LayerNorm(dim)
        self.fn = fn


class _Transformer(nn.Module):
    def __init__(self, dim, depth, heads, dim_head, mlp_dim):
        super().__init__()
        self.layers = nn.ModuleList([nn.ModuleList([_PreNorm(dim, _Attention(dim, heads, dim_head)), _PreNorm(dim, _FeedForward(dim, mlp_dim))])
                                     for _ in range(depth)])


class AudioTransformer_80(nn.Module):
    """The ViT encoder over (B, T, 80) log-mels: BatchNorm2d(80), 4 x 80 patches, cls token, 12 pre-norm blocks, mlp_head -> (B, T / 4 + 1, 527).
    Runs on the GPU through the owning ACT's engine (it is only ever used inside ACT)."""

    def __init__(self, patch_size=PATCH, num_classes=NUM_CLASSES, dim=EMBED_DIM, depth=DEPTH, heads=HEADS, mlp_dim=MLP_DIM, dim_head=64, dropout=0.):
        super().__init__()
        if tuple(patch_size) != PATCH or dim_head != 64 or dim != heads * dim_head:
            raise ValueError("AudioTransformer_80 runs the reference's (4, 80) patches with head_dim 64")
        self.bn0 = nn.BatchNorm2d(80)
        self.patch_embed = nn.Sequential(OrderedDict([("rerange", _PatchRows()), ("proj", nn.Linear(PATCH[0] * PATCH[1], dim))]))
        self.pos_embedding = nn.Parameter(torch.randn(1, 215 + 1, dim))
        self.cls_token = nn.Parameter(torch.randn(1, 1, dim))
        self.dropout = nn.Dropout(dropout)
        self.blocks = _Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.to_latent = nn.Identity()
        self.mlp_head = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, num_classes))


class PositionalEncoding(nn.Module):
    """The sinusoidal table pe (max_len, 1, d_model) of TransModel.py, built with the reference's fp32 arithmetic."""

    def __init__(self, d_model, dropout=0.1, max_len=2000):
        super().__init__()
        self.dropout = nn.Dropout(p=dropout)
        pe = torch.zeros(max_len, d_model)
        position = torch.arange(0, max_len, dtype=torch.float).unsqueeze(1)
        div_term = torch.exp(torch.arange(0, d_model, 2).float() * (-math.log(10000.0) / d_model))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        self.register_buffer("pe", pe.unsqueeze(0).transpose(0, 1))


def _cfg(config, *path):
    for k in path:
        config = config[k] if isinstance(config, dict) else getattr(config, k)
    return config


class ACT(EngineModule):
    """ACT(config, ntoken): the reference's constructor (config.encoder.pretrained loads config.path.encoder, config.word_embedding.pretrained
    needs gensim) and module tree; encode / decode / forward run on the GPU (the module must live on a CUDA device)."""

    def __init__(self, config, ntoken):
        super().__init__()
        self.ntoken = ntoken
        self.encoder = AudioTransformer_80(PATCH, NUM_CLASSES, EMBED_DIM, DEPTH, HEADS, MLP_DIM, dropout=0.2)
        if _cfg(config, "encoder", "pretrained"):
            pretrained = torch.load(_cfg(config, "path", "encoder"), map_location="cpu")["model"]
            if _cfg(config, "encoder", "model") == "deit":
                new = self.encoder.state_dict().copy()
                for k in [k for k in pretrained.keys() if not ("head" in k or "pos" in k)]:
                    new[k] = pretrained[k]
                self.encoder.load_state_dict(new)
            else:
                self.encoder.load_state_dict(pretrained)
        if _cfg(config, "encoder", "freeze"):
            for p in self.encoder.parameters():
                p.requires_grad = False
        nhead, nlayers = _cfg(config, "decoder", "nhead"), _cfg(config, "decoder", "nlayers")
        dim_feedforward, activation = _cfg(config, "decoder", "dim_feedforward"), _cfg(config, "decoder", "activation")
        dropout = _cfg(config, "decoder", "dropout")
        self.nhid = _cfg(config, "decoder", "nhid")
        if activation != "gelu":
            raise ValueError(f"decoder activation {activation!r} unsupported: the caption engine runs the reference's 'gelu'")
        self.encoder_linear = nn.Linear(NUM_CLASSES, self.nhid)
        self.pos_encoder = PositionalEncoding(self.nhid, dropout)
        layer = nn.TransformerDecoderLayer(self.nhid, nhead, dim_feedforward, dropout, activation)
        self.transformer_decoder = nn.TransformerDecoder(layer, nlayers)
        self.word_emb = nn.Embedding(ntoken, self.nhid)
        self.dec_fc = nn.Linear(self.nhid, ntoken)
        if _cfg(config, "word_embedding", "freeze"):
            self.word_emb.weight.requires_grad = False
        if _cfg(config, "word_embedding", "pretrained"):
            self.word_emb.weight.data = _align_word_embedding(_cfg(config, "path", "vocabulary"), _cfg(config, "path", "word2vec"), self.nhid)
        self.engine = CaptionEngine(self)

    def generate_square_subsequent_mask(self, sz):
        mask = (torch.triu(torch.ones(sz, sz)) == 1).transpose(0, 1)
        return mask.float().masked_fill(mask == 0, float("-inf")).masked_fill(mask == 1, float(0.0))

    @torch.no_grad()
    def encode(self, src):
        """src (B, T, n_mels=80) -> (T / 4 + 1, B, nhid) = relu(encoder_linear(encoder(src))).transpose(0, 1)."""
        _refuse_training(self)
        return self.engine.encode(src).transpose(0, 1)

    @torch.no_grad()
    def decode(self, encoded_feats, tgt, input_mask=None, target_mask=None, target_padding_mask=None):
        """encoded_feats (Lm, B, nhid), tgt (B, n) -> logits (n, B, ntoken) under the causal mask (the default target_mask)."""
        _refuse_training(self)
        if input_mask is not None or target_padding_mask is not None:
            raise NotImplementedError("ACT.decode runs without memory or padding masks, as the reference's decoders call it")
        if target_mask is not None and target_mask.size(0) == tgt.shape[1]:
            causal = self.generate_square_subsequent_mask(tgt.shape[1]).to(target_mask.device)
            if not torch.equal(target_mask, causal):
                raise NotImplementedError("ACT.decode runs the causal target mask only")
        return self.engine.decode(encoded_feats.transpose(0, 1), tgt)

    def forward(self, src, tgt, input_mask=None, target_mask=None, target_padding_mask=None):
        return self.decode(self.encode(src), tgt, input_mask=input_mask, target_mask=target_mask, target_padding_mask=target_padding_mask)


def _align_word_embedding(words_list_path, model_path, nhid):
    """tools/utils.py align_word_embedding: word2vec vectors of the vocabulary, in vocabulary order."""
    try:
        from gensim.models.word2vec import Word2Vec
    except ImportError as e:
        raise ImportError("config.word_embedding.pretrained needs gensim (gensim.models.word2vec.Word2Vec), which is not installed") from e
    import pickle

    import numpy as np
    with open(words_list_path, "rb") as f:
        words_list = pickle.load(f)
    w2v = Word2Vec.load(model_path)
    weights = np.zeros((len(words_list), nhid))
    for i, word in enumerate(words_list):
        weights[i] = w2v.wv[word]
    return torch.from_numpy(weights).float()
