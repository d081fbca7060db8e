"""Drop-in for sound_synthesis/modeling/embeddings/clip_text_embedding.py::CLIPTextEmbedding (SURVEY.md section 8f N2).

Same constructor arguments, state_dict keys (token_embedding.weight, positional_embedding, transformer.resblocks.N.{attn.in_proj_weight, ...},
ln_final.*, text_projection) and forward(index) contract; the transformer runs on the CUDA kernels of TextTowerEngine.  The reference downloads
OpenAI's CLIP weights in __init__ (clip.load) -- there is no network here, so the module is built with CLIP's initialisation and takes its
weights from `clip_ckpt_path` (a CLIP state_dict / TorchScript archive saved by the user) or a later load_state_dict(); the sub-modules only
hold parameters."""
from __future__ import annotations

import torch
from torch import nn

from ... import ops
from ...engine_base import EngineModule
from ...text_engine import TextTowerEngine

_TEXT_CONFIGS = {"ViT-B/32": dict(width=512, layers=12, heads=8, ctx=77, embed=512), "ViT-B/16": dict(width=512, layers=12, heads=8, ctx=77, embed=512)}


class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} only stores parameters; compute runs in TextTowerEngine (CUDA kernels)")


class _ResBlock(_Holder):
    def __init__(self, width, heads):
        super().__init__()
        self.attn = nn.MultiheadAttention(width, heads)   # parameter container: in_proj_weight / in_proj_bias / out_proj.*
        self.ln_1 = nn.LayerNorm(width)
        self.mlp = nn.Sequential()
        self.mlp.add_module("c_fc", nn.Linear(width, 4 * width))
        self.mlp.add_module("gelu", _Holder())
        self.mlp.add_module("c_proj", nn.Linear(4 * width, width))
        self.ln_2 = nn.LayerNorm(width)


class _Transformer(_Holder):
    def __init__(self, width, layers, heads):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(*[_ResBlock(width, heads) for _ in range(layers)])


class CLIPTextEmbedding(EngineModule):
    def __init__(self, clip_name="ViT-B/32", num_embed=49408, normalize=True, pick_last_embedding=True, keep_seq_len_dim=False,
                 additional_last_embedding=False, embed_dim=1024, clip_ckpt_path=None, text_layers=None):
        super().__init__()
        cfg = dict(_TEXT_CONFIGS[clip_name])
        if text_layers is not None:
            cfg["layers"] = text_layers
        self.num_embed, self.clip_name, self.normalize = num_embed, clip_name, normalize
        self.pick_last_embedding, self.keep_seq_len_dim, self.additional_last_embedding = pick_last_embedding, keep_seq_len_dim, additional_last_embedding
        W = cfg["width"]
        self.token_embedding = nn.Embedding(num_embed, W)
        self.positional_embedding = nn.Parameter(torch.empty(cfg["ctx"], W))
        self.transformer = _Transformer(W, cfg["layers"], cfg["heads"])
        self.ln_final = nn.LayerNorm(W)
        self.text_projection = nn.Parameter(torch.empty(W, cfg["embed"]))
        self._init(cfg)
        self.embed_dim = cfg["embed"] * 2 if embed_dim == 1024 else cfg["embed"]
        self.trainable = False
        for p in self.parameters():
            p.requires_grad = False
        self.eval()
        self.engine = TextTowerEngine(self)
        if clip_ckpt_path is not None:
            self.load_clip_checkpoint(clip_ckpt_path)

    def _init(self, cfg):  # CLIP.initialize_parameters (modules/clip/model.py:300-321)
        W, NL = cfg["width"], cfg["layers"]
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        proj_std, attn_std, fc_std = (W ** -0.5) * ((2 * NL) ** -0.5), W ** -0.5, (2 * W) ** -0.5
        for blk in self.transformer.resblocks:
            nn.init.normal_(blk.attn.in_proj_weight, std=attn_std)
            nn.init.normal_(blk.attn.out_proj.weight, std=proj_std)
            nn.init.normal_(blk.mlp.c_fc.weight, std=fc_std)
            nn.init.normal_(blk.mlp.c_proj.weight, std=proj_std)
        nn.init.normal_(self.text_projection, std=W ** -0.5)

    def load_clip_checkpoint(self, path):
        """A CLIP state_dict (torch.save(model.state_dict())) or OpenAI's TorchScript archive: only the text-side keys are used."""
        try:
            sd = torch.jit.load(path, map_location="cpu").state_dict()
        except RuntimeError:
            sd = torch.load(path, map_location="cpu")
            sd = sd.get("state_dict", sd)
        mine = self.state_dict()
        self.load_state_dict({k: v.float() for k, v in sd.items() if k in mine}, strict=True)

    def train(self, mode=True):  # BaseEmbedding.train: a frozen embedding stays in eval mode
        self.training = mode and self.trainable
        return self

    @property
    def dtype(self):
        return self.transformer.resblocks[0].attn.in_proj_weight.dtype

    @torch.no_grad()
    def encode_text(self, text):
        x = self.engine.forward(text, normalize=False)                       # ln_final output (B, L, W)
        if self.pick_last_embedding:
            idx = text.clamp(min=0).argmax(dim=-1)
            last = x[torch.arange(x.shape[0], device=x.device), idx].contiguous()
            x = ops.gemm_f32(last, self.text_projection.detach().float().t().contiguous())
            if self.keep_seq_len_dim:
                x = x.unsqueeze(1)
        return x

    @torch.no_grad()
    def forward(self, index, **kwargs):
        """index (B, L) int64 token ids -> (B, L, 512) per-token features (Diffsound: pick_last_embedding=False, embed_dim=512, normalize=True)."""
        assert index.dim() == 2
        feat = self.encode_text(index)
        out = torch.cat((feat, feat), dim=2) if self.embed_dim == 1024 and feat.dim() == 3 else feat
        if self.normalize:
            out = ops.l2_normalize_rows_(out.contiguous())
        if self.additional_last_embedding:
            idx = index.clamp(min=0).argmax(dim=-1)
            last = feat[torch.arange(feat.shape[0], device=feat.device), idx].contiguous()
            last = ops.gemm_f32(last, self.text_projection.detach().float().t().contiguous())
            return out, (last.unsqueeze(1) if self.keep_seq_len_dim else last)
        return out
