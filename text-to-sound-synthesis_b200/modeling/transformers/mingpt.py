"""Drop-in for Codebook/specvqgan/modules/transformer/mingpt.py (GPT, GPTFeats and their blocks): the autoregressive transformer that
Net2NetTransformer samples token by token.  Same constructor arguments, the same parameter / buffer names (a reference checkpoint's
state_dict loads unchanged, including blocks.N.attn.mask) and the same seeded initialisation order.

The modules hold the parameters; compute runs in `AREngine` (ar_engine.py): a KV-cached decode with CUDA kernels, teacher-forced or sampling,
and a full-sequence causal pass that scores given targets.  Attention maps are not materialised: forward() returns (logits, loss, None) where the
reference returns (logits, loss, att).  Only the forward is implemented: training (gradients), embedders other than Conv1d(kernel_size=1) and
n_unmasked > 0 are not.
"""
from __future__ import annotations

import copy

import torch
from torch import nn

from ... import ops
from ...ar_engine import AREngine, check_ar_shapes
from ...engine_base import EngineModule
from ...utils.misc import instantiate_from_config


class GPTConfig:
    """Same fields as mingpt.py:21-32."""
    embd_pdrop = 0.1
    resid_pdrop = 0.1
    attn_pdrop = 0.1

    def __init__(self, vocab_size, block_size, **kwargs):
        self.vocab_size = vocab_size
        self.block_size = block_size
        for k, v in kwargs.items():
            setattr(self, k, v)


class CausalSelfAttention(nn.Module):
    """Parameters of mingpt.py:53-94 (key / query / value / proj Linears and the causal mask buffer)."""

    def __init__(self, config):
        super().__init__()
        assert config.n_embd % config.n_head == 0
        self.key = nn.Linear(config.n_embd, config.n_embd)
        self.query = nn.Linear(config.n_embd, config.n_embd)
        self.value = nn.Linear(config.n_embd, config.n_embd)
        self.attn_drop = nn.Dropout(config.attn_pdrop)
        self.resid_drop = nn.Dropout(config.resid_pdrop)
        self.proj = nn.Linear(config.n_embd, config.n_embd)
        mask = torch.tril(torch.ones(config.block_size, config.block_size))
        if hasattr(config, "n_unmasked"):
            mask[:config.n_unmasked, :config.n_unmasked] = 1
        self.register_buffer("mask", mask.view(1, 1, config.block_size, config.block_size))
        self.n_head = config.n_head

    def forward(self, *a, **k):
        raise RuntimeError("CausalSelfAttention only stores parameters; compute runs in AREngine (CUDA kernels)")


class Block(nn.Module):
    """Pre-LN block of mingpt.py:111-138: ln1, attn, ln2, mlp = Linear(D, 4D) -> GELU (erf) -> Linear(4D, D) -> Dropout."""

    def __init__(self, config):
        super().__init__()
        self.ln1 = nn.LayerNorm(config.n_embd)
        self.ln2 = nn.LayerNorm(config.n_embd)
        self.attn = CausalSelfAttention(config)
        self.mlp = nn.Sequential(
            nn.Linear(config.n_embd, 4 * config.n_embd),
            nn.GELU(),
            nn.Linear(4 * config.n_embd, config.n_embd),
            nn.Dropout(config.resid_pdrop),
        )

    def forward(self, *a, **k):
        raise RuntimeError("Block only stores parameters; compute runs in AREngine (CUDA kernels)")


class GPT(EngineModule):
    """mingpt.py:141-187: tok_emb, pos_emb (1, block_size, D), blocks, ln_f, head (no bias)."""

    def __init__(self, vocab_size, block_size, n_layer=12, n_head=8, n_embd=256, embd_pdrop=0., resid_pdrop=0., attn_pdrop=0., n_unmasked=0):
        super().__init__()
        config = GPTConfig(vocab_size=vocab_size, block_size=block_size, embd_pdrop=embd_pdrop, resid_pdrop=resid_pdrop, attn_pdrop=attn_pdrop,
                           n_layer=n_layer, n_head=n_head, n_embd=n_embd, n_unmasked=n_unmasked)
        self.tok_emb = nn.Embedding(config.vocab_size, config.n_embd)
        self.pos_emb = nn.Parameter(torch.zeros(1, config.block_size, config.n_embd))
        self.drop = nn.Dropout(config.embd_pdrop)
        self.blocks = nn.Sequential(*[Block(config) for _ in range(config.n_layer)])
        self.ln_f = nn.LayerNorm(config.n_embd)
        self.head = nn.Linear(config.n_embd, config.vocab_size, bias=False)
        self.block_size = config.block_size
        self.apply(self._init_weights)
        self.config = config
        self.engine = AREngine(self)

    def get_block_size(self):
        return self.block_size

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def _check(self, n_pos: int) -> None:
        """Refusals, before anything is launched: kernel limits, then the reference's block-size assert (mingpt.py:170)."""
        c = self.config
        check_ar_shapes(c.vocab_size, c.n_embd, c.n_head, self.block_size)
        if getattr(c, "n_unmasked", 0):
            raise NotImplementedError("n_unmasked > 0 (a bidirectional prefix) is not implemented by the KV-cached decode")
        assert n_pos <= self.block_size, "Cannot forward, model block size is exhausted."
        if self.head.weight.device.type != "cuda":
            raise RuntimeError("the autoregressive transformer runs on CUDA only (no CPU fallback): move the module to a CUDA device")

    def _refuse_training(self, what):
        if self.training:
            raise NotImplementedError(f"{what} in training mode: only the forward (logits and loss) is implemented; training (gradients) is not. "
                                      "Call .eval() to score.")

    @torch.no_grad()
    def forward(self, idx, embeddings=None, targets=None):
        """Logits of every position (B, Tc + n, V) for idx (B, n) after `embeddings` (B, Tc, D).  Without targets: (logits, None, None) from the
        teacher-forced KV-cached decode (the logits sample() sees).  With targets (B, Tc + n) int64 (ignore_index -100): (logits, loss, None)
        from one causal pass, loss = F.cross_entropy(logits.view(-1, V), targets.view(-1)) (mingpt.py:183-185); eval mode only.  Attention maps
        are not materialised."""
        Tc = 0 if embeddings is None else embeddings.shape[1]
        n_pos = Tc + idx.shape[1]
        if targets is not None:
            self._refuse_training("GPT.forward with targets")
            if tuple(targets.shape) != (idx.shape[0], n_pos):
                raise ValueError(f"targets {tuple(targets.shape)} must be (B, T) = {(idx.shape[0], n_pos)}")
        self._check(n_pos)
        B = idx.shape[0]
        if embeddings is None:
            embeddings = torch.zeros(B, 0, self.config.n_embd, device=idx.device)
        if targets is not None:
            logits, loss, _ = self.engine.prefill(embeddings.float(), idx, targets, first_row=0)
            return logits, loss, None
        _, logits = self.engine.run(embeddings.float(), idx, n_pos, n_pos, record_logits=True)
        return logits, None, None


class GPTFeats(GPT):
    """mingpt.py:270-293: GPT with a feature embedder whose output (B, Tc, D) is prepended to the token embeddings.  Only
    Conv1d(kernel_size=1) embedders are implemented (the caps configs' Conv1d(512, n_embd, 1))."""

    def __init__(self, feat_embedding_config, GPT_config):
        super().__init__(**GPT_config)
        cfg = copy.deepcopy(dict(feat_embedding_config))
        if cfg["target"].split(".")[-1] in ["LSTM", "GRU"]:
            for p in ["in_channels", "out_channels", "padding", "kernel_size"]:
                cfg.get("params", {}).pop(p, None)
        self.embedder = instantiate_from_config(config=cfg)

    def _check_embedder(self):
        e = self.embedder
        if not (isinstance(e, nn.Conv1d) and tuple(e.kernel_size) == (1,) and tuple(e.stride) == (1,) and tuple(e.padding) == (0,)
                and tuple(e.dilation) == (1,) and e.groups == 1):
            raise NotImplementedError(f"GPTFeats embedder {type(e).__name__}: only Conv1d(kernel_size=1) is implemented")

    @torch.no_grad()
    def forward(self, idx, feats):
        """feats (B, Cf, Tc), idx (B, n) -> (logits (B, Tc + n, V), None, None), teacher-forced through the KV-cached decode."""
        self._check_embedder()
        self._check(feats.shape[-1] + idx.shape[1])
        return super().forward(idx, embeddings=self.engine.embed_condition(feats))

    @torch.no_grad()
    def forward_loss(self, idx, feats, targets, first_row):
        """Net2NetTransformer.shared_step's scoring in one causal pass: logits of GPTFeats.forward(idx (B, n), feats (B, Cf, Tc)) from row
        `first_row` on, and F.cross_entropy of those rows against targets (B, T - first_row) (cond_transformer.py:106, :359).  Returns (logits
        (B, T - first_row, V), loss (), per-row NLL (B, T - first_row))."""
        self._refuse_training("Net2NetTransformer.shared_step")
        self._check_embedder()
        T = feats.shape[-1] + idx.shape[1]
        if tuple(targets.shape) != (idx.shape[0], T - first_row):
            raise ValueError(f"targets {tuple(targets.shape)} must be (B, T - first_row) = {(idx.shape[0], T - first_row)}")
        self._check(T)
        logits, loss, nll = self.engine.prefill(self.engine.embed_condition(feats), idx, targets, first_row=first_row)
        return logits[:, first_row:], loss, nll

    @torch.no_grad()
    def sample_tokens(self, x, feats, steps, *, temperature=1.0, sample=False, top_k=None, callback=None, record_logits=False):
        """The decode loop of Net2NetTransformer.sample (cond_transformer.py:166-190): x (B, n0) given tokens, `steps` new ones.  Returns
        (ids (B, n0 + steps), logits history (B, Tc + n0 + steps - 1, V) or None)."""
        self._check_embedder()
        Tc = feats.shape[-1]
        n0 = x.shape[1]
        n_pos = Tc + n0 + steps - 1
        if Tc + n0 < 1:
            raise ValueError("sampling needs a condition or at least one given token")
        ops.check_ar_sampler_args(self.config.vocab_size, top_k, temperature)
        self._check(n_pos)
        cond = self.engine.embed_condition(feats)
        return self.engine.run(cond, x, n_pos, Tc + n0 - 1, temperature=temperature, top_k=top_k, sample=sample, record_logits=record_logits,
                               callback=callback)
