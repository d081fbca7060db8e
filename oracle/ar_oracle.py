"""CPU fp32 restatement of the autoregressive SpecVQGAN transformer (Codebook/specvqgan/modules/transformer/mingpt.py GPTFeats.forward) and of
Net2NetTransformer.sample's loop (Codebook/specvqgan/models/cond_transformer.py:124-194) -- test infrastructure.

forward() recomputes the whole prefix, as the reference does, from a state_dict with the reference's key names, with the same torch ops in the
same order (so CPU results agree with the reference bit for bit in practice).  sample() runs the reference loop; the multinomial draw either is
torch.multinomial itself (CPU generator) or takes q from the caller, argmax(probs / q) per row -- the formula of torch.multinomial's
one-sample path -- so a test can feed the oracle the exact draws the CUDA generator made.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch
import torch.nn.functional as F


def forward(sd: dict, idx: torch.Tensor, feats: torch.Tensor, *, n_layer: int, n_head: int, prefix: str = "") -> torch.Tensor:
    """GPTFeats.forward(idx (B, n), feats (B, Cf, Tc)) -> logits (B, Tc + n, V), fp32, full-prefix recompute."""
    g = lambda k: sd[prefix + k].float()
    c = F.conv1d(feats.float(), g("embedder.weight"), g("embedder.bias")).permute(0, 2, 1)
    x = torch.cat((c, F.embedding(idx, g("tok_emb.weight"))), dim=1)
    T = x.shape[1]
    x = x + g("pos_emb")[:, :T, :]
    B, _, C = x.shape
    hd = C // n_head
    mask = torch.tril(torch.ones(T, T, device=x.device))
    for i in range(n_layer):
        b = f"blocks.{i}."
        h = F.layer_norm(x, (C,), g(b + "ln1.weight"), g(b + "ln1.bias"))
        k = F.linear(h, g(b + "attn.key.weight"), g(b + "attn.key.bias")).view(B, T, n_head, hd).transpose(1, 2)
        q = F.linear(h, g(b + "attn.query.weight"), g(b + "attn.query.bias")).view(B, T, n_head, hd).transpose(1, 2)
        v = F.linear(h, g(b + "attn.value.weight"), g(b + "attn.value.bias")).view(B, T, n_head, hd).transpose(1, 2)
        att = (q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(k.size(-1)))
        att = att.masked_fill(mask == 0, float("-inf"))
        att = F.softmax(att, dim=-1)
        y = (att @ v).transpose(1, 2).contiguous().view(B, T, C)
        x = x + F.linear(y, g(b + "attn.proj.weight"), g(b + "attn.proj.bias"))
        h = F.layer_norm(x, (C,), g(b + "ln2.weight"), g(b + "ln2.bias"))
        h = F.linear(F.gelu(F.linear(h, g(b + "mlp.0.weight"), g(b + "mlp.0.bias"))), g(b + "mlp.2.weight"), g(b + "mlp.2.bias"))
        x = x + h
    x = F.layer_norm(x, (C,), g("ln_f.weight"), g("ln_f.bias"))
    return F.linear(x, g("head.weight"))


def top_k_logits(logits: torch.Tensor, k: int) -> torch.Tensor:
    v, _ = torch.topk(logits, k)
    out = logits.clone()
    out[out < v[..., [-1]]] = -float("Inf")
    return out


def step_probs(logits_last: torch.Tensor, temperature: float, top_k: Optional[int]) -> torch.Tensor:
    """cond_transformer.py:171-177: probs (B, V) from the last position's logits."""
    logits = logits_last / temperature
    if top_k is not None:
        logits = top_k_logits(logits, top_k)
    return F.softmax(logits, dim=-1)


def pick(probs: torch.Tensor, sample: bool, q: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(B, 1) ids: torch.multinomial(probs, 1) (CPU generator) or, with q given, argmax(probs / q) (its one-sample formula); greedy: argmax."""
    if not sample:
        return torch.topk(probs, k=1, dim=-1)[1]
    if q is None:
        return torch.multinomial(probs, num_samples=1)
    return torch.argmax(probs / q, dim=-1, keepdim=True)


def sample(sd: dict, x: torch.Tensor, feats: torch.Tensor, steps: int, *, n_layer: int, n_head: int, temperature: float = 1.0, sample: bool = False,
           top_k: Optional[int] = None, q_fn: Optional[Callable[[int], torch.Tensor]] = None, prefix: str = "", return_logits: bool = False):
    """Net2NetTransformer.sample for GPTFeats: x (B, n0) -> (B, n0 + steps).  q_fn(k) -> (B, V) exponential draws of step k (None: multinomial)."""
    seen = []
    for k in range(steps):
        logits = forward(sd, x, feats, n_layer=n_layer, n_head=n_head, prefix=prefix)[:, -1, :]
        seen.append(logits)
        probs = step_probs(logits, temperature, top_k)
        ix = pick(probs, sample, None if q_fn is None else q_fn(k))
        x = torch.cat((x, ix), dim=1)
    return (x, torch.stack(seen, 1)) if return_logits else x


def make_state_dict(*, V: int, D: int, n_layer: int, n_head: int, Cf: int, block_size: int = 266, seed: int = 0, scale: float = 1.0) -> dict:
    """Seeded GPTFeats state_dict (reference key names, no `transformer.` prefix) with non-trivial pos_emb and LayerNorm affines: Linear
    weights N(0, 0.02 * scale), biases N(0, 0.02), embeddings N(0, 0.02 * scale)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, std=0.02: torch.randn(*s, generator=g) * std
    sd = {"tok_emb.weight": r(V, D, std=0.02 * scale), "pos_emb": r(1, block_size, D, std=0.02 * scale),
          "embedder.weight": r(D, Cf, 1, std=1.0 / math.sqrt(Cf)), "embedder.bias": r(D)}
    for i in range(n_layer):
        b = f"blocks.{i}."
        for ln in ("ln1", "ln2"):
            sd[b + ln + ".weight"] = 1.0 + r(D, std=0.1)
            sd[b + ln + ".bias"] = r(D)
        for n in ("key", "query", "value", "proj"):
            sd[b + f"attn.{n}.weight"] = r(D, D, std=0.02 * scale)
            sd[b + f"attn.{n}.bias"] = r(D)
        sd[b + "attn.mask"] = torch.tril(torch.ones(block_size, block_size)).view(1, 1, block_size, block_size)
        sd[b + "mlp.0.weight"] = r(4 * D, D, std=0.02 * scale)
        sd[b + "mlp.0.bias"] = r(4 * D)
        sd[b + "mlp.2.weight"] = r(D, 4 * D, std=0.02 * scale)
        sd[b + "mlp.2.bias"] = r(D)
    sd["ln_f.weight"] = 1.0 + r(D, std=0.1)
    sd["ln_f.bias"] = r(D)
    sd["head.weight"] = r(V, D, std=0.02 * scale)
    return sd


TINY = dict(n_embd=128, n_layer=2, n_head=2, Cf=16)  # the teacher-forced / sampling fixture configs (head_dim 64)


@torch.no_grad()
def perturb_(sd: dict, seed: int) -> dict:
    """In place, on a GPTFeats state_dict (reference key names): pos_emb (zero at init) N(0, 0.02), LayerNorm weights 1 + N(0, 0.1), LayerNorm /
    Linear / embedder biases (zero or tiny at init) N(0, 0.02); keys visited in sorted order from one seeded generator."""
    g = torch.Generator().manual_seed(seed)
    for k in sorted(sd):
        t = sd[k]
        if k == "pos_emb" or k.endswith(".bias"):
            t.copy_(torch.randn(t.shape, generator=g) * 0.02)
        elif (".ln" in k or k.startswith("ln_f")) and k.endswith(".weight"):
            t.copy_(1.0 + torch.randn(t.shape, generator=g) * 0.1)
    return sd


def gpt_config(V: int, n_embd: int, n_layer: int, n_head: int, Cf: int, block_size: int = 266):
    """(feat_embedding_config, GPT_config) of a GPTFeats, as the caps_transformer configs write them."""
    return (dict(target="torch.nn.Conv1d", params=dict(in_channels=Cf, out_channels=n_embd, kernel_size=1, padding=0)),
            dict(vocab_size=V, block_size=block_size, n_layer=n_layer, n_head=n_head, n_embd=n_embd))
