"""Restatement of the ACT audio-captioning transformer (Codebook/AudiocaptionLoss/models/TransModel.py, models/AudioTransformer.py) and of its
decoders (tools/utils.py greedy_decode, tools/beam.py beam_decode) in plain torch on a state_dict, in any dtype: fp64 for the tests, fp32 for
the benchmark's reference algorithm (the whole prefix re-run for every expanded node, one clip at a time).  Also the seeded weights and mels
the fixtures use: an integer hash (splitmix64), so they do not depend on any library's random generator."""
from __future__ import annotations

import math
import queue

import numpy as np
import torch
import torch.nn.functional as F

ENC_DIM, ENC_DEPTH, ENC_HEADS, ENC_MLP, NUM_CLASSES = 768, 12, 12, 3072, 527


# ---------------------------------------------------------------- seeded tensors
def hash_uniform(seed: int, n: int) -> np.ndarray:
    """n values in [-1, 1) from splitmix64(seed * 2^32 + i), exact integer arithmetic."""
    with np.errstate(over="ignore"):
        z = (np.arange(n, dtype=np.uint64) + np.uint64(seed) * np.uint64(1 << 32)) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -52 - 1.0


def seeded_state_dict(template: dict, seed: int, eos_ind: int | None = None, eos_bias: float = 0.0) -> dict:
    """Weights for every entry of `template` (name -> tensor; shapes only): Linear / embedding weights uniform with variance 1 / fan_in,
    LayerNorm / BatchNorm weights 1 + 0.1 u, biases 0.02 u, running_var 0.5 + 0.5 |u|, running_mean 0.1 u, cls / pos 0.02 u, pe kept.
    eos_bias is added to dec_fc.bias[eos_ind]."""
    out = {}
    for i, (k, v) in enumerate(template.items()):
        shape, n = tuple(v.shape), v.numel()
        if k.endswith("num_batches_tracked") or k == "pos_encoder.pe":
            out[k] = v.clone()
            continue
        u = hash_uniform(seed * 1000 + i, n).reshape(shape)
        if k.endswith("running_var"):
            a = 0.5 + 0.5 * np.abs(u)
        elif k.endswith("running_mean"):
            a = 0.1 * u
        elif k.endswith("bias"):
            a = 0.02 * u
        elif v.dim() == 1:
            a = 1.0 + 0.1 * u
        elif k.endswith(("cls_token", "pos_embedding")):
            a = 0.02 * u
        else:
            a = u * math.sqrt(3.0 / shape[-1])
        out[k] = torch.from_numpy(np.ascontiguousarray(a)).float()
    if eos_ind is not None:
        out["dec_fc.bias"][eos_ind] += eos_bias
    return out


def seeded_mels(seed: int, B: int, T: int = 848) -> torch.Tensor:
    """(B, T, 80) fp32 in [0, 1], the range pipeline.save_clip writes."""
    return torch.from_numpy(0.5 + 0.5 * hash_uniform(seed, B * T * 80).reshape(B, T, 80)).float()


# ---------------------------------------------------------------- model
def _ln(x, sd, p, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"].to(x), sd[p + ".bias"].to(x), eps)


def _lin(x, sd, p):
    return F.linear(x, sd[p + ".weight"].to(x), sd[p + ".bias"].to(x))


def encode(sd: dict, spec: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    """spec (B, T, 80) -> memory (B, T / 4 + 1, nhid) = relu(encoder_linear(AudioTransformer_80(spec))) in eval mode."""
    g = lambda k: sd[k].to(dtype)
    x = spec.to(dtype)
    B, T, _ = x.shape
    x = (x - g("encoder.bn0.running_mean")) / torch.sqrt(g("encoder.bn0.running_var") + 1e-5) * g("encoder.bn0.weight") + g("encoder.bn0.bias")
    x = _lin(x.reshape(B, T // 4, 320), sd, "encoder.patch_embed.proj")
    x = torch.cat([g("encoder.cls_token").expand(B, 1, ENC_DIM), x], 1) + g("encoder.pos_embedding")[:, :T // 4 + 1]
    hd = ENC_DIM // ENC_HEADS
    for i in range(ENC_DEPTH):
        p = f"encoder.blocks.layers.{i}"
        q, k, v = _lin(_ln(x, sd, p + ".0.norm"), sd, p + ".0.fn.qkv").chunk(3, -1)
        q, k, v = (t.reshape(B, -1, ENC_HEADS, hd).transpose(1, 2) for t in (q, k, v))
        a = torch.softmax(q @ k.transpose(-1, -2) * hd ** -0.5, -1) @ v
        x = _lin(a.transpose(1, 2).reshape(B, -1, ENC_DIM), sd, p + ".0.fn.proj.0") + x
        h = _ln(x, sd, p + ".1.norm")
        x = _lin(F.gelu(_lin(h, sd, p + ".1.fn.mlp.fc1")), sd, p + ".1.fn.mlp.fc2") + x
    x = _lin(_ln(x, sd, "encoder.mlp_head.0"), sd, "encoder.mlp_head.1")
    return torch.relu(_lin(x, sd, "encoder_linear"))


def _mha(xq, xkv, sd, p, nhead, causal):
    D = xq.shape[-1]
    w, b = sd[p + ".in_proj_weight"].to(xq), sd[p + ".in_proj_bias"].to(xq)
    q, k, v = F.linear(xq, w[:D], b[:D]), F.linear(xkv, w[D:2 * D], b[D:2 * D]), F.linear(xkv, w[2 * D:], b[2 * D:])
    B, Lq, Lk, hd = xq.shape[0], xq.shape[1], xkv.shape[1], D // nhead
    q, k, v = (t.reshape(B, -1, nhead, hd).transpose(1, 2) for t in (q, k, v))
    s = q @ k.transpose(-1, -2) / math.sqrt(hd)
    if causal:
        s = s.masked_fill(torch.ones(Lq, Lk, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    a = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, Lq, D)
    return _lin(a, sd, p + ".out_proj")


def decode(sd: dict, memory: torch.Tensor, tgt: torch.Tensor, nhead: int, dtype=torch.float64) -> torch.Tensor:
    """ACT.decode with the causal mask: memory (B, Lm, nhid), tgt (B, n) -> logits (B, n, ntoken) (batch-first)."""
    mem = memory.to(dtype)
    D = mem.shape[-1]
    n = tgt.shape[1]
    x = sd["word_emb.weight"].to(dtype)[tgt] * math.sqrt(D) + sd["pos_encoder.pe"].to(dtype)[:n, 0]
    nl = len({k.split(".")[2] for k in sd if k.startswith("transformer_decoder.layers.")})
    for i in range(nl):
        p = f"transformer_decoder.layers.{i}"
        x = _ln(x + _mha(x, x, sd, p + ".self_attn", nhead, True), sd, p + ".norm1")
        x = _ln(x + _mha(x, mem, sd, p + ".multihead_attn", nhead, False), sd, p + ".norm2")
        x = _ln(x + _lin(F.gelu(_lin(x, sd, p + ".linear1")), sd, p + ".linear2"), sd, p + ".norm3")
    return _lin(x, sd, "dec_fc")


def greedy_decode(sd, memory, nhead, sos_ind, max_len=30, dtype=torch.float64):
    """utils.py greedy_decode on the memory: (B, max_len + 1), full prefix re-run per position."""
    ys = torch.full((memory.shape[0], 1), sos_ind, dtype=torch.int64, device=memory.device)
    for _ in range(max_len):
        out = decode(sd, memory, ys, nhead, dtype)[:, -1]
        ys = torch.cat([ys, torch.argmax(torch.softmax(out, -1), 1, keepdim=True)], 1)
    return ys


def next_logprobs(sd, memory_row, words, nhead, dtype=torch.float64):
    """log_softmax of the last position after the prefix `words` of one clip (memory_row (Lm, nhid))."""
    out = decode(sd, memory_row[None], torch.tensor([words], device=memory_row.device), nhead, dtype)[0, -1]
    return F.log_softmax(out, -1)


class _Node:
    def __init__(self, prev, words, logp, leng):
        self.prevNode, self.words, self.logp, self.leng = prev, words, logp, leng

    def __lt__(self, other):
        return self.logp < other.logp

    def eval(self):
        return self.logp / float(self.leng - 1 + 1e-6) + 1.0 * 0


def beam_decode_one(logprobs_of, sos_ind, eos_ind, beam_width, top_k):
    """beam.py's search for one clip, as the reference runs it (PriorityQueue); logprobs_of(words) -> the fp32 log-probs of the next word."""
    endnodes, number_required = [], min(top_k + 1, top_k)
    nodes = queue.PriorityQueue()
    node = _Node(None, [sos_ind], 0, 1)
    nodes.put((-node.eval(), node))
    qsize = 1
    while qsize <= 2000:
        score, n = nodes.get()
        if n.words[-1] == eos_ind and n.prevNode is not None:
            endnodes.append((score, n))
            if len(endnodes) >= number_required:
                break
            continue
        lp, ix = torch.topk(logprobs_of(n.words).float(), beam_width)
        for k in range(beam_width):
            c = _Node(n, n.words + [int(ix[k])], n.logp + lp[k].item(), n.leng + 1)
            nodes.put((-c.eval(), c))
        qsize += beam_width - 1
    if not endnodes:
        endnodes = [nodes.get() for _ in range(top_k)]
    ends = sorted(endnodes, key=lambda t: t[0])
    return [ends[i][1].words for i in range(top_k)]
