"""Drop-in for sound_synthesis/modeling/transformers/transformer_utils.py::Text2ImageTransformer.

Same constructor arguments and the same state_dict keys (SURVEY.md section 8b), so reference checkpoints load unchanged;
``forward`` runs the hand-written sm_90a kernels through ``DenoiserEngine`` instead of ATen ops (inference);
training goes through ``DenoiserTrainEngine`` (called from DiffusionTransformer._train_loss).  The sub-modules
below only HOLD parameters under the reference's names -- they have no torch forward (there is no fallback path).
"""
import math

import torch
from torch import nn

from ...engine import DenoiserEngine
from ...engine_base import EngineModule
from ...train_engine import DenoiserTrainEngine
from ...utils.misc import instantiate_from_config


class _ParamOnly(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} only stores parameters; the compute path is DenoiserEngine (CUDA kernels)")


class GELU2(_ParamOnly):
    pass


class FullAttention(_ParamOnly):
    def __init__(self, n_embd, n_head):
        super().__init__()
        assert n_embd % n_head == 0
        self.key = nn.Linear(n_embd, n_embd)
        self.query = nn.Linear(n_embd, n_embd)
        self.value = nn.Linear(n_embd, n_embd)
        self.proj = nn.Linear(n_embd, n_embd)
        self.n_head = n_head


class CrossAttention(_ParamOnly):
    def __init__(self, n_embd, condition_embd, n_head, seq_len):
        super().__init__()
        self.key = nn.Linear(condition_embd, n_embd)
        self.query = nn.Linear(n_embd, n_embd)
        self.value = nn.Linear(condition_embd, n_embd)
        self.proj = nn.Linear(n_embd, n_embd)
        self.n_head = n_head
        # dead buffer the reference registers from its causal=True default (transformer_utils.py:87-89); kept for key parity
        self.register_buffer("mask", torch.tril(torch.ones(seq_len, seq_len)).view(1, 1, seq_len, seq_len))


class AdaLayerNorm(_ParamOnly):
    def __init__(self, n_embd, diffusion_step, emb_type="adalayernorm"):
        super().__init__()
        if "abs" in emb_type:
            raise NotImplementedError("sinusoidal ('abs') timestep embedding is not used by the Diffsound configs")
        self.emb = nn.Embedding(diffusion_step, n_embd)
        self.linear = nn.Linear(n_embd, n_embd * 2)


class Block(_ParamOnly):
    def __init__(self, condition_seq_len, n_embd, n_head, seq_len, mlp_hidden_times, activate, condition_dim, diffusion_step, timestep_type):
        super().__init__()
        assert activate == "GELU2", "the fused MLP epilogue implements GELU2 (block_activate of every Diffsound config)"
        self.ln1 = AdaLayerNorm(n_embd, diffusion_step, timestep_type)
        self.ln2 = nn.LayerNorm(n_embd)
        self.attn1 = FullAttention(n_embd, n_head)
        self.attn2 = CrossAttention(n_embd, condition_dim, n_head, seq_len)
        self.ln1_1 = AdaLayerNorm(n_embd, diffusion_step, timestep_type)
        self.mlp = nn.Sequential(nn.Linear(n_embd, mlp_hidden_times * n_embd), GELU2(), nn.Linear(mlp_hidden_times * n_embd, n_embd), nn.Dropout(0.0))


class Text2ImageTransformer(EngineModule):
    def __init__(self, condition_seq_len=77, n_layer=14, n_embd=1024, n_head=16, content_seq_len=1024, attn_pdrop=0, resid_pdrop=0,
                 mlp_hidden_times=4, block_activate=None, attn_type="selfcross", content_spatial_size=[32, 32], condition_dim=512,
                 diffusion_step=1000, timestep_type="adalayernorm", content_emb_config=None, mlp_type="fc", checkpoint=False,
                 precision="f16x3", train_precision="bf16"):
        super().__init__()
        assert attn_type == "selfcross"
        assert mlp_type == "fc", "conv_mlp is not used by the Diffsound configs"
        if attn_pdrop or resid_pdrop:
            raise NotImplementedError("dropout > 0 (training) is outside the inference hot path")
        self.use_checkpoint = checkpoint
        self.content_emb = instantiate_from_config(content_emb_config)
        if content_spatial_size is None:
            s = int(math.sqrt(content_seq_len))
            assert s * s == content_seq_len
            content_spatial_size = (s, s)
        self.blocks = nn.Sequential(*[Block(condition_seq_len, n_embd, n_head, content_seq_len, mlp_hidden_times, block_activate, condition_dim,
                                            diffusion_step, timestep_type) for _ in range(n_layer)])
        out_cls = self.content_emb.num_embed - 1
        self.to_logits = nn.Sequential(nn.LayerNorm(n_embd), nn.Linear(n_embd, out_cls))
        self.condition_seq_len = condition_seq_len
        self.content_seq_len = content_seq_len
        self.n_embd, self.n_head, self.diffusion_step = n_embd, n_head, diffusion_step
        self.apply(self._init_weights)
        self.engine = DenoiserEngine(self, precision=precision)
        self.train_engine = DenoiserTrainEngine(self, precision=train_precision)  # forward-with-activations + backward (A13)

    def _init_weights(self, module):  # same distribution as the reference (:355-363)
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm) and module.elementwise_affine:
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def _apply(self, fn, *a, **k):  # .cuda() / .to(): the training engine's operands and workspaces go stale too
        out = super()._apply(fn, *a, **k)
        if hasattr(self, "train_engine"):
            self.train_engine.reset()
        return out

    @torch.no_grad()
    def forward(self, input, cond_emb, t):
        """input (B,L) int64 ids, cond_emb (B,Lc,condition_dim) fp32, t (B,) int64 -> logits (B, K, L) (view, as the reference's rearrange)."""
        kv = self.engine.encode_condition(cond_emb)  # repacks first if the parameters changed (optimizer.step(), EMA swap, ...)
        logits = self.engine.forward(input.contiguous(), kv, t.to(input.device).contiguous(), cond_emb.shape[1])
        self.engine.check_token_range(*input.shape)
        return logits.clone().permute(0, 2, 1)  # clone: the engine reuses its workspace on the next call
