"""Drop-in for Codebook/specvqgan/models/cond_transformer.py::Net2NetTransformer, the autoregressive SpecVQGAN baseline (the caps_transformer*.yaml
configs): same constructor arguments and state_dict keys (`transformer.*`, `first_stage_model.*`, the permuter buffers), the same `forward`,
`sample`, `encode_to_z`, `encode_to_c`, `decode_to_img`, `top_k_logits`, `get_input`, `get_xc`, `shared_step` and `validation_step`.

`sample` runs the KV-cached decode of `GPTFeats` (ar_engine.py): one fixed launch sequence per position, replayed from a CUDA graph, with the
top-k / softmax / multinomial step in-kernel (torch.multinomial(probs, 1)'s CUDA draw replayed from the default CUDA generator, which is left
where the reference leaves it).  Attention maps are not materialised: `sample` returns (x, None) where the reference returns (x, att).
`shared_step` / `validation_step` score a batch (the validation loss) with one causal pass of `GPTFeats.forward_loss`, in eval mode only.
Training (`training_step`, `configure_optimizers`, pkeep < 1 corruption) and the pkeep <= 0 single-pass branch are not implemented.
"""
import torch
from torch import nn

from ...utils.misc import instantiate_from_config, retarget_config
from ..transformers.mingpt import GPTFeats


def disabled_train(self, mode=True):
    return self


class Net2NetTransformer(nn.Module):
    def __init__(self, transformer_config, first_stage_config, cond_stage_config, first_stage_permuter_config=None, cond_stage_permuter_config=None,
                 ckpt_path=None, ignore_keys=[], first_stage_key="image", cond_stage_key="depth", downsample_cond_size=-1, pkeep=1.0):
        super().__init__()
        model = instantiate_from_config(retarget_config(first_stage_config)).eval()
        model.train = disabled_train.__get__(model)
        self.first_stage_model = model
        self.cond_stage_model = instantiate_from_config(retarget_config(cond_stage_config)).eval()
        if first_stage_permuter_config is None:
            first_stage_permuter_config = {"target": "specvqgan.modules.transformer.permuter.Identity"}
        if cond_stage_permuter_config is None:
            cond_stage_permuter_config = {"target": "specvqgan.modules.transformer.permuter.Identity"}
        self.first_stage_permuter = instantiate_from_config(retarget_config(first_stage_permuter_config))
        self.cond_stage_permuter = instantiate_from_config(retarget_config(cond_stage_permuter_config))
        self.transformer = instantiate_from_config(retarget_config(transformer_config))
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys)
        self.first_stage_key = first_stage_key
        self.cond_stage_key = cond_stage_key
        self.downsample_cond_size = downsample_cond_size
        self.pkeep = pkeep

    def init_from_ckpt(self, path, ignore_keys=list()):
        sd = torch.load(path, map_location="cpu")["state_dict"]
        for k in list(sd.keys()):
            if any(k.startswith(ik) for ik in ignore_keys):
                del sd[k]
        self.load_state_dict(sd, strict=False)
        print(f"Restored from {path}")

    def _feats_transformer(self):
        if not isinstance(self.transformer, GPTFeats):
            raise NotImplementedError(f"transformer {type(self.transformer).__name__}: only GPTFeats (the caps_transformer configs) is implemented")
        return self.transformer

    @torch.no_grad()
    def forward(self, x, c):
        """cond_transformer.py:69-125 at inference: (logits (B, 265, V) of p(z_i | z_<i, c), target z_indices)."""
        if self.training and self.pkeep < 1.0:
            raise NotImplementedError("training-time token corruption (pkeep < 1) is not implemented")
        _, z_indices = self.encode_to_z(x)
        _, c_indices = self.encode_to_c(c)
        logits, _, _ = self._feats_transformer()(z_indices[:, :-1], c)
        cond_size = c.size(-1)
        return logits[:, cond_size - 1:], z_indices

    def top_k_logits(self, logits, k):
        v, ix = torch.topk(logits, k)
        out = logits.clone()
        out[out < v[..., [-1]]] = -float("Inf")
        return out

    @torch.no_grad()
    def sample(self, x, c, steps, temperature=1.0, sample=False, top_k=None, callback=lambda k: None):
        """cond_transformer.py:124-194: x (B, n0) given tokens, c (B, Cf, Tc) features -> (x (B, n0 + steps), None).  The new tokens come from
        the in-kernel top-k / softmax / multinomial (or argmax) step; the default CUDA generator advances as torch.multinomial's would.
        callback(k) is called on the host before token k.  Attention maps are not materialised (None in place of att)."""
        tr = self._feats_transformer()
        assert not tr.training
        if self.pkeep <= 0.0:
            raise NotImplementedError("Implement for GPTFeats")
        if steps == 0:
            return x, None
        ids, _ = tr.sample_tokens(x, c, steps, temperature=temperature, sample=sample, top_k=top_k, callback=callback)
        return ids, None

    def get_input(self, key, batch):
        """cond_transformer.py:318-335 for string keys: 'feature' / 'target' through the condition stage ((B, Tc, Cf) -> (B, Cf, Tc)), anything else
        (a mel (B, H, W) or (B, H, W, C)) to (B, C, H, W); doubles become floats."""
        if not isinstance(key, str):
            raise NotImplementedError("get_input: only string batch keys are implemented (the caps configs' 'image' / 'feature')")
        if key in ["feature", "target"]:
            x = self.cond_stage_model.get_input(batch, key)
        else:
            x = batch[key]
            if len(x.shape) == 3:
                x = x[..., None]
            x = x.permute(0, 3, 1, 2).to(memory_format=torch.contiguous_format)
        if x.dtype == torch.double:
            x = x.float()
        return x

    def get_xc(self, batch, N=None):
        """cond_transformer.py:337-351."""
        x = self.get_input(self.first_stage_key, batch)
        c = self.get_input(self.cond_stage_key, batch)
        if N is not None:
            x, c = x[:N], c[:N]
        return x, c

    @torch.no_grad()
    def shared_step(self, batch, batch_idx=None):
        """cond_transformer.py:353-360 in eval mode: z = encode_to_z(mel), logits of z[:, :-1] after the condition from row cond_size - 1 on,
        loss = F.cross_entropy(logits.reshape(-1, V), z.reshape(-1)), from one causal pass.  Returns the loss (0-dim fp32 tensor)."""
        if self.training:
            raise NotImplementedError("Net2NetTransformer.shared_step in training mode: only the forward (the loss) is implemented; training "
                                      "(gradients) is not. Call .eval() to score.")
        x, c = self.get_xc(batch)
        x, c = x.to(self.transformer.head.weight.device), c.to(self.transformer.head.weight.device)
        _, z_indices = self.encode_to_z(x)
        _, c = self.encode_to_c(c)
        _, loss, _ = self._feats_transformer().forward_loss(z_indices[:, :-1], c, z_indices, c.size(-1) - 1)
        return loss

    def validation_step(self, batch, batch_idx=None):
        """cond_transformer.py:367-370: the shared_step loss (`val/loss`; logging is left to the caller)."""
        return self.shared_step(batch, batch_idx)

    @torch.no_grad()
    def encode_to_z(self, x):
        quant_z, _, info = self.first_stage_model.encode(x)
        indices = info[2].view(quant_z.shape[0], -1)
        indices = self.first_stage_permuter(indices)
        return quant_z, indices

    @torch.no_grad()
    def encode_to_c(self, c):
        if self.downsample_cond_size > -1:
            raise NotImplementedError("downsample_cond_size is not implemented (the caps configs use raw features)")
        quant_c, _, info = self.cond_stage_model.encode(c)
        return quant_c, info[2]

    @torch.no_grad()
    def decode_to_img(self, index, zshape, stage="first"):
        if stage != "first":
            raise NotImplementedError
        index = self.first_stage_permuter(index, reverse=True)
        bhwc = (zshape[0], zshape[2], zshape[3], zshape[1])
        quant_z = self.first_stage_model.quantize.get_codebook_entry(index.reshape(-1), shape=bhwc)
        return self.first_stage_model.decode(quant_z)
