"""Drop-in for sound_synthesis/modeling/transformers/diffusion_transformer.py::DiffusionTransformer (inference side).

Same constructor arguments, buffers and state_dict keys as the reference (ckpt['ema'] loads unchanged).  The 100-step
loop carries token ids (not (B,K+1,L) log-one-hot tensors); each step is  denoiser (DenoiserEngine)  ->  one fused
posterior/truncation/Gumbel kernel, optionally replayed as a CUDA graph.  The reference's separately callable methods
(`predict_start`, `q_posterior`, `log_sample_categorical`, `p_sample`, `p_pred`) are kept -- and stay re-bindable
instance attributes, because reference code monkey-patches them (models/dalle_spec.py:207-210) -- each mapped onto the
same kernel through its stage flags.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import nn

from ... import ops
from ... import train_ops
from ...graphs import capture
from ...utils.misc import instantiate_from_config

_SCHED_ROWS = ["log_at", "log_bt", "log_ct", "log_1_min_ct", "log_cumprod_at", "log_cumprod_bt", "log_cumprod_ct", "log_1_min_cumprod_ct"]


def alpha_schedule(time_step, N=100, att_1=0.99999, att_T=0.000009, ctt_1=0.000009, ctt_T=0.9):
    """fp64 mask-and-uniform schedule; must stay bit-identical to the reference (diffusion_transformer.py:122-151)."""
    att = np.arange(0, time_step) / (time_step - 1) * (att_T - att_1) + att_1
    att = np.concatenate(([1], att))
    at = att[1:] / att[:-1]
    ctt = np.arange(0, time_step) / (time_step - 1) * (ctt_T - ctt_1) + ctt_1
    ctt = np.concatenate(([0], ctt))
    one_minus_ctt = 1 - ctt
    one_minus_ct = one_minus_ctt[1:] / one_minus_ctt[:-1]
    ct = 1 - one_minus_ct
    bt = (1 - at - ct) / N
    att = np.concatenate((att[1:], [1]))
    ctt = np.concatenate((ctt[1:], [0]))
    btt = (1 - att - ctt) / N
    return at, bt, ct, att, btt, ctt


def parse_truncation(sample_type):
    """'top0.85r' -> (1, 0.85, 0); 'top20p' -> (2, 0, 20); None/'normal' -> (0, 0, 0)   (dalle_spec.py:146-177)."""
    if not sample_type:
        return 0, 0.0, 0
    head = sample_type.split(",")[0]
    if head[:3] != "top":
        return 0, 0.0, 0
    if head[-1] == "r":
        return 1, float(head[3:-1]), 0
    if head[-1] == "p":
        return 2, 0.0, int(head[3:-1])
    raise ValueError(f"wrong sample type {sample_type!r}")


class DiffusionTransformer(nn.Module):
    def __init__(self, *, content_emb_config=None, condition_emb_config=None, transformer_config=None, diffusion_step=100,
                 alpha_init_type="cos", auxiliary_loss_weight=0, adaptive_auxiliary_loss=False, mask_weight=[1, 1]):
        super().__init__()
        if condition_emb_config is None:
            self.condition_emb = None
        else:
            self.condition_emb = instantiate_from_config(condition_emb_config)
            self.condition_dim = self.condition_emb.embed_dim
        transformer_config["params"]["diffusion_step"] = diffusion_step  # the reference mutates the config the same way (:177-178)
        transformer_config["params"]["content_emb_config"] = content_emb_config
        self.transformer = instantiate_from_config(transformer_config)
        self.content_seq_len = transformer_config["params"]["content_seq_len"]
        self.amp = False
        self.num_classes = self.transformer.content_emb.num_embed  # K + 1
        self.loss_type = "vb_stochastic"
        self.shape = transformer_config["params"]["content_seq_len"]
        self.num_timesteps = diffusion_step
        self.parametrization = "x0"
        self.auxiliary_loss_weight = auxiliary_loss_weight
        self.adaptive_auxiliary_loss = adaptive_auxiliary_loss
        self.mask_weight = mask_weight
        if alpha_init_type != "alpha1":
            raise ValueError("alpha_init_type must be 'alpha1' (the reference only prints a warning and then fails, :196-199)")
        at, bt, ct, att, btt, ctt = alpha_schedule(self.num_timesteps, N=self.num_classes)
        t64 = lambda a: torch.tensor(a.astype("float64"))
        log_at, log_bt, log_ct = torch.log(t64(at)), torch.log(t64(bt)), torch.log(t64(ct))
        log_cumprod_at, log_cumprod_bt, log_cumprod_ct = torch.log(t64(att)), torch.log(t64(btt)), torch.log(t64(ctt))
        log_1_min_a = lambda a: torch.log(1 - a.exp() + 1e-40)
        log_1_min_ct = log_1_min_a(log_ct)
        log_1_min_cumprod_ct = log_1_min_a(log_cumprod_ct)
        lae = lambda a, b: torch.max(a, b) + torch.log(torch.exp(a - torch.max(a, b)) + torch.exp(b - torch.max(a, b)))
        assert lae(log_ct, log_1_min_ct).abs().sum().item() < 1.0e-5
        assert lae(log_cumprod_ct, log_1_min_cumprod_ct).abs().sum().item() < 1.0e-5
        self.diffusion_acc_list = [0] * self.num_timesteps
        self.diffusion_keep_list = [0] * self.num_timesteps
        for name, v in (("log_at", log_at), ("log_bt", log_bt), ("log_ct", log_ct), ("log_cumprod_at", log_cumprod_at),
                        ("log_cumprod_bt", log_cumprod_bt), ("log_cumprod_ct", log_cumprod_ct), ("log_1_min_ct", log_1_min_ct),
                        ("log_1_min_cumprod_ct", log_1_min_cumprod_ct)):
            self.register_buffer(name, v.float())
        self.register_buffer("Lt_history", torch.zeros(self.num_timesteps))
        self.register_buffer("Lt_count", torch.zeros(self.num_timesteps))
        # knobs of the fused path (not in the reference): truncation applied inside the sampler kernel, CUDA-graph replay
        self.truncation = None
        self.resample_rate = 0.0  # 'q' sample types: probability of repeating a step's p_sample at the same t
        self.use_cuda_graph = True
        self._sched_cache = None
        self._graphs = {}
        self.last_gpu_launches = 0

    def __deepcopy__(self, memo):
        """EMA's shadow copy (reference engine/ema.py:19): captured CUDA graphs / schedule caches belong to this instance only."""
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = {} if k == "_graphs" else (None if k == "_sched_cache" else copy.deepcopy(v, memo))
        return new

    # ------------------------------------------------------------------ helpers
    @property
    def device(self):
        return self.transformer.to_logits[-1].weight.device

    def _sched(self) -> torch.Tensor:
        """(8, T+1) fp32 table in the row order dsb_posterior_sample expects, rebuilt if the buffers moved/changed."""
        key = (self.log_at.data_ptr(), self.log_at.device)
        if self._sched_cache is None or self._sched_cache[0] != key:
            T = self.num_timesteps
            s = torch.zeros(8, T + 1, dtype=torch.float32, device=self.log_at.device)
            for i, n in enumerate(_SCHED_ROWS):
                b = getattr(self, n)
                s[i, : b.numel()] = b
            self._sched_cache = (key, s)
        return self._sched_cache[1]

    def _trunc(self):
        return parse_truncation(self.truncation)

    def _sampler_ops(self):
        """(posterior_sample, posterior_sample_loop) for this codebook: one warp per column up to K = 1055, one CTA per column above."""
        if self.num_classes - 1 > ops.WARP_SAMPLER_MAX_K:
            return ops.posterior_sample_wide, ops.posterior_sample_wide_loop
        return ops.posterior_sample, ops.posterior_sample_loop

    # ------------------------------------------------------------------ reference-compatible stage methods
    @torch.no_grad()
    def predict_start(self, log_x_t, cond_emb, t):
        """p(x0|xt): (B,K+1,L) log-one-hot -> log_pred (B,K+1,L)  (diffusion_transformer.py:269-291); applies self.truncation if set."""
        x_t = log_x_t.argmax(1)
        out = self.transformer(x_t, cond_emb, t)  # (B,K,L) view of the (B,L,K) kernel output
        assert out.size(0) == x_t.size(0) and out.size(1) == self.num_classes - 1 and out.size()[2:] == x_t.size()[1:]
        blk = out.permute(0, 2, 1)
        assert blk.is_contiguous()
        B, L, K = blk.shape
        log_pred = torch.empty(B, K + 1, L, dtype=torch.float32, device=blk.device)
        mode, r, k = self._trunc()
        self._sampler_ops()[0](blk, None, None, None, None, T=self.num_timesteps, trunc_mode=mode, trunc_r=r, trunc_k=k, log_prob_out=log_pred,
                               stage=ops.STAGE_SKIP_POSTERIOR | ops.STAGE_SKIP_SAMPLE)
        return log_pred

    @torch.no_grad()
    def q_posterior(self, log_x_start, log_x_t, t):
        """log p_theta(x_{t-1}|x_t) (diffusion_transformer.py:293-339); log_x_t is a log-one-hot (only its argmax is used)."""
        assert t.min().item() >= 0 and t.max().item() < self.num_timesteps
        x_t = log_x_t.argmax(1).contiguous()
        out = torch.empty_like(log_x_start, memory_format=torch.contiguous_format)
        self._sampler_ops()[0](log_x_start.contiguous().float(), x_t, t.contiguous(), None, self._sched(), T=self.num_timesteps, trunc_mode=0,
                               log_prob_out=out, stage=ops.STAGE_INPUT_LOGPROB | ops.STAGE_SKIP_SAMPLE)
        return out

    @torch.no_grad()
    def log_sample_categorical(self, logits, return_index=False):
        """Gumbel-argmax with torch.rand_like's stream (diffusion_transformer.py:359-368); returns the log-one-hot re-encoding."""
        uniform = torch.rand_like(logits)
        ids = self._sampler_ops()[0](logits.contiguous().float(), None, None, uniform, None, T=self.num_timesteps, trunc_mode=0,
                                     stage=ops.STAGE_INPUT_LOGPROB | ops.STAGE_SKIP_POSTERIOR)
        return ids if return_index else index_to_log_onehot(ids, self.num_classes)

    def p_pred(self, log_x, cond_emb, t):
        log_x_recon = self.predict_start(log_x, cond_emb, t)
        return self.q_posterior(log_x_start=log_x_recon, log_x_t=log_x, t=t)

    @torch.no_grad()
    def p_sample(self, log_x, cond_emb, t):
        return self.log_sample_categorical(self.p_pred(log_x, cond_emb, t))

    @torch.no_grad()
    def q_sample(self, log_x_start, t, return_index=False):
        """x_t ~ q(x_t | x_0) (diffusion_transformer.py:370-377): q_pred + Gumbel-argmax in one kernel, uniforms from torch.rand_like's stream."""
        x0 = log_x_start.argmax(1).contiguous()
        uniform = torch.rand_like(log_x_start, memory_format=torch.contiguous_format)
        ids = train_ops.q_sample(x0, t.contiguous(), uniform, self._sched(), self.num_timesteps)
        return ids if return_index else index_to_log_onehot(ids, self.num_classes)

    def sample_time(self, b, device, method="uniform"):
        """Importance-sampled timesteps (diffusion_transformer.py:379-406); host-side policy on two 100-element buffers."""
        if method == "importance":
            if not (self.Lt_count > 10).all():
                return self.sample_time(b, device, method="uniform")
            Lt_sqrt = torch.sqrt(self.Lt_history + 1e-10) + 0.0001
            Lt_sqrt[0] = Lt_sqrt[1]
            pt_all = Lt_sqrt / Lt_sqrt.sum()
            t = torch.multinomial(pt_all, num_samples=b, replacement=True)
            return t, pt_all.gather(dim=0, index=t)
        if method == "uniform":
            t = torch.randint(0, self.num_timesteps, (b,), device=device).long()
            return t, torch.ones_like(t).float() / self.num_timesteps
        raise ValueError(method)

    def _train_loss(self, x, cond_emb, is_train=True, want_prob=True):
        """KL training loss (diffusion_transformer.py:408-476).  Returns (exp(log_model_prob) or None, vb_loss (B,), loss scalar) where the scalar
        already carries forward()'s normalisation (:568-569) and is differentiable w.r.t. the transformer parameters."""
        assert self.loss_type == "vb_stochastic"
        B, L = x.shape
        x = x.contiguous()
        oob = ((x < 0) | (x >= self.num_classes)).any()  # read together with the accuracy flags below (no extra sync point)
        t, pt = self.sample_time(B, x.device, "importance")
        uniform = torch.rand(B, self.num_classes, L, dtype=torch.float32, device=x.device)  # == rand_like(log_EV_qxt_x0), :360
        x_t = train_ops.q_sample(x, t.contiguous(), uniform, self._sched(), self.num_timesteps)
        loss, prob, vb, hits = denoiser_loss(self, x, x_t, cond_emb, t.contiguous(), pt.float().contiguous(), bool(is_train), bool(want_prob))
        # accuracy bookkeeping of :424-436 (one small D2H copy instead of 2B .item() calls)
        rate = hits.float().mean(dim=1).cpu()
        if bool(oob):  # the reference asserts in index_to_log_onehot (diffusion_transformer.py:46-47)
            raise AssertionError(f"Error: content token id outside [0, {self.num_classes})")
        for i, this_t in enumerate(t.tolist()):
            self.diffusion_acc_list[this_t] = float(rate[i, 0]) * 0.1 + self.diffusion_acc_list[this_t] * 0.9
            self.diffusion_keep_list[this_t] = float(rate[i, 1]) * 0.1 + self.diffusion_keep_list[this_t] * 0.9
        return prob, vb, loss

    # ------------------------------------------------------------------ fused fast path
    def _stages_overridden(self) -> bool:
        """True when a caller re-bound one of the stage methods on the instance (e.g. the reference DALLE's truncation wrapper)."""
        return any(n in self.__dict__ for n in ("predict_start", "q_posterior", "log_sample_categorical", "p_sample", "p_pred"))

    @torch.no_grad()
    def _fused_step(self, st):
        """One p_sample on ids: denoiser -> fused sampler.  Every launch is a kernel of this library: the sampler draws its own uniforms (bit-for-bit
        the stream torch.rand_like(model_log_prob) would produce, diffusion_transformer.py:360), writes x in place and advances t / t_post / the RNG
        offset on the device, so the captured step needs no host-side update between replays."""
        eng = self.transformer.engine
        logits = eng.forward(st["x"], st["kv"], st["t"], st["Lc"])
        mode, r, k = st["trunc"]
        self._sampler_ops()[1](logits, st["x"], st["t"], st["t_post"], self._sched(), st["ctrl"], st["t_sched"], st["tp_sched"], T=self.num_timesteps,
                               trunc_mode=mode, trunc_r=r, trunc_k=k)

    def _arm_loop(self, st, steps, post_steps, seed, offset, counter_offset, nthreads):
        """(Re)load the device-side loop state: RNG (seed, offset), the timestep schedule, step 0's t / t_post.  One small H2D copy per sample()."""
        n = len(steps)
        if n > st["t_sched"].numel():
            raise RuntimeError(f"sampling schedule of {n} steps exceeds the captured capacity {st['t_sched'].numel()}")
        host = st["host"]
        host[:n] = torch.tensor(steps, dtype=torch.int64)
        host[st["cap"]:st["cap"] + n] = torch.tensor(post_steps, dtype=torch.int64)
        c = host[2 * st["cap"]:]
        c[0] = np.array([seed & (2 ** 64 - 1)], dtype=np.uint64).view(np.int64)[0].item()
        c[1], c[2], c[3], c[4], c[5], c[6] = offset, counter_offset, nthreads, 0, n, 0
        st["dev"].copy_(host)  # blocking: the pinned staging buffer is rewritten by the next call
        st["t"].fill_(steps[0])
        st["t_post"].fill_(post_steps[0])

    def _run_steps(self, cond_emb, batch_size, steps, post_steps, x_init=None):
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("DiffusionTransformer sampling needs a CUDA device (no CPU fallback)")
        eng = self.transformer.engine
        K, L, B = self.num_classes - 1, self.shape, batch_size
        kv = eng.encode_condition(cond_emb)  # (re)packs the weights if they changed
        key = (B, cond_emb.shape[1], self.truncation)
        st = self._graphs.get(key) if self.use_cuda_graph else None
        if st is not None and st["generation"] != eng.generation:
            st = None  # weights were repacked: the captured graph holds stale pointers
        if st is None:
            cap = max(4 * self.num_timesteps, len(steps))  # schedule capacity ('q' re-sampling can double the step count)
            devbuf = torch.zeros(2 * cap + 8, dtype=torch.int64, device=dev)
            st = dict(x=torch.empty(B, L, dtype=torch.int64, device=dev), t=torch.zeros(B, dtype=torch.int64, device=dev),
                      t_post=torch.zeros(B, dtype=torch.int64, device=dev), kv=torch.empty_like(kv), Lc=cond_emb.shape[1], trunc=self._trunc(),
                      graph=None, generation=eng.generation, cap=cap, dev=devbuf, host=torch.zeros(2 * cap + 8, dtype=torch.int64).pin_memory(),
                      t_sched=devbuf[:cap], tp_sched=devbuf[cap:2 * cap], ctrl=devbuf[2 * cap:])
        st["kv"].copy_(kv)
        # the reference draws torch.rand_like(logits) once per step from the default CUDA generator: replay exactly that stream, then leave the
        # generator where the reference would have left it
        gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
        seed, offset = gen.initial_seed(), gen.get_offset()
        nthreads, counter_offset = ops.aten_rand_geometry(B * (K + 1) * L, dev)
        if self.use_cuda_graph and st["graph"] is None:  # the warm-up runs one step: the loop state is re-armed afterwards
            self._arm_loop(st, steps, post_steps, seed, offset, counter_offset, nthreads)
            st["x"].fill_(K)
            st["graph"] = capture(lambda: self._fused_step(st), dev)
            self._graphs[key] = st
        self._arm_loop(st, steps, post_steps, seed, offset, counter_offset, nthreads)
        if x_init is None:
            st["x"].fill_(K)  # all-[MASK] start state (diffusion_transformer.py:633-636)
        else:
            st["x"].copy_(x_init)
        for _ in steps:
            if st["graph"] is not None:
                st["graph"].replay()
            else:
                self._fused_step(st)
        gen.set_offset(offset + len(steps) * counter_offset)
        self.last_gpu_launches = len(steps) * (eng.launches_per_forward + 1)
        out = st["x"].clone()
        eng.check_token_range(B, L)  # a token id >= num_embed raises like the reference's embedding lookup (one 4-byte read after the loop)
        return out

    def _cond(self, condition_token, condition_embed):
        if self.condition_emb is not None:
            with torch.no_grad():
                return self.condition_emb(condition_token).float()
        return condition_embed.float() if condition_embed is not None else None

    @torch.no_grad()
    def sample(self, condition_token, condition_mask, condition_embed, content_token=None, filter_ratio=0.5, temperature=1.0,
               return_att_weight=False, return_logits=False, content_logits=None, print_log=True, **kwargs):
        """Reference signature (diffusion_transformer.py:587-659).  filter_ratio=0 (the only value the inference script uses,
        generate_samples_batch.py:164) starts from all-[MASK]."""
        batch_size = condition_token.shape[0] if condition_token is not None else kwargs["batch_size"]
        start_step = int(self.num_timesteps * filter_ratio)
        cond_emb = self._cond(condition_token, condition_embed)
        x_init = None
        if start_step != 0:  # content-conditioned: noise the given tokens to t = start_step-1, then denoise from there (:647-655)
            t0 = torch.full((batch_size,), start_step - 1, device=self.device, dtype=torch.long)
            x_init = self.q_sample(index_to_log_onehot(content_token, self.num_classes), t0, return_index=True)
        steps = list(range((start_step or self.num_timesteps) - 1, -1, -1))
        if self.resample_rate > 0:  # host-side coin per step, like the reference's wrapper (python `random`, dalle_spec.py:139-141)
            import random
            steps = [s_ for t_ in steps for s_ in ([t_, t_] if random.random() < self.resample_rate else [t_])]
        if self._stages_overridden():
            content_token = self._sample_unfused(cond_emb, batch_size, steps, steps, x_init=x_init)
        else:
            content_token = self._run_steps(cond_emb, batch_size, steps, steps, x_init=x_init)
        output = {"content_token": content_token}
        if return_logits:
            output["logits"] = torch.exp(index_to_log_onehot(content_token, self.num_classes))
        return output

    @torch.no_grad()
    def sample_uniform_only(self, condition_token, condition_mask, condition_embed, content_token=None, filter_ratio=0.5, temperature=1.0,
                            return_att_weight=False, return_logits=False, content_logits=None, print_log=True, **kwargs):
        """Reference :661-746: as sample(), but filter_ratio = 0 starts from tokens drawn uniformly from [0, K-1) (the reference's
        `torch.randint(0, self.num_classes-2, ...)` on the CPU generator) instead of all-[MASK]."""
        batch_size = condition_token.shape[0] if condition_token is not None else kwargs["batch_size"]
        start_step = int(self.num_timesteps * filter_ratio)
        cond_emb = self._cond(condition_token, condition_embed)
        if start_step == 0:
            x_init = torch.randint(0, self.num_classes - 2, (batch_size, self.shape)).to(self.device)
            start_step = self.num_timesteps
        else:
            t0 = torch.full((batch_size,), start_step - 1, device=self.device, dtype=torch.long)
            x_init = self.q_sample(index_to_log_onehot(content_token, self.num_classes), t0, return_index=True)
        steps = list(range(start_step - 1, -1, -1))
        if self._stages_overridden():
            content_token = self._sample_unfused(cond_emb, batch_size, steps, steps, x_init=x_init)
        else:
            content_token = self._run_steps(cond_emb, batch_size, steps, steps, x_init=x_init)
        output = {"content_token": content_token}
        if return_logits:
            output["logits"] = torch.exp(index_to_log_onehot(content_token, self.num_classes))
        return output

    @torch.no_grad()
    def sample_fast(self, condition_token, condition_mask, condition_embed, content_token=None, filter_ratio=0.5, temperature=1.0,
                    return_att_weight=False, return_logits=False, content_logits=None, print_log=True, skip_step=1, **kwargs):
        """Skip-step sampler (diffusion_transformer.py:748-812): the denoiser sees t, q_posterior sees t - skip_step."""
        batch_size = condition_token.shape[0] if condition_token is not None else kwargs["batch_size"]
        assert int(self.num_timesteps * filter_ratio) == 0
        cond_emb = self._cond(condition_token, condition_embed)
        steps = list(range(self.num_timesteps - 1, -1, -1 - skip_step))
        if steps[-1] != 0:
            steps.append(0)
        post = [s - skip_step if s > skip_step else s for s in steps]
        if self._stages_overridden():
            content_token = self._sample_unfused(cond_emb, batch_size, steps, post)
        else:
            content_token = self._run_steps(cond_emb, batch_size, steps, post)
        output = {"content_token": content_token}
        if return_logits:
            output["logits"] = torch.exp(index_to_log_onehot(content_token, self.num_classes))
        return output

    @torch.no_grad()
    def _sample_unfused(self, cond_emb, batch_size, steps, post_steps, x_init=None):
        """Stage-by-stage loop through the (possibly re-bound) reference-named methods; every stage is still a CUDA kernel."""
        dev = self.device
        K, L = self.num_classes - 1, self.shape
        log_z = index_to_log_onehot(torch.full((batch_size, L), K, dtype=torch.int64, device=dev) if x_init is None else x_init, self.num_classes)
        for ti, tp in zip(steps, post_steps):
            t = torch.full((batch_size,), ti, device=dev, dtype=torch.long)
            if ti == tp:
                log_z = self.p_sample(log_z, cond_emb, t)
            else:
                log_x_recon = self.predict_start(log_z, cond_emb, t)
                log_z = self.log_sample_categorical(self.q_posterior(log_x_start=log_x_recon, log_x_t=log_z,
                                                                     t=torch.full((batch_size,), tp, device=dev, dtype=torch.long)))
        return log_z.argmax(1)

    def parameters(self, recurse=True, name=None):
        """Reference override (diffusion_transformer.py:483-537): with a name, return AdamW groups -- Linear weights decayed (0.01), biases /
        LayerNorm / Embedding weights not (the minGPT split).  The reference's own named branch trips its completeness assert (its name sets keep
        the 'transformer.' prefix, its param_dict does not; the shipped configs only ever pass name='none'); this is the intended behaviour."""
        if name is None or name == "none":
            return super().parameters(recurse=recurse)
        decay, no_decay = set(), set()
        for mn, m in self.named_modules():
            for pn, _ in m.named_parameters(recurse=False):
                fpn = f"{mn}.{pn}" if mn else pn
                if pn.endswith("bias"):
                    no_decay.add(fpn)
                elif pn.endswith("weight") and isinstance(m, nn.Linear):
                    decay.add(fpn)
                elif pn.endswith("weight") and isinstance(m, (nn.LayerNorm, nn.Embedding)):
                    no_decay.add(fpn)
        strip = lambda names: {n[len("transformer."):] for n in names if n.startswith("transformer.")}
        decay, no_decay = strip(decay), strip(no_decay)
        param_dict = dict(self.transformer.named_parameters())
        assert not (decay & no_decay) and not (param_dict.keys() - (decay | no_decay))
        return [{"params": [param_dict[pn] for pn in sorted(decay)], "weight_decay": 0.01},
                {"params": [param_dict[pn] for pn in sorted(no_decay)], "weight_decay": 0.0}]

    def forward(self, input, return_loss=False, return_logits=True, return_att_weight=False, is_train=True, **kwargs):
        """Training / validation entry (diffusion_transformer.py:539-584): {'logits': exp(log_model_prob), 'loss': scalar}."""
        if kwargs.get("autocast") is True:
            self.amp = True  # kept for interface parity; the engine's GEMM precision is fixed at construction (train_precision)
        sample_image = input["content_token"]
        if self.condition_emb is not None:
            with torch.no_grad():
                cond_emb = self.condition_emb(input["condition_token"]).float()
        else:
            cond_emb = input["condition_embed_token"].float() if input.get("condition_embed_token") is not None else None
        out = {}
        if is_train:
            prob, _, loss = self._train_loss(sample_image, cond_emb, want_prob=return_logits)
            if return_logits:
                out["logits"] = prob
            if return_loss:
                out["loss"] = loss
        self.amp = False
        return out


def denoiser_loss(dt, x0, x_t, cond_emb, t, pt, is_train=True, want_prob=True):
    """(loss, exp(log_model_prob) or empty, vb_loss, accuracy flags) with the hand-written backward attached.
    One autograd node per backward segment (tail <- layer 0 <- ... <- layer NL-1 <- head/loss): a layer's parameter gradients reach autograd -- and
    DistributedDataParallel's bucketed all-reduce (solver_spec.py:109) -- as soon as that layer's backward graph has been launched, so the NCCL traffic
    of layer l overlaps the backward of layers l-1 ... 0 instead of starting after the whole backward pass."""
    eng = dt.transformer.train_engine
    named = dict(dt.transformer.named_parameters())
    carrier = None
    for seg in ["tail"] + [("layer", li) for li in range(len(dt.transformer.blocks))]:
        names = tuple(eng.segment_names(seg))
        carrier = _SegmentGrad.apply(eng, seg, names, carrier, *[named[n] for n in names])
    names = tuple(eng.segment_names("head"))
    return _DenoiserLoss.apply(dt, x0, x_t, cond_emb, t, pt, is_train, want_prob, names, carrier, *[named[n] for n in names])


class _DenoiserLoss(torch.autograd.Function):
    """loss = _train_loss(denoiser(x_t, cond, t)) with a hand-written backward: forward runs DenoiserTrainEngine.forward and the fused loss
    kernel (which also emits d loss / d logits); backward runs DenoiserTrainEngine.backward and hands every parameter its gradient."""

    @staticmethod
    def forward(ctx, dt, x0, x_t, cond_emb, t, pt, is_train, want_prob, names, carrier, *params):
        eng = dt.transformer.train_engine
        B, L = x0.shape
        K = dt.num_classes - 1
        dev = x0.device
        logits = eng.forward(x_t, cond_emb, t)
        need_grad = any(ctx.needs_input_grad[9:])  # the carrier (-> earlier segments' parameters) or a head parameter
        dlogits = eng.dlogits_buffer() if need_grad else None  # engine-owned: the static input of its backward graph
        prob = torch.empty(B, K + 1, L, dtype=torch.float32, device=dev) if want_prob else None
        hits = torch.empty(B, L, 2, dtype=torch.int32, device=dev)
        aux = float(dt.auxiliary_loss_weight) if is_train else 0.0
        res = train_ops.train_loss(logits, x0, x_t, t, pt, dt._sched(), dt.num_timesteps, aux_weight=aux, adaptive=bool(dt.adaptive_auxiliary_loss),
                                   mask_weight=dt.mask_weight, dlogits=dlogits, log_model_prob=prob, hits=hits, lt_history=dt.Lt_history,
                                   lt_count=dt.Lt_count, prob_as_exp=True)
        ctx.eng, ctx.dlogits, ctx.names, ctx.forward_id = eng, dlogits, names, eng.forward_id
        loss = res["loss"].clone().reshape(())
        vb = res["vb_loss"].clone()
        if prob is None:
            prob = torch.empty(0, device=dev)
        ctx.mark_non_differentiable(prob, vb, hits)
        return loss, prob, vb, hits

    @staticmethod
    def backward(ctx, gloss, gprob, gvb, ghits):
        if ctx.forward_id != ctx.eng.forward_id:
            raise RuntimeError("DiffusionTransformer: backward() of a loss whose activations were overwritten by a later forward(); the training "
                               "engine keeps one forward's activations (call loss.backward() before the next forward, as Solver.step does)")
        ctx.eng.backward_begin(ctx.dlogits, scale=gloss.detach().float().reshape(1).contiguous())
        grads = ctx.eng.backward_segment("head")
        return (None,) * 9 + (torch.zeros((), device=gloss.device),) + tuple(grads[n] for n in ctx.names)


class _SegmentGrad(torch.autograd.Function):
    """Autograd node of one backward segment ('tail' or ('layer', li)): forward only threads a scalar carrier through the chain (the actual forward
    pass runs inside _DenoiserLoss.forward, the last node); backward launches that segment of DenoiserTrainEngine's backward and returns its
    parameters' gradients."""

    @staticmethod
    def forward(ctx, eng, seg, names, carrier, *params):
        ctx.eng, ctx.seg, ctx.names, ctx.has_carrier = eng, seg, names, carrier is not None
        return params[0].new_zeros(()) if len(params) else torch.zeros(())

    @staticmethod
    def backward(ctx, g):
        grads = ctx.eng.backward_segment(ctx.seg)
        return (None, None, None, torch.zeros((), device=g.device) if ctx.has_carrier else None) + tuple(grads[n] for n in ctx.names)


def index_to_log_onehot(x, num_classes):
    """log(clamp(one_hot, 1e-30)) carrier (diffusion_transformer.py:45-56); memory-format plumbing only."""
    out = torch.full((x.shape[0], num_classes, x.shape[1]), float(np.log(np.float32(1e-30))), dtype=torch.float32, device=x.device)
    out.scatter_(1, x.unsqueeze(1), 0.0)
    return out
