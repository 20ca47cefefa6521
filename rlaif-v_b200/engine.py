"""DPO training-step engine: the public call a user makes for one optimisation step.

`DPOStepEngine.train_step(batch)` takes the reference collator's batch dict
(DataCollatorForDPODataset.__call__, muffin/train/train_muffin.py:43-112 — host tensors), copies
the step's inputs host->device, runs policy forward on chosen+rejected, the DPO loss + gradient
kernel, the hand-written backward, the (ZeRO-2) gradient reduction and the fused AdamW, and
returns the metrics of LLaVA15DPOTrainer.compute_loss (muffin/train/trainers.py:279-311).
"""
import os

import torch
import torch.distributed as dist

from . import lib as _lib
from . import ops
from .model import LlavaDPOPolicy
from .zero2 import OffloadAdamW, Zero2AdamW, cosine_lr

_F32 = torch.float32

METRIC_NAMES = ("loss", "rewards_train/chosen", "rewards_train/rejected", "rewards_train/accuracies",
                "rewards_train/margins", "logps_train/rejected", "logps_train/chosen",
                "logps_train/ref_rejected", "logps_train/ref_chosen")


class DPOStepEngine:
    def __init__(self, policy: LlavaDPOPolicy, lr=5e-7, weight_decay=0.01, betas=(0.9, 0.999), eps=1e-8,
                 total_steps=2672, warmup_ratio=0.05, dpo_use_average=False, micro_pairs=None,
                 rank=0, world=1, group=None, constant_lr=False, hf_deepspeed_input_cast=False,
                 dpo_token_weighted=False, offload_optimizer=False, offload_budget=None, batch_pairs=None,
                 optim="adamw_torch"):
        """optim: the optimizer state format, "adamw_torch" (fp32 moments) or "adamw_8bit" (blockwise 8-bit moments,
        zero2.state_format of --optim adamw_bnb_8bit / adamw_8bit)."""
        self.policy = policy
        self.rank, self.world, self.group = rank, world, group
        if offload_optimizer:
            # one GPU, full fine-tuning of a model whose fp32 optimizer state does not fit next to the weights,
            # gradients and activations: the state that does not fit is streamed from pinned host memory
            # (zero2.OffloadAdamW; DeepSpeed offload_optimizer.device = "cpu"). offload_budget: device bytes for
            # optimizer state. By default it is what is free after the activations of the micro-batch the step runs
            # (micro_pairs, else the whole per-device batch `batch_pairs`) at the model's maximum sequence length
            # (dims.max_len bounds T after the image-token splice) and the fp32 embedding-gradient buffer; the OmniLMM
            # policy adds its resampler and EVA tower (policy.activation_reserve_bytes).
            d = policy.dims
            reserve = 0
            if offload_budget is None:
                pairs = micro_pairs or batch_pairs
                if not pairs:
                    raise ValueError("offload_optimizer: the device budget is sized from the micro-batch; pass "
                                     "micro_pairs or batch_pairs (pairs per step), or an explicit offload_budget")
                reserve = policy.activation_reserve_bytes(pairs, d.max_len)
            self.opt = OffloadAdamW(policy.trainable_buckets(), lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                    rank=rank, world=world, group=group, gather_order=policy.param_need_order(),
                                    device_budget=offload_budget, activation_reserve=reserve, optim=optim)
        else:
            self.opt = Zero2AdamW(policy.trainable_buckets(), lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                  rank=rank, world=world, group=group, gather_order=policy.param_need_order(),
                                  optim=optim)
        self.base_lr, self.total_steps, self.warmup_ratio = lr, total_steps, warmup_ratio
        self.constant_lr = constant_lr
        self.dpo_use_average = dpo_use_average
        # --dpo_token_weighted (muffin/train/trainers.py:246-261): log-probs become token-weighted sums. The reference
        # refuses it for LLaVA-1.5 (:246-248: weights live in text positions, log-probs in spliced positions). Here the
        # LLaVA policy maps the weights through the splice (ops.splice_token_weight) and reduces the cached reference
        # per-token log-probs with the same spliced weights; it needs the collator's keep_spliced_per_token=True keys.
        self.dpo_token_weighted = dpo_token_weighted
        self._spliced_weights = dpo_token_weighted and policy.dims.frontend == "clip_mlp"
        self.micro_pairs = micro_pairs
        # HF Trainer._prepare_inputs casts every floating input to bf16 under DeepSpeed-bf16, which
        # rounds the reference log-probs (|logp| ~ 5e3 -> granularity 32) before dpo_loss. The drop-in
        # trainer (trainers.LLaVA15DPOTrainer) switches this on to reproduce the shipped recipe; the
        # engine itself takes get_beta_and_logps' inputs as they are.
        self.hf_deepspeed_input_cast = hf_deepspeed_input_cast
        self.global_step = 0
        self._metrics = torch.zeros(9, dtype=_F32, device=policy.device)
        self._last_micro = False
        self._stepping = False
        # ZeRO-2 overlap: reduce a layer's bucket as soon as its backward finished (last micro-batch only)
        policy.on_layer_grads_ready = self._layer_ready
        policy.on_head_grads_ready = self._head_ready
        if hasattr(policy, "on_bucket_grads_ready"):      # front-end buckets that finish inside the backward (EVA tower)
            policy.on_bucket_grads_ready = self._bucket_ready
        policy.param_ready = self.opt.wait_bucket

    def load_optimizer_state(self, sd):
        """Resume the optimizer from a state_dict of Zero2AdamW / OffloadAdamW. The policy may first refuse a checkpoint
        written for another set of trainable parameters with a message that names the mismatch (OmniLMM: trained vs
        frozen vision tower); the optimizer refuses any other size mismatch."""
        check = getattr(self.policy, "check_optimizer_state", None)
        if check is not None:
            check(sd, self.opt.owned, self.world)
        self.opt.load_state_dict(sd)

    def _layer_ready(self, layer):
        if self._last_micro:
            name = self.policy.layer_bucket_name(layer)
            self.opt.reduce_bucket(name)
            if self._stepping:            # gradients final, weights no longer read this step: update now,
                self.opt.step_bucket(name)    # overlapped with the rest of the backward

    def _bucket_ready(self, name):
        if self._last_micro and name not in self.policy.tail_bucket_names():
            self.opt.reduce_bucket(name)
            if self._stepping:
                self.opt.step_bucket(name)

    def _head_ready(self):
        if self._last_micro:
            self.opt.reduce_bucket("head")      # head bucket: final right after its backward
            if self._stepping:
                self.opt.step_bucket("head")

    def _h2d(self, t, dtype=None):
        if not t.is_cuda:
            if not t.is_pinned():
                t = t.pin_memory()
            t = t.to(self.policy.device, non_blocking=True)
        return t if dtype is None else t.to(dtype)

    def train_step(self, batch, optimizer_step=True):
        """batch: dict with concatenated_input_ids/labels [2B,L] (win rows first), images [B,3,S,S],
        ref_win_logp / ref_rej_logp [B] (or the *_avg_* variants when dpo_use_average), beta."""
        pol = self.policy
        _lib.bind_stream(torch.cuda.current_stream())
        try:
            return self._train_step(batch, optimizer_step)
        finally:
            _lib.bind_stream(None)

    def _train_step(self, batch, optimizer_step):
        pol = self.policy
        ids = self._h2d(batch["concatenated_input_ids"])
        labels = self._h2d(batch["concatenated_labels"])
        images = self._h2d(batch["images"])
        tw = ref_pt = None
        if self._spliced_weights:
            if "ref_win_per_token_logp_spliced" not in batch:
                raise KeyError("dpo_token_weighted on the LLaVA policy needs the un-truncated reference per-token "
                               "log-probs: DataCollatorForDPODataset(keep_spliced_per_token=True)")
            tw = self._h2d(batch["concatenated_token_weight"]).to(_F32).contiguous()       # [2B, L-1], text positions
            pw_, pr_ = batch["ref_win_per_token_logp_spliced"], batch["ref_rej_per_token_logp_spliced"]
            n = max(pw_.shape[1], pr_.shape[1])
            ref_pt = torch.zeros((2 * pw_.shape[0], n), dtype=_F32, device=pw_.device)
            ref_pt[: pw_.shape[0], : pw_.shape[1]] = pw_
            ref_pt[pw_.shape[0]:, : pr_.shape[1]] = pr_
            ref_pt = self._h2d(ref_pt)
            rw = rr = None
        elif self.dpo_token_weighted:
            from .trainers import compute_weighted_logp     # host tensors from the collator, [B, L-1] each
            rw = self._h2d(compute_weighted_logp(batch["ref_win_per_token_logp"], batch["win_labels"],
                                                 batch["win_token_weight"], self.dpo_use_average)).to(_F32)
            rr = self._h2d(compute_weighted_logp(batch["ref_rej_per_token_logp"], batch["rej_labels"],
                                                 batch["rej_token_weight"], self.dpo_use_average)).to(_F32)
            tw = self._h2d(batch["concatenated_token_weight"]).to(_F32).contiguous()       # [2B, L-1]
        else:
            key = "avg_logp" if self.dpo_use_average else "logp"
            rw = self._h2d(batch["ref_win_" + key]).to(_F32)
            rr = self._h2d(batch["ref_rej_" + key]).to(_F32)
        if self.hf_deepspeed_input_cast and rw is not None:
            rw = rw.to(torch.bfloat16).to(_F32)
            rr = rr.to(torch.bfloat16).to(_F32)
        beta = float(batch["beta"])
        B = images.shape[0]
        mp = self.micro_pairs or B
        sft_w = float(os.environ.get("SFT_weight", 0.0))     # muffin/train/trainers.py:299-300
        dpo_w = float(os.environ.get("DPO_weight", 1.0))
        self._metrics.zero_()
        self._stepping = bool(optimizer_step)
        if optimizer_step:
            lr = self.base_lr if self.constant_lr else cosine_lr(self.global_step, self.total_steps, self.base_lr,
                                                                 self.warmup_ratio)
            self.opt.begin_step(lr)
        n_micro = (B + mp - 1) // mp
        for mi in range(n_micro):
            lo, hi = mi * mp, min(B, (mi + 1) * mp)
            b = hi - lo
            self._last_micro = mi == n_micro - 1
            mids = torch.cat([ids[lo:hi], ids[B + lo:B + hi]], 0)
            mlab = torch.cat([labels[lo:hi], labels[B + lo:B + hi]], 0)
            out = pol.forward_logps(mids, mlab, images[lo:hi], keep_stash=True)
            lp = out["avg_logp"] if self.dpo_use_average else out["logp"]
            mtw = wsum = None
            mrw, mrr = (rw[lo:hi].contiguous(), rr[lo:hi].contiguous()) if rw is not None else (None, None)
            if tw is not None:
                mtw = torch.cat([tw[lo:hi], tw[B + lo:B + hi]], 0).contiguous()
                if self._spliced_weights:
                    T = out["T"]
                    mtw = ops.splice_token_weight(pol._stash["src"], mtw, T)              # text -> spliced positions
                    mref = torch.zeros((2 * b, T - 1), dtype=_F32, device=mtw.device)
                    n = min(T - 1, ref_pt.shape[1])
                    mref[:b, :n] = ref_pt[lo:hi, :n]
                    mref[b:, :n] = ref_pt[B + lo:B + hi, :n]
                    rlw, raw_, _ = ops.logp_weighted_reduce(mref, out["labels"], mtw)       # reference side, same weights
                    rsel = raw_ if self.dpo_use_average else rlw
                    mrw, mrr = rsel[:b].contiguous(), rsel[b:].contiguous()
                    if self.hf_deepspeed_input_cast:
                        mrw, mrr = mrw.to(torch.bfloat16).to(_F32), mrr.to(torch.bfloat16).to(_F32)
                lw, aw, wsum = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], mtw)
                lp = aw if self.dpo_use_average else lw
            _, _, _, dpw, dpr, out9 = ops.dpo_loss(lp[:b].contiguous(), lp[b:].contiguous(), mrw, mrr, beta, dpo_w, sft_w,
                                                   grad_scale=(b / B) / self.world)
            self._metrics.add_(out9, alpha=b / B)
            pol.backward_logps(torch.cat([dpw, dpr]).contiguous(), use_average=self.dpo_use_average,
                               accumulate=mi > 0, token_weight=mtw, weight_sum=wsum)
        pol.finalize_embed_grad()
        if self.world > 1:
            for name in pol.tail_bucket_names():
                self.opt.reduce_bucket(name)
        if optimizer_step:
            self.opt.finish_step()
            self.global_step += 1
            if pol.lora is not None:
                pol.lora.step = self.global_step
        return self._metrics

    def metrics_dict(self, metrics=None):
        """One small all-reduce + one D2H for the 9 scalars (the reference does 7 gathers + 7 syncs)."""
        m = (self._metrics if metrics is None else metrics).clone()
        if self.world > 1:
            dist.all_reduce(m, op=dist.ReduceOp.SUM, group=self.group)
            m /= self.world
        vals = m.tolist()
        return dict(zip(METRIC_NAMES, vals))
