"""Drop-in trainer glue: same names / signatures / return values as muffin/train/trainers.py.

  dpo_loss(...)                      muffin/train/trainers.py:91-126   -> CUDA dpo_loss kernel
  get_beta_and_logps(...)            muffin/train/trainers.py:161-275  -> fused policy forward (the seam)
  forward_DPO(...)                   muffin/train/trainers.py:66-88    -> generic branch (OmniLMM policy)
  compute_weighted_logp(...)         muffin/train/trainers.py:128-137  (--dpo_token_weighted)
  collect_preference_metrics(...)    muffin/train/trainers.py:140-158
  LLaVA15DPOTrainer.compute_loss     muffin/train/trainers.py:279-311  (textually the same flow)

The reference subclasses HF `Trainer` (unusable here: needs `accelerate`, and its loop would go
through DeepSpeed).  `LLaVA15DPOTrainer` below keeps the surface the reference entry point touches
(`train(resume_from_checkpoint=)`, `save_state`, `_save`, `log`, `args.should_save`,
`_get_train_sampler` = RandomSampler like ZephyrTrainer, `_nested_gather`) on a small loop that
drives DPOStepEngine: ZeRO-2 reduce-scatter, fused AdamW, cosine schedule, checkpoints.
`compute_loss` stays autograd-compatible: policy log-probs come from a torch.autograd.Function whose
backward launches the hand-written backward kernels.
"""
import glob
import json
import math
import os
import time

import torch
import torch.distributed as dist

from . import ops
from .engine import DPOStepEngine, METRIC_NAMES
from .zero2 import OffloadAdamW, state_format

_F32 = torch.float32


# ------------------------------------------------------------------------------------------------
class _PolicyLogps(torch.autograd.Function):
    """forward: fused policy forward -> logp_sum / logp_avg [2B]; backward: kernels fill ParamStore.grad."""

    @staticmethod
    def forward(ctx, anchor, policy, input_ids, labels, images, use_average):
        # (inside Function.forward grad mode is off: the anchor carries the caller's intent)
        out = policy.forward_logps(input_ids, labels, images, keep_stash=anchor.requires_grad)
        ctx.policy, ctx.use_average = policy, use_average
        return (out["avg_logp"] if use_average else out["logp"]).clone()

    @staticmethod
    def backward(ctx, d_logp):
        pol = ctx.policy
        pol.backward_logps(d_logp.to(_F32).contiguous(), use_average=ctx.use_average,
                           accumulate=getattr(pol, "_grad_accumulate", False))
        pol.finalize_embed_grad()
        return None, None, None, None, None, None


class _DPOLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pw, pr, rw, rr, beta):
        losses, cr, rj, dpw, dpr, _ = ops.dpo_loss(pw.contiguous(), pr.contiguous(), rw.to(_F32).contiguous(),
                                                   rr.to(_F32).contiguous(), beta)
        B = pw.numel()
        ctx.save_for_backward(dpw * B, dpr * B)     # kernel grads are d(mean)/d logp: undo the 1/B
        ctx.mark_non_differentiable(cr, rj)
        return losses, cr, rj

    @staticmethod
    def backward(ctx, g_losses, _g1, _g2):
        dpw, dpr = ctx.saved_tensors
        return g_losses * dpw, g_losses * dpr, None, None, None


def dpo_loss(policy_chosen_logps, policy_rejected_logps, reference_chosen_logps, reference_rejected_logps,
             beta, reference_free=False):
    """(losses, chosen_rewards, rejected_rewards), all [B] fp32."""
    if reference_free:
        # ref_logratios = 0 for the loss; the rewards still use the provided references (trainers.py:117-124)
        losses, cr, _ = _DPOLoss.apply(policy_chosen_logps, policy_rejected_logps, reference_chosen_logps,
                                       reference_chosen_logps, float(beta))
        rj = float(beta) * (policy_rejected_logps.detach() - reference_rejected_logps.to(policy_rejected_logps.device))
        return losses, cr, rj
    return _DPOLoss.apply(policy_chosen_logps, policy_rejected_logps, reference_chosen_logps,
                          reference_rejected_logps, float(beta))


def compute_weighted_logp(per_token_logp, labels, token_weight, use_average):
    """muffin/train/trainers.py:128-137, for host-side tensors (the frozen-reference per-token log-probs the collator
    delivers). The policy side of the token-weighted loss runs in the CUDA library (ops.logp_weighted_reduce /
    ops.logp_bwd(token_weight=...) through DPOStepEngine(dpo_token_weighted=True)); the reference — and this drop-in —
    raise NotImplementedError for LLaVA-1.5 (:246-248), the branch exists for the OmniLMM / MiniCPM-style models."""
    loss_mask = labels[:, 1:] != -100
    weighted_mask = token_weight * loss_mask
    logp = (per_token_logp * weighted_mask).sum(-1)
    if use_average:
        return logp / weighted_mask.sum(-1)
    return logp


class _PolicyPerTokenLogps(torch.autograd.Function):
    """forward: per-token log-probs [2B, T-1] (forward_DPO(token_weighted=True)); backward: an arbitrary per-token
    gradient is exactly the token-weighted backward with d_logp = 1 and token_weight = d_per_token."""

    @staticmethod
    def forward(ctx, anchor, policy, input_ids, labels, images):
        out = policy.forward_logps(input_ids, labels, images, keep_stash=anchor.requires_grad)
        ctx.policy = policy
        return out["per_token_logps"].clone()

    @staticmethod
    def backward(ctx, d_pt):
        pol = ctx.policy
        ones = torch.ones(d_pt.shape[0], dtype=_F32, device=d_pt.device)
        pol.backward_logps(ones, token_weight=d_pt.to(_F32).contiguous(),
                           accumulate=getattr(pol, "_grad_accumulate", False))
        pol.finalize_embed_grad()
        return None, None, None, None, None


def forward_DPO(model, input_ids, labels, attention_mask, images, **kwargs):
    """muffin/train/trainers.py:66-88 for a policy of this package (OmniLMMDPOPolicy: `images` = the vision tower's
    output tokens, B or — as the reference passes them, :190 — 2B of them): summed / averaged log-probs [2B], or the
    per-token log-probs [2B, L-1] with token_weighted=True; autograd-connected to the hand-written backward."""
    token_weighted = kwargs.pop("token_weighted", False)
    dpo_use_average = kwargs.pop("dpo_use_average", False)
    if kwargs.pop("is_minicpm", False):
        raise NotImplementedError("MiniCPM-V branch")
    if attention_mask is not None:
        raise NotImplementedError("attention_mask=None path only (muffin/train/trainers.py:199 sets it to None)")
    policy = model.policy if hasattr(model, "policy") else model
    anchor = torch.zeros((), device=policy.device, requires_grad=torch.is_grad_enabled())
    if token_weighted:
        return _PolicyPerTokenLogps.apply(anchor, policy, input_ids, labels, images)
    return _PolicyLogps.apply(anchor, policy, input_ids, labels, images, bool(dpo_use_average))


def get_beta_and_logps(data_dict, model, args, is_minicpm=False, is_llava15=False):
    """Same contract as the reference (muffin/train/trainers.py:161-275): pops the collator keys, returns
    (policy_win_logp, policy_rej_logp, ref_win_logp, ref_rej_logp, beta). is_llava15=True: LLaVA-1.5 policy;
    otherwise the generic `forward_DPO` branch (:233-261) on an OmniLMM policy, including --dpo_token_weighted."""
    if is_minicpm:
        raise NotImplementedError("MiniCPM-V branch")
    token_weighted = bool(getattr(args, "dpo_token_weighted", False))
    if token_weighted and is_llava15:
        raise NotImplementedError          # muffin/train/trainers.py:246-248 (is_llava15)
    if getattr(args, "task", "DPO") != "DPO":
        raise NotImplementedError("KTO task")
    win_input_ids = data_dict.pop("win_input_ids")
    rej_input_ids = data_dict.pop("rej_input_ids")
    win_labels, rej_labels = data_dict.pop("win_labels", None), data_dict.pop("rej_labels", None)
    ref_win_pt, ref_rej_pt = data_dict.pop("ref_win_per_token_logp", None), data_dict.pop("ref_rej_per_token_logp", None)
    win_tw, rej_tw = data_dict.pop("win_token_weight", None), data_dict.pop("rej_token_weight", None)
    cat_tw = data_dict.pop("concatenated_token_weight", None)
    for k in ("win_attention_mask", "rej_attention_mask", "concatenated_attention_mask"):
        data_dict.pop(k, None)
    ref_win_avg_logp = data_dict.pop("ref_win_avg_logp")
    ref_rej_avg_logp = data_dict.pop("ref_rej_avg_logp")
    ref_win_logp = data_dict.pop("ref_win_logp")
    ref_rej_logp = data_dict.pop("ref_rej_logp")
    if args.dpo_use_average:
        ref_win_logp, ref_rej_logp = ref_win_avg_logp, ref_rej_avg_logp
    beta = data_dict.pop("beta")
    images = data_dict.pop("images")
    ids = data_dict.pop("concatenated_input_ids")
    labels = data_dict.pop("concatenated_labels")
    policy = model.policy if hasattr(model, "policy") else model
    dev = policy.device
    if is_llava15 != (policy.dims.frontend == "clip_mlp"):
        raise ValueError("is_llava15=%s does not match the policy's vision front-end %r" % (is_llava15,
                                                                                             policy.dims.frontend))
    if is_llava15:
        anchor = torch.zeros((), device=dev, requires_grad=torch.is_grad_enabled())
        logp = _PolicyLogps.apply(anchor, policy, ids, labels, images, bool(args.dpo_use_average))
    else:
        logp = forward_DPO(model, ids, labels, None, images, token_weighted=token_weighted,
                           dpo_use_average=args.dpo_use_average)
        if token_weighted:                                  # trainers.py:246-261
            ua = bool(args.dpo_use_average)
            ref_win_logp = compute_weighted_logp(ref_win_pt, win_labels, win_tw, ua)
            ref_rej_logp = compute_weighted_logp(ref_rej_pt, rej_labels, rej_tw, ua)
            logp = compute_weighted_logp(logp, labels.to(dev), cat_tw.to(dev), ua)
    win_size, rej_size = win_input_ids.shape[0], rej_input_ids.shape[0]
    assert win_size == rej_size
    policy_win_logp, policy_rej_logp = logp.split([win_size, rej_size])
    return policy_win_logp, policy_rej_logp, ref_win_logp.to(dev), ref_rej_logp.to(dev), beta


def collect_preference_metrics(metrics, task, chosen_rewards, rejected_rewards, policy_rej_logp, policy_win_logp,
                               ref_rej_logp, ref_win_logp, reward_accuracies, preprocess_func):
    t = task
    m = {f"rewards_{t}/chosen": preprocess_func(chosen_rewards),
         f"rewards_{t}/rejected": preprocess_func(rejected_rewards),
         f"logps_{t}/rejected": preprocess_func(policy_rej_logp),
         f"logps_{t}/chosen": preprocess_func(policy_win_logp),
         f"logps_{t}/ref_rejected": preprocess_func(ref_rej_logp),
         f"logps_{t}/ref_chosen": preprocess_func(ref_win_logp),
         f"rewards_{t}/accuracies": preprocess_func(reward_accuracies)}
    m[f"rewards_{t}/margins"] = m[f"rewards_{t}/chosen"] - m[f"rewards_{t}/rejected"]
    return m


# ------------------------------------------------------------------------------------------------
class LLaVA15DPOTrainer:
    def __init__(self, model=None, tokenizer=None, args=None, train_dataset=None, eval_dataset=None,
                 data_collator=None):
        self.model, self.tokenizer, self.args = model, tokenizer, args
        self.train_dataset, self.eval_dataset, self.data_collator = train_dataset, eval_dataset, data_collator
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        a = args
        self.engine = DPOStepEngine(model.policy, lr=a.learning_rate, weight_decay=a.weight_decay,
                                    betas=(getattr(a, "adam_beta1", 0.9), getattr(a, "adam_beta2", 0.999)),
                                    eps=getattr(a, "adam_epsilon", 1e-8), total_steps=max(1, a.max_steps),
                                    warmup_ratio=a.warmup_ratio, dpo_use_average=a.dpo_use_average,
                                    dpo_token_weighted=bool(getattr(a, "dpo_token_weighted", False)),
                                    micro_pairs=getattr(a, "micro_pairs", None), rank=self.rank, world=self.world,
                                    offload_optimizer=bool(getattr(a, "offload_optimizer", False)),
                                    batch_pairs=getattr(a, "per_device_train_batch_size", None),
                                    optim=state_format(getattr(a, "optim", "adamw_torch")),
                                    hf_deepspeed_input_cast=bool(getattr(a, "bf16", True) and getattr(a, "deepspeed", None)),
                                    constant_lr=getattr(a, "lr_scheduler_type", "cosine") == "constant")
        self.state = {"global_step": 0, "log_history": []}
        if not hasattr(a, "should_save"):
            a.should_save = self.rank == 0
        if not hasattr(a, "past_index"):
            a.past_index = -1

    # ---- HF-Trainer surface used by the reference ----
    def _get_train_sampler(self, *unused):
        if self.train_dataset is None or not hasattr(self.train_dataset, "__len__"):
            return None
        g = torch.Generator().manual_seed(int(getattr(self.args, "seed", 42)))
        return torch.utils.data.RandomSampler(self.train_dataset, generator=g)     # ZephyrTrainer, trainers.py:45-51

    def _nested_gather(self, x):
        if self.world == 1:
            return x.reshape(1)
        out = [torch.zeros_like(x) for _ in range(self.world)]
        dist.all_gather(out, x)
        return torch.stack(out)

    def log(self, logs):
        logs = dict(logs)
        logs["step"] = self.state["global_step"]
        self.state["log_history"].append(logs)
        if self.rank == 0:
            print(json.dumps({k: (round(v, 6) if isinstance(v, float) else v) for k, v in logs.items()}), flush=True)

    def compute_loss(self, model, inputs, return_outputs=False):
        if self.args.past_index >= 0:
            raise NotImplementedError

        def gather_and_do_mean(x):
            return self._nested_gather(x.mean()).mean().item()

        data_dict = inputs
        policy_win_logp, policy_rej_logp, ref_win_logp, ref_rej_logp, beta = get_beta_and_logps(
            data_dict, model, self.args, is_llava15=True)
        losses, chosen_rewards, rejected_rewards = dpo_loss(policy_win_logp, policy_rej_logp, ref_win_logp,
                                                            ref_rej_logp, beta=beta)
        reward_accuracies = (chosen_rewards > rejected_rewards).float()
        SFT_weight = float(os.environ.get("SFT_weight", 0.0))
        DPO_weight = float(os.environ.get("DPO_weight", 1.0))
        loss = DPO_weight * losses.mean() - SFT_weight * policy_win_logp.mean()
        t = "train" if model.training else "test"
        metrics = collect_preference_metrics({}, t, chosen_rewards, rejected_rewards, policy_rej_logp.detach(),
                                             policy_win_logp.detach(), ref_rej_logp, ref_win_logp, reward_accuracies,
                                             gather_and_do_mean)
        self.log(metrics)
        return loss

    # ---- training loop ----
    def training_step(self, model, inputs):
        """Fused path: forward + DPO loss/grad kernel + backward + reduce-scatter + AdamW."""
        return self.engine.train_step(inputs)

    def _dataloader(self, epoch=0):
        """One epoch's loader; the shuffle is a pure function of (seed, epoch) so that a resumed run replays the
        order of the interrupted one."""
        a = self.args
        sampler = self._get_train_sampler()
        seed = int(getattr(a, "seed", 42)) + epoch
        if self.world > 1 and sampler is not None:
            sampler = torch.utils.data.distributed.DistributedSampler(self.train_dataset, self.world, self.rank,
                                                                      shuffle=True, seed=seed)
        elif isinstance(sampler, torch.utils.data.RandomSampler):
            sampler.generator = torch.Generator().manual_seed(seed)
        return torch.utils.data.DataLoader(self.train_dataset, batch_size=a.per_device_train_batch_size,
                                           sampler=sampler, collate_fn=self.data_collator,
                                           num_workers=getattr(a, "dataloader_num_workers", 0), drop_last=True,
                                           pin_memory=True)

    def _steps_per_epoch(self):
        """Batches one epoch's loader yields on this rank: DistributedSampler (drop_last=False) pads every rank to
        ceil(len / world) samples, the DataLoader then drops the ragged last batch."""
        if not hasattr(self.train_dataset, "__len__"):
            return 1 << 60
        n = len(self.train_dataset)
        if self.world > 1:
            n = -(-n // self.world)
        return n // self.args.per_device_train_batch_size

    def train(self, resume_from_checkpoint=None):
        a = self.args
        if resume_from_checkpoint:
            self._load_checkpoint(a.output_dir)
        self.model.train()
        step = self.state["global_step"]
        self.engine.global_step = step
        pol = self.model.policy
        if pol.lora is not None:
            # LoRA dropout streams are a function of (optimisation step, forward count): restore both so a resumed
            # run draws the masks the uninterrupted run would have drawn
            pol.lora.step = step
            pol._fwd_count = self.state.get("fwd_count", pol._fwd_count)
        t0 = time.time()
        while step < a.max_steps:
            loader = self._dataloader(epoch=step // max(1, self._steps_per_epoch()))
            skip = step % max(1, self._steps_per_epoch())       # batches of this epoch consumed before a resume
            for bi, batch in enumerate(loader):
                if bi < skip:
                    continue
                m = self.training_step(self.model, batch)
                step += 1
                self.state["global_step"] = step
                self.state["fwd_count"] = self.model.policy._fwd_count
                if a.logging_steps and step % a.logging_steps == 0:
                    logs = self.engine.metrics_dict(m)
                    logs["learning_rate"] = self.engine.opt._lr       # the rate begin_step() was given this step
                    logs["elapsed_s"] = time.time() - t0
                    self.log(logs)
                if getattr(a, "save_strategy", "no") == "steps" and a.save_steps and step % a.save_steps == 0:
                    self._save_checkpoint(os.path.join(a.output_dir, f"checkpoint-{step}"))
                if step >= a.max_steps:
                    break
        return self.state

    # ---- checkpoints ----
    def _write_config(self, output_dir):
        """`config.json` next to the weights (HF `save_pretrained` does this for the reference; the LoRA run script
        copies it into every checkpoint dir, script/train/llava15_train_lora.sh:51-69)."""
        cfg = dict(vars(self.model.config))
        cfg.update(model_type="llava_llama", architectures=["LlavaLlamaForCausalLM"], torch_dtype="bfloat16")
        with open(os.path.join(output_dir, "config.json"), "w") as f:
            json.dump(cfg, f, indent=1)

    def save_adapter(self, output_dir):
        """LoRA run: peft-layout adapter (`adapter_model.bin` + `adapter_config.json`) and the non-LoRA trainables
        (`non_lora_trainables.bin` = mm_projector), muffin/train/train_llava15_lora.py:184-197 — what
        llava/model/builder.py:52-86 loads back."""
        pol = self.model.policy
        os.makedirs(output_dir, exist_ok=True)
        if pol.param_ready is not None:                       # pending ZeRO-2 all-gathers of the last step
            for b in pol.lora.buckets:
                pol.param_ready(b.name)
        torch.cuda.synchronize()
        ad = {"base_model.model." + k: v.cpu() for k, v in pol.lora.hf_views().items()}
        torch.save(ad, os.path.join(output_dir, "adapter_model.bin"))
        with open(os.path.join(output_dir, "adapter_config.json"), "w") as f:
            json.dump({"peft_type": "LORA", "r": pol.lora.r, "lora_alpha": pol.lora.scaling * pol.lora.r,
                       "lora_dropout": pol.lora.dropout, "bias": "none", "task_type": "CAUSAL_LM",
                       "base_model_name_or_path": getattr(self.args, "model_name_or_path", None),
                       "target_modules": ["q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj",
                                          "down_proj"]}, f, indent=1)
        non_lora = {"base_model.model." + k: v.cpu() for k, v in self.model.state_dict().items()
                    if "mm_projector" in k}
        torch.save(non_lora, os.path.join(output_dir, "non_lora_trainables.bin"))
        self._write_config(output_dir)

    def load_adapter(self, path):
        pol = self.model.policy
        ad = torch.load(os.path.join(path, "adapter_model.bin"), map_location="cpu")
        pol.lora.load_hf({k[len("base_model.model."):]: v for k, v in ad.items()})
        nl = torch.load(os.path.join(path, "non_lora_trainables.bin"), map_location="cpu")
        views = pol.store.hf_views()
        for k, v in nl.items():
            views[k[len("base_model.model."):]].copy_(v)

    def _save(self, output_dir, state_dict=None):
        os.makedirs(output_dir, exist_ok=True)
        if self.model.policy.lora is not None and state_dict is None:
            self.save_adapter(output_dir)                      # frozen base weights are not rewritten
            return
        sd = state_dict if state_dict is not None else {k: v.cpu() for k, v in self.model.state_dict().items()}
        torch.save(sd, os.path.join(output_dir, "pytorch_model.bin"))
        self._write_config(output_dir)

    def save_state(self):
        if self.args.should_save:
            os.makedirs(self.args.output_dir, exist_ok=True)
            with open(os.path.join(self.args.output_dir, "trainer_state.json"), "w") as f:
                json.dump(self.state, f)

    def _save_checkpoint(self, path):
        # every rank writes its optimizer shard: the tail buckets' reduce-scatter wait / AdamW / all-gather of the
        # last step may still be queued on the optimizer side stream — drain them first on ALL ranks
        self.engine.opt.wait_all()
        torch.cuda.synchronize()
        os.makedirs(path, exist_ok=True)
        if self.args.should_save:
            self._save(path)
            with open(os.path.join(path, "trainer_state.json"), "w") as f:
                json.dump(self.state, f)
        torch.save(self.engine.opt.state_dict(), os.path.join(path, f"optimizer_rank{self.rank}.pt"))
        if self.world > 1:
            dist.barrier()        # pruning / a resume must never see a half-written checkpoint
        limit = getattr(self.args, "save_total_limit", None)
        if limit and self.args.should_save:
            ck = sorted(glob.glob(os.path.join(self.args.output_dir, "checkpoint-*")),
                        key=lambda p: int(p.rsplit("-", 1)[1]))
            for old in ck[:-limit]:
                for fn in os.listdir(old):
                    os.remove(os.path.join(old, fn))
                os.rmdir(old)

    def _load_checkpoint(self, output_dir):
        ck = sorted(glob.glob(os.path.join(output_dir, "checkpoint-*")), key=lambda p: int(p.rsplit("-", 1)[1]))
        if not ck:
            return
        path = ck[-1]
        if self.model.policy.lora is not None:
            self.load_adapter(path)
        else:
            self.model.load_state_dict(torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu"))
        # an offloaded optimizer's state does not fit on the device: load it on the host and let it place the parts
        offloaded = isinstance(self.engine.opt, OffloadAdamW)
        self.engine.load_optimizer_state(torch.load(os.path.join(path, f"optimizer_rank{self.rank}.pt"),
                                                    map_location="cpu" if offloaded else self.model.device))
        with open(os.path.join(path, "trainer_state.json")) as f:
            self.state = json.load(f)
