"""Training entry point — drop-in for `muffin/train/train_llava15.py` (same flag names as
script/train/llava15_train.sh:6-48, same three argument groups, same train() flow):

    torchrun --nproc-per-node 8 -m rlaifv_b200.train_llava15 --deepspeed ./script/zero2.json \
        --model_name_or_path ... --data_dir ... --task DPO --dpo_beta 0.1 ...

Differences forced by the environment (SURVEY.md §8b "environment drift"): arguments are parsed by
a small dataclass parser instead of HfArgumentParser/transformers.TrainingArguments (which refuses
--deepspeed/--bf16 without `accelerate`), the launcher is torchrun (one process per GPU, NCCL)
instead of `deepspeed`, and `--deepspeed <json>` is read only for its ZeRO stage (2 = what this
engine implements natively) and `offload_optimizer.device` ("cpu": full fine-tuning on one GPU with
the optimizer state streamed from pinned host memory, script/zero2_offload.json).
"""
import argparse
import dataclasses
import glob
import json
import os
import pathlib
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.distributed as dist


@dataclass
class ModelArguments:                      # muffin/train/train_llava15.py:32-46
    model_name_or_path: Optional[str] = "facebook/opt-125m"
    version: Optional[str] = "llava_v1"
    freeze_backbone: bool = False
    tune_mm_mlp_adapter: bool = False
    vision_tower: Optional[str] = None
    mm_vision_select_layer: Optional[int] = -1
    pretrain_mm_mlp_adapter: Optional[str] = None
    mm_projector_type: Optional[str] = "linear"
    mm_use_im_start_end: bool = False
    mm_use_im_patch_token: bool = True
    mm_patch_merge_type: Optional[str] = "flat"
    mm_vision_select_feature: Optional[str] = "patch"


@dataclass
class DataArguments:                       # muffin/train/train_llava15.py:49-69
    lazy_preprocess: bool = False
    is_multimodal: bool = False
    image_token_len: int = 0
    image_folder: Optional[str] = None
    image_aspect_ratio: str = "square"
    parquet: bool = False
    data_source_names: str = "unimm-chat"
    data_source_weights: str = "100"
    eval_data_source_names: Optional[str] = None
    data_dir: str = "./RLAIF-V-Dataset/"
    kto_win_data_source_names: str = "100"
    kto_win_data_source_weights: str = "100"
    kto_rej_data_source_names: str = "100"
    kto_rej_data_source_weights: str = "100"
    dpo_beta: float = 0.5
    dpo_token_weight: float = 3.0
    shuffle_data: bool = True


@dataclass
class TrainingArguments:                   # muffin/train/train_llava15.py:72-100 + the HF fields the script sets
    output_dir: str = "./checkpoints"
    cache_dir: Optional[str] = None
    optim: str = "adamw_torch"
    remove_unused_columns: bool = False
    freeze_mm_mlp_adapter: bool = False
    force_fsdp: bool = False
    model_max_length: int = 512
    max_steps: int = 1000
    no_randaug: bool = False
    task: str = "LM"
    dpo_use_average: bool = False
    dpo_token_weighted: bool = False
    mm_projector_lr: Optional[float] = None
    group_by_modality_length: bool = False
    fully_tune: bool = False
    deepspeed: Optional[str] = None
    bf16: bool = False
    tf32: bool = False
    num_train_epochs: float = 3.0
    per_device_train_batch_size: int = 8
    per_device_eval_batch_size: int = 8
    gradient_accumulation_steps: int = 1
    evaluation_strategy: str = "no"
    save_strategy: str = "steps"
    save_steps: int = 500
    save_total_limit: Optional[int] = None
    learning_rate: float = 5e-5
    weight_decay: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_epsilon: float = 1e-8
    warmup_ratio: float = 0.0
    lr_scheduler_type: str = "linear"
    logging_steps: int = 500
    logging_dir: Optional[str] = None
    gradient_checkpointing: bool = False
    report_to: str = "none"
    run_name: Optional[str] = None
    dataloader_num_workers: int = 0
    seed: int = 42
    local_rank: int = -1
    micro_pairs: Optional[int] = None      # engine knob: pairs per micro-batch (None = whole batch)
    # decoder rows a preference pair shares (prompt + image up to the first response token) computed once
    share_prompt_prefix: bool = False
    # muffin/train/train_llava15_lora.py:112-117
    lora_enable: bool = False
    lora_r: int = 64
    lora_alpha: int = 16
    lora_dropout: float = 0.05
    lora_weight_path: Optional[str] = None
    lora_bias: str = "none"
    # the decoder's frozen base matrices in FP8 e4m3 (DESIGN.md §3 "FP8 frozen base"); needs --lora_enable True
    base_fp8: bool = False


def _add_fields(parser, cls):
    for f in dataclasses.fields(cls):
        typ = f.type
        base = typ.__args__[0] if getattr(typ, "__args__", None) else typ
        if base is bool:
            parser.add_argument("--" + f.name, type=lambda s: str(s).lower() in ("1", "true", "yes"),
                                nargs="?", const=True, default=f.default)
        else:
            parser.add_argument("--" + f.name, type=base, default=f.default)


def parse_args_into_dataclasses(argv=None):
    parser = argparse.ArgumentParser(allow_abbrev=False)
    for cls in (ModelArguments, DataArguments, TrainingArguments):
        _add_fields(parser, cls)
    ns, unknown = parser.parse_known_args(argv)
    if unknown:
        raise SystemExit("unknown arguments: %s" % unknown)
    out = []
    for cls in (ModelArguments, DataArguments, TrainingArguments):
        out.append(cls(**{f.name: getattr(ns, f.name) for f in dataclasses.fields(cls)}))
    return tuple(out)


def zero_stage(path):
    if not path:
        return 0
    with open(path) as f:
        return int(json.load(f).get("zero_optimization", {}).get("stage", 0))


def offload_optimizer(path):
    """DeepSpeed `zero_optimization.offload_optimizer.device` of the --deepspeed JSON: True for "cpu" (the optimizer
    state that does not fit on the GPU lives in pinned host memory, zero2.OffloadAdamW), False when absent or "none".
    "nvme" is not implemented."""
    if not path:
        return False
    with open(path) as f:
        block = json.load(f).get("zero_optimization", {}).get("offload_optimizer") or {}
    device = str(block.get("device", "none")).lower()
    if device == "nvme":
        raise NotImplementedError("offload_optimizer.device = nvme: only \"cpu\" (pinned host memory) is implemented")
    if device not in ("cpu", "none"):
        raise ValueError("offload_optimizer.device = %r: expected \"cpu\" or \"none\"" % device)
    return device == "cpu"


def safe_save_model_for_hf_trainer(trainer, output_dir):
    """muffin/train/train_llava15.py:102-112 — full state dict to CPU, saved by the main process.
    LoRA (train_llava15_lora.py:184-197): adapter weights + `non_lora_trainables.bin` (the projector)."""
    pol = trainer.model.policy
    if pol.lora is not None:
        if trainer.args.should_save:
            trainer.save_adapter(output_dir)
        return
    if trainer.args.should_save:
        trainer._save(output_dir, state_dict={k: v.cpu() for k, v in trainer.model.state_dict().items()})


def init_distributed():
    if "RANK" in os.environ and int(os.environ.get("WORLD_SIZE", "1")) > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    return int(os.environ.get("LOCAL_RANK", "0"))


def dims_from_checkpoint(model_dir, vision_tower_dir, select_layer, max_len):
    """LlavaDims from the checkpoint's config.json (+ the CLIP directory's config.json) — what
    `LlavaLlamaForCausalLM.from_pretrained` / `CLIPVisionModel.from_pretrained` read in the reference
    (muffin/train/train_llava15.py:206-214, llava/model/multimodal_encoder/clip_encoder.py:25-34).
    Missing files / keys fall back to the LLaVA-1.5-7B + CLIP-ViT-L/14-336 defaults."""
    from .model import LlavaDims
    kw = dict(select_layer=select_layer, max_len=max_len)

    def read(d):
        p = os.path.join(d, "config.json") if d and os.path.isdir(d) else None
        if p and os.path.exists(p):
            with open(p) as f:
                return json.load(f)
        return {}
    c = read(model_dir)
    for src, dst in (("vocab_size", "vocab_size"), ("hidden_size", "hidden_size"),
                     ("intermediate_size", "intermediate_size"), ("num_hidden_layers", "num_layers"),
                     ("num_attention_heads", "num_heads"), ("rms_norm_eps", "rms_eps"), ("rope_theta", "rope_theta")):
        if c.get(src) is not None:
            kw[dst] = c[src]
    if c.get("num_key_value_heads") and c["num_key_value_heads"] != c.get("num_attention_heads"):
        kw["num_kv_heads"] = c["num_key_value_heads"]
    v = read(vision_tower_dir)
    v = v.get("vision_config", v)
    for src, dst in (("hidden_size", "clip_hidden"), ("intermediate_size", "clip_intermediate"),
                     ("num_hidden_layers", "clip_layers"), ("num_attention_heads", "clip_heads"),
                     ("image_size", "image_size"), ("patch_size", "patch_size"), ("layer_norm_eps", "clip_eps")):
        if v.get(src) is not None:
            kw[dst] = v[src]
    return LlavaDims(**kw)


def check_base_fp8(training_args):
    if training_args.base_fp8 and not training_args.lora_enable:
        raise ValueError("--base_fp8 True needs --lora_enable True: the FP8 base is frozen and gets no gradient")


def init_model(model_args, data_args, training_args, attn_implementation=None, source_rows=None):
    """muffin/train/train_llava15.py:198-281: policy model (+ frozen reference used once for the
    log-prob pre-pass inside the dataset), tokenizer, data module."""
    from .llava_model import LlavaLlamaForCausalLM
    from .model import LlavaDims
    from .data import make_dpo_data_module, load_tokenizer, load_hf_checkpoint
    from .image_processing import ClipImageProcessor, PixelValues
    local_rank = init_distributed()
    dims = dims_from_checkpoint(model_args.model_name_or_path, model_args.vision_tower,
                                select_layer=model_args.mm_vision_select_layer,
                                max_len=training_args.model_max_length)
    check_base_fp8(training_args)
    state = load_hf_checkpoint(model_args.model_name_or_path, model_args.vision_tower)
    # the base's storage format is fixed when the model is built, before enable_lora
    model = LlavaLlamaForCausalLM(dims, torch.device("cuda", local_rank), hf_state=state,
                                  base_fp8=bool(training_args.base_fp8))
    model.config.use_cache = False
    model.policy.share_prefix = bool(training_args.share_prompt_prefix)
    if training_args.lora_enable:
        if training_args.lora_bias != "none":
            raise NotImplementedError("lora_bias=%r (the shipped recipe uses 'none')" % training_args.lora_bias)
        model.policy.enable_lora(r=training_args.lora_r, alpha=training_args.lora_alpha,
                                 dropout=training_args.lora_dropout)
        if training_args.lora_weight_path:                    # continue from a saved adapter
            ad = torch.load(os.path.join(training_args.lora_weight_path, "adapter_model.bin"), map_location="cpu")
            model.policy.lora.load_hf({k[len("base_model.model."):]: v for k, v in ad.items()})
    tokenizer = load_tokenizer(model_args.model_name_or_path, training_args.model_max_length)
    data_args.is_multimodal = True
    data_args.image_token_len = dims.num_patches
    # extension: --dpo_token_weighted on LLaVA-1.5 needs the un-truncated (spliced-position) reference per-token lists
    data_args.keep_spliced_per_token = bool(training_args.dpo_token_weighted)
    # muffin/train/train_llava15.py:244: `lambda x: vision_tower.image_processor(x)['pixel_values'][0]`
    data_args.image_processor = PixelValues(ClipImageProcessor.from_pretrained(model_args.vision_tower,
                                                                               dims.image_size))
    data_module = make_dpo_data_module(tokenizer=tokenizer, data_args=data_args, reference_model=model,
                                       source_rows=source_rows)
    return model, data_module, tokenizer


def train(attn_implementation=None, argv=None, source_rows=None):
    """`source_rows`: raw preference rows for the reference-log-prob pre-pass when `data_dir` holds no *logp* parquet
    yet (the reference downloads openbmb/RLAIF-V-Dataset from the hub at this point, muffin/data/datasets.py:38-50)."""
    model_args, data_args, training_args = parse_args_into_dataclasses(argv)
    data_args.data_source_names = data_args.data_source_names.split("#")
    data_args.data_source_weights = [int(x) for x in data_args.data_source_weights.split("#")]
    if data_args.eval_data_source_names is not None:
        data_args.eval_data_source_names = data_args.eval_data_source_names.split("#")
    if zero_stage(training_args.deepspeed) not in (0, 2):
        raise NotImplementedError("only ZeRO stage 2 (script/zero2.json) is implemented natively")
    training_args.offload_optimizer = offload_optimizer(training_args.deepspeed)
    if training_args.gradient_accumulation_steps != 1:
        # the shipped recipes use 1 (script/train/llava15_train.sh:33); inside one step the engine's own
        # --micro_pairs splits the per-device batch with gradient accumulation in the wgrad epilogues
        raise NotImplementedError("gradient_accumulation_steps=%d: use --micro_pairs to split the per-device batch"
                                  % training_args.gradient_accumulation_steps)
    model, data_module, tokenizer = init_model(model_args, data_args, training_args, attn_implementation, source_rows)
    if training_args.task != "DPO":
        raise NotImplementedError
    from .trainers import LLaVA15DPOTrainer
    training_args.model_name_or_path = model_args.model_name_or_path
    trainer = LLaVA15DPOTrainer(model=model, tokenizer=tokenizer, args=training_args, **data_module)
    if list(pathlib.Path(training_args.output_dir).glob("checkpoint-*")):
        print("Resume from checkpoint.")
        trainer.train(resume_from_checkpoint=True)
    else:
        print("Train from start.")
        trainer.train()
    trainer.save_state()
    safe_save_model_for_hf_trainer(trainer=trainer, output_dir=training_args.output_dir)
    return trainer


if __name__ == "__main__":
    train(attn_implementation="flash_attention_2")
