"""Training entry point for OmniLMM-12B / RLAIF-V-12B DPO (BASELINE config d; SURVEY.md §8 a13 / f3).

The reference ships no OmniLMM train script (SURVEY §8 a13: "no train script in tree"); the pieces it does ship fix the
contract this entry follows: the model (`OmniLMMForCausalLM`, omnilmm/model/omnilmm.py:268-346, `tune_clip=True`), the
generic `forward_DPO` branch of `get_beta_and_logps` (muffin/train/trainers.py:66-88, 233-261), the sample encoding
(`omni_preprocess`, omnilmm/train/train_utils.py:50-151, with `<im_start><im_patch>*64<im_end>` expansion), the image
transform (`build_transform`, omnilmm/model/utils.py:421-462), the preference collator and the parquet / cached
reference-log-prob dataset of the LLaVA recipe, and ZeRO (script/zero3.json for the 12B model).

    torchrun --nproc-per-node 8 -m rlaifv_b200.train_omnilmm --model_name_or_path <ckpt dir> --data_dir <parquet dir> \
        --task DPO --dpo_beta 0.1 --deepspeed ./script/zero3.json --bf16 True ...

Flags are those of train_llava15 (same three argument groups) plus --num_query / --image_size / --tune_clip.
`--tune_clip False` freezes the EVA tower as the reference does (it runs forward only and is never updated; the resampler
and the decoder train); the default `True` trains it.
ZeRO: `--deepspeed` may name a stage-2 or stage-3 config; the engine runs its native ZeRO-2 either way: the 23.5 GB of
bf16 parameters replicate on every GPU and the fp32 optimizer state is sharded. With the tower trained that is 11.7 B
trainable parameters: 23.5 GB of gradients and 141 GB of fp32 state, so at N = 4 each GPU holds 23.5 + 23.5 + 35 GB
before any activation, more than an 80 GB card; N = 8 leaves room (not measured). With `--tune_clip False` 7.3 B
parameters train (14.7 GB of gradients, 88 GB of state).
One GPU: `--deepspeed script/zero2_offload.json` keeps the fp32 state that does not fit in pinned host memory
(zero2.OffloadAdamW). The device budget subtracts the activation reserve of `--micro_pairs` pairs at
`--model_max_length` (decoder, resampler, the tower's working set and, when it trains, its stash; DESIGN.md §2). With
`--tune_clip False --micro_pairs 2 --model_max_length 1024` on an 80 GB H100, 59 GB of state is streamed and
MemAvailable must show 68 GB; with the tower trained (`--micro_pairs 1`) 117 GB is streamed and 126 GB is needed, which
the optimizer refuses up front where MemAvailable is smaller.
"""
import dataclasses
import json
import os
import pathlib
from dataclasses import dataclass
from types import SimpleNamespace

import torch
import torch.distributed as dist
from torch.utils.data import Dataset

from . import train_llava15 as T15


@dataclass
class OmniArguments:
    num_query: int = 64                 # omnilmm/model/omnilmm.py:46-51 (resampler queries = <im_patch> tokens per image)
    image_size: int = 448
    tune_clip: bool = True              # True: the tower is trained; False: frozen, forward only (omnilmm.py:57-70)


class OmniLMMForCausalLM:
    """Facade with the surface the trainer touches (policy, config, state_dict, train/eval)."""

    def __init__(self, dims, eva_dims, device="cuda", hf_state=None, seed=0, tune_clip=True):
        from .omnilmm_model import OmniLMMDPOPolicy
        self.dims = dims
        self.policy = OmniLMMDPOPolicy(dims, device, hf_state=hf_state, seed=seed, eva_dims=eva_dims,
                                       tune_clip=tune_clip)
        self.device, self.dtype, self.training = self.policy.device, torch.bfloat16, True
        self.config = SimpleNamespace(hidden_size=dims.hidden_size, vocab_size=dims.vocab_size,
                                      num_hidden_layers=dims.num_layers, num_attention_heads=dims.num_heads,
                                      num_key_value_heads=dims.kv_heads, intermediate_size=dims.intermediate_size,
                                      rms_norm_eps=dims.rms_eps, num_query=dims.num_query, image_size=eva_dims.img_size,
                                      mm_vision_tower="eva02_enormous_patch14_clip_224.laion2b_plus", use_cache=False)

    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def state_dict(self):
        for b in self.policy.trainable_buckets():
            self.policy._need(b.name)
        return self.policy.hf_views()

    def load_state_dict(self, state, strict=True):
        pol = self.policy
        pol.store.load_hf(state)
        pre = "model.resampler."
        pol.resampler.load_state_dict({k[len(pre):]: v for k, v in state.items() if k.startswith(pre)})
        pre = "model.vision_tower."
        pol.tower.load_timm_state({k[len(pre):]: v for k, v in state.items() if k.startswith(pre)})


class OmniDPODataset(Dataset):
    """Preference rows (parquet with cached reference log-probs, muffin/data/datasets.py contract) encoded for OmniLMM."""

    def __init__(self, tokenizer, data_dir, multimodal_cfg, reference_model=None, source_rows=None):
        from .data import RLAIFVDataset
        self.tokenizer, self.cfg = tokenizer, dict(multimodal_cfg, keep_image_tag=False)
        have = os.path.isdir(data_dir) and any(f.endswith(".parquet") and "logp" in f for f in os.listdir(data_dir))
        if not have:
            assert reference_model is not None and source_rows is not None, \
                "no *logp*.parquet in %s: pass the raw rows and a reference model for the log-prob pre-pass" % data_dir
            omni_inference_logp(reference_model, tokenizer, source_rows, data_dir, self.cfg)
        self.rows = RLAIFVDataset(data_dir, None, tokenizer)

    def __len__(self):
        return len(self.rows)

    def __getitem__(self, i):
        from .omnilmm_data import encode_omni_preference_sample
        return encode_omni_preference_sample(self.rows[i], self.tokenizer, self.cfg)


def omni_inference_logp(model, tokenizer, rows, cache_dir, cfg, batch_size=4):
    """Frozen-reference log-prob pre-pass (muffin/eval/muffin_inference_logp.py:213-344) for the OmniLMM policy: one
    fused forward per batch of pairs, same parquet contract as the LLaVA recipe."""
    from functools import partial
    from .collator import preference_collator_fn
    from .data import bytes_to_PIL_image, write_logp_to_preference_parquet
    from .omnilmm_data import encode_omni_preference_sample
    os.makedirs(cache_dir, exist_ok=True)
    rank = dist.get_rank() if dist.is_initialized() else 0
    world = dist.get_world_size() if dist.is_initialized() else 1
    mine = list(range(rank, len(rows), world))
    outs = {}
    collate = partial(preference_collator_fn, pad_token_id=tokenizer.pad_token_id)
    for lo in range(0, len(mine), batch_size):
        idx = mine[lo:lo + batch_size]
        inst = []
        for i in idx:
            s = rows[i]
            src = {"image": bytes_to_PIL_image(s["image"]["bytes"]),
                   "question": {"from": "human", "value": f"<image>\n{s['question']}"},
                   "chosen": {"from": "gpt", "value": s["chosen"]}, "rejected": {"from": "gpt", "value": s["rejected"]}}
            inst.append(encode_omni_preference_sample(src, tokenizer, cfg))
        b = collate(inst)
        res = model.policy.forward_logps(b["concatenated_input_ids"], b["concatenated_labels"], b["images"],
                                         keep_stash=False)
        pt, lp, av = res["per_token_logps"].float().cpu(), res["logp"].float().cpu(), res["avg_logp"].float().cpu()
        B = len(idx)
        for j, i in enumerate(idx):
            nw, nr = int(b["win_attention_mask"][j].sum()), int(b["rej_attention_mask"][j].sum())
            outs[i] = (float(lp[j]), float(av[j]), pt[j, : nw - 1].tolist(),
                       float(lp[B + j]), float(av[B + j]), pt[B + j, : nr - 1].tolist())
    if world > 1:
        gathered = [None] * world
        dist.all_gather_object(gathered, outs)
        outs = {k: v for g in gathered for k, v in g.items()}
    write_logp_to_preference_parquet(rows, cache_dir, [outs[i] for i in range(len(rows))], overwrite_logps=False)


def dims_from_config(model_dir, omni_args, max_len):
    from .eva_tower import EvaDims
    from .omnilmm_model import omnilmm_dims
    cfg = {}
    p = os.path.join(model_dir, "config.json") if model_dir and os.path.isdir(model_dir) else None
    if p and os.path.exists(p):
        with open(p) as f:
            cfg = json.load(f)
    kw = {}
    for src, dst in (("vocab_size", "vocab_size"), ("hidden_size", "hidden_size"), ("intermediate_size", "intermediate_size"),
                     ("num_hidden_layers", "num_layers"), ("num_attention_heads", "num_heads"),
                     ("num_key_value_heads", "num_kv_heads"), ("rms_norm_eps", "rms_eps"), ("rope_theta", "rope_theta"),
                     ("im_patch_token", "im_patch_token"), ("im_start_token", "im_start_token"),
                     ("im_end_token", "im_end_token")):
        if cfg.get(src) is not None:
            kw[dst] = cfg[src]
    v = cfg.get("vision_tower_config", {})
    dims = omnilmm_dims(num_query=cfg.get("num_query", omni_args.num_query), max_len=max_len,
                        vision_width=v.get("embed_dim", 1792), **kw)
    eva = EvaDims(embed_dim=v.get("embed_dim", 1792), depth=v.get("depth", 64), num_heads=v.get("num_heads", 16),
                  mlp_hidden=v.get("mlp_hidden", 15360), patch_size=v.get("patch_size", 14),
                  pretrain_img=v.get("pretrain_img", 224), img_size=cfg.get("image_size", omni_args.image_size))
    return dims, eva


def load_tokenizer(model_name_or_path, model_max_length):
    import transformers
    tok = transformers.AutoTokenizer.from_pretrained(model_name_or_path, model_max_length=model_max_length,
                                                     padding_side="right")
    from .omnilmm_data import DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN
    tok.add_tokens([DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN], special_tokens=True)   # chat.py:48-49
    return tok


def init_model(model_args, data_args, training_args, omni_args, source_rows=None):
    from .collator import DataCollatorForDPODataset
    from .data import load_hf_checkpoint
    from .image_processing import SquareResizeProcessor
    local_rank = T15.init_distributed()
    dims, eva = dims_from_config(model_args.model_name_or_path, omni_args, training_args.model_max_length)
    has_weights = os.path.isdir(model_args.model_name_or_path) and any(
        f.endswith((".bin", ".safetensors")) for f in os.listdir(model_args.model_name_or_path))
    state = load_hf_checkpoint(model_args.model_name_or_path) if has_weights else None
    tokenizer = load_tokenizer(model_args.model_name_or_path, training_args.model_max_length)
    if dims.im_patch_token < 0 or state is None:
        from .omnilmm_data import DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN
        ids = tokenizer.convert_tokens_to_ids([DEFAULT_IMAGE_PATCH_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IM_END_TOKEN])
        dims = dataclasses.replace(dims, im_patch_token=ids[0], im_start_token=ids[1], im_end_token=ids[2])
    model = OmniLMMForCausalLM(dims, eva, torch.device("cuda", local_rank), hf_state=state, tune_clip=omni_args.tune_clip)
    cfg = dict(is_multimodal=True, image_token_len=dims.num_query, use_im_start_end=True,
               image_processor=SquareResizeProcessor(eva.img_size))
    train = OmniDPODataset(tokenizer, data_args.data_dir, cfg, reference_model=model, source_rows=source_rows)
    print(f"Train data size is {len(train)}", flush=True)
    collator = DataCollatorForDPODataset(tokenizer=tokenizer, beta=data_args.dpo_beta,
                                         mod_token_weight=data_args.dpo_token_weight)
    return model, dict(train_dataset=train, eval_dataset=None, data_collator=collator), tokenizer


def train(argv=None, source_rows=None):
    import argparse
    parser = argparse.ArgumentParser(allow_abbrev=False)
    for cls in (T15.ModelArguments, T15.DataArguments, T15.TrainingArguments, OmniArguments):
        T15._add_fields(parser, cls)
    ns, unknown = parser.parse_known_args(argv)
    if unknown:
        raise SystemExit("unknown arguments: %s" % unknown)
    model_args, data_args, training_args, omni_args = (
        cls(**{f.name: getattr(ns, f.name) for f in dataclasses.fields(cls)})
        for cls in (T15.ModelArguments, T15.DataArguments, T15.TrainingArguments, OmniArguments))
    if training_args.task != "DPO":
        raise NotImplementedError
    if T15.zero_stage(training_args.deepspeed) not in (0, 2, 3):
        raise NotImplementedError("unsupported ZeRO stage")
    training_args.offload_optimizer = T15.offload_optimizer(training_args.deepspeed)
    model, data_module, tokenizer = init_model(model_args, data_args, training_args, omni_args, source_rows)
    from .trainers import LLaVA15DPOTrainer
    training_args.model_name_or_path = model_args.model_name_or_path
    trainer = LLaVA15DPOTrainer(model=model, tokenizer=tokenizer, args=training_args, **data_module)
    resume = bool(list(pathlib.Path(training_args.output_dir).glob("checkpoint-*")))
    print("Resume from checkpoint." if resume else "Train from start.")
    trainer.train(resume_from_checkpoint=resume or None)
    trainer.save_state()
    T15.safe_save_model_for_hf_trainer(trainer=trainer, output_dir=training_args.output_dir)
    return trainer


if __name__ == "__main__":
    train()
