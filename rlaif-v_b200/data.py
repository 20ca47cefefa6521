"""Host-side data path of the DPO step, interface-compatible with the reference:

  tokenizer_image_token / preprocess_v1 / encode_multimodal_preference_sample
                                  muffin/train/train_utils.py:176-349 (llava_v1 template, label masking)
  RLAIFVDataset                   muffin/data/datasets.py:27-91   (parquet rows with cached ref log-probs)
  DPODataset / make_dpo_data_module   muffin/train/train_llava15.py:124-195
  PreferenceInferenceDataset / InferenceSampler / get_multimodal_sample_logps /
  write_logp_to_preference_parquet / inference_logp
                                  muffin/eval/muffin_inference_logp.py:55-79,117-164,213-344
      — the frozen-reference log-prob pre-pass (SURVEY.md §8f-1).  Here it runs on the same H100
        forward kernels as training: win and rej of a pair in ONE forward sharing the encoded image
        (the reference runs 2 forwards per pair and encodes the image twice), batched, and writes the
        identical on-disk contract: column `logps` = json.dumps({'logps': [win_sum, win_avg,
        win_per_tok[], rej_sum, rej_avg, rej_per_tok[]]}), files
        `RLAIF-V-Dataset-withlogp_{idx:03}-{n}.parquet` of 5000 rows.

Everything here is Python on the host (strings, token lists, parquet I/O); the arithmetic is in
the policy's kernels.
"""
import copy
import io
import itertools
import json
import os
from functools import partial

import torch
import torch.distributed as dist
from torch.utils.data import Dataset

from .collator import DataCollatorForDPODataset, preference_collator_fn

IGNORE_INDEX = -100
IMAGE_TOKEN_INDEX = -200
DEFAULT_IMAGE_TOKEN = "<image>"

LLAVA_V1_SYSTEM = ("A chat between a curious human and an artificial intelligence assistant. "
                   "The assistant gives helpful, detailed, and polite answers to the human's questions.")
LLAVA_V1_ROLES = ("USER", "ASSISTANT")
LLAVA_V1_SEP, LLAVA_V1_SEP2 = " ", "</s>"


def llava_v1_prompt(messages):
    """SeparatorStyle.TWO prompt of conv_llava_v1 (muffin/conversation.py:54-63, :325-335)."""
    seps = (LLAVA_V1_SEP, LLAVA_V1_SEP2)
    out = LLAVA_V1_SYSTEM + seps[0]
    for i, (role, msg) in enumerate(messages):
        out += (role + ": " + msg + seps[i % 2]) if msg else (role + ":")
    return out


def tokenizer_image_token(prompt, tokenizer, image_token_index=IMAGE_TOKEN_INDEX, return_tensors=None):
    chunks = [tokenizer(c).input_ids for c in prompt.split(DEFAULT_IMAGE_TOKEN)]
    ids, offset = [], 0
    if chunks and chunks[0] and chunks[0][0] == tokenizer.bos_token_id:
        offset = 1
        ids.append(chunks[0][0])
    for i, c in enumerate(chunks):
        if i > 0:
            ids.append(image_token_index)        # one -200 per <image> tag, between the text chunks
        ids.extend(c[offset:])
    if return_tensors == "pt":
        return torch.tensor(ids, dtype=torch.long)
    if return_tensors is not None:
        raise ValueError(f"Unsupported tensor type: {return_tensors}")
    return ids


def preprocess_v1(sources, tokenizer, has_image=False):
    """llava_v1 template + label masking: only assistant turns are supervised."""
    role_of = {"human": LLAVA_V1_ROLES[0], "gpt": LLAVA_V1_ROLES[1]}
    convs = []
    for src in sources:
        if role_of[src[0]["from"]] != LLAVA_V1_ROLES[0]:
            src = src[1:]
        msgs = []
        for j, s in enumerate(src):
            assert role_of[s["from"]] == LLAVA_V1_ROLES[j % 2]
            msgs.append((role_of[s["from"]], s["value"]))
        convs.append(llava_v1_prompt(msgs))
    if has_image:
        input_ids = torch.stack([tokenizer_image_token(c, tokenizer, return_tensors="pt") for c in convs], 0)
        count = lambda text: len(tokenizer_image_token(text, tokenizer))          # noqa: E731
    else:
        input_ids = tokenizer(convs, return_tensors="pt", padding="longest", max_length=tokenizer.model_max_length,
                              truncation=True).input_ids
        count = lambda text: len(tokenizer(text).input_ids)                       # noqa: E731
    targets = input_ids.clone()
    sep = LLAVA_V1_SEP + LLAVA_V1_ROLES[1] + ": "
    legacy = getattr(tokenizer, "legacy", True)
    for conv, tgt in zip(convs, targets):
        total = int(tgt.ne(tokenizer.pad_token_id).sum())
        cur = 1
        tgt[:cur] = IGNORE_INDEX
        for i, rnd in enumerate(conv.split(LLAVA_V1_SEP2)):
            if rnd == "":
                break
            parts = rnd.split(sep)
            if len(parts) != 2:
                break
            round_len = count(rnd)
            instr_len = count(parts[0] + sep) - 2
            if i != 0 and not legacy:
                round_len -= 1
                instr_len -= 1
            tgt[cur:cur + instr_len] = IGNORE_INDEX
            cur += round_len
        tgt[cur:] = IGNORE_INDEX
        if cur < tokenizer.model_max_length and cur != total:
            tgt[:] = IGNORE_INDEX
            print(f"WARNING: tokenization mismatch: {cur} vs. {total}. (ignored)")
    return {"input_ids": input_ids, "labels": targets}


def encode_multimodal_preference_sample(source, tokenizer, multimodal_cfg, preprocess_func=None):
    """-> (rej_dict, win_dict) with input_ids, labels, image and the cached reference log-probs."""
    if isinstance(source["chosen"], list):
        win_conv, rej_conv = source["chosen"], source["rejected"]
    else:
        win_conv = copy.deepcopy([source["question"], source["chosen"]])
        rej_conv = copy.deepcopy([source["question"], source["rejected"]])
    fn = preprocess_func or partial(preprocess_v1, has_image=True)
    image = multimodal_cfg["image_processor"](source["image"]) if "image" in source else None
    out = []
    for conv in (rej_conv, win_conv):
        enc = fn([conv], tokenizer)
        out.append({"input_ids": enc["input_ids"][0], "labels": enc["labels"][0]})
    rej, win = out
    if image is not None:
        rej["image"] = win["image"] = image
    elif multimodal_cfg.get("is_multimodal"):
        cs = multimodal_cfg["image_processor"].crop_size
        rej["image"] = win["image"] = torch.zeros(3, cs["height"], cs["width"])
    if "ref_win_logp" in source:
        for k in ("logp", "avg_logp", "per_token_logp"):
            rej[f"ref_rej_{k}"] = source[f"ref_rej_{k}"]
            win[f"ref_win_{k}"] = source[f"ref_win_{k}"]
    return rej, win


def bytes_to_PIL_image(buf):
    from PIL import Image
    return Image.open(io.BytesIO(buf)).convert("RGB")


def _load_parquet_dir(data_dir):
    import pyarrow.parquet as pq
    files = sorted(f for f in os.listdir(data_dir) if f.endswith(".parquet"))
    tables = [pq.read_table(os.path.join(data_dir, f)) for f in files]
    rows = []
    for t in tables:
        rows.extend(t.to_pylist())
    return rows


class RLAIFVDataset(Dataset):
    """Rows of the preference parquet(s) with cached reference log-probs; runs the pre-pass if absent."""

    def __init__(self, data_dir, reference_model=None, tokenizer=None, image_token_len=None, img_processor=None,
                 use_im_start_end=True, is_llava15=False, source_rows=None):
        os.makedirs(data_dir, exist_ok=True)
        have = [f for f in os.listdir(data_dir) if f.endswith(".parquet") and "logp" in f]
        if not have:
            assert reference_model is not None, "`reference_model` is mandatory when logps do not exist."
            if source_rows is None:
                raise FileNotFoundError("no *logp*.parquet in %s and no source rows given (the HF hub dataset "
                                        "openbmb/RLAIF-V-Dataset cannot be downloaded offline)" % data_dir)
            inference_logp(reference_model, tokenizer, source_rows, data_dir, image_token_len, img_processor,
                           use_im_start_end, is_llava15=is_llava15)
            if dist.is_initialized():
                dist.barrier()
        self.data = _load_parquet_dir(data_dir)
        self.line_idx = list(range(len(self.data)))

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        s = self.data[self.line_idx[index]]
        d = {"image": bytes_to_PIL_image(s["image"]["bytes"]),
             "question": {"from": "human", "value": f"<image>\n{s['question']}"},
             "chosen": {"from": "gpt", "value": s["chosen"]},
             "rejected": {"from": "gpt", "value": s["rejected"]},
             "idx": s["idx"],
             "metainfo": {"origin_dataset": s.get("origin_dataset"), "origin_split": s.get("origin_split"),
                          "origin_idx": s["idx"], "image_id": s.get("image_path")}}
        logps = json.loads(s["logps"])
        vals = logps if isinstance(logps, list) else logps["logps"]
        (d["ref_win_logp"], d["ref_win_avg_logp"], d["ref_win_per_token_logp"],
         d["ref_rej_logp"], d["ref_rej_avg_logp"], d["ref_rej_per_token_logp"]) = vals
        return d


class DPODataset(Dataset):
    def __init__(self, tokenizer, data_dir, multimodal_cfg, reference_model=None, source_rows=None):
        self.tokenizer = tokenizer
        self.list_data_dict = RLAIFVDataset(data_dir, reference_model, tokenizer, multimodal_cfg["image_token_len"],
                                            multimodal_cfg["image_processor"], multimodal_cfg["use_im_start_end"],
                                            is_llava15=True, source_rows=source_rows)
        self.multimodal_cfg = dict(multimodal_cfg, keep_image_tag=True)

    def __len__(self):
        return len(self.list_data_dict)

    def __getitem__(self, i):
        return encode_multimodal_preference_sample(self.list_data_dict[i], self.tokenizer, self.multimodal_cfg,
                                                   preprocess_func=partial(preprocess_v1, has_image=True))


def make_dpo_data_module(tokenizer, data_args, reference_model, source_rows=None):
    cfg = dict(is_multimodal=data_args.is_multimodal, image_token_len=data_args.image_token_len,
               image_folder=data_args.image_folder, image_aspect_ratio=data_args.image_aspect_ratio,
               use_im_start_end=getattr(data_args, "mm_use_im_start_end", False),
               image_processor=getattr(data_args, "image_processor", None),
               data_source_names=data_args.data_source_names, data_source_weights=data_args.data_source_weights,
               shuffle_data=data_args.shuffle_data)
    train = DPODataset(tokenizer, data_args.data_dir, cfg, reference_model, source_rows)
    print(f"Train data size is {len(train)}", flush=True)
    collator = DataCollatorForDPODataset(tokenizer=tokenizer, beta=data_args.dpo_beta,
                                         mod_token_weight=data_args.dpo_token_weight,
                                         keep_spliced_per_token=bool(getattr(data_args, "keep_spliced_per_token", False)))
    return dict(train_dataset=train, eval_dataset=None, data_collator=collator)


# ------------------------------------------------------------------------------------------------
# frozen-reference log-prob pre-pass
# ------------------------------------------------------------------------------------------------
class InferenceSampler(torch.utils.data.sampler.Sampler):
    """Contiguous shard of [0, size) per rank (muffin/eval/muffin_inference_logp.py:55-79)."""

    def __init__(self, size):
        self._size = int(size)
        rank = dist.get_rank() if dist.is_initialized() else 0
        world = dist.get_world_size() if dist.is_initialized() else 1
        per, rem = divmod(self._size, world)
        sizes = [per + (r < rem) for r in range(world)]
        begin = sum(sizes[:rank])
        self._local_indices = range(begin, min(begin + sizes[rank], self._size))

    def __iter__(self):
        yield from self._local_indices

    def __len__(self):
        return len(self._local_indices)


class PreferenceInferenceDataset(Dataset):
    def __init__(self, data, tokenizer, image_token_len, img_processor, use_im_start_end=True):
        self.data = data
        self.tokenizer = tokenizer
        self.mm_cfg = {"image_token_len": image_token_len, "is_multimodal": True, "use_im_start_end": use_im_start_end,
                       "image_processor": img_processor, "keep_image_tag": True}

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        s = self.data[index]
        src = {"image": bytes_to_PIL_image(s["image"]["bytes"]),
               "question": {"from": "human", "value": f"<image>\n{s['question']}"},
               "chosen": {"from": "gpt", "value": s["chosen"]},
               "rejected": {"from": "gpt", "value": s["rejected"]}, "idx": s["idx"]}
        return encode_multimodal_preference_sample(src, self.tokenizer, self.mm_cfg,
                                                   preprocess_func=partial(preprocess_v1, has_image=True))


def get_multimodal_sample_logps(model, dataloader, tokenizer=None, is_llava15=True):
    """-> six lists (win sum/avg/per-token, rej sum/avg/per-token). One fused forward per batch of pairs."""
    policy = model.policy if hasattr(model, "policy") else model
    outs = [[] for _ in range(6)]
    for batch in dataloader:
        B = batch["win_input_ids"].shape[0]
        res = policy.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"],
                                   keep_stash=False)
        per_tok = res["per_token_logps"].float().cpu()
        logp, avg = res["logp"].float().cpu(), res["avg_logp"].float().cpu()
        T = res["T"]
        P = policy.dims.num_patches
        for i in range(B):
            for kind, row, base in (("win", i, 0), ("rej", B + i, 3)):
                # per-token list of the un-padded sequence, as the reference's batch-size-1 pass yields it
                n = int(batch[f"{kind}_attention_mask"][i].sum()) if f"{kind}_attention_mask" in batch else T
                has_img = bool((batch[f"{kind}_input_ids"][i] == IMAGE_TOKEN_INDEX).any())
                t_len = min(n - 1 + P, policy.dims.max_len) if has_img else n
                outs[base].append(float(logp[row]))
                outs[base + 1].append(float(avg[row]))
                outs[base + 2].append(per_tok[row, : t_len - 1].tolist())
    return tuple(outs)


def write_logp_to_preference_parquet(origin_data, cache_file, logps, overwrite_logps=False):
    import pandas as pd
    rows = []
    for i in range(len(logps)):
        line = dict(origin_data[i])
        if "logps" in line:
            assert overwrite_logps, "Found existing logp data, pass overwrite_logps=True to force overwritting"
        else:
            assert all(k in line for k in ("question", "chosen", "rejected")), \
                f"Undefined data structure, expecting [Q, Win, Rej] in keys, got {line.keys()}"
        line["logps"] = json.dumps({"logps": logps[i]})
        rows.append(line)
    if not dist.is_initialized() or dist.get_rank() == 0:
        step = 5000
        for idx, start in enumerate(range(0, len(rows), step)):
            chunk = rows[start:start + step]
            pd.DataFrame(chunk).to_parquet(
                os.path.join(cache_file, f"RLAIF-V-Dataset-withlogp_{idx:03}-{len(chunk)}.parquet"))
    if dist.is_initialized():
        dist.barrier()


def inference_logp(model, tokenizer, hf_data, cache_file, image_token_len, img_processor, use_im_start_end,
                   is_llava15=True, batch_size=8):
    ds = PreferenceInferenceDataset(hf_data, tokenizer, image_token_len, img_processor, use_im_start_end)
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False, sampler=InferenceSampler(len(ds)),
                                         collate_fn=partial(preference_collator_fn, pad_token_id=tokenizer.pad_token_id))
    outs = get_multimodal_sample_logps(model, loader, tokenizer, is_llava15=is_llava15)
    if dist.is_initialized() and dist.get_world_size() > 1:
        merged = []
        for o in outs:
            bucket = [None] * dist.get_world_size()
            dist.all_gather_object(bucket, o)
            merged.append(list(itertools.chain.from_iterable(bucket)))
        outs = tuple(merged)
    write_logp_to_preference_parquet(ds.data, cache_file, list(zip(*outs)), overwrite_logps=False)


# ------------------------------------------------------------------------------------------------
# checkpoint / tokenizer loading (plumbing; no weights exist offline in the build environment)
# ------------------------------------------------------------------------------------------------
def load_tokenizer(model_name_or_path, model_max_length):
    import transformers
    tok = transformers.AutoTokenizer.from_pretrained(model_name_or_path, model_max_length=model_max_length,
                                                     padding_side="right", use_fast=False)
    tok.pad_token = tok.unk_token            # muffin/train/train_llava15.py:219-228
    return tok


def load_hf_checkpoint(model_dir, vision_tower_dir=None):
    """HF-format LLaVA-1.5 checkpoint directory (+ CLIP directory) -> flat HF-named state dict."""
    def read_dir(d):
        state = {}
        files = sorted(os.listdir(d))
        st = [f for f in files if f.endswith(".safetensors")]
        if st:
            from safetensors.torch import load_file
            for f in st:
                state.update(load_file(os.path.join(d, f)))
        else:
            for f in files:
                if f.endswith(".bin") and f.startswith("pytorch_model"):
                    state.update(torch.load(os.path.join(d, f), map_location="cpu"))
        return state
    if not os.path.isdir(model_dir):
        raise FileNotFoundError("checkpoint directory %r not found (hub downloads are not available)" % model_dir)
    state = read_dir(model_dir)
    if vision_tower_dir and os.path.isdir(vision_tower_dir):
        for k, v in read_dir(vision_tower_dir).items():
            if k.startswith("vision_model."):
                state["model.vision_tower.vision_tower." + k] = v
    return state
