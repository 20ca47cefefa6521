"""-m gpu end-to-end drop-in flow on a synthetic preference dataset: rows without cached log-probs ->
RLAIFVDataset triggers the frozen-reference pre-pass on the H100 forward kernels -> parquet cache in the
reference's on-disk format -> DPODataset / DataCollatorForDPODataset -> LLaVA15DPOTrainer.train().
(muffin/data/datasets.py:27-91, muffin/eval/muffin_inference_logp.py:213-344, muffin/train/train_llava15.py:124-195)"""
import io
import json
import os
from types import SimpleNamespace

import pytest
import torch

from oracle import llava_dpo_oracle as O
from oracle.toy_tokenizer import ToyTokenizer

pytestmark = pytest.mark.gpu


def png_bytes(seed, size=56):
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    arr = (torch.rand(size, size, 3, generator=g) * 255).to(torch.uint8).numpy()
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, format="PNG")
    return buf.getvalue()


def image_processor(pil):
    import numpy as np
    x = torch.from_numpy(np.asarray(pil, dtype="float32") / 255.0).permute(2, 0, 1)
    return (x - 0.5) / 0.25


def test_prepass_parquet_dataset_collator_trainer(tmp_path):
    from rlaifv_b200.data import DPODataset, RLAIFVDataset, make_dpo_data_module
    from rlaifv_b200.llava_model import LlavaLlamaForCausalLM
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.trainers import LLaVA15DPOTrainer
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    params = O.make_params(c, seed=0, scale=0.4)
    model = LlavaLlamaForCausalLM(dims, "cuda", hf_state=params)
    tok = ToyTokenizer()
    words = "a red bus on the street near two small dogs and one cat under blue sky with trees".split()
    rows = []
    for i in range(6):
        rows.append({"image": {"bytes": png_bytes(i)}, "question": "what is shown in picture %d ?" % i,
                     "chosen": " ".join(words[i:i + 6]), "rejected": " ".join(words[::-1][i:i + 4 + i % 3]),
                     "idx": i, "origin_dataset": "synthetic", "origin_split": "train", "image_path": "img%d" % i})
    data_dir = str(tmp_path / "data")
    data_args = SimpleNamespace(is_multimodal=True, image_token_len=c.num_patches, image_folder=None,
                                image_aspect_ratio="pad", image_processor=image_processor, data_source_names=[""],
                                data_source_weights=[1], shuffle_data=True, dpo_beta=0.1, dpo_token_weight=1.0,
                                data_dir=data_dir)
    dm = make_dpo_data_module(tok, data_args, reference_model=model, source_rows=rows)
    # --- on-disk contract of the pre-pass ---
    files = sorted(os.listdir(data_dir))
    assert files == ["RLAIF-V-Dataset-withlogp_000-6.parquet"]
    ds = dm["train_dataset"]
    assert len(ds) == 6
    raw = ds.list_data_dict.data[2]
    logps = json.loads(raw["logps"])["logps"]
    assert len(logps) == 6 and isinstance(logps[2], list) and isinstance(logps[5], list)
    rej, win = ds[2]
    n_win = len(win["input_ids"])
    assert len(logps[2]) == n_win - 1 + c.num_patches - 1          # per-token list of the spliced sequence
    assert abs(win["ref_win_logp"] - logps[0]) < 1e-6 and abs(rej["ref_rej_logp"] - logps[3]) < 1e-6
    # --- the cached reference log-probs are the model's own: policy == reference at step 0 -> loss ln 2 ---
    batch = dm["data_collator"]([ds[i] for i in range(3)])
    out = model.policy.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"],
                                     keep_stash=False)
    ref = torch.cat([batch["ref_win_logp"], batch["ref_rej_logp"]]).cuda().float()
    assert float((out["logp"] - ref).abs().max()) <= 1e-3 * float(ref.abs().max())
    # a second construction finds the cache and does not need a reference model
    ds2 = RLAIFVDataset(data_dir, reference_model=None, tokenizer=tok)
    assert len(ds2) == 6
    # --- train two steps through the drop-in trainer on that dataset ---
    args = SimpleNamespace(learning_rate=1e-3, weight_decay=0.0, max_steps=2, warmup_ratio=0.0, dpo_use_average=False,
                           dpo_token_weighted=False, task="DPO", output_dir=str(tmp_path / "ckpt"), logging_steps=1,
                           save_strategy="no", save_steps=0, save_total_limit=None, per_device_train_batch_size=3,
                           dataloader_num_workers=0, lr_scheduler_type="constant", bf16=True, deepspeed=None, seed=1)
    tr = LLaVA15DPOTrainer(model=model, tokenizer=tok, args=args, **dm)
    tr.train()
    torch.cuda.synchronize()
    losses = [h["loss"] for h in tr.state["log_history"] if "loss" in h]
    assert len(losses) == 2 and abs(losses[0] - 0.693147) < 5e-3     # first step: policy == reference
    assert all(l == l and abs(l) < 10 for l in losses)
