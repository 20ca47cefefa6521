#!/usr/bin/env python
"""Ragged preference batches on packed decoder rows vs the padded layout, on one GPU.

    python tools/ragged_step.py [--layers 32] [--steps 5] [--warmup 3] [--rounds 2] [--micro-pairs 4]

Workload: bench.py's LoRA-DPO recipe (LLaVA-1.5-7B, r = 64, alpha = 16, 8 pairs, 336 px, 48-token prompt, R = 512,
micro-batches of 4 pairs), except that every response length is uniform in [R/2, R] (SURVEY.md §8d's second canonical
run; per step `torch.Generator().manual_seed(1234 + step)`), so the batch is right-padded.

Before timing, on the same weights: the training forward of each micro-batch with and without packing must give the
same bits (log-probs, average log-probs, per-token log-probs, spliced labels), and so must the 9 metrics of a step
without update; an equal-length batch (bench.py's headline inputs) must not be packed. Then the two layouts alternate,
`--rounds` times: `--warmup` steps, then `--steps` timed steps each (the timed steps update the weights). Prints one JSON
line: pairs/s, ms per step, decoder rows, causal attention tiles per head, peak memory, card, power limit, median SM
clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from bench import IMAGE_POS, PAIRS_PER_GPU, PROMPT_LEN, RESP_LEN, ClockSampler, synthetic_batch  # noqa: E402


def ragged_batch(step, B):
    """bench.synthetic_batch with response lengths uniform in [R/2, R], right-padded with id 0 / label -100."""
    g = torch.Generator().manual_seed(1234 + step)
    L = PROMPT_LEN + RESP_LEN
    ids = torch.zeros((2 * B, L), dtype=torch.int64)
    labels = torch.full((2 * B, L), -100, dtype=torch.int64)
    for i in range(B):
        prompt = torch.randint(3, 32000, (PROMPT_LEN,), generator=g)
        prompt[0] = 1
        prompt[IMAGE_POS] = -200
        for row in (i, B + i):
            R = int(torch.randint(RESP_LEN // 2, RESP_LEN + 1, (1,), generator=g))
            resp = torch.randint(3, 32000, (R,), generator=g)
            resp[-1] = 2
            ids[row, :PROMPT_LEN + R] = torch.cat([prompt, resp])
            labels[row, PROMPT_LEN:PROMPT_LEN + R] = resp
    images = torch.randn(B, 3, 336, 336, generator=g)
    return {"concatenated_input_ids": ids, "concatenated_labels": labels, "images": images, "beta": 0.1}


def micro_batches(batch, B, micro):
    for lo in range(0, B, micro):
        hi = min(B, lo + micro)
        ids = torch.cat([batch["concatenated_input_ids"][lo:hi], batch["concatenated_input_ids"][B + lo:B + hi]])
        lab = torch.cat([batch["concatenated_labels"][lo:hi], batch["concatenated_labels"][B + lo:B + hi]])
        yield lo, hi, ids, lab, batch["images"][lo:hi]


def work_counts(policy, batch, B, micro):
    """(padded rows, packed rows, padded tiles, packed tiles): decoder rows and causal (query, key) 128-row tile pairs
    per head of attention, summed over the micro-batches."""
    from rlaifv_b200.model import packed_lengths
    rows_pad = rows_pk = tiles_pad = tiles_pk = 0
    for lo, hi, ids, lab, img in micro_batches(batch, B, micro):
        _, new_labels, _, T = policy.splice(ids.cuda(), lab.cuda(), torch.zeros(
            (hi - lo) * policy.dims.num_patches, policy.dims.hidden_size, dtype=torch.bfloat16, device="cuda"), hi - lo,
            (torch.arange(ids.shape[0], dtype=torch.int32, device="cuda") % (hi - lo)).contiguous())
        lens = packed_lengths(new_labels).tolist()
        n = (T + 127) // 128
        rows_pad += len(lens) * T
        rows_pk += sum(lens)
        tiles_pad += len(lens) * n * (n + 1) // 2
        tiles_pk += sum((ln + 127) // 128 * ((ln + 127) // 128 + 1) // 2 for ln in lens)
    return rows_pad, rows_pk, tiles_pad, tiles_pk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--micro-pairs", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_step.py measures on a GPU; none is visible")
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    B, micro = PAIRS_PER_GPU, args.micro_pairs
    policy = LlavaDPOPolicy(LlavaDims(num_layers=args.layers), "cuda", seed=0)
    policy.enable_lora(r=64, alpha=16)
    engine = DPOStepEngine(policy, lr=1e-5, weight_decay=0.01, total_steps=2672, micro_pairs=micro)

    batches = [ragged_batch(s, B) for s in range(2)]
    for hb in batches:                      # frozen-reference log-probs = the initial policy's (step-0 loss ln 2)
        rw, rr = [], []
        for lo, hi, ids, lab, img in micro_batches(hb, B, micro):
            out = policy.forward_logps(ids, lab, img, keep_stash=False)
            rw.append(out["logp"][: hi - lo].float().cpu())
            rr.append(out["logp"][hi - lo:].float().cpu())
        hb["ref_win_logp"], hb["ref_rej_logp"] = torch.cat(rw), torch.cat(rr)
    dev = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()} for hb in batches]

    # identity on the same weights, before any update
    identical, packed_taken = True, []
    for lo, hi, ids, lab, img in micro_batches(dev[0], B, micro):
        outs = []
        for packed in (False, True):
            policy.pack_rows = packed
            out = policy.forward_logps(ids, lab, img, keep_stash=True)
            packed_taken.append(policy._stash["pack"] is not None)
            outs.append({k: out[k].clone() for k in ("logp", "avg_logp", "per_token_logps", "labels")})
            policy._stash = None
        identical &= all(torch.equal(outs[0][k], outs[1][k]) for k in outs[0])
    metrics = []
    for packed in (False, True):
        policy.pack_rows = packed
        metrics.append(engine.train_step(dev[0], optimizer_step=False).clone().cpu())
    metrics_identical = torch.equal(metrics[0], metrics[1])
    policy.pack_rows = True
    eq = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synthetic_batch(0, 0, B).items()}
    lo, hi, ids, lab, img = next(micro_batches(eq, B, micro))
    policy.forward_logps(ids, lab, img, keep_stash=True)
    equal_length_packed = policy._stash["pack"] is not None
    policy._stash = None
    rows_pad, rows_pk, tiles_pad, tiles_pk = work_counts(policy, dev[0], B, micro)

    timings = {"padded": [], "packed": []}
    peak = {}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for _ in range(args.rounds):
        for name in ("padded", "packed"):
            policy.pack_rows = name == "packed"
            for s in range(args.warmup):
                engine.train_step(dev[s % 2])
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            for s in range(args.steps):
                engine.train_step(dev[s % 2])
            torch.cuda.synchronize()
            timings[name].append((time.perf_counter() - t0) / args.steps)
            peak[name] = max(peak.get(name, 0), torch.cuda.max_memory_allocated())
    clocks = sampler.stop()
    card = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"workload": "LoRA-DPO LLaVA-1.5-7B, %d layers, %d pairs, micro %d, R uniform in [%d, %d]"
                       % (args.layers, B, micro, RESP_LEN // 2, RESP_LEN),
           "forward_identical": bool(identical), "step_metrics_identical": bool(metrics_identical),
           "packed_path_taken": packed_taken[1::2], "equal_length_batch_packed": equal_length_packed,
           "rows": {"padded": rows_pad, "packed": rows_pk}, "attention_tiles_per_head": {"padded": tiles_pad,
                                                                                        "packed": tiles_pk},
           "card": card, "clocks": clocks}
    for name in ("padded", "packed"):
        ms = [1e3 * t for t in timings[name]]
        res[name] = {"ms_per_step": [round(x, 1) for x in ms], "pairs_per_s": [round(B / (x / 1e3), 3) for x in ms],
                     "peak_mem_gb": round(peak[name] / 1e9, 2)}
    res["speedup"] = round(min(timings["padded"]) / min(timings["packed"]), 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
