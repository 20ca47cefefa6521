#!/usr/bin/env python
"""Shared prompt prefixes (policy.share_prefix) against today's layout, on one GPU.

    python tools/prefix_step.py [--layers 32] [--steps 5] [--warmup 3] [--rounds 2] [--micro-pairs 4]

Workloads: bench.py's LoRA-DPO headline (LLaVA-1.5-7B, r = 64, alpha = 16, dropout 0, 8 pairs, micro-batches of 4
pairs, bench.py's synthetic inputs: equal-length responses, so today's layout is the padded one) and its ragged variant
(responses uniform in [R/2, R], tools/ragged_step.py's batches, where today's layout is packed rows). For each, before
timing and on the same weights: the training forward of every micro-batch with sharing off and on must give the same
bits (log-probs, average log-probs, per-token log-probs, spliced labels), and so must the 9 metrics of a step without
update. Then the two layouts alternate, `--rounds` times: `--warmup` steps, then `--steps` timed steps each. Also the
attention of one layer on each layout's rows (random q/k/v, CUDA events over 20 launches, forward and backward).
Prints one JSON line: decoder rows and causal attention tile pairs per head per step, ms per step, pairs/s, peak
memory, attention times, card, power limit and median SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

import torch  # noqa: E402

from bench import PAIRS_PER_GPU, ClockSampler, synthetic_batch  # noqa: E402
from ragged_step import micro_batches, ragged_batch  # noqa: E402


def layouts(policy, batch, B, micro, share):
    """The RowPacking (or None = padded) and padded length of each micro-batch with sharing off / on."""
    from rlaifv_b200.model import pack_rows, splice_sources
    out = []
    for lo, hi, ids, lab, img in micro_batches(batch, B, micro):
        ids, lab = ids.cuda(), lab.cuda()
        _, new_labels, src, T = policy.splice(ids, lab, torch.zeros(
            (hi - lo) * policy.dims.num_patches, policy.dims.hidden_size, dtype=torch.bfloat16, device="cuda"), hi - lo,
            (torch.arange(ids.shape[0], dtype=torch.int32, device="cuda") % (hi - lo)).contiguous())
        out.append((pack_rows(new_labels, splice_sources(src, ids) if share else None), ids.shape[0], T))
    return out


def work_counts(lays):
    """(decoder rows, causal 128-row (query, key) tile pairs per head) summed over the micro-batches."""
    rows = tiles = 0
    for pk, nseq, T in lays:
        if pk is None:
            n = (T + 127) // 128
            rows, tiles = rows + nseq * T, tiles + nseq * n * (n + 1) // 2
            continue
        rows += pk.M
        own = (pk.cu[1:] - pk.cu[:-1]).tolist()
        p0 = pk.pos0_h.tolist() if pk.shared else [0] * nseq
        for p, n in zip(p0, own):
            a, e = p // 128, (p + n + 127) // 128     # query tiles a .. e-1, each over key tiles 0 .. itself
            tiles += e * (e + 1) // 2 - a * (a + 1) // 2
    return rows, tiles


def attention_ms(lay, dims, reps=20):
    """(forward ms, backward ms) of one decoder layer's attention on this layout's rows."""
    from rlaifv_b200 import ops
    pk, nseq, T = lay
    nh, hd, H = dims.num_heads, dims.head_dim, dims.hidden_size
    M = nseq * T if pk is None else pk.M
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(M, 3 * H, device="cuda", generator=g).to(torch.bfloat16)
    att, lse = torch.empty(M, H, dtype=torch.bfloat16, device="cuda"), torch.empty(nh * M, device="cuda")
    d_o, dqkv, delta = torch.randn_like(att), torch.empty_like(qkv), torch.empty(nh * M, device="cuda")
    q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    scale = hd ** -0.5
    if pk is None:
        fwd = lambda: ops.attention_fwd(q, k, v, nseq, T, nh, hd, True, scale, out=att,  # noqa: E731
                                        lse=lse.view(nseq, nh, T))
        bwd = lambda: ops.attention_bwd_split(q, k, v, att, d_o, lse.view(nseq, nh, T), nseq, T, T, nh, hd,  # noqa: E731
                                              True, scale, dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:],
                                              delta_ws=delta.view(nseq, nh, T))
    else:
        f, b = (ops.attention_varlen_prefix_fwd, ops.attention_varlen_prefix_bwd) if pk.shared else \
            (ops.attention_varlen_fwd, ops.attention_varlen_bwd)
        fwd = lambda: f(q, k, v, pk, nh, hd, scale, att, lse)  # noqa: E731
        bwd = lambda: b(q, k, v, att, d_o, lse, pk, nh, hd, scale, dqkv[:, :H], dqkv[:, H:2 * H],  # noqa: E731
                        dqkv[:, 2 * H:], delta)
    res = []
    for fn in (fwd, bwd):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(round(e0.elapsed_time(e1) / reps, 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--micro-pairs", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prefix_step.py measures on a GPU; none is visible")
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    B, micro = PAIRS_PER_GPU, args.micro_pairs
    policy = LlavaDPOPolicy(LlavaDims(num_layers=args.layers), "cuda", seed=0)
    policy.enable_lora(r=64, alpha=16)
    engine = DPOStepEngine(policy, lr=1e-5, weight_decay=0.01, total_steps=2672, micro_pairs=micro)

    res = {"workload": "LoRA-DPO LLaVA-1.5-7B, %d layers, r 64, dropout 0, %d pairs, micro %d" % (args.layers, B, micro)}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for wl, make in (("equal", lambda s: synthetic_batch(s, 0, B)), ("ragged", lambda s: ragged_batch(s, B))):
        batches = [make(s) for s in range(2)]
        policy.share_prefix = False
        for hb in batches:                  # frozen-reference log-probs = the initial policy's
            rw, rr = [], []
            for lo, hi, ids, lab, img in micro_batches(hb, B, micro):
                out = policy.forward_logps(ids, lab, img, keep_stash=False)
                rw.append(out["logp"][: hi - lo].float().cpu())
                rr.append(out["logp"][hi - lo:].float().cpu())
            hb["ref_win_logp"], hb["ref_rej_logp"] = torch.cat(rw), torch.cat(rr)
        dev = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()} for hb in batches]
        r = {}
        identical, shared_taken = True, []
        for lo, hi, ids, lab, img in micro_batches(dev[0], B, micro):
            outs = []
            for share in (False, True):
                policy.share_prefix = share
                out = policy.forward_logps(ids, lab, img, keep_stash=True)
                pk = policy._stash["pack"]
                shared_taken.append(pk is not None and pk.shared)
                outs.append({k: out[k].clone() for k in ("logp", "avg_logp", "per_token_logps", "labels")})
                policy._stash = None
            identical &= all(torch.equal(outs[0][k], outs[1][k]) for k in outs[0])
        metrics = []
        for share in (False, True):
            policy.share_prefix = share
            metrics.append(engine.train_step(dev[0], optimizer_step=False).clone().cpu())
        r.update(forward_identical=bool(identical), step_metrics_identical=torch.equal(metrics[0], metrics[1]),
                 shared_path_taken=shared_taken[1::2])
        timings, peak = {"off": [], "on": []}, {}
        for _ in range(args.rounds):
            for name in ("off", "on"):
                policy.share_prefix = name == "on"
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
        for name in ("off", "on"):
            lays = layouts(policy, dev[0], B, micro, name == "on")
            rows, tiles = work_counts(lays)
            ms = [1e3 * t for t in timings[name]]
            r[name] = {"rows_per_step": rows, "attention_tile_pairs_per_head_per_step": tiles,
                       "ms_per_step": [round(x, 1) for x in ms], "pairs_per_s": [round(B / (x / 1e3), 3) for x in ms],
                       "peak_mem_gb": round(peak[name] / 1e9, 2),
                       "attention_ms_fwd_bwd_first_micro_batch": attention_ms(lays[0], policy.dims)}
        r["speedup"] = round(min(timings["off"]) / min(timings["on"]), 4)
        res[wl] = r
    res["clocks"] = sampler.stop()
    res["card"] = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                                  "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
