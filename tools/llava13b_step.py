#!/usr/bin/env python
"""LoRA-DPO of LLaVA-1.5-13B on one GPU: step time, model FLOP rate, memory, and the RMSNorm kernels at 5120 columns.

    python tools/llava13b_step.py [--layers 40] [--steps 5] [--warmup 3] [--micro-pairs 8]

Workload: bench.py's LoRA-DPO recipe at 13B widths (hidden 5120, ffn 13824, 40 heads of 128, 40 layers, vocab 32000;
CLIP-ViT-L/14-336 and the 1024 -> 5120 -> 5120 projector), LoRA r = 64 / alpha = 16 on q,k,v,o,gate,up,down, seeded
random weights, bench's synthetic inputs (8 pairs, 336 px, 48-token prompt, R = 512, T = 1135). The frozen-reference
log-probs are the initial policy's, so the step-0 loss is ln 2. The micro-batch starts at --micro-pairs and is halved
on out-of-memory, as bench.py does. Then --warmup steps and --steps timed steps (CUDA events).

Model FLOPs per pair (SURVEY.md §8d, LoRA form): 2 T [4 (N_dec + N_head) + 6 N_lora] + 3 x causal attention + F_clip +
3 F_proj, with N_dec = 40 (4 H^2 + 3 H F), N_head = H V and N_lora = 250 347 520 (base weight gradients are not computed).

RMSNorm: forward and backward (with the residual gradient, as the decoder runs it) at [9080, 5120] and [9080, 4096],
bytes moved over CUDA-event time. Prints one JSON line, with the card's name, power limit and median SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from bench import PAIRS_PER_GPU, PROMPT_LEN, RESP_LEN, ClockSampler, synthetic_batch  # noqa: E402

H, F, V, HEADS, C = 5120, 13824, 32000, 40, 1024
N_LORA = 250_347_520          # r = 64 on q,k,v,o,gate,up,down of 40 layers: 40 * 64 * (11 H + 3 F)


def flops_per_pair(T, layers):
    n_dec = layers * (4 * H ** 2 + 3 * H * F)
    n_head = H * V
    attn_seq = layers * 4 * T * T * H * 0.5
    f_clip = 2 * 23 * (4 * C ** 2 + 2 * C * 4096) * 577 + 23 * 4 * 577 ** 2 * C + 2 * 588 * C * 576
    f_proj = 2 * (C * H + H ** 2) * 576
    n_lora = N_LORA * layers // 40
    return 2 * T * (4 * (n_dec + n_head) + 6 * n_lora) + 3 * 2 * attn_seq + f_clip + 3 * f_proj


def rmsnorm_rates(M, width, iters=50):
    """GB/s of rmsnorm_fwd (x in, y out, fp32 rstd) and rmsnorm_bwd (dy, x, dres in, dx out; dw partials) on
    [M, width] bf16 rows."""
    from rlaifv_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(width)
    x = torch.randn(M, width, generator=g, device="cuda").to(torch.bfloat16)
    dy, dres = torch.randn_like(x), torch.randn_like(x)
    w = torch.ones(width, dtype=torch.bfloat16, device="cuda")
    rstd = torch.empty(M, dtype=torch.float32, device="cuda")
    y, dx, dw = torch.empty_like(x), torch.empty_like(x), torch.empty_like(w)
    parts = ops._l.load().rlaifv_rmsnorm_bwd_partials()
    grid = min(parts, (M + 1) // 2)

    def fwd():
        ops.rmsnorm_fwd(x, w, 1e-5, out=y, rstd=rstd)

    def bwd():
        ops.rmsnorm_bwd(dy, x, w, rstd, dx, dw, dres=dres)

    out = {}
    for name, f, nbytes in (("fwd", fwd, 2 * M * width * 2 + 4 * M),
                            ("bwd", bwd, 4 * M * width * 2 + 4 * M + 2 * grid * width * 4)):
        for _ in range(5):
            f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            f()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / iters
        out[name] = {"us": round(ms * 1e3, 1), "gb_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--micro-pairs", type=int, default=PAIRS_PER_GPU)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("llava13b_step.py measures on a GPU; none is visible")
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    B, micro = PAIRS_PER_GPU, args.micro_pairs
    dims = LlavaDims(hidden_size=H, intermediate_size=F, num_layers=args.layers, num_heads=HEADS)
    T = PROMPT_LEN + RESP_LEN - 1 + dims.num_patches
    norms = {"%dx%d" % (9080, wd): rmsnorm_rates(9080, wd) for wd in (5120, 4096)}
    policy = LlavaDPOPolicy(dims, "cuda", seed=0)
    policy.enable_lora(r=64, alpha=16)
    weights_gb = policy.store.flat.numel() * 2 / 1e9
    engine = DPOStepEngine(policy, lr=1e-5, weight_decay=0.01, total_steps=2672, micro_pairs=micro)
    host = [synthetic_batch(0, s, B) for s in range(2)]
    loss0 = None
    while loss0 is None:
        try:
            for hb in host:              # frozen-reference log-probs = the initial policy's (step-0 loss ln 2)
                rw, rr = [], []
                for lo in range(0, B, micro):
                    hi = min(B, lo + micro)
                    ids = torch.cat([hb["concatenated_input_ids"][lo:hi], hb["concatenated_input_ids"][B + lo:B + hi]])
                    lab = torch.cat([hb["concatenated_labels"][lo:hi], hb["concatenated_labels"][B + lo:B + hi]])
                    out = policy.forward_logps(ids, lab, hb["images"][lo:hi], keep_stash=False)
                    rw.append(out["logp"][: hi - lo].float().cpu())
                    rr.append(out["logp"][hi - lo:].float().cpu())
                hb["ref_win_logp"], hb["ref_rej_logp"] = torch.cat(rw), torch.cat(rr)
            dev = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()} for hb in host]
            loss0 = float(engine.train_step(dev[0], optimizer_step=False)[0].item())
        except torch.OutOfMemoryError:
            policy._stash = None
            policy._bufs.clear()
            torch.cuda.empty_cache()
            if micro == 1:
                raise
            micro = max(1, micro // 2)
            engine.micro_pairs = micro
    for s in range(args.warmup):
        engine.train_step(dev[s % 2])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for s in range(args.steps):
        m = engine.train_step(dev[s % 2])
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1) / args.steps
    last_loss = float(m[0].item())
    card = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    f_pair = flops_per_pair(T, args.layers)
    pairs_s = B / (ms * 1e-3)
    res = {"workload": "LoRA(r=64)-DPO LLaVA-1.5-13B widths, %d layers, %d pairs, 336 px, T = %d, seeded random "
                       "weights" % (args.layers, B, T),
           "step0_loss": loss0, "ln2": 0.6931471805599453, "last_loss": last_loss,
           "micro_pairs": micro, "steps": args.steps, "warmup": args.warmup,
           "ms_per_step": round(ms, 1), "pairs_per_s": round(pairs_s, 3),
           "model_tflop_per_pair": round(f_pair / 1e12, 2), "model_tflops": round(pairs_s * f_pair / 1e12, 1),
           "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2), "base_weights_gb": round(weights_gb, 2),
           "rmsnorm": norms, "card": card, "clocks": clocks}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
