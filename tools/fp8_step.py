#!/usr/bin/env python
"""The FP8 frozen base (--base_fp8) against the bf16 base, on one GPU.

    python tools/fp8_step.py [--out results.json] [--skip-13b]

1. Kernels: the 8 frozen-base GEMM launches of a LoRA (r = 64) step at the 7B and 13B widths, M = 9080 rows, four
   variants alternating (CUDA events, median of rounds): the shipped bf16 launch (gemm_dual / gemm_swiglu_bwd), gemm_fp8
   alone, gemm_fp8 plus the quantization of its input, and cuBLAS FP8 through torch._scaled_mm with row-wise scales (a
   plain product without second source or epilogue: a yardstick only). ms and TFLOP/s of the base product (2 M N K),
   and the quantizers' GB/s (bytes read + written).
2. 7B LoRA-DPO step (bench.py's inputs, 8 pairs, micro-batches of 4): both bases resident, alternating, 2 rounds of 3
   warm-up and 5 timed steps; pairs/s, the peak memory with both resident and each base's parameter and gradient
   storage, the step-0 loss (reference log-probs from the same policy), and the loss of 20 steps from one seed.
3. 13B LoRA-DPO step: the largest micro-batch of 8, 4 or 2 pairs that fits with the FP8 base, against the bf16 base
   at 2 pairs.
Prints one JSON line with the card, its power limit and the median SM clock.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from bench import PAIRS_PER_GPU, ClockSampler, synthetic_batch  # noqa: E402

M = 9080
R = 64
WIDTHS = {"7b": dict(hidden_size=4096, intermediate_size=11008, num_heads=32),
          "13b": dict(hidden_size=5120, intermediate_size=13824, num_heads=40)}


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q


def events_ms(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def shapes(w):
    """(name, N, K, dgrad, k2, n_sub, residual, glu) of the 8 frozen-base launches (model._lin_fwd / _lin_bwd)."""
    H, F = w["hidden_size"], w["intermediate_size"]
    return [("qkv_fwd", 3 * H, H, False, R, H, False, False), ("o_fwd", H, H, False, R, 0, True, False),
            ("gu_fwd", 2 * F, H, False, R, F, False, False), ("down_fwd", H, F, False, R, 0, True, False),
            ("down_dgrad_swiglu", F, H, True, R, 0, False, True), ("gu_dgrad", H, 2 * F, True, 2 * R, 0, False, False),
            ("o_dgrad", H, H, True, R, 0, False, False), ("qkv_dgrad", H, 3 * H, True, 3 * R, 0, False, False)]


def kernels(reps=10, rounds=3):
    from rlaifv_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {}
    for wname, w in WIDTHS.items():
        for name, N, K, dgrad, k2, n_sub, res, glu in shapes(w):
            Nw, Kw = (K, N) if dgrad else (N, K)                 # W [Nw, Kw]
            wb = (torch.randn((Nw, Kw), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
            fw = ops.Fp8Weight(Nw, Kw, "cuda")
            ops.quant_fp8_blocks(wb, fw.q, fw.qt, fw.s)
            x = torch.randn((M, K), generator=g, device="cuda").to(torch.bfloat16)
            a2 = torch.randn((M, (N // n_sub) * R if n_sub else k2), generator=g, device="cuda").to(torch.bfloat16)
            b2 = (torch.randn((k2, N) if dgrad else (N, k2), generator=g, device="cuda") * 0.02).to(torch.bfloat16)
            resid = torch.randn((M, N), generator=g, device="cuda").to(torch.bfloat16) if res else None
            gu = torch.randn((M, 2 * N), generator=g, device="cuda").to(torch.bfloat16) if glu else None
            c = torch.empty((M, 2 * N if glu else N), dtype=torch.bfloat16, device="cuda")
            xq, xs = ops.quant_fp8_rows(x)
            if glu:
                bf16 = lambda: ops.gemm_swiglu_bwd(x, wb, gu, c, b_mn=True, a2=a2, b2=b2)  # noqa: E731
            else:
                bf16 = lambda: ops.gemm_dual(x, wb, a2, b2, c, k2=k2 if not n_sub else R, r=R, n_sub=n_sub,  # noqa: E731
                                             b_mn=dgrad, residual=resid)
            kw = dict(dgrad=dgrad, a2=a2, b2=b2, k2=R if n_sub else k2, r=R, n_sub=n_sub, residual=resid, glu=gu)
            fp8 = lambda: ops.gemm_fp8(xq, xs, fw, c, **kw)  # noqa: E731
            fp8q = lambda: ops.gemm_fp8(*ops.quant_fp8_rows(x, xq, xs), fw, c, **kw)  # noqa: E731
            bq = fw.qt if dgrad else fw.q                         # [N, K] row-major = column-major [K, N]
            sa_row = torch.rand((M, 1), device="cuda") + 0.5
            sb_row = torch.rand((1, N), device="cuda") + 0.5
            cub = lambda: torch._scaled_mm(xq, bq.t(), scale_a=sa_row, scale_b=sb_row,  # noqa: E731
                                           out_dtype=torch.bfloat16)
            quant = lambda: ops.quant_fp8_rows(x, xq, xs)  # noqa: E731
            t = {k: [] for k in ("bf16", "fp8", "fp8_with_quant", "cublas_fp8_rowwise", "quant_rows")}
            for _ in range(rounds):
                for k, fn in (("bf16", bf16), ("fp8", fp8), ("fp8_with_quant", fp8q), ("cublas_fp8_rowwise", cub),
                              ("quant_rows", quant)):
                    t[k].append(events_ms(fn, reps))
            flop = 2.0 * M * N * K
            r = {}
            for k, v in t.items():
                ms = sorted(v)[len(v) // 2]
                r[k + "_ms"] = round(ms, 4)
                if k != "quant_rows":
                    r[k + "_tflops"] = round(flop / ms / 1e9, 1)
            r["quant_rows_gbps"] = round((M * K * 2 + M * K + 4 * M * K / 128) / r["quant_rows_ms"] / 1e6, 1)
            wq = events_ms(lambda: ops.quant_fp8_blocks(wb, fw.q, fw.qt, fw.s), 3)
            r["quant_blocks_gbps"] = round((Nw * Kw * 4) / wq / 1e6, 1)
            r["fp8_speedup_vs_bf16"] = round(r["bf16_ms"] / r["fp8_ms"], 3)
            r["fp8_with_quant_speedup_vs_bf16"] = round(r["bf16_ms"] / r["fp8_with_quant_ms"], 3)
            out["%s_%s" % (wname, name)] = r
            del wb, fw, x, a2, b2, resid, gu, c, xq, xs
            torch.cuda.empty_cache()
    return out


def make_policy(width, layers, base_fp8, micro):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    pol = LlavaDPOPolicy(LlavaDims(num_layers=layers, **width), "cuda", seed=0, base_fp8=base_fp8)
    pol.enable_lora(r=R, alpha=16)
    eng = DPOStepEngine(pol, lr=1e-5, weight_decay=0.01, total_steps=2672, micro_pairs=micro)
    return pol, eng


def batches(pol, micro, n=2):
    """bench.py's inputs with frozen-reference log-probs from this policy (its initial state)."""
    B = PAIRS_PER_GPU
    out = []
    for s in range(n):
        hb = synthetic_batch(0, s, B)
        rw, rr = [], []
        for lo in range(0, B, micro):
            hi = min(B, lo + micro)
            ids = torch.cat([hb["concatenated_input_ids"][lo:hi], hb["concatenated_input_ids"][B + lo:B + hi]])
            lab = torch.cat([hb["concatenated_labels"][lo:hi], hb["concatenated_labels"][B + lo:B + hi]])
            o = pol.forward_logps(ids, lab, hb["images"][lo:hi], keep_stash=False)
            rw.append(o["logp"][:hi - lo].float().cpu())
            rr.append(o["logp"][hi - lo:].float().cpu())
        hb["ref_win_logp"], hb["ref_rej_logp"] = torch.cat(rw), torch.cat(rr)
        out.append({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()})
    return out


def step_7b(layers=32, micro=4, warmup=3, steps=5, rounds=2, traj=20):
    runs = {}
    for name, fp8 in (("bf16", False), ("fp8", True)):
        pol, eng = make_policy(WIDTHS["7b"], layers, fp8, micro)
        runs[name] = dict(pol=pol, eng=eng, dev=batches(pol, micro), losses=[], times=[], peak=0)
    for _ in range(rounds):
        for r in runs.values():
            for s in range(warmup):
                r["losses"].append(float(r["eng"].train_step(r["dev"][len(r["losses"]) % 2])[0]))
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            for s in range(steps):
                r["losses"].append(float(r["eng"].train_step(r["dev"][len(r["losses"]) % 2])[0]))
            torch.cuda.synchronize()
            r["times"].append((time.perf_counter() - t0) / steps)
            r["peak"] = max(r["peak"], torch.cuda.max_memory_allocated())
    for r in runs.values():
        while len(r["losses"]) < traj:
            r["losses"].append(float(r["eng"].train_step(r["dev"][len(r["losses"]) % 2])[0]))
    res = {}
    for name, r in runs.items():
        best = min(r["times"])
        st, f8 = r["pol"].store, r["pol"].fp8
        res[name] = dict(pairs_per_s=round(PAIRS_PER_GPU / best, 3),
                         pairs_per_s_rounds=[round(PAIRS_PER_GPU / t, 3) for t in r["times"]],
                         peak_gb_both_resident=round(r["peak"] / 1e9, 2),
                         base_and_store_gb=round((2 * st.flat.numel() + (2 * st.grad.numel() if st.grad is not None
                                                  else 0) + (f8.nbytes() if f8 is not None else 0)) / 1e9, 2),
                         step0_loss=round(r["losses"][0], 6), loss_trajectory=[round(v, 5) for v in r["losses"][:traj]])
    del r
    runs.clear()
    gc.collect()                    # policy <-> engine hooks form cycles
    torch.cuda.empty_cache()
    return res


def step_13b(layers=40, warmup=3, steps=5):
    res = {}
    for name, fp8, micros in (("fp8", True, (8, 4, 2)), ("bf16", False, (2,))):
        for micro in micros:
            pol = eng = None
            try:
                pol, eng = make_policy(WIDTHS["13b"], layers, fp8, micro)
                dev = batches(pol, micro)
                for s in range(warmup):
                    eng.train_step(dev[s % 2])
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                for s in range(steps):
                    eng.train_step(dev[s % 2])
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) / steps
                res[name] = dict(micro_pairs=micro, pairs_per_s=round(PAIRS_PER_GPU / dt, 3),
                                 peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
                break
            except torch.cuda.OutOfMemoryError:
                res.setdefault(name + "_oom_at", []).append(micro)
            finally:
                del pol, eng
                dev = None
                gc.collect()
                torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-13b", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_step.py measures on a GPU; none is visible")
    res = {"card": card()}
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    res["kernels"] = kernels()
    res["step_7b"] = step_7b()
    if not args.skip_13b:
        res["step_13b"] = step_13b()
    res["clock"] = sampler.stop()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
