"""Time the frozen-base GEMMs of one LLaVA-1.5 LoRA-DPO step shape by shape, against cuBLAS on the same card.

    python tools/gemm_step_shapes.py --out DIR [--dims 7b|13b] [--stalls] [--min-seconds 1.0]

The calls are recorded, not re-typed: one training step of a one-decoder-layer LoRA(r=64) policy at the benchmark's
batch (8 pairs, micro-batches of 4, T = 1135) runs with ops.gemm, ops.gemm_dual and ops.gemm_swiglu_bwd wrapped, so
every shape keeps its operand layouts, epilogue and LoRA second source. A decoder layer's calls repeat once per layer
per step: 32 times for LLaVA-1.5-7B (--dims 7b, hidden 4096, ffn 11008), 40 times for LLaVA-1.5-13B (--dims 13b,
hidden 5120, ffn 13824). Per frozen-base shape, in one process, alternating between the variants:

  ours           the shipped path, automatic tile choice
  ours-register  the same launch with the register epilogue (rlaifv_gemm_set_tuning(0, 2)): threads store C straight
                 from their accumulators instead of through shared memory and TMA stores; same bits
  ours-mainloop  the same launch with the epilogue skipped (rlaifv_gemm_set_tuning(0, 1)): the difference to
                 `ours` is the epilogue the tensor cores wait for
  cublas         torch.matmul on the same tensors and layouts (x @ W.t(), dy @ W), no fused epilogue and no second
                 source: compare it with ours-mainloop

Each variant gets at least --min-seconds of timed work (CUDA events, after warm-up). One more line sums every rank-r
adapter GEMM of the step. --stalls also builds the library with -DRLAIFV_GEMM_STALLS into DIR and reports, per shape,
the consumers' cycles waiting on `full` barriers, the producer's waiting on `empty` barriers and the epilogue cycles
(gemm.cu: GemmStall). The card name, power limit and the SM clock sampled during the timing are part of the output.
Writes DIR/gemm_step_shapes.json.
"""
import argparse
import ctypes
import importlib.util
import json
import math
import os
import subprocess
import sys
import threading
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

# decoder widths and layers of each model: the recorded one-layer calls repeat `layers` times per step
DIMS = {"7b": dict(hidden_size=4096, intermediate_size=11008, num_heads=32, layers=32),
        "13b": dict(hidden_size=5120, intermediate_size=13824, num_heads=40, layers=40)}
PAIRS, MICRO_PAIRS = 8, 4   # bench.py: pairs per step and per micro-batch
STALL_FIELDS = ("ctas", "tiles", "cons_total", "cons_full_wait", "cons_epilogue", "prod_total", "prod_empty_wait")


def shape_names(H, F, lora=True):
    """Names of the frozen-base shapes: (function, N, K) -> name; N / K are the launch's output columns / first-source
    depth. The two H x H launches are told apart by the layout of B. Full fine-tuning (lora=False) runs the same
    shapes as plain gemm launches, the fused SwiGLU backward included."""
    dual = "gemm_dual" if lora else "gemm"
    return {(dual, 3 * H, H): "qkv forward", (dual, H, H, False): "o forward",
            (dual, 2 * F, H): "gate|up forward", (dual, H, F): "down forward",
            ("gemm_swiglu_bwd", F, H): "down dgrad (SwiGLU bwd)", (dual, H, 2 * F): "gate|up dgrad",
            (dual, H, H, True): "o dgrad", (dual, H, 3 * H): "qkv dgrad"}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="output directory (JSON, stall-accounting build)")
    ap.add_argument("--dims", choices=sorted(DIMS), default="7b", help="decoder widths: LLaVA-1.5-7B or -13B")
    ap.add_argument("--min-seconds", type=float, default=1.0, help="timed work per variant and shape")
    ap.add_argument("--adapter-seconds", type=float, default=0.2, help="timed work per adapter GEMM shape")
    ap.add_argument("--stalls", action="store_true", help="build and run the stall-accounting variant too")
    ap.add_argument("--no-cublas", action="store_true")
    ap.add_argument("--group-m", type=int, default=0, help="rlaifv_gemm_set_tuning group size (0: library default)")
    ap.add_argument("--l2", type=int, default=-1, help="rlaifv_gemm_set_l2 bits (-1: automatic policy)")
    ap.add_argument("--tag", default="", help="label stored with the results")
    return ap.parse_args(argv)


def build_stall_library(out_dir):
    """gemm.cu with -DRLAIFV_GEMM_STALLS, linked with the in-tree objects of the other sources (build.py's flags)."""
    spec = importlib.util.spec_from_file_location("_rlaifv_build", os.path.join(REPO, "rlaif-v_b200", "build.py"))
    bld = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bld)
    bld.build(verbose=False)
    d = os.path.join(os.path.abspath(out_dir), "stalls")
    os.makedirs(d, exist_ok=True)
    obj = os.path.join(d, "gemm_stalls.o")
    cmd = [bld.NVCC] + bld.FLAGS + ["-DRLAIFV_GEMM_STALLS", "-Xptxas", "-v", "-c", os.path.join(bld.CSRC, "gemm.cu"),
                                    "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    spills = [ln for ln in r.stderr.splitlines() if "spill" in ln and not ln.strip().startswith("0 bytes spill")
              and " 0 bytes spill stores, 0 bytes spill loads" not in ln]
    others = [os.path.join(bld.OBJ, s[:-3] + ".o") for s in bld._sources() if s != "gemm.cu"]
    so = os.path.join(d, "librlaifv_b200_stalls.so")
    r = subprocess.run([bld.NVCC, "-shared", "-o", so, obj] + others + ["-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return so, spills


class ClockSampler:
    """nvidia-smi SM clock and power samples while the timings run (read-only queries)."""

    def __init__(self):
        self.lines, self.proc = [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,power.draw",
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=lambda: [self.lines.append(x.strip()) for x in self.proc.stdout],
                             daemon=True).start()
        except OSError:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {"sm_mhz_median": None, "power_w_median": None, "samples": 0}
        self.proc.terminate()
        self.proc.wait()
        sm, pw = [], []
        for ln in self.lines:
            try:
                a, b = [float(x) for x in ln.split(",")[:2]]
            except ValueError:
                continue
            sm.append(a)
            pw.append(b)
        med = lambda v: sorted(v)[len(v) // 2] if v else None    # noqa: E731
        return {"sm_mhz_median": med(sm), "power_w_median": med(pw), "samples": len(sm)}


def card_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_max_clock"] = [x.strip() for x in q.split(",")[:2]]
    except (OSError, ValueError, subprocess.SubprocessError):
        info["power_limit"] = info["sm_max_clock"] = "unknown"
    return info


def record_step_calls(dims, lora=True):
    """One DPO training step of a one-layer policy at the benchmark's batch, LoRA(r=64) or (lora=False) full
    fine-tuning: every GEMM call with its tensors."""
    import torch
    import bench
    from rlaifv_b200 import ops
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    policy = LlavaDPOPolicy(LlavaDims(num_layers=1, hidden_size=dims["hidden_size"],
                                      intermediate_size=dims["intermediate_size"], num_heads=dims["num_heads"]),
                            torch.device("cuda", 0), seed=0)
    if lora:
        policy.enable_lora(r=64, alpha=16)
    engine = DPOStepEngine(policy, lr=1e-5, weight_decay=0.01, total_steps=2672, micro_pairs=MICRO_PAIRS)
    hb = bench.synthetic_batch(0, 0, PAIRS)
    batch = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()}
    batch["ref_win_logp"] = torch.zeros(PAIRS, device="cuda")
    batch["ref_rej_logp"] = torch.zeros(PAIRS, device="cuda")
    calls, orig = [], {n: getattr(ops, n) for n in ("gemm", "gemm_dual", "gemm_swiglu_bwd")}

    def wrap(name):
        def f(*a, **kw):
            r = orig[name](*a, **kw)
            calls.append((name, a, dict(kw), r))
            return r
        return f

    for n in orig:
        setattr(ops, n, wrap(n))
    try:
        engine.train_step(batch, optimizer_step=False)
        torch.cuda.synchronize()
    finally:
        for n, f in orig.items():
            setattr(ops, n, f)
    return calls, (policy, engine, batch)


def describe(name, a, kw, r):
    """(signature, shape dict) of one recorded call. The signature is what makes two calls the same launch."""
    t_sig = tuple((tuple(x.shape), tuple(x.stride())) if hasattr(x, "shape") else x for x in a)
    kw_sig = tuple(sorted((k, (tuple(v.shape), tuple(v.stride())) if hasattr(v, "shape") else v) for k, v in kw.items()))
    if name == "gemm":
        a_mn, b_mn = kw.get("a_mn", False), kw.get("b_mn", False)
        M, N = r.shape
        K = a[0].shape[0] if a_mn else a[0].shape[1]
        k2 = 0
        epi = "+".join(e for e in ("bias", "residual") if kw.get(e) is not None) or "none"
        if kw.get("accumulate"):
            epi = "accumulate"
    elif name == "gemm_dual":
        a_mn, b_mn = False, kw.get("b_mn", False)
        M, N = a[4].shape
        K, k2 = a[0].shape[1], kw["k2"]
        epi = "residual" if kw.get("residual") is not None else "none"
    else:
        a_mn, b_mn = False, kw.get("b_mn", True)
        M, K = a[0].shape
        N = a[1].shape[1] if b_mn else a[1].shape[0]
        k2 = kw["a2"].shape[1] if kw.get("a2") is not None else 0
        epi = "swiglu_bwd"
    d = {"fn": name, "M": M, "N": N, "K": K, "K2": k2, "A": "MN" if a_mn else "K", "B": "MN" if b_mn else "K",
         "epilogue": epi}
    return (name, t_sig, kw_sig), d


def shape_name(d, dims, lora=True):
    H = dims["hidden_size"]
    key = (d["fn"], d["N"], d["K"])
    if d["fn"] != "gemm_swiglu_bwd" and d["N"] == d["K"] == H:
        key = key + (d["B"] == "MN",)
    return shape_names(H, dims["intermediate_size"], lora).get(key)


def is_adapter(d, r=64):
    return d["fn"] == "gemm" and any(x in (r, 2 * r, 3 * r) for x in (d["M"], d["N"], d["K"]))


def time_variants(variants, min_seconds, rounds=4):
    """variants: {name: fn}. Alternates the variants in `rounds` blocks; returns ms per call for each."""
    import torch
    for f in variants.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    est = {}
    for n, f in variants.items():
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(3):
            f()
        e.record()
        e.synchronize()
        est[n] = max(s.elapsed_time(e) / 3, 1e-3)
    reps = {n: max(1, math.ceil(min_seconds * 1e3 / est[n] / rounds)) for n in variants}
    tot = {n: 0.0 for n in variants}
    cnt = {n: 0 for n in variants}
    for _ in range(rounds):
        for n, f in variants.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(reps[n]):
                f()
            e.record()
            e.synchronize()
            tot[n] += s.elapsed_time(e)
            cnt[n] += reps[n]
    return {n: tot[n] / cnt[n] for n in variants}


def main(argv=None):
    args = parse_args(argv)
    os.makedirs(args.out, exist_ok=True)
    stall_so = None
    dims = DIMS[args.dims]
    result = {"tag": args.tag, "group_m": args.group_m, "l2": args.l2, "dims": args.dims}
    if args.stalls:
        stall_so, spills = build_stall_library(args.out)
        result["stall_build"] = {"library": os.path.relpath(stall_so, args.out), "ptxas_spill_lines": spills}
        print("stall-accounting build: %s (%d ptxas lines with spills)" % (stall_so, len(spills)), flush=True)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gemm_step_shapes.py times kernels on a CUDA device: none is visible")
    from rlaifv_b200 import lib, ops
    L = lib.load()
    result["card"] = card_info()
    for tile_n in (512, 256):
        n = ctypes.c_int(0)
        try:
            lib.call("rlaifv_gemm_max_active_clusters", tile_n, ctypes.byref(n))
            result["card"]["max_active_clusters_tile%d" % tile_n] = n.value
        except AttributeError:               # a library from before the query existed
            result["card"]["max_active_clusters_tile%d" % tile_n] = None
    print("card:", json.dumps(result["card"]), flush=True)
    if args.group_m or args.l2 >= 0:
        L.rlaifv_gemm_set_tuning(args.group_m, 0)
        L.rlaifv_gemm_set_l2(args.l2)

    calls, keep = record_step_calls(dims)
    uniq = {}
    for name, a, kw, r in calls:
        sig, d = describe(name, a, kw, r)
        if sig not in uniq:
            uniq[sig] = [d, (name, a, kw, r), 0]
        uniq[sig][2] += 1
    # in LoRA mode every frozen-base decoder GEMM is a dual-source launch (gemm_dual / gemm_swiglu_bwd)
    frozen = [(v[0], v[1], v[2]) for v in uniq.values() if v[0]["fn"] != "gemm"]
    adapters = [(v[0], v[1], v[2]) for v in uniq.values() if is_adapter(v[0])]
    print("recorded %d GEMM calls (%d distinct); %d frozen-base shapes, %d adapter shapes"
          % (len(calls), len(uniq), len(frozen), len(adapters)), flush=True)

    def ours_fn(call):
        name, a, kw, _ = call
        f = getattr(ops, name)
        return lambda: f(*a, **kw)

    def debug_fn(call, bits):
        g = ours_fn(call)

        def f():
            L.rlaifv_gemm_set_tuning(0, bits)
            g()
            L.rlaifv_gemm_set_tuning(0, 0)
        return f

    def cublas_fn(call, d):
        name, a, kw, _ = call
        x, w = a[0], a[1]
        out = torch.empty((d["M"], d["N"]), dtype=torch.bfloat16, device="cuda")
        wt = w if d["B"] == "MN" else w.t()
        return lambda: torch.matmul(x, wt, out=out)

    sampler = ClockSampler()
    sampler.start()
    rows = []
    ad_ms = ad_fl = 0.0
    ad_calls = 0
    try:   # the sampler is a child process: stop it whatever happens to the timings
        for d, call, count in frozen:
            per_step = count * dims["layers"]      # the recorded step already holds both micro-batches
            v = {"ours": ours_fn(call), "ours-register": debug_fn(call, 2), "ours-mainloop": debug_fn(call, 1)}
            if not args.no_cublas:
                v["cublas"] = cublas_fn(call, d)
            ms = time_variants(v, args.min_seconds)
            fl = 2.0 * d["M"] * d["N"] * (d["K"] + d["K2"])
            fl_cublas = 2.0 * d["M"] * d["N"] * d["K"]
            row = dict(d, name=shape_name(d, dims), calls_per_step=per_step, gflop=fl / 1e9)
            for n, t in ms.items():
                f = fl_cublas if n == "cublas" else fl
                row[n] = {"ms_per_call": t, "ms_per_step": t * per_step, "tflops": f / (t * 1e-3) / 1e12}
            if "cublas" in ms:
                rate = fl_cublas / (ms["cublas"] * 1e-3)
                row["ms_per_step_saved_at_cublas_rate"] = (ms["ours"] - fl / rate * 1e3) * per_step
            rows.append(row)
            print("%-26s M=%d N=%d K=%d+%d A %s B %s epi %-10s x%-4d" % (row["name"], d["M"], d["N"], d["K"], d["K2"],
                  d["A"], d["B"], d["epilogue"], per_step) +
                  "  ".join(" %s %.3f ms %.0f TF/s" % (n, row[n]["ms_per_call"], row[n]["tflops"]) for n in ms), flush=True)
        for d, call, count in adapters:
            per_step = count * dims["layers"]
            t = time_variants({"ours": ours_fn(call)}, args.adapter_seconds, rounds=1)["ours"]
            ad_ms += t * per_step
            ad_fl += 2.0 * d["M"] * d["N"] * d["K"] * per_step
            ad_calls += per_step
    finally:
        result["clocks"] = sampler.stop()
    result["shapes"] = rows
    result["adapters"] = {"calls_per_step": ad_calls, "ms_per_step": ad_ms, "tflop_per_step": ad_fl / 1e12,
                          "tflops": ad_fl / (ad_ms * 1e-3) / 1e12 if ad_ms else None}
    tot = {n: sum(r[n]["ms_per_step"] for r in rows if n in r) for n in ("ours", "ours-register", "ours-mainloop",
                                                                            "cublas")}
    result["total_ms_per_step"] = tot
    print("frozen-base GEMMs per step: " + ", ".join("%s %.1f ms" % kv for kv in tot.items()))
    print("rank-64 adapter GEMMs per step: %d calls, %.1f ms, %.2f TFLOP" % (ad_calls, ad_ms, ad_fl / 1e12))
    print("clocks during the timings:", json.dumps(result["clocks"]), flush=True)

    if stall_so:
        lib._lib = None                      # every following launch goes to the stall-accounting build
        lib.LIB_PATH = stall_so
        S = lib.load()
        S.rlaifv_gemm_stalls_read.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
        buf = (ctypes.c_ulonglong * len(STALL_FIELDS))()
        if args.group_m or args.l2 >= 0:
            S.rlaifv_gemm_set_tuning(args.group_m, 0)
            S.rlaifv_gemm_set_l2(args.l2)
        for row, (d, call, _) in zip(rows, frozen):
            f = ours_fn(call)
            for _ in range(3):
                f()
            S.rlaifv_gemm_stalls_read(buf, 1)
            for _ in range(10):
                f()
            S.rlaifv_gemm_stalls_read(buf, 1)
            st = dict(zip(STALL_FIELDS, list(buf)))
            st["cons_full_wait_frac"] = st["cons_full_wait"] / max(1, st["cons_total"])
            st["cons_epilogue_frac"] = st["cons_epilogue"] / max(1, st["cons_total"])
            st["prod_empty_wait_frac"] = st["prod_empty_wait"] / max(1, st["prod_total"])
            row["stalls"] = st
            print("stalls %-26s consumers: full-wait %.1f %%, epilogue %.1f %%; producer: empty-wait %.1f %%; "
                  "%.1f tiles per CTA" % (row["name"], 100 * st["cons_full_wait_frac"], 100 * st["cons_epilogue_frac"],
                                          100 * st["prod_empty_wait_frac"], st["tiles"] / max(1, 2 * st["ctas"])),
                  flush=True)
    with open(os.path.join(args.out, "gemm_step_shapes.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    del keep


if __name__ == "__main__":
    main()
