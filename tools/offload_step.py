"""Full-parameter DPO of LLaVA-1.5-7B on one GPU with the offloaded optimizer (zero2.OffloadAdamW), measured.

    python tools/offload_step.py --out DIR [--skip-identity] [--skip-config-b] [--steps 5] [--warmup 3]

1. Identity at real widths: LLaVA-1.5-7B dimensions at --identity-layers decoder layers (default 4). Three optimizer
   steps with the on-device Zero2AdamW, then three from the same seed with offload and a device budget that keeps only
   embed, projector, layer0 and layer1 resident. Reports whether the metrics, every bf16 parameter and the fp32
   master / exp_avg / exp_avg_sq are bit-identical.
2. Config (b): full width and depth, full fine-tuning, 8 pairs of T = 1135 (bench.py's synthetic batch), offload on,
   with the engine's own default device budget, as the training CLI plans it with --micro_pairs --micro-pairs and
   --model_max_length --max-len: what is free after the activations of the micro-batch at max-len and the fp32
   embedding gradient. Step 0 (no update) is checked against ln 2, then --warmup and --steps timed steps.
3. One JSON line (also DIR/offload_step.json): pairs/s and ms/step; resident, streamed and pinned bytes; peak device
   memory; the optimizer's exposed time per step (end of the last backward kernel -> last update done, and -> last
   D2H done); the H2D and D2H GB/s the streams achieved during the step; a plain cudaMemcpyAsync H2D and D2H of the
   same pinned buffer, one direction at a time and both at the same moment on two streams; the staging ring on its
   own (no backward beside it); the median SM clock; the GPU name and power limit.

    python tools/offload_step.py --omnilmm --tune-clip {0,1} --out DIR [--max-len 1024] [--micro-pairs 2]

    python tools/offload_step.py --optim adamw_8bit --out DIR [--steps 5] [--warmup 3]

AdamW with blockwise 8-bit moments, written to DIR/offload_step_8bit.json (each leg can be skipped, see --help):
1. Kernel throughput: rlaifv_adamw8bit_step against the fp32 adamw_kernel on one 2^30-element shard, CUDA events, GB/s
   of algorithmic bytes (master 8 B, grad / param 4 B, codes 2 B per element, absmax 16 B per 256).
2. Identity: LLaVA-1.5-7B widths at --identity-layers layers, three steps on the device, then offloaded with a mixed
   and an all-streamed split: metrics, bf16 parameters, master, codes and absmax bit for bit.
3. Loss trajectory: 7B widths at 2 layers, 20 steps of each optimizer from one seed on bench.py's inputs: the largest
   |delta loss| and the master weights' relative difference.
4. Config (b) offloaded with adamw_torch and adamw_8bit, alternating (torch, 8-bit, torch, 8-bit) in one process.
5. 13B full fine-tuning (1 pair at 2048 tokens per micro-batch) and OmniLMM-12B with a trained tower, with 8-bit
   moments: measured where MemAvailable holds the streamed state, otherwise the refusal with MemAvailable recorded.

OmniLMM-12B (config d), written to DIR/offload_step_omnilmm.json:
1. Identity at OmniLMM widths, --identity-layers decoder layers and --identity-eva-blocks EVA blocks, in both tower
   modes: three steps on the device, then three from the same seed offloaded with a mixed split (embed, resampler and
   the first tower / decoder buckets resident) and with every bucket streamed. Bit identity of the metrics, the bf16
   parameters of decoder, resampler and tower, and the fp32 master / exp_avg / exp_avg_sq; with a frozen tower, also
   that its weights are still the initial ones.
2. Config (d): the whole model, 8 pairs of 448 px and 512-token responses (T = 625, bench.py's OmniLMM batch), the tower
   mode of --tune-clip, the engine's default budget for --micro-pairs at --max-len; the same report as config (b).
3. The trained-tower recipe (--micro_pairs 1): the planner's split and the host memory it needs. It runs where
   MemAvailable holds the streamed state; otherwise the optimizer's refusal is recorded.
"""
import argparse
import gc
import json
import math
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

import bench  # noqa: E402  (synthetic_batch, ClockSampler, PAIRS_PER_GPU; bench.py itself is not changed)


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--micro-pairs", type=int, default=2, help="config (b)'s micro-batch (--micro_pairs of the CLI)")
    ap.add_argument("--max-len", type=int, default=None,
                    help="model_max_length the engine sizes the activation reserve for (default: the LLaVA recipe's "
                         "2048; 1024 with --omnilmm)")
    ap.add_argument("--identity-layers", type=int, default=4)
    ap.add_argument("--skip-identity", action="store_true")
    ap.add_argument("--skip-config-b", action="store_true")
    ap.add_argument("--omnilmm", action="store_true",
                    help="OmniLMM-12B (config d) instead of LLaVA-1.5-7B: identity in both tower modes, config (d) "
                         "with the tower mode of --tune-clip, and the trained-tower plan")
    ap.add_argument("--tune-clip", type=int, choices=(0, 1), default=0,
                    help="with --omnilmm: 1 trains the EVA tower in the config (d) leg, 0 freezes it")
    ap.add_argument("--identity-eva-blocks", type=int, default=4)
    ap.add_argument("--skip-config-d", action="store_true")
    ap.add_argument("--skip-trained-tower", action="store_true")
    ap.add_argument("--optim", choices=("adamw_torch", "adamw_8bit"), default="adamw_torch",
                    help="adamw_8bit: the 8-bit legs (kernel, identity, loss trajectory, config (b) both ways, 13B, "
                         "trained-tower OmniLMM) instead of the legs above")
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-trajectory", action="store_true")
    ap.add_argument("--skip-13b", action="store_true")
    args = ap.parse_args(argv)
    if args.max_len is None:
        args.max_len = 1024 if args.omnilmm else 2048
    return args


def gpu_name_and_power():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:          # noqa: BLE001 — reported, not fatal
        return "unknown (%s)" % e, None


def make_engine(layers, micro, offload_budget=None, offload=False, seed=0, optim="adamw_torch"):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    policy = LlavaDPOPolicy(LlavaDims(num_layers=layers), torch.device("cuda", 0), seed=seed)
    eng = DPOStepEngine(policy, lr=5e-7, weight_decay=0.01, total_steps=2672, micro_pairs=micro,
                        offload_optimizer=offload, offload_budget=offload_budget, optim=optim)
    return eng


def add_reference_logps(policy, batches, B, micro):
    """Frozen-reference log-probs = the initial policy's (step-0 loss = ln 2), as bench.py does."""
    for hb in batches:
        rw, rr = [], []
        for lo in range(0, B, micro):
            hi = min(B, lo + micro)
            ids = torch.cat([hb["concatenated_input_ids"][lo:hi], hb["concatenated_input_ids"][B + lo:B + hi]])
            lab = torch.cat([hb["concatenated_labels"][lo:hi], hb["concatenated_labels"][B + lo:B + hi]])
            out = policy.forward_logps(ids, lab, hb["images"][lo:hi], keep_stash=False)
            rw.append(out["logp"][: hi - lo].float().cpu())
            rr.append(out["logp"][hi - lo:].float().cpu())
        hb["ref_win_logp"] = torch.cat(rw)
        hb["ref_rej_logp"] = torch.cat(rr)


def identity(layers):
    """Three steps on the device, three offloaded from the same seed; compare everything bit for bit."""
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    B, micro = 4, 2
    batches = [bench.synthetic_batch(0, s, B) for s in range(3)]
    results = {}
    for mode in ("device", "offload"):
        budget = None
        if mode == "offload":
            budget = STATE_BYTES_PER_ELEM * sum(sizes[n] for n in ("embed", "projector", "layer0", "layer1"))
        eng = make_engine(layers, micro, offload_budget=budget, offload=mode == "offload")
        if mode == "device":
            sizes = {b.name: b.size for b in eng.policy.trainable_buckets()}
            add_reference_logps(eng.policy, batches, B, micro)
        metrics = [eng.train_step(hb).clone() for hb in batches]
        eng.opt.wait_all()
        torch.cuda.synchronize()
        sd = eng.opt.state_dict()
        results[mode] = {"metrics": torch.stack(metrics).cpu(), "params": eng.policy.store.flat.cpu(),
                         **{k: sd[k].cpu() for k in ("master", "exp_avg", "exp_avg_sq")}}
        if mode == "offload":
            split = {"resident": eng.opt.resident_names, "streamed": eng.opt.streamed_names}
            eng.opt.close()
        del eng, sd
        gc.collect()                  # the policy and the engine reference each other (the backward hooks)
        torch.cuda.empty_cache()
    d, o = results["device"], results["offload"]
    return {"layers": layers, "pairs": B, "micro_pairs": micro, "steps": 3, **split,
            "metrics_identical": bool(torch.equal(d["metrics"], o["metrics"])),
            "params_identical": bool(torch.equal(d["params"], o["params"])),
            **{k + "_identical": bool(torch.equal(d[k], o[k])) for k in ("master", "exp_avg", "exp_avg_sq")}}


def plain_copy_gbs(host, reps=5):
    """cudaMemcpyAsync H2D and D2H of a pinned buffer (torch copy_ with non_blocking), CUDA-event timed."""
    dev = torch.empty(host.numel(), dtype=host.dtype, device="cuda")
    s = torch.cuda.Stream()
    out = {}
    for name, fn in (("h2d", lambda: dev.copy_(host, non_blocking=True)),
                     ("d2h", lambda: host.copy_(dev, non_blocking=True))):
        with torch.cuda.stream(s):
            fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            for _ in range(reps):
                fn()
            e1.record(s)
        s.synchronize()
        out[name] = reps * host.numel() * host.element_size() / (e0.elapsed_time(e1) * 1e-3) / 1e9
    del dev
    return out


def concurrent_copy_gbs(host, reps=5):
    """A plain H2D of the first half of a pinned buffer and a D2H into its second half, at the same moment on two
    streams (the D2H writes back what the buffer held). GB/s per direction."""
    h = host.numel() // 2
    src, dst = host[:h], host[h:2 * h]
    dev_in = torch.empty(h, dtype=host.dtype, device="cuda")
    dev_out = dst.to("cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record(s1)
    ev[2].record(s2)
    with torch.cuda.stream(s1):
        for _ in range(reps):
            dev_in.copy_(src, non_blocking=True)
    with torch.cuda.stream(s2):
        for _ in range(reps):
            dst.copy_(dev_out, non_blocking=True)
    ev[1].record(s1)
    ev[3].record(s2)
    torch.cuda.synchronize()
    b = reps * h * host.element_size()
    out = {"h2d": b / (ev[0].elapsed_time(ev[1]) * 1e-3) / 1e9, "d2h": b / (ev[2].elapsed_time(ev[3]) * 1e-3) / 1e9}
    del dev_in, dev_out
    return out


def ring_alone_gbs(opt, reps=3):
    """rlaifv_adamw_offload_bucket on its own (no backward beside it) over a scratch range of 2^27 elements, through
    the optimizer's staging ring: state GB/s per direction (H2D and D2H run at the same time)."""
    from rlaifv_b200 import ops
    n = min(1 << 27, opt.host_master.numel())
    host = [torch.zeros(n, dtype=torch.float32).pin_memory() for _ in range(3)]
    grad = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    param = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(opt.h2d_stream)
    from rlaifv_b200 import lib
    with torch.cuda.stream(s), lib.use_stream(s):
        for step in range(1, reps + 1):
            ops.adamw_offload_bucket(*host, grad, param, n, opt.ring, opt.slot_elems, 1e-6, 0.9, 0.999, 1e-8, 0.0,
                                     step, opt.h2d_stream, opt.d2h_stream)
    e1.record(opt.d2h_stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    del host, grad, param
    return {"slots": opt.ring.shape[0], "slot_elems": opt.slot_elems, "elements": n, "reps": reps, "ms": ms,
            "gbs_each_way": reps * 12 * n / (ms * 1e-3) / 1e9}


def config_b(args, optim="adamw_torch"):
    """Config (b) through the engine's own default device budget, as `train_llava15.py --deepspeed
    script/zero2_offload.json --micro_pairs M --model_max_length L` plans it."""
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    B = bench.PAIRS_PER_GPU
    dims = LlavaDims(max_len=args.max_len)
    T = bench.PROMPT_LEN + bench.RESP_LEN - 1 + dims.num_patches
    gc.collect()
    torch.cuda.empty_cache()
    policy = LlavaDPOPolicy(dims, torch.device("cuda", 0), seed=0)
    return timed_offload_run(args, policy, [bench.synthetic_batch(0, s, B) for s in range(2)], B, T, optim)


def timed_offload_run(args, policy, host_batches, B, T, optim="adamw_torch"):
    """The measured run of a full-size policy with the engine's own default device budget for --micro-pairs at
    dims.max_len: step 0 against ln 2, --warmup and --steps timed steps, then the copy rates."""
    from rlaifv_b200.engine import DPOStepEngine
    import rlaifv_b200.zero2 as z
    dims = policy.dims
    micro = args.micro_pairs
    free = torch.cuda.mem_get_info()[0]
    reserve = policy.activation_reserve_bytes(micro, dims.max_len)
    t0 = time.perf_counter()
    eng = DPOStepEngine(policy, lr=5e-7, weight_decay=0.01, total_steps=2672, micro_pairs=micro,
                        offload_optimizer=True, batch_pairs=B, optim=optim)
    setup_s = time.perf_counter() - t0
    opt = eng.opt
    add_reference_logps(policy, host_batches, B, micro)
    batches = [{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()} for hb in host_batches]
    while True:
        try:
            loss0 = float(eng.train_step(batches[0], optimizer_step=False)[0].item())
            break
        except torch.OutOfMemoryError:
            policy._stash = None
            policy._bufs.clear()
            torch.cuda.empty_cache()
            if micro > 1:
                micro = max(1, micro // 2)
                eng.micro_pairs = micro
            else:
                raise
    # exposed optimizer time: the backward's last kernel is enqueued when finish_step is called
    marks = []
    orig_finish = opt.finish_step

    def timed_finish():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record(torch.cuda.current_stream())
        orig_finish()                        # world 1: ends with the current stream waiting for every update
        ev[1].record(torch.cuda.current_stream())
        ev[2].record(opt.d2h_stream)
        marks.append(ev)
    opt.finish_step = timed_finish

    def run(n):
        for s in range(n):
            eng.train_step(batches[s % len(batches)])
        opt.wait_all()
        torch.cuda.current_stream().wait_stream(opt.d2h_stream)    # the last step's stores belong to the window

    run(args.warmup)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    marks.clear()
    sampler = bench.ClockSampler(0)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(args.steps)
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    ms = e0.elapsed_time(e1) / args.steps
    exposed_upd = sorted(a.elapsed_time(b) for a, b, _ in marks)
    exposed_d2h = sorted(a.elapsed_time(c) for a, _, c in marks)
    peak_alloc, peak_reserved = torch.cuda.max_memory_allocated(), torch.cuda.max_memory_reserved()

    # copy rates the streams achieved: one more step with each offloaded bucket's H2D / D2H spans event-timed
    spans = []
    entry = "adamw_offload_bucket" if optim == "adamw_torch" else "adamw8bit_offload_bucket"
    orig_off = getattr(z.ops, entry)

    def timed_off(hm, *a, **kw):
        h2d, d2h = a[-2], a[-1]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record(h2d)
        ev[2].record(d2h)
        orig_off(hm, *a, **kw)
        ev[1].record(h2d)
        ev[3].record(d2h)
        spans.append((ev, z.state_bytes(hm.numel(), optim)))
    setattr(z.ops, entry, timed_off)
    try:
        run(1)
        torch.cuda.synchronize()
    finally:
        setattr(z.ops, entry, orig_off)
    streamed_bytes = sum(b for _, b in spans)
    h2d_ms = sum(ev[0].elapsed_time(ev[1]) for ev, _ in spans)
    d2h_ms = sum(ev[2].elapsed_time(ev[3]) for ev, _ in spans)
    first_h2d, last_d2h = spans[0][0][0], spans[-1][0][3]
    pipeline_ms = first_h2d.elapsed_time(last_d2h)
    plain = plain_copy_gbs(opt.host_master[: min(opt.host_master.numel(), 1 << 28)])
    plain["both_at_once"] = concurrent_copy_gbs(opt.host_master[: min(opt.host_master.numel(), 1 << 28)])
    ring_alone = ring_alone_gbs(opt) if optim == "adamw_torch" else None
    gbs = lambda b, t: b / (t * 1e-3) / 1e9 if t > 0 else None           # noqa: E731
    med = lambda xs: xs[len(xs) // 2] if xs else None                     # noqa: E731
    out = {
        "pairs": B, "T": T, "micro_pairs": micro, "max_len": dims.max_len, "steps": args.steps, "warmup": args.warmup,
        "step0_loss": loss0, "ln2": math.log(2.0), "step0_ok": abs(loss0 - math.log(2.0)) < 1e-3,
        "ms_per_step": ms, "pairs_per_s": B / (ms * 1e-3),
        "device_free_before_optimizer_bytes": free, "activation_reserve_bytes": reserve,
        "optim": optim, "device_budget_bytes": opt.device_budget,
        "resident_bytes": sum(z.state_bytes(s1 - s0, optim) for (b, s0, s1, _), st in zip(opt.slices, opt._is_streamed)
                              if not st),
        "streamed_bytes": opt.pinned_bytes, "pinned_host_bytes": opt.pinned_bytes,
        "resident_buckets": len(opt.resident_names), "streamed_buckets": len(opt.streamed_names),
        "optimizer_setup_s": setup_s,
        "peak_device_allocated_bytes": peak_alloc, "peak_device_reserved_bytes": peak_reserved,
        "exposed_optimizer_ms_to_update": med(exposed_upd), "exposed_optimizer_ms_to_d2h": med(exposed_d2h),
        "streaming": {"bytes_each_way": streamed_bytes, "h2d_busy_ms": h2d_ms, "d2h_busy_ms": d2h_ms,
                      "h2d_gbs": gbs(streamed_bytes, h2d_ms), "d2h_gbs": gbs(streamed_bytes, d2h_ms),
                      "first_h2d_to_last_d2h_ms": pipeline_ms},
        "plain_copy_gbs": plain,
        "ring_alone": ring_alone,
        "sm_clock": clocks,
    }
    opt.close()
    return out


# ---- OmniLMM-12B (config d) ---------------------------------------------------------------------------------------
def omni_policy(layers, eva_blocks, tune_clip, max_len, seed=0):
    """OmniLMM policy at real widths: `layers` decoder layers, `eva_blocks` live EVA blocks (None: all 63)."""
    from rlaifv_b200.eva_tower import EvaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy, omnilmm_dims
    dims = omnilmm_dims(num_layers=layers, max_len=max_len)
    eva = EvaDims() if eva_blocks is None else EvaDims(depth=eva_blocks + 1)
    return OmniLMMDPOPolicy(dims, torch.device("cuda", 0), seed=seed, eva_dims=eva, tune_clip=bool(tune_clip))


def omni_batches(policy, B, n=2):
    """bench.py's OmniLMM batch (T = 625) with 448 px pixels in place of the tower's tokens, as bench.py builds it."""
    out = []
    for s in range(n):
        hb = bench.synthetic_omni_batch(0, s, B, policy.dims)
        g = torch.Generator().manual_seed(4321 + s)
        img = policy.tower.dims.img_size
        hb["images"] = torch.randn(B, 3, img, img, generator=g).pin_memory()
        out.append(hb)
    return out


def omni_snapshot(eng):
    pol = eng.policy
    sd = eng.opt.state_dict()
    return {"params": torch.cat([pol.store.flat.cpu(), pol.resampler.flat.cpu(), pol.tower.flat.cpu()]),
            **{k: sd[k].cpu() for k in ("master", "exp_avg", "exp_avg_sq")}}


def omni_identity(layers, eva_blocks, tune_clip):
    """OmniLMM widths at `layers` decoder layers and `eva_blocks` EVA blocks, one tower mode: three steps on the device,
    then three offloaded from the same seed with a mixed split and with every bucket streamed."""
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    B, micro = 4, 2

    def engine(budget):
        pol = omni_policy(layers, eva_blocks, tune_clip, 1024)
        return DPOStepEngine(pol, lr=5e-7, weight_decay=0.01, total_steps=2672, micro_pairs=micro,
                             offload_optimizer=budget is not None, offload_budget=budget)

    eng = engine(None)
    sizes = {b.name: b.size for b in eng.policy.trainable_buckets()}
    batches = omni_batches(eng.policy, B, 3)
    add_reference_logps(eng.policy, batches, B, micro)
    dev_metrics = torch.stack([eng.train_step(hb).clone() for hb in batches]).cpu()
    eng.opt.wait_all()
    torch.cuda.synchronize()
    ref = omni_snapshot(eng)
    tower_frozen_ok = None
    if not tune_clip:                                    # the frozen tower's weights are the initial ones
        tower_frozen_ok = bool(torch.equal(eng.policy.tower.flat.cpu(),
                                           omni_policy(layers, eva_blocks, tune_clip, 1024).tower.flat.cpu()))
    del eng
    gc.collect()
    torch.cuda.empty_cache()
    first = ["embed", "resampler"] + (["eva_embed", "eva0"] if tune_clip else ["layer0"])
    out = {"layers": layers, "eva_blocks": eva_blocks, "tune_clip": bool(tune_clip), "pairs": B, "micro_pairs": micro,
           "steps": 3, "trainable_buckets": len(sizes), "tower_bit_unchanged": tower_frozen_ok, "splits": {}}
    for split, budget in (("mixed", STATE_BYTES_PER_ELEM * sum(sizes[n] for n in first)), ("all_streamed", 0)):
        eng = engine(budget)
        metrics = torch.stack([eng.train_step(hb).clone() for hb in batches]).cpu()
        eng.opt.wait_all()
        torch.cuda.synchronize()
        got = omni_snapshot(eng)
        out["splits"][split] = {
            "resident": eng.opt.resident_names, "streamed": len(eng.opt.streamed_names),
            "metrics_identical": bool(torch.equal(dev_metrics, metrics)),
            **{k + "_identical": bool(torch.equal(ref[k], got[k])) for k in ("params", "master", "exp_avg", "exp_avg_sq")}}
        eng.opt.close()
        del eng
        gc.collect()
        torch.cuda.empty_cache()
    return out


def mem_available():
    from rlaifv_b200.zero2 import _read_meminfo, mem_available_bytes
    return mem_available_bytes(_read_meminfo())


def config_d(args, tune_clip):
    """Config (d): the whole OmniLMM-12B (63 EVA blocks, 448 px, 32 decoder layers), 8 pairs of T = 625, through the
    engine's own default device budget, as `train_omnilmm.py --deepspeed script/zero2_offload.json --tune_clip ...
    --micro_pairs M --model_max_length L` plans it."""
    gc.collect()
    torch.cuda.empty_cache()
    B = bench.PAIRS_PER_GPU
    policy = omni_policy(32, None, tune_clip, args.max_len)
    T = bench.PROMPT_LEN + bench.RESP_LEN - 1 + policy.dims.num_query + 2
    out = timed_offload_run(args, policy, omni_batches(policy, B), B, T)
    out["tune_clip"] = bool(tune_clip)
    return out


def trained_tower_plan(args, optim="adamw_torch"):
    """The trained-tower recipe (--micro_pairs 1): the planner's numbers, then the run itself where MemAvailable holds
    the streamed state, otherwise the optimizer's refusal."""
    from rlaifv_b200.engine import DPOStepEngine
    gc.collect()
    torch.cuda.empty_cache()
    policy = omni_policy(32, None, 1, args.max_len)
    return planned_run(args, policy, omni_batches, bench.PROMPT_LEN + bench.RESP_LEN - 1 + policy.dims.num_query + 2,
                       optim)


def planned_run(args, policy, make_batches, T, optim="adamw_torch"):
    """The planner's split for `policy` with micro-batches of one pair and the host memory it needs; then the timed run
    where MemAvailable holds the streamed state, otherwise the optimizer's refusal."""
    from rlaifv_b200.zero2 import (DEFAULT_SLOT_ELEMS, DEFAULT_SLOTS, DEVICE_MARGIN, HOST_MARGIN, offload_plan,
                                   ring_bytes, ring_slot_elems, state_bytes)
    gc.collect()
    torch.cuda.empty_cache()
    B, micro = bench.PAIRS_PER_GPU, 1
    sizes = [(b.name, b.size) for b in policy.trainable_buckets()]
    free = torch.cuda.mem_get_info()[0]
    reserve = policy.activation_reserve_bytes(micro, policy.dims.max_len)
    ring = ring_bytes(DEFAULT_SLOTS, ring_slot_elems(max(n for _, n in sizes), DEFAULT_SLOT_ELEMS, optim), optim)
    budget = free - reserve - ring - DEVICE_MARGIN
    resident, streamed = offload_plan(sizes, budget, optim)
    n_of = dict(sizes)
    streamed_bytes = sum(state_bytes(n_of[n], optim) for n in streamed)
    plan = {"optim": optim, "micro_pairs": micro, "max_len": policy.dims.max_len, "trainable_elems": sum(n_of.values()),
            "device_free_before_optimizer_bytes": free, "activation_reserve_bytes": reserve,
            "device_budget_bytes": budget, "resident_bytes": sum(state_bytes(n_of[n], optim) for n in resident),
            "streamed_bytes": streamed_bytes, "host_needed_bytes": streamed_bytes + HOST_MARGIN,
            "mem_available_bytes": mem_available(), "resident_buckets": len(resident), "streamed_buckets": len(streamed)}
    a = argparse.Namespace(**vars(args))
    a.micro_pairs = micro
    try:        # the engine's optimizer refuses before it pins anything when MemAvailable is too small
        plan["run"] = timed_offload_run(a, policy, make_batches(policy, B), B, T, optim)
    except MemoryError as e:
        plan["refused"] = str(e)
    return plan


# ---- AdamW with blockwise 8-bit moments (--optim adamw_8bit) -----------------------------------------------------------
def kernel_throughput(n=1 << 30, reps=20):
    """rlaifv_adamw8bit_step against the fp32 rlaifv_adamw_step (adamw_kernel) on one n-element shard, CUDA events.
    Algorithmic bytes per element: fp32 master read + write 8, bf16 grad 2 and param 2, codes read + write 4 (8-bit:
    16 B + 16 B per 256 elements for the absmax) or fp32 m and v read + write 16 (fp32: 28 B)."""
    from rlaifv_b200 import ops
    from rlaifv_b200.zero2 import dynamic_map
    g = torch.Generator(device="cuda").manual_seed(0)
    grad = (torch.randn(n, generator=g, device="cuda") * 1e-3).bfloat16()
    param = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    master = torch.randn(n, generator=g, device="cuda") * 0.02
    out = {"elements": n, "reps": reps}
    nb = (n + 255) // 256
    state8 = [torch.full((n,), 127, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.uint8, device="cuda"),
              torch.zeros(nb, device="cuda"), torch.zeros(nb, device="cuda")]
    maps = [dynamic_map(True).cuda(), dynamic_map(False).cuda()]
    run8 = lambda st: ops.adamw8bit_step(master, *state8, grad, param, n, *maps, 1e-6, 0.9, 0.999, 1e-8, 0.01, st)  # noqa
    for name, fn, bpe in (("adamw_8bit", run8, 16 + 16 / 256), ("adamw_torch", None, 28)):
        if fn is None:
            m, v = torch.zeros_like(master), torch.zeros_like(master)
            fn = lambda st: ops.adamw_step(master, m, v, grad, param, 1e-6, 0.9, 0.999, 1e-8, 0.01, st)  # noqa
        for st in range(1, 4):
            fn(st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for st in range(4, 4 + reps):
            fn(st)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[name] = {"ms": ms, "bytes_per_elem": bpe, "gbs": bpe * n / (ms * 1e-3) / 1e9}
        if fn is not run8:
            del m, v
    return out


def identity8(layers):
    """Three steps with 8-bit moments on the device, then from the same seed offloaded with a mixed and an all-streamed
    split: metrics, bf16 parameters and every state tensor bit for bit."""
    from rlaifv_b200.zero2 import state_bytes, state_parts
    B, micro = 4, 2
    batches = [bench.synthetic_batch(0, s, B) for s in range(3)]
    keys = [k for k, _, _ in state_parts("adamw_8bit")]
    results, splits = {}, {}
    for mode in ("device", "mixed", "all_streamed"):
        budget = None
        if mode == "mixed":
            budget = sum(state_bytes(sizes[n], "adamw_8bit") for n in ("embed", "projector", "layer0", "layer1"))
        elif mode == "all_streamed":
            budget = 0
        eng = make_engine(layers, micro, offload_budget=budget, offload=budget is not None, optim="adamw_8bit")
        if mode == "device":
            sizes = {b.name: b.size for b in eng.policy.trainable_buckets()}
            add_reference_logps(eng.policy, batches, B, micro)
        metrics = [eng.train_step(hb).clone() for hb in batches]
        eng.opt.wait_all()
        torch.cuda.synchronize()
        sd = eng.opt.state_dict()
        results[mode] = {"metrics": torch.stack(metrics).cpu(), "params": eng.policy.store.flat.cpu(),
                         **{k: sd[k].cpu() for k in keys}}
        if budget is not None:
            splits[mode] = {"resident": eng.opt.resident_names, "streamed": len(eng.opt.streamed_names)}
            eng.opt.close()
        del eng, sd
        gc.collect()
        torch.cuda.empty_cache()
    d = results["device"]
    out = {"layers": layers, "pairs": B, "micro_pairs": micro, "steps": 3}
    for mode in ("mixed", "all_streamed"):
        o = results[mode]
        out[mode] = {**splits[mode], **{k + "_identical": bool(torch.equal(d[k], o[k])) for k in d}}
    return out


def loss_trajectory(steps=20, layers=2):
    """7B widths at `layers` layers, `steps` steps of each optimizer from one seed on bench.py's inputs (4 pairs,
    micro-batches of 2, lr 5e-7 as in the recipe): the largest |delta loss| over the steps and the relative difference
    of the fp32 master weights at the end."""
    B, micro = 4, 2
    batches = [bench.synthetic_batch(0, s, B) for s in range(steps)]
    res = {}
    for optim in ("adamw_torch", "adamw_8bit"):
        eng = make_engine(layers, micro, optim=optim)
        if optim == "adamw_torch":
            add_reference_logps(eng.policy, batches, B, micro)
            m0 = eng.opt.master.cpu()
        losses = [float(eng.train_step(hb)[0]) for hb in batches]
        eng.opt.wait_all()
        torch.cuda.synchronize()
        res[optim] = (losses, eng.opt.master.cpu())
        del eng
        gc.collect()
        torch.cuda.empty_cache()
    (l32, m32), (l8, m8) = res["adamw_torch"], res["adamw_8bit"]
    return {"layers": layers, "steps": steps, "pairs": B, "lr": 5e-7, "loss_adamw_torch": l32, "loss_adamw_8bit": l8,
            "max_abs_delta_loss": max(abs(a - b) for a, b in zip(l32, l8)),
            "master_rel_diff": float((m8 - m32).norm() / m32.norm()),
            "master_rel_diff_of_update": float((m8 - m32).norm() / (m32 - m0).norm())}


def llava13b_full_ft(args):
    """13B full fine-tuning with 8-bit moments: 8 pairs of bench.py's T in micro-batches of one pair, model_max_length
    2048, seeded weights; measured where MemAvailable holds the streamed state, otherwise the refusal."""
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    gc.collect()
    torch.cuda.empty_cache()
    dims = LlavaDims(hidden_size=5120, intermediate_size=13824, num_layers=40, num_heads=40, max_len=2048)
    policy = LlavaDPOPolicy(dims, torch.device("cuda", 0), seed=0)
    T = bench.PROMPT_LEN + bench.RESP_LEN - 1 + dims.num_patches
    return planned_run(args, policy, lambda pol, B: [bench.synthetic_batch(0, s, B) for s in range(2)], T,
                       "adamw_8bit")


def adamw8bit_main(args, line):
    path = os.path.join(args.out, "offload_step_8bit.json")
    line["mem_available_bytes"] = mem_available()

    def dump(key):
        print(json.dumps({key: line[key]}), flush=True)
        with open(path, "w") as f:
            json.dump(line, f, indent=1)
    legs = [("kernel", args.skip_kernel, kernel_throughput),
            ("identity", args.skip_identity, lambda: identity8(args.identity_layers)),
            ("loss_trajectory", args.skip_trajectory, loss_trajectory),
            ("config_b", args.skip_config_b, lambda: [config_b(args, optim) for optim in
                                                      ("adamw_torch", "adamw_8bit", "adamw_torch", "adamw_8bit")]),
            ("llava13b_full_ft", args.skip_13b, lambda: llava13b_full_ft(args)),
            ("omnilmm_trained_tower", args.skip_trained_tower, lambda: trained_tower_plan(argparse.Namespace(**dict(vars(args), max_len=1024)),
                                                                     "adamw_8bit"))]
    for key, skip, fn in legs:
        if skip:
            continue
        try:
            line[key] = fn()
        except torch.OutOfMemoryError as e:
            line[key] = {"out_of_memory": str(e).splitlines()[0]}
        gc.collect()
        torch.cuda.empty_cache()
        dump(key)
    print(json.dumps(line), flush=True)


def omnilmm_main(args, line):
    path = os.path.join(args.out, "offload_step_omnilmm.json")

    def dump():
        with open(path, "w") as f:
            json.dump(line, f, indent=1)
    if not args.skip_identity:
        line["identity"] = [omni_identity(args.identity_layers, args.identity_eva_blocks, tc) for tc in (0, 1)]
        print(json.dumps({"identity": line["identity"]}), flush=True)
        dump()
    if not args.skip_config_d:
        line["config_d"] = config_d(args, args.tune_clip)
        print(json.dumps({"config_d": line["config_d"]}), flush=True)
        dump()
    if not args.skip_trained_tower:
        line["trained_tower"] = trained_tower_plan(args)
        dump()
    print(json.dumps(line), flush=True)


def main(argv=None):
    args = parse_args(argv)
    os.makedirs(args.out, exist_ok=True)
    if not torch.cuda.is_available():
        raise SystemExit("offload_step.py measures on a GPU; no CUDA device found")
    name, power = gpu_name_and_power()
    line = {"gpu": name, "power_limit": power}
    if args.omnilmm:
        return omnilmm_main(args, line)
    if args.optim == "adamw_8bit":
        return adamw8bit_main(args, line)
    if not args.skip_identity:
        line["identity"] = identity(args.identity_layers)
        print(json.dumps({"identity": line["identity"]}), flush=True)
        torch.cuda.empty_cache()
    if not args.skip_config_b:
        line["config_b"] = config_b(args)
    print(json.dumps(line), flush=True)
    with open(os.path.join(args.out, "offload_step.json"), "w") as f:
        json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
