"""ZeRO-2 style data-parallel AdamW over the flat parameter buckets (script/zero2.json:16-22;
optimizer = adamw_torch, muffin/train/train_llava15.py:75; lr/wd/schedule flags of
script/train/llava15_train.sh:31-34).

Every bucket of ParamStore (embed | layer i | head | projector) is cut into `world` equal slices;
rank r owns slice r of every bucket: fp32 master weights and Adam moments exist only for owned
slices (12 B/param / world; about 6 B with optim="adamw_8bit"), gradients are reduce-scattered in
place into the owned slice as soon as a bucket's backward has finished (overlapping the rest of the backward on a side stream), the
fused AdamW kernel updates the slice and writes bf16 straight into the parameter buffer, and an
in-place all-gather redistributes the updated parameters.  With world == 1 the collectives vanish.
OffloadAdamW (world == 1) keeps the state that does not fit on the device in pinned host memory and
streams it through the GPU each step (script/zero2_offload.json); the policy's activation reserve sizes its default
device budget (activation_reserve_bytes for the decoder, omnilmm_activation_reserve_bytes for OmniLMM).

torch.distributed (NCCL) is the transport; nothing here computes on the host.
"""
import math

import torch
import torch.distributed as dist

from . import lib as _lib
from . import ops

_F32 = torch.float32
_U8 = torch.uint8

# ---- optimizer state formats ------------------------------------------------------------------------------------------
# adamw_torch: fp32 master, exp_avg and exp_avg_sq (12 B per element; torch.optim.AdamW, the default).
# adamw_8bit: fp32 master, one uint8 code each for exp_avg and exp_avg_sq, and per block of QBLOCK consecutive elements
# of a slice one fp32 absmax each (bitsandbytes AdamW8bit, Dettmers et al. 2022; HF --optim adamw_bnb_8bit / adamw_8bit).
# Blocks are counted from the start of each owned slice; a slice's last block may be partial.
OPTIMS = ("adamw_torch", "adamw_8bit")
QBLOCK = 256
STATE_BYTES_PER_ELEM = 12            # adamw_torch: fp32 master + exp_avg + exp_avg_sq


def state_format(hf_optim):
    """The state format of an HF TrainingArguments.optim value: adamw_bnb_8bit and adamw_8bit (HF's alias) train with
    8-bit moments; every other value keeps the fp32 AdamW state."""
    return "adamw_8bit" if hf_optim in ("adamw_bnb_8bit", "adamw_8bit") else "adamw_torch"


def _check_optim(optim):
    if optim not in OPTIMS:
        raise ValueError("optimizer state format %r: expected one of %s" % (optim, ", ".join(OPTIMS)))


def n_blocks(n):
    """Quantization blocks of a slice of n elements."""
    return (n + QBLOCK - 1) // QBLOCK


def state_bytes(n, optim="adamw_torch"):
    """Exact bytes of optimizer state of one slice of n elements."""
    _check_optim(optim)
    return STATE_BYTES_PER_ELEM * n if optim == "adamw_torch" else 6 * n + 8 * n_blocks(n)


def state_parts(optim):
    """The flat state tensors of a format, as (name, dtype, "elem" | "block"): one entry per element of the owned slices,
    or one per quantization block. The names are the state_dict keys and the optimizer's attribute names."""
    _check_optim(optim)
    if optim == "adamw_torch":
        return (("master", _F32, "elem"), ("exp_avg", _F32, "elem"), ("exp_avg_sq", _F32, "elem"))
    return (("master", _F32, "elem"), ("exp_avg_q", _U8, "elem"), ("exp_avg_sq_q", _U8, "elem"),
            ("absmax", _F32, "block"), ("absmax_sq", _F32, "block"))


def dynamic_map(signed):
    """The 256-entry code map of 8-bit AdamW, built as bitsandbytes' create_dynamic_map builds it: for i in 0..6, the
    midpoints of linspace(0.1, 1, k) with k = 2^i + 1 (signed) or 2^(i+1) + 1 (unsigned), scaled by 10^(i-6), and for
    the signed map their negatives too; then 0 and 1. Strictly increasing fp32."""
    vals = [torch.tensor([0.0, 1.0], dtype=_F32)]
    for i in range(7):
        k = 2 ** i + 1 if signed else 2 ** (i + 1) + 1
        b = torch.linspace(0.1, 1, k, dtype=_F32)
        pos = 10 ** (i - 6) * ((b[:-1] + b[1:]) / 2)
        vals += [pos, -pos] if signed else [pos]
    return torch.sort(torch.cat(vals)).values


def _initial_code(name):
    """What a fresh state tensor holds: the code of 0 for the moments (index 127 of the signed map, 0 of the unsigned
    one), zero for the rest (master is copied from the parameters)."""
    return 127 if name == "exp_avg_q" else 0


def cosine_lr(step, total_steps, base_lr, warmup_ratio=0.05):
    """HF get_cosine_schedule_with_warmup value used for optimizer step `step` (0-based)."""
    warm = math.ceil(total_steps * warmup_ratio)
    if step < warm:
        return base_lr * step / max(1, warm)
    prog = (step - warm) / max(1, total_steps - warm)
    return base_lr * max(0.0, 0.5 * (1.0 + math.cos(math.pi * prog)))


class OptBucket:
    """One trainable bucket as the optimizer sees it: flat bf16 parameter / gradient views of equal length
    (a multiple of 8*world), of which the first `decay_size` elements get weight decay."""

    def __init__(self, name, flat, grad, decay_size):
        self.name, self.flat, self.grad, self.decay_size = name, flat, grad, decay_size
        self.size = flat.numel()


class Zero2AdamW:
    def __init__(self, buckets, lr=5e-7, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, rank=0, world=1,
                 group=None, gather_order=None, optim="adamw_torch"):
        """optim: the state format, "adamw_torch" (fp32 moments) or "adamw_8bit" (blockwise 8-bit moments)."""
        _check_optim(optim)
        self.optim = optim
        self.buckets = list(buckets)
        self.index = {b.name: i for i, b in enumerate(self.buckets)}
        self.lr, self.betas, self.eps, self.wd = lr, betas, eps, weight_decay
        self.rank, self.world, self.group = rank, world, group
        self.step_count = 0
        dev = self.buckets[0].flat.device
        self.slices = []   # (bucket, s0, s1, offset into the owned fp32 state), s0/s1 relative to the bucket
        self.block_offsets = []     # per slice: its first block in the owned block-indexed state (absmax, absmax_sq)
        total = blocks = 0
        for b in self.buckets:
            assert b.size % (world * 8) == 0, (b.name, b.size)
            n = b.size // world
            self.slices.append((b, rank * n, (rank + 1) * n, total))
            self.block_offsets.append(blocks)
            total += n
            blocks += n_blocks(n)
        self.owned, self.owned_blocks = total, blocks
        self.state_nbytes = sum(state_bytes(s1 - s0, optim) for _, s0, s1, _ in self.slices)
        if optim == "adamw_8bit":
            self.map_m = dynamic_map(True).to(dev)
            self.map_v = dynamic_map(False).to(dev)
        self._init_state(dev)
        self.comm_stream = torch.cuda.Stream(device=dev) if world > 1 else None
        self.opt_stream = None
        self._gathered = {}
        self._reduced = {}
        self._done = set()
        # order in which the next forward needs the parameters (default: as given)
        self.gather_order = [self.index[n] for n in gather_order if n in self.index] if gather_order else \
            list(range(len(self.buckets)))

    def _new_state(self, n_elems, n_blk, device, prefix=""):
        """Fresh flat state tensors of this format (state_parts) for n_elems elements in n_blk blocks, set as the
        attributes prefix + name. The master is left for the caller to fill."""
        for name, dtype, per in state_parts(self.optim):
            shape = (n_elems if per == "elem" else n_blk,)
            t = torch.empty(shape, dtype=dtype, device=device) if name == "master" else \
                torch.full(shape, _initial_code(name), dtype=dtype, device=device)
            setattr(self, prefix + name, t)

    def _init_state(self, dev):
        """fp32 master copy of the owned slices and fresh moments, all on the device."""
        self._new_state(self.owned, self.owned_blocks, dev)
        for b, s0, s1, o in self.slices:
            self.master[o:o + (s1 - s0)].copy_(b.flat[s0:s1])

    # ---- gradient reduction (called from the backward as buckets complete) ----
    def reduce_bucket(self, bucket_index):
        if self.world == 1:
            return
        if isinstance(bucket_index, str):
            if bucket_index not in self.index:
                return
            bucket_index = self.index[bucket_index]
        b, s0, s1, _ = self.slices[bucket_index]
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            dist.reduce_scatter_tensor(b.grad[s0:s1], b.grad, op=dist.ReduceOp.SUM, group=self.group)
            done = torch.cuda.Event()
            done.record(self.comm_stream)
        self._reduced[bucket_index] = done

    def reduce_all(self):
        for i in range(len(self.slices)):
            self.reduce_bucket(i)

    # ---- optimizer step ----
    def _adamw_bucket(self, bi, lr):
        b, s0, s1, o = self.slices[bi]
        b1, b2 = self.betas
        if self.optim == "adamw_8bit":      # one launch per slice: blocks never split at the decay edge
            n, q = s1 - s0, self.block_offsets[bi]
            nb = n_blocks(n)
            ops.adamw8bit_step(self.master[o:o + n], self.exp_avg_q[o:o + n], self.exp_avg_sq_q[o:o + n],
                               self.absmax[q:q + nb], self.absmax_sq[q:q + nb], b.grad[s0:s1], b.flat[s0:s1],
                               min(n, max(0, b.decay_size - s0)), self.map_m, self.map_v, lr, b1, b2, self.eps,
                               self.wd, self.step_count)
            return
        dec_end = min(s1, b.decay_size)
        if dec_end > s0:
            n = dec_end - s0
            ops.adamw_step(self.master[o:o + n], self.exp_avg[o:o + n], self.exp_avg_sq[o:o + n],
                           b.grad[s0:dec_end], b.flat[s0:dec_end], lr, b1, b2, self.eps, self.wd, self.step_count)
        nd0 = max(s0, b.decay_size)
        if s1 > nd0:
            n = s1 - nd0
            oo = o + (nd0 - s0)
            ops.adamw_step(self.master[oo:oo + n], self.exp_avg[oo:oo + n], self.exp_avg_sq[oo:oo + n],
                           b.grad[nd0:s1], b.flat[nd0:s1], lr, b1, b2, self.eps, 0.0, self.step_count)

    def begin_step(self, lr=None):
        """Open an optimizer step whose buckets are updated one by one (`step_bucket`) while the backward
        is still running; `finish_step` updates whatever is left and closes the step."""
        self._lr = self.lr if lr is None else lr
        self.step_count += 1
        self._done = set()
        if self.opt_stream is None:
            self.opt_stream = torch.cuda.Stream(device=self.buckets[0].flat.device)

    def step_bucket(self, name):
        """AdamW (+ parameter all-gather) of one bucket on the optimizer side stream, ordered after everything
        enqueued so far on the current stream and after this bucket's gradient reduce-scatter. The caller
        guarantees the bucket's gradients are final and its parameters are no longer read this step."""
        bi = self.index.get(name, -1)
        if bi < 0 or bi in self._done:
            return
        self._done.add(bi)
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        self.opt_stream.wait_event(ev)
        if self.world > 1:
            rs = self._reduced.pop(bi, None)
            if rs is not None:
                self.opt_stream.wait_event(rs)
        with torch.cuda.stream(self.opt_stream), _lib.use_stream(self.opt_stream):
            self._adamw_bucket(bi, self._lr)
            if self.world > 1:
                b, s0, s1, _ = self.slices[bi]
                dist.all_gather_into_tensor(b.flat, b.flat[s0:s1], group=self.group)
            done = torch.cuda.Event()
            done.record(self.opt_stream)
        self._gathered[bi] = done

    def finish_step(self):
        for bi in self.gather_order:
            self.step_bucket(self.buckets[bi].name)
        # single-GPU callers read the parameters right away on the main stream: order it after the side stream
        if self.world == 1:
            self.wait_all()

    def step(self, lr=None):
        """Whole optimizer step at once (no overlap with the backward)."""
        self.begin_step(lr)
        if self.world > 1:
            torch.cuda.current_stream().wait_stream(self.comm_stream)
        self.finish_step()

    def wait_bucket(self, bucket_index):
        """Make the current stream wait for bucket's parameter all-gather of the last step (no-op if none)."""
        if isinstance(bucket_index, str):
            if bucket_index not in self.index:
                raise KeyError("wait_bucket: %r is not a bucket of this optimizer (%s ...)"
                               % (bucket_index, ", ".join(list(self.index)[:4])))
            bucket_index = self.index[bucket_index]
        ev = self._gathered.pop(bucket_index, None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)

    def wait_all(self):
        for bi in list(self._gathered):
            self.wait_bucket(bi)

    def _format_keys(self):
        """state_dict entries that record the format: none for adamw_torch (its checkpoints predate the choice)."""
        return {} if self.optim == "adamw_torch" else {"optim": self.optim, "block": QBLOCK}

    def state_dict(self):
        return {"step": self.step_count, **{k: getattr(self, k) for k, _, _ in state_parts(self.optim)},
                **self._format_keys(), "rank": self.rank, "world": self.world}

    def check_format(self, sd):
        """Refuse (ValueError) a checkpoint written with the other optimizer state format."""
        fmt = sd.get("optim", "adamw_torch")
        if sd.get("block", QBLOCK) != QBLOCK:
            fmt = "%s (blocks of %s)" % (fmt, sd["block"])
        if fmt != self.optim:
            raise ValueError("optimizer checkpoint holds %s state, but this optimizer keeps %s state: converting "
                             "between formats is not supported; resume with the --optim it was written with"
                             % (fmt, self.optim))

    def check_state_size(self, sd):
        """Refuse (ValueError) a checkpoint whose flat state was written for another set of trainable buckets."""
        n = sd["master"].numel()
        if n != self.owned:
            raise ValueError("optimizer checkpoint holds %d fp32 elements per state tensor, but this optimizer owns %d "
                             "over its %d buckets (%s ...): it was written for a different set of trainable parameters"
                             % (n, self.owned, len(self.buckets), ", ".join(b.name for b in self.buckets[:4])))

    def load_state_dict(self, sd):
        assert sd["world"] == self.world and sd["rank"] == self.rank
        self.check_format(sd)
        self.check_state_size(sd)
        self.step_count = sd["step"]
        for k, _, _ in state_parts(self.optim):
            getattr(self, k).copy_(sd[k])


# ------------------------------------------------------------------------------------------------
# Offloaded AdamW (one GPU): the fp32 state that does not fit on the device lives in pinned host memory and is streamed
# through a small device staging ring each step (DeepSpeed `offload_optimizer: {device: cpu}`, script/zero2_offload.json;
# the update itself stays on the GPU). DESIGN.md §2 has the memory plan, §3 the pipeline.
# ------------------------------------------------------------------------------------------------
DEFAULT_SLOT_ELEMS = 8 << 20         # 8 Mi elements: 96 MB per ring slot (master | m | v), 48 MB with 8-bit moments
DEFAULT_SLOTS = 3                    # load of chunk i+1 | update of chunk i | store of chunk i-1
DEVICE_MARGIN = 2 << 30              # allocator fragmentation, CLIP tower and head buffers, library workspaces
HOST_MARGIN = 8 << 30                # what MemAvailable must still show after the streamed state is pinned


def offload_priority(names):
    """Bucket names in the order they should stay on the device: the buckets whose gradients become final last first.
    Their updates run after the whole backward and can overlap nothing; the head and the last layers finish first, so
    their copies overlap the rest of the backward. LLaVA: embed, projector, layer0, layer1, ..., head.
    OmniLMM with a trained tower: the tail buckets embed and resampler are stepped after the whole backward; the tower's
    backward runs after the decoder's and finishes with its embedding (eva62 first, eva_embed last), so the order is
    embed, resampler, eva_embed, eva0, ..., eva62, layer0, ..., layer31, head. Keeping the first tower blocks resident
    also keeps the first buckets the next forward reads off the copy streams."""
    def numbered(prefix):
        k = len(prefix)
        return sorted((n for n in names if n.startswith(prefix) and n[k:].isdigit()), key=lambda n: int(n[k:]))
    layers, eva = numbered("layer"), numbered("eva")
    eva_embed = [n for n in names if n == "eva_embed"]
    head = [n for n in names if n == "head"]
    ordered = set(layers + eva + eva_embed + head)
    rest = [n for n in names if n not in ordered]
    return rest + eva_embed + eva + layers + head


def offload_plan(sizes, budget_bytes, optim="adamw_torch"):
    """Resident / streamed split of the optimizer state. sizes: [(bucket name, elements)]. Buckets are taken in
    offload_priority order while their state (state_bytes in format `optim`) fits in budget_bytes; the first one that
    does not fit and every one after it are streamed. Returns (resident names, streamed names), each in priority order."""
    n_of = dict(sizes)
    order = offload_priority([n for n, _ in sizes])
    used, k = 0, 0
    while k < len(order) and used + state_bytes(n_of[order[k]], optim) <= budget_bytes:
        used += state_bytes(n_of[order[k]], optim)
        k += 1
    return order[:k], order[k:]


def ring_slot_elems(largest, slot_elems, optim="adamw_torch"):
    """Elements per staging-ring slot: slot_elems, or less when the largest owned slice is smaller (rounded up to 4
    elements for adamw_torch, to a whole block for adamw_8bit, whose chunks must start on block edges)."""
    q = 4 if optim == "adamw_torch" else QBLOCK
    return min(slot_elems, (largest + q - 1) // q * q)


def adamw8bit_slot_bytes(slot_elems):
    """Bytes of one 8-bit ring slot: master | code_m | code_v | absmax_m | absmax_v of slot_elems (% 256 == 0) elements,
    rounded up to 256 bytes (the layout rlaifv_adamw8bit_offload_bucket reads)."""
    return (6 * slot_elems + 8 * (slot_elems // QBLOCK) + 255) // 256 * 256


def ring_bytes(n_slots, slot_elems, optim="adamw_torch"):
    """Device bytes of the staging ring."""
    return n_slots * (3 * slot_elems * 4 if optim == "adamw_torch" else adamw8bit_slot_bytes(slot_elems))


def offload_chunks(n, slot_elems, decay_size):
    """The chunks rlaifv_adamw_offload_bucket cuts a streamed bucket of n elements into: [(offset, length, elements
    that get weight decay)]. Mirrors the loop of the C entry point (pinned by the CPU tests)."""
    out = []
    for off in range(0, n, slot_elems):
        c = min(slot_elems, n - off)
        out.append((off, c, min(c, max(0, decay_size - off))))
    return out


def activation_reserve_bytes(dims, pairs, seq_len, stash_act=False):
    """Device bytes the step's activations need for `pairs` preference pairs (2 * pairs sequences) of seq_len tokens.
    Per decoder layer and token (DESIGN.md §2): bf16 x, fused qkv, attention output, x2 and gate|up, fp32 rstd1/rstd2
    and the attention LSE (92 KB at 7B widths), plus the SwiGLU product when it is stashed. Per token once: eight bf16
    rows of width H for the step's working buffers."""
    H, F, KV = dims.hidden_size, dims.intermediate_size, dims.kv_size
    per_layer = 2 * (4 * H + 2 * KV + 2 * F) + 8 + 4 * dims.num_heads + (2 * F if stash_act else 0)
    tokens = 2 * pairs * seq_len
    return tokens * (per_layer * dims.num_layers + 16 * H)


def eva_stash_bytes_per_image(e):
    """What the trained EVA tower's forward keeps for its backward, per image (EvaTower.forward(keep_stash=True)). Per
    live block and token (1 + grid^2 tokens): bf16 qkv (3 x padded width), attention output (padded width), the
    attention projection, x_mid, the fc1 output, the MLP output and the block output, plus the fp32 LSE per head.
    Once per image: the im2col columns and the embedding output (block 0's input)."""
    S, C = e.n_tokens + 1, e.embed_dim
    per_block = S * (2 * (4 * e.hp + 4 * C + e.mlp_hidden) + 4 * e.num_heads)
    return e.live_blocks * per_block + e.n_tokens * 2 * e.patch_k_pad + S * 2 * C


def eva_working_bytes_per_image(e, trained):
    """The EVA tower's reused buffers (EvaTower._bufs, which live as long as the tower) per image, plus its output.
    Frozen (forward without stash): qkv, attention output, attention projection, x_mid, fc1 output, MLP output, two
    block outputs, the LayerNorm and GELU outputs and the LSE. Trained: the forward keeps only the LayerNorm and GELU
    buffers (the rest is stash); the backward adds dy, dx (two), dm, dh, df, d(att), dqkv and the fp32 delta.
    Both: the final LayerNorm output and the tokens without the prefix."""
    S, C, Hd, HP = e.n_tokens + 1, e.embed_dim, e.mlp_hidden, e.hp
    if trained:
        elems = (C + Hd) + (5 * C + 2 * Hd + 4 * HP)
    else:
        elems = 4 * HP + 6 * C + 2 * Hd
    return S * (2 * elems + 4 * e.num_heads) + S * 2 * C + e.n_tokens * 2 * C


def resampler_bytes_per_image(dims, n_tokens):
    """The resampler's stash and backward temporaries per image of n_tokens vision tokens (resampler.Resampler): per
    token the bf16 input, kv_proj output, its LayerNorm, k input, k and v (stash) and dk, dv, dxn, dxk and the input
    gradient (backward); per query row the attention output, out_proj output and ln_post output."""
    E, W, Q = dims.hidden_size, dims.vision_width, dims.num_query
    return n_tokens * 2 * (2 * W + 9 * E) + Q * 2 * 3 * E


def omnilmm_activation_reserve_bytes(dims, eva, pairs, seq_len, tune_clip=True, stash_act=False):
    """activation_reserve_bytes for the OmniLMM policy: the GQA decoder (kv_size, intermediate_size of dims) at seq_len
    for `pairs` pairs, plus per image (one per pair) the resampler and, when the policy has its EVA tower (`eva`), the
    tower's working set and, with tune_clip, its stash."""
    r = activation_reserve_bytes(dims, pairs, seq_len, stash_act)
    n_tokens = eva.n_tokens if eva is not None else 1024
    r += pairs * resampler_bytes_per_image(dims, n_tokens)
    if eva is not None:
        r += pairs * eva_working_bytes_per_image(eva, tune_clip)
        if tune_clip:
            r += pairs * eva_stash_bytes_per_image(eva)
    return r


def mem_available_bytes(meminfo_text):
    """MemAvailable of a /proc/meminfo text, in bytes (None if the line is missing)."""
    for line in meminfo_text.splitlines():
        if line.startswith("MemAvailable:"):
            f = line.split()
            return int(f[1]) * (1024 if len(f) > 2 and f[2].lower() == "kb" else 1)
    return None


def check_host_memory(need_bytes, meminfo_text, margin=HOST_MARGIN):
    """Refuse (MemoryError) to pin need_bytes of optimizer state unless MemAvailable covers it plus `margin`: on a shared
    host the kernel's OOM killer must never be the one to say no."""
    avail = mem_available_bytes(meminfo_text)
    if avail is None:
        raise MemoryError("offload_optimizer: no MemAvailable line in /proc/meminfo; cannot check host memory")
    if need_bytes + margin > avail:
        raise MemoryError("offload_optimizer: the streamed optimizer state needs %.2f GB of pinned host memory plus a "
                          "%.2f GB margin, but MemAvailable is %.2f GB. Give the device a larger budget, use more GPUs "
                          "(ZeRO-2 without offload), or free host memory."
                          % (need_bytes / 1e9, margin / 1e9, avail / 1e9))
    return avail


def _read_meminfo(path="/proc/meminfo"):
    with open(path) as f:
        return f.read()


class OffloadAdamW(Zero2AdamW):
    """Zero2AdamW for one GPU whose optimizer state does not all fit on the device. offload_plan keeps as many buckets'
    state on the device as `device_budget` allows (resident buckets run the on-device path unchanged); the others'
    state is in pinned host memory and rlaifv_adamw_offload_bucket streams it through a staging ring of n_slots x
    slot_elems on two copy streams while the update runs on the optimizer stream. Results are bit-identical to
    Zero2AdamW: both paths run the same per-element update (adamw_elem in rowops.cu).

    device_budget: bytes of optimizer state allowed on the device. None: free device memory minus
    `activation_reserve`, the staging ring and DEVICE_MARGIN.

    Ordering: the event wait_bucket hands to the next forward is recorded after the bucket's update, not after its D2H,
    so the copies out run under the next step's forward; a bucket's next H2D waits for its last D2H; state_dict and
    load_state_dict wait for the copies in flight."""

    def __init__(self, buckets, lr=5e-7, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, rank=0, world=1,
                 group=None, gather_order=None, device_budget=None, activation_reserve=0,
                 slot_elems=DEFAULT_SLOT_ELEMS, n_slots=DEFAULT_SLOTS, host_margin=HOST_MARGIN, meminfo=None,
                 optim="adamw_torch"):
        if world != 1:
            raise NotImplementedError("offload_optimizer runs on one GPU; with two or more, ZeRO-2 shards the state "
                                      "(offloading each rank's slice is not implemented)")
        assert slot_elems > 0 and slot_elems % (4 if optim == "adamw_torch" else QBLOCK) == 0 and 2 <= n_slots <= 8
        self._cfg = dict(device_budget=device_budget, activation_reserve=activation_reserve, slot_elems=slot_elems,
                         n_slots=n_slots, host_margin=host_margin, meminfo=meminfo)
        self._host = []
        self._stored = {}
        self.ring = None
        super().__init__(buckets, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, rank=rank, world=world,
                         group=group, gather_order=gather_order, optim=optim)

    def _init_state(self, dev):
        cfg = self._cfg
        largest = max(s1 - s0 for _, s0, s1, _ in self.slices)
        self.slot_elems = ring_slot_elems(largest, cfg["slot_elems"], self.optim)
        ring_b = ring_bytes(cfg["n_slots"], self.slot_elems, self.optim)
        budget = cfg["device_budget"]
        if budget is None:
            budget = torch.cuda.mem_get_info(dev)[0] - cfg["activation_reserve"] - ring_b - DEVICE_MARGIN
        self.device_budget = budget
        self.resident_names, self.streamed_names = offload_plan(
            [(b.name, s1 - s0) for b, s0, s1, _ in self.slices], budget, self.optim)
        streamed = set(self.streamed_names)
        self._global = [o for _, _, _, o in self.slices]       # offsets in the checkpoint's flat layout
        self._global_blocks = list(self.block_offsets)         # block offsets in the checkpoint's flat layout
        self._is_streamed = [b.name in streamed for b, _, _, _ in self.slices]
        local, local_blocks, n_dev, n_host, nb_dev, nb_host = [], [], 0, 0, 0, 0
        host_bytes = 0
        for (b, s0, s1, _), st in zip(self.slices, self._is_streamed):
            local.append(n_host if st else n_dev)
            local_blocks.append(nb_host if st else nb_dev)
            if st:
                n_host += s1 - s0
                nb_host += n_blocks(s1 - s0)
                host_bytes += state_bytes(s1 - s0, self.optim)
            else:
                n_dev += s1 - s0
                nb_dev += n_blocks(s1 - s0)
        self.resident_elems, self.streamed_elems = n_dev, n_host
        if n_host:
            check_host_memory(host_bytes, (cfg["meminfo"] or _read_meminfo)(), cfg["host_margin"])
        # resident buckets index the device tensors exactly as Zero2AdamW does (so _adamw_bucket is reused as is);
        # streamed buckets index the host tensors
        self.slices = [(b, s0, s1, lo) for (b, s0, s1, _), lo in zip(self.slices, local)]
        self.block_offsets = local_blocks
        self._new_state(n_dev, nb_dev, dev)
        # Plain CPU tensors of the exact size, pinned with cudaHostRegister: torch's pinned allocator rounds every block
        # up to a power of two, which would turn ~45 GB of state into 64 GB.
        self._new_state(n_host, nb_host, "cpu", prefix="host_")
        for name, _, _ in state_parts(self.optim):
            t = getattr(self, "host_" + name)
            if t.numel():
                self._register(t)
        for (b, s0, s1, o), st in zip(self.slices, self._is_streamed):
            (self.host_master if st else self.master)[o:o + (s1 - s0)].copy_(b.flat[s0:s1])
        if n_host:
            if self.optim == "adamw_torch":
                self.ring = torch.empty((cfg["n_slots"], 3 * self.slot_elems), dtype=_F32, device=dev)
            else:
                self.ring = torch.empty((cfg["n_slots"], adamw8bit_slot_bytes(self.slot_elems)), dtype=_U8, device=dev)
            self.h2d_stream = torch.cuda.Stream(device=dev)
            self.d2h_stream = torch.cuda.Stream(device=dev)
        self.pinned_bytes = sum(t.numel() * t.element_size() for t in self._host)

    def _register(self, t):
        rt = torch.cuda.cudart()
        err = rt.cudaHostRegister(t.data_ptr(), t.numel() * t.element_size(), 0)
        if int(err) != 0:
            raise RuntimeError("cudaHostRegister of %.2f GB failed: %s"
                               % (t.numel() * t.element_size() / 1e9, rt.cudaGetErrorString(err)))
        self._host.append(t)

    def close(self):
        """Wait for the copies in flight, release the library's events for the staging ring, free the ring and unpin
        the host state (also done when the object is collected)."""
        if not self._host:
            return
        self._drain()
        if self.ring is not None:
            ops.adamw_offload_release(self.ring)
            self.ring = None
        rt = torch.cuda.cudart()
        for t in self._host:
            rt.cudaHostUnregister(t.data_ptr())
        self._host = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _drain(self):
        if self.ring is not None:
            self.h2d_stream.synchronize()
            self.d2h_stream.synchronize()
        self._stored.clear()

    def _adamw_bucket(self, bi, lr):
        if not self._is_streamed[bi]:
            return super()._adamw_bucket(bi, lr)
        if not self._host:
            raise RuntimeError("OffloadAdamW used after close()")
        b, s0, s1, o = self.slices[bi]
        n = s1 - s0
        prev = self._stored.pop(bi, None)
        if prev is not None:                 # this step's loads read what the last step's stores wrote
            self.h2d_stream.wait_event(prev)
        b1, b2 = self.betas
        decay_n = min(n, max(0, b.decay_size - s0))
        if self.optim == "adamw_8bit":
            q, nb = self.block_offsets[bi], n_blocks(n)
            ops.adamw8bit_offload_bucket(self.host_master[o:o + n], self.host_exp_avg_q[o:o + n],
                                         self.host_exp_avg_sq_q[o:o + n], self.host_absmax[q:q + nb],
                                         self.host_absmax_sq[q:q + nb], b.grad[s0:s1], b.flat[s0:s1], decay_n,
                                         self.map_m, self.map_v, self.ring, self.slot_elems, lr, b1, b2, self.eps,
                                         self.wd, self.step_count, self.h2d_stream, self.d2h_stream)
        else:
            ops.adamw_offload_bucket(self.host_master[o:o + n], self.host_exp_avg[o:o + n],
                                     self.host_exp_avg_sq[o:o + n], b.grad[s0:s1], b.flat[s0:s1], decay_n, self.ring,
                                     self.slot_elems, lr, b1, b2, self.eps, self.wd, self.step_count, self.h2d_stream,
                                     self.d2h_stream)
        ev = torch.cuda.Event()
        ev.record(self.d2h_stream)
        self._stored[bi] = ev

    def _state_parts(self):
        """(name, device tensor, host tensor, checkpoint length, [(global offset, local offset, length)] per slice) of
        every state tensor."""
        out = []
        for name, _, per in state_parts(self.optim):
            spans = []
            for (b, s0, s1, o), g, q, gq in zip(self.slices, self._global, self.block_offsets, self._global_blocks):
                spans.append((g, o, s1 - s0) if per == "elem" else (gq, q, n_blocks(s1 - s0)))
            total = self.owned if per == "elem" else self.owned_blocks
            out.append((name, getattr(self, name), getattr(self, "host_" + name), total, spans))
        return out

    def state_dict(self):
        """The Zero2AdamW layout (full flat tensors, here on the host), so either optimizer resumes the other's
        checkpoint of the same format. The tensors take state_bytes per slice of host memory on top of the pinned state
        (81 GB at 7B with fp32 moments): MemAvailable is checked first, so a checkpoint that does not fit raises
        MemoryError instead of waking the kernel's OOM killer."""
        check_host_memory(self.state_nbytes, (self._cfg["meminfo"] or _read_meminfo)(), self._cfg["host_margin"])
        self.wait_all()
        torch.cuda.current_stream().synchronize()
        if self.opt_stream is not None:
            self.opt_stream.synchronize()
        self._drain()
        out = {}
        for key, dev_t, host_t, total, spans in self._state_parts():
            full = torch.empty(total, dtype=dev_t.dtype)
            for (g, o, n), st in zip(spans, self._is_streamed):
                full[g:g + n].copy_((host_t if st else dev_t)[o:o + n])
            out[key] = full
        return {"step": self.step_count, **out, **self._format_keys(), "rank": self.rank, "world": self.world}

    def load_state_dict(self, sd):
        assert sd["world"] == self.world and sd["rank"] == self.rank
        self.check_format(sd)
        self.check_state_size(sd)
        self.wait_all()
        if self.opt_stream is not None:
            self.opt_stream.synchronize()
        self._drain()
        self.step_count = sd["step"]
        for key, dev_t, host_t, _, spans in self._state_parts():
            src = sd[key]
            for (g, o, n), st in zip(spans, self._is_streamed):
                (host_t if st else dev_t)[o:o + n].copy_(src[g:g + n])
        torch.cuda.current_stream().synchronize()
