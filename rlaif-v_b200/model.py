"""LLaVA-1.5 DPO policy on the H100 kernels: parameter storage + hand-written forward / backward.

Mirrors what the reference executes in `get_beta_and_logps(..., is_llava15=True)`
(muffin/train/trainers.py:205-231): CLIP tower (frozen, llava/model/multimodal_encoder/clip_encoder.py:46-58)
-> mm_projector (llava/model/multimodal_projector/builder.py:39-46) -> image-token splice
(llava/model/llava_arch.py:150-330) -> Llama decoder (llava/model/language_model/llava_llama.py:57-102)
-> per-token log-prob gather (muffin/eval/muffin_inference_logp.py:82-115) — and the backward of
all trainable parts.  There is no autograd here: the backward is an explicit sequence of kernel
launches over an activation stash.

All arithmetic runs in the C-ABI library (ops.*); torch supplies device memory, streams and
zero-fills.  Parameters live in ONE flat bf16 buffer cut into buckets (embed | layer i | head |
projector); gradients in a same-layout flat buffer, so the ZeRO-2 optimizer (zero2.py) can
reduce-scatter / update / all-gather bucket slices in place.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import ops

IGNORE_INDEX = -100
IMAGE_TOKEN_INDEX = -200
_BF = torch.bfloat16
_F32 = torch.float32


@dataclass
class LlavaDims:
    """Dimensions (defaults = LLaVA-1.5-7B + CLIP-ViT-L/14-336; script/train/llava15_train.sh:8,11)."""
    vocab_size: int = 32000
    hidden_size: int = 4096
    intermediate_size: int = 11008
    num_layers: int = 32
    num_heads: int = 32
    num_kv_heads: int = 0          # 0 = num_heads; fewer = grouped-query attention (Mistral-7B: 32 / 8)
    rms_eps: float = 1e-5
    rope_theta: float = 10000.0
    max_len: int = 2048
    clip_hidden: int = 1024
    clip_intermediate: int = 4096
    clip_layers: int = 24
    clip_heads: int = 16
    image_size: int = 336
    patch_size: int = 14
    clip_eps: float = 1e-5
    select_layer: int = -2
    # vision front-end: "clip_mlp" = frozen CLIP tower + trainable mlp2x_gelu projector (LLaVA-1.5);
    # "resampler" = OmniLMM-12B: external vision-tower tokens -> trainable perceiver resampler -> in-place
    # <im_patch> splice (omnilmm_model.OmniLMMDPOPolicy; omnilmm/model/omnilmm.py:107-120, 183-265)
    frontend: str = "clip_mlp"
    num_query: int = 64            # resampler queries = <im_patch> tokens per image (omnilmm.py:46-51)
    vision_width: int = 1792       # EVA-02-E token width
    im_patch_token: int = -1
    im_start_token: int = -1
    im_end_token: int = -1

    @property
    def head_dim(self):
        return self.hidden_size // self.num_heads

    @property
    def kv_heads(self):
        return self.num_kv_heads or self.num_heads

    @property
    def kv_size(self):
        return self.kv_heads * self.head_dim

    @property
    def num_patches(self):
        return (self.image_size // self.patch_size) ** 2

    @property
    def clip_layers_used(self):
        return self.clip_layers + 1 + self.select_layer if self.select_layer < 0 else self.select_layer

    @property
    def patch_k(self):
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_k_pad(self):
        return (self.patch_k + 63) // 64 * 64


@dataclass
class Segment:
    name: str           # storage name (fused tensors have their own names)
    shape: tuple
    offset: int         # element offset in the flat buffer
    decay: bool


@dataclass
class Bucket:
    name: str
    start: int
    size: int            # padded to a multiple of PAD
    decay_size: int      # leading part that gets weight decay; the rest (norm weights, biases) does not
    segments: list = field(default_factory=list)


class FlatStore:
    """Flat bf16 parameter storage cut into optimizer buckets, a same-layout gradient buffer and named views of both.

    layout: [(bucket name, [(segment name, shape)] with weight decay, [(segment name, shape)] without)]. A bucket is
    its decay prefix (matrices), its no-decay tail (norms, biases), then zero padding up to a multiple of PAD.
    `p` / `g` map segment names to views of `flat` / `grad` in segment order. grads=False (a frozen module): `grad` is
    None, `g` is empty and there are no optimizer buckets.
    """
    # Zero2AdamW cuts every bucket into `world` equal slices whose length must be a multiple of 8 elements (16 B of
    # bf16); 1024-element buckets divide that way for every power-of-two world size up to 128
    PAD = 1024

    def __init__(self, layout, device, grads=True):
        self.buckets, off = [], 0
        for name, decay, nodecay in layout:
            b = Bucket(name=name, start=off, size=0, decay_size=sum(math.prod(shape) for _, shape in decay))
            o = off
            for segs, dec in ((decay, True), (nodecay, False)):
                for nm, shape in segs:
                    b.segments.append(Segment(nm, shape, o, dec))
                    o += math.prod(shape)
            b.size = (o - off + self.PAD - 1) // self.PAD * self.PAD
            off += b.size
            self.buckets.append(b)
        self.numel = off
        self.flat = torch.zeros(off, dtype=_BF, device=device)
        self.grad = torch.zeros(off, dtype=_BF, device=device) if grads else None
        self.p = self._views(self.flat)
        self.g = self._views(self.grad) if grads else {}

    def _views(self, buf):
        return {s.name: buf[s.offset:s.offset + math.prod(s.shape)].view(s.shape)
                for b in self.buckets for s in b.segments}

    def opt_buckets(self, names=None):
        """zero2.OptBuckets of the buckets (optionally only the named ones), in bucket order."""
        from .zero2 import OptBucket
        if self.grad is None:
            return []
        return [OptBucket(b.name, self.flat[b.start:b.start + b.size], self.grad[b.start:b.start + b.size],
                          b.decay_size) for b in self.buckets if names is None or b.name in names]

    def zero_grad(self):
        if self.grad is not None:
            self.grad.zero_()

    def load_hf(self, state):
        """Copy a (possibly fp32, CPU) HF-named state dict into the flat storage through the subclass's hf_views()."""
        for k, v in self.hf_views().items():
            v.copy_(state[k].to(device=v.device, dtype=_BF))


# the decoder's frozen-base matrices of one layer (an FP8 base keeps them in Fp8BaseStore instead)
BASE_GROUPS = ("qkv", "o", "gu", "down")


class ParamStore(FlatStore):
    """The decoder's (and LLaVA's projector's) parameters and gradients.

    Storage tensors: embed, per layer {qkv [3H,H], o [H,H], gu [2F,H], down [H,F], ln1 [H], ln2 [H]},
    norm [H], lm_head [V,H], projector {w0 [H,C], w2 [H,H], b0 [H], b2 [H]}.
    HF state-dict names map onto (views of) these — see hf_views().
    base=False (FP8 frozen base): the layers hold only ln1 / ln2; qkv, o, gu and down live in Fp8BaseStore and have
    neither a bf16 copy nor gradient storage.
    """

    def __init__(self, dims: LlavaDims, device, base=True):
        self.dims = dims
        self.base = base
        super().__init__(self.layout(dims, base), device)

    @staticmethod
    def layout(d, base=True):
        H, F, V, C, KV = d.hidden_size, d.intermediate_size, d.vocab_size, d.clip_hidden, d.kv_size
        layout = [("embed", [("embed", (V, H))], [])]
        layout += [(f"layer{i}",
                    [(f"l{i}.qkv", (H + 2 * KV, H)), (f"l{i}.o", (H, H)), (f"l{i}.gu", (2 * F, H)),
                     (f"l{i}.down", (H, F))] if base else [],
                    [(f"l{i}.ln1", (H,)), (f"l{i}.ln2", (H,))]) for i in range(d.num_layers)]
        layout.append(("head", [("lm_head", (V, H))], [("norm", (H,))]))
        if d.frontend == "clip_mlp":
            layout.append(("projector", [("proj.w0", (H, C)), ("proj.w2", (H, H))],
                           [("proj.b0", (H,)), ("proj.b2", (H,))]))
        return layout

    def hf_views(self, grads=False):
        """HF state-dict name -> view into the fused parameter (or, with grads, gradient) storage
        (LlavaLlamaForCausalLM naming)."""
        d, src = self.dims, (self.g if grads else self.p)
        H, F, KV = d.hidden_size, d.intermediate_size, d.kv_size
        out = {"model.embed_tokens.weight": src["embed"], "model.norm.weight": src["norm"],
               "lm_head.weight": src["lm_head"]}
        if d.frontend == "clip_mlp":
            out.update({"model.mm_projector.0.weight": src["proj.w0"], "model.mm_projector.0.bias": src["proj.b0"],
                        "model.mm_projector.2.weight": src["proj.w2"], "model.mm_projector.2.bias": src["proj.b2"]})
        for i in range(d.num_layers):
            pre = f"model.layers.{i}."
            out[pre + "input_layernorm.weight"] = src[f"l{i}.ln1"]
            out[pre + "post_attention_layernorm.weight"] = src[f"l{i}.ln2"]
            if not self.base:
                continue
            qkv, gu = src[f"l{i}.qkv"], src[f"l{i}.gu"]
            out[pre + "self_attn.q_proj.weight"] = qkv[0:H]
            out[pre + "self_attn.k_proj.weight"] = qkv[H:H + KV]
            out[pre + "self_attn.v_proj.weight"] = qkv[H + KV:H + 2 * KV]
            out[pre + "self_attn.o_proj.weight"] = src[f"l{i}.o"]
            out[pre + "mlp.gate_proj.weight"] = gu[0:F]
            out[pre + "mlp.up_proj.weight"] = gu[F:2 * F]
            out[pre + "mlp.down_proj.weight"] = src[f"l{i}.down"]
        return out

    def hf_grad_views(self):
        return self.hf_views(grads=True)


class Fp8BaseStore:
    """The decoder's frozen-base matrices in e4m3 (DESIGN.md §3 "FP8 frozen base"): per layer one ops.Fp8Weight each
    for qkv [H+2KV, H], o [H, H], gu [2F, H] and down [H, F], quantized one HF tensor at a time as they arrive (the
    128-row blocks of q / k / v and of gate / up never straddle two of them: H and F are multiples of 128)."""

    # HF linear of layer i -> (group, first row of its block of the fused matrix)
    @staticmethod
    def hf_rows(d):
        H, F, KV = d.hidden_size, d.intermediate_size, d.kv_size
        return {"self_attn.q_proj": ("qkv", 0), "self_attn.k_proj": ("qkv", H), "self_attn.v_proj": ("qkv", H + KV),
                "self_attn.o_proj": ("o", 0), "mlp.gate_proj": ("gu", 0), "mlp.up_proj": ("gu", F),
                "mlp.down_proj": ("down", 0)}

    @staticmethod
    def check_dims(d):
        H, F, KV = d.hidden_size, d.intermediate_size, d.kv_size
        if H % 128 or F % 128 or KV % 128:
            raise ValueError("base_fp8: hidden_size (%d), intermediate_size (%d) and the k/v width (%d) must be "
                             "multiples of 128 (the FP8 block size)" % (H, F, KV))

    def __init__(self, dims: LlavaDims, device):
        self.check_dims(dims)
        d = self.dims = dims
        H, F, KV = d.hidden_size, d.intermediate_size, d.kv_size
        shapes = {"qkv": (H + 2 * KV, H), "o": (H, H), "gu": (2 * F, H), "down": (H, F)}
        self.w = [{g: ops.Fp8Weight(*shapes[g], device) for g in BASE_GROUPS} for _ in range(d.num_layers)]

    def quantize(self, i, group, row0, w):
        """Rows [row0, row0 + w.shape[0]) of layer i's `group` matrix from the bf16 (device) tensor w."""
        ops.quant_fp8_blocks(w, *self.w[i][group].rows(row0, w.shape[0]))

    def load_hf(self, state):
        """Stream the 7 HF linears of each layer through the quantizer, one tensor on the device at a time."""
        dev = self.w[0]["qkv"].q.device
        for i in range(self.dims.num_layers):
            for name, (group, row0) in self.hf_rows(self.dims).items():
                w = state[f"model.layers.{i}.{name}.weight"].to(device=dev, dtype=_BF).contiguous()
                self.quantize(i, group, row0, w)
                del w

    def nbytes(self):
        return sum(w.nbytes() for layer in self.w for w in layer.values())


class LoraStore(FlatStore):
    """Flat bf16 storage of the LoRA adapters (config e; muffin/train/train_llava15_lora.py:112-134, 304-318:
    r=64, alpha=16 on q,k,v,o,gate,up,down of every decoder layer; lm_head / projector / vision excluded).
    One bucket per layer: A_qkv [3r,H] (the three lora_A stacked — q,k,v share their input), B_q/B_k/B_v [H,r],
    A_o [r,H], B_o [H,r], A_gu [2r,H], B_g/B_u [F,r], A_d [r,F], B_d [H,r]. Adapters get weight decay like any
    other matrix (HF decay groups exclude only norms and biases)."""

    def __init__(self, dims: LlavaDims, device, r=64, alpha=16, seed=7, init_b_zero=True, dropout=0.0):
        self.dims, self.r, self.scaling = dims, r, alpha / r
        self.dropout = float(dropout)      # applied to the adapter input while training (peft lora_dropout)
        self.rng_seed = 0x5EED0000 + seed
        self.step = 0                      # advanced by the engine once per optimisation step
        H, F = dims.hidden_size, dims.intermediate_size
        shapes = [("A_qkv", (3 * r, H)), ("B_q", (H, r)), ("B_k", (H, r)), ("B_v", (H, r)), ("A_o", (r, H)),
                  ("B_o", (H, r)), ("A_gu", (2 * r, H)), ("B_g", (F, r)), ("B_u", (F, r)), ("A_d", (r, F)),
                  ("B_d", (H, r))]
        super().__init__([(f"lora{i}", [(f"l{i}.{nm}", shape) for nm, shape in shapes], [])
                          for i in range(dims.num_layers)], device)
        # peft init: lora_A kaiming_uniform(a=sqrt(5)) = U(-1/sqrt(in), 1/sqrt(in)), lora_B = 0
        g = torch.Generator(device=device).manual_seed(seed)
        for name, v in self.p.items():
            if ".A_" in name:
                bound = 1.0 / math.sqrt(v.shape[1])
                v.copy_((torch.rand(v.shape, generator=g, device=device) * 2 - 1) * bound)
            elif not init_b_zero:
                v.copy_(torch.randn(v.shape, generator=g, device=device) * 0.02)
        for i, b in enumerate(self.buckets):   # stacked lora_B views (adjacent segments) = second-source B operand
            offset = {s.name: s.offset for s in b.segments}
            oq, og = offset[f"l{i}.B_q"], offset[f"l{i}.B_g"]
            for src, base in ((self.p, self.flat), (self.g, self.grad)):
                src[f"l{i}.B_qkv"] = base[oq:oq + 3 * H * r].view(3 * H, r)
                src[f"l{i}.B_gu"] = base[og:og + 2 * F * r].view(2 * F, r)
                src[f"l{i}.B_o_cat"] = src[f"l{i}.B_o"]
                src[f"l{i}.B_d_cat"] = src[f"l{i}.B_d"]

    _PEFT = {"q_proj": ("A_qkv", 0, "B_q"), "k_proj": ("A_qkv", 1, "B_k"), "v_proj": ("A_qkv", 2, "B_v"),
             "o_proj": ("A_o", 0, "B_o"), "gate_proj": ("A_gu", 0, "B_g"), "up_proj": ("A_gu", 1, "B_u"),
             "down_proj": ("A_d", 0, "B_d")}

    def hf_views(self, grads=False):
        """`model.layers.{i}.{self_attn|mlp}.{x}_proj.lora_{A,B}.weight` -> views (peft adapter naming minus the
        `base_model.model.` prefix and the adapter name)."""
        src = self.g if grads else self.p
        r, out = self.r, {}
        for i in range(self.dims.num_layers):
            for proj, (a_name, idx, b_name) in self._PEFT.items():
                mod = "self_attn" if proj in ("q_proj", "k_proj", "v_proj", "o_proj") else "mlp"
                pre = f"model.layers.{i}.{mod}.{proj}."
                out[pre + "lora_A.weight"] = src[f"l{i}.{a_name}"][idx * r:(idx + 1) * r]
                out[pre + "lora_B.weight"] = src[f"l{i}.{b_name}"]
        return out


@dataclass
class RowPacking:
    """Packed rows of a training forward (DESIGN.md §3). Sequence s keeps its first len_s rows, len_s = 1 + the last
    position whose spliced label is supervised (1 if there is none): attention is causal, so no supervised log-prob
    depends on a later row, and the compact head gives those rows exactly zero gradient. Sequence s occupies packed
    rows [cu[s], cu[s] + len_s - pos0[s]); packed row cu[s] + t - pos0[s] is position t. With a shared prefix
    (pos0[s] > 0, DESIGN.md §3 "Shared prompt prefixes") positions t < pos0[s] are the lender's rows
    cu[partner[s]] + t; without one, pos0 is None and every sequence starts at position 0."""
    nseq: int
    T: int                   # padded length
    M: int                   # packed rows: sum of the own rows
    max_len: int             # most own rows of a sequence
    cu: torch.Tensor         # int32 [nseq + 1]
    pos: torch.Tensor        # int32 [M]: position t of each packed row (its RoPE position)
    rows: torch.Tensor       # int32 [M]: the padded row s*T + t of each packed row
    pos0: Optional[torch.Tensor] = None        # int32 [nseq] (device): first own position, a multiple of 128
    partner: Optional[torch.Tensor] = None     # int32 [nseq] (device): lender of a borrower, borrower of a lender, or -1
    pos0_h: Optional[torch.Tensor] = None      # the same two on the host (the attention entry points check them)
    partner_h: Optional[torch.Tensor] = None

    @property
    def shared(self):
        return self.pos0 is not None

    def packed_rows(self, row_pos):
        """Padded rows s*T + t (-1 = unused slot, kept) -> packed rows (a borrower's t < pos0[s]: the lender's row)."""
        rp = row_pos.long().clamp(min=0)
        s = torch.div(rp, self.T, rounding_mode="floor")
        if self.pos0 is None:
            return torch.where(row_pos >= 0, self.cu.long()[s] + rp - s * self.T, -1).to(torch.int32)
        t = rp - s * self.T
        p0 = self.pos0.long()[s]
        cu = self.cu.long()
        r = torch.where(t < p0, cu[self.partner.long()[s].clamp(min=0)] + t, cu[s] + t - p0)
        return torch.where(row_pos >= 0, r, -1).to(torch.int32)


# sequences one attention launch with shared prefixes takes (PREFIX_MAX_SEQ in csrc/attention.cu)
PREFIX_MAX_SEQ = 64
# shared prefixes end on a multiple of the attention kernels' 128-row tiles (why: DESIGN.md §3)
PREFIX_ALIGN = 128


def packed_lengths(labels):
    """len_s of spliced labels [nseq, T] (int64): 1 + the last supervised position, 1 if none."""
    t = torch.arange(labels.shape[1], device=labels.device)
    return (torch.where(labels != IGNORE_INDEX, t, -1).amax(dim=1) + 1).clamp(min=1)


def splice_sources(src, input_ids):
    """What each spliced position holds, [nseq, T] int64: its token id, or the negative splice code of its image
    feature row (or of padding). Two positions with equal values have equal decoder inputs."""
    return torch.where(src >= 0, input_ids.gather(1, src.clamp(min=0).long()), src.long())


def shared_prefix_lengths(labels, sources):
    """pos0 of a preference batch [2b, T] (pair i = sequences i and b + i), int64 [2b] on the device: 0 for the
    chosen side, and for the rejected side 128 * floor(min(p_i, f_i) / 128). p_i is the first position where the two
    sides' sources differ (T if none); f_i the smaller of their first supervised rows (row t is supervised when the
    label at t + 1 is; 0 for a side without one), so no shared row reaches the head."""
    nseq, T = labels.shape
    b = nseq // 2
    t = torch.arange(T, device=labels.device)
    p = torch.where(sources[:b] != sources[b:], t, T).amin(dim=1)
    sup = labels[:, 1:] != IGNORE_INDEX
    first = torch.where(sup.any(dim=1), torch.where(sup, t[:-1], T).amin(dim=1), 0)
    f = torch.minimum(first[:b], first[b:])
    pos0 = torch.div(torch.minimum(p, f), PREFIX_ALIGN, rounding_mode="floor") * PREFIX_ALIGN
    return torch.cat([torch.zeros_like(pos0), pos0])


def pack_rows(labels, sources=None):
    """RowPacking of spliced labels [nseq, T], or None when it would drop no row. sources (splice_sources of a
    preference batch, nseq = 2b): the rejected side of pair i also drops its first shared_prefix_lengths rows and
    reads them from the chosen side. Reads the lengths to the host once."""
    nseq, T = labels.shape
    lens = packed_lengths(labels)
    share = sources is not None and nseq % 2 == 0 and 0 < nseq <= PREFIX_MAX_SEQ
    if share:
        pos0 = shared_prefix_lengths(labels, sources)
        lens_h, pos0_h = torch.stack([lens, pos0]).cpu()
        share = bool(pos0_h.any())
    else:
        lens_h = lens.cpu()
    own, own_h = (lens - pos0, lens_h - pos0_h) if share else (lens, lens_h)
    M = int(own_h.sum())
    if M == nseq * T:
        return None
    dev = labels.device
    cu = torch.zeros(nseq + 1, dtype=torch.int64, device=dev)
    cu[1:] = torch.cumsum(own, 0)
    seq = torch.repeat_interleave(torch.arange(nseq, device=dev), own, output_size=M)
    pos = torch.arange(M, device=dev) - cu[seq]
    if not share:
        return RowPacking(nseq, T, M, int(own_h.max()), cu.int(), pos.int(), (seq * T + pos).int())
    pos += pos0[seq]

    def partners(p0):                        # built twice (device, host): an upload would wait for the stream
        other = torch.arange(nseq, device=p0.device).roll(nseq // 2)
        return torch.where((p0 > 0) | (p0.roll(nseq // 2) > 0), other, -1).int()
    return RowPacking(nseq, T, M, int(own_h.max()), cu.int(), pos.int(), (seq * T + pos).int(),
                      pos0.int(), partners(pos0), pos0_h.int(), partners(pos0_h))


class ClipWeights:
    """Frozen CLIP-ViT weights in kernel-friendly form (fused qkv, padded patch-embedding matrix)."""

    def __init__(self, dims: LlavaDims, device, state=None, seed=1):
        d = dims
        C, I = d.clip_hidden, d.clip_intermediate
        vp = "model.vision_tower.vision_tower.vision_model."
        if state is None:
            g = torch.Generator().manual_seed(seed)
            state = {}

            def rnd(name, *shape, s=0.02):
                state[name] = torch.randn(*shape, generator=g) * s

            rnd(vp + "embeddings.class_embedding", C)
            rnd(vp + "embeddings.patch_embedding.weight", C, 3, d.patch_size, d.patch_size)
            rnd(vp + "embeddings.position_embedding.weight", d.num_patches + 1, C)
            state[vp + "pre_layrnorm.weight"] = torch.ones(C)
            state[vp + "pre_layrnorm.bias"] = torch.zeros(C)
            for i in range(d.clip_layers_used):
                pre = vp + f"encoder.layers.{i}."
                for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
                    rnd(pre + f"self_attn.{nm}.weight", C, C)
                    state[pre + f"self_attn.{nm}.bias"] = torch.zeros(C)
                rnd(pre + "mlp.fc1.weight", I, C)
                state[pre + "mlp.fc1.bias"] = torch.zeros(I)
                rnd(pre + "mlp.fc2.weight", C, I)
                state[pre + "mlp.fc2.bias"] = torch.zeros(C)
                for ln in ("layer_norm1", "layer_norm2"):
                    state[pre + ln + ".weight"] = torch.ones(C)
                    state[pre + ln + ".bias"] = torch.zeros(C)

        def dev(t):
            return t.to(device=device, dtype=_BF).contiguous()

        self.cls = dev(state[vp + "embeddings.class_embedding"])
        w = state[vp + "embeddings.patch_embedding.weight"].reshape(C, -1).to(_BF)
        wp = torch.zeros(C, d.patch_k_pad, dtype=_BF)
        wp[:, : d.patch_k] = w
        self.patch_w = wp.to(device)
        self.pos = dev(state[vp + "embeddings.position_embedding.weight"])
        self.pre_ln_w = dev(state[vp + "pre_layrnorm.weight"])
        self.pre_ln_b = dev(state[vp + "pre_layrnorm.bias"])
        self.layers = []
        for i in range(d.clip_layers_used):
            pre = vp + f"encoder.layers.{i}."
            L = {}
            L["qkv_w"] = dev(torch.cat([state[pre + f"self_attn.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")], 0))
            L["qkv_b"] = dev(torch.cat([state[pre + f"self_attn.{n}.bias"] for n in ("q_proj", "k_proj", "v_proj")], 0))
            L["o_w"] = dev(state[pre + "self_attn.out_proj.weight"])
            L["o_b"] = dev(state[pre + "self_attn.out_proj.bias"])
            L["fc1_w"] = dev(state[pre + "mlp.fc1.weight"])
            L["fc1_b"] = dev(state[pre + "mlp.fc1.bias"])
            L["fc2_w"] = dev(state[pre + "mlp.fc2.weight"])
            L["fc2_b"] = dev(state[pre + "mlp.fc2.bias"])
            for ln in ("layer_norm1", "layer_norm2"):
                L[ln + "_w"] = dev(state[pre + ln + ".weight"])
                L[ln + "_b"] = dev(state[pre + ln + ".bias"])
            self.layers.append(L)


class LlavaDPOPolicy:
    """Forward (policy log-probs) and backward (gradients into ParamStore.grad) of one micro-batch."""

    def __init__(self, dims: LlavaDims, device="cuda", hf_state=None, seed=0, init_std=0.02, base_fp8=False):
        self.dims = dims
        self.device = torch.device(device)
        # base_fp8: the decoder's qkv / o / gu / down are stored only in e4m3 (Fp8BaseStore) and their forward and dgrad
        # GEMMs run on FP8 tensor cores; trains only with LoRA (the base gets no gradient)
        self.base_fp8 = bool(base_fp8)
        self.fp8 = Fp8BaseStore(dims, self.device) if self.base_fp8 else None
        self.store = ParamStore(dims, self.device, base=not self.base_fp8)
        has_clip = dims.frontend == "clip_mlp"
        if hf_state is not None:
            self.store.load_hf(hf_state)
            if self.fp8 is not None:
                self.fp8.load_hf(hf_state)
            self.clip = ClipWeights(dims, self.device, hf_state) if has_clip else None
        else:
            self._random_init(seed, init_std)
            self.clip = ClipWeights(dims, self.device, None, seed + 1) if has_clip else None
        self._rope = {}
        self._bufs = {}
        # True: also stash the normalised inputs and the SwiGLU product (22 KB/token/layer more memory,
        # 3 fewer row passes per layer in the backward). The engine turns it on when HBM allows.
        self.stash_extra = False
        # middle ground for one GPU (unsharded 81 GB optimizer state): stash only the SwiGLU product (22 KB/token/layer,
        # 12.8 GB at config b) — saves the largest of the three recompute passes
        self.stash_act = False
        # training forward sends only the supervised positions through final norm / lm_head / log-softmax
        # (forward_logps); inference / the reference log-prob pre-pass keep the full head (per-token values of every
        # position are part of the parquet contract)
        self.compact_head = True
        # attention backward as two kernels (dK/dV, dQ) without fp32 atomics; False = the fused round-1 kernel
        self.split_attention_bwd = True
        # ragged training batches run the decoder on packed rows (RowPacking) when that drops any row; False = always
        # the padded layout (the reference the packed path is tested against). A policy on the CPU only serves host-side
        # dry runs of the padded launch sequence, so it packs only when asked.
        self.pack_rows = self.device.type == "cuda"
        # with packed rows: the rejected sequence of a pair reads the rows it shares with the chosen one (same inputs up
        # to its first supervised row, whole 128-row tiles) from the chosen copy instead of computing them again
        # (DESIGN.md §3 "Shared prompt prefixes"). Forward bits are unchanged; gradient sums change order. Not with
        # LoRA dropout, which draws a separate mask for each copy.
        self.share_prefix = False
        # SwiGLU backward inside the epilogue of the down-projection dgrad (no d(act) round trip, one launch less per
        # layer); False = separate swiglu_bwd pass
        self.fuse_swiglu_bwd = True
        self.embed_grad_f32 = None   # fp32 scatter target for embedding rows (allocated lazily)
        self._stash = None
        self.lora = None             # LoraStore: base weights frozen, adapters + mm_projector trainable

    def enable_lora(self, r=64, alpha=16, seed=7, init_b_zero=True, dropout=0.0):
        if self.dims.kv_heads != self.dims.num_heads:
            raise NotImplementedError("LoRA adapters on a grouped-query decoder (unequal q/k/v widths)")
        self.lora = LoraStore(self.dims, self.device, r=r, alpha=alpha, seed=seed, init_b_zero=init_b_zero,
                              dropout=dropout)
        return self.lora

    training = True

    def _lora_seed(self, i, group):
        """One dropout stream per (optimisation step, micro-batch forward, layer, linear group)."""
        L = self.lora
        g = ("qkv", "o", "gu", "down").index(group)
        return (L.rng_seed * 1000003 + L.step) * 4099 + (self._fwd_count * 131 + i) * 4 + g

    _fwd_count = 0

    # ---- what the optimizer trains / in which order the forward needs it ----
    def trainable_buckets(self):
        if self.lora is None:
            self._refuse_fp8_full()
            return self.store.opt_buckets()
        return self.lora.opt_buckets() + self.store.opt_buckets(names={"projector"})

    def _refuse_fp8_full(self):
        if self.base_fp8:
            raise ValueError("base_fp8: an FP8 frozen base trains only with LoRA adapters (enable_lora); full "
                             "fine-tuning needs the bf16 base weights and their gradients")

    def param_need_order(self):
        d = self.dims
        if self.lora is None:
            return ["projector", "embed"] + [f"layer{i}" for i in range(d.num_layers)] + ["head"]
        return ["projector"] + [f"lora{i}" for i in range(d.num_layers)]

    def activation_reserve_bytes(self, pairs, seq_len):
        """Device bytes a training micro-batch of `pairs` pairs at seq_len tokens needs next to the weights, gradients
        and optimizer state: the decoder's activations (zero2.activation_reserve_bytes) and, in full fine-tuning, the
        fp32 embedding-gradient buffer. The offloaded optimizer sizes its default device budget with it."""
        from .zero2 import activation_reserve_bytes
        d = self.dims
        reserve = activation_reserve_bytes(d, pairs, seq_len, self.stash_act)
        if self.base_fp8:
            # one reused pair of FP8 scratch buffers: codes (1 B) and row scales (4 B per 128) of the widest input
            widest = max(d.hidden_size + 2 * d.kv_size, 2 * d.intermediate_size)
            reserve += 2 * pairs * seq_len * widest * (1 + 4 / 128)
        if self.lora is None:
            reserve += 4 * d.vocab_size * d.hidden_size
        return reserve

    def layer_bucket_name(self, i):
        return f"layer{i}" if self.lora is None else f"lora{i}"

    def tail_bucket_names(self):
        """Buckets whose gradients are final only after the whole backward (reduced at the end of the step)."""
        return ["embed", "projector"]

    # ---- one linear group = base GEMM (+ LoRA adapters sharing the input) ----
    _GROUPS = {"qkv": ("A_qkv", ("B_q", "B_k", "B_v"), "B_qkv"), "o": ("A_o", ("B_o",), "B_o_cat"),
               "gu": ("A_gu", ("B_g", "B_u"), "B_gu"), "down": ("A_d", ("B_d",), "B_d_cat")}

    def _lin_fwd(self, i, group, x, out, residual=None, ls=None):
        """out = x @ W^T (+ residual). LoRA: t = s * x @ A^T (all sub-linears' lora_A stacked), then ONE GEMM
        accumulates x @ W^T and t_j @ B_j^T in the same accumulator tile (rlaifv_gemm_bf16_dual)."""
        if self.lora is None:
            if self.base_fp8:
                return ops.gemm_fp8(*self._fp8_quant(x), self.fp8.w[i][group], out, residual=residual)
            return ops.gemm(x, self.store.p[f"l{i}.{group}"], out, residual=residual)
        L = self.lora
        a_name, b_names, bcat = self._GROUPS[group]
        A = L.p[f"l{i}.{a_name}"]
        M = x.shape[0]
        t = torch.empty((M, A.shape[0]), dtype=_BF, device=self.device) if ls is not None else \
            self.buf("lora_t_" + group, (M, A.shape[0]))
        xa = x
        if L.dropout > 0.0 and self.training and ls is not None:
            # the sub-linears of a fused group share one mask (peft draws one per adapter; same marginal law)
            seed = self._lora_seed(i, group)
            xa = ops.dropout_fwd(x, L.dropout, seed, out=self.buf("lora_xd_%d" % x.shape[1], tuple(x.shape)),
                                 rows=ls.get("rows"))
            ls["seed_" + group] = seed
        ops.gemm(xa, A, t, alpha=L.scaling)
        n_sub = out.shape[1] // len(b_names) if len(b_names) > 1 else 0
        if self.base_fp8:
            ops.gemm_fp8(*self._fp8_quant(x), self.fp8.w[i][group], out, a2=t, b2=L.p[f"l{i}.{bcat}"], k2=L.r, r=L.r,
                         n_sub=n_sub, residual=residual)
        else:
            ops.gemm_dual(x, self.store.p[f"l{i}.{group}"], t, L.p[f"l{i}.{bcat}"], out, k2=L.r, r=L.r, n_sub=n_sub,
                          residual=residual)
        if ls is not None:
            ls["t_" + group] = t
        return out

    def _lin_bwd(self, i, group, dy, x, dx_out, ls, acc, glu=None):
        """dx = dy @ W (+ adapter path); weight gradients: base (full FT) or adapters (LoRA).
        glu (down projection only): the layer's gate|up pre-activations [M, 2F]; dx_out is then [M, 2F] and receives
        swiglu_bwd(glu, dy @ W) from the GEMM epilogue — d(act) stays in the accumulator (ops.gemm_swiglu_bwd)."""
        if self.lora is None:
            self._refuse_fp8_full()
            W = self.store.p[f"l{i}.{group}"]
            ops.gemm(dy, x, self.store.g[f"l{i}.{group}"], a_mn=True, b_mn=True, accumulate=acc)
            if glu is not None:
                return ops.gemm_swiglu_bwd(dy, W, glu, dx_out)
            return ops.gemm(dy, W, dx_out, b_mn=True)
        L = self.lora
        W = None if self.base_fp8 else self.store.p[f"l{i}.{group}"]
        a_name, b_names, _ = self._GROUPS[group]
        A = L.p[f"l{i}.{a_name}"]
        r, M = L.r, x.shape[0]
        t = ls["t_" + group]                      # already scaled by s
        dt = self.buf("lora_dt_" + group, (M, A.shape[0]))
        n_out = dy.shape[1] // len(b_names)
        for j, bn in enumerate(b_names):
            dy_j = dy[:, j * n_out:(j + 1) * n_out]
            ops.gemm(dy_j, L.p[f"l{i}.{bn}"], dt[:, j * r:(j + 1) * r], b_mn=True, alpha=L.scaling)   # dt_j = s dy_j B_j
            ops.gemm(dy_j, t[:, j * r:(j + 1) * r], L.g[f"l{i}.{bn}"], a_mn=True, b_mn=True, accumulate=acc)  # dB_j
        seed = ls.get("seed_" + group)
        if seed is not None:
            # dropout on the adapter input: dA sees the dropped input, and the adapter's dx passes through the mask
            xd = ops.dropout_fwd(x, L.dropout, seed, out=self.buf("lora_xd_%d" % x.shape[1], tuple(x.shape)),
                                 rows=ls.get("rows"))
            ops.gemm(dt, xd, L.g[f"l{i}.{a_name}"], a_mn=True, b_mn=True, accumulate=acc)             # dA = dt^T drop(x)
            dx_plain = dx_out if glu is None else self.buf("dact", tuple(x.shape))
            if self.base_fp8:
                ops.gemm_fp8(*self._fp8_quant(dy), self.fp8.w[i][group], dx_plain, dgrad=True)
            else:
                ops.gemm(dy, W, dx_plain, b_mn=True)
            pa = ops.gemm(dt, A, self.buf("lora_xd_%d" % x.shape[1], tuple(x.shape)), b_mn=True)                       # dt @ A
            ops.dropout_bwd_add(dx_plain, pa, L.dropout, seed, rows=ls.get("rows"))
            return dx_plain if glu is None else ops.swiglu_bwd(glu, dx_plain, dx_out)
        ops.gemm(dt, x, L.g[f"l{i}.{a_name}"], a_mn=True, b_mn=True, accumulate=acc)                  # dA = dt^T x
        # dx = dy @ W + dt @ A in one pass (second source = stacked lora_A, MN-major like W)
        if self.base_fp8:
            return ops.gemm_fp8(*self._fp8_quant(dy), self.fp8.w[i][group], dx_out, dgrad=True, a2=dt, b2=A,
                                k2=A.shape[0], glu=glu)
        if glu is not None:
            return ops.gemm_swiglu_bwd(dy, W, glu, dx_out, a2=dt, b2=A)
        return ops.gemm_dual(dy, W, dt, A, dx_out, k2=A.shape[0], r=r, n_sub=0, b_mn=True)

    # ------------------------------------------------------------------ init / buffers
    def _fp8_quant(self, x):
        """(codes, row scales) of a GEMM input, in one pair of buffers every frozen-base GEMM reuses (each consumes
        them before the next quantization on the same stream)."""
        d = self.dims
        M, K = x.shape
        widest = max(d.hidden_size + 2 * d.kv_size, 2 * d.intermediate_size)
        q = self.buf("fp8_q", (M * widest,), torch.float8_e4m3fn)[:M * K].view(M, K)
        Mp = ops.fp8_scale_rows(M)
        s = self.buf("fp8_s", (Mp * (widest // 128),), _F32)[:Mp * (K // 128)].view(K // 128, Mp)
        return ops.quant_fp8_rows(x, q, s)

    def _random_init(self, seed, std):
        """The bf16 layout's draws in its order, so a bf16 and an FP8 policy of one seed hold the same weights (an FP8
        base matrix is drawn into a temporary and quantized right away)."""
        g = torch.Generator(device=self.device).manual_seed(seed)
        for _, decay, nodecay in ParamStore.layout(self.dims):
            for name, shape in decay + nodecay:
                s = Segment(name, shape, 0, True)
                v = self.store.p.get(name)
                if v is None:
                    v = torch.empty(shape, dtype=_BF, device=self.device)
                if len(s.shape) == 1 and (s.name.endswith("ln1") or s.name.endswith("ln2") or s.name == "norm"):
                    v.fill_(1.0)
                elif len(s.shape) == 1:
                    v.zero_()
                else:
                    # chunked normal_ to bound the fp32 temporary
                    flat = v.view(-1)
                    step = 1 << 26
                    for o in range(0, flat.numel(), step):
                        n = min(step, flat.numel() - o)
                        flat[o:o + n].copy_(torch.randn(n, generator=g, device=self.device, dtype=_F32) * std)
                    if name not in self.store.p:
                        i, group = name[1:].split(".")
                        self.fp8.quantize(int(i), group, 0, v)

    def buf(self, key, shape, dtype=_BF):
        t = self._bufs.get(key)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(shape, dtype=dtype, device=self.device)
            self._bufs[key] = t
        return t

    def rope_tables(self, T):
        if T not in self._rope:
            d = self.dims
            hd = d.head_dim
            inv_freq = 1.0 / (d.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
            pos = torch.arange(T, dtype=_F32)
            emb = torch.cat([pos[:, None] * inv_freq[None, :]] * 2, dim=-1)
            self._rope[T] = (emb.cos().to(_BF).to(self.device).contiguous(),
                             emb.sin().to(_BF).to(self.device).contiguous())
        return self._rope[T]

    # ------------------------------------------------------------------ CLIP (frozen, forward only)
    def encode_images(self, images):
        """images [b,3,S,S] (any float dtype) -> CLIP patch features [b*P, C] (bf16)."""
        d, cw = self.dims, self.clip
        b = images.shape[0]
        P, C = d.num_patches, d.clip_hidden
        T = P + 1
        img = images.to(device=self.device, dtype=_BF).contiguous()
        cols = ops.clip_im2col(img, d.patch_size, d.patch_k_pad)
        patch = ops.gemm(cols, cw.patch_w)
        x = ops.clip_embed(patch, cw.cls, cw.pos, b, P)
        x = ops.layernorm_fwd(x, cw.pre_ln_w, cw.pre_ln_b, d.clip_eps)
        nh = d.clip_heads
        hd = C // nh
        scale = hd ** -0.5
        for L in cw.layers:
            h = ops.layernorm_fwd(x, L["layer_norm1_w"], L["layer_norm1_b"], d.clip_eps, out=self.buf("clip_h", x.shape))
            qkv = ops.gemm(h, L["qkv_w"], self.buf("clip_qkv", (b * T, 3 * C)), bias=L["qkv_b"])
            att, _ = ops.attention_fwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], b, T, nh, hd, False, scale,
                                       out=self.buf("clip_att", (b * T, C)), lse=self.buf("clip_lse", (b, nh, T), _F32))
            x2 = ops.gemm(att, L["o_w"], self.buf("clip_x2", x.shape), bias=L["o_b"], residual=x)
            h = ops.layernorm_fwd(x2, L["layer_norm2_w"], L["layer_norm2_b"], d.clip_eps, out=self.buf("clip_h", x.shape))
            f = ops.gemm(h, L["fc1_w"], self.buf("clip_f", (b * T, d.clip_intermediate)), bias=L["fc1_b"],
                         act=ops.ACT_QUICK_GELU)
            x = ops.gemm(f, L["fc2_w"], self.buf("clip_x", x.shape), bias=L["fc2_b"], residual=x2)
        return ops.clip_drop_cls(x, b, P)

    # ------------------------------------------------------------------ splice
    def splice(self, input_ids, labels, image_rows, n_blocks, img_index=None, T_hint=None):
        """llava_arch.prepare_inputs_labels_for_multimodal (attention_mask=None path).

        image_rows: [n_blocks*P, H] projected features; img_index[i] = feature block used by the
        i-th image slot (default: identity).  Returns (embeds [nseq*T,H], new_labels [nseq,T], src, T)."""
        d = self.dims
        nseq, L = input_ids.shape
        n_img, lens = ops.splice_count(input_ids, d.num_patches, d.max_len)
        if T_hint is None:
            T = int(lens.max().item())       # one tiny D2H per step (the reference syncs ~4x per sample)
            n_slots = int(torch.clamp(n_img, min=1).sum().item())
        else:
            T, n_slots = T_hint
        if img_index is None:
            img_index = torch.arange(n_slots, dtype=torch.int32, device=self.device)
        src, new_labels = ops.splice_map(input_ids, labels, n_img, img_index, d.num_patches, T, d.max_len)
        embeds = ops.splice_gather(src, input_ids, self.store.p["embed"], image_rows,
                                   out=self.buf("x0", (nseq * T, d.hidden_size)))
        return embeds, new_labels, src, T

    # ------------------------------------------------------------------ decoder layers
    def _run_layers(self, x, nseq, T, st, pk=None):
        """32 x [RMSNorm -> fused qkv GEMM -> RoPE -> causal attention -> o GEMM(+res) -> RMSNorm ->
        fused gate|up GEMM -> SwiGLU -> down GEMM(+res)]; st (dict or None) receives the per-layer stash.
        pk (RowPacking): x holds the packed rows, attention and RoPE run variable-length."""
        d, P, dev = self.dims, self.store.p, self.device
        H, F, KV = d.hidden_size, d.intermediate_size, d.kv_size
        nh, hd, nkv = d.num_heads, d.head_dim, d.kv_heads
        QKV = H + 2 * KV
        M = nseq * T if pk is None else pk.M
        cos, sin = self.rope_tables(T)
        scale = hd ** -0.5
        keep_stash = st is not None
        lse_shape = (nseq, nh, T) if pk is None else (nh * M,)
        for i in range(d.num_layers):
            self._need(self.layer_bucket_name(i))
            ls = None
            if keep_stash:
                ls = {"x": x} if pk is None else {"x": x, "rows": pk.rows}
                qkv = torch.empty((M, QKV), dtype=_BF, device=dev)
                att = torch.empty((M, H), dtype=_BF, device=dev)
                x2 = torch.empty((M, H), dtype=_BF, device=dev)
                gu = torch.empty((M, 2 * F), dtype=_BF, device=dev)
                x3 = torch.empty((M, H), dtype=_BF, device=dev)
                rstd1 = torch.empty(M, dtype=_F32, device=dev)
                rstd2 = torch.empty(M, dtype=_F32, device=dev)
                lse = torch.empty(lse_shape, dtype=_F32, device=dev)
            else:
                qkv, att = self.buf("qkv", (M, QKV)), self.buf("att", (M, H))
                x2, gu = self.buf("x2", (M, H)), self.buf("gu", (M, 2 * F))
                x3 = self.buf("x3_%d" % (i & 1), (M, H))
                rstd1 = rstd2 = None
                lse = self.buf("lse", lse_shape, _F32)
            extra = keep_stash and self.stash_extra
            n1 = ops.rmsnorm_fwd(x, P[f"l{i}.ln1"], d.rms_eps,
                                 out=torch.empty((M, H), dtype=_BF, device=dev) if extra else self.buf("n", (M, H)),
                                 rstd=rstd1)
            self._lin_fwd(i, "qkv", n1, qkv, ls=ls if keep_stash else None)
            if pk is None:
                ops.rope_fwd(qkv, cos, sin, T, nh, hd, n_kv_heads=nkv)
                ops.attention_fwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], nseq, T, nh, hd, True, scale, out=att,
                                  lse=lse, n_kv_heads=nkv)
            else:
                ops.rope_pos_fwd(qkv, cos, sin, pk.pos, nh, hd, n_kv_heads=nkv)
                att_fwd = ops.attention_varlen_prefix_fwd if pk.shared else ops.attention_varlen_fwd
                att_fwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], pk, nh, hd, scale, att, lse, n_kv_heads=nkv)
            self._lin_fwd(i, "o", att, x2, residual=x, ls=ls if keep_stash else None)
            n2 = ops.rmsnorm_fwd(x2, P[f"l{i}.ln2"], d.rms_eps,
                                 out=torch.empty((M, H), dtype=_BF, device=dev) if extra else self.buf("n", (M, H)),
                                 rstd=rstd2)
            self._lin_fwd(i, "gu", n2, gu, ls=ls if keep_stash else None)
            keep_act = extra or (keep_stash and self.stash_act)
            act = ops.swiglu_fwd(gu, torch.empty((M, F), dtype=_BF, device=dev) if keep_act else self.buf("act", (M, F)))
            self._lin_fwd(i, "down", act, x3, residual=x2, ls=ls if keep_stash else None)
            if keep_stash:
                ls.update(qkv=qkv, att=att, x2=x2, gu=gu, rstd1=rstd1, rstd2=rstd2, lse=lse)
                if extra:
                    ls.update(n1=n1, n2=n2, act=act)
                elif keep_act:
                    ls.update(act=act)
                st["layers"].append(ls)
            x = x3
        return x

    def decoder_logits(self, inputs_embeds):
        """inputs_embeds [nseq,T,H] bf16 -> logits [nseq,T,V] bf16 (inference form, no stash)."""
        d = self.dims
        nseq, T, H = inputs_embeds.shape
        x = inputs_embeds.to(device=self.device, dtype=_BF).reshape(nseq * T, H).contiguous()
        x = self._run_layers(x, nseq, T, None)
        self._need("head")
        hn = ops.rmsnorm_fwd(x, self.store.p["norm"], d.rms_eps, out=self.buf("hn", (nseq * T, H)))
        logits = ops.gemm(hn, self.store.p["lm_head"])
        return logits.view(nseq, T, d.vocab_size)

    # ------------------------------------------------------------------ forward
    def forward_logps(self, input_ids, labels, images, keep_stash=True, return_per_token=True, T_hint=None):
        """input_ids/labels [2b, L] int64 (win rows first, then rej — preference_collator_fn order),
        images [b,3,S,S].  Returns dict(per_token_logps [2b,T-1], logp [2b], avg_logp [2b], labels [2b,T])."""
        d, P = self.dims, self.store.p
        dev = self.device
        input_ids = input_ids.to(dev).contiguous()
        labels = labels.to(dev).contiguous()
        nseq = input_ids.shape[0]
        b = images.shape[0]
        H, F, V = d.hidden_size, d.intermediate_size, d.vocab_size
        nh, hd = d.num_heads, d.head_dim
        st = {"layers": []} if keep_stash else None
        self._fwd_count += 1

        proj = self._frontend_fwd(images, st)                                # [b*Pn, H] image rows
        # images are shared by the win and rej copy of a pair (trainers.py:190 cat([images, images]))
        n_slots = nseq
        img_index = (torch.arange(n_slots, dtype=torch.int32, device=dev) % b).contiguous() if nseq == 2 * b \
            else torch.arange(n_slots, dtype=torch.int32, device=dev)
        self._need("embed")
        x, new_labels, src, T = self.splice(input_ids, labels, proj, b, img_index,
                                            T_hint=(T_hint, n_slots) if T_hint is not None else None)
        compact = keep_stash and self.compact_head
        # training on a ragged batch: the decoder runs only each sequence's rows up to its last supervised position
        pk = None
        if compact and self.pack_rows:
            share = self.share_prefix and nseq == 2 * b and not (self.lora is not None and self.lora.dropout > 0.0)
            pk = pack_rows(new_labels, splice_sources(src, input_ids) if share else None)
        if pk is not None:
            x = ops.rows_gather(pk.rows, x, out=self.buf("xp", (pk.M, H)))
        if keep_stash:
            st.update(src=src, input_ids=input_ids, labels=new_labels, T=T, nseq=nseq, b=b,
                      n_feat_rows=proj.shape[0], pack=pk)
        x = self._run_layers(x, nseq, T, st, pk)
        self._need("head")
        row_pos = None
        if compact:
            # training: only the positions whose next token is supervised reach the final norm / lm_head / log-softmax
            # (get_batch_logps masks the rest out of the sum, muffin_inference_logp.py:93-104). A row of the collator
            # holds at most L labels, so L slots per sequence always suffice — no host sync for the count.
            # row_pos (padded positions) locates labels / per_tok; x_rows locates the rows of x.
            row_pos = ops.supervised_rows(new_labels, input_ids.shape[1])
            x_rows = row_pos if pk is None else pk.packed_rows(row_pos)
            x = ops.rows_gather(x_rows, x, out=self.buf("xc", (row_pos.numel(), H)))
            st.update(row_pos=row_pos, x_rows=x_rows)
        R, sfx = x.shape[0], "_c" if compact else ""      # rows that reach the head (M, or the compact row count)
        rstd_f = torch.empty(R, dtype=_F32, device=dev) if keep_stash else None
        hn = ops.rmsnorm_fwd(x, P["norm"], d.rms_eps, out=self.buf("hn" + sfx, (R, H)), rstd=rstd_f)
        logits = ops.gemm(hn, P["lm_head"], self.buf("logits" + sfx, (R, V)))
        per_tok, lse_v, logp, avg, count = ops.logp_fwd(logits, new_labels, nseq, T, row_pos=row_pos)
        if keep_stash:
            st.update(x_final=x, rstd_f=rstd_f, hn=hn, logits=logits, lse_v=lse_v, count=count)
            self._stash = st
        return dict(per_token_logps=per_tok, logp=logp, avg_logp=avg, labels=new_labels, T=T)

    # ------------------------------------------------------------------ backward
    def backward_logps(self, d_logp, use_average=False, accumulate=False, token_weight=None, weight_sum=None):
        """Gradients of sum_b d_logp[b] * logp[b] into store.grad (bf16; `accumulate` adds to what is
        there — used for the 2nd.. micro-batch of a step). token_weight [nseq, T-1] fp32: logp is the token-weighted
        sum of compute_weighted_logp (muffin/train/trainers.py:128-137); with use_average also pass weight_sum."""
        st = self._stash
        assert st is not None, "forward_logps(keep_stash=True) must precede backward_logps"
        d, P, G = self.dims, self.store.p, self.store.g
        dev = self.device
        nseq, T, b, pk = st["nseq"], st["T"], st["b"], st["pack"]
        M = nseq * T if pk is None else pk.M
        H, F, V, KV = d.hidden_size, d.intermediate_size, d.vocab_size, d.kv_size
        nh, hd, nkv = d.num_heads, d.head_dim, d.kv_heads
        scale = hd ** -0.5
        cos, sin = self.rope_tables(T)
        acc = bool(accumulate)

        row_pos = st.get("row_pos")               # compact head (training): logits hold the supervised rows only
        if token_weight is not None:
            assert not use_average or weight_sum is not None
        norm = (weight_sum if token_weight is not None else st["count"]) if use_average else None
        dlogits = ops.logp_bwd(st["logits"], st["labels"], st["lse_v"], d_logp, nseq, T, row_pos=row_pos,
                               token_weight=token_weight, norm=norm)
        frozen = self.lora is not None            # LoRA: lm_head / norms / embeddings / base matrices are frozen
        scratch_h = self.buf("frozen_dw", (H,)) if frozen else None
        Mh = dlogits.shape[0]                     # rows that went through the head (M, or the compact row count)
        if not frozen:
            ops.gemm(dlogits, st["hn"], G["lm_head"], a_mn=True, b_mn=True, accumulate=acc)    # dW = dlogits^T hn
        dhn = ops.gemm(dlogits, P["lm_head"], self.buf("dn_c" if row_pos is not None else "dn", (Mh, H)), b_mn=True)               # dhn = dlogits W
        dx = ops.rmsnorm_bwd(dhn, st["x_final"], P["norm"], st["rstd_f"],
                             self.buf("dx_c" if row_pos is not None else "dx_a", (Mh, H)),
                             scratch_h if frozen else G["norm"], dw_accumulate=acc and not frozen)
        if row_pos is not None:                   # back to the [M, H] residual stream (zeros at unsupervised positions)
            full = self.buf("dx_a", (M, H))
            full.zero_()
            dx = ops.rows_scatter(st["x_rows"], dx, full)
        if self.on_head_grads_ready is not None:
            self.on_head_grads_ready()
        for i in reversed(range(d.num_layers)):
            ls = st["layers"][i]
            # ---- MLP ----
            act = ls["act"] if "act" in ls else ops.swiglu_fwd(ls["gu"], self.buf("act", (M, F)))   # recompute
            if self.fuse_swiglu_bwd and F % 64 == 0:
                # d(act) = dx @ W_down never leaves the GEMM: its epilogue applies the SwiGLU backward (DESIGN.md §3)
                dgu = self._lin_bwd(i, "down", dx, act, self.buf("dgu", (M, 2 * F)), ls, acc, glu=ls["gu"])
            else:
                dact = self._lin_bwd(i, "down", dx, act, self.buf("dact", (M, F)), ls, acc)
                dgu = ops.swiglu_bwd(ls["gu"], dact, self.buf("dgu", (M, 2 * F)))
            n2 = ls["n2"] if "n2" in ls else ops.rmsnorm_fwd(ls["x2"], P[f"l{i}.ln2"], d.rms_eps,
                                                             out=self.buf("n", (M, H)))             # recompute
            dn2 = self._lin_bwd(i, "gu", dgu, n2, self.buf("dn", (M, H)), ls, acc)
            dx2 = ops.rmsnorm_bwd(dn2, ls["x2"], P[f"l{i}.ln2"], ls["rstd2"], self.buf("dx_b", (M, H)),
                                  scratch_h if frozen else G[f"l{i}.ln2"], dres=dx, dw_accumulate=acc and not frozen)
            # ---- attention ----
            datt = self._lin_bwd(i, "o", dx2, ls["att"], self.buf("datt", (M, H)), ls, acc)
            qkv = ls["qkv"]
            dqkv = self.buf("dqkv", (M, H + 2 * KV))
            if pk is not None:
                att_bwd = ops.attention_varlen_prefix_bwd if pk.shared else ops.attention_varlen_bwd
                att_bwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], ls["att"], datt, ls["lse"], pk, nh, hd, scale,
                        dqkv[:, :H], dqkv[:, H:H + KV], dqkv[:, H + KV:], self.buf("delta", (nh * M,), _F32),
                        n_kv_heads=nkv)
                ops.rope_pos_bwd(dqkv, cos, sin, pk.pos, nh, hd, n_kv_heads=nkv)
            elif self.split_attention_bwd:
                # dK/dV kernel + dQ kernel: dQ lands in the q block of dqkv as bf16, rotated back in place
                ops.attention_bwd_split(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], ls["att"], datt, ls["lse"], nseq,
                                        T, T, nh, hd, True, scale, dqkv[:, :H], dqkv[:, H:H + KV], dqkv[:, H + KV:],
                                        n_kv_heads=nkv, delta_ws=self.buf("delta", (nseq, nh, T), _F32))
                ops.rope_bwd(dqkv, None, cos, sin, T, nh, hd, n_kv_heads=nkv)
            else:
                dq32 = self.buf("dq32", (M, H), _F32)
                dq32.zero_()
                ops.attention_bwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], ls["att"], datt, ls["lse"], nseq, T, nh,
                                  hd, scale, dq32, dqkv[:, H:H + KV], dqkv[:, H + KV:],
                                  self.buf("delta", (nseq, nh, T), _F32), n_kv_heads=nkv)
                ops.rope_bwd(dqkv, dq32, cos, sin, T, nh, hd, n_kv_heads=nkv)
            n1 = ls["n1"] if "n1" in ls else ops.rmsnorm_fwd(ls["x"], P[f"l{i}.ln1"], d.rms_eps,
                                                             out=self.buf("n", (M, H)))             # recompute
            dn1 = self._lin_bwd(i, "qkv", dqkv, n1, self.buf("dn", (M, H)), ls, acc)
            dx = ops.rmsnorm_bwd(dn1, ls["x"], P[f"l{i}.ln1"], ls["rstd1"], self.buf("dx_a", (M, H)),
                                 scratch_h if frozen else G[f"l{i}.ln1"], dres=dx2, dw_accumulate=acc and not frozen)
            st["layers"][i] = None   # release this layer's stash
            if self.on_layer_grads_ready is not None:
                self.on_layer_grads_ready(i)
        # ---- splice backward: embedding rows + projected image rows ----
        if frozen:
            pass
        elif self.embed_grad_f32 is None:
            self.embed_grad_f32 = torch.zeros((V, H), dtype=_F32, device=dev)
        elif not acc:
            self.embed_grad_f32.zero_()
        n_feat_rows = st["n_feat_rows"]
        dfeat32 = self.buf("dfeat32", (n_feat_rows, H), _F32)
        dfeat32.zero_()
        src, ids = st["src"], st["input_ids"]
        if pk is not None:
            # scatter straight from the packed rows: one "sequence" of M rows over the flattened ids, a token's source
            # index offset by its sequence's start in them
            L = ids.shape[1]
            src = src.view(-1)[pk.rows.long()]
            src = torch.where(src >= 0, src + torch.div(pk.rows, T, rounding_mode="floor") * L, src).view(1, -1)
            ids = ids.view(1, -1)
        ops.splice_scatter(src, ids, dx, None if frozen else self.embed_grad_f32, dfeat32)
        dproj = ops.f32_to_bf16(dfeat32, self.buf("dproj", (n_feat_rows, H)))
        self._frontend_bwd(dproj, st, acc)
        self._stash = None

    # ------------------------------------------------------------------ vision front-end (LLaVA-1.5: CLIP + projector)
    def _frontend_fwd(self, images, st):
        """images [b,3,S,S] -> projected image rows [b*P, H]; st (dict or None) receives what the backward needs."""
        P, H = self.store.p, self.dims.hidden_size
        feats = self.encode_images(images)                                   # [b*Pn, C]
        self._need("projector")
        pre = ops.gemm(feats, P["proj.w0"], self.buf("proj_pre", (feats.shape[0], H)), bias=P["proj.b0"])
        post = ops.gelu_fwd(pre, self.buf("proj_post", pre.shape))
        proj = ops.gemm(post, P["proj.w2"], self.buf("proj_out", pre.shape), bias=P["proj.b2"])
        if st is not None:
            st.update(feats=feats, proj_pre=pre, proj_post=post)
        return proj

    def _frontend_bwd(self, dproj, st, acc):
        """dproj [b*P, H] bf16 = gradient of the image rows -> mm_projector gradients (the CLIP tower is frozen)."""
        P, G, H = self.store.p, self.store.g, self.dims.hidden_size
        n_feat_rows = dproj.shape[0]
        ops.gemm(dproj, st["proj_post"], G["proj.w2"], a_mn=True, b_mn=True, accumulate=acc)
        ops.colsum(dproj, G["proj.b2"], accumulate=acc)
        dpost = ops.gemm(dproj, P["proj.w2"], self.buf("dpost", (n_feat_rows, H)), b_mn=True)
        dpre = ops.gelu_bwd(st["proj_pre"], dpost, self.buf("dpre", (n_feat_rows, H)))
        ops.gemm(dpre, st["feats"], G["proj.w0"], a_mn=True, b_mn=True, accumulate=acc)
        ops.colsum(dpre, G["proj.b0"], accumulate=acc)

    on_layer_grads_ready = None
    on_head_grads_ready = None
    param_ready = None          # callable(bucket_name): wait for that bucket's parameter all-gather (ZeRO-2)

    def _need(self, bucket):
        """Order the current stream after `bucket`'s ZeRO-2 parameter all-gather. Frozen buckets (LoRA: embed / head /
        base layers) are not the optimizer's and need no wait; an unknown trainable name is a bug and raises."""
        if self.param_ready is None:
            return
        if self.lora is not None and not (bucket.startswith("lora") or bucket in ("projector", "resampler")):
            return
        self.param_ready(bucket)

    def finalize_embed_grad(self):
        """fp32 embedding-row accumulator -> bf16 flat gradient (once per optimizer step)."""
        if self.lora is not None:
            return
        ops.f32_to_bf16(self.embed_grad_f32.view(-1), self.store.g["embed"].view(-1))
