"""Perceiver resampler of OmniLMM-12B (BASELINE config d; SURVEY.md §8 a13) on the CUDA library — forward and
backward, all arithmetic in the sm_90a kernels (wgmma GEMMs, cross-attention with S/O in registers, LayerNorm fwd/bwd).

Mirrors `Resampler` of omnilmm/model/resampler.py:93-168 (same parameter names, so `state_dict()` keys line up with
`model.resampler.*` of an OmniLMM checkpoint):

    x  [B, N, kv_dim] vision tokens  ->  ln_kv(kv_proj(x))                       (:153-154)
    q  = ln_q(query) + pos_embed,  k = x + get_abs_pos(pos_embed, N),  v = x     (:157-162)
    out = MultiheadAttention(q, k, v)  ->  ln_post  ->  @ proj                   (:158-168)

The learned queries are identical for every image, so their LayerNorm, position add and q-projection are computed
once ([Q,E] instead of [B,Q,E]); the cross-attention kernel reads that one block for every image (`q_shared`) and its
backward's fp32 dQ reduction sums over the batch. The frozen sin-cos position table and its bicubic resize
(`get_abs_pos`, :23-39) are constants prepared on the host at construction.
"""
import math

import numpy as np
import torch

from . import ops
from .model import FlatStore

_BF = torch.bfloat16
_F32 = torch.float32

# storage order = weight-decay group first (matrices and the learned queries), then what HF's Trainer exempts
# (biases and LayerNorm parameters), so the flat buffer is one optimizer bucket with a `decay_size` prefix
DECAY_PARAMS = ("query", "proj", "kv_proj.weight", "attn.in_proj_weight", "attn.out_proj.weight")
NO_DECAY_PARAMS = ("attn.in_proj_bias", "attn.out_proj.bias", "ln_q.weight", "ln_q.bias", "ln_kv.weight", "ln_kv.bias",
                   "ln_post.weight", "ln_post.bias")


def _sincos_1d(dim, pos):
    omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float32) / (dim / 2.0))
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def sincos_pos_embed(embed_dim, grid_size):
    """2-D sin-cos table of the query grid (resampler.py:42-87): channels [0,E/2) encode the column index, [E/2,E)
    the row index."""
    ar = np.arange(grid_size, dtype=np.float32)
    grid = np.stack(np.meshgrid(ar, ar), axis=0).reshape(2, 1, grid_size, grid_size)
    emb = np.concatenate([_sincos_1d(embed_dim // 2, grid[0]), _sincos_1d(embed_dim // 2, grid[1])], axis=1)
    return torch.from_numpy(emb).float()


def resize_pos_embed(pos_embed, n_tokens):
    """get_abs_pos (resampler.py:23-39): bicubic resize of the [g*g, E] table to n_tokens = t*t positions (host-side
    constant preparation)."""
    src, tgt = int(math.sqrt(pos_embed.shape[0])), int(math.sqrt(n_tokens))
    if src == tgt:
        return pos_embed
    t = pos_embed.float().reshape(1, src, src, -1).permute(0, 3, 1, 2)
    t = torch.nn.functional.interpolate(t, size=(tgt, tgt), mode="bicubic", align_corners=False)
    return t.permute(0, 2, 3, 1).flatten(0, 2)


class Resampler(FlatStore):
    def __init__(self, grid_size, embed_dim, num_heads, kv_dim, device="cuda", state=None, seed=0, eps=1e-6):
        assert embed_dim % num_heads == 0 and embed_dim // num_heads == 128, "cross-attention kernels need head_dim 128"
        assert kv_dim % 8 == 0 and embed_dim % 8 == 0
        self.num_queries, self.embed_dim, self.num_heads, self.kv_dim = grid_size ** 2, embed_dim, num_heads, kv_dim
        self.head_dim, self.eps, self.device = 128, eps, torch.device(device)
        E, Q = embed_dim, self.num_queries
        shapes = {"query": (Q, E), "proj": (E, E), "kv_proj.weight": (E, kv_dim), "attn.in_proj_weight": (3 * E, E),
                  "attn.in_proj_bias": (3 * E,), "attn.out_proj.weight": (E, E), "attn.out_proj.bias": (E,),
                  "ln_q.weight": (E,), "ln_q.bias": (E,), "ln_kv.weight": (E,), "ln_kv.bias": (E,),
                  "ln_post.weight": (E,), "ln_post.bias": (E,)}
        super().__init__([("resampler", [(n, shapes[n]) for n in DECAY_PARAMS],
                           [(n, shapes[n]) for n in NO_DECAY_PARAMS])], self.device)
        pos = sincos_pos_embed(E, grid_size)
        if state is not None:
            self.load_state_dict(state)
            if "pos_embed" in state:
                pos = state["pos_embed"].float().cpu()
        else:
            g = torch.Generator().manual_seed(seed)
            for name, t in self.p.items():                                  # resampler.py:133-147 initialisation
                if name.endswith("bias"):
                    t.zero_()
                elif name.startswith("ln_"):
                    t.fill_(1.0)
                elif name == "proj":
                    t.copy_((E ** -0.5 * torch.randn(t.shape, generator=g)).to(_BF))
                else:
                    t.copy_((0.02 * torch.randn(t.shape, generator=g).clamp_(-2, 2)).to(_BF))
        self.pos_embed_f32 = pos                                            # frozen (requires_grad_(False), :115-118)
        self.pos_q = pos.to(self.device, _BF).contiguous()
        self._pos_kv = {}
        self._stash = None

    # ---- nn.Module-ish surface ----
    def state_dict(self):
        sd = {k: v for k, v in self.p.items()}
        sd["pos_embed"] = self.pos_embed_f32
        return sd

    def load_state_dict(self, state):
        for k, v in self.p.items():
            v.copy_(state[k].to(device=self.device, dtype=_BF))

    def _pos_for(self, n_tokens):
        if n_tokens not in self._pos_kv:
            self._pos_kv[n_tokens] = resize_pos_embed(self.pos_embed_f32, n_tokens).to(self.device, _BF).contiguous()
        return self._pos_kv[n_tokens]

    # ---- forward ----
    def forward(self, x, keep_stash=True):
        """x [B, N, kv_dim] bf16 -> [B, Q, E] bf16."""
        P, E, Q, H = self.p, self.embed_dim, self.num_queries, self.num_heads
        B, N, _ = x.shape
        x2 = x.reshape(B * N, self.kv_dim).contiguous()
        wq, wk, wv = P["attn.in_proj_weight"][:E], P["attn.in_proj_weight"][E:2 * E], P["attn.in_proj_weight"][2 * E:]
        bq, bk, bv = P["attn.in_proj_bias"][:E], P["attn.in_proj_bias"][E:2 * E], P["attn.in_proj_bias"][2 * E:]
        xk = ops.gemm(x2, P["kv_proj.weight"])                                   # [BN, E]
        xn = ops.layernorm_fwd(xk, P["ln_kv.weight"], P["ln_kv.bias"], self.eps)
        k_in = ops.add_rows_bcast(xn, self._pos_for(N))
        k = ops.gemm(k_in, wk, bias=bk)
        v = ops.gemm(xn, wv, bias=bv)
        qn = ops.layernorm_fwd(P["query"], P["ln_q.weight"], P["ln_q.bias"], self.eps)
        q_in = ops.add_rows_bcast(qn, self.pos_q)
        qp = ops.gemm(q_in, wq, bias=bq)                                         # [Q, E], shared by the batch
        att, lse = ops.cross_attention_fwd(qp, k, v, B, Q, N, H, self.head_dim, 1.0 / math.sqrt(self.head_dim),
                                           q_shared=True)
        o = ops.gemm(att, P["attn.out_proj.weight"], bias=P["attn.out_proj.bias"])
        y = ops.layernorm_fwd(o, P["ln_post.weight"], P["ln_post.bias"], self.eps)
        z = ops.gemm(y, P["proj"], b_mn=True)                                    # y @ proj
        if keep_stash:
            self._stash = dict(B=B, N=N, x2=x2, xk=xk, xn=xn, k_in=k_in, k=k, v=v, q_in=q_in, qp=qp, att=att, lse=lse,
                               o=o, y=y)
        return z.view(B, Q, E)

    __call__ = forward

    # ---- backward ----
    def backward(self, d_out, input_grad=True):
        """d_out [B, Q, E] -> d_x [B, N, kv_dim]; parameter gradients are ACCUMULATED into `self.g` (bf16).
        input_grad=False (nothing upstream trains, e.g. a frozen vision tower): the backward stops at the parameters,
        the last dgrad GEMM is skipped and None is returned."""
        st, P, G, E, Q, H = self._stash, self.p, self.g, self.embed_dim, self.num_queries, self.num_heads
        assert st is not None, "backward() needs forward(keep_stash=True)"
        B, N = st["B"], st["N"]
        dz = d_out.reshape(B * Q, E).contiguous()
        wq, wk, wv = P["attn.in_proj_weight"][:E], P["attn.in_proj_weight"][E:2 * E], P["attn.in_proj_weight"][2 * E:]
        gwq, gwk, gwv = G["attn.in_proj_weight"][:E], G["attn.in_proj_weight"][E:2 * E], G["attn.in_proj_weight"][2 * E:]
        gbq, gbk, gbv = G["attn.in_proj_bias"][:E], G["attn.in_proj_bias"][E:2 * E], G["attn.in_proj_bias"][2 * E:]
        # z = y @ proj
        ops.gemm(st["y"], dz, G["proj"], a_mn=True, b_mn=True, accumulate=True)          # d proj = y^T dz
        dy = ops.gemm(dz, P["proj"])                                                      # dz @ proj^T
        do = torch.empty_like(dy)
        ops.layernorm_bwd(dy, st["o"], P["ln_post.weight"], self.eps, do, G["ln_post.weight"], G["ln_post.bias"])
        # out_proj
        ops.gemm(do, st["att"], G["attn.out_proj.weight"], a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(do, G["attn.out_proj.bias"])
        datt = ops.gemm(do, P["attn.out_proj.weight"], b_mn=True)
        # cross-attention
        dq32 = torch.zeros((Q, E), dtype=_F32, device=self.device)
        dk = torch.empty((B * N, E), dtype=_BF, device=self.device)
        dv = torch.empty((B * N, E), dtype=_BF, device=self.device)
        ops.cross_attention_bwd(st["qp"], st["k"], st["v"], st["att"], datt, st["lse"], B, Q, N, H, self.head_dim,
                                1.0 / math.sqrt(self.head_dim), dq32, dk, dv, q_shared=True)
        dqp = ops.f32_to_bf16(dq32, torch.empty((Q, E), dtype=_BF, device=self.device))
        # in_proj (q | k | v rows of the packed weight)
        ops.gemm(dqp, st["q_in"], gwq, a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(dqp, gbq)
        ops.gemm(dk, st["k_in"], gwk, a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(dk, gbk)
        ops.gemm(dv, st["xn"], gwv, a_mn=True, b_mn=True, accumulate=True)
        ops.colsum(dv, gbv)
        dq_in = ops.gemm(dqp, wq, b_mn=True)                                              # [Q, E]
        dxn = ops.gemm(dk, wk, b_mn=True)                                                 # d k_in (pos add: identity)
        ops.gemm(dv, wv, dxn, b_mn=True, accumulate=True)                                 # + d via v
        # ln_q / ln_kv
        dquery = torch.empty_like(dq_in)
        ops.layernorm_bwd(dq_in, P["query"], P["ln_q.weight"], self.eps, dquery, G["ln_q.weight"], G["ln_q.bias"])
        ops.add_rows_bcast(G["query"], dquery, out=G["query"])                            # d query += (in place)
        dxk = torch.empty_like(dxn)
        ops.layernorm_bwd(dxn, st["xk"], P["ln_kv.weight"], self.eps, dxk, G["ln_kv.weight"], G["ln_kv.bias"])
        # kv_proj
        ops.gemm(dxk, st["x2"], G["kv_proj.weight"], a_mn=True, b_mn=True, accumulate=True)
        self._stash = None
        if not input_grad:
            return None
        dx = ops.gemm(dxk, P["kv_proj.weight"], b_mn=True)
        return dx.view(B, N, self.kv_dim)
