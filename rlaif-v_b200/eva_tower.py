"""OmniLMM-12B's vision tower (BASELINE config d; SURVEY.md §8 a13 / f3) on the CUDA library — forward AND backward
(the tower is trainable in OmniLMM: `tune_clip=True`, omnilmm/model/omnilmm.py:57-70).

What the reference runs: `timm.create_model('eva02_enormous_patch14_clip_224.laion2b_plus', pretrained=False,
num_classes=0, dynamic_img_size=True, dynamic_img_pad=True)` with the last block replaced by Identity
(omnilmm/model/omnilmm.py:31-43), consumed as `forward_features(pixel_values)[:, num_prefix_tokens:]`
(omnilmm.py:107-118).  In timm 0.9.10 (timm/models/eva.py) that model is a post-norm ViT: patch 14, width 1792,
64 blocks (63 live), 16 heads of width **112**, GELU MLP 1792 -> 15360 -> 1792, absolute position embedding of the
16x16 pre-training grid bicubically resampled to the 32x32 grid of a 448 px input, LayerNorm eps 1e-6, final LayerNorm
on every token.  (The tests' CPU restatement of it lives under oracle/; timm is absent from the image, so that
restatement is parity-unpinned.)

Kernel mapping — nothing here is a new kernel family; the tower is built from the library's existing pieces:
  * every contraction is the wgmma GEMM (bias / residual epilogues, dgrad, wgrad straight into the flat bf16
    gradient bucket);
  * attention is the register-resident non-causal wgmma kernel pair (d = 128).  The model's head width is 112, so the fused qkv
    / proj weights are stored PADDED per head to 128 (16 zero rows per head in `qkv`, 16 zero columns per head in
    `proj`): q.k^T and P.V are unchanged by zero padding, every gradient that lands on a padded element is exactly
    zero (dQ_pad = dS.K_pad = 0, dK_pad = dS^T.Q_pad = 0, dV_pad = P^T.dO_pad with dO_pad = d(att).Wo_pad^T = 0), and
    AdamW keeps an exact zero at zero gradient, so the padding never leaks into the timm-named state dict;
  * the position-embedding resample is linear in `pos_embed`, so it is ONE small GEMM with a host-built constant
    matrix R [1 + 32*32, 1 + 16*16]; its backward (and the sum over the batch, and d cls_token) is one wgrad-form GEMM
    against the batch-tiled R;
  * LayerNorm fwd/bwd, GELU fwd/bwd, bias column sums, im2col patch extraction are the row kernels of rowops.cu.
Parameters live in one flat bf16 buffer cut into ZeRO-2 buckets `eva_embed | eva0 .. eva62` (decay prefix = matrices,
cls_token, pos_embed; no-decay tail = biases and LayerNorm parameters, HF Trainer's grouping).
"""
import torch

from . import ops
from .model import FlatStore

_BF = torch.bfloat16
_F32 = torch.float32
PADDED_HEAD = 128


class EvaDims:
    def __init__(self, embed_dim=1792, depth=64, num_heads=16, mlp_hidden=15360, patch_size=14, pretrain_img=224,
                 img_size=448, eps=1e-6):
        self.embed_dim, self.depth, self.num_heads, self.mlp_hidden = embed_dim, depth, num_heads, mlp_hidden
        self.patch_size, self.pretrain_img, self.img_size, self.eps = patch_size, pretrain_img, img_size, eps
        assert embed_dim % num_heads == 0 and embed_dim % 8 == 0 and mlp_hidden % 8 == 0
        self.head_dim = embed_dim // num_heads
        assert self.head_dim <= PADDED_HEAD
        self.live_blocks = depth - 1                    # blocks[-1] = Identity (omnilmm.py:43)
        self.grid = img_size // patch_size
        self.pretrain_grid = pretrain_img // patch_size
        self.n_tokens = self.grid ** 2                  # patch tokens per image (prefix token excluded)
        self.hp = num_heads * PADDED_HEAD               # padded width of q / k / v
        self.patch_k = 3 * patch_size * patch_size
        self.patch_k_pad = (self.patch_k + 63) // 64 * 64
        self.n_pos = 1 + self.pretrain_grid ** 2
        self.n_pos_pad = (self.n_pos + 7) // 8 * 8


def pos_resample_matrix(d: EvaDims):
    """R [1 + grid^2, n_pos]: timm's resample_abs_pos_embed (bicubic, antialias, align_corners=False, fp32) as a
    matrix — the prefix (cls) row passes through, the grid rows are the interpolation of the basis vectors."""
    import torch.nn.functional as F
    old, new = d.pretrain_grid, d.grid
    R = torch.zeros(1 + new * new, d.n_pos)
    R[0, 0] = 1.0
    if old == new:
        R[1:, 1:] = torch.eye(old * old)
        return R
    eye = torch.eye(old * old).reshape(1, old, old, old * old).permute(0, 3, 1, 2)       # channel c = basis c
    up = F.interpolate(eye, size=(new, new), mode="bicubic", antialias=True, align_corners=False)
    R[1:, 1:] = up.permute(0, 2, 3, 1).reshape(new * new, old * old)
    return R


class EvaTower(FlatStore):
    """forward(images [B,3,S,S]) -> tokens [B, grid^2, C]; backward(d_tokens) accumulates parameter gradients.

    trainable=False (OmniLMM's `tune_clip=False`): the tower is forward-only. It has no gradient buffer and no optimizer
    buckets, and backward() refuses."""

    def __init__(self, dims: EvaDims, device="cuda", state=None, seed=0, trainable=True):
        self.dims = d = dims
        self.device = torch.device(device)
        self.trainable = bool(trainable)
        C, Hd, HP = d.embed_dim, d.mlp_hidden, d.hp
        layout = [("eva_embed", [("patch_w", (C, d.patch_k_pad)), ("cls", (C,)), ("pos", (d.n_pos_pad, C))],
                   [("patch_b", (C,)), ("norm_w", (C,)), ("norm_b", (C,))])]
        layout += [(f"eva{i}",
                    [(f"b{i}.qkv_w", (3 * HP, C)), (f"b{i}.proj_w", (C, HP)), (f"b{i}.fc1_w", (Hd, C)),
                     (f"b{i}.fc2_w", (C, Hd))],
                    [(f"b{i}.qkv_b", (3 * HP,)), (f"b{i}.proj_b", (C,)), (f"b{i}.n1_w", (C,)), (f"b{i}.n1_b", (C,)),
                     (f"b{i}.fc1_b", (Hd,)), (f"b{i}.fc2_b", (C,)), (f"b{i}.n2_w", (C,)), (f"b{i}.n2_b", (C,))])
                   for i in range(d.live_blocks)]
        super().__init__(layout, self.device, grads=self.trainable)
        R = pos_resample_matrix(d)                                                   # [1+N, n_pos] fp32
        Rp = torch.zeros(R.shape[0], d.n_pos_pad)
        Rp[:, : d.n_pos] = R
        self.R = Rp.to(self.device, _BF).contiguous()
        self._R_tiled = {}
        self._bufs = {}
        self._stash = None
        self.param_ready = None          # callable(bucket name): ZeRO-2 parameter all-gather wait
        self.on_block_grads_ready = None  # callable(block index) / ("embed")
        if state is not None:
            self.load_timm_state(state)
        else:
            self._random_init(seed)

    # ------------------------------------------------------------------ parameters
    def _random_init(self, seed):
        """timm's Eva init: trunc_normal(0.02) for matrices / cls / pos, zeros for biases, ones for LayerNorm
        weights — written through load_timm_state so that the head padding is exactly zero."""
        d = self.dims
        g = torch.Generator().manual_seed(seed)
        C, Hd = d.embed_dim, d.mlp_hidden

        def tn(*shape):
            return (0.02 * torch.randn(*shape, generator=g)).clamp_(-0.04, 0.04)
        st = {"patch_embed.proj.weight": tn(C, 3, d.patch_size, d.patch_size), "patch_embed.proj.bias": torch.zeros(C),
              "cls_token": tn(1, 1, C), "pos_embed": tn(1, d.n_pos, C), "norm.weight": torch.ones(C),
              "norm.bias": torch.zeros(C)}
        self._load_top(st)
        for i in range(d.live_blocks):
            pre = f"blocks.{i}."
            self._load_block(i, {pre + "attn.qkv.weight": tn(3 * C, C), pre + "attn.q_bias": torch.zeros(C),
                                 pre + "attn.v_bias": torch.zeros(C), pre + "attn.proj.weight": tn(C, C),
                                 pre + "attn.proj.bias": torch.zeros(C), pre + "norm1.weight": torch.ones(C),
                                 pre + "norm1.bias": torch.zeros(C), pre + "mlp.fc1.weight": tn(Hd, C),
                                 pre + "mlp.fc1.bias": torch.zeros(Hd), pre + "mlp.fc2.weight": tn(C, Hd),
                                 pre + "mlp.fc2.bias": torch.zeros(C), pre + "norm2.weight": torch.ones(C),
                                 pre + "norm2.bias": torch.zeros(C)})

    def _dev(self, t):
        return t.to(device=self.device, dtype=_BF)

    def _load_top(self, st):
        d, P = self.dims, self.p
        P["patch_w"].zero_()
        P["patch_w"][:, : d.patch_k].copy_(self._dev(st["patch_embed.proj.weight"].reshape(d.embed_dim, -1)))
        P["patch_b"].copy_(self._dev(st["patch_embed.proj.bias"]))
        P["cls"].copy_(self._dev(st["cls_token"].reshape(-1)))
        P["pos"].zero_()
        P["pos"][: d.n_pos].copy_(self._dev(st["pos_embed"].reshape(d.n_pos, d.embed_dim)))
        P["norm_w"].copy_(self._dev(st["norm.weight"]))
        P["norm_b"].copy_(self._dev(st["norm.bias"]))

    def _load_block(self, i, st):
        d, P = self.dims, self.p
        C, nh, hd = d.embed_dim, d.num_heads, d.head_dim
        pre = f"blocks.{i}."
        qw = P[f"b{i}.qkv_w"].view(3, nh, PADDED_HEAD, C)
        qw.zero_()
        qw[:, :, :hd].copy_(self._dev(st[pre + "attn.qkv.weight"]).view(3, nh, hd, C))
        qb = P[f"b{i}.qkv_b"].view(3, nh, PADDED_HEAD)
        qb.zero_()
        qb[0, :, :hd].copy_(self._dev(st[pre + "attn.q_bias"]).view(nh, hd))
        qb[2, :, :hd].copy_(self._dev(st[pre + "attn.v_bias"]).view(nh, hd))       # k_bias is a zero buffer in timm
        pw = P[f"b{i}.proj_w"].view(C, nh, PADDED_HEAD)
        pw.zero_()
        pw[:, :, :hd].copy_(self._dev(st[pre + "attn.proj.weight"]).view(C, nh, hd))
        for src, dst in (("attn.proj.bias", "proj_b"), ("norm1.weight", "n1_w"), ("norm1.bias", "n1_b"),
                         ("mlp.fc1.weight", "fc1_w"), ("mlp.fc1.bias", "fc1_b"), ("mlp.fc2.weight", "fc2_w"),
                         ("mlp.fc2.bias", "fc2_b"), ("norm2.weight", "n2_w"), ("norm2.bias", "n2_b")):
            P[f"b{i}.{dst}"].copy_(self._dev(st[pre + src]))

    def load_timm_state(self, state):
        self._load_top(state)
        for i in range(self.dims.live_blocks):
            self._load_block(i, state)

    def timm_state(self, grads=False):
        """timm-named tensors (copies: the padded head layout is not expressible as a view of the timm shapes)."""
        d, S = self.dims, (self.g if grads else self.p)
        C, nh, hd = d.embed_dim, d.num_heads, d.head_dim
        out = {"patch_embed.proj.weight": S["patch_w"][:, : d.patch_k].reshape(C, 3, d.patch_size, d.patch_size).clone(),
               "patch_embed.proj.bias": S["patch_b"].clone(), "cls_token": S["cls"].reshape(1, 1, C).clone(),
               "pos_embed": S["pos"][: d.n_pos].reshape(1, d.n_pos, C).clone(), "norm.weight": S["norm_w"].clone(),
               "norm.bias": S["norm_b"].clone()}
        for i in range(d.live_blocks):
            pre = f"blocks.{i}."
            out[pre + "attn.qkv.weight"] = S[f"b{i}.qkv_w"].view(3, nh, PADDED_HEAD, C)[:, :, :hd].reshape(3 * C, C)
            qb = S[f"b{i}.qkv_b"].view(3, nh, PADDED_HEAD)
            out[pre + "attn.q_bias"] = qb[0, :, :hd].reshape(C)
            out[pre + "attn.v_bias"] = qb[2, :, :hd].reshape(C)
            out[pre + "attn.proj.weight"] = S[f"b{i}.proj_w"].view(C, nh, PADDED_HEAD)[:, :, :hd].reshape(C, C)
            for src, dst in (("attn.proj.bias", "proj_b"), ("norm1.weight", "n1_w"), ("norm1.bias", "n1_b"),
                             ("mlp.fc1.weight", "fc1_w"), ("mlp.fc1.bias", "fc1_b"), ("mlp.fc2.weight", "fc2_w"),
                             ("mlp.fc2.bias", "fc2_b"), ("norm2.weight", "n2_w"), ("norm2.bias", "n2_b")):
                out[pre + src] = S[f"b{i}.{dst}"].clone()
        return out

    def buf(self, key, shape, dtype=_BF):
        t = self._bufs.get(key)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(shape, dtype=dtype, device=self.device)
            self._bufs[key] = t
        return t

    def _need(self, bucket):
        if self.param_ready is not None:
            self.param_ready(bucket)

    def _R_for_batch(self, B):
        if B not in self._R_tiled:
            self._R_tiled[B] = self.R.repeat(B, 1).contiguous()          # [B*(1+N), n_pos_pad]
        return self._R_tiled[B]

    # ------------------------------------------------------------------ forward
    def forward(self, images, keep_stash=True):
        d, P, dev = self.dims, self.p, self.device
        C, Hd, HP, nh = d.embed_dim, d.mlp_hidden, d.hp, d.num_heads
        B = images.shape[0]
        assert images.shape[2] == d.img_size and images.shape[3] == d.img_size, "tower is built for one input size"
        N, S = d.n_tokens, d.n_tokens + 1
        M = B * S
        scale = d.head_dim ** -0.5
        img = images.to(device=dev, dtype=_BF).contiguous()
        self._need("eva_embed")
        cols = ops.clip_im2col(img, d.patch_size, d.patch_k_pad)                               # [B*N, k_pad]
        patch = ops.gemm(cols, P["patch_w"], bias=P["patch_b"])                                # conv 14x14 / 14
        pos = ops.gemm(self.R, P["pos"], b_mn=True)                                            # [1+N, C] resampled
        x = ops.clip_embed(patch, P["cls"], pos, B, N)                                         # cat(cls, patches) + pos
        st = {"B": B, "cols": cols, "blocks": []} if keep_stash else None
        for i in range(d.live_blocks):
            self._need(f"eva{i}")
            if keep_stash:
                qkv = torch.empty((M, 3 * HP), dtype=_BF, device=dev)
                att = torch.empty((M, HP), dtype=_BF, device=dev)
                a = torch.empty((M, C), dtype=_BF, device=dev)
                x_mid = torch.empty((M, C), dtype=_BF, device=dev)
                f = torch.empty((M, Hd), dtype=_BF, device=dev)
                m = torch.empty((M, C), dtype=_BF, device=dev)
                x_out = torch.empty((M, C), dtype=_BF, device=dev)
                lse = torch.empty((B, nh, S), dtype=_F32, device=dev)
            else:
                qkv, att, a = self.buf("qkv", (M, 3 * HP)), self.buf("att", (M, HP)), self.buf("a", (M, C))
                x_mid, f, m = self.buf("x_mid", (M, C)), self.buf("f", (M, Hd)), self.buf("m", (M, C))
                x_out, lse = self.buf("x_%d" % (i & 1), (M, C)), self.buf("lse", (B, nh, S), _F32)
            ops.gemm(x, P[f"b{i}.qkv_w"], qkv, bias=P[f"b{i}.qkv_b"])
            ops.cross_attention_fwd(qkv[:, :HP], qkv[:, HP:2 * HP], qkv[:, 2 * HP:], B, S, S, nh, PADDED_HEAD, scale,
                                    q_shared=False, out=att, lse=lse)
            ops.gemm(att, P[f"b{i}.proj_w"], a, bias=P[f"b{i}.proj_b"])
            n1 = ops.layernorm_fwd(a, P[f"b{i}.n1_w"], P[f"b{i}.n1_b"], d.eps, out=self.buf("n", (M, C)))
            ops.add_rows_bcast(x, n1, out=x_mid)                                               # x + norm1(attn(x))
            ops.gemm(x_mid, P[f"b{i}.fc1_w"], f, bias=P[f"b{i}.fc1_b"])
            h = ops.gelu_fwd(f, self.buf("h", (M, Hd)))
            ops.gemm(h, P[f"b{i}.fc2_w"], m, bias=P[f"b{i}.fc2_b"])
            n2 = ops.layernorm_fwd(m, P[f"b{i}.n2_w"], P[f"b{i}.n2_b"], d.eps, out=self.buf("n", (M, C)))
            ops.add_rows_bcast(x_mid, n2, out=x_out)                                           # x + norm2(mlp(x))
            if keep_stash:
                st["blocks"].append(dict(x=x, qkv=qkv, att=att, a=a, x_mid=x_mid, f=f, m=m, lse=lse))
            x = x_out
        y = ops.layernorm_fwd(x, P["norm_w"], P["norm_b"], d.eps)
        if keep_stash:
            st["x_final"] = x
            self._stash = st
        return ops.clip_drop_cls(y, B, N).view(B, N, C)                                        # prefix token dropped

    __call__ = forward

    # ------------------------------------------------------------------ backward
    def backward(self, d_tokens, accumulate=False):
        """d_tokens [B, N, C] (gradient of the tower's output tokens). Parameter gradients go to `self.g`
        (overwritten unless `accumulate`)."""
        assert self.trainable, "this tower is frozen (trainable=False): it has no backward"
        st = self._stash
        assert st is not None, "backward() needs forward(keep_stash=True)"
        d, P, G, dev = self.dims, self.p, self.g, self.device
        C, Hd, HP, nh = d.embed_dim, d.mlp_hidden, d.hp, d.num_heads
        B = st["B"]
        N, S = d.n_tokens, d.n_tokens + 1
        M = B * S
        acc = bool(accumulate)
        scale = d.head_dim ** -0.5
        # final LayerNorm: the prefix token's output is unused -> zero gradient on those rows
        dy = self.buf("dy", (M, C))
        dy.zero_()
        dy.view(B, S, C)[:, 1:].copy_(d_tokens.to(device=dev, dtype=_BF).reshape(B, N, C))
        dx = ops.layernorm_bwd(dy, st["x_final"], P["norm_w"], d.eps, self.buf("dx_a", (M, C)), G["norm_w"], G["norm_b"],
                               accumulate=acc)
        for i in reversed(range(d.live_blocks)):
            bs = st["blocks"][i]
            # ---- x_out = x_mid + norm2(fc2(gelu(fc1(x_mid)))) ----
            dm = ops.layernorm_bwd(dx, bs["m"], P[f"b{i}.n2_w"], d.eps, self.buf("dm", (M, C)), G[f"b{i}.n2_w"],
                                   G[f"b{i}.n2_b"], accumulate=acc)
            h = ops.gelu_fwd(bs["f"], self.buf("h", (M, Hd)))                                   # recompute
            ops.gemm(dm, h, G[f"b{i}.fc2_w"], a_mn=True, b_mn=True, accumulate=acc)
            ops.colsum(dm, G[f"b{i}.fc2_b"], accumulate=acc)
            dh = ops.gemm(dm, P[f"b{i}.fc2_w"], self.buf("dh", (M, Hd)), b_mn=True)
            df = ops.gelu_bwd(bs["f"], dh, self.buf("df", (M, Hd)))
            ops.gemm(df, bs["x_mid"], G[f"b{i}.fc1_w"], a_mn=True, b_mn=True, accumulate=acc)
            ops.colsum(df, G[f"b{i}.fc1_b"], accumulate=acc)
            dx_mid = ops.gemm(df, P[f"b{i}.fc1_w"], self.buf("dx_b", (M, C)), b_mn=True, residual=dx)
            # ---- x_mid = x + norm1(proj(attn(qkv(x)))) ----
            da = ops.layernorm_bwd(dx_mid, bs["a"], P[f"b{i}.n1_w"], d.eps, self.buf("dm", (M, C)), G[f"b{i}.n1_w"],
                                   G[f"b{i}.n1_b"], accumulate=acc)
            ops.gemm(da, bs["att"], G[f"b{i}.proj_w"], a_mn=True, b_mn=True, accumulate=acc)
            ops.colsum(da, G[f"b{i}.proj_b"], accumulate=acc)
            datt = ops.gemm(da, P[f"b{i}.proj_w"], self.buf("datt", (M, HP)), b_mn=True)
            qkv = bs["qkv"]
            dqkv = self.buf("dqkv", (M, 3 * HP))
            ops.attention_bwd_split(qkv[:, :HP], qkv[:, HP:2 * HP], qkv[:, 2 * HP:], bs["att"], datt, bs["lse"], B, S, S,
                                    nh, PADDED_HEAD, False, scale, dqkv[:, :HP], dqkv[:, HP:2 * HP], dqkv[:, 2 * HP:],
                                    delta_ws=self.buf("delta", (B, nh, S), _F32))
            ops.gemm(dqkv, bs["x"], G[f"b{i}.qkv_w"], a_mn=True, b_mn=True, accumulate=acc)
            if acc:
                kb_old = G[f"b{i}.qkv_b"][HP:2 * HP].clone()
            ops.colsum(dqkv, G[f"b{i}.qkv_b"], accumulate=acc)
            if acc:
                G[f"b{i}.qkv_b"][HP:2 * HP].copy_(kb_old)
            else:
                G[f"b{i}.qkv_b"][HP:2 * HP].zero_()        # k_bias is a constant zero buffer in timm (not trained)
            dx = ops.gemm(dqkv, P[f"b{i}.qkv_w"], self.buf("dx_a", (M, C)), b_mn=True, residual=dx_mid)
            st["blocks"][i] = None
            if self.on_block_grads_ready is not None:
                self.on_block_grads_ready(i)
        # ---- embeddings: x0[b] = cat(cls, patch[b]) + R @ pos ----
        # d pos (incl. the sum over the batch) = tile(R, B)^T @ dx0 ; d cls = the prefix row of the same sum
        ops.gemm(self._R_for_batch(B), dx, G["pos"], a_mn=True, b_mn=True, accumulate=acc)
        dcls = self.buf("dcls", (8, C))
        ops.gemm(self._cls_selector(B), dx, dcls, a_mn=True, b_mn=True)
        if acc:
            ops.add_rows_bcast(G["cls"].view(1, C), dcls[:1], out=G["cls"].view(1, C))
        else:
            G["cls"].copy_(dcls[0])
        dpatch = ops.clip_drop_cls(dx, B, N)                                                   # [B*N, C]
        ops.gemm(dpatch, st["cols"], G["patch_w"], a_mn=True, b_mn=True, accumulate=acc)
        ops.colsum(dpatch, G["patch_b"], accumulate=acc)
        self._stash = None
        if self.on_block_grads_ready is not None:
            self.on_block_grads_ready("embed")

    def _cls_selector(self, B):
        """[B*(1+N), 8] bf16 with a one in column 0 at every image's prefix row: dcls = selector^T @ dx0 (row 0)."""
        key = ("sel", B)
        if key not in self._R_tiled:
            S = self.dims.n_tokens + 1
            sel = torch.zeros(B * S, 8, dtype=_BF, device=self.device)
            sel[::S, 0] = 1.0
            self._R_tiled[key] = sel
        return self._R_tiled[key]
