"""-m gpu: the packed-row (variable-length) decoder of ragged training batches against the padded one.

Kernels: varlen attention forward / backward, RoPE at per-row positions and row-keyed LoRA dropout give the bits the
fixed-length kernels give the same sequences padded. Models: the training forward on packed rows is bit-identical to
the padded one (log-probs, per-token log-probs, spliced labels, DPO loss and metrics); gradients differ only by the
summation order over rows (per bucket: norm within 1e-3 relative, max |diff| <= 1e-2 max |g|)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import llava_dpo_oracle as O
from oracle import omnilmm_oracle as OM

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
LENS = [1, 63, 64, 127, 128, 129, 1135, 2048]


def _packing(lens):
    from rlaifv_b200.model import pack_rows
    T = max(lens)
    labels = torch.full((len(lens), T), -100, dtype=torch.int64)
    for s, n in enumerate(lens):
        labels[s, n - 1] = 5
    return pack_rows(labels.cuda())


def _padded(packed, pk, fill):
    """Rows of `packed` [M, C] placed at their padded rows; the other rows hold `fill` (same shape as the result)."""
    out = fill.clone()
    out[pk.rows.long()] = packed
    return out


@pytest.mark.parametrize("n_kv", [32, 8], ids=["mha32", "gqa32_8"])
def test_varlen_attention_matches_fixed_length_kernels(n_kv):
    from rlaifv_b200 import ops
    nh, hd = 32, 128
    H, KV = nh * hd, n_kv * hd
    pk = _packing(LENS)
    nseq, T, M = len(LENS), max(LENS), pk.M
    assert pk.max_len == T and int(pk.cu[-1]) == M          # the last sequence ends at the buffer end
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(M, H + 2 * KV, device="cuda", generator=g).to(torch.bfloat16)
    qkv_pad = _padded(qkv, pk, torch.randn(nseq * T, H + 2 * KV, device="cuda", generator=g).to(torch.bfloat16))
    scale = hd ** -0.5
    att, lse = torch.empty(M, H, dtype=torch.bfloat16, device="cuda"), torch.empty(nh * M, device="cuda")
    ops.attention_varlen_fwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], pk, nh, hd, scale, att, lse, n_kv_heads=n_kv)
    att_pad, lse_pad = ops.attention_fwd(qkv_pad[:, :H], qkv_pad[:, H:H + KV], qkv_pad[:, H + KV:], nseq, T, nh, hd, True,
                                         scale, n_kv_heads=n_kv)
    rows = pk.rows.long()
    assert torch.equal(att, att_pad[rows])
    cu = pk.cu.tolist()
    for s, n in enumerate(LENS):
        assert torch.equal(lse[nh * cu[s]:nh * cu[s + 1]].view(nh, n), lse_pad[s, :, :n]), s
    # backward: the padded rows past each sequence's end get zero dO, as in the decoder
    d_o = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16)
    d_o_pad = _padded(d_o, pk, torch.zeros(nseq * T, H, dtype=torch.bfloat16, device="cuda"))
    dqkv = torch.empty_like(qkv)
    ops.attention_varlen_bwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], att, d_o, lse, pk, nh, hd, scale,
                             dqkv[:, :H], dqkv[:, H:H + KV], dqkv[:, H + KV:], torch.empty(nh * M, device="cuda"),
                             n_kv_heads=n_kv)
    dqkv_pad = torch.empty_like(qkv_pad)
    ops.attention_bwd_split(qkv_pad[:, :H], qkv_pad[:, H:H + KV], qkv_pad[:, H + KV:], att_pad, d_o_pad, lse_pad, nseq,
                            T, T, nh, hd, True, scale, dqkv_pad[:, :H], dqkv_pad[:, H:H + KV], dqkv_pad[:, H + KV:],
                            n_kv_heads=n_kv)
    torch.cuda.synchronize()
    for name, cols in (("dq", slice(0, H)), ("dk", slice(H, H + KV)), ("dv", slice(H + KV, H + 2 * KV))):
        assert torch.equal(dqkv[:, cols], dqkv_pad[rows, cols]), name
    assert float(dqkv.float().abs().max()) > 0


def test_rope_positions_and_row_keyed_dropout_match_padded_layout():
    from rlaifv_b200 import ops
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    nh, nkv, hd = 32, 8, 128
    pk = _packing([5, 300, 129, 77])
    nseq, T, M = 4, pk.T, pk.M
    d = LlavaDims(hidden_size=nh * hd, num_heads=nh, num_kv_heads=nkv, num_layers=1)
    cos, sin = LlavaDPOPolicy.rope_tables(SimpleNamespace(_rope={}, dims=d, device=torch.device("cuda")), T)
    g = torch.Generator(device="cuda").manual_seed(1)
    W = (nh + 2 * nkv) * hd
    x = torch.randn(M, W, device="cuda", generator=g).to(torch.bfloat16)
    xp = _padded(x, pk, torch.randn(nseq * T, W, device="cuda", generator=g).to(torch.bfloat16))
    rows = pk.rows.long()
    a, b = ops.rope_pos_fwd(x.clone(), cos, sin, pk.pos, nh, hd, n_kv_heads=nkv), ops.rope_fwd(xp.clone(), cos, sin, T,
                                                                                               nh, hd, n_kv_heads=nkv)
    assert torch.equal(a, b[rows])
    a, b = ops.rope_pos_bwd(x.clone(), cos, sin, pk.pos, nh, hd, n_kv_heads=nkv), ops.rope_bwd(xp.clone(), None, cos,
                                                                                               sin, T, nh, hd,
                                                                                               n_kv_heads=nkv)
    assert torch.equal(a, b[rows])
    for width in (4096, 11008):
        x = torch.randn(M, width, device="cuda", generator=g).to(torch.bfloat16)
        xp = _padded(x, pk, torch.randn(nseq * T, width, device="cuda", generator=g).to(torch.bfloat16))
        a, b = ops.dropout_fwd(x, 0.05, 77, rows=pk.rows), ops.dropout_fwd(xp, 0.05, 77)
        assert torch.equal(a, b[rows]) and not torch.equal(a, x)
        gr = torch.randn_like(x)
        a = ops.dropout_bwd_add(x.clone(), gr, 0.05, 78, rows=pk.rows)
        b = ops.dropout_bwd_add(xp.clone(), _padded(gr, pk, torch.zeros_like(xp)), 0.05, 78)
        assert torch.equal(a, b[rows])


# ---------------------------------------------------------------------------------------------------------- models
def _step(pol, ids, labels, images, packed, token_weight=None):
    """Training forward + DPO loss + backward on a zeroed gradient; -> (outputs, out9, {bucket: grad}, packed?)."""
    from rlaifv_b200 import ops
    pol.pack_rows = packed
    for st in (pol.store, pol.lora, getattr(pol, "resampler", None)):
        if st is not None:
            st.zero_grad()
    pol._fwd_count = 0                      # the same LoRA dropout streams on both layouts
    out = pol.forward_logps(ids, labels, images, keep_stash=True)
    took = pol._stash["pack"] is not None
    nseq = ids.shape[0]
    B = nseq // 2
    lp, wsum = out["logp"], None
    if token_weight is not None:
        lp, _, wsum = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], token_weight)
    ref = torch.linspace(-120.0, -80.0, nseq, device="cuda")
    _, _, _, dpw, dpr, out9 = ops.dpo_loss(lp[:B].contiguous(), lp[B:].contiguous(), ref[:B].contiguous(),
                                           ref[B:].contiguous(), 0.1)
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous(), token_weight=token_weight, weight_sum=wsum)
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    grads = {b.name: b.grad.float().clone() for b in pol.trainable_buckets()}
    keep = {k: out[k].clone() for k in ("logp", "avg_logp", "per_token_logps", "labels")}
    return keep, out9.clone(), grads, took


def _compare(pol, ids, labels, images, token_weight=None):
    o_pad, m_pad, g_pad, took_pad = _step(pol, ids, labels, images, False, token_weight)
    o_pk, m_pk, g_pk, took_pk = _step(pol, ids, labels, images, True, token_weight)
    assert took_pk and not took_pad
    for k in o_pad:
        assert torch.equal(o_pk[k], o_pad[k]), k
    assert torch.equal(m_pk, m_pad)
    worst = (0.0, 0.0)
    for name, ref in g_pad.items():
        got = g_pk[name]
        n_ref = float(ref.double().norm())
        dn = abs(float(got.double().norm()) - n_ref) / max(n_ref, 1e-30)
        dm = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
        worst = (max(worst[0], dn), max(worst[1], dm))
        assert dn <= 1e-3 and dm <= 1e-2, (name, dn, dm)
    print(f"gradient gap packed vs padded: norm {worst[0]:.2e}, max|diff|/max|g| {worst[1]:.2e}")
    return o_pk


def _llava(cfg, scale, seed=0):
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = cfg
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, num_kv_heads=c.num_kv_heads,
                     clip_hidden=c.clip_hidden, clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers,
                     clip_heads=c.clip_heads, image_size=c.image_size, patch_size=c.patch_size)
    return LlavaDPOPolicy(dims, "cuda", hf_state=O.make_params(c, seed=seed, scale=scale))


@pytest.mark.parametrize("name", ["tiny_ragged_b2", "cool_ragged_b2", "gqa_ragged_b2"])
def test_tiny_llava_packed_matches_padded_on_ragged_fixture(name):
    fx = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = O.CONFIGS[str(fx["cfg_name"])] if "cfg_name" in fx.files else O.TINY
    pol = _llava(cfg, float(fx["param_scale"]))
    out = _compare(pol, torch.from_numpy(fx["concatenated_input_ids"]), torch.from_numpy(fx["concatenated_labels"]),
                   torch.from_numpy(fx["images"]))
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))


def test_tiny_lora_with_dropout_packed_matches_padded_on_ragged_fixture():
    fx = np.load(os.path.join(GOLDEN, "lora", "lora_ragged_b2.npz"))
    c = O.TINY
    pol = _llava(c, float(fx["param_scale"]))
    pol.enable_lora(r=int(fx["r"]), alpha=float(fx["alpha"]), dropout=0.05).load_hf(
        O.make_lora_params(c, r=int(fx["r"]), seed=int(fx["lora_seed"]), b_std=float(fx["lora_b_std"])))
    _compare(pol, torch.from_numpy(fx["concatenated_input_ids"]), torch.from_numpy(fx["concatenated_labels"]),
             torch.from_numpy(fx["images"]))


@pytest.mark.parametrize("name", ["omni_ragged_b2", "omni_weighted_b2"])
def test_tiny_omnilmm_packed_matches_padded_on_ragged_fixture(name):
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    fx = np.load(os.path.join(GOLDEN, "omnilmm", name + ".npz"))
    d, r, t = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    dims = LlavaDims(frontend="resampler", vocab_size=d.vocab_size, hidden_size=d.hidden_size,
                     intermediate_size=d.intermediate_size, num_layers=d.num_layers, num_heads=d.num_heads,
                     num_kv_heads=d.num_kv_heads, rms_eps=d.rms_eps, num_query=r.num_queries, vision_width=r.kv_dim,
                     im_patch_token=t.im_patch, im_start_token=t.im_start, im_end_token=t.im_end)
    B, seed = int(fx["B"]), int(fx["seed"])
    pol = OmniLMMDPOPolicy(dims, "cuda", hf_state=OM.make_omnilmm_params(d, r, seed))
    batch = OM.synthetic_omni_batch(d, r, t, B, 28, 20, seed=seed + 7, ragged=bool(fx["ragged"]))
    tw = torch.from_numpy(fx["token_weight"]).cuda() if "token_weight" in fx.files else None
    _compare(pol, batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"], tw)


@pytest.mark.parametrize("n_kv,ffn", [(32, 11008), (8, 14336)], ids=["llava7b", "mistral7b_gqa"])
def test_7b_width_two_layers_packed_matches_padded(n_kv, ffn):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    dims = LlavaDims(num_layers=2, num_kv_heads=n_kv, intermediate_size=ffn, clip_layers=3)
    batch = O.synthetic_pair_batch(SimpleNamespace(vocab_size=dims.vocab_size, image_size=dims.image_size), 2, 60, 500,
                                   seed=11, image_pos=5, ragged=True)
    ids, labels, images = batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"]
    pol = LlavaDPOPolicy(dims, "cuda", seed=3)
    out = _compare(pol, ids, labels, images)
    assert out["labels"].shape[1] > 1000
    # one engine step each way from the same weights: the 9 step metrics are the same bits
    batch.update(ref_win_logp=torch.tensor([-900.0, -950.0]), ref_rej_logp=torch.tensor([-905.0, -940.0]), beta=0.1)
    metrics = []
    for packed in (False, True):
        pol = LlavaDPOPolicy(dims, "cuda", seed=3)
        pol.pack_rows = packed
        eng = DPOStepEngine(pol, lr=1e-5, total_steps=10, constant_lr=True)
        metrics.append(eng.train_step(batch).clone())
        del eng, pol
    assert torch.equal(metrics[0], metrics[1])


def test_equal_length_batch_is_not_packed():
    pol = _llava(O.TINY, 0.4)
    batch = O.synthetic_pair_batch(O.TINY, 2, 24, 20, seed=5, image_pos=7, ragged=False)
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"], keep_stash=True)
    assert pol._stash["pack"] is None
