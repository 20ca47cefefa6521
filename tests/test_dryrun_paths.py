"""CPU test: the Python orchestration (forward + backward launch sequences, full fine-tuning and LoRA)
runs end to end against a recording stand-in for the C ABI — catches host-side breakage (shapes, views,
missing methods, argument counts vs the ctypes table) without a GPU. No arithmetic is checked here."""
import ctypes

import pytest
import torch

from oracle import llava_dpo_oracle as O

# argument positions of rlaifv_logp_fwd / rlaifv_logp_bwd (include/rlaifv_b200.h)
ROW_POS, TOKEN_WEIGHT = 3, 7


def _nonnull(p):
    return p.value is not None      # ops passes None as c_void_p(0), whose value is None


@pytest.mark.parametrize("use_lora,cfg_name", [(False, "TINY"), (True, "TINY"), (False, "TINY_GQA")])
def test_launch_sequence_and_head_arguments_dry_run(monkeypatch, use_lora, cfg_name):
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = O.CONFIGS[cfg_name]
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, num_kv_heads=c.num_kv_heads,
                     clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    calls, argv = [], {}

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name       # argument count matches the ctypes table
        calls.append(name)
        argv.setdefault(name, []).append(args)

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    if cfg_name == "TINY_GQA":
        assert pol.store.p["l0.qkv"].shape == (512 + 2 * 256, 512)
        with pytest.raises(NotImplementedError):
            pol.enable_lora()
    if use_lora:
        pol.enable_lora(r=8, alpha=2.0)
    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    monkeypatch.setattr(pol, "splice", lambda ids, labels, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), torch.full((4, T), -100),
        torch.zeros(4, T, dtype=torch.int32), T))
    out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    assert out["logp"].shape == (4,) and out["per_token_logps"].shape == (4, T - 1)
    n_fwd = len(calls)
    pol.backward_logps(torch.zeros(4))
    pol.finalize_embed_grad()
    assert len(calls) > 2 * n_fwd * 0.8
    per_layer_gemm = 4
    # the down-projection dgrad carries the SwiGLU backward in its epilogue (no separate swiglu_bwd pass)
    assert calls.count("rlaifv_gemm_bf16_swiglu_bwd") == dims.num_layers and calls.count("rlaifv_swiglu_bwd") == 0
    if use_lora:
        assert calls.count("rlaifv_gemm_bf16_dual") == (2 * per_layer_gemm - 1) * dims.num_layers   # fwd + dgrad
        assert "rlaifv_f32_to_bf16" in calls                # projected-image-row gradients still flow
    else:
        assert calls.count("rlaifv_gemm_bf16_dual") == 0
    gqa = dims.kv_heads != dims.num_heads
    assert calls.count("rlaifv_attention_fwd") + calls.count("rlaifv_attention_fwd_gqa") == \
        dims.num_layers + dims.clip_layers_used
    assert calls.count("rlaifv_attention_fwd_gqa") == (dims.num_layers if gqa else 0)
    # decoder backward: the split dK/dV + dQ kernels (one C-ABI entry for MHA and GQA)
    assert calls.count("rlaifv_attention_bwd_split") == dims.num_layers
    # compact head: the log-prob forward and backward run on the rows supervised_rows picked
    assert calls.count("rlaifv_supervised_rows") == 1 and calls.count("rlaifv_rows_scatter") == 1
    (rows,), (fwd,), (bwd,) = argv["rlaifv_supervised_rows"], argv["rlaifv_logp_fwd"], argv["rlaifv_logp_bwd"]
    assert _nonnull(fwd[ROW_POS]) and fwd[ROW_POS].value == bwd[ROW_POS].value == rows[4].value
    assert not _nonnull(bwd[TOKEN_WEIGHT])
    names = {b.name for b in pol.trainable_buckets()}
    assert ("projector" in names) and (("lora0" in names) == use_lora) and (("embed" in names) != use_lora)


def test_resampler_launch_sequence_dry_run(monkeypatch):
    """Perceiver resampler (config d piece): forward + backward orchestration against the recording C ABI."""
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.resampler import Resampler
    from oracle import resampler_oracle as R
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append(name)

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    c = R.TINY_R
    m = Resampler(c.grid_size, c.embed_dim, c.num_heads, c.kv_dim, device="cpu", state=R.make_resampler_params(c, 1))
    assert set(m.state_dict()) == set(R.PARAM_SHAPES(c)) | {"pos_embed"}
    x = torch.zeros(3, c.kv_tokens, c.kv_dim, dtype=torch.bfloat16)
    y = m(x)
    assert y.shape == (3, c.num_queries, c.embed_dim)
    assert calls.count("rlaifv_cross_attention_fwd") == 1 and calls.count("rlaifv_layernorm_fwd") == 3
    dx = m.backward(torch.zeros_like(y))
    assert dx.shape == x.shape
    assert calls.count("rlaifv_cross_attention_bwd") == 1 and calls.count("rlaifv_layernorm_bwd") == 3
    # bicubic position table for the 12x12 vision grid was prepared from the 4x4 query grid
    assert m._pos_for(144).shape == (144, c.embed_dim)
    assert torch.allclose(m.pos_embed_f32, R.sincos_2d(c.embed_dim, c.grid_size), atol=1e-6)


def test_omnilmm_policy_launch_sequence_and_head_arguments_dry_run(monkeypatch):
    """OmniLMM policy (resampler front-end + in-place splice + GQA decoder) against the recording C ABI; also runs the
    bf16 oracle path once so the GPU parity test's CPU half is known to work."""
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy, omnilmm_dims
    from oracle import omnilmm_oracle as OM
    calls, argv = [], {}

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append(name)
        argv.setdefault(name, []).append(args)

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    d, r, t = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    dims = LlavaDims(frontend="resampler", vocab_size=d.vocab_size, hidden_size=d.hidden_size,
                     intermediate_size=d.intermediate_size, num_layers=d.num_layers, num_heads=d.num_heads,
                     num_kv_heads=d.num_kv_heads, num_query=r.num_queries, vision_width=r.kv_dim,
                     im_patch_token=t.im_patch, im_start_token=t.im_start, im_end_token=t.im_end)
    params = OM.make_omnilmm_params(d, r, 1)
    pol = OmniLMMDPOPolicy(dims, "cpu", hf_state=params)
    assert "projector" not in {b.name for b in pol.store.buckets} and pol.clip is None
    names = [b.name for b in pol.trainable_buckets()]
    assert names[-1] == "resampler" and "embed" in names and pol.tail_bucket_names() == ["embed", "resampler"]
    assert all(b.size % 64 == 0 for b in pol.trainable_buckets())
    assert set(pol.hf_views()) == set(params)
    batch = OM.synthetic_omni_batch(d, r, t, 2, 28, 20, seed=2)
    out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"])
    L = batch["concatenated_input_ids"].shape[1]
    assert out["T"] == L and out["per_token_logps"].shape == (4, L - 1)
    pol.backward_logps(torch.zeros(4))
    pol.finalize_embed_grad()
    assert calls.count("rlaifv_splice_map_inplace") == 1 and calls.count("rlaifv_cross_attention_bwd") == 1
    assert calls.count("rlaifv_attention_fwd_gqa") == d.num_layers and "rlaifv_clip_im2col" not in calls
    assert pol.vision_token_grad.shape == batch["vision_tokens"].shape
    # token-weighted variant (--dpo_token_weighted): weighted reduce + the backward with token weights
    out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"])
    tw = torch.ones(4, L - 1)
    lw, aw, ws = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], tw)
    pol.backward_logps(torch.zeros(4), use_average=True, token_weight=tw, weight_sum=ws)
    # compact head: the weighted and the plain backward share one entry point (token_weight / norm arguments)
    fwds, bwds = argv["rlaifv_logp_fwd"], argv["rlaifv_logp_bwd"]
    assert len(fwds) == len(bwds) == 2 and all(_nonnull(a[ROW_POS]) for a in fwds + bwds)
    assert not _nonnull(bwds[0][TOKEN_WEIGHT]) and _nonnull(bwds[1][TOKEN_WEIGHT])
    # generic get_beta_and_logps branch (forward_DPO) incl. --dpo_token_weighted, autograd bridge end to end
    from types import SimpleNamespace
    from rlaifv_b200 import trainers
    ids, labels = batch["concatenated_input_ids"], batch["concatenated_labels"]
    for weighted in (False, True):
        dd = {"win_input_ids": ids[:2], "rej_input_ids": ids[2:], "win_labels": labels[:2], "rej_labels": labels[2:],
              "ref_win_per_token_logp": torch.zeros(2, L - 1), "ref_rej_per_token_logp": torch.zeros(2, L - 1),
              "win_token_weight": tw[:2], "rej_token_weight": tw[2:], "concatenated_token_weight": tw,
              "ref_win_avg_logp": torch.zeros(2), "ref_rej_avg_logp": torch.zeros(2), "ref_win_logp": torch.zeros(2),
              "ref_rej_logp": torch.zeros(2), "beta": 0.1, "images": batch["vision_tokens"],
              "concatenated_input_ids": ids, "concatenated_labels": labels, "concatenated_attention_mask": None}
        args = SimpleNamespace(dpo_use_average=False, dpo_token_weighted=weighted, task="DPO")
        n_w = len(argv["rlaifv_logp_bwd"])
        pw, pr, rw, rr, beta = trainers.get_beta_and_logps(dd, pol, args, is_llava15=False)
        assert pw.shape == (2,) and pr.shape == (2,) and pw.requires_grad and not dd
        losses, cr, rj = trainers.dpo_loss(pw, pr, rw, rr, beta)
        losses.mean().backward()
        assert len(argv["rlaifv_logp_bwd"]) == n_w + 1
        bwd = argv["rlaifv_logp_bwd"][-1]
        assert _nonnull(bwd[ROW_POS]) and _nonnull(bwd[TOKEN_WEIGHT]) == weighted
    with pytest.raises(ValueError):
        trainers.get_beta_and_logps({**{k: None for k in ("win_input_ids", "rej_input_ids", "ref_win_avg_logp",
                                                          "ref_rej_avg_logp", "ref_win_logp", "ref_rej_logp", "beta",
                                                          "images", "concatenated_input_ids", "concatenated_labels")}},
                                    pol, SimpleNamespace(dpo_use_average=False, dpo_token_weighted=False, task="DPO"),
                                    is_llava15=True)
    full = omnilmm_dims()
    assert full.kv_size == 1024 and full.intermediate_size == 14336 and full.vocab_size % 8 == 0
    # bf16 evaluation order of the oracle (used as the second comparison point on the GPU)
    pb = {k: v.to(torch.bfloat16) for k, v in params.items()}
    ob = OM.omnilmm_policy_logps(pb, d, r, t, batch["concatenated_input_ids"], batch["concatenated_labels"],
                                 batch["vision_tokens"].to(torch.bfloat16))
    assert ob["logp"].shape == (4,) and bool(torch.isfinite(ob["logp"].float()).all())
