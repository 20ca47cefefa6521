"""-m gpu: the DPO step at LLaVA-1.5-13B widths (hidden 5120, ffn 13824, 40 heads of 128, vocab 32000, CLIP-ViT-L/14-336).

- RMSNorm forward and backward at [9080, 5120] against fp64 per element, with the bounds of test_gpu_rowop_bounds.py
  (the backward caches three 8-element chunks per thread at this width).
- Full fine-tuning forward and backward against the fixtures of the unmodified reference at 13B widths and 2 layers
  (oracle/gen_golden_llava13b.py), with the gates of test_gpu_model_parity.py.
- Packed and padded decoder rows on the ragged fixture, with the gates of test_gpu_packed_rows.py.
- The LoRA step against the merged-weight reference fixture, with the gates of test_gpu_lora.py.
- The shipped entry point with --lora_enable on a 13B-width checkpoint.
"""
import os

import numpy as np
import pytest
import torch

import test_gpu_rowop_bounds as RB
from oracle import llava_dpo_oracle as O
from oracle.gen_golden_llava13b import W13B, grad_index

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "llava13b")
FULL_FT = ["w13b_ragged_b2", "w13b_long_b1"]


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


# ---------------------------------------------------------------------------------------------------------- RMSNorm
@pytest.mark.parametrize("M,H", [(9080, 5120)])
def test_rmsnorm_bounds_at_13b_width(M, H, monkeypatch):
    from rlaifv_b200 import ops
    # the backward keeps ceil(H / 8 / 256) = 3 chunks per thread at H = 5120: its row sums are that deep
    monkeypatch.setattr(RB, "NORM_MAXCH", 3)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator().manual_seed(5120 + M)
    x = RB.norm_rows(M, H, gen, RB.DEV)
    w = (1.0 + 0.3 * torch.randn(H, generator=gen)).to(RB.BF).to(RB.DEV)
    rstd = torch.empty(M, dtype=RB.F32, device=RB.DEV)
    y = ops.rmsnorm_fwd(x, w, 1e-5, rstd=rstd)
    torch.cuda.synchronize()
    (yr, yb), (rr, rb) = RB.rmsnorm_fwd_ref(x, w, 1e-5)
    RB.assert_within("rmsnorm_fwd y [%d,%d]" % (M, H), y, yr, yb)
    RB.assert_within("rmsnorm_fwd rstd [%d,%d]" % (M, H), rstd, rr, rb)
    del yr, yb
    dy = RB.norm_rows(M, H, gen, RB.DEV)
    dres = RB.norm_rows(M, H, gen, RB.DEV)
    grid = RB.rmsnorm_bwd_grid(M, sms)
    for use_dres in (False, True):
        for acc in (False, True):
            dx = torch.full_like(x, float("nan"))
            dw = (torch.randn(H, generator=gen) * 4).to(RB.BF).to(RB.DEV)
            old = dw.clone()
            ops.rmsnorm_bwd(dy, x, w, rstd, dx, dw, dres=dres if use_dres else None, dw_accumulate=acc)
            torch.cuda.synchronize()
            (dxr, dxb), (dwr, dwb) = RB.rmsnorm_bwd_ref(dy, x, w, rstd, dres if use_dres else None, grid,
                                                        old if acc else None)
            RB.assert_within("rmsnorm_bwd dx [%d,%d] dres=%d" % (M, H, use_dres), dx, dxr, dxb)
            RB.assert_within("rmsnorm_bwd dw [%d,%d] acc=%d" % (M, H, acc), dw, dwr, dwb)


def test_rmsnorm_bwd_refuses_rows_wider_than_6144():
    from rlaifv_b200 import lib, ops
    x = torch.zeros(4, 6152, dtype=torch.bfloat16, device="cuda")
    w = torch.ones(6152, dtype=torch.bfloat16, device="cuda")
    rstd = torch.ones(4, dtype=torch.float32, device="cuda")
    with pytest.raises(lib.B200Error, match=r"shape \[4,6152\] unsupported"):
        ops.rmsnorm_bwd(x, x, w, rstd, torch.empty_like(x), torch.empty_like(w))


# ---------------------------------------------------------------------------------------------------------- models
def dims13(c=W13B):
    from rlaifv_b200.model import LlavaDims
    return LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)


_POL = {}


def full_ft_policy(scale):
    """One 13B-width policy for the full fine-tuning tests (1.3 B parameters: build it once)."""
    from rlaifv_b200.model import LlavaDPOPolicy
    if scale not in _POL:
        _POL.clear()
        params = O.make_params(W13B, seed=0, scale=scale)
        _POL[scale] = (LlavaDPOPolicy(dims13(), "cuda", hf_state=params), O.params_checksum(params))
        del params
    return _POL[scale]


def fixture_inputs(fx):
    """The fixture's batch, regenerated from its seed (the images are not stored) and checked against it."""
    b = O.synthetic_pair_batch(W13B, int(fx["B"]), int(fx["prompt_len"]), int(fx["resp_len"]), int(fx["seed"]),
                               image_pos=int(fx["image_pos"]), ragged=bool(int(fx["ragged"])))
    ids, labels = torch.from_numpy(fx["concatenated_input_ids"]), torch.from_numpy(fx["concatenated_labels"])
    assert torch.equal(b["concatenated_input_ids"], ids) and torch.equal(b["concatenated_labels"], labels)
    chk = float(fx["images_checksum"])
    assert abs(float(b["images"].double().abs().sum()) - chk) <= 1e-9 * chk
    return ids, labels, b["images"]


@pytest.mark.parametrize("name", FULL_FT)
def test_13b_width_forward_matches_reference_fixture(name):
    fx = np.load(os.path.join(GOLDEN, name + ".npz"))
    pol, checksum = full_ft_policy(float(fx["param_scale"]))
    assert abs(checksum - float(fx["params_checksum"])) < 1e-6 * float(fx["params_checksum"])
    ids, labels, images = fixture_inputs(fx)
    out = pol.forward_logps(ids, labels, images, keep_stash=False)
    torch.cuda.synchronize()
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))
    logp = out["logp"].cpu()
    ref32 = torch.cat([torch.from_numpy(fx["policy_win_logp"]), torch.from_numpy(fx["policy_rej_logp"])])
    refbf = torch.cat([torch.from_numpy(fx["bf16_policy_win_logp"]), torch.from_numpy(fx["bf16_policy_rej_logp"])])
    e_bf, e_32 = rel(logp, refbf), rel(logp, ref32)
    print(f"summed logp {logp.tolist()}: rel err vs bf16 reference {e_bf:.2e}, vs fp32 {e_32:.2e} "
          f"(reference bf16-vs-fp32 {rel(refbf, ref32):.2e})")
    assert e_bf <= 1e-3 and e_32 <= 1e-3
    mask = torch.from_numpy(fx["spliced_labels"])[:, 1:] != -100
    pt = out["per_token_logps"].cpu()[mask]
    pt32, ptbf = torch.from_numpy(fx["per_token_logps"])[mask], torch.from_numpy(fx["bf16_per_token_logps"])[mask]
    own = rel(ptbf, pt32)
    e_pbf, e_p32 = rel(pt, ptbf), rel(pt, pt32)
    print(f"per-token rel err vs bf16 reference {e_pbf:.2e}, vs fp32 {e_p32:.2e}; reference's own gap {own:.2e}; "
          f"mean per-token logp {float(pt32.mean()):.3f}")
    assert e_pbf <= max(1e-3, 2.5 * own) and e_pbf <= 1e-2
    assert e_p32 <= max(1e-3, 2.5 * own) and e_p32 <= 1e-2
    # CLIP features and projected image rows: per-row sums and seeded samples
    feats = pol.encode_images(images).float().cpu()
    proj = pol._frontend_fwd(images, None).float().cpu()
    torch.cuda.synchronize()
    for got, key in ((feats, "clip_features"), (proj, "projected_rows")):
        idx = torch.from_numpy(fx[key + "_index"])
        s, s32, sbf = got.flatten()[idx], torch.from_numpy(fx[key + "_sample"]), torch.from_numpy(fx["bf16_" + key + "_sample"])
        own = float((sbf - s32).abs().mean() / s32.abs().mean())
        e_bf = float((s - sbf).abs().mean() / sbf.abs().mean())
        e_32 = float((s - s32).abs().mean() / s32.abs().mean())
        rs = got.double().sum(-1).reshape(fx[key + "_rowsum"].shape)
        rs32, rsbf = torch.from_numpy(fx[key + "_rowsum"]), torch.from_numpy(fx["bf16_" + key + "_rowsum"])
        own_rs, e_rs = rel(rsbf, rs32), rel(rs, rsbf)
        print(f"{key}: sample mean-abs rel err vs bf16 reference {e_bf:.2e}, vs fp32 {e_32:.2e}, reference's own "
              f"{own:.2e}; row sums vs bf16 {e_rs:.2e} (own {own_rs:.2e})")
        assert e_bf <= own
        assert e_32 <= 1.25 * max(own, 1e-3)
        assert rel(s, sbf) <= 3e-2
        assert e_rs <= max(2.5 * own_rs, 1e-3)


@pytest.mark.parametrize("name", FULL_FT)
def test_13b_width_dpo_loss_and_grads_match_reference_fixture(name):
    from rlaifv_b200 import ops
    fx = np.load(os.path.join(GOLDEN, name + ".npz"))
    pol, _ = full_ft_policy(float(fx["param_scale"]))
    ids, labels, images = fixture_inputs(fx)
    B = int(fx["B"])
    pol.store.zero_grad()
    out = pol.forward_logps(ids, labels, images, keep_stash=True)
    losses, cr, rj, dpw, dpr, out9 = ops.dpo_loss(out["logp"][:B].contiguous(), out["logp"][B:].contiguous(),
                                                  torch.from_numpy(fx["ref_win_logp"]).cuda(),
                                                  torch.from_numpy(fx["ref_rej_logp"]).cuda(), float(fx["beta"]))
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous())
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    e_bf, e_32, own = rel(losses, fx["bf16_losses"]), rel(losses, fx["losses"]), rel(fx["bf16_losses"], fx["losses"])
    print(f"DPO losses rel err: vs bf16 reference {e_bf:.2e}, vs fp32 {e_32:.2e}; reference bf16-vs-fp32 {own:.2e}")
    # The loss is -logsigmoid(beta * (difference of summed log-probs)). At |logp| ~ 400-1560 a summed log-prob within
    # 5e-5 relative of the reference still moves the loss by up to 0.5 %, and the reference's own bf16 run sits that far
    # from its fp32 run (1.9e-3 and 7.2e-3 on these fixtures): the 1e-3 gate widens to that gap and no further.
    assert e_bf <= max(1e-3, own)
    assert e_32 <= max(2e-3, 2.5 * own)
    assert rel(cr, fx["bf16_chosen_rewards"]) <= 2e-3
    grads = pol.store.hf_grad_views()
    names = [k.split(":", 1)[1] for k in fx.files if k.startswith("gradsample:")]
    # every tensor class of the decoder and projector: embeddings, q/k/v/o, gate/up/down, both norms, final norm, head
    assert len(names) == 2 * 9 + 7
    for name_ in names:
        g = grads[name_].float().flatten().cpu()
        idx = grad_index(g.numel())
        ref = torch.from_numpy(fx["gradsample:" + name_])
        gn = float(fx["gradnorm:" + name_])
        scale = float(ref.abs().max()) + 1e-12
        err = float((g[idx] - ref).abs().max())
        nrm = float(g.double().norm())
        own_s = float(np.abs(fx["bf16_gradsample:" + name_] - fx["gradsample:" + name_]).max()) / scale
        own_n = abs(float(fx["bf16_gradnorm:" + name_]) - gn) / gn
        print(f"{name_}: sample err {err / scale:.2e} (own {own_s:.2e}); norm err {abs(nrm - gn) / gn:.2e} "
              f"(own {own_n:.2e})")
        assert abs(nrm - gn) <= 1e-2 * gn, name_
        assert err <= max(2.5 * own_s, 2e-2) * scale, name_


def test_13b_width_packed_matches_padded_on_ragged_fixture():
    from test_gpu_packed_rows import _compare
    fx = np.load(os.path.join(GOLDEN, "w13b_ragged_b2.npz"))
    pol, _ = full_ft_policy(float(fx["param_scale"]))
    ids, labels, images = fixture_inputs(fx)
    try:
        out = _compare(pol, ids, labels, images)
    finally:
        pol.pack_rows = True
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))


def test_13b_width_lora_matches_merged_weight_reference_fixture():
    from rlaifv_b200 import ops
    from rlaifv_b200.model import LlavaDPOPolicy
    _POL.clear()
    fx = np.load(os.path.join(GOLDEN, "w13b_lora_b1.npz"))
    params = O.make_params(W13B, seed=0, scale=float(fx["param_scale"]))
    lora = O.make_lora_params(W13B, r=int(fx["r"]), seed=int(fx["lora_seed"]), b_std=float(fx["lora_b_std"]))
    assert abs(O.params_checksum(lora) - float(fx["lora_checksum"])) <= 1e-9 * float(fx["lora_checksum"])
    pol = LlavaDPOPolicy(dims13(), "cuda", hf_state=params)
    del params
    pol.enable_lora(r=int(fx["r"]), alpha=float(fx["alpha"])).load_hf(lora)
    ids, labels, images = fixture_inputs(fx)
    out = pol.forward_logps(ids, labels, images, keep_stash=True)
    B = int(fx["B"])
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))
    ref = torch.cat([torch.from_numpy(fx["policy_win_logp"]), torch.from_numpy(fx["policy_rej_logp"])])
    e_sum = rel(out["logp"], ref)
    losses, cr, rj, dpw, dpr, out9 = ops.dpo_loss(out["logp"][:B].contiguous(), out["logp"][B:].contiguous(),
                                                  torch.from_numpy(fx["ref_win_logp"]).cuda(),
                                                  torch.from_numpy(fx["ref_rej_logp"]).cuda(), float(fx["beta"]))
    pol.store.grad.zero_()
    pol.lora.grad.zero_()
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous())
    torch.cuda.synchronize()
    e_loss = rel(losses, fx["losses"])
    print(f"summed logp rel err vs merged-weight reference {e_sum:.2e}; losses {e_loss:.2e}")
    assert e_sum <= 1e-3
    assert e_loss <= 5e-3
    assert rel(cr, fx["chosen_rewards"]) <= 5e-3
    gl = dict(pol.lora.hf_views(grads=True))
    gl.update({k: v for k, v in pol.store.hf_grad_views().items() if "mm_projector" in k})
    worst_n = worst_s = 0.0
    keys = [k for k in fx.files if k.startswith("gradsample:")]
    assert len(keys) == 2 * 7 * 2 + 4
    for key in keys:
        name = key.split(":", 1)[1]
        g = gl[name].float().flatten().cpu()
        idx = grad_index(g.numel())
        refs = torch.from_numpy(fx[key])
        gn = float(fx["gradnorm:" + name])
        en = abs(float(g.double().norm()) - gn) / gn
        es = float((g[idx] - refs).abs().max()) / (float(refs.abs().max()) + 1e-12)
        worst_n, worst_s = max(worst_n, en), max(worst_s, es)
        assert en <= 3e-2, (name, en)
        assert es <= 6e-2, (name, es)
    print(f"adapter + projector gradients: worst norm err {worst_n:.2e}, worst sample err {worst_s:.2e}")


def test_train_llava15_lora_entry_at_13b_width(tmp_path, monkeypatch):
    """`train_llava15.train(... --lora_enable True ...)` for two steps on a 13B-width, 2-layer checkpoint with the toy
    vocabulary: config.json-driven widths, reference log-prob pre-pass, LoRA r = 64, and a peft-layout adapter saved."""
    import io
    import json
    from PIL import Image
    from oracle.toy_tokenizer import ToyTokenizer
    from rlaifv_b200 import data as D
    from rlaifv_b200 import train_llava15 as TL
    _POL.clear()
    c = O.OracleConfig(vocab_size=O.TINY.vocab_size, hidden_size=5120, intermediate_size=13824, num_layers=2,
                       num_heads=40, clip_hidden=128, clip_intermediate=256, clip_layers=3, clip_heads=2,
                       image_size=56, patch_size=14)
    params = O.make_params(c, seed=0, scale=0.09, dtype=torch.bfloat16)
    ckpt, vt = tmp_path / "ckpt", tmp_path / "clip"
    ckpt.mkdir()
    vt.mkdir()
    vp = "model.vision_tower.vision_tower."
    torch.save({k: v for k, v in params.items() if not k.startswith(vp)}, ckpt / "pytorch_model.bin")
    torch.save({k[len(vp):]: v for k, v in params.items() if k.startswith(vp)}, vt / "pytorch_model.bin")
    del params
    (ckpt / "config.json").write_text(json.dumps({
        "vocab_size": c.vocab_size, "hidden_size": c.hidden_size, "intermediate_size": c.intermediate_size,
        "num_hidden_layers": c.num_layers, "num_attention_heads": c.num_heads, "num_key_value_heads": c.num_heads,
        "rms_norm_eps": c.rms_eps}))
    (vt / "config.json").write_text(json.dumps({"vision_config": {
        "hidden_size": c.clip_hidden, "intermediate_size": c.clip_intermediate, "num_hidden_layers": c.clip_layers,
        "num_attention_heads": c.clip_heads, "image_size": c.image_size, "patch_size": c.patch_size}}))
    (vt / "preprocessor_config.json").write_text(json.dumps({
        "size": {"shortest_edge": c.image_size}, "crop_size": {"height": c.image_size, "width": c.image_size},
        "image_mean": [0.48145466, 0.4578275, 0.40821073], "image_std": [0.26862954, 0.26130258, 0.27577711]}))
    monkeypatch.setattr(D, "load_tokenizer", lambda path, max_len: ToyTokenizer())
    g = torch.Generator().manual_seed(2)
    words = "a red bus on the street near two small dogs and one cat under blue sky with trees".split()
    rows = []
    for i in range(4):
        arr = (torch.rand(70 + 10 * i, 90, 3, generator=g) * 255).to(torch.uint8).numpy()
        buf = io.BytesIO()
        Image.fromarray(arr).save(buf, format="PNG")
        rows.append({"image": {"bytes": buf.getvalue()}, "question": "what is shown in picture %d ?" % i,
                     "chosen": " ".join(words[i:i + 6]), "rejected": " ".join(words[::-1][i:i + 4]), "idx": i,
                     "origin_dataset": "synthetic", "origin_split": "train", "image_path": "img%d" % i})
    out_dir = tmp_path / "out"
    tr = TL.train(argv=["--model_name_or_path", str(ckpt), "--vision_tower", str(vt), "--mm_vision_select_layer", "-2",
                        "--data_dir", str(tmp_path / "data"), "--data_source_names", "", "--data_source_weights", "1",
                        "--task", "DPO", "--dpo_beta", "0.1", "--dpo_token_weight", "1.0", "--learning_rate", "2e-4",
                        "--lora_enable", "True", "--lora_r", "64", "--lora_alpha", "16",
                        "--max_steps", "2", "--per_device_train_batch_size", "2", "--logging_steps", "1",
                        "--save_strategy", "no", "--lr_scheduler_type", "constant", "--model_max_length", "2048",
                        "--output_dir", str(out_dir), "--bf16", "True", "--image_aspect_ratio", "pad"], source_rows=rows)
    torch.cuda.synchronize()
    pol = tr.model.policy
    assert pol.dims.hidden_size == 5120 and pol.dims.num_heads == 40 and pol.lora is not None
    losses = [h["loss"] for h in tr.state["log_history"] if "loss" in h]
    assert len(losses) == 2 and abs(losses[0] - 0.693147) < 5e-3 and all(l == l for l in losses)
    cfg = json.load(open(out_dir / "adapter_config.json"))
    assert cfg["r"] == 64 and cfg["lora_alpha"] == 16 and cfg["peft_type"] == "LORA"
    ad = torch.load(out_dir / "adapter_model.bin")
    assert ad["base_model.model.model.layers.1.mlp.down_proj.lora_A.weight"].shape == (64, 13824)
    assert ad["base_model.model.model.layers.0.self_attn.q_proj.lora_B.weight"].shape == (5120, 64)
    assert float(ad["base_model.model.model.layers.0.self_attn.q_proj.lora_B.weight"].float().abs().max()) > 0
    assert set(torch.load(out_dir / "non_lora_trainables.bin")) == {
        "base_model.model.model.mm_projector.%d.%s" % (i, n) for i in (0, 2) for n in ("weight", "bias")}
