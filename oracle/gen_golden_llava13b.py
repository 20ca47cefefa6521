"""ORACLE TOOLING — pins the DPO step at LLaVA-1.5-13B widths against the UNMODIFIED reference.

    PYTHONDONTWRITEBYTECODE=1 python oracle/gen_golden_llava13b.py          (build container only)

W13B is llava-v1.5-13b's config.json (hidden 5120, ffn 13824, 40 heads of 128, vocab 32000, rms_norm_eps 1e-5, RoPE
theta 1e4) cut to 2 decoder layers, with the real CLIP-ViT-L/14-336 tower (24 layers, select layer -2, 576 patches)
and the mlp2x_gelu projector 1024 -> 5120 -> 5120.  Three fixtures go to tests/golden/llava13b/:

  w13b_ragged_b2   B = 2 ragged pairs, full fine-tuning: gen_golden.py's recipe (reference in fp32 and as shipped in
                   bf16, the oracle checked against the fp32 run)
  w13b_long_b1     B = 1, a 150-token response, same recipe
  w13b_lora_b1     LoRA r = 64 / alpha = 16 on q,k,v,o,gate,up,down: gen_golden_lora.py's recipe (the reference run
                   with merged weights W + s B A; adapter gradients by the chain rule)

PARAM_SCALE = 0.09 is the `cool_*` fixtures' 0.4 at hidden 256 carried to hidden 5120 (0.4 * sqrt(256 / 5120) = 0.089):
every projection's output std is sqrt(H) * std * scale, so logits and per-layer activations keep the cool cases'
magnitude, and per-token log-probs sit near -ln(32000) as a real checkpoint's do on random tokens.

A [576, 5120] projected image is 11.8 MB in fp32, so the fixtures keep per-row sums and SAMPLE_N seeded samples of the
CLIP features and projected rows, and 64 samples plus the norm of every gradient tensor.  The images are not stored:
they are regenerated from the case seed by `synthetic_pair_batch` and pinned by `images_checksum`.

Run time on 8 CPU cores (AVX-512 with AMX-BF16), 62 GB RAM: about 5 minutes, peak resident memory 39 GB.
"""
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle.llava_dpo_oracle import OracleConfig  # noqa: E402

W13B = OracleConfig(vocab_size=32000, hidden_size=5120, intermediate_size=13824, num_layers=2, num_heads=40)
PARAM_SCALE = 0.09
SAMPLE_N = 4096
LORA_R, LORA_ALPHA = 64, 16.0          # the shipped recipe (scaling 0.25)
CASES = {
    # name: (B, prompt_len, resp_len, seed, image_pos, ragged)
    "w13b_ragged_b2": (2, 24, 40, 51, 9, True),
    "w13b_long_b1": (1, 30, 150, 52, 20, False),
}
LORA_CASE = ("w13b_lora_b1", (1, 20, 40, 53, 5, False), 7, 0.02)     # (name, case, lora_seed, lora_b_std)


def sample_index(numel, seed):
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:SAMPLE_N].sort().values


def summarize_rows(prefix, t, idx):
    """Per-row sums (fp64) and seeded samples of a [..., rows, width] tensor."""
    t = t.detach().float()
    return {prefix + "_rowsum": t.double().sum(-1).numpy(), prefix + "_sample": t.flatten()[idx].numpy()}


def grad_index(numel):
    """64 evenly spaced flat indices, first and last included (in fp64: an fp32 linspace rounds past the end of the
    163 840 000-element embedding)."""
    return (torch.arange(64, dtype=torch.float64) * ((numel - 1) / 63)).long()


def grad_entries(fx, name, g, prefix=""):
    flat = g.detach().float().flatten()
    idx = grad_index(flat.numel())
    fx[prefix + "gradnorm:" + name] = np.float64(float(flat.double().norm()))
    fx[prefix + "gradsample:" + name] = flat[idx].numpy()


def rel(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


class Tok:
    pad_token_id = 0


class Args:
    dpo_use_average = False
    dpo_token_weighted = False
    task = "DPO"


def collate(R, O, cfg, case, ref_center):
    B, P, Rl, seed, ipos, ragged = case
    from oracle import gen_golden as G
    batch = O.synthetic_pair_batch(cfg, B, P, Rl, seed, image_pos=ipos, ragged=ragged)
    g = torch.Generator().manual_seed(seed + 100)
    ref = {k: (ref_center + 3.0 * torch.randn(B, generator=g)) for k in ("ref_win_logp", "ref_rej_logp")}
    ref["ref_win_avg_logp"] = ref["ref_win_logp"] / Rl
    ref["ref_rej_avg_logp"] = ref["ref_rej_logp"] / Rl
    data = R["DataCollatorForDPODataset"](tokenizer=Tok(), beta=0.1, mod_token_weight=1.0)(
        G.make_instances(batch, ref, B))
    assert torch.equal(data["concatenated_input_ids"], batch["concatenated_input_ids"])
    assert torch.equal(data["concatenated_labels"], batch["concatenated_labels"])
    return batch, ref, data


def case_header(case, params):
    B, P, Rl, seed, ipos, ragged = case
    from oracle import llava_dpo_oracle as O
    return dict(B=np.int64(B), prompt_len=np.int64(P), resp_len=np.int64(Rl), seed=np.int64(seed),
                image_pos=np.int64(ipos), ragged=np.int64(int(ragged)), param_scale=np.float64(PARAM_SCALE),
                params_checksum=np.float64(O.params_checksum(params)), cfg_name=np.array("W13B"),
                sample_n=np.int64(SAMPLE_N))


def full_ft_case(R, O, model, params, name, case, out_dir):
    from oracle import gen_golden as G
    cfg = W13B
    B = case[0]
    batch, ref, data = collate(R, O, cfg, case, -40.0)
    model.zero_grad(set_to_none=True)
    with torch.no_grad():
        _, _, _, _, ref_embeds, ref_labels = model.prepare_inputs_labels_for_multimodal(
            input_ids=data["concatenated_input_ids"].clone(), position_ids=None, attention_mask=None,
            past_key_values=None, labels=data["concatenated_labels"].clone(),
            images=torch.cat([data["images"], data["images"]], 0))
        ref_per_tok, _, _ = R["get_batch_logps"](model.forward(inputs_embeds=ref_embeds, labels=None).logits.float(),
                                                ref_labels, return_all=True)
        ref_feats = model.get_model().get_vision_tower()(data["images"])
        ref_proj = model.get_model().mm_projector(ref_feats)
    pw, pr, rw, rr, beta = R["get_beta_and_logps"](dict(data), model, Args(), is_llava15=True)
    losses, cr, rj = R["dpo_loss"](pw, pr, rw, rr, beta=beta)
    loss = losses.mean()
    loss.backward()
    ref_grads = {k: v.grad.detach().clone() for k, v in model.named_parameters() if v.grad is not None}
    assert all("vision_tower" not in k for k in ref_grads), "CLIP must stay frozen"
    model.zero_grad(set_to_none=True)
    rb = G.reference_bf16_run(R, model, data, Args)
    # --- the oracle against the fp32 reference (gen_golden.py's assertion) ---
    op = {k: v.clone().requires_grad_(k.startswith(O.TRAINABLE_PREFIXES)) for k, v in params.items()}
    oo = O.dpo_step(op, cfg, dict(batch, ref_win_logp=ref["ref_win_logp"], ref_rej_logp=ref["ref_rej_logp"]), beta=0.1)
    oo["loss"].backward()
    assert torch.equal(oo["labels"], ref_labels), "splice labels not bit-exact"
    # the spliced rows are compared like every other fp32 result: at these widths the BLAS blocks the projector GEMM by
    # its row count, and the reference projects the image twice (win and rej copies) where the oracle projects it once
    checks = {"inputs_embeds": rel(oo["inputs_embeds"].detach(), ref_embeds),
              "per_token_logps": rel(oo["per_token_logps"].detach(), ref_per_tok),
              "policy_win_logp": rel(oo["policy_win_logp"].detach(), pw.detach()),
              "policy_rej_logp": rel(oo["policy_rej_logp"].detach(), pr.detach()),
              "losses": rel(oo["losses"].detach(), losses.detach()),
              "chosen_rewards": rel(oo["chosen_rewards"], cr)}
    for k in ref_grads:
        checks["grad:" + k] = rel(op[k].grad, ref_grads[k])
    del op, oo
    worst = max(checks.values())
    print(f"[{name}] oracle vs reference: worst rel err {worst:.3e} over {len(checks)} quantities; "
          f"loss={float(loss):.6f} T={ref_labels.shape[1]}")
    assert worst < 2e-5, {k: v for k, v in checks.items() if v >= 2e-5}
    mask = ref_labels[:, 1:] != O.IGNORE_INDEX
    print(f"    per-token logp mean {float(ref_per_tok[mask].mean()):.3f}; reference bf16 vs fp32: summed logp "
          f"{rel(torch.cat([rb['policy_win_logp'], rb['policy_rej_logp']]), torch.cat([pw, pr]).detach()):.2e}")
    fi = sample_index(ref_feats.numel(), case[3] + 1)
    pi = sample_index(ref_proj.numel(), case[3] + 2)
    fx = case_header(case, params)
    fx.update(images_checksum=np.float64(float(batch["images"].double().abs().sum())),
              concatenated_input_ids=data["concatenated_input_ids"].numpy(),
              concatenated_labels=data["concatenated_labels"].numpy(),
              ref_win_logp=ref["ref_win_logp"].numpy(), ref_rej_logp=ref["ref_rej_logp"].numpy(), beta=np.float64(0.1),
              spliced_labels=ref_labels.numpy(), spliced_embeds_rowsum=ref_embeds.double().sum(-1).numpy(),
              per_token_logps=ref_per_tok.numpy(), policy_win_logp=pw.detach().numpy(),
              policy_rej_logp=pr.detach().numpy(), losses=losses.detach().numpy(), chosen_rewards=cr.numpy(),
              rejected_rewards=rj.numpy(), loss=np.float64(float(loss)),
              clip_features_index=fi.numpy(), projected_rows_index=pi.numpy(),
              bf16_per_token_logps=rb["per_token_logps"].numpy(), bf16_policy_win_logp=rb["policy_win_logp"].numpy(),
              bf16_policy_rej_logp=rb["policy_rej_logp"].numpy(), bf16_losses=rb["losses"].numpy(),
              bf16_chosen_rewards=rb["chosen_rewards"].numpy(), bf16_rejected_rewards=rb["rejected_rewards"].numpy(),
              bf16_loss=np.float64(rb["loss"]))
    fx.update(summarize_rows("clip_features", ref_feats, fi))
    fx.update(summarize_rows("projected_rows", ref_proj, pi))
    fx.update(summarize_rows("bf16_clip_features", rb["clip_features"], fi))
    fx.update(summarize_rows("bf16_projected_rows", rb["projected_rows"], pi))
    for k, gk in ref_grads.items():
        grad_entries(fx, k, gk)
        grad_entries(fx, k, rb["grads"][k], prefix="bf16_")
    np.savez_compressed(os.path.join(out_dir, name + ".npz"), **fx)


def lora_case(R, O, params, out_dir):
    from oracle import gen_golden as G
    from oracle import gen_golden_lora as GL
    cfg = W13B
    name, case, lseed, bstd = LORA_CASE
    B = case[0]
    scaling = LORA_ALPHA / LORA_R
    lora = O.make_lora_params(cfg, r=LORA_R, seed=lseed, b_std=bstd)
    model = G.build_reference_model(R, cfg, GL.merged_params(O, cfg, params, lora, scaling))
    model.train()
    batch, ref, data = collate(R, O, cfg, case, -150.0)
    with torch.no_grad():
        _, _, _, _, emb, new_labels = model.prepare_inputs_labels_for_multimodal(
            input_ids=data["concatenated_input_ids"].clone(), position_ids=None, attention_mask=None,
            past_key_values=None, labels=data["concatenated_labels"].clone(),
            images=torch.cat([data["images"], data["images"]], 0))
        ref_per_tok, _, _ = R["get_batch_logps"](model.forward(inputs_embeds=emb, labels=None).logits.float(),
                                                new_labels, return_all=True)
    model.zero_grad(set_to_none=True)
    pw, pr, rw, rr, beta = R["get_beta_and_logps"](dict(data), model, Args(), is_llava15=True)
    losses, cr, rj = R["dpo_loss"](pw, pr, rw, rr, beta=beta)
    losses.mean().backward()
    gW = {k: v.grad.detach() for k, v in model.named_parameters() if v.grad is not None}
    ref_grads = {}
    for i in range(cfg.num_layers):
        for t in O.LORA_TARGETS:
            n = f"model.layers.{i}.{t}"
            A, Bm, dW = lora[n + ".lora_A.weight"], lora[n + ".lora_B.weight"], gW[n + ".weight"]
            ref_grads[n + ".lora_A.weight"] = scaling * (Bm.t() @ dW)
            ref_grads[n + ".lora_B.weight"] = scaling * (dW @ A.t())
    for k in ("model.mm_projector.0.weight", "model.mm_projector.0.bias", "model.mm_projector.2.weight",
              "model.mm_projector.2.bias"):
        ref_grads[k] = gW[k]
    del model, gW
    op = {k: v.clone().requires_grad_(k.startswith("model.mm_projector.")) for k, v in params.items()}
    op.update({k: v.clone().requires_grad_(True) for k, v in lora.items()})
    oo = O.dpo_step(op, cfg, dict(batch, ref_win_logp=ref["ref_win_logp"], ref_rej_logp=ref["ref_rej_logp"]), beta=0.1)
    oo["loss"].backward()
    assert torch.equal(oo["labels"], new_labels)
    checks = {"per_token_logps": rel(oo["per_token_logps"].detach(), ref_per_tok),
              "policy_win_logp": rel(oo["policy_win_logp"].detach(), pw.detach()),
              "policy_rej_logp": rel(oo["policy_rej_logp"].detach(), pr.detach()),
              "losses": rel(oo["losses"].detach(), losses.detach())}
    for k, v in ref_grads.items():
        checks["grad:" + k] = rel(op[k].grad, v)
    del op, oo
    worst = max(checks.values())
    print(f"[{name}] oracle LoRA branch vs merged-weight reference: worst rel err {worst:.3e} over {len(checks)} "
          f"quantities; loss={float(losses.mean()):.6f}")
    assert worst < 5e-5, {k: v for k, v in checks.items() if v >= 5e-5}
    with torch.no_grad():
        base = O.policy_logps(params, cfg, batch["concatenated_input_ids"], batch["concatenated_labels"],
                              batch["images"])
    assert rel(base["logp"], torch.cat([pw, pr]).detach()) > 1e-3, "the adapters must change the output"
    fx = case_header(case, params)
    fx.update(lora_seed=np.int64(lseed), lora_b_std=np.float64(bstd), r=np.int64(LORA_R), alpha=np.float64(LORA_ALPHA),
              lora_checksum=np.float64(O.params_checksum(lora)),
              images_checksum=np.float64(float(batch["images"].double().abs().sum())),
              concatenated_input_ids=data["concatenated_input_ids"].numpy(),
              concatenated_labels=data["concatenated_labels"].numpy(),
              ref_win_logp=ref["ref_win_logp"].numpy(), ref_rej_logp=ref["ref_rej_logp"].numpy(), beta=np.float64(0.1),
              spliced_labels=new_labels.numpy(), per_token_logps=ref_per_tok.numpy(),
              policy_win_logp=pw.detach().numpy(), policy_rej_logp=pr.detach().numpy(),
              losses=losses.detach().numpy(), chosen_rewards=cr.numpy(), rejected_rewards=rj.numpy(),
              loss=np.float64(float(losses.mean())))
    for k, v in ref_grads.items():
        grad_entries(fx, k, v)
    np.savez_compressed(os.path.join(out_dir, name + ".npz"), **fx)


def main():
    import time
    from oracle import gen_golden as G
    from oracle import llava_dpo_oracle as O
    t0 = time.time()
    torch.set_grad_enabled(True)
    R = G.import_reference()
    out_dir = os.path.join(REPO, "tests", "golden", "llava13b")
    os.makedirs(out_dir, exist_ok=True)
    params = O.make_params(W13B, seed=0, scale=PARAM_SCALE)
    model = G.build_reference_model(R, W13B, params)
    model.train()
    for name, case in CASES.items():
        full_ft_case(R, O, model, params, name, case, out_dir)
        print(f"    {time.time() - t0:.0f} s")
    del model
    lora_case(R, O, params, out_dir)
    print(f"13B-width fixtures written to {out_dir} in {time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()
