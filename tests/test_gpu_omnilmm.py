"""-m gpu: OmniLMM-12B DPO policy downstream of the vision tower (BASELINE config d, SURVEY.md §8 a13) through the
C ABI — resampler, in-place <im_patch> splice (index map bit-exact), Mistral GQA decoder, log-prob gather, DPO loss,
full backward — against the oracle and the fixtures of the unmodified reference OmniLMMForCausalLM."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import omnilmm_oracle as OM

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "omnilmm", "*.npz")))


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def tiny_dims():
    from rlaifv_b200.model import LlavaDims
    d, r, t = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    return LlavaDims(frontend="resampler", vocab_size=d.vocab_size, hidden_size=d.hidden_size,
                     intermediate_size=d.intermediate_size, num_layers=d.num_layers, num_heads=d.num_heads,
                     num_kv_heads=d.num_kv_heads, rms_eps=d.rms_eps, num_query=r.num_queries, vision_width=r.kv_dim,
                     im_patch_token=t.im_patch, im_start_token=t.im_start, im_end_token=t.im_end)


def test_inplace_splice_map_bit_exact_and_errors():
    from rlaifv_b200 import ops
    tok, Q = OM.TINY_OMNI_TOK, 16
    b = OM.synthetic_omni_batch(OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, tok, 3, 30, 12, seed=5)
    ids = b["concatenated_input_ids"].clone()
    ids[1, :] = torch.randint(3, 400, (ids.shape[1],))                          # a text-only row consumes no image
    slots = torch.tensor([2, 0, 1, 2, 0], dtype=torch.int32)                     # arbitrary image-of-slot table
    want = OM.inplace_splice_map(ids, tok, Q, image_of_slot=slots)
    src, status = ops.splice_map_inplace(ids.cuda(), slots.cuda(), Q, tok.im_patch, tok.im_start, tok.im_end)
    assert int(status.item()) == 0 and torch.equal(src.cpu().long(), want)
    bad = ids.clone()
    bad[0, 4 + Q + 1] = 7                                                        # <im_end> missing -> count mismatch
    _, status = ops.splice_map_inplace(bad.cuda(), slots.cuda(), Q, tok.im_patch, tok.im_start, tok.im_end)
    assert int(status.item()) & 1
    bad = ids.clone()
    bad[0, 4 + Q + 1], bad[0, 4 + Q + 3] = 7, tok.im_end                        # <im_end> displaced
    _, status = ops.splice_map_inplace(bad.cuda(), slots.cuda(), Q, tok.im_patch, tok.im_start, tok.im_end)
    assert int(status.item()) & 2


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_omnilmm_policy_matches_oracle_and_reference_fixture(path):
    from rlaifv_b200 import ops
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    fx = np.load(path)
    dec, res, tok = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    B, seed = int(fx["B"]), int(fx["seed"])
    params = OM.make_omnilmm_params(dec, res, seed)
    pol = OmniLMMDPOPolicy(tiny_dims(), "cuda", hf_state=params)
    batch = OM.synthetic_omni_batch(dec, res, tok, B, 28, 20, seed=seed + 7, ragged=bool(fx["ragged"]))
    ids, labels, vt = batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"]
    out = pol.forward_logps(ids, labels, vt, keep_stash=True)
    # integer work: bit exact
    slots = torch.arange(2 * B) % B
    assert torch.equal(pol._stash["src"].cpu().long(), OM.inplace_splice_map(ids, tok, res.num_queries, slots))
    assert torch.equal(out["labels"].cpu(), labels) and out["T"] == ids.shape[1]
    # bf16-op-order oracle on the same bf16-rounded parameters / inputs, and the fp32 reference fixture
    pb = {k: v.to(torch.bfloat16) for k, v in params.items()}
    ob = OM.omnilmm_policy_logps(pb, dec, res, tok, ids, labels, vt.to(torch.bfloat16))
    weighted = "token_weight" in fx.files                  # --dpo_token_weighted fixture (trainers.py:246-261)
    tw = wsum = None
    if weighted:
        tw = torch.from_numpy(fx["token_weight"]).cuda()
        lw, aw, wsum = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], tw)
        ob["logp"] = OM.compute_weighted_logp(ob["per_token_logps"].float(), labels, tw.cpu())
        logp_dev = lw
        wm = tw.cpu() * (labels[:, 1:] != -100)
        assert torch.allclose(wsum.cpu(), wm.sum(-1)) and torch.allclose(aw.cpu(), lw.cpu() / wm.sum(-1), rtol=1e-6)
    else:
        logp_dev = out["logp"]
    logp = logp_dev.cpu()
    ref_fp32 = torch.from_numpy(fx["logp"])
    inherent = rel(ob["logp"], ref_fp32)
    e_ref, e_orc = rel(logp, ref_fp32), rel(logp, ob["logp"])
    print(f"summed logp rel err: cuda-vs-fp32ref {e_ref:.2e}, cuda-vs-bf16oracle {e_orc:.2e}, inherent {inherent:.2e}")
    assert e_orc <= 1e-3 and e_ref <= 1e-3
    mask = labels[:, 1:] != -100
    pt, ref_pt = out["per_token_logps"].cpu(), torch.from_numpy(fx["per_token_logps"])
    inh_pt = rel(ob["per_token_logps"].float()[mask], ref_pt[mask])
    e_pt = rel(pt[mask], ref_pt[mask])
    print(f"per-token rel err: cuda-vs-fp32ref {e_pt:.2e}, inherent {inh_pt:.2e}")
    assert e_pt <= max(1e-3, 2.5 * inh_pt) and e_pt <= 1e-2
    # DPO loss + backward
    rw, rr = torch.from_numpy(fx["ref_win_logp"]).cuda(), torch.from_numpy(fx["ref_rej_logp"]).cuda()
    losses, cr, rj, dpw, dpr, out9 = ops.dpo_loss(logp_dev[:B].contiguous(), logp_dev[B:].contiguous(), rw, rr, 0.1)
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous(), token_weight=tw, weight_sum=wsum)
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    assert rel(losses, fx["losses"]) <= 2e-2 and rel(out9[0], fx["loss"]) <= 2e-2
    grads = dict(pol.store.hf_grad_views())
    grads.update({"model.resampler." + k: v for k, v in pol.resampler.g.items()})
    for key in fx.files:
        if not key.startswith("gradnorm:"):
            continue
        name = key.split(":", 1)[1]
        g = grads[name].float().flatten().cpu()
        ref = torch.from_numpy(fx["gradsample:" + name])
        got = g[torch.linspace(0, g.numel() - 1, min(64, g.numel())).long()]
        gn, nrm = float(fx[key]), float(g.double().norm())
        err, scale = float((got - ref).abs().max()), float(ref.abs().max()) + 1e-12
        print(f"{name}: sample max err {err:.3e} (ref max {scale:.3e}); norm {nrm:.4e} vs ref {gn:.4e}")
        assert abs(nrm - gn) <= 3e-2 * gn, name
        assert err <= 6e-2 * scale, name
    dv = pol.vision_token_grad.float()
    assert abs(float(dv.norm()) - float(fx["dvision_norm"])) <= 3e-2 * float(fx["dvision_norm"])


def test_omnilmm_engine_step_trains_decoder_and_resampler():
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    dec, res, tok = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    pol = OmniLMMDPOPolicy(tiny_dims(), "cuda", hf_state=OM.make_omnilmm_params(dec, res, 3))
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, micro_pairs=1)
    assert [b.name for b in eng.opt.buckets][-1] == "resampler"
    batch = OM.synthetic_omni_batch(dec, res, tok, 2, 28, 20, seed=9)
    ref = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"],
                            keep_stash=False)["logp"].float().cpu()
    batch.update(images=batch["vision_tokens"], ref_win_logp=ref[:2], ref_rej_logp=ref[2:], beta=0.1)
    w0, r0 = pol.store.flat.clone(), pol.resampler.flat.clone()
    m = eng.train_step(batch)
    torch.cuda.synchronize()
    loss1 = float(m[0])                                     # (the engine reuses its metrics tensor)
    assert abs(loss1 - 0.6931472) < 1e-4                    # policy == reference -> loss ln 2
    assert not torch.equal(pol.store.flat, w0) and not torch.equal(pol.resampler.flat, r0)
    m2 = eng.train_step(batch)
    torch.cuda.synchronize()
    assert float(m2[0]) < loss1                             # one AdamW step on the same batch lowers the loss


def test_weighted_logp_reduce_and_backward_match_torch():
    """rlaifv_logp_weighted_reduce / rlaifv_logp_bwd with token weights vs fp32 torch (sum and average mode)."""
    from rlaifv_b200 import ops
    g = torch.Generator().manual_seed(2)
    nseq, T, V = 3, 37, 320
    logits = (torch.randn(nseq * T, V, generator=g) * 2).to(torch.bfloat16).cuda()
    labels = torch.randint(0, V, (nseq, T), generator=g)
    labels[:, :9] = -100
    labels[1, 30:] = -100
    tw = torch.where(torch.rand(nseq, T - 1, generator=g) < 0.4, 3.0, 1.0)
    d = torch.tensor([0.7, -1.3, 0.2])
    for use_avg in (False, True):
        lf = logits.float().cpu().view(nseq, T, V).clone().requires_grad_(True)
        pt = torch.gather(torch.log_softmax(lf[:, :-1], -1), 2, labels[:, 1:].clamp_min(0).unsqueeze(-1)).squeeze(-1)
        wm = tw * (labels[:, 1:] != -100)
        ref = (pt * wm).sum(-1) / (wm.sum(-1) if use_avg else 1.0)
        (ref * d).sum().backward()
        lg = logits.clone()
        per_tok, lse, _, _, _ = ops.logp_fwd(lg, labels.cuda(), nseq, T)
        lw, aw, ws = ops.logp_weighted_reduce(per_tok, labels.cuda(), tw.cuda())
        got = (aw if use_avg else lw).cpu()
        assert rel(got, ref.detach()) < 2e-3
        ops.logp_bwd(lg, labels.cuda(), lse, d.cuda(), nseq, T, token_weight=tw.cuda(), norm=ws if use_avg else None)
        torch.cuda.synchronize()
        want = lf.grad.view(nseq * T, V)
        assert float((lg.float().cpu() - want).norm() / want.norm()) < 8e-3
        assert float(lg.float().cpu().view(nseq, T, V)[:, -1].abs().max()) == 0.0      # last position: no target


def test_engine_token_weighted_step_and_llava_refusal():
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    dec, res, tok = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    pol = OmniLMMDPOPolicy(tiny_dims(), "cuda", hf_state=OM.make_omnilmm_params(dec, res, 3))
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, dpo_token_weighted=True)
    batch = OM.synthetic_omni_batch(dec, res, tok, 2, 28, 20, seed=9)
    ids, labels = batch["concatenated_input_ids"], batch["concatenated_labels"]
    g = torch.Generator().manual_seed(1)
    tw = torch.where(torch.rand(4, ids.shape[1] - 1, generator=g) < 0.3, 3.0, 1.0)
    ref_pt = pol.forward_logps(ids, labels, batch["vision_tokens"], keep_stash=False)["per_token_logps"].float().cpu()
    batch.update(images=batch["vision_tokens"], beta=0.1, concatenated_token_weight=tw, win_token_weight=tw[:2],
                 rej_token_weight=tw[2:], win_labels=labels[:2], rej_labels=labels[2:],
                 ref_win_per_token_logp=ref_pt[:2], ref_rej_per_token_logp=ref_pt[2:])
    m = eng.train_step(batch)
    torch.cuda.synchronize()
    loss1 = float(m[0])
    assert abs(loss1 - 0.6931472) < 1e-4                    # weighted policy == weighted reference -> ln 2
    want_chosen = OM.compute_weighted_logp(ref_pt[:2], labels[:2], tw[:2]).mean()
    assert abs(float(m[6]) - float(want_chosen)) < 1e-2 * abs(float(want_chosen))     # logps_train/chosen is weighted
    assert float(eng.train_step(batch)[0]) < loss1
    c = __import__("oracle.llava_dpo_oracle", fromlist=["TINY"]).TINY
    llava = LlavaDPOPolicy(LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size,
                                     intermediate_size=c.intermediate_size, num_layers=c.num_layers,
                                     num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers,
                                     clip_heads=c.clip_heads, image_size=c.image_size, patch_size=c.patch_size), "cuda")
    # LLaVA-1.5: the drop-in seam keeps the reference's refusal (trainers.py:246-248); the ENGINE accepts it as an
    # extension but only with the collator's un-truncated (spliced-position) reference per-token log-probs
    from types import SimpleNamespace
    from rlaifv_b200 import trainers as TR
    with pytest.raises(NotImplementedError):
        TR.get_beta_and_logps({}, SimpleNamespace(policy=llava), SimpleNamespace(dpo_token_weighted=True, dpo_use_average=False,
                                                                                 task="DPO"), is_llava15=True)
    eng_l = DPOStepEngine(llava, dpo_token_weighted=True)
    with pytest.raises(KeyError):
        eng_l.train_step({"concatenated_input_ids": torch.zeros(2, 8, dtype=torch.long),
                          "concatenated_labels": torch.zeros(2, 8, dtype=torch.long),
                          "images": torch.zeros(1, 3, c.image_size, c.image_size), "beta": 0.1})


@pytest.mark.parametrize("case", ["omni_ragged_b2", "omni_weighted_b2"])
def test_generic_get_beta_and_logps_branch_matches_reference_fixture(case):
    """trainers.get_beta_and_logps(is_llava15=False) -> forward_DPO (-> compute_weighted_logp) -> dpo_loss -> autograd
    backward through the hand-written kernels, against the reference fixture (muffin/train/trainers.py:233-275)."""
    from types import SimpleNamespace
    from rlaifv_b200 import trainers
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    fx = np.load([p for p in GOLDEN if case in p][0])
    dec, res, tok = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    B, seed = int(fx["B"]), int(fx["seed"])
    pol = OmniLMMDPOPolicy(tiny_dims(), "cuda", hf_state=OM.make_omnilmm_params(dec, res, seed))
    batch = OM.synthetic_omni_batch(dec, res, tok, B, 28, 20, seed=seed + 7, ragged=True)
    ids, labels = batch["concatenated_input_ids"], batch["concatenated_labels"]
    L = ids.shape[1]
    weighted = "token_weight" in fx.files
    tw = torch.from_numpy(fx["token_weight"]) if weighted else torch.ones(2 * B, L - 1)
    rw, rr = torch.from_numpy(fx["ref_win_logp"]), torch.from_numpy(fx["ref_rej_logp"])
    # per-token reference log-probs whose weighted sums are the fixture's reference log-probs
    ref_pt = torch.zeros(2 * B, L - 1)
    first = (labels[:, 1:] != -100).float().argmax(-1)
    for b in range(2 * B):
        ref_pt[b, first[b]] = (rw[b] if b < B else rr[b - B]) / tw[b, first[b]]
    dd = {"win_input_ids": ids[:B], "rej_input_ids": ids[B:], "win_labels": labels[:B], "rej_labels": labels[B:],
          "ref_win_per_token_logp": ref_pt[:B], "ref_rej_per_token_logp": ref_pt[B:], "win_token_weight": tw[:B],
          "rej_token_weight": tw[B:], "concatenated_token_weight": tw, "ref_win_avg_logp": rw / 10,
          "ref_rej_avg_logp": rr / 10, "ref_win_logp": rw, "ref_rej_logp": rr, "beta": 0.1,
          "images": batch["vision_tokens"], "concatenated_input_ids": ids, "concatenated_labels": labels,
          "concatenated_attention_mask": torch.ones_like(ids), "win_attention_mask": None, "rej_attention_mask": None}
    args = SimpleNamespace(dpo_use_average=False, dpo_token_weighted=weighted, task="DPO")
    pol.resampler.zero_grad()
    pw, pr, rw_d, rr_d, beta = trainers.get_beta_and_logps(dd, pol, args, is_llava15=False)
    assert not dd and beta == 0.1
    assert rel(torch.cat([pw, pr]).detach(), fx["logp"]) <= 1e-3
    assert torch.allclose(rw_d.cpu(), rw, rtol=1e-5) and torch.allclose(rr_d.cpu(), rr, rtol=1e-5)
    losses, cr, rj = trainers.dpo_loss(pw, pr, rw_d, rr_d, beta)
    assert rel(losses.detach(), fx["losses"]) <= 2e-2
    losses.mean().backward()
    torch.cuda.synchronize()
    grads = dict(pol.store.hf_grad_views())
    grads.update({"model.resampler." + k: v for k, v in pol.resampler.g.items()})
    for name in ("lm_head.weight", "model.layers.0.self_attn.q_proj.weight", "model.layers.1.mlp.down_proj.weight",
                 "model.resampler.proj", "model.resampler.attn.in_proj_weight", "model.embed_tokens.weight"):
        gn = float(fx["gradnorm:" + name])
        assert abs(float(grads[name].float().norm()) - gn) <= 3e-2 * gn, name
