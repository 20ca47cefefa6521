"""-m gpu: OmniLMM-12B with a frozen EVA tower (`tune_clip=False`) and the offloaded optimizer on the OmniLMM policy.

* Frozen vs trained tower at the same weights and batch: log-probs, loss, resampler and decoder gradients bit-identical;
  three engine steps leave the tower's weights bit-unchanged; the device footprint drops by at least the tower's
  gradient buffer.
* The frozen-tower policy meets the gates of the reference fixtures tests/golden/omnilmm/*.
* Offloaded vs on-device AdamW at tiny OmniLMM dimensions with the tower, both tower modes, mixed and all-streamed
  splits: bit-identical; a streamed tower block's update is waited on before the next forward reads it.
* Checkpoint save / resume with the frozen tower under offload; a resume across tower modes is refused.
* `train_omnilmm --tune_clip False --deepspeed script/zero2_offload.json` end to end, with a resume."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import eva_oracle as E
from oracle import omnilmm_oracle as OM
from oracle import resampler_oracle as R

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "omnilmm", "*.npz")))


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def eva_dims(t=E.TINY_EVA):
    from rlaifv_b200.eva_tower import EvaDims
    return EvaDims(embed_dim=t.embed_dim, depth=t.depth, num_heads=t.num_heads, mlp_hidden=t.mlp_hidden,
                   patch_size=t.patch_size, pretrain_img=t.pretrain_img, img_size=t.img_size, eps=t.eps)


def setup(tune_clip, B=2, seed=3):
    """Tiny whole OmniLMM (tower -> resampler -> GQA decoder) from fixed parameters, and a pixel batch."""
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    t, dec, tok = E.TINY_EVA, OM.TINY_OMNI_DEC, OM.TINY_OMNI_TOK
    res = R.ResamplerConfig(grid_size=4, embed_dim=dec.hidden_size, num_heads=dec.hidden_size // 128,
                            kv_dim=t.embed_dim, kv_tokens=t.grid ** 2)
    params = OM.make_omnilmm_params(dec, res, seed)
    params.update({"model.vision_tower." + k: v for k, v in E.make_eva_params(t, seed=seed + 9).items()})
    dims = LlavaDims(frontend="resampler", vocab_size=dec.vocab_size, hidden_size=dec.hidden_size,
                     intermediate_size=dec.intermediate_size, num_layers=dec.num_layers, num_heads=dec.num_heads,
                     num_kv_heads=dec.num_kv_heads, rms_eps=dec.rms_eps, num_query=res.num_queries,
                     vision_width=res.kv_dim, im_patch_token=tok.im_patch, im_start_token=tok.im_start,
                     im_end_token=tok.im_end)
    pol = OmniLMMDPOPolicy(dims, "cuda", hf_state=params, eva_dims=eva_dims(t), tune_clip=tune_clip)
    return pol, params


def pixel_batch(step, B=2, seed=3):
    t, dec, tok = E.TINY_EVA, OM.TINY_OMNI_DEC, OM.TINY_OMNI_TOK
    res = R.ResamplerConfig(grid_size=4, embed_dim=dec.hidden_size, num_heads=dec.hidden_size // 128,
                            kv_dim=t.embed_dim, kv_tokens=t.grid ** 2)
    batch = OM.synthetic_omni_batch(dec, res, tok, B, 28, 20, seed=seed + 7 + step, ragged=True)
    g = torch.Generator().manual_seed(seed + 11 + step)
    batch["images"] = torch.randn(B, 3, t.img_size, t.img_size, generator=g)
    batch["ref_win_logp"] = torch.tensor([-60.0, -62.0])[:B]
    batch["ref_rej_logp"] = torch.tensor([-61.0, -60.5])[:B]
    batch["beta"] = 0.1
    del batch["vision_tokens"]
    return batch


# ---- frozen vs trained ----------------------------------------------------------------------------------------------
def test_frozen_tower_bit_identical_to_trained_downstream():
    from rlaifv_b200 import ops
    batch = pixel_batch(0)
    B = 2
    outs = {}
    for tc in (True, False):
        pol, _ = setup(tc)
        out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
        _, _, _, dpw, dpr, out9 = ops.dpo_loss(out["logp"][:B].contiguous(), out["logp"][B:].contiguous(),
                                               batch["ref_win_logp"].cuda(), batch["ref_rej_logp"].cuda(), 0.1)
        pol.backward_logps(torch.cat([dpw, dpr]).contiguous())
        pol.finalize_embed_grad()
        torch.cuda.synchronize()
        outs[tc] = dict(logp=out["logp"].clone(), pt=out["per_token_logps"].clone(), m=out9.clone(),
                        g=pol.store.grad.clone(), rg=pol.resampler.grad.clone(), vg=pol.vision_token_grad)
        del pol
    t, f = outs[True], outs[False]
    assert torch.equal(t["logp"], f["logp"]) and torch.equal(t["pt"], f["pt"]) and torch.equal(t["m"], f["m"])
    assert torch.equal(t["g"], f["g"]), "decoder gradients differ"
    assert torch.equal(t["rg"], f["rg"]), "resampler gradients differ"
    assert float(t["g"].float().abs().max()) > 0 and float(t["rg"].float().abs().max()) > 0
    assert t["vg"] is not None and f["vg"] is None                  # the frozen tower skips the input gradient


def _footprint(tc):
    from rlaifv_b200.engine import DPOStepEngine
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    pol, _ = setup(tc)
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True)
    torch.cuda.synchronize()
    return eng, torch.cuda.memory_allocated() - before


def test_frozen_tower_three_steps_and_footprint():
    eng_t, foot_t = _footprint(True)
    tower_grad_bytes = eng_t.policy.tower.numel * 2
    del eng_t
    eng, foot_f = _footprint(False)
    pol = eng.policy
    assert foot_t - foot_f >= tower_grad_bytes, (foot_t, foot_f, tower_grad_bytes)
    assert not any(b.name.startswith("eva") for b in eng.opt.buckets)
    w_tower, w_res, w_dec = pol.tower.flat.clone(), pol.resampler.flat.clone(), pol.store.flat.clone()
    losses = []
    for s in range(3):
        b = pixel_batch(0)
        if s == 0:
            out = pol.forward_logps(b["concatenated_input_ids"], b["concatenated_labels"], b["images"],
                                    keep_stash=False)
            ref = out["logp"].float().cpu()
        b["ref_win_logp"], b["ref_rej_logp"] = ref[:2], ref[2:]
        losses.append(float(eng.train_step(b)[0]))
    eng.opt.wait_all()
    torch.cuda.synchronize()
    assert abs(losses[0] - 0.693147) < 2e-3 and losses[2] < losses[0]
    assert torch.equal(pol.tower.flat, w_tower), "the frozen tower's weights changed"
    assert not torch.equal(pol.resampler.flat, w_res) and not torch.equal(pol.store.flat, w_dec)
    # micro-batches of one pair run the tower forward-only as well
    eng.micro_pairs = 1
    m = float(eng.train_step(pixel_batch(1))[0])
    torch.cuda.synchronize()
    assert m == m
    assert torch.equal(pol.tower.flat, w_tower)


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_frozen_tower_policy_meets_reference_fixture_gates(path):
    """The gates test_gpu_omnilmm.py applies to the policy without a tower, on a frozen-tower policy fed the fixture's
    vision tokens; the input gradient of the resampler is not computed (vision_token_grad stays None)."""
    from rlaifv_b200 import ops
    from rlaifv_b200.eva_tower import EvaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    from test_gpu_omnilmm import tiny_dims
    fx = np.load(path)
    dec, res, tok = OM.TINY_OMNI_DEC, OM.TINY_OMNI_RES, OM.TINY_OMNI_TOK
    B, seed = int(fx["B"]), int(fx["seed"])
    params = OM.make_omnilmm_params(dec, res, seed)
    eva = EvaDims(embed_dim=res.kv_dim, depth=3, num_heads=2, mlp_hidden=2 * res.kv_dim, patch_size=14,
                  pretrain_img=56, img_size=14 * int(round(res.kv_tokens ** 0.5)))
    pol = OmniLMMDPOPolicy(tiny_dims(), "cuda", hf_state=params, eva_dims=eva, tune_clip=False)
    batch = OM.synthetic_omni_batch(dec, res, tok, B, 28, 20, seed=seed + 7, ragged=bool(fx["ragged"]))
    ids, labels, vt = batch["concatenated_input_ids"], batch["concatenated_labels"], batch["vision_tokens"]
    out = pol.forward_logps(ids, labels, vt, keep_stash=True)
    slots = torch.arange(2 * B) % B
    assert torch.equal(pol._stash["src"].cpu().long(), OM.inplace_splice_map(ids, tok, res.num_queries, slots))
    pb = {k: v.to(torch.bfloat16) for k, v in params.items()}
    ob = OM.omnilmm_policy_logps(pb, dec, res, tok, ids, labels, vt.to(torch.bfloat16))
    tw = wsum = None
    if "token_weight" in fx.files:
        tw = torch.from_numpy(fx["token_weight"]).cuda()
        logp_dev, _, wsum = ops.logp_weighted_reduce(out["per_token_logps"], out["labels"], tw)
        ob["logp"] = OM.compute_weighted_logp(ob["per_token_logps"].float(), labels, tw.cpu())
    else:
        logp_dev = out["logp"]
    ref_fp32 = torch.from_numpy(fx["logp"])
    assert rel(logp_dev.cpu(), ob["logp"]) <= 1e-3 and rel(logp_dev.cpu(), ref_fp32) <= 1e-3
    mask = labels[:, 1:] != -100
    pt, ref_pt = out["per_token_logps"].cpu(), torch.from_numpy(fx["per_token_logps"])
    inh_pt = rel(ob["per_token_logps"].float()[mask], ref_pt[mask])
    e_pt = rel(pt[mask], ref_pt[mask])
    assert e_pt <= max(1e-3, 2.5 * inh_pt) and e_pt <= 1e-2
    rw, rr = torch.from_numpy(fx["ref_win_logp"]).cuda(), torch.from_numpy(fx["ref_rej_logp"]).cuda()
    losses, _, _, dpw, dpr, out9 = ops.dpo_loss(logp_dev[:B].contiguous(), logp_dev[B:].contiguous(), rw, rr, 0.1)
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous(), token_weight=tw, weight_sum=wsum)
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    assert rel(losses, fx["losses"]) <= 2e-2 and rel(out9[0], fx["loss"]) <= 2e-2
    grads = dict(pol.store.hf_grad_views())
    grads.update({"model.resampler." + k: v for k, v in pol.resampler.g.items()})
    n_checked = 0
    for key in fx.files:
        if not key.startswith("gradnorm:"):
            continue
        name = key.split(":", 1)[1]
        g = grads[name].float().flatten().cpu()
        ref = torch.from_numpy(fx["gradsample:" + name])
        got = g[torch.linspace(0, g.numel() - 1, min(64, g.numel())).long()]
        gn, nrm = float(fx[key]), float(g.double().norm())
        assert abs(nrm - gn) <= 3e-2 * gn, name
        assert float((got - ref).abs().max()) <= 6e-2 * (float(ref.abs().max()) + 1e-12), name
        n_checked += 1
    assert n_checked > 0
    assert pol.vision_token_grad is None


# ---- offloaded optimizer on the OmniLMM policy ---------------------------------------------------------------------
def _engine(tc, budget=None, slot_elems=None):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.zero2 import OffloadAdamW
    pol, _ = setup(tc)
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, micro_pairs=1,
                        offload_optimizer=budget is not None and slot_elems is None, offload_budget=budget)
    if slot_elems is not None:            # small ring slots: several chunks per bucket
        eng.opt = OffloadAdamW(pol.trainable_buckets(), lr=1e-3, gather_order=pol.param_need_order(),
                               device_budget=budget, slot_elems=slot_elems)
        pol.param_ready = eng.opt.wait_bucket
    return eng


def _run(eng, steps, first=0):
    out = [eng.train_step(pixel_batch(s)).clone() for s in range(first, first + steps)]
    eng.opt.wait_all()
    torch.cuda.synchronize()
    return out


def _assert_same(e1, e2, m1, m2):
    for a, b in zip(m1, m2):
        assert torch.equal(a, b), (a, b)
    p1, p2 = e1.policy, e2.policy
    assert torch.equal(p1.store.flat, p2.store.flat)
    assert torch.equal(p1.resampler.flat, p2.resampler.flat)
    assert torch.equal(p1.tower.flat, p2.tower.flat)
    s1, s2 = e1.opt.state_dict(), e2.opt.state_dict()
    assert s1["step"] == s2["step"]
    for k in ("master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(s1[k].cpu(), s2[k].cpu()), k


@pytest.mark.parametrize("split", ["mixed", "all_streamed"])
@pytest.mark.parametrize("tune_clip", [True, False], ids=["trained_tower", "frozen_tower"])
def test_offload_bit_identical_with_tower(tune_clip, split):
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    ref = _engine(tune_clip)
    sz = {b.name: b.size for b in ref.opt.buckets}
    first = ["embed", "resampler"] + (["eva_embed", "eva0"] if tune_clip else ["layer0"])
    budget = STATE_BYTES_PER_ELEM * sum(sz[n] for n in first) if split == "mixed" else 0
    off = _engine(tune_clip, budget, slot_elems=None if split == "mixed" else 1 << 14)
    assert off.opt.streamed_names and bool(off.opt.resident_names) == (split == "mixed")
    if split == "mixed":
        assert off.opt.resident_names == first
        if tune_clip:
            assert "eva1" in off.opt.streamed_names
    if tune_clip:
        # the next forward waits for each tower block's update (recorded after it, also for streamed blocks) before
        # the block reads its weights: record the waits of the second step's forward
        waits = []
        orig = off.opt.wait_bucket
        off.policy.param_ready = lambda name: (waits.append(name), orig(name))[1]
    m_ref, m_off = _run(ref, 3), _run(off, 3)
    _assert_same(ref, off, m_ref, m_off)
    if tune_clip:
        nb = off.policy.tower.dims.live_blocks
        tower = [w for w in waits if w.startswith("eva")]
        assert tower[: nb + 1] == ["eva_embed"] + ["eva%d" % i for i in range(nb)]
        assert waits.index("eva%d" % (nb - 1)) < waits.index("resampler")
    off.opt.close()


def test_checkpoint_resume_frozen_tower_offload_and_cross_mode_refusal():
    """Frozen tower, offloaded optimizer with streamed buckets: the saved model state keeps the tower's (unchanged)
    weights; a policy built from it plus the optimizer checkpoint continues bit-identically. A trained-tower engine
    refuses the frozen-tower optimizer checkpoint, and the reverse."""
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    src = _engine(False, budget=0)
    sz = {b.name: b.size for b in src.opt.buckets}
    budget = STATE_BYTES_PER_ELEM * (sz["embed"] + sz["resampler"])
    src.opt.close()
    src = _engine(False, budget=budget)
    tower0 = {k: v.clone() for k, v in src.policy.tower.timm_state().items()}
    _run(src, 2)
    for b in src.policy.trainable_buckets():
        src.policy._need(b.name)
    state = {k: v.detach().cpu().clone() for k, v in src.policy.hf_views().items()}
    for k, v in tower0.items():
        assert torch.equal(state["model.vision_tower." + k], v.cpu()), k
    opt_sd = src.opt.state_dict()
    dst_pol = OmniLMMDPOPolicy(src.policy.dims, "cuda", hf_state=state, eva_dims=src.policy.tower.dims,
                               tune_clip=False)
    dst = DPOStepEngine(dst_pol, lr=1e-3, total_steps=10, constant_lr=True, micro_pairs=1, offload_optimizer=True,
                        offload_budget=budget)
    dst.load_optimizer_state(opt_sd)
    dst.global_step = src.global_step
    assert torch.equal(dst_pol.store.flat, src.policy.store.flat) and torch.equal(dst_pol.tower.flat, src.policy.tower.flat)
    m_src, m_dst = _run(src, 1, first=2), _run(dst, 1, first=2)
    _assert_same(src, dst, m_src, m_dst)
    trained = _engine(True, budget=budget)
    with pytest.raises(ValueError, match=r"tune_clip=False"):
        trained.load_optimizer_state(opt_sd)
    _run(trained, 1)
    with pytest.raises(ValueError, match=r"tune_clip=True"):
        dst.load_optimizer_state(trained.opt.state_dict())
    for e in (src, dst, trained):
        e.opt.close()


def test_train_omnilmm_frozen_tower_offload_end_to_end(tmp_path, monkeypatch):
    """`train_omnilmm --tune_clip False --deepspeed script/zero2_offload.json` on a tiny checkpoint directory: two steps
    with a checkpoint, first loss ln 2, the tower's weights in the saved model unchanged; a second run resumes from the
    checkpoint; a run with the tower trained refuses that checkpoint."""
    import io
    import json
    from PIL import Image
    from oracle.toy_tokenizer import CharChatTokenizer
    from rlaifv_b200 import train_omnilmm as TO
    from rlaifv_b200.zero2 import OffloadAdamW

    class Tok(CharChatTokenizer):
        SPECIALS = {"<im_patch>": 500, "<im_start>": 501, "<im_end>": 502, "</s>": 2}
        unk_token = pad_token = "<unk>"

        def convert_tokens_to_ids(self, toks):
            return [self.SPECIALS[t] for t in toks]

    monkeypatch.setattr(TO, "load_tokenizer", lambda path, max_len: Tok())
    ckpt = tmp_path / "ckpt"
    ckpt.mkdir()
    t = E.TINY_EVA
    (ckpt / "config.json").write_text(json.dumps({
        "vocab_size": 512, "hidden_size": 512, "intermediate_size": 768, "num_hidden_layers": 2,
        "num_attention_heads": 4, "num_key_value_heads": 2, "rms_norm_eps": 1e-5, "num_query": 16, "image_size": t.img_size,
        "im_patch_token": 500, "im_start_token": 501, "im_end_token": 502,
        "vision_tower_config": {"embed_dim": t.embed_dim, "depth": t.depth, "num_heads": t.num_heads,
                                "mlp_hidden": t.mlp_hidden, "patch_size": t.patch_size, "pretrain_img": t.pretrain_img}}))
    g = torch.Generator().manual_seed(0)
    rows = []
    words = "a red bus on the street near two small dogs and one cat under blue sky".split()
    for i in range(4):
        arr = (torch.rand(40 + 8 * i, 52, 3, generator=g) * 255).to(torch.uint8).numpy()
        buf = io.BytesIO()
        Image.fromarray(arr).save(buf, format="PNG")
        rows.append({"image": {"bytes": buf.getvalue()}, "question": "what is in picture %d ?" % i,
                     "chosen": " ".join(words[i:i + 5]), "rejected": " ".join(words[::-1][i:i + 3]), "idx": i,
                     "origin_dataset": "synthetic", "origin_split": "train", "image_path": "img%d" % i})
    out_dir = tmp_path / "out"

    def argv(steps, tune_clip):
        return ["--model_name_or_path", str(ckpt), "--data_dir", str(tmp_path / "data"), "--task", "DPO",
                "--dpo_beta", "0.1", "--dpo_token_weight", "1.0", "--learning_rate", "1e-3", "--max_steps", str(steps),
                "--per_device_train_batch_size", "2", "--micro_pairs", "1", "--logging_steps", "1",
                "--save_strategy", "steps", "--save_steps", "2", "--lr_scheduler_type", "constant",
                "--model_max_length", "1024", "--output_dir", str(out_dir), "--bf16", "True", "--num_query", "16",
                "--image_size", str(t.img_size), "--tune_clip", tune_clip,
                "--deepspeed", os.path.join(REPO, "script", "zero2_offload.json")]

    tr = TO.train(argv=argv(2, "False"), source_rows=rows)
    torch.cuda.synchronize()
    pol = tr.model.policy
    assert isinstance(tr.engine.opt, OffloadAdamW) and pol.frozen_tower
    assert not any(b.name.startswith("eva") for b in tr.engine.opt.buckets)
    losses = [h["loss"] for h in tr.state["log_history"] if "loss" in h]
    assert len(losses) == 2 and abs(losses[0] - 0.693147) < 5e-3 and all(l == l for l in losses)
    sd = torch.load(out_dir / "pytorch_model.bin")
    ck = torch.load(ckpt.parent / "out" / "checkpoint-2" / "pytorch_model.bin")
    init = TO.OmniLMMForCausalLM(*TO.dims_from_config(str(ckpt), TO.OmniArguments(num_query=16, image_size=t.img_size),
                                                      1024), tune_clip=False).state_dict()
    for k in init:
        if k.startswith("model.vision_tower."):
            assert torch.equal(sd[k], init[k].cpu()) and torch.equal(ck[k], init[k].cpu()), k
    tr.engine.opt.close()
    tr2 = TO.train(argv=argv(3, "False"), source_rows=rows)
    torch.cuda.synchronize()
    assert tr2.state["global_step"] == 3
    assert [h["step"] for h in tr2.state["log_history"] if "loss" in h][-1] == 3
    tr2.engine.opt.close()
    with pytest.raises(ValueError, match=r"tune_clip=False"):
        TO.train(argv=argv(4, "True"), source_rows=rows)
