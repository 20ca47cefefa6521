"""-m gpu parity tests: the CUDA path (through the C ABI) vs the oracle and the golden fixtures that
were produced by the unmodified reference (oracle/gen_golden.py).

The fixtures hold the outputs of the unmodified reference twice: in fp32, and AS SHIPPED — `model.bfloat16()`, bf16
images, fp32 logits (gen_golden.reference_bf16_run; keys `bf16_*`).  The bf16-op-order oracle reproduces that bf16
reference run bit-for-bit on the ragged fixtures, so it is a pinned yardstick, not a guess.

Tolerances (north_star: "within 1e-3 relative in bf16 vs the reference HF path, bit-exact for token-index gathers"):
  splice labels                              bit-exact
  summed log-probs vs the bf16 reference     <= 1e-3   (and vs the bf16-order oracle; vs fp32: the reference's own gap)
  DPO losses vs the bf16 reference           <= 1e-3 of max(|loss|) on the realistically scaled fixtures
  per-token log-probs                        within 2.5x of the reference's OWN bf16-vs-fp32 gap, never worse than 1e-2
  CLIP features / projected image rows       closer to the bf16 reference than that is to the fp32 reference
  gradients                                  norm within 1e-2, samples within 2.5x of the reference's own bf16-vs-fp32 gap
"""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import llava_dpo_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


def cfg_of(fx):
    return O.CONFIGS[str(fx["cfg_name"])] if "cfg_name" in fx.files else O.TINY


def tiny_dims(c=O.TINY):
    from rlaifv_b200.model import LlavaDims
    return LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, num_kv_heads=c.num_kv_heads,
                     clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)


_POL = {}


def policy_for(scale, cfg=O.TINY):
    from rlaifv_b200.model import LlavaDPOPolicy
    key = (scale, id(cfg))
    if key not in _POL:
        params = O.make_params(cfg, seed=0, scale=scale)
        _POL[key] = (LlavaDPOPolicy(tiny_dims(cfg), "cuda", hf_state=params), params)
    return _POL[key]


def rel(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_forward_matches_reference_fixture(path):
    fx = np.load(path)
    cfg = cfg_of(fx)
    pol, params = policy_for(float(fx["param_scale"]), cfg)
    assert abs(O.params_checksum(params) - float(fx["params_checksum"])) < 1e-6 * float(fx["params_checksum"])
    ids = torch.from_numpy(fx["concatenated_input_ids"])
    labels = torch.from_numpy(fx["concatenated_labels"])
    images = torch.from_numpy(fx["images"])
    out = pol.forward_logps(ids, labels, images, keep_stash=False)
    torch.cuda.synchronize()
    # integer work: bit exact
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))
    # bf16-op-order oracle on the same bf16-rounded parameters
    pb = {k: v.to(torch.bfloat16) for k, v in params.items()}
    ob = O.policy_logps(pb, cfg, ids, labels, images.to(torch.bfloat16))
    B = ids.shape[0] // 2
    logp = out["logp"].cpu()
    print("logp cuda", logp.tolist(), "oracle bf16", ob["logp"].tolist(),
          "ref fp32", fx["policy_win_logp"].tolist(), fx["policy_rej_logp"].tolist())
    ref_fp32 = torch.cat([torch.from_numpy(fx["policy_win_logp"]), torch.from_numpy(fx["policy_rej_logp"])])
    # summed log-probs: the 1e-3 gate of BASELINE.md §5, against both the bf16-op-order oracle and
    # the fp32 outputs of the unmodified reference
    inherent_sum = rel(ob["logp"], ref_fp32)       # what the reference's own bf16 op order costs
    e_sum_ref, e_sum_orc = rel(logp, ref_fp32), rel(logp, ob["logp"])
    print(f"summed logp rel err: cuda-vs-fp32ref {e_sum_ref:.2e}, cuda-vs-bf16oracle {e_sum_orc:.2e}, "
          f"inherent {inherent_sum:.2e}")
    assert e_sum_orc <= 1e-3
    # the reference as shipped (model.bfloat16(), fp32 logits): north_star's 1e-3 on the summed log-probs
    ref_bf16 = torch.cat([torch.from_numpy(fx["bf16_policy_win_logp"]), torch.from_numpy(fx["bf16_policy_rej_logp"])])
    e_sum_bf = rel(logp, ref_bf16)
    print(f"summed logp rel err vs the bf16 reference run {e_sum_bf:.2e} (bf16-order oracle vs that run "
          f"{rel(ob['logp'], ref_bf16):.2e})")
    assert e_sum_bf <= 1e-3
    if float(fx["param_scale"]) < 1.0:
        assert e_sum_ref <= 1e-3                   # strict gate on realistically scaled logits
    else:
        assert e_sum_ref <= max(1e-3, 1.5 * inherent_sum)
    # per-token log-probs: a single bf16 logit of magnitude ~2 carries up to 8e-3 absolute rounding
    # error, so two valid bf16 evaluation orders differ by a few 1e-3 relative per token.  The gate
    # is therefore: the CUDA path is as close to the fp32 reference as the reference's own bf16
    # op order is (x2.5 — max-error statistics over a few hundred tokens), and never worse than 1e-2.
    mask = torch.from_numpy(fx["spliced_labels"])[:, 1:] != -100
    pt = out["per_token_logps"].cpu()
    ref_pt = torch.from_numpy(fx["per_token_logps"])
    inherent = rel(ob["per_token_logps"][mask], ref_pt[mask])
    e_ref = rel(pt[mask], ref_pt[mask])
    e_orc = rel(pt[mask], ob["per_token_logps"][mask])
    print(f"per-token rel err: cuda-vs-fp32ref {e_ref:.2e}, cuda-vs-bf16oracle {e_orc:.2e}, "
          f"bf16oracle-vs-fp32ref (inherent) {inherent:.2e}")
    assert e_ref <= max(1e-3, 2.5 * inherent) and e_ref <= 1e-2
    assert e_orc <= max(1e-3, 2.5 * inherent) and e_orc <= 1e-2
    bf_pt = torch.from_numpy(fx["bf16_per_token_logps"])
    e_bf = rel(pt[mask], bf_pt[mask])
    print(f"per-token rel err vs the bf16 reference run {e_bf:.2e}; mean abs {float((pt[mask] - bf_pt[mask]).abs().mean()):.2e}")
    assert e_bf <= max(1e-3, 2.5 * inherent) and e_bf <= 1e-2


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_clip_features_and_projected_rows_match_reference_fixture(path):
    """SURVEY §8 a3 / a4 on their own: CLIP tower output (layer -2, CLS dropped) and mm_projector rows against the
    reference's `get_vision_tower()(images)` / `mm_projector(...)` (clip_encoder.py:46-58, llava_arch.py:141-148)."""
    fx = np.load(path)
    cfg = cfg_of(fx)
    pol, params = policy_for(float(fx["param_scale"]), cfg)
    images = torch.from_numpy(fx["images"])
    feats = pol.encode_images(images).float().cpu()
    proj = pol._frontend_fwd(images, None).float().cpu()
    torch.cuda.synchronize()
    for got, key in ((feats, "clip_features"), (proj, "projected_rows")):
        ref_bf = torch.from_numpy(fx["bf16_" + key]).reshape(got.shape)
        ref_32 = torch.from_numpy(fx[key]).reshape(got.shape)
        own = float((ref_bf - ref_32).abs().mean() / ref_32.abs().mean())      # the reference's bf16-vs-fp32 gap
        e_bf = float((got - ref_bf).abs().mean() / ref_bf.abs().mean())
        e_32 = float((got - ref_32).abs().mean() / ref_32.abs().mean())
        e_max = rel(got, ref_bf)
        print(f"{key}: mean-abs rel err vs bf16 reference {e_bf:.2e} (max {e_max:.2e}), vs fp32 {e_32:.2e}; "
              f"reference bf16-vs-fp32 {own:.2e}")
        # two bf16 evaluations that round at the same points still differ by ~2^-10 per element per rounding; the
        # yardstick is the reference itself: the CUDA path must sit closer to the reference's bf16 run than that run
        # sits to the reference's fp32 run 
        assert e_bf <= own
        assert e_32 <= 1.25 * max(own, 1e-3)
        assert e_max <= 3e-2


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_dpo_loss_and_grads_match_reference_fixture(path):
    from rlaifv_b200 import ops
    fx = np.load(path)
    pol, params = policy_for(float(fx["param_scale"]), cfg_of(fx))
    ids = torch.from_numpy(fx["concatenated_input_ids"])
    labels = torch.from_numpy(fx["concatenated_labels"])
    images = torch.from_numpy(fx["images"])
    B = int(fx["B"])
    out = pol.forward_logps(ids, labels, images, keep_stash=True)
    rw = torch.from_numpy(fx["ref_win_logp"]).cuda()
    rr = torch.from_numpy(fx["ref_rej_logp"]).cuda()
    losses, cr, rj, dpw, dpr, out9 = ops.dpo_loss(out["logp"][:B].contiguous(), out["logp"][B:].contiguous(), rw, rr,
                                                  float(fx["beta"]))
    pol.backward_logps(torch.cat([dpw, dpr]).contiguous())
    pol.finalize_embed_grad()
    torch.cuda.synchronize()
    # DPO loss against the reference run in bf16 (as shipped). The loss is -logsigmoid(beta * (difference of summed
    # log-probs)): on the realistically scaled ("cool") fixtures the 1e-3 of north_star holds; on the hot random
    # networks (scale 1.0: logits of std ~10, an ill-conditioned case no checkpoint looks like) the reference's own
    # two evaluation orders already disagree by more, so the gate there is the reference's own bf16-vs-fp32 gap.
    e_loss_bf = rel(losses, fx["bf16_losses"])
    e_loss_32 = rel(losses, fx["losses"])
    own_loss = rel(fx["bf16_losses"], fx["losses"])
    print(f"DPO losses rel err: vs bf16 reference {e_loss_bf:.2e}, vs fp32 reference {e_loss_32:.2e}; "
          f"reference bf16-vs-fp32 {own_loss:.2e}")
    if float(fx["param_scale"]) < 1.0:
        assert e_loss_bf <= 1e-3
    else:
        assert e_loss_bf <= max(1e-3, 1.5 * own_loss)
    assert e_loss_32 <= max(2e-3, 2.5 * own_loss)
    assert rel(cr, fx["bf16_chosen_rewards"]) <= 2e-3
    grads = pol.store.hf_grad_views()
    for key in fx.files:
        if not key.startswith("gradsample:"):
            continue
        name = key.split(":", 1)[1]
        g = grads[name].float().flatten().cpu()
        idx = torch.linspace(0, g.numel() - 1, 64).long()
        got = g[idx]
        ref = torch.from_numpy(fx[key])
        gn = float(fx["gradnorm:" + name])
        err = float((got - ref).abs().max())
        scale = float(ref.abs().max()) + 1e-12
        nrm = float(g.double().norm())
        own_s = float(np.abs(fx["bf16_gradsample:" + name] - fx[key]).max()) / scale   # reference bf16 vs fp32
        own_n = abs(float(fx["bf16_gradnorm:" + name]) - gn) / gn
        print(f"{name}: sample err {err / scale:.2e} (reference's own bf16-vs-fp32 {own_s:.2e}); "
              f"norm err {abs(nrm - gn) / gn:.2e} (own {own_n:.2e})")
        assert abs(nrm - gn) <= 1e-2 * gn, name
        assert err <= max(2.5 * own_s, 2e-2) * scale, name
