"""-m gpu: BASELINE.json configs[0] at full width AND full depth (LLaVA-1.5-7B + CLIP-L/14-336, 1 pair, 336 px,
64-token responses, T = 687) — the CUDA path against the outputs of the UNMODIFIED reference on the same seeded weights
(tests/golden_full/config_a.npz, written by oracle/gen_golden_config_a.py: reference in fp32 and, as shipped,
model.bfloat16() + fp32 logits).

The 7B weights are regenerated from the seed and streamed to the GPU tensor by tensor (oracle.iter_params), so no
weight file is committed and the host never holds more than one matrix.

Gates (north_star: "within 1e-3 relative in bf16 vs the reference HF path, bit-exact for token-index gathers"):
  spliced labels                       bit-exact
  summed log-probs  vs bf16 AND fp32 reference   <= 1e-3
  DPO loss          kernel = closed form (1e-5); deviation from the reference bounded by the log-prob deviations
                    (the loss is ill-conditioned at |logp| = 700: the reference's own bf16 run moves it by 2.4e-2)
  per-token log-probs: mean and max abs error <= 1.5x the reference's own bf16-vs-fp32 spread
and the same quantities against the fp32 reference are printed beside the reference's own bf16-vs-fp32 gap.
"""
import os
import time

import numpy as np
import pytest
import torch

from oracle import llava_dpo_oracle as O

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(__file__), "golden_full", "config_a.npz")


def rel(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def stream_policy(cfg, scale, device="cuda"):
    """LlavaDPOPolicy whose parameters are oracle.make_params(cfg, seed=0, scale) — streamed, not materialised."""
    from rlaifv_b200.model import ClipWeights, LlavaDims, LlavaDPOPolicy
    dims = LlavaDims(num_layers=cfg.num_layers)
    pol = LlavaDPOPolicy(dims, device, seed=0)
    views = pol.store.hf_views()
    clip_state, checksum, seen = {}, {}, set()
    for name, t in O.iter_params(cfg, seed=0, scale=scale):
        checksum[name] = float(t.double().abs().sum())
        if name in views:
            views[name].copy_(t.to(device=device, dtype=torch.bfloat16))
            seen.add(name)
        else:
            clip_state[name] = t
    assert seen == set(views), sorted(set(views) - seen)[:4]
    pol.clip = ClipWeights(dims, pol.device, clip_state)
    total = 0.0
    for k in sorted(checksum):
        total += checksum[k]
    return pol, total


@pytest.mark.skipif(not os.path.exists(FIXTURE), reason="tests/golden_full/config_a.npz not generated")
def test_config_a_full_depth_matches_reference():
    from rlaifv_b200 import ops
    fx = np.load(FIXTURE)
    free, _ = torch.cuda.mem_get_info()
    if free < 40 * 2 ** 30:
        pytest.skip("needs ~30 GB of free HBM")
    cfg = O.OracleConfig()
    t0 = time.time()
    pol, checksum = stream_policy(cfg, float(fx["param_scale"]))
    print("7B weights regenerated and streamed in %.0fs" % (time.time() - t0))
    assert abs(checksum - float(fx["params_checksum"])) <= 1e-9 * float(fx["params_checksum"])
    batch = O.synthetic_pair_batch(cfg, 1, int(fx["prompt_len"]), int(fx["resp_len"]), seed=int(fx["seed"]),
                                   image_pos=int(fx["image_pos"]))
    assert np.array_equal(batch["concatenated_input_ids"].numpy(), fx["concatenated_input_ids"])
    assert abs(float(batch["images"].double().abs().sum()) - float(fx["images_checksum"])) <= 1e-9 * float(fx["images_checksum"])
    out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"],
                            keep_stash=False)
    torch.cuda.synchronize()
    assert torch.equal(out["labels"].cpu(), torch.from_numpy(fx["spliced_labels"]))          # index work: bit-exact
    logp = out["logp"].float().cpu()
    ref_bf = torch.cat([torch.from_numpy(fx["bf16_policy_win_logp"]), torch.from_numpy(fx["bf16_policy_rej_logp"])])
    ref_32 = torch.cat([torch.from_numpy(fx["policy_win_logp"]), torch.from_numpy(fx["policy_rej_logp"])])
    losses, cr, rj, _, _, out9 = ops.dpo_loss(out["logp"][:1].contiguous(), out["logp"][1:].contiguous(),
                                              torch.from_numpy(fx["ref_win_logp"]).cuda(),
                                              torch.from_numpy(fx["ref_rej_logp"]).cuda(), float(fx["beta"]))
    mask = torch.from_numpy(fx["spliced_labels"])[:, 1:] != -100
    pt = out["per_token_logps"].float().cpu()[mask]
    pt_bf = torch.from_numpy(fx["bf16_per_token_logps"])[mask]
    pt_32 = torch.from_numpy(fx["per_token_logps"])[mask]
    e_sum_bf, e_sum_32, inh_sum = rel(logp, ref_bf), rel(logp, ref_32), rel(ref_bf, ref_32)
    e_loss_bf, e_loss_32 = rel(losses, fx["bf16_losses"]), rel(losses, fx["losses"])
    inh_loss = rel(fx["bf16_losses"], fx["losses"])
    print("summed logp: cuda %s | ref bf16 %s | ref fp32 %s" % (logp.tolist(), ref_bf.tolist(), ref_32.tolist()))
    print("summed logp rel err: vs bf16 reference %.2e, vs fp32 reference %.2e (reference bf16-vs-fp32 %.2e)"
          % (e_sum_bf, e_sum_32, inh_sum))
    print("DPO loss: cuda %.6f | ref bf16 %.6f | ref fp32 %.6f ; rel err vs bf16 %.2e, vs fp32 %.2e (reference's own %.2e)"
          % (float(losses[0]), float(fx["bf16_losses"][0]), float(fx["losses"][0]), e_loss_bf, e_loss_32, inh_loss))
    print("per-token logp vs bf16 reference: max abs %.3e mean abs %.3e ; vs fp32: max %.3e mean %.3e ; reference's own "
          "bf16-vs-fp32: max %.3e mean %.3e" % (float((pt - pt_bf).abs().max()), float((pt - pt_bf).abs().mean()),
                                                float((pt - pt_32).abs().max()), float((pt - pt_32).abs().mean()),
                                                float((pt_bf - pt_32).abs().max()), float((pt_bf - pt_32).abs().mean())))
    assert e_sum_bf <= 1e-3
    assert e_sum_32 <= 1e-3
    # DPO loss = -logsigmoid(beta * (difference of two log-prob sums of magnitude 700)): a relative tolerance of 1e-3
    # on the sums admits 0.7 absolute on each, i.e. up to beta * 1.4 on the loss, so at 7B depth the loss is
    # ill-conditioned — the reference's OWN bf16 run moves it by 2.4e-2 relative from its fp32 run, and two builds
    # of this repo (different but equally valid summation orders in attention) landed 1.5e-2 and 3.9e-2 from the bf16
    # reference. What CAN be held exactly is consistency: (1) the loss kernel on the CUDA log-probs equals the closed
    # form in fp64 to 1e-5, and (2) the deviation from the reference's loss is bounded by the log-prob deviations that
    # the 1e-3 gates above admit: |dL| <= beta * (|d pi_w| + |d pi_r|)   (|d/dz -logsigmoid(z)| <= 1).
    beta = float(fx["beta"])
    z = beta * ((logp[0].double() - logp[1].double()) - (float(fx["ref_win_logp"][0]) - float(fx["ref_rej_logp"][0])))
    closed = float(torch.nn.functional.softplus(-z))
    assert abs(float(losses[0]) - closed) <= 1e-5 * max(1.0, closed)
    for ref_lp, ref_loss in ((ref_bf, fx["bf16_losses"]), (ref_32, fx["losses"])):
        bound = beta * float((logp.double() - ref_lp.double()).abs().sum())
        assert abs(float(losses[0]) - float(ref_loss[0])) <= bound + 1e-6
    assert e_loss_bf <= 5e-2 and e_loss_32 <= 5e-2          # regression guard, ~2x the reference's own 2.4e-2
    # per token (|log p| ~ 10.5): no worse than 1.5x the reference's own bf16-vs-fp32 spread, mean and max
    own_mean, own_max = float((pt_bf - pt_32).abs().mean()), float((pt_bf - pt_32).abs().max())
    assert float((pt - pt_bf).abs().mean()) <= 1.5 * own_mean and float((pt - pt_32).abs().mean()) <= 1.5 * own_mean
    assert float((pt - pt_bf).abs().max()) <= 1.5 * own_max and float((pt - pt_32).abs().max()) <= 1.5 * own_max
