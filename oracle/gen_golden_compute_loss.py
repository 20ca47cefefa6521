"""ORACLE TOOLING — stores what tests/test_gpu_trainer_compat.py::test_reference_compute_loss_text_on_rebound_seam
compares the engine against: the reference's own `LLaVA15DPOTrainer.compute_loss` (from the staged oracle/_ref copy,
__graft_entry__.build() stages it where the reference source is present) with `get_beta_and_logps` / `dpo_loss` rebound
to this repo's, on the test's batch and weights. Needs a GPU and oracle/_ref:

    python oracle/gen_golden_compute_loss.py [OUT.npz]      (default tests/golden/trainer/compute_loss_rebound.npz)
"""
import importlib.util
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(REPO, "tests", "golden", "trainer", "compute_loss_rebound.npz")
    spec = importlib.util.spec_from_file_location("_seam", os.path.join(REPO, "tests", "test_gpu_trainer_compat.py"))
    t = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(t)
    from oracle import llava_dpo_oracle as O
    from oracle import stage_ref
    if not stage_ref.available():
        raise SystemExit("oracle/_ref is not staged: run __graft_entry__.build() where the reference source is present")
    loss, logged, grad = t.run_reference_compute_loss(t.seam_batch(), O.make_params(O.TINY, seed=0, scale=0.4))
    idx = t.seam_grad_index(grad.numel())
    rec = {"loss": np.float64(loss), "grad_sample": grad[idx.to(grad.device)].cpu().numpy().astype(np.float32)}
    rec.update({"metric:" + k: np.float64(logged[k]) for k in t.SEAM_METRICS})
    os.makedirs(os.path.dirname(out), exist_ok=True)
    np.savez_compressed(out, **rec)
    print("wrote", out, "loss", loss)


if __name__ == "__main__":
    main()
