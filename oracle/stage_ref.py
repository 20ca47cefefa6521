"""ORACLE TOOLING — stages the UNMODIFIED reference under oracle/_ref/ so that it can travel to the GPU box.

The reference is Python: nothing to compile, but its own `pip install` (the one offline install the task allows) puts
its packages (`llava`, `muffin`, `omnilmm`, `utils`, ~1.4 MB of source) into a directory of our choosing:

    python -m pip install --no-index --no-build-isolation --no-deps --target oracle/_ref <copy of /root/reference>

oracle/_ref/ is git-ignored (never in history, the copy detector never sees it) but NOT gpurun-ignored, so
`bench.py --impl reference` on the GPU box's host cores drives the reference's OWN code
(prepare_inputs_labels_for_multimodal -> forward -> get_batch_logps -> dpo_loss -> backward -> torch.optim.AdamW)
instead of the oracle port.  __graft_entry__.build() calls stage() wherever /root/reference exists; where it does not
(the GPU box) the already-staged copy is used as is.  The install runs from a pruned copy under /tmp because
/root/reference is read-only and setuptools writes build/ and *.egg-info into the source tree.
"""
import os
import shutil
import subprocess
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference"
TARGET = os.path.join(HERE, "_ref")
PACKAGES = ("llava", "muffin", "utils")


def available():
    return all(os.path.isdir(os.path.join(TARGET, p)) for p in PACKAGES)


def stage(force=False, verbose=False):
    """Returns True when oracle/_ref is usable afterwards."""
    if available() and not force:
        return True
    if not os.path.isdir(REF_SRC):
        return False
    tmp = tempfile.mkdtemp(prefix="rlaifv_ref_")
    try:
        src = os.path.join(tmp, "src")
        skip = shutil.ignore_patterns(".git", "examples", "*.png", "*.jpg", "*.jpeg", "*.gif", "*.pdf", "*.parquet",
                                      "__pycache__")
        shutil.copytree(REF_SRC, src, ignore=skip)
        if os.path.isdir(TARGET):
            shutil.rmtree(TARGET)
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps", "--quiet",
               "--target", TARGET, src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            if verbose:
                print("staging the reference failed:\n" + r.stdout[-2000:] + r.stderr[-2000:])
            return False
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if verbose:
        print("staged the reference under", TARGET)
    return available()


def import_reference(root=None):
    """Imports the reference's own modules from `root` (default: the staged oracle/_ref) and returns the callables of
    the DPO step path. `matplotlib` is stubbed (utils/utils.py:19 imports it at module top; it is not installed)."""
    root = root or TARGET
    if not os.path.isdir(os.path.join(root, "llava")):
        raise ImportError("reference not found under %s" % root)
    sys.dont_write_bytecode = True
    if root not in sys.path:
        sys.path.insert(0, root)
    for name in ("matplotlib", "matplotlib.pyplot"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    from llava.model import LlavaLlamaForCausalLM, LlavaConfig                      # noqa
    from llava.model.multimodal_encoder.clip_encoder import CLIPVisionTower        # noqa
    from llava.model.multimodal_projector.builder import build_vision_projector    # noqa
    from muffin.train.trainers import get_beta_and_logps, dpo_loss                 # noqa
    from muffin.train.train_muffin import DataCollatorForDPODataset                # noqa
    from muffin.eval.muffin_inference_logp import get_batch_logps                  # noqa
    from transformers import CLIPVisionModel, CLIPVisionConfig                     # noqa
    return dict(LlavaLlamaForCausalLM=LlavaLlamaForCausalLM, LlavaConfig=LlavaConfig,
                CLIPVisionTower=CLIPVisionTower, build_vision_projector=build_vision_projector,
                get_beta_and_logps=get_beta_and_logps, dpo_loss=dpo_loss,
                DataCollatorForDPODataset=DataCollatorForDPODataset, get_batch_logps=get_batch_logps,
                CLIPVisionModel=CLIPVisionModel, CLIPVisionConfig=CLIPVisionConfig)


def build_reference_model(R, cfg, params=None, load=True):
    """SURVEY.md Appendix A recipe: random-init LlavaLlamaForCausalLM with a CLIP tower attached without network
    (bypasses CLIPVisionTower.load_model's from_pretrained, llava/model/multimodal_encoder/clip_encoder.py:25-34)."""
    import torch
    lc = R["LlavaConfig"](vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size,
                          intermediate_size=cfg.intermediate_size, num_hidden_layers=cfg.num_layers,
                          num_attention_heads=cfg.num_heads, num_key_value_heads=cfg.kv_heads,
                          rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta, max_position_embeddings=4096,
                          attn_implementation="eager", tie_word_embeddings=False, pad_token_id=0,
                          bos_token_id=1, eos_token_id=2)
    lc.pretraining_tp = 1
    model = R["LlavaLlamaForCausalLM"](lc)
    vt = R["CLIPVisionTower"].__new__(R["CLIPVisionTower"])
    torch.nn.Module.__init__(vt)
    vt.is_loaded = True
    vt.vision_tower_name = "synthetic"
    vt.select_layer = cfg.select_layer
    vt.select_feature = "patch"
    vc = R["CLIPVisionConfig"](hidden_size=cfg.clip_hidden, intermediate_size=cfg.clip_intermediate,
                               num_hidden_layers=cfg.clip_layers, num_attention_heads=cfg.clip_heads,
                               image_size=cfg.image_size, patch_size=cfg.patch_size, hidden_act="quick_gelu",
                               layer_norm_eps=cfg.clip_eps, attn_implementation="eager")
    vt.vision_tower = R["CLIPVisionModel"](vc)
    vt.vision_tower.requires_grad_(False)
    model.model.vision_tower = vt
    model.config.mm_projector_type = "mlp2x_gelu"
    model.config.mm_hidden_size = cfg.clip_hidden
    model.model.mm_projector = R["build_vision_projector"](model.config)
    model.config.tokenizer_model_max_length = cfg.max_len
    model.config.tokenizer_padding_side = "right"
    model.float()
    if not load or params is None:      # caller assigns the parameters itself, or keeps HF's random init
        return model
    missing, unexpected = model.load_state_dict({k: v.clone() for k, v in params.items()}, strict=False)
    missing = [m for m in missing if "rotary" not in m and "position_ids" not in m]
    assert not missing and not unexpected, (missing, unexpected)
    return model


if __name__ == "__main__":
    ok = stage(force="--force" in sys.argv, verbose=True)
    print("oracle/_ref available:", ok)
