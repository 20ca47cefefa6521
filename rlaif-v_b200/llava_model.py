"""Model facade with the reference's duck-typed protocol (SURVEY.md §8b inner contract).

`LlavaLlamaForCausalLM` here exposes what the reference's trainer / logp code touches on its model:

  prepare_inputs_labels_for_multimodal(input_ids, position_ids, attention_mask, past_key_values, labels, images)
      -> (None, position_ids, attention_mask, past_key_values, inputs_embeds, labels)
         llava/model/llava_arch.py:150-330 (attention_mask=None path, the one get_beta_and_logps uses)
  encode_images(images)                   llava/model/llava_arch.py:141-148
  forward(inputs_embeds=..., labels=None) -> object with .logits      llava_llama.py:57-102
  state_dict() / load_state_dict()        HF names (fused storage is exposed through views)

All arithmetic runs in the CUDA library through LlavaDPOPolicy. `forward` is the inference form
(no activation stash); training goes through trainers.get_beta_and_logps / engine.DPOStepEngine.
"""
from types import SimpleNamespace

import torch

from . import ops
from .model import LlavaDims, LlavaDPOPolicy

_BF = torch.bfloat16


class LlavaLlamaForCausalLM:
    def __init__(self, dims: LlavaDims = None, device="cuda", hf_state=None, seed=0, base_fp8=False):
        self.dims = dims or LlavaDims()
        self.policy = LlavaDPOPolicy(self.dims, device, hf_state=hf_state, seed=seed, base_fp8=base_fp8)
        self.device = self.policy.device
        self.dtype = _BF
        self.training = True
        d = self.dims
        self.config = SimpleNamespace(hidden_size=d.hidden_size, vocab_size=d.vocab_size,
                                      num_hidden_layers=d.num_layers, num_attention_heads=d.num_heads,
                                      intermediate_size=d.intermediate_size, rms_norm_eps=d.rms_eps,
                                      mm_projector_type="mlp2x_gelu", mm_hidden_size=d.clip_hidden,
                                      mm_vision_select_layer=d.select_layer, mm_vision_select_feature="patch",
                                      tokenizer_model_max_length=d.max_len, tokenizer_padding_side="right",
                                      use_cache=False)

    # ---- nn.Module-ish surface the trainer touches ----
    def train(self, mode=True):
        self.training = mode
        return self

    def eval(self):
        return self.train(False)

    def get_model(self):
        return self

    def get_vision_tower(self):
        return self.policy.clip

    def state_dict(self):
        for b in self.policy.store.buckets:              # pending ZeRO-2 parameter all-gathers
            self.policy._need(b.name)
        return {k: v for k, v in self.policy.store.hf_views().items()}

    def load_state_dict(self, state, strict=True):
        self.policy.store.load_hf(state)

    def parameters(self):
        return iter(self.policy.store.hf_views().values())

    # ---- reference protocol ----
    def encode_images(self, images):
        """[n,3,S,S] -> projected image features [n, P, hidden] (bf16)."""
        pol, P = self.policy, self.policy.store.p
        feats = pol.encode_images(images)
        pol._need("projector")
        pre = ops.gemm(feats, P["proj.w0"], bias=P["proj.b0"])
        post = ops.gelu_fwd(pre)
        out = ops.gemm(post, P["proj.w2"], bias=P["proj.b2"])
        return out.view(images.shape[0], self.dims.num_patches, self.dims.hidden_size)

    def prepare_inputs_labels_for_multimodal(self, input_ids, position_ids, attention_mask, past_key_values, labels,
                                             images, image_sizes=None):
        if images is None or input_ids.shape[1] == 1:
            return input_ids, position_ids, attention_mask, past_key_values, None, labels
        if attention_mask is not None:
            raise NotImplementedError("only the attention_mask=None path of the DPO step is implemented "
                                      "(muffin/train/trainers.py:199 sets it to None)")
        pol = self.policy
        input_ids = input_ids.to(pol.device).contiguous()
        lab = None if labels is None else labels.to(pol.device).contiguous()
        feats = self.encode_images(images)
        n_blocks = feats.shape[0]
        embeds, new_labels, _, T = pol.splice(input_ids, lab, feats.reshape(-1, self.dims.hidden_size), n_blocks)
        embeds = embeds.view(input_ids.shape[0], T, self.dims.hidden_size).clone()
        return None, position_ids, attention_mask, past_key_values, embeds, (new_labels if labels is not None else None)

    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                inputs_embeds=None, labels=None, images=None, **kwargs):
        """Inference-form decoder pass on spliced embeddings -> logits [nseq, T, V] (bf16)."""
        if inputs_embeds is None:
            _, _, _, _, inputs_embeds, labels = self.prepare_inputs_labels_for_multimodal(
                input_ids, position_ids, attention_mask, past_key_values, labels, images)
        logits = self.policy.decoder_logits(inputs_embeds)
        return SimpleNamespace(logits=logits, loss=None)

    __call__ = forward
