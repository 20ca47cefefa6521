"""OmniLMM-12B DPO policy (BASELINE config d; SURVEY.md §8 a13) on the H100 kernels: EVA vision tower (eva_tower.py,
trained or frozen) -> perceiver resampler -> in-place <im_patch> splice -> Mistral decoder (grouped-query attention) ->
per-token log-prob gather, and the backward of all of it.

Mirrors what `forward_DPO` (muffin/train/trainers.py:66-88) executes on an `OmniLMMForCausalLM`
(omnilmm/model/omnilmm.py:268-346): `OmniLMMModel.forward` (:183-265) embeds the ids, replaces the num_query rows after
each <im_start> by `get_vision_embedding(images)` (:107-120 = tower -> drop prefix tokens -> `Resampler`), runs the HF
Mistral stack and `lm_head`; `get_batch_logps` (muffin/eval/muffin_inference_logp.py:82-115) follows.

`images` are pixels [B, 3, S, S] when the policy was built with `eva_dims` (the whole config-(d) model), or — for a
policy built without a tower — the tower's output tokens [B, N, vision_width] (prefix tokens already dropped; the
gradient w.r.t. them is left in `self.vision_token_grad`). The decoder, loss, optimizer and ZeRO-2 plumbing are the
LLaVA path's; the tower's blocks are extra ZeRO-2 buckets whose reduce-scatter / AdamW start as each block's backward
finishes.

`tune_clip=False` is the reference's frozen tower (`OmniLMMModel` keeps it in a Python list, omnilmm.py:58-70 and
:74-94, so it is not in `parameters()`): the tower runs forward every step without a stash and is never updated, while
the resampler and the decoder train. It has no gradient buffer and no optimizer buckets, the resampler's backward stops
at its own parameters (`vision_token_grad` stays None), and with ZeRO-2 the tower is replicated and never reduced or
gathered, like LLaVA's CLIP. `hf_views()` (and so a saved checkpoint) still holds the tower's unchanged weights, so the
model loads like a trained-tower one; the reference's `state_dict()` would drop them.
"""
import torch

from . import ops
from .model import LlavaDims, LlavaDPOPolicy
from .resampler import Resampler

_BF = torch.bfloat16


def omnilmm_dims(**kw):
    """Mistral-7B decoder + 64-query resampler over 1024 EVA-02-E tokens (omnilmm/model/omnilmm.py:31-52;
    HF MistralConfig of the 7B: ffn 14336, 32 query / 8 key-value heads, rms eps 1e-5)."""
    base = dict(frontend="resampler", hidden_size=4096, intermediate_size=14336, num_layers=32, num_heads=32,
                num_kv_heads=8, rms_eps=1e-5, rope_theta=10000.0, vocab_size=32008, num_query=64, vision_width=1792,
                im_patch_token=32000, im_start_token=32001, im_end_token=32002)
    base.update(kw)
    return LlavaDims(**base)


class OmniLMMDPOPolicy(LlavaDPOPolicy):
    def __init__(self, dims: LlavaDims, device="cuda", hf_state=None, seed=0, init_std=0.02, eva_dims=None,
                 tune_clip=True):
        assert dims.frontend == "resampler" and dims.hidden_size % 128 == 0
        assert min(dims.im_patch_token, dims.im_start_token, dims.im_end_token) >= 0, "set the <im_*> token ids"
        super().__init__(dims, device, hf_state=hf_state, seed=seed, init_std=init_std)
        grid = int(round(dims.num_query ** 0.5))
        assert grid * grid == dims.num_query
        pre = "model.resampler."
        rstate = None if hf_state is None else {k[len(pre):]: v for k, v in hf_state.items() if k.startswith(pre)}
        self.resampler = Resampler(grid, dims.hidden_size, dims.hidden_size // 128, dims.vision_width, self.device,
                                   state=rstate, seed=seed + 2)
        self.vision_token_grad = None
        self.tower = None
        self.tune_clip = bool(tune_clip)
        if eva_dims is not None:
            from .eva_tower import EvaTower
            assert eva_dims.embed_dim == dims.vision_width
            tpre = "model.vision_tower."
            tstate = None if hf_state is None else {k[len(tpre):]: v for k, v in hf_state.items() if k.startswith(tpre)}
            self.tower = EvaTower(eva_dims, self.device, state=tstate or None, seed=seed + 3, trainable=self.tune_clip)
            if self.tune_clip:        # a frozen tower's weights are no optimizer's: nothing to wait for, nothing to step
                self.tower.param_ready = self._need
                self.tower.on_block_grads_ready = self._tower_block_ready

    @property
    def frozen_tower(self):
        return self.tower is not None and not self.tune_clip

    on_bucket_grads_ready = None     # callable(bucket name), set by the engine (reduce-scatter + AdamW of that bucket)

    def _tower_block_ready(self, i):
        if self.on_bucket_grads_ready is not None:
            self.on_bucket_grads_ready("eva_embed" if i == "embed" else "eva%d" % i)

    def enable_lora(self, *a, **k):
        raise NotImplementedError("the reference has no LoRA recipe for OmniLMM")

    # ---- optimizer view ----
    def trainable_buckets(self):
        tower = self.tower.opt_buckets() if self.tower is not None else []
        return self.store.opt_buckets() + self.resampler.opt_buckets() + tower

    def param_need_order(self):
        tower = [b.name for b in self.tower.buckets] if self.tower is not None and self.tune_clip else []
        return tower + ["resampler", "embed"] + [f"layer{i}" for i in range(self.dims.num_layers)] + ["head"]

    def _need(self, bucket):
        if self.frozen_tower and (bucket == "eva_embed" or (bucket.startswith("eva") and bucket[3:].isdigit())):
            return                                # frozen tower: no optimizer owns its buckets
        super()._need(bucket)

    def activation_reserve_bytes(self, pairs, seq_len):
        """LlavaDPOPolicy.activation_reserve_bytes plus, per image, the resampler and the EVA tower: its working set,
        and its stash when it trains (zero2.omnilmm_activation_reserve_bytes)."""
        from .zero2 import omnilmm_activation_reserve_bytes
        d = self.dims
        eva = self.tower.dims if self.tower is not None else None
        return (omnilmm_activation_reserve_bytes(d, eva, pairs, seq_len, tune_clip=self.tune_clip,
                                                 stash_act=self.stash_act) + 4 * d.vocab_size * d.hidden_size)

    def check_optimizer_state(self, sd, owned, world=1):
        """Refuse an optimizer checkpoint written in the other tower mode: a frozen tower's run has no state for the
        tower's buckets, which follow every other bucket in the flat layout."""
        if self.tower is None:
            return
        n, tower = sd["master"].numel(), self.tower.numel // world
        if self.tune_clip and n == owned - tower:
            raise ValueError("optimizer checkpoint was written with the EVA tower frozen (tune_clip=False): it has no "
                             "state for the tower's %d buckets, but this policy trains the tower (tune_clip=True). "
                             "Resume with --tune_clip False or start a new run." % len(self.tower.buckets))
        if not self.tune_clip and n == owned + tower:
            raise ValueError("optimizer checkpoint was written with the EVA tower trained (tune_clip=True): it holds "
                             "state for the tower's %d buckets, but this policy freezes the tower (tune_clip=False). "
                             "Resume with --tune_clip True or start a new run." % len(self.tower.buckets))

    def tail_bucket_names(self):
        # the tower's buckets are reduced / stepped block by block from its backward (on_bucket_grads_ready)
        return ["embed", "resampler"]

    def hf_views(self):
        out = dict(self.store.hf_views())
        out.update({"model.resampler." + k: v for k, v in self.resampler.state_dict().items()})
        if self.tower is not None:
            out.update({"model.vision_tower." + k: v for k, v in self.tower.timm_state().items()})
        return out

    # ---- vision front-end: resampler on the tower's tokens ----
    def _frontend_fwd(self, images, st):
        d = self.dims
        if images.dim() == 4:                       # pixels: get_vision_embedding (omnilmm.py:107-120) tower first
            assert self.tower is not None, "this policy was built without the vision tower (pass eva_dims)"
            trained = self.tune_clip and st is not None
            tokens = self.tower.forward(images, keep_stash=trained)
            if trained:
                st["tower_ran"] = True
        else:
            tokens = images.to(device=self.device, dtype=_BF)
        assert tokens.dim() == 3 and tokens.shape[2] == d.vision_width, \
            "OmniLMM policy takes pixels [B,3,S,S] or the vision tower's output tokens [B, N, vision_width]"
        self._need("resampler")
        feats = self.resampler.forward(tokens, keep_stash=st is not None)       # [b, Q, H]
        return feats.view(tokens.shape[0] * d.num_query, d.hidden_size)

    def _frontend_bwd(self, dproj, st, acc):
        if not acc:
            self.resampler.zero_grad()            # first micro-batch of the step overwrites, later ones accumulate
        b = st["b"]
        # frozen tower: nothing upstream of the resampler trains, so its input gradient is not computed
        self.vision_token_grad = self.resampler.backward(dproj.view(b, self.dims.num_query, self.dims.hidden_size),
                                                         input_grad=not self.frozen_tower)
        if self.on_bucket_grads_ready is not None:
            self.on_bucket_grads_ready("resampler")
        if st.get("tower_ran"):
            self.tower.backward(self.vision_token_grad, accumulate=acc)

    # ---- in-place splice (length unchanged, labels unchanged) ----
    def splice(self, input_ids, labels, image_rows, n_blocks, img_index=None, T_hint=None):
        d = self.dims
        nseq, L = input_ids.shape
        if img_index is None:
            img_index = torch.arange(nseq, dtype=torch.int32, device=self.device)
        src, status = ops.splice_map_inplace(input_ids, img_index, d.num_query, d.im_patch_token, d.im_start_token,
                                             d.im_end_token)
        if T_hint is None:                        # same single tiny D2H per step as the LLaVA path's length query
            code = int(status.item())
            if code & 1:
                raise ValueError("The number of image start tokens and image end tokens should be the same.")
            if code & 2:
                raise ValueError("The image end token should follow the image start token.")
        embeds = ops.splice_gather(src, input_ids, self.store.p["embed"], image_rows,
                                   out=self.buf("x0", (nseq * L, d.hidden_size)))
        return embeds, labels, src, L
