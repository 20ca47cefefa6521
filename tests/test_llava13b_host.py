"""CPU tests: LLaVA-1.5-13B on the host side — the widths read from its config.json, the memory plan of LoRA and full
fine-tuning at those widths, and the launch sequence of a decoder wider than 4096."""
import ctypes
import json

import pytest
import torch

from oracle import llava_dpo_oracle as O

# llava-v1.5-13b/config.json (the decoder) and clip-vit-large-patch14-336/config.json (the tower), the keys
# dims_from_checkpoint reads; llava-v1.5-13b carries no rope_theta, so HF's default 1e4 applies
LLAVA13B_CONFIG = {"architectures": ["LlavaLlamaForCausalLM"], "model_type": "llava", "hidden_size": 5120,
                   "intermediate_size": 13824, "num_attention_heads": 40, "num_hidden_layers": 40,
                   "num_key_value_heads": 40, "rms_norm_eps": 1e-05, "vocab_size": 32000, "mm_hidden_size": 1024,
                   "mm_projector_type": "mlp2x_gelu", "mm_vision_select_layer": -2,
                   "mm_vision_tower": "openai/clip-vit-large-patch14-336", "max_position_embeddings": 4096,
                   "tie_word_embeddings": False}
CLIP_L336_CONFIG = {"vision_config": {"hidden_size": 1024, "intermediate_size": 4096, "num_hidden_layers": 24,
                                      "num_attention_heads": 16, "image_size": 336, "patch_size": 14,
                                      "layer_norm_eps": 1e-05}}


def dims13b():
    from rlaifv_b200.model import LlavaDims
    return LlavaDims(hidden_size=5120, intermediate_size=13824, num_layers=40, num_heads=40)


def test_dims_from_a_llava13b_checkpoint(tmp_path):
    from rlaifv_b200.train_llava15 import dims_from_checkpoint
    (tmp_path / "llm").mkdir()
    (tmp_path / "clip").mkdir()
    (tmp_path / "llm" / "config.json").write_text(json.dumps(LLAVA13B_CONFIG))
    (tmp_path / "clip" / "config.json").write_text(json.dumps(CLIP_L336_CONFIG))
    d = dims_from_checkpoint(str(tmp_path / "llm"), str(tmp_path / "clip"), -2, 2048)
    assert d == dims13b()
    assert (d.head_dim, d.kv_heads, d.num_patches, d.clip_layers_used) == (128, 40, 576, 23)
    assert (d.rms_eps, d.rope_theta, d.max_len) == (1e-5, 10000.0, 2048)


def test_13b_parameter_counts_and_activation_reserve():
    """Full fine-tuning trains 13.05 B parameters (26.1 GB bf16, 156.6 GB of fp32 master / m / v); LoRA r = 64 trains
    250 347 520 adapter parameters plus the 31 467 520-parameter projector. A decoder layer keeps 116 904 bytes of
    activations per token (92 KB at 7B widths)."""
    from rlaifv_b200.model import LlavaDims, LoraStore, ParamStore
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM, activation_reserve_bytes
    d = dims13b()
    store = ParamStore(d, "meta")                   # layout only: no memory behind it
    n = {b.name: b.size for b in store.buckets}
    assert store.numel == sum(n.values()) == 13_047_331_840
    assert n["projector"] == 31_467_520 and n["embed"] == 163_840_000 and n["layer0"] == 317_204_480
    assert STATE_BYTES_PER_ELEM * store.numel == 156_567_982_080
    one_layer = LoraStore(LlavaDims(hidden_size=5120, intermediate_size=13824, num_layers=1, num_heads=40), "cpu", r=64)
    assert one_layer.numel * d.num_layers == 250_347_520
    per_token_layer = (activation_reserve_bytes(d, 1, 1) - 2 * 16 * d.hidden_size) // (2 * d.num_layers)
    assert per_token_layer == 116_904
    assert activation_reserve_bytes(d, 1, 2048) == 19_489_095_680
    assert activation_reserve_bytes(d, 4, 1135) == 4 * activation_reserve_bytes(d, 1, 1135)


def test_13b_full_ft_offload_plan_on_one_80gb_card():
    """Full fine-tuning of 13B on one 80 GB card: after 26.1 GB of bf16 weights and 26.1 GB of gradients, the reserve
    for one pair at 2048 tokens, the staging ring and the device margin, 5.2 GB of optimizer state fits on the device
    (embed and projector). The other 154.2 GB is streamed from pinned host memory, and the planner refuses unless
    MemAvailable covers it plus the 8 GiB host margin (162.8 GB)."""
    from rlaifv_b200.model import ParamStore
    from rlaifv_b200.zero2 import (DEFAULT_SLOT_ELEMS, DEFAULT_SLOTS, DEVICE_MARGIN, HOST_MARGIN, STATE_BYTES_PER_ELEM,
                                   activation_reserve_bytes, check_host_memory, offload_plan)
    d = dims13b()
    store = ParamStore(d, "meta")
    sizes = [(b.name, b.size) for b in store.buckets]
    n_of = dict(sizes)
    free = 80 * 10 ** 9 - 2 * 2 * store.numel                              # bf16 weights + bf16 gradients
    reserve = activation_reserve_bytes(d, 1, d.max_len) + 4 * d.vocab_size * d.hidden_size
    ring = DEFAULT_SLOTS * 3 * min(DEFAULT_SLOT_ELEMS, max(n_of.values())) * 4
    budget = free - reserve - ring - DEVICE_MARGIN
    assert budget == 5_216_743_424
    resident, streamed = offload_plan(sizes, budget)
    assert resident == ["embed", "projector"]
    assert streamed == [f"layer{i}" for i in range(40)] + ["head"]
    assert sorted(resident + streamed) == sorted(n_of)                     # every bucket exactly once
    dev_bytes = STATE_BYTES_PER_ELEM * sum(n_of[k] for k in resident)
    host_bytes = STATE_BYTES_PER_ELEM * sum(n_of[k] for k in streamed)
    assert dev_bytes <= budget
    assert dev_bytes + host_bytes == STATE_BYTES_PER_ELEM * store.numel
    assert host_bytes == 154_224_291_840
    need_kb = (host_bytes + HOST_MARGIN) // 1024
    meminfo = "MemTotal: 2113470464 kB\nMemAvailable: %d kB\n"
    assert check_host_memory(host_bytes, meminfo % (need_kb + 1)) == (need_kb + 1) * 1024
    with pytest.raises(MemoryError, match="154.22 GB of pinned host memory"):
        check_host_memory(host_bytes, meminfo % (need_kb - 1))


def test_launch_sequence_dry_run_wider_than_4096(monkeypatch):
    """The decoder at H = 5120 (40 heads of 128) runs its forward and backward launch sequence on the host, full
    fine-tuning and LoRA; every RMSNorm backward gets the 5120-wide rows."""
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = O.OracleConfig(vocab_size=512, hidden_size=5120, intermediate_size=1024, num_layers=1, num_heads=40,
                       clip_hidden=128, clip_intermediate=256, clip_layers=3, clip_heads=2, image_size=56, patch_size=14)
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    calls, argv = [], {}

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append(name)
        argv.setdefault(name, []).append(args)

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    params = O.make_params(c, seed=0, scale=0.09)
    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    for use_lora in (False, True):
        calls.clear()
        argv.clear()
        pol = LlavaDPOPolicy(dims, "cpu", hf_state=params)
        if use_lora:
            pol.enable_lora(r=64, alpha=16.0)
        monkeypatch.setattr(pol, "splice", lambda ids, labels, rows, nb, idx, T_hint=None: (
            torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), torch.full((4, T), -100),
            torch.zeros(4, T, dtype=torch.int32), T))
        out = pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
        assert out["logp"].shape == (4,)
        pol.backward_logps(torch.zeros(4))
        pol.finalize_embed_grad()
        assert calls.count("rlaifv_attention_fwd") == dims.num_layers + dims.clip_layers_used
        assert calls.count("rlaifv_attention_bwd_split") == dims.num_layers
        # two norms per layer and the final norm, forward and backward, all 5120 wide
        assert calls.count("rlaifv_rmsnorm_fwd") >= 2 * dims.num_layers + 1
        assert calls.count("rlaifv_rmsnorm_bwd") == 2 * dims.num_layers + 1
        H_POS = 10          # rlaifv_rmsnorm_bwd(dy, x, w, rstd, dres, dx, dw, acc, workspace, M, H, stream)
        assert all(a[H_POS] == 5120 for a in argv["rlaifv_rmsnorm_bwd"])
        assert calls.count("rlaifv_gemm_bf16_dual") == ((2 * 4 - 1) * dims.num_layers if use_lora else 0)
