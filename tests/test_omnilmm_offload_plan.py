"""CPU tests of the OmniLMM-12B (config d) side of the offloaded optimizer: the activation reserve in both tower modes
against hand arithmetic from the shapes, the resident order of OmniLMM's buckets, `train_omnilmm --tune_clip False` with
script/zero2_offload.json building an OffloadAdamW engine on a faked device, and the host-memory refusal at the
trained-tower plan."""
import json
import os

import pytest
import torch

from test_offload_plan import MEMINFO, _fake_cuda

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GB = 1 << 30

# config (d) shapes: Mistral-7B decoder (H 4096, ffn 14336, 32 q / 8 kv heads of 128, V 32008), 64-query resampler,
# EVA-02-E at 448 px (1792 wide, 16 heads padded to 128, mlp 15360, 63 live blocks, 1 + 32 * 32 tokens)
DEC_PER_TOKEN = 32 * (2 * (4 * 4096 + 2 * 1024 + 2 * 14336) + 8 + 4 * 32) + 16 * 4096
RESAMPLER_PER_IMAGE = 1024 * 2 * (2 * 1792 + 9 * 4096) + 64 * 2 * 3 * 4096
EVA_OUT_PER_IMAGE = 1025 * 2 * 1792 + 1024 * 2 * 1792            # final LayerNorm output + tokens without the prefix
EVA_FROZEN_WORK = 1025 * (2 * (4 * 2048 + 6 * 1792 + 2 * 15360) + 4 * 16) + EVA_OUT_PER_IMAGE
EVA_TRAINED_WORK = 1025 * (2 * ((1792 + 15360) + (5 * 1792 + 2 * 15360 + 4 * 2048)) + 4 * 16) + EVA_OUT_PER_IMAGE
EVA_STASH = 63 * 1025 * (2 * (4 * 2048 + 4 * 1792 + 15360) + 4 * 16) + 1024 * 2 * 640 + 1025 * 2 * 1792
EMBED_GRAD = 4 * 32008 * 4096


def _no_init(monkeypatch):
    """Full-size policies are built on the meta device for their shapes; skip the random initialisation."""
    from rlaifv_b200.eva_tower import EvaTower
    from rlaifv_b200.model import LlavaDPOPolicy
    monkeypatch.setattr(LlavaDPOPolicy, "_random_init", lambda self, seed, std: None)
    monkeypatch.setattr(EvaTower, "_random_init", lambda self, seed: None)


def _config_d(max_len):
    from rlaifv_b200.eva_tower import EvaDims
    from rlaifv_b200.omnilmm_model import omnilmm_dims
    return omnilmm_dims(max_len=max_len), EvaDims()


@pytest.mark.parametrize("tune_clip,pairs,max_len", [(False, 2, 1024), (False, 2, 2048), (True, 1, 1024)])
def test_reserve_matches_hand_arithmetic(tune_clip, pairs, max_len):
    from rlaifv_b200.zero2 import activation_reserve_bytes, omnilmm_activation_reserve_bytes
    dims, eva = _config_d(max_len)
    got = omnilmm_activation_reserve_bytes(dims, eva, pairs, max_len, tune_clip=tune_clip)
    want = 2 * pairs * max_len * DEC_PER_TOKEN + pairs * RESAMPLER_PER_IMAGE
    want += pairs * (EVA_TRAINED_WORK + EVA_STASH if tune_clip else EVA_FROZEN_WORK)
    assert got == want
    # the decoder part is the LLaVA formula at the GQA widths
    assert activation_reserve_bytes(dims, pairs, max_len) == 2 * pairs * max_len * DEC_PER_TOKEN
    # the issue-level numbers: 12.6 GB of decoder activations for 2 pairs at 1024, ~4 GB of tower stash per image
    assert 12.6e9 < 2 * pairs * max_len * DEC_PER_TOKEN * (1024 / max_len) * (2 / pairs) < 12.7e9
    assert 3.9e9 < EVA_STASH < 4.1e9 and EVA_FROZEN_WORK < 0.12e9


def test_policy_reserve_adds_the_embedding_gradient(monkeypatch):
    """The policy's reserve (what the engine's default budget subtracts) = the OmniLMM formula + the fp32 [V, H] buffer;
    a frozen tower drops its stash and the larger backward working set."""
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    _no_init(monkeypatch)
    dims, eva = _config_d(1024)
    frozen = OmniLMMDPOPolicy(dims, "meta", eva_dims=eva, tune_clip=False)
    trained = OmniLMMDPOPolicy(dims, "meta", eva_dims=eva, tune_clip=True)
    base = 2 * 2 * 1024 * DEC_PER_TOKEN + 2 * RESAMPLER_PER_IMAGE + EMBED_GRAD
    assert frozen.activation_reserve_bytes(2, 1024) == base + 2 * EVA_FROZEN_WORK
    assert trained.activation_reserve_bytes(2, 1024) == base + 2 * (EVA_TRAINED_WORK + EVA_STASH)
    # frozen: no gradient buffer and no optimizer buckets for the tower
    assert frozen.tower.grad is None and frozen.tower.opt_buckets() == []
    names = [b.name for b in frozen.trainable_buckets()]
    assert not any(n.startswith("eva") for n in names) and "resampler" in names
    assert not any(n.startswith("eva") for n in frozen.param_need_order())
    assert [b.name for b in trained.trainable_buckets()][-64:] == ["eva_embed"] + ["eva%d" % i for i in range(63)]
    assert trained.param_need_order()[:2] == ["eva_embed", "eva0"]


def test_llava_reserve_unchanged(monkeypatch):
    """LLaVA's reserve through the policy is the decoder formula plus the embedding gradient, as before."""
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    from rlaifv_b200.zero2 import activation_reserve_bytes
    _no_init(monkeypatch)
    d = LlavaDims(max_len=2048)
    pol = LlavaDPOPolicy(d, "meta")
    assert pol.activation_reserve_bytes(2, 2048) == activation_reserve_bytes(d, 2, 2048) + 4 * d.vocab_size * d.hidden_size


def test_omnilmm_resident_order_pinned():
    """Resident first: the buckets whose gradients become final last. embed and resampler are stepped after the whole
    backward; the tower's backward ends with eva0 and eva_embed; then the decoder from layer0 up; the head last."""
    from rlaifv_b200.zero2 import offload_plan, offload_priority
    names = (["embed"] + ["layer%d" % i for i in range(32)] + ["head", "resampler", "eva_embed"]
             + ["eva%d" % i for i in range(63)])
    want = (["embed", "resampler", "eva_embed"] + ["eva%d" % i for i in range(63)] + ["layer%d" % i for i in range(32)]
            + ["head"])
    assert offload_priority(names) == want
    assert offload_priority(names[::-1]) == ["resampler", "embed"] + want[2:]      # only the tail keeps input order
    frozen = [n for n in names if not n.startswith("eva")]
    assert offload_priority(frozen) == ["embed", "resampler"] + ["layer%d" % i for i in range(32)] + ["head"]
    res, streamed = offload_plan([(n, 10) for n in names], 12 * 10 * 5)
    assert res == ["embed", "resampler", "eva_embed", "eva0", "eva1"] and streamed == want[5:]


def _tiny_omni_ckpt(tmp_path):
    ckpt = tmp_path / "ckpt"
    ckpt.mkdir()
    (ckpt / "config.json").write_text(json.dumps({
        "vocab_size": 512, "hidden_size": 512, "intermediate_size": 768, "num_hidden_layers": 2,
        "num_attention_heads": 4, "num_key_value_heads": 2, "rms_norm_eps": 1e-5, "num_query": 16, "image_size": 84,
        "im_patch_token": 500, "im_start_token": 501, "im_end_token": 502,
        "vision_tower_config": {"embed_dim": 224, "depth": 4, "num_heads": 2, "mlp_hidden": 448, "patch_size": 14,
                                "pretrain_img": 56}}))
    return ckpt


def test_train_omnilmm_frozen_tower_offload_engine(tmp_path, monkeypatch):
    """`train_omnilmm --tune_clip False --deepspeed script/zero2_offload.json --micro_pairs 1 --model_max_length 256`
    builds an OffloadAdamW engine on the frozen-tower policy whose default budget is the free memory minus the policy's
    reserve for one pair at 256 tokens, the ring and the margin."""
    from rlaifv_b200 import train_llava15 as T15
    from rlaifv_b200 import train_omnilmm as TO
    from rlaifv_b200 import trainers
    from rlaifv_b200.zero2 import DEFAULT_SLOT_ELEMS, DEFAULT_SLOTS, DEVICE_MARGIN, STATE_BYTES_PER_ELEM, OffloadAdamW
    _fake_cuda(monkeypatch)
    ckpt = _tiny_omni_ckpt(tmp_path)
    seen = {}

    def fake_init_model(model_args, data_args, training_args, omni_args, source_rows=None):
        dims, eva = TO.dims_from_config(model_args.model_name_or_path, omni_args, training_args.model_max_length)
        seen.update(tune_clip=omni_args.tune_clip, offload=training_args.offload_optimizer, dims=dims)
        model = TO.OmniLMMForCausalLM(dims, eva, "cpu", tune_clip=omni_args.tune_clip)
        seen["model"] = model
        return model, dict(train_dataset=None, eval_dataset=None, data_collator=None), None

    free = 1 << 40
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (free, 80 << 30))
    monkeypatch.setattr(TO, "init_model", fake_init_model)
    monkeypatch.setattr(trainers.LLaVA15DPOTrainer, "train", lambda self, resume_from_checkpoint=None: self.state)
    monkeypatch.setattr(trainers.LLaVA15DPOTrainer, "save_state", lambda self: None)
    monkeypatch.setattr(T15, "safe_save_model_for_hf_trainer", lambda trainer, output_dir: None)
    tr = TO.train(argv=["--model_name_or_path", str(ckpt), "--data_dir", str(tmp_path / "data"), "--task", "DPO",
                        "--deepspeed", os.path.join(REPO, "script", "zero2_offload.json"), "--tune_clip", "False",
                        "--micro_pairs", "1", "--per_device_train_batch_size", "2", "--model_max_length", "256",
                        "--output_dir", str(tmp_path / "out"), "--image_size", "84", "--num_query", "16"])
    assert seen["tune_clip"] is False and seen["offload"] is True
    pol = seen["model"].policy
    assert pol.frozen_tower and pol.tower.grad is None
    opt = tr.engine.opt
    assert isinstance(opt, OffloadAdamW)
    assert not any(b.name.startswith("eva") for b in opt.buckets)
    sizes = {b.name: b.size for b in opt.buckets}
    ring = DEFAULT_SLOTS * 3 * min(DEFAULT_SLOT_ELEMS, max(sizes.values())) * 4
    assert opt.device_budget == free - pol.activation_reserve_bytes(1, 256) - ring - DEVICE_MARGIN
    assert pol.activation_reserve_bytes(1, 256) > pol.activation_reserve_bytes(1, 128)
    assert opt.streamed_names == [] and opt.master.numel() == opt.owned == sum(sizes.values())
    assert STATE_BYTES_PER_ELEM * opt.owned <= opt.device_budget
    # the default stays tune_clip=True
    from rlaifv_b200.train_omnilmm import OmniArguments
    assert OmniArguments().tune_clip is True


def test_optimizer_checkpoint_across_tower_modes_refused(monkeypatch):
    """A frozen-tower optimizer checkpoint has no tower buckets: resuming it with a trained tower (and the reverse) is
    refused with a message that names the mismatch; any other size mismatch is refused by the optimizer."""
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    from rlaifv_b200 import train_omnilmm as TO
    _fake_cuda(monkeypatch)
    dims, eva = TO.dims_from_config(None, TO.OmniArguments(num_query=16, image_size=84), 256)
    import dataclasses
    from rlaifv_b200.eva_tower import EvaDims
    dims = dataclasses.replace(dims, vocab_size=512, hidden_size=512, intermediate_size=768, num_layers=2, num_heads=4,
                               num_kv_heads=2, vision_width=224, im_patch_token=500, im_start_token=501,
                               im_end_token=502)
    eva = EvaDims(embed_dim=224, depth=4, num_heads=2, mlp_hidden=448, patch_size=14, pretrain_img=56, img_size=84)
    engines = {tc: DPOStepEngine(OmniLMMDPOPolicy(dims, "cpu", eva_dims=eva, tune_clip=tc)) for tc in (False, True)}
    sd = {tc: e.opt.state_dict() for tc, e in engines.items()}
    with pytest.raises(ValueError, match=r"frozen \(tune_clip=False\).*trains the tower"):
        engines[True].load_optimizer_state(sd[False])
    with pytest.raises(ValueError, match=r"trained \(tune_clip=True\).*freezes the tower"):
        engines[False].load_optimizer_state(sd[True])
    bad = dict(sd[False], master=sd[False]["master"][:-8])
    with pytest.raises(ValueError, match="different set of trainable parameters"):
        engines[False].load_optimizer_state(bad)
    engines[False].load_optimizer_state(sd[False])                 # same mode resumes


def test_trained_tower_plan_refused_by_host_memory(monkeypatch):
    """The trained-tower recipe (--micro_pairs 1 --model_max_length 1024) on one 80 GB card streams ~120 GB of state;
    with less MemAvailable than that plus the margin the optimizer refuses before allocating or pinning anything. The
    frozen-tower recipe at the same free memory streams under half of it."""
    from rlaifv_b200 import zero2
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy
    from rlaifv_b200.zero2 import DEFAULT_SLOTS, DEFAULT_SLOT_ELEMS, DEVICE_MARGIN, STATE_BYTES_PER_ELEM, offload_plan
    _fake_cuda(monkeypatch)
    _no_init(monkeypatch)
    registered = []
    monkeypatch.setattr(zero2.OffloadAdamW, "_register", lambda self, t: registered.append(t))
    dims, eva = _config_d(1024)
    ring = DEFAULT_SLOTS * 3 * DEFAULT_SLOT_ELEMS * 4
    streamed = {}
    for tc in (True, False):
        pol = OmniLMMDPOPolicy(dims, "meta", eva_dims=eva, tune_clip=tc)
        sizes = [(b.name, b.size) for b in pol.trainable_buckets()]
        weights = 2 * (pol.store.flat.numel() + pol.resampler.flat.numel() + pol.tower.numel)
        grads = 2 * sum(n for _, n in sizes)
        free = 85 * 10 ** 9 - weights - grads                      # an 80 GB H100 after weights and gradients
        micro = 1 if tc else 2
        budget = free - pol.activation_reserve_bytes(micro, 1024) - ring - DEVICE_MARGIN
        res, st = offload_plan(sizes, budget)
        n_of = dict(sizes)
        streamed[tc] = STATE_BYTES_PER_ELEM * sum(n_of[n] for n in st)
        assert res[:2] == ["embed", "resampler"] and st[-1] == "head"
        if tc:
            monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (free, 80 << 30))
            monkeypatch.setattr("rlaifv_b200.zero2._read_meminfo", lambda: MEMINFO % (100 * GB // 1024))
            with pytest.raises(MemoryError, match=r"needs 1[0-9][0-9]\.\d\d GB of pinned host memory.*MemAvailable is "
                                                  r"107\.37 GB"):
                DPOStepEngine(pol, offload_optimizer=True, micro_pairs=micro)
            assert not registered
    assert 110e9 < streamed[True] < 130e9
    assert 50e9 < streamed[False] < 70e9


def test_frozen_tower_zero2_world2_leaves_the_tower_out(monkeypatch):
    """ZeRO-2 at world 2 with a frozen tower: no tower bucket is sharded, reduced or gathered, and the forward's
    parameter waits skip the tower (a wait on a bucket no optimizer owns would raise)."""
    import dataclasses
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.eva_tower import EvaDims
    from rlaifv_b200.omnilmm_model import OmniLMMDPOPolicy, omnilmm_dims
    _fake_cuda(monkeypatch)
    dims = dataclasses.replace(omnilmm_dims(), vocab_size=512, hidden_size=512, intermediate_size=768, num_layers=2,
                               num_heads=4, num_kv_heads=2, vision_width=224, num_query=16, im_patch_token=500,
                               im_start_token=501, im_end_token=502)
    eva = EvaDims(embed_dim=224, depth=4, num_heads=2, mlp_hidden=448, patch_size=14, pretrain_img=56, img_size=84)
    pol = OmniLMMDPOPolicy(dims, "cpu", eva_dims=eva, tune_clip=False)
    eng = DPOStepEngine(pol, rank=1, world=2)
    opt = eng.opt
    assert not any(b.name.startswith("eva") for b in opt.buckets)
    assert opt.owned == sum(b.size for b in opt.buckets) // 2
    reduced = []
    monkeypatch.setattr(opt, "reduce_bucket", lambda name: reduced.append(name))
    eng._last_micro = True
    for name in ("eva_embed", "eva0"):
        pol._need(name)                          # no KeyError from wait_bucket
    assert pol.tower.param_ready is None and pol.tower.on_block_grads_ready is None
    eng._bucket_ready("resampler")
    assert reduced == []                          # a tail bucket: reduced after the whole backward
    with pytest.raises(KeyError):
        opt.wait_bucket("eva0")
