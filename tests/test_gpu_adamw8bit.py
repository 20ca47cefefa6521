"""GPU tests of AdamW with blockwise 8-bit moments (rlaifv_adamw8bit_step, rlaifv_adamw8bit_offload_bucket,
optim="adamw_8bit"): the quantizer against the reference bit for bit, general betas within bounds, the offloaded
optimizer against the on-device one bit for bit, checkpoints, footprints, entry-point refusals, training sanity, the
trainer's --optim adamw_bnb_8bit end to end, and two ranks."""
import dataclasses
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import adamw8bit_oracle as Q
from oracle import llava_dpo_oracle as O

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
LR, EPS, WD = 1e-3, 1e-8, 0.01


def _maps():
    return [m.to(DEV) for m in Q.maps()]


def _rand_state(n, seed):
    """A state in the 8-bit format with random codes and scales (what earlier steps could have left)."""
    g = torch.Generator().manual_seed(seed)
    nb = (n + 255) // 256
    master = torch.randn(n, generator=g) * 0.02
    qm = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8)
    qv = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8)
    am = torch.rand(nb, generator=g) * 1e-2
    av = torch.rand(nb, generator=g) * 1e-4
    return [master, qm, qv, am, av]


def _grad(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g) * torch.logspace(-5, 0, n)[torch.randperm(n, generator=g)]
    x[256:512] = 0.0                                     # an all-zero block
    x[512:768] = 0.0
    x[700] = -0.75                                       # a block with a single non-zero
    return x.bfloat16()


def _kernel_step(state, grad, decay_n, b1, b2, step):
    from rlaifv_b200 import ops
    mm, mv = _maps()
    master, qm, qv, am, av = [t.to(DEV) for t in state]
    g = grad.to(DEV)
    p = torch.empty_like(g)
    ops.adamw8bit_step(master, qm, qv, am, av, g, p, decay_n, mm, mv, LR, b1, b2, EPS, WD, step)
    torch.cuda.synchronize()
    return [t.cpu() for t in (master, qm, qv, am, av, p)]


@pytest.mark.parametrize("n,decay_n", [(256 * 40, 256 * 40), (256 * 40 + 72, 256 * 3 + 40), (4104, 0)])
def test_quantizer_bit_exact_with_zero_betas(n, decay_n):
    """beta1 = beta2 = 0: the new moments are g and g * g under any FMA contraction, so codes and absmax equal the
    reference bit for bit: random data, an all-zero block, a block with one non-zero, a partial last block
    (n % 256 = 72 or 8) and a decay edge inside a block."""
    state = _rand_state(n, 1)
    grad = _grad(n, 2)
    got = _kernel_step(state, grad, decay_n, 0.0, 0.0, 1)
    ref = Q.step(*state, grad, decay_n, LR, 0.0, 0.0, EPS, WD, 1)
    for name, a, b in zip(("code_m", "code_v", "absmax_m", "absmax_v"), got[1:5], ref[1:5]):
        assert torch.equal(a, b), (name, int((a != b).sum()))
    assert float(got[3][1]) == 0.0 and float(got[4][1]) == 0.0 and bool((got[1][256:512] == 127).all())
    assert float(got[3][2]) == 0.75 and int(got[1][700]) == 0 and int(got[2][700]) == 255
    # the master: the same operations, FMA contraction aside
    assert torch.allclose(got[0], ref[0], rtol=2 ** -20, atol=LR * 2 ** -18)
    assert torch.equal(got[5], got[0].bfloat16())


def test_general_betas_five_steps_within_bounds():
    """beta1 = 0.9, beta2 = 0.999, five steps; each step's reference starts from the kernel's state. fp32 FMA
    contraction may move a moment across a code midpoint: codes differ on at most 1e-3 of the elements and only by one
    code. A contracted m = b1 m + (1 - b1) g rounds once instead of twice, so it may differ by an ulp of its
    uncancelled terms |b1 m| + |(1 - b1) g|: absmax within 2^-20 of that per block, and the master within 2^-20 of
    |p| + lr / bc1 * (|b1 m| + |(1 - b1) g|) / denom."""
    n, decay_n = 256 * 4096 + 136, 256 * 2000 + 24
    state = _rand_state(n, 3)
    mm, mv = Q.maps()
    for step in range(1, 6):
        grad = _grad(n, 10 + step)
        got = _kernel_step(state, grad, decay_n, 0.9, 0.999, step)
        ref = Q.step(*state, grad, decay_n, LR, 0.9, 0.999, EPS, WD, step)
        for a, b in ((got[1], ref[1]), (got[2], ref[2])):
            d = (a.int() - b.int()).abs()
            assert int(d.max()) <= 1 and int((d > 0).sum()) <= 1e-3 * n, (int(d.max()), int((d > 0).sum()))
        m_old = Q.dequantize(state[1], state[3], mm)
        terms = 0.9 * m_old.abs() + 0.1 * grad.float().abs()
        assert bool(((got[3] - ref[3]).abs() <= 2 ** -20 * Q.block_absmax(terms, n)).all())
        assert bool(((got[4] - ref[4]).abs() <= 2 ** -20 * ref[4]).all())
        bc1 = 1 - 0.9 ** step
        denom = ref[6].sqrt() / math.sqrt(1 - 0.999 ** step) + EPS
        tol = 2 ** -20 * (ref[0].abs() + LR / bc1 * terms / denom)
        assert bool(((got[0] - ref[0]).abs() <= tol).all()), float(((got[0] - ref[0]).abs() / tol).max())
        dm = Q.dequantize(got[1], got[3], mm) - Q.dequantize(ref[1], ref[3], mm)
        assert float(dm.abs().max()) <= 0.05 * float(ref[3].max())     # one code of the signed map, at most
        dv = Q.dequantize(got[2], got[4], mv) - Q.dequantize(ref[2], ref[4], mv)
        assert float(dv.abs().max()) <= 0.05 * float(ref[4].max())
        state = got[:5]


def test_offload_entry_point_matches_on_device_bit_for_bit():
    """Three steps over a range of several chunks, the last partial, with the decay edge inside a block."""
    from rlaifv_b200 import ops
    from rlaifv_b200.zero2 import adamw8bit_slot_bytes
    slot, n, decay_n = 4096, 4096 * 3 + 1000, 4096 + 300
    mm, mv = _maps()
    host = [t.pin_memory() for t in _rand_state(n, 5)]
    dev = [t.to(DEV) for t in host]
    p_dev = host[0].to(DEV).bfloat16()
    p_off = p_dev.clone()
    ring = torch.empty((3, adamw8bit_slot_bytes(slot)), dtype=torch.uint8, device=DEV)
    h2d, d2h = torch.cuda.Stream(), torch.cuda.Stream()
    for step in (1, 2, 3):
        grad = _grad(n, 20 + step).to(DEV)
        ops.adamw8bit_step(*dev, grad, p_dev, decay_n, mm, mv, LR, 0.9, 0.999, EPS, WD, step)
        ops.adamw8bit_offload_bucket(*host, grad, p_off, decay_n, mm, mv, ring, slot, LR, 0.9, 0.999, EPS, WD, step,
                                     h2d, d2h)
        torch.cuda.synchronize()
    assert torch.equal(p_off, p_dev)
    for h, d in zip(host, dev):
        assert torch.equal(h, d.cpu())
    ops.adamw_offload_release(ring)


def test_entry_points_refuse_bad_input():
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.zero2 import adamw8bit_slot_bytes
    n, slot = 4096, 1024
    mm, mv = _maps()
    grad = torch.zeros(n, dtype=torch.bfloat16, device=DEV)
    p = torch.zeros_like(grad)
    ring = torch.empty((3, adamw8bit_slot_bytes(slot)), dtype=torch.uint8, device=DEV)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    pageable = _rand_state(n, 6)
    with pytest.raises(lib.B200Error, match="pinned host"):
        ops.adamw8bit_offload_bucket(*pageable, grad, p, n, mm, mv, ring, slot, LR, 0.9, 0.999, EPS, WD, 1, s1, s2)
    pinned = [t.pin_memory() for t in pageable]
    with pytest.raises(lib.B200Error, match="multiple of 256"):
        ops.adamw8bit_offload_bucket(*pinned, grad, p, n, mm, mv, ring, slot - 8, LR, 0.9, 0.999, EPS, WD, 1, s1, s2)
    m = 4092                                             # n % 8 != 0
    bad = [t.to(DEV) for t in _rand_state(m, 7)]
    with pytest.raises(lib.B200Error, match="n % 8"):
        ops.adamw8bit_step(*bad, grad[:m], p[:m], m, mm, mv, LR, 0.9, 0.999, EPS, WD, 1)
    with pytest.raises(lib.B200Error, match="n % 8"):
        ops.adamw8bit_offload_bucket(*[t.pin_memory() for t in _rand_state(m, 7)], grad[:m], p[:m], m, mm, mv, ring,
                                     slot, LR, 0.9, 0.999, EPS, WD, 1, s1, s2)
    torch.cuda.synchronize()


# ---- whole engine -------------------------------------------------------------------------------------------------
CFG4 = dataclasses.replace(O.TINY, num_layers=4)


def _dims(c):
    from rlaifv_b200.model import LlavaDims
    return LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)


def _engine(optim="adamw_8bit", offload=None, slot_elems=None, c=CFG4, lr=1e-3):
    """Tiny LLaVA engine, micro_pairs 1 < B = 2. offload: None (Zero2AdamW) or a device budget in bytes."""
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDPOPolicy
    from rlaifv_b200.zero2 import OffloadAdamW
    pol = LlavaDPOPolicy(_dims(c), DEV, hf_state=O.make_params(c, seed=0, scale=0.4))
    eng = DPOStepEngine(pol, lr=lr, total_steps=10, constant_lr=True, micro_pairs=1, optim=optim,
                        offload_optimizer=offload is not None and slot_elems is None, offload_budget=offload)
    if slot_elems is not None:            # small ring slots: several chunks per bucket
        eng.opt = OffloadAdamW(pol.trainable_buckets(), lr=lr, gather_order=pol.param_need_order(),
                               device_budget=offload, slot_elems=slot_elems, optim=optim)
        pol.param_ready = eng.opt.wait_bucket
    return eng


def _batch(step, c=CFG4):
    batch = O.synthetic_pair_batch(c, 2, 24, 20, seed=5 + step, image_pos=7, ragged=True)
    batch["ref_win_logp"] = torch.tensor([-60.0, -70.0])
    batch["ref_rej_logp"] = torch.tensor([-61.0, -69.0])
    batch["beta"] = 0.1
    return batch


def _run(eng, steps, first=0):
    out = [eng.train_step(_batch(s)).clone() for s in range(first, first + steps)]
    eng.opt.wait_all()
    torch.cuda.synchronize()
    return out


def _assert_same(e1, e2, m1, m2):
    from rlaifv_b200.zero2 import state_parts
    for a, b in zip(m1, m2):
        assert torch.equal(a, b), (a, b)
    assert torch.equal(e1.policy.store.flat, e2.policy.store.flat)
    s1, s2 = e1.opt.state_dict(), e2.opt.state_dict()
    assert s1["step"] == s2["step"] and s1["optim"] == s2["optim"] == "adamw_8bit"
    for k, _, _ in state_parts("adamw_8bit"):
        assert torch.equal(s1[k].cpu(), s2[k].cpu()), k


def _sizes(eng):
    return {b.name: b.size for b in eng.policy.trainable_buckets()}


def _budget(sz, names):
    from rlaifv_b200.zero2 import state_bytes
    return sum(state_bytes(sz[k], "adamw_8bit") for k in names)


@pytest.mark.parametrize("split", ["mixed", "all_streamed"])
def test_engine_offload_bit_identical(split):
    """4 decoder layers, three steps: the offloaded 8-bit optimizer gives the on-device one's metrics, bf16
    parameters, master, codes and absmax bit for bit."""
    ref = _engine()
    sz = _sizes(ref)
    budget = _budget(sz, ("embed", "projector", "layer0")) if split == "mixed" else 0
    off = _engine(offload=budget, slot_elems=None if split == "mixed" else 1 << 14)
    assert off.opt.streamed_names and (bool(off.opt.resident_names) == (split == "mixed"))
    if split == "all_streamed":
        assert max(sz.values()) > off.opt.slot_elems            # several chunks per bucket
    m_ref, m_off = _run(ref, 3), _run(off, 3)
    _assert_same(ref, off, m_ref, m_off)
    off.opt.close()


@pytest.mark.parametrize("direction", ["device_to_offload", "offload_to_device"])
def test_checkpoint_resume_bit_identical(direction):
    """A state_dict written by one optimizer resumes with the other, and the resumed step equals continuing without
    the checkpoint bit for bit. A checkpoint of the other format is refused."""
    sz = _sizes(_engine())
    budget = _budget(sz, ("embed", "projector"))
    src = _engine() if direction == "device_to_offload" else _engine(offload=budget)
    _run(src, 2)
    dst = _engine(offload=budget) if direction == "device_to_offload" else _engine()
    dst.policy.store.flat.copy_(src.policy.store.flat)
    sd = src.opt.state_dict()
    sd = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in sd.items()}
    assert sd["optim"] == "adamw_8bit" and sd["exp_avg_q"].dtype == torch.uint8
    dst.load_optimizer_state(sd)
    dst.global_step = src.global_step
    torch.cuda.synchronize()
    m_src, m_dst = _run(src, 1, first=2), _run(dst, 1, first=2)
    _assert_same(src, dst, m_src, m_dst)
    other = _engine(optim="adamw_torch", offload=None if direction == "offload_to_device" else 0, slot_elems=None)
    with pytest.raises(ValueError, match="adamw_8bit state.*adamw_torch state"):
        other.load_optimizer_state(sd)
    with pytest.raises(ValueError, match="adamw_torch state.*adamw_8bit state"):
        dst.load_optimizer_state(other.opt.state_dict())
    for e in (src, dst, other):
        if hasattr(e.opt, "close"):
            e.opt.close()


def test_footprints():
    """On the device the state takes exactly state_bytes per slice; offloaded, the pinned bytes are the streamed
    state and the device holds only the ring."""
    from rlaifv_b200.zero2 import OffloadAdamW, Zero2AdamW, adamw8bit_slot_bytes, state_bytes, state_parts
    eng = _engine(optim="adamw_torch")
    pol = eng.policy
    expect = sum(state_bytes(b.size, "adamw_8bit") for b in pol.trainable_buckets())
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    opt = Zero2AdamW(pol.trainable_buckets(), optim="adamw_8bit")
    own = sum(getattr(opt, k).numel() * getattr(opt, k).element_size() for k, _, _ in state_parts("adamw_8bit"))
    assert own == expect == opt.state_nbytes
    assert torch.cuda.memory_allocated() - before <= expect + 2 * 256 * 4 + (1 << 20)
    del opt
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    off = OffloadAdamW(pol.trainable_buckets(), device_budget=0, slot_elems=1 << 14, optim="adamw_8bit")
    torch.cuda.synchronize()
    ring = 3 * adamw8bit_slot_bytes(1 << 14)
    assert off.ring.numel() == ring and off.resident_names == []
    assert torch.cuda.memory_allocated() - before <= ring + (1 << 20)
    assert off.pinned_bytes == expect
    for k, _, _ in state_parts("adamw_8bit"):
        assert getattr(off, "host_" + k).is_pinned()
    off.close()
    assert not off.host_master.is_pinned()


def _train(eng, batch, steps):
    losses = [float(eng.train_step(batch)[0]) for _ in range(steps)]
    eng.opt.wait_all()
    torch.cuda.synchronize()
    return losses


# Bound on the final-loss gap between the two optimizers after 10 steps, as a fraction of the fp32 run's loss drop.
# Measured on an NVIDIA H100 80GB HBM3 (700 W): tiny fixture, lr 1e-3: gap 2.1e-5 of a 0.686 drop (3.1e-5 of it);
# 7B widths at 2 layers, lr 5e-7: gap 7.2e-4 of a 0.643 drop (1.1e-3 of it).
GAP_BOUND = {"tiny": 1e-3, "7b_width_2_layers": 1e-2}


def test_training_sanity_tiny():
    """Both optimizers lower the loss from ln 2 over 10 steps on one batch, and end close to each other."""
    res = {}
    for optim in ("adamw_torch", "adamw_8bit"):
        eng = _engine(optim=optim, c=O.TINY, lr=1e-3)
        batch = _batch(0, O.TINY)
        ids, lab, img = batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"]
        ref = []
        for i in range(2):                # reference log-probs of the initial policy, per micro-batch of one pair
            out = eng.policy.forward_logps(ids[i::2].to(DEV), lab[i::2].to(DEV), img[i:i + 1].to(DEV),
                                           keep_stash=False)
            ref.append(out["logp"].float().cpu())
        batch["ref_win_logp"] = torch.stack([r[0] for r in ref])
        batch["ref_rej_logp"] = torch.stack([r[1] for r in ref])
        res[optim] = _train(eng, batch, 11)
    _check_sanity(res, "tiny")


def _check_sanity(res, key):
    l32, l8 = res["adamw_torch"], res["adamw_8bit"]
    print(key, "fp32", l32, "8bit", l8)
    for ls in (l32, l8):
        assert abs(ls[0] - math.log(2)) < 1e-3 and ls[-1] < ls[0] - 1e-3
    drop = l32[0] - l32[-1]
    assert abs(l8[-1] - l32[-1]) <= GAP_BOUND[key] * drop, (l8[-1], l32[-1], drop)


def test_training_sanity_7b_width_2_layers():
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    sys.path.insert(0, REPO)
    import bench
    B, micro = 2, 2
    res = {}
    for optim in ("adamw_torch", "adamw_8bit"):
        pol = LlavaDPOPolicy(LlavaDims(num_layers=2), torch.device("cuda", 0), seed=0)
        eng = DPOStepEngine(pol, lr=5e-7, weight_decay=0.01, total_steps=10, constant_lr=True, micro_pairs=micro,
                            optim=optim)
        hb = bench.synthetic_batch(0, 0, B)
        out = pol.forward_logps(hb["concatenated_input_ids"], hb["concatenated_labels"], hb["images"],
                                keep_stash=False)
        hb["ref_win_logp"], hb["ref_rej_logp"] = out["logp"][:B].float().cpu(), out["logp"][B:].float().cpu()
        res[optim] = _train(eng, hb, 11)
        del eng, pol
        torch.cuda.empty_cache()
    _check_sanity(res, "7b_width_2_layers")


def test_train_llava15_entry_with_adamw_bnb_8bit(tmp_path, monkeypatch):
    """train_llava15.train(--optim adamw_bnb_8bit) end to end on a tiny checkpoint: the optimizer keeps 8-bit moments,
    two steps run from ln 2 and the parameters move."""
    import io
    import json
    from PIL import Image
    from oracle.toy_tokenizer import ToyTokenizer
    from rlaifv_b200 import data as D
    from rlaifv_b200 import train_llava15 as TL
    c = O.TINY
    params = O.make_params(c, seed=0, scale=0.4)
    ckpt, vt = tmp_path / "ckpt", tmp_path / "clip"
    ckpt.mkdir()
    vt.mkdir()
    vp = "model.vision_tower.vision_tower."
    torch.save({k: v for k, v in params.items() if not k.startswith(vp)}, ckpt / "pytorch_model.bin")
    torch.save({k[len(vp):]: v for k, v in params.items() if k.startswith(vp)}, vt / "pytorch_model.bin")
    (ckpt / "config.json").write_text(json.dumps({
        "vocab_size": c.vocab_size, "hidden_size": c.hidden_size, "intermediate_size": c.intermediate_size,
        "num_hidden_layers": c.num_layers, "num_attention_heads": c.num_heads, "rms_norm_eps": c.rms_eps}))
    (vt / "config.json").write_text(json.dumps({"vision_config": {
        "hidden_size": c.clip_hidden, "intermediate_size": c.clip_intermediate, "num_hidden_layers": c.clip_layers,
        "num_attention_heads": c.clip_heads, "image_size": c.image_size, "patch_size": c.patch_size}}))
    (vt / "preprocessor_config.json").write_text(json.dumps({
        "size": {"shortest_edge": c.image_size}, "crop_size": {"height": c.image_size, "width": c.image_size},
        "image_mean": [0.48145466, 0.4578275, 0.40821073], "image_std": [0.26862954, 0.26130258, 0.27577711]}))
    monkeypatch.setattr(D, "load_tokenizer", lambda path, max_len: ToyTokenizer())
    g = torch.Generator().manual_seed(1)
    words = "a red bus on the street near two small dogs and one cat under blue sky with trees".split()
    rows = []
    for i in range(6):
        arr = (torch.rand(70 + 10 * i, 90, 3, generator=g) * 255).to(torch.uint8).numpy()
        buf = io.BytesIO()
        Image.fromarray(arr).save(buf, format="PNG")
        rows.append({"image": {"bytes": buf.getvalue()}, "question": "what is shown in picture %d ?" % i,
                     "chosen": " ".join(words[i:i + 6]), "rejected": " ".join(words[::-1][i:i + 4]), "idx": i,
                     "origin_dataset": "synthetic", "origin_split": "train", "image_path": "img%d" % i})
    out_dir = tmp_path / "out"
    tr = TL.train(argv=["--model_name_or_path", str(ckpt), "--vision_tower", str(vt), "--mm_vision_select_layer", "-2",
                        "--data_dir", str(tmp_path / "data"), "--data_source_names", "", "--data_source_weights", "1",
                        "--task", "DPO", "--dpo_beta", "0.1", "--dpo_token_weight", "1.0", "--learning_rate", "1e-3",
                        "--max_steps", "2", "--per_device_train_batch_size", "3", "--logging_steps", "1",
                        "--save_strategy", "no", "--lr_scheduler_type", "constant", "--model_max_length", "2048",
                        "--output_dir", str(out_dir), "--bf16", "True", "--image_aspect_ratio", "pad",
                        "--optim", "adamw_bnb_8bit"], source_rows=rows)
    torch.cuda.synchronize()
    assert tr.engine.opt.optim == "adamw_8bit"
    assert tr.engine.opt.exp_avg_q.dtype == torch.uint8 and int(tr.engine.opt.absmax.count_nonzero()) > 0
    losses = [h["loss"] for h in tr.state["log_history"] if "loss" in h]
    assert len(losses) == 2 and abs(losses[0] - 0.693147) < 5e-3 and all(l == l for l in losses)
    w0 = params["model.layers.0.mlp.down_proj.weight"].to(torch.bfloat16)
    w2 = tr.model.state_dict()["model.layers.0.mlp.down_proj.weight"].cpu()
    assert float((w2.float() - w0.float()).abs().max()) > 0
    assert os.path.exists(out_dir / "pytorch_model.bin")


TWO_RANK = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, %(repo)r)
from oracle import llava_dpo_oracle as O
from rlaifv_b200.engine import DPOStepEngine
from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
dist.init_process_group("nccl")
rank, world = dist.get_rank(), dist.get_world_size()
torch.cuda.set_device(rank)
c = O.TINY
dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                 num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                 clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                 image_size=c.image_size, patch_size=c.patch_size)
batch = O.synthetic_pair_batch(c, 4, 24, 20, seed=5, image_pos=7, ragged=True)
batch["ref_win_logp"] = torch.tensor([-60.0, -70.0, -65.0, -62.0])
batch["ref_rej_logp"] = torch.tensor([-61.0, -69.0, -64.0, -63.0])
batch["beta"] = 0.1
def run(r, w, group):
    pol = LlavaDPOPolicy(dims, "cuda:%%d" %% torch.cuda.current_device(), hf_state=O.make_params(c, seed=0, scale=0.4))
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, rank=r, world=w, group=group,
                        optim="adamw_8bit")
    B = 4 // w
    sub = {k: (torch.cat([v[r * B:(r + 1) * B], v[4 + r * B:4 + (r + 1) * B]]) if k.startswith("concatenated")
               else v[r * B:(r + 1) * B]) if torch.is_tensor(v) else v for k, v in batch.items()}
    for _ in range(2):
        m = eng.train_step(sub)
    eng.opt.wait_all()
    torch.cuda.synchronize()
    return eng.metrics_dict(m)["loss"], pol.store.flat.float().cpu()
loss2, flat2 = run(rank, world, None)
if rank == 0:
    torch.save({"loss": loss2, "flat": flat2}, os.environ["OUT2"])
dist.destroy_process_group()
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_8bit_step_matches_single_gpu(tmp_path):
    """Two ZeRO-2 ranks with 8-bit moments (bucket sizes are multiples of 1024, so each rank's slices start on block
    edges and the block layout is the one GPU's) take two steps on the global batch that one GPU takes alone: loss and
    parameters within 1e-3 relative (the gradients' reduction order differs)."""
    script = tmp_path / "two_rank.py"
    script.write_text(TWO_RANK % {"repo": REPO})
    env = dict(os.environ, OUT2=str(tmp_path / "two.pt"))
    port = str(29500 + os.getpid() % 500)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", port, str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0
    two = torch.load(tmp_path / "two.pt")
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDPOPolicy
    c = O.TINY
    pol = LlavaDPOPolicy(_dims(c), DEV, hf_state=O.make_params(c, seed=0, scale=0.4))
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, optim="adamw_8bit")
    batch = O.synthetic_pair_batch(c, 4, 24, 20, seed=5, image_pos=7, ragged=True)
    batch["ref_win_logp"] = torch.tensor([-60.0, -70.0, -65.0, -62.0])
    batch["ref_rej_logp"] = torch.tensor([-61.0, -69.0, -64.0, -63.0])
    batch["beta"] = 0.1
    for _ in range(2):
        m = eng.train_step(batch)
    eng.opt.wait_all()
    torch.cuda.synchronize()
    loss1 = eng.metrics_dict(m)["loss"]
    flat1 = pol.store.flat.float().cpu()
    assert abs(two["loss"] - loss1) <= 1e-3 * abs(loss1)
    assert float((two["flat"] - flat1).norm() / flat1.norm()) <= 1e-3
