"""GPU tests of the offloaded AdamW (rlaifv_adamw_offload_bucket / zero2.OffloadAdamW): bit-identity with the on-device
optimizer at the kernel, bucket and whole-engine level, its device footprint, checkpoint interchange with Zero2AdamW,
and the entry point's rejection of pageable host memory."""
import pytest
import torch

from oracle import llava_dpo_oracle as O

pytestmark = pytest.mark.gpu

LR, B1, B2, EPS, WD = 1e-3, 0.9, 0.999, 1e-8, 0.01


def _state(n, seed, pinned):
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(n, generator=g)
    e = torch.randn(n, generator=g).abs() * 1e-3
    v = torch.randn(n, generator=g).square() * 1e-6
    out = [m, e, v]
    return [t.pin_memory() for t in out] if pinned else out


def test_entry_point_matches_adamw_step():
    """Three steps over a range that is not a multiple of the chunk, with the decay boundary inside a chunk."""
    from rlaifv_b200 import ops
    slot, n, decay = 4096, 4096 * 3 + 1000, 4096 + 500
    dev = "cuda:0"
    hm, hv1, hv2 = _state(n, 1, pinned=True)
    dm, dv1, dv2 = hm.to(dev), hv1.to(dev), hv2.to(dev)
    p_ref = hm.to(dev).bfloat16()
    p_off = p_ref.clone()
    ring = torch.empty((3, 3 * slot), dtype=torch.float32, device=dev)
    h2d, d2h = torch.cuda.Stream(), torch.cuda.Stream()
    g = torch.Generator(device=dev).manual_seed(7)
    for step in (1, 2, 3):
        grad = (torch.randn(n, generator=g, device=dev) * 1e-2).bfloat16()
        ops.adamw_step(dm[:decay], dv1[:decay], dv2[:decay], grad[:decay], p_ref[:decay], LR, B1, B2, EPS, WD, step)
        ops.adamw_step(dm[decay:], dv1[decay:], dv2[decay:], grad[decay:], p_ref[decay:], LR, B1, B2, EPS, 0.0, step)
        ops.adamw_offload_bucket(hm, hv1, hv2, grad, p_off, decay, ring, slot, LR, B1, B2, EPS, WD, step, h2d, d2h)
        torch.cuda.synchronize()
    assert torch.equal(p_off, p_ref)
    assert torch.equal(hm, dm.cpu()) and torch.equal(hv1, dv1.cpu()) and torch.equal(hv2, dv2.cpu())


def test_entry_point_rejects_pageable_host_memory():
    from rlaifv_b200 import lib, ops
    n, slot = 4096, 1024
    hm, hv1, hv2 = _state(n, 2, pinned=False)
    grad = torch.zeros(n, dtype=torch.bfloat16, device="cuda:0")
    p = torch.zeros_like(grad)
    ring = torch.empty((3, 3 * slot), dtype=torch.float32, device="cuda:0")
    with pytest.raises(lib.B200Error, match="pinned host"):
        ops.adamw_offload_bucket(hm, hv1, hv2, grad, p, n, ring, slot, LR, B1, B2, EPS, WD, 1,
                                 torch.cuda.Stream(), torch.cuda.Stream())
    torch.cuda.synchronize()


# ---- whole engine -------------------------------------------------------------------------------------------------
def _dims():
    from rlaifv_b200.model import LlavaDims
    c = O.TINY
    return c, LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                        num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                        clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                        image_size=c.image_size, patch_size=c.patch_size)


def _engine(offload=None, slot_elems=None):
    """Tiny LLaVA engine, micro_pairs 1 < B = 2. offload: None (Zero2AdamW) or a device budget in bytes."""
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDPOPolicy
    from rlaifv_b200.zero2 import OffloadAdamW
    c, dims = _dims()
    pol = LlavaDPOPolicy(dims, "cuda:0", hf_state=O.make_params(c, seed=0, scale=0.4))
    eng = DPOStepEngine(pol, lr=1e-3, total_steps=10, constant_lr=True, micro_pairs=1,
                        offload_optimizer=offload is not None and slot_elems is None, offload_budget=offload)
    if slot_elems is not None:            # small ring slots: several chunks per bucket
        eng.opt = OffloadAdamW(pol.trainable_buckets(), lr=1e-3, gather_order=pol.param_need_order(),
                               device_budget=offload, slot_elems=slot_elems)
        pol.param_ready = eng.opt.wait_bucket
    return eng


def _batch(step):
    c = O.TINY
    batch = O.synthetic_pair_batch(c, 2, 24, 20, seed=5 + step, image_pos=7, ragged=True)
    batch["ref_win_logp"] = torch.tensor([-60.0, -70.0])
    batch["ref_rej_logp"] = torch.tensor([-61.0, -69.0])
    batch["beta"] = 0.1
    return batch


def _run(eng, steps, first=0):
    out = []
    for s in range(first, first + steps):
        out.append(eng.train_step(_batch(s)).clone())
    eng.opt.wait_all()
    torch.cuda.synchronize()
    return out


def _assert_same(e1, e2, m1=None, m2=None):
    if m1 is not None:
        for a, b in zip(m1, m2):
            assert torch.equal(a, b), (a, b)
    assert torch.equal(e1.policy.store.flat, e2.policy.store.flat)
    s1, s2 = e1.opt.state_dict(), e2.opt.state_dict()
    assert s1["step"] == s2["step"]
    for k in ("master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(s1[k].cpu(), s2[k].cpu()), k


def _sizes(eng):
    return {b.name: b.size for b in eng.policy.trainable_buckets()}


@pytest.mark.parametrize("split", ["mixed", "all_streamed"])
def test_engine_offload_bit_identical(split):
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    ref = _engine()
    sz = _sizes(ref)
    budget = STATE_BYTES_PER_ELEM * (sz["embed"] + sz["projector"] + sz["layer0"]) if split == "mixed" else 0
    off = _engine(offload=budget, slot_elems=None if split == "mixed" else 1 << 14)
    assert off.opt.streamed_names and (bool(off.opt.resident_names) == (split == "mixed"))
    if split == "all_streamed":
        assert max(sz.values()) > off.opt.slot_elems            # several chunks per bucket
    m_ref, m_off = _run(ref, 3), _run(off, 3)
    _assert_same(ref, off, m_ref, m_off)
    off.opt.close()


def test_offload_device_footprint_and_pinning():
    from rlaifv_b200.zero2 import OffloadAdamW
    eng = _engine()
    pol = eng.policy
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    opt = OffloadAdamW(pol.trainable_buckets(), device_budget=0, slot_elems=1 << 14)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    ring_bytes = opt.ring.numel() * 4
    assert opt.resident_names == [] and opt.master.numel() == 0
    assert grown <= ring_bytes + (1 << 20), (grown, ring_bytes)
    for t in (opt.host_master, opt.host_exp_avg, opt.host_exp_avg_sq):
        assert t.is_pinned() and t.numel() == opt.owned
    assert opt.pinned_bytes == 12 * opt.owned
    opt.close()
    assert not opt.host_master.is_pinned()


@pytest.mark.parametrize("direction", ["device_to_offload", "offload_to_device"])
def test_checkpoint_interchange(direction):
    """A state_dict written by one optimizer resumes with the other: after one more step on each, bit-identical."""
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM
    sz = _sizes(_engine())
    budget = STATE_BYTES_PER_ELEM * (sz["embed"] + sz["projector"])
    src = _engine() if direction == "device_to_offload" else _engine(offload=budget)
    _run(src, 2)
    dst = _engine(offload=budget) if direction == "device_to_offload" else _engine()
    dst.policy.store.flat.copy_(src.policy.store.flat)
    dst.opt.load_state_dict(src.opt.state_dict())
    dst.global_step = src.global_step
    torch.cuda.synchronize()
    m_src, m_dst = _run(src, 1, first=2), _run(dst, 1, first=2)
    _assert_same(src, dst, m_src, m_dst)
    for e in (src, dst):
        if hasattr(e.opt, "close"):
            e.opt.close()
