"""CPU tests of AdamW with blockwise 8-bit moments (optim="adamw_8bit"): the two code maps, the reference quantizer,
the block layout of the owned slices, the exact state size and the memory plans it gives, and the path from
--optim adamw_bnb_8bit / adamw_8bit to the optimizer in a dry run against a recording stand-in for the C ABI."""
import ctypes
import hashlib
from contextlib import nullcontext
from types import SimpleNamespace

import pytest
import torch

from oracle import adamw8bit_oracle as Q
from oracle import llava_dpo_oracle as O

MEMINFO = "MemTotal: 2113470464 kB\nMemAvailable: %d kB\n"


def test_dynamic_maps_are_pinned():
    from rlaifv_b200.zero2 import dynamic_map
    for signed, sha, lo in ((True, "e732639a65f497b4", -0.99296875), (False, "305f002cc11278fb", 0.0)):
        m = dynamic_map(signed)
        assert m.dtype == torch.float32 and m.numel() == 256
        assert bool((m[1:] > m[:-1]).all())
        assert hashlib.sha256(m.numpy().tobytes()).hexdigest().startswith(sha)
        assert float(m[0]) == float(torch.tensor(lo, dtype=torch.float32)) and float(m[-1]) == 1.0
    assert float(dynamic_map(True)[127]) == 0.0          # the code of 0 a fresh exp_avg holds
    assert float(dynamic_map(False)[0]) == 0.0


@pytest.mark.parametrize("signed", [True, False])
def test_oracle_round_trip_within_half_the_local_gap(signed):
    """Quantize -> dequantize moves each element by at most half the map gap next to its code, times the absmax."""
    qmap = Q.maps()[0 if signed else 1]
    g = torch.Generator().manual_seed(3)
    n = 256 * 40 + 72                                    # a partial last block
    x = torch.randn(n, generator=g) * torch.logspace(-6, 2, n)[torch.randperm(n, generator=g)]
    x = x if signed else x * x
    x[256:512] = 0.0                                     # an all-zero block
    x[512:768] = 0.0
    x[600] = -3.5 if signed else 3.5                     # a single non-zero
    am = Q.block_absmax(x.abs(), n)
    codes = Q.quantize_blocks(x, am, qmap)
    back = Q.dequantize(codes, am, qmap)
    c = codes.long()
    gap = torch.maximum(qmap[(c + 1).clamp(max=255)] - qmap[c], qmap[c] - qmap[(c - 1).clamp(min=0)])
    scale = am.repeat_interleave(256)[:n]
    # slack: the fp32 map's outermost signed entry lies 4e-6 (relative) beyond half its gap from -1, and the dequantized
    # product rounds once (at most half an ulp of absmax)
    assert bool(((back - x).abs() <= 0.5 * gap * scale * (1 + 1e-5) + scale * 2.0 ** -24).all())
    assert bool((back[256:512] == 0).all()) and int(codes[600]) == (0 if signed else 255)
    assert int(codes[256]) == (127 if signed else 0)     # a zero absmax stores the code of 0


def test_oracle_quantizer_ties_go_to_the_lower_code():
    qmap = Q.maps()[1]
    mids = (qmap[:-1] + qmap[1:]) / 2
    exact = (mids - qmap[:-1]) == (qmap[1:] - mids)      # midpoints that are exact ties in fp32
    codes = Q.quantize(mids[exact], qmap)
    assert exact.any() and bool((codes == torch.nonzero(exact).flatten()).all())
    assert bool((Q.quantize(qmap, qmap) == torch.arange(256)).all())
    assert int(Q.quantize(torch.tensor([-1.0]), Q.maps()[0])) == 0


def _fake_buckets(sizes):
    from rlaifv_b200.zero2 import OptBucket
    return [OptBucket("b%d" % i, torch.zeros(n, dtype=torch.bfloat16), torch.zeros(n, dtype=torch.bfloat16), n - 8)
            for i, n in enumerate(sizes)]


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_block_layout_per_slice(monkeypatch, world):
    """Blocks are counted from each owned slice's start, one table entry per slice; the last block of a slice may be
    partial. Bucket sizes are multiples of 1024, so at world <= 4 every slice edge is a block edge and the blocks
    cover each bucket exactly as at world 1."""
    from rlaifv_b200.zero2 import Zero2AdamW, n_blocks, state_bytes
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: None)
    sizes = [1024 * 3, 1024 * 5, 1024, 1024 * 9]
    cover_w1 = {}
    for rank in range(world):
        opt = Zero2AdamW(_fake_buckets(sizes), rank=rank, world=world, optim="adamw_8bit")
        total = 0
        for (b, s0, s1, o), q in zip(opt.slices, opt.block_offsets):
            n = s1 - s0
            assert q == total and n == b.size // world
            total += n_blocks(n)
            for k in range(n_blocks(n)):
                cover_w1.setdefault(b.name, []).append((s0 + 256 * k, min(s1, s0 + 256 * (k + 1))))
        assert opt.owned_blocks == total == opt.absmax.numel() == opt.absmax_sq.numel()
        assert opt.exp_avg_q.numel() == opt.owned and opt.exp_avg_q.dtype == torch.uint8
        assert bool((opt.exp_avg_q == 127).all()) and bool((opt.exp_avg_sq_q == 0).all())
        assert opt.state_nbytes == sum(state_bytes(s1 - s0, "adamw_8bit") for _, s0, s1, _ in opt.slices)
    for b, n in zip(_fake_buckets(sizes), sizes):
        blocks = sorted(cover_w1[b.name])
        world1 = [(256 * k, min(n, 256 * (k + 1))) for k in range(n_blocks(n))]
        assert (blocks == world1) == (world <= 4 or n % (256 * world) == 0)
        if world == 8 and n == 1024:     # 1024 / 8 = 128: each rank's slice is one partial block
            assert blocks == [(128 * r, 128 * (r + 1)) for r in range(8)]


def test_state_bytes_and_formats():
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM, state_bytes, state_format, state_parts
    assert state_bytes(1024) == STATE_BYTES_PER_ELEM * 1024 == state_bytes(1024, "adamw_torch")
    assert state_bytes(256, "adamw_8bit") == 256 * 6 + 8
    assert state_bytes(264, "adamw_8bit") == 264 * 6 + 16           # a partial block still has both scales
    assert state_bytes(8 << 20, "adamw_8bit") / (8 << 20) == pytest.approx(6.03125)
    with pytest.raises(ValueError, match="adamw_8bit"):
        state_bytes(8, "adamw_4bit")
    assert [k for k, _, _ in state_parts("adamw_8bit")] == ["master", "exp_avg_q", "exp_avg_sq_q", "absmax",
                                                            "absmax_sq"]
    assert state_format("adamw_bnb_8bit") == state_format("adamw_8bit") == "adamw_8bit"
    for other in ("adamw_torch", "adamw_hf", "adafactor", "sgd"):
        assert state_format(other) == "adamw_torch"


def _plan(d, pairs, optim):
    from rlaifv_b200.model import ParamStore
    from rlaifv_b200.zero2 import (DEFAULT_SLOT_ELEMS, DEFAULT_SLOTS, DEVICE_MARGIN, activation_reserve_bytes,
                                   offload_plan, ring_bytes, ring_slot_elems, state_bytes)
    store = ParamStore(d, "meta")
    sizes = [(b.name, b.size) for b in store.buckets]
    n_of = dict(sizes)
    free = 80 * 10 ** 9 - 2 * 2 * store.numel                              # bf16 weights + bf16 gradients
    reserve = activation_reserve_bytes(d, pairs, d.max_len) + 4 * d.vocab_size * d.hidden_size
    ring = ring_bytes(DEFAULT_SLOTS, ring_slot_elems(max(n_of.values()), DEFAULT_SLOT_ELEMS, optim), optim)
    budget = free - reserve - ring - DEVICE_MARGIN
    resident, streamed = offload_plan(sizes, budget, optim)
    assert sorted(resident + streamed) == sorted(n_of)
    dev = sum(state_bytes(n_of[k], optim) for k in resident)
    host = sum(state_bytes(n_of[k], optim) for k in streamed)
    assert dev <= budget
    return store, ring, budget, resident, dev, host


def test_13b_full_ft_plan_with_8bit_moments():
    """13B full fine-tuning, 1 pair at 2048 tokens, on an 80 GB card: 78.7 GB of state instead of 156.6 GB. Four
    buckets (5.0 GB) stay on the device and 73.7 GB is streamed, so MemAvailable must show 82.3 GB instead of 162.8."""
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.zero2 import HOST_MARGIN, check_host_memory
    d = LlavaDims(hidden_size=5120, intermediate_size=13824, num_layers=40, num_heads=40)
    store, ring, budget, resident, dev, host = _plan(d, 1, "adamw_8bit")
    assert ring == 151_781_376 and budget == 5_366_951_936
    assert resident == ["embed", "projector", "layer0", "layer1"]
    assert (dev, host) == (5_004_227_520, 73_687_492_640)
    assert dev + host == 78_691_720_160
    assert round((host + HOST_MARGIN) / 1e9, 1) == 82.3
    need_kb = (host + HOST_MARGIN) // 1024
    assert check_host_memory(host, MEMINFO % (need_kb + 1)) == (need_kb + 1) * 1024
    assert check_host_memory(host, MEMINFO % (101_300_000_000 // 1024))      # the 101.3 GB host
    with pytest.raises(MemoryError, match="73.69 GB of pinned host memory"):
        check_host_memory(host, MEMINFO % (need_kb - 1))
    # the fp32 plan at the same budget rule is the one test_llava13b_host pins
    _, _, _, res32, dev32, host32 = _plan(d, 1, "adamw_torch")
    assert res32 == ["embed", "projector"] and host32 == 154_224_291_840


def test_7b_config_b_plan_with_8bit_moments():
    """7B full fine-tuning with micro-batches of 2 pairs at 2048 tokens: 23.7 GB resident / 57.4 GB streamed with fp32
    moments, 24.1 / 16.7 GB (21 buckets resident) with 8-bit moments."""
    from rlaifv_b200.model import LlavaDims
    d = LlavaDims(max_len=2048)
    _, _, _, res32, dev32, host32 = _plan(d, 2, "adamw_torch")
    _, _, _, res8, dev8, host8 = _plan(d, 2, "adamw_8bit")
    assert (len(res32), dev32, host32) == (11, 23_682_023_424, 57_430_720_512)
    assert (len(res8), dev8, host8) == (21, 24_108_930_048, 16_658_673_024)


# ---- dry run of the engine's optimizer step against a recording C ABI ----
class _FakeStream:
    cuda_stream = 0

    def __init__(self, *a, **k):
        pass

    def wait_event(self, ev):
        pass

    def wait_stream(self, s):
        pass

    def synchronize(self):
        pass


class _FakeEvent:
    def __init__(self, *a, **k):
        pass

    def record(self, stream=None):
        pass


class _FakeCudart:
    def __init__(self):
        self.registered = {}

    def cudaHostRegister(self, ptr, size, flags):
        self.registered[ptr] = size
        return 0

    def cudaHostUnregister(self, ptr):
        self.registered.pop(ptr)
        return 0


def _tiny_policy():
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    return c, dims, LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))


@pytest.mark.parametrize("hf_optim", ["adamw_bnb_8bit", "adamw_8bit", "adamw_torch"])
def test_optim_flag_reaches_the_optimizer_dry_run(monkeypatch, hf_optim):
    """LLaVA15DPOTrainer maps --optim to the state format. With 8-bit moments, resident buckets get one
    rlaifv_adamw8bit_step per bucket and streamed ones rlaifv_adamw8bit_offload_bucket, head first; adamw_torch
    builds today's optimizer and calls today's entry points."""
    from rlaifv_b200 import lib, ops, trainers
    from rlaifv_b200.train_llava15 import parse_args_into_dataclasses
    from rlaifv_b200.zero2 import OffloadAdamW, adamw8bit_slot_bytes, state_bytes
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append((name, args))

    cudart = _FakeCudart()
    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    monkeypatch.setattr(torch.cuda, "Stream", _FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _FakeStream())
    monkeypatch.setattr(torch.cuda, "stream", lambda s: nullcontext())
    monkeypatch.setattr(torch.cuda, "cudart", lambda: cudart)
    monkeypatch.setattr("rlaifv_b200.zero2._read_meminfo", lambda: MEMINFO % (1 << 40))

    _, _, training_args = parse_args_into_dataclasses(["--optim", hf_optim, "--output_dir", "unused"])
    assert training_args.optim == hf_optim
    c, dims, pol = _tiny_policy()
    fmt = "adamw_torch" if hf_optim == "adamw_torch" else "adamw_8bit"
    sizes = {b.name: b.size for b in pol.trainable_buckets()}
    budget = sum(state_bytes(sizes[k], fmt) for k in ("embed", "projector", "layer0"))
    real_engine = trainers.DPOStepEngine
    monkeypatch.setattr(trainers, "DPOStepEngine",
                        lambda policy, **kw: real_engine(policy, **dict(kw, offload_budget=budget)))
    args = SimpleNamespace(learning_rate=1e-4, weight_decay=0.01, max_steps=10, warmup_ratio=0.0,
                           dpo_use_average=False, per_device_train_batch_size=2, offload_optimizer=True,
                           optim=training_args.optim)
    eng = trainers.LLaVA15DPOTrainer(model=SimpleNamespace(policy=pol), args=args).engine
    opt = eng.opt
    assert isinstance(opt, OffloadAdamW) and opt.optim == fmt
    assert opt.resident_names == ["embed", "projector", "layer0"]
    if fmt == "adamw_8bit":
        assert opt.slot_elems % 256 == 0
        assert opt.ring.dtype == torch.uint8 and opt.ring.shape == (3, adamw8bit_slot_bytes(opt.slot_elems))
        assert len(cudart.registered) == 5
        assert opt.pinned_bytes == sum(state_bytes(sizes[k], fmt) for k in opt.streamed_names)
    else:
        assert opt.ring.dtype == torch.float32 and len(cudart.registered) == 3

    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    monkeypatch.setattr(pol, "splice", lambda ids, labels, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), torch.full((4, T), -100),
        torch.zeros(4, T, dtype=torch.int32), T))
    opt.begin_step(1e-4)
    eng._stepping, eng._last_micro = True, True
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    calls.clear()
    pol.backward_logps(torch.zeros(4))
    pol.finalize_embed_grad()
    opt.finish_step()
    names = [n for n, _ in calls]
    nl = dims.num_layers
    if fmt == "adamw_8bit":
        assert "rlaifv_adamw_step" not in names and "rlaifv_adamw_offload_bucket" not in names
        assert names.count("rlaifv_adamw8bit_step") == 3                     # one launch per resident slice
        off = [a for n, a in calls if n == "rlaifv_adamw8bit_offload_bucket"]
        assert [a[7] for a in off] == [sizes["head"]] + [sizes["layer%d" % i] for i in reversed(range(1, nl))]
        head_b = pol.store.buckets[[b.name for b in pol.store.buckets].index("head")]
        assert off[0][8] == head_b.decay_size
        assert all(a[12] == 3 and a[13] == opt.slot_elems and a[19] == 1 for a in off)
        sd = opt.state_dict()
        assert sd["optim"] == "adamw_8bit" and sd["block"] == 256
        assert set(sd) == {"step", "optim", "block", "master", "exp_avg_q", "exp_avg_sq_q", "absmax", "absmax_sq",
                           "rank", "world"}
        assert sd["absmax"].numel() == opt.owned_blocks and sd["exp_avg_q"].numel() == opt.owned
    else:
        assert "rlaifv_adamw8bit_step" not in names and "rlaifv_adamw8bit_offload_bucket" not in names
        assert len([n for n in names if n == "rlaifv_adamw_offload_bucket"]) == nl
        sd = opt.state_dict()
        assert set(sd) == {"step", "master", "exp_avg", "exp_avg_sq", "rank", "world"}
    opt.close()
    assert not cudart.registered


def test_cross_format_checkpoint_is_refused(monkeypatch):
    from rlaifv_b200.zero2 import Zero2AdamW
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: None)
    sizes = [2048, 1024]
    o8 = Zero2AdamW(_fake_buckets(sizes), optim="adamw_8bit")
    o32 = Zero2AdamW(_fake_buckets(sizes))
    with pytest.raises(ValueError, match="adamw_torch state.*adamw_8bit state"):
        o8.load_state_dict(o32.state_dict())
    with pytest.raises(ValueError, match="adamw_8bit state.*adamw_torch state"):
        o32.load_state_dict(o8.state_dict())
    with pytest.raises(ValueError, match="adamw_4bit"):
        Zero2AdamW(_fake_buckets(sizes), optim="adamw_4bit")
    o8.load_state_dict(o8.state_dict())
