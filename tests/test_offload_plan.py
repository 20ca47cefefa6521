"""CPU tests of the offloaded optimizer's host side: the resident / streamed planner, the chunking of a streamed bucket,
the host-memory refusal, the DeepSpeed `offload_optimizer` parsing, and a dry run of the engine's optimizer step against
a recording stand-in for the C ABI."""
import ctypes
import json
from contextlib import nullcontext

import pytest
import torch

from oracle import llava_dpo_oracle as O

NAMES = ["embed"] + ["layer%d" % i for i in range(4)] + ["head", "projector"]


def test_priority_order():
    from rlaifv_b200.zero2 import offload_priority
    assert offload_priority(NAMES) == ["embed", "projector", "layer0", "layer1", "layer2", "layer3", "head"]
    # layer numbers sort numerically, not as strings
    names = ["layer%d" % i for i in (10, 2, 1)] + ["head"]
    assert offload_priority(names) == ["layer1", "layer2", "layer10", "head"]


@pytest.mark.parametrize("budget_elems,resident", [
    (0, []),
    (99, []),
    (100, ["embed"]),
    (100 + 10, ["embed", "projector"]),
    (100 + 10 + 50 * 2, ["embed", "projector", "layer0", "layer1"]),
    (100 + 10 + 50 * 2 + 49, ["embed", "projector", "layer0", "layer1"]),
    (100 + 10 + 50 * 4, ["embed", "projector", "layer0", "layer1", "layer2", "layer3"]),
    (10 ** 9, ["embed", "projector", "layer0", "layer1", "layer2", "layer3", "head"]),
])
def test_plan_split(budget_elems, resident):
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM, offload_plan
    sizes = [("embed", 100)] + [("layer%d" % i, 50) for i in range(4)] + [("head", 100), ("projector", 10)]
    res, streamed = offload_plan(sizes, budget_elems * STATE_BYTES_PER_ELEM)
    assert res == resident
    # the streamed buckets are the rest, the first to become final first: head, layer3, layer2, ...
    assert streamed == [n for n in ["embed", "projector", "layer0", "layer1", "layer2", "layer3", "head"]
                        if n not in resident]
    assert sorted(res + streamed) == sorted(n for n, _ in sizes)


@pytest.mark.parametrize("n,slot,decay", [(13288, 4096, 4596), (4096, 4096, 4096), (4100, 4096, 0),
                                          (1 << 20, 1000, (1 << 20) - 4), (8, 4, 5)])
def test_chunks_cover_once_and_decay_boundary(n, slot, decay):
    from rlaifv_b200.zero2 import offload_chunks
    ch = offload_chunks(n, slot, decay)
    covered = torch.zeros(n, dtype=torch.int32)
    decayed = torch.zeros(n, dtype=torch.bool)
    for off, c, dn in ch:
        assert 0 < c <= slot and 0 <= dn <= c
        covered[off:off + c] += 1
        decayed[off:off + dn] = True
    assert bool((covered == 1).all())                     # every element exactly once
    assert bool(decayed[:decay].all()) and not bool(decayed[decay:].any())
    straddling = [x for x in ch if 0 < x[2] < x[1]]
    assert len(straddling) == (1 if decay % slot and 0 < decay < n else 0)   # the boundary chunk is one launch


MEMINFO = """MemTotal:       2113470464 kB
MemFree:         1500000000 kB
MemAvailable:    %d kB
Buffers:            1234 kB
"""


def test_host_memory_refusal():
    from rlaifv_b200.zero2 import check_host_memory, mem_available_bytes
    assert mem_available_bytes(MEMINFO % 1000) == 1024000
    gb = 1 << 30
    assert check_host_memory(40 * gb, MEMINFO % (60 * gb // 1024), margin=8 * gb) == 60 * gb
    with pytest.raises(MemoryError, match="MemAvailable"):
        check_host_memory(40 * gb, MEMINFO % (45 * gb // 1024), margin=8 * gb)
    with pytest.raises(MemoryError):
        check_host_memory(1, "MemTotal: 5 kB\n")


def test_offload_refuses_before_pinning(monkeypatch):
    """The refusal happens before any host buffer is allocated or registered."""
    from rlaifv_b200 import zero2
    registered = []
    monkeypatch.setattr(zero2.OffloadAdamW, "_register", lambda self, t: registered.append(t))
    monkeypatch.setattr(torch.cuda, "Stream", lambda device=None: None)
    b = zero2.OptBucket("layer0", torch.zeros(1024, dtype=torch.bfloat16), torch.zeros(1024, dtype=torch.bfloat16), 1000)
    with pytest.raises(MemoryError):
        zero2.OffloadAdamW([b], device_budget=0, host_margin=0, meminfo=lambda: MEMINFO % 1)
    assert not registered
    with pytest.raises(NotImplementedError):
        zero2.OffloadAdamW([b], world=2, device_budget=0)


def test_deepspeed_offload_parsing(tmp_path):
    from rlaifv_b200.train_llava15 import offload_optimizer, zero_stage
    import os
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    assert offload_optimizer(os.path.join(repo, "script", "zero2_offload.json")) is True
    assert zero_stage(os.path.join(repo, "script", "zero2_offload.json")) == 2
    assert offload_optimizer(os.path.join(repo, "script", "zero2.json")) is False
    assert offload_optimizer(None) is False

    def cfg(block):
        p = tmp_path / ("c%d.json" % len(list(tmp_path.iterdir())))
        z = {"stage": 2}
        if block is not None:
            z["offload_optimizer"] = block
        p.write_text(json.dumps({"zero_optimization": z}))
        return str(p)
    assert offload_optimizer(cfg({"device": "cpu", "pin_memory": True})) is True
    assert offload_optimizer(cfg({"device": "none"})) is False
    assert offload_optimizer(cfg(None)) is False
    with pytest.raises(NotImplementedError):
        offload_optimizer(cfg({"device": "nvme", "nvme_path": "/local_nvme"}))


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

    def synchronize(self):
        pass


class _FakeCudart:
    def __init__(self):
        self.registered = set()

    def cudaHostRegister(self, ptr, size, flags):
        self.registered.add(ptr)
        return 0

    def cudaHostUnregister(self, ptr):
        self.registered.discard(ptr)
        return 0


def test_engine_offload_dry_run(monkeypatch):
    """One optimizer step of the engine with offload on, against the recording C ABI: resident buckets go through
    rlaifv_adamw_step, streamed ones through rlaifv_adamw_offload_bucket with an argument count that matches the ctypes
    table, in the order their gradients become final (head first)."""
    from rlaifv_b200 import lib, ops
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    from rlaifv_b200.zero2 import STATE_BYTES_PER_ELEM, OffloadAdamW
    c = O.TINY
    dims = LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size)
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name       # argument count matches the ctypes table
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
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    sizes = {b.name: b.size for b in pol.trainable_buckets()}
    budget = STATE_BYTES_PER_ELEM * (sizes["embed"] + sizes["projector"] + sizes["layer0"])
    monkeypatch.setattr("rlaifv_b200.zero2._read_meminfo", lambda: MEMINFO % (1 << 40))
    eng = DPOStepEngine(pol, offload_optimizer=True, offload_budget=budget)
    opt = eng.opt
    assert isinstance(opt, OffloadAdamW)
    nl = dims.num_layers
    assert opt.resident_names == ["embed", "projector", "layer0"]
    assert opt.streamed_names == ["layer%d" % i for i in range(1, nl)] + ["head"]
    assert opt.master.numel() == budget // STATE_BYTES_PER_ELEM
    assert opt.host_master.numel() == sum(sizes[n] for n in opt.streamed_names)
    assert len(cudart.registered) == 3 and opt.pinned_bytes == STATE_BYTES_PER_ELEM * opt.host_master.numel()
    # the host master holds the initial parameters of the streamed buckets
    b_head = opt.buckets[opt.index["head"]]
    o_head = opt.slices[opt.index["head"]][3]
    assert torch.equal(opt.host_master[o_head:o_head + b_head.size], b_head.flat.float())

    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    monkeypatch.setattr(pol, "splice", lambda ids, labels, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, dims.hidden_size, dtype=torch.bfloat16), torch.full((4, T), -100),
        torch.zeros(4, T, dtype=torch.int32), T))
    # the engine's step, as _train_step drives it: begin_step, backward with the per-bucket hooks, finish_step
    opt.begin_step(1e-4)
    eng._stepping, eng._last_micro = True, True
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    calls.clear()
    pol.backward_logps(torch.zeros(4))
    pol.finalize_embed_grad()
    opt.finish_step()
    off = [a for n, a in calls if n == "rlaifv_adamw_offload_bucket"]
    assert len(off) == nl                                   # layers 1..nl-1 and the head
    assert [a[5] for a in off] == [sizes["head"]] + [sizes["layer%d" % i] for i in reversed(range(1, nl))]
    head_b = pol.store.buckets[[b.name for b in pol.store.buckets].index("head")]
    assert off[0][6] == head_b.decay_size                  # decay boundary handed through
    assert all(a[8] == 3 and a[15] == 1 for a in off)      # 3 ring slots, step 1
    # resident buckets: the unchanged on-device path (decay + no-decay launch per bucket with a no-decay tail)
    adam = [n for n, _ in calls if n == "rlaifv_adamw_step"]
    assert 3 <= len(adam) <= 6
    sd = opt.state_dict()
    assert sd["master"].numel() == opt.owned and not sd["master"].is_cuda
    assert set(sd) == {"step", "master", "exp_avg", "exp_avg_sq", "rank", "world"}
    g_head = opt._global[opt.index["head"]]
    assert torch.equal(sd["master"][g_head:g_head + b_head.size], opt.host_master[o_head:o_head + b_head.size])
    n_calls = len(calls)
    opt.close()
    assert not cudart.registered
    # close() hands the ring's events back to the library, once
    assert [n for n, _ in calls[n_calls:]] == ["rlaifv_adamw_offload_release"] and opt.ring is None
    opt.close()
    assert len(calls) == n_calls + 1


def _tiny_dims():
    from rlaifv_b200.model import LlavaDims
    c = O.TINY
    return c, LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                        num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                        clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                        image_size=c.image_size, patch_size=c.patch_size)


@pytest.mark.parametrize("micro_pairs,batch_pairs,pairs", [(None, 1, 1), (None, 8, 8), (2, 8, 2), (3, None, 3)])
def test_engine_default_budget(monkeypatch, micro_pairs, batch_pairs, pairs):
    """Without an explicit budget the engine sizes the activation reserve from the micro-batch the step runs
    (micro_pairs, else the per-device batch) at dims.max_len, and plans against a faked mem_get_info."""
    from rlaifv_b200 import lib
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDPOPolicy
    from rlaifv_b200.zero2 import (DEFAULT_SLOT_ELEMS, DEFAULT_SLOTS, DEVICE_MARGIN, STATE_BYTES_PER_ELEM,
                                   activation_reserve_bytes, offload_plan)
    _fake_cuda(monkeypatch)
    c, dims = _tiny_dims()
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    sizes = [(b.name, b.size) for b in pol.trainable_buckets()]
    slot = min(DEFAULT_SLOT_ELEMS, max(n for _, n in sizes))
    ring = DEFAULT_SLOTS * 3 * slot * 4
    reserve = activation_reserve_bytes(dims, pairs, dims.max_len) + 4 * dims.vocab_size * dims.hidden_size
    # free memory that leaves room for exactly embed + projector + layer0 after the reserve, ring and margin
    n_of = dict(sizes)
    keep = STATE_BYTES_PER_ELEM * (n_of["embed"] + n_of["projector"] + n_of["layer0"])
    free = reserve + ring + DEVICE_MARGIN + keep
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (free, 80 << 30))
    eng = DPOStepEngine(pol, offload_optimizer=True, micro_pairs=micro_pairs, batch_pairs=batch_pairs)
    assert eng.opt.device_budget == keep
    assert eng.opt.resident_names == ["embed", "projector", "layer0"]
    assert (eng.opt.resident_names, eng.opt.streamed_names) == offload_plan(sizes, keep)
    eng.opt.close()


def test_engine_default_budget_needs_the_batch(monkeypatch):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDPOPolicy
    _fake_cuda(monkeypatch)
    c, dims = _tiny_dims()
    pol = LlavaDPOPolicy(dims, "cpu", hf_state=O.make_params(c, seed=0))
    with pytest.raises(ValueError, match="micro_pairs"):
        DPOStepEngine(pol, offload_optimizer=True)


def test_default_reserve_at_7b_widths():
    """At LLaVA-1.5-7B widths and the recipe's model_max_length 2048, the reserve for the shipped per-device batch of
    1 pair is ~12.5 GB, and for micro-batches of 2 pairs ~25 GB: both leave tens of GB of an 80 GB card for state."""
    from rlaifv_b200.model import LlavaDims
    from rlaifv_b200.zero2 import activation_reserve_bytes
    d = LlavaDims(max_len=2048)
    one, two = activation_reserve_bytes(d, 1, 2048), activation_reserve_bytes(d, 2, 2048)
    assert 12e9 < one < 13e9 and two == 2 * one


def test_trainer_passes_the_per_device_batch(monkeypatch):
    from types import SimpleNamespace
    from rlaifv_b200 import trainers
    seen = {}
    monkeypatch.setattr(trainers, "DPOStepEngine", lambda policy, **kw: seen.update(kw) or SimpleNamespace())
    args = SimpleNamespace(learning_rate=1e-6, weight_decay=0.0, max_steps=10, warmup_ratio=0.03,
                           dpo_use_average=False, per_device_train_batch_size=1, offload_optimizer=True)
    trainers.LLaVA15DPOTrainer(model=SimpleNamespace(policy=None), args=args)
    assert seen["offload_optimizer"] is True and seen["batch_pairs"] == 1 and seen["micro_pairs"] is None


def _fake_cuda(monkeypatch):
    from rlaifv_b200 import lib, ops
    monkeypatch.setattr(lib, "call", lambda name, *args: None)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    monkeypatch.setattr(torch.cuda, "Stream", _FakeStream)
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: _FakeStream())
    monkeypatch.setattr(torch.cuda, "cudart", lambda: _FakeCudart())
    monkeypatch.setattr("rlaifv_b200.zero2._read_meminfo", lambda: MEMINFO % (1 << 40))
