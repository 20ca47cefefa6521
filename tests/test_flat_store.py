"""CPU tests of the flat bucketed parameter store (model.FlatStore) that the decoder, the LoRA adapters, the EVA tower
and the resampler share: bucket sizes and decay boundaries at the real widths against hand arithmetic, the named views
aliasing the flat buffers, the stacked LoRA B operands, and a store without gradients."""
import math

import torch

META = torch.device("meta")
PAD = 1024


def _pad(n):
    return -(-n // PAD) * PAD


def _sizes(store):
    return [(b.name, b.size, b.decay_size) for b in store.buckets]


def test_llava_7b_layout():
    from rlaifv_b200.model import LlavaDims, ParamStore
    st = ParamStore(LlavaDims(), META)
    H, F, V, C = 4096, 11008, 32000, 1024
    layer_decay = 3 * H * H + H * H + 2 * F * H + H * F
    assert layer_decay == 202_375_168 and _pad(layer_decay + 2 * H) == 202_383_360
    assert _sizes(st) == ([("embed", V * H, V * H)] + [(f"layer{i}", 202_383_360, 202_375_168) for i in range(32)]
                          + [("head", _pad(V * H + H), V * H), ("projector", _pad(H * C + H * H + 2 * H), H * C + H * H)])
    assert len(st.buckets) == 35 and st.numel == st.flat.numel() == 6_759_395_328
    assert [b.start for b in st.buckets] == [sum(b.size for b in st.buckets[:i]) for i in range(35)]


def test_omnilmm_decoder_layout():
    from rlaifv_b200.model import ParamStore
    from rlaifv_b200.omnilmm_model import omnilmm_dims
    st = ParamStore(omnilmm_dims(), META)
    H, KV, F, V = 4096, 1024, 14336, 32008
    layer_decay = (H + 2 * KV) * H + H * H + 2 * F * H + H * F
    assert _sizes(st) == ([("embed", V * H, V * H)] + [(f"layer{i}", _pad(layer_decay + 2 * H), layer_decay)
                                                       for i in range(32)] + [("head", _pad(V * H + H), V * H)])
    assert len(st.buckets) == 34 and st.numel == 7_241_797_632


def test_lora_r64_layout_and_stacked_b_views():
    from rlaifv_b200.model import LlavaDims, LoraStore
    H, F, r = 4096, 11008, 64
    st = LoraStore(LlavaDims(num_layers=2), "cpu", r=r, init_b_zero=False)
    per_layer = 3 * r * H + 3 * H * r + r * H + H * r + 2 * r * H + 2 * F * r + r * F + H * r
    assert per_layer == 4_997_120 == _pad(per_layer)
    assert _sizes(st) == [("lora0", per_layer, per_layer), ("lora1", per_layer, per_layer)]
    assert 32 * per_layer == 159_907_840                  # bench.py's LoRA parameter count at 32 layers
    assert all(s.decay for b in st.buckets for s in b.segments)
    st.grad.copy_(torch.randn(st.numel, generator=torch.Generator().manual_seed(0)))
    for i in range(2):
        for src, base in ((st.p, st.flat), (st.g, st.grad)):
            assert src[f"l{i}.B_qkv"].shape == (3 * H, r) and src[f"l{i}.B_gu"].shape == (2 * F, r)
            assert torch.equal(src[f"l{i}.B_qkv"], torch.cat([src[f"l{i}.B_{x}"] for x in "qkv"]))
            assert torch.equal(src[f"l{i}.B_gu"], torch.cat([src[f"l{i}.B_{x}"] for x in "gu"]))
            assert src[f"l{i}.B_qkv"].storage_offset() == src[f"l{i}.B_q"].storage_offset()
            assert src[f"l{i}.B_gu"].storage_offset() == src[f"l{i}.B_g"].storage_offset()
            assert src[f"l{i}.B_o_cat"] is src[f"l{i}.B_o"] and src[f"l{i}.B_d_cat"] is src[f"l{i}.B_d"]
            b_g = src[f"l{i}.B_g"].clone()
            src[f"l{i}.B_gu"][F:].fill_(5.0)               # writes through the stacked view land in B_u only
            assert bool((src[f"l{i}.B_u"] == 5.0).all()) and torch.equal(src[f"l{i}.B_g"], b_g)
            assert src[f"l{i}.B_qkv"].untyped_storage().data_ptr() == base.untyped_storage().data_ptr()


def test_resampler_layout():
    from rlaifv_b200.resampler import Resampler
    rs = Resampler(8, 4096, 32, 1792, META)
    E, kv, Q = 4096, 1792, 64
    decay = Q * E + E * E + E * kv + 3 * E * E + E * E
    assert decay == 91_488_256
    assert _sizes(rs) == [("resampler", 91_529_216, decay)] and rs.numel == _pad(decay + 3 * E + E + 6 * E)
    [b] = rs.opt_buckets()
    assert (b.name, b.size, b.decay_size) == ("resampler", rs.numel, decay)


def test_eva_tower_layout(monkeypatch):
    from rlaifv_b200.eva_tower import EvaDims, EvaTower
    monkeypatch.setattr(EvaTower, "_random_init", lambda self, seed: None)
    tower = EvaTower(EvaDims(depth=3), META)
    C, Hd, HP = 1792, 15360, 16 * 128
    embed_decay = C * 640 + C + 264 * C                   # patch 3*14*14 = 588 -> 640, 1 + 16*16 = 257 -> 264 positions
    block_decay = 3 * HP * C + C * HP + Hd * C + C * Hd
    block_tail = 3 * HP + C + 2 * C + Hd + C + 2 * C
    assert _pad(embed_decay + 3 * C) == 1_627_136 and _pad(block_decay + block_tail) == 69_763_072
    assert _sizes(tower) == [("eva_embed", 1_627_136, embed_decay), ("eva0", 69_763_072, block_decay),
                             ("eva1", 69_763_072, block_decay)]
    assert tower.numel == 141_153_280


def _small_store(grads):
    from rlaifv_b200.model import FlatStore
    return FlatStore([("a", [("w", (24, 8)), ("v", (5, 8))], [("b", (7,))]), ("c", [], [("n", (3,))])], "cpu",
                     grads=grads)


def test_views_alias_the_flat_buffers_in_segment_order():
    st = _small_store(grads=True)
    assert _sizes(st) == [("a", PAD, 232), ("c", PAD, 0)] and st.numel == 2 * PAD
    segs = [s for b in st.buckets for s in b.segments]
    assert [s.name for s in segs] == list(st.p) == list(st.g) == ["w", "v", "b", "n"]
    assert [(s.offset, s.decay) for s in segs] == [(0, True), (192, True), (232, False), (PAD, False)]
    for views, base in ((st.p, st.flat), (st.g, st.grad)):
        base.copy_(torch.arange(st.numel) % 251)
        for s in segs:
            v = views[s.name]
            assert v.untyped_storage().data_ptr() == base.untyped_storage().data_ptr()
            assert v.storage_offset() == s.offset and tuple(v.shape) == s.shape
            assert torch.equal(v.reshape(-1), base[s.offset:s.offset + math.prod(s.shape)])
    ob = st.opt_buckets()
    assert [(b.name, b.size, b.decay_size, b.flat.storage_offset()) for b in ob] == [("a", PAD, 232, 0),
                                                                                    ("c", PAD, 0, PAD)]
    assert ob[1].grad.untyped_storage().data_ptr() == st.grad.untyped_storage().data_ptr()
    assert [b.name for b in st.opt_buckets(names={"c"})] == ["c"]
    st.zero_grad()
    assert not bool(st.grad.any()) and bool(st.flat.any())


def test_store_without_gradients():
    st = _small_store(grads=False)
    assert st.grad is None and st.g == {} and st.opt_buckets() == [] and list(st.p) == ["w", "v", "b", "n"]
    st.zero_grad()
