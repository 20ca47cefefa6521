"""-m gpu: shared prompt prefixes (a pair's rejected sequence reads the rows below pos0 from its chosen sequence).

Kernels: attention_varlen_prefix_fwd / bwd give the bits the fixed-length kernels give the pair laid out padded (O,
LSE and dQ at every own row, dK/dV at every row that is not shared); the shared rows' dK/dV, the sum of both copies'
gradients, is held to an fp64 reference with the bounds of test_gpu_kernel_bounds. Models: with share_prefix on,
the training forward is bit-identical to the padded layout and gradients stay within the packed-row bounds; with LoRA
dropout the layout does not share; the 13B-width reference fixtures pass their gates with sharing on."""
from types import SimpleNamespace

import pytest
import torch

import test_gpu_llava13b as L13
import test_gpu_packed_rows as PR
from oracle import llava_dpo_oracle as O
from test_gpu_kernel_bounds import F64, FTZ_FLOOR, assert_within, attention_ref, expand_kv, group_sum, heads

pytestmark = pytest.mark.gpu

# (pos0, chosen rows, rejected own rows); a third sequence of 300 rows neither lends nor borrows
CASES = [(128, 129, 129), (512, 1135, 623), (1024, 2048, 1024), (256, 700, 1)]
OTHER = 300


def _layout(P, Lc, R):
    from rlaifv_b200.model import RowPacking
    own, pos0, partner = [Lc, R, OTHER], [0, P, 0], [1, 0, -1]
    T = max(Lc, P + R, OTHER)
    cu = torch.tensor([0, Lc, Lc + R, Lc + R + OTHER], dtype=torch.int32)
    pos = torch.cat([torch.arange(Lc), torch.arange(P, P + R), torch.arange(OTHER)])
    rows = pos + torch.repeat_interleave(torch.arange(3), torch.tensor(own)) * T
    p0, pa = torch.tensor(pos0, dtype=torch.int32), torch.tensor(partner, dtype=torch.int32)
    return RowPacking(3, T, sum(own), max(own), cu.cuda(), pos.int().cuda(), rows.int().cuda(), p0.cuda(), pa.cuda(),
                      p0, pa)


@pytest.mark.parametrize("n_kv", [32, 8], ids=["mha32", "gqa32_8"])
@pytest.mark.parametrize("P,Lc,R", CASES)
def test_prefix_attention_matches_fixed_length_kernels(P, Lc, R, n_kv):
    from rlaifv_b200 import ops
    nh, hd = 32, 128
    H, KV, W = nh * hd, n_kv * hd, (nh + 2 * n_kv) * hd
    pk = _layout(P, Lc, R)
    nseq, T, M = 3, pk.T, pk.M
    g = torch.Generator(device="cuda").manual_seed(P + R)
    qkv = torch.randn(M, W, device="cuda", generator=g).to(torch.bfloat16)
    qkv_pad = PR._padded(qkv, pk, torch.randn(nseq * T, W, device="cuda", generator=g).to(torch.bfloat16))
    qkv_pad[T:T + P] = qkv[:P]                                   # the rejected copy of the shared rows
    scale = hd ** -0.5
    att, lse = torch.empty(M, H, dtype=torch.bfloat16, device="cuda"), torch.empty(nh * M, device="cuda")
    ops.attention_varlen_prefix_fwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], pk, nh, hd, scale, att, lse,
                                    n_kv_heads=n_kv)
    att_pad, lse_pad = ops.attention_fwd(qkv_pad[:, :H], qkv_pad[:, H:H + KV], qkv_pad[:, H + KV:], nseq, T, nh, hd, True,
                                         scale, n_kv_heads=n_kv)
    rows = pk.rows.long()
    assert torch.equal(att, att_pad[rows])
    cu = pk.cu.tolist()
    for s, (p0, n) in enumerate(zip([0, P, 0], [Lc, R, OTHER])):
        assert torch.equal(lse[nh * cu[s]:nh * cu[s + 1]].view(nh, n), lse_pad[s, :, p0:p0 + n]), s
    # backward: dO is zero on padding and on the rejected copy of the shared rows (the shared rows' dO is the chosen one)
    d_o = torch.randn(M, H, device="cuda", generator=g).to(torch.bfloat16)
    d_o_pad = PR._padded(d_o, pk, torch.zeros(nseq * T, H, dtype=torch.bfloat16, device="cuda"))
    dqkv = torch.empty_like(qkv)
    ops.attention_varlen_prefix_bwd(qkv[:, :H], qkv[:, H:H + KV], qkv[:, H + KV:], att, d_o, lse, pk, nh, hd, scale,
                                    dqkv[:, :H], dqkv[:, H:H + KV], dqkv[:, H + KV:],
                                    torch.empty(nh * M, device="cuda"), n_kv_heads=n_kv)
    dqkv_pad = torch.empty_like(qkv_pad)
    ops.attention_bwd_split(qkv_pad[:, :H], qkv_pad[:, H:H + KV], qkv_pad[:, H + KV:], att_pad, d_o_pad, lse_pad, nseq,
                            T, T, nh, hd, True, scale, dqkv_pad[:, :H], dqkv_pad[:, H:H + KV], dqkv_pad[:, H + KV:],
                            n_kv_heads=n_kv)
    torch.cuda.synchronize()
    assert torch.equal(dqkv[:, :H], dqkv_pad[rows, :H]), "dq"
    own = torch.ones(M, dtype=torch.bool, device="cuda")
    own[:P] = False                                             # the shared rows: the chosen sequence's first P
    assert torch.equal(dqkv[own, H:], dqkv_pad[rows[own], H:]), "dk / dv of rows that are not shared"
    assert not torch.equal(dqkv[:P, H:], dqkv_pad[:P, H:])      # the rejected queries' share arrived
    # shared rows: the sum of both copies' dK / dV against fp64
    q = heads(qkv_pad[:2 * T, :H], 2, T, nh, hd)
    k = expand_kv(heads(qkv_pad[:2 * T, H:H + KV], 2, T, n_kv, hd), nh)
    v = expand_kv(heads(qkv_pad[:2 * T, H + KV:], 2, T, n_kv, hd), nh)
    r = attention_ref(q, k, v, scale, True, d_out=heads(d_o_pad[:2 * T], 2, T, nh, hd))
    for name, cols in (("dk", slice(H, H + KV)), ("dv", slice(H + KV, W))):
        ref = group_sum(r[name][:, :, :P].sum(0), n_kv)
        bound = group_sum(r[name + "_t"][:, :, :P].sum(0), n_kv) + 2.0 ** -8 * ref.abs() + FTZ_FLOOR
        got = dqkv[:P, cols].view(P, n_kv, hd).permute(1, 0, 2).to(F64)
        assert_within(f"shared {name} P={P} R={R} nkv={n_kv}", got, ref, bound)


# ---------------------------------------------------------------------------------------------------------- models
@pytest.fixture
def shared_layouts(monkeypatch):
    """The RowPacking of every training forward (to check that the batch shared rows)."""
    from rlaifv_b200 import model
    seen, pack = [], model.pack_rows

    def record(labels, sources=None):
        pk = pack(labels, sources)
        seen.append(pk)
        return pk
    monkeypatch.setattr(model, "pack_rows", record)
    return seen


def _shared_step_matches_padded(pol, batch, seen):
    pol.share_prefix = True
    out = PR._compare(pol, batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    assert seen[-1] is not None and seen[-1].shared and int(seen[-1].pos0_h.max()) >= 512
    return out


@pytest.mark.parametrize("n_kv,ffn,ragged", [(32, 11008, False), (32, 11008, True), (8, 14336, True)],
                         ids=["llava7b_equal", "llava7b_ragged", "mistral7b_gqa_ragged"])
def test_7b_width_two_layers_shared_matches_padded(n_kv, ffn, ragged, shared_layouts):
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    dims = LlavaDims(num_layers=2, num_kv_heads=n_kv, intermediate_size=ffn, clip_layers=3)
    batch = O.synthetic_pair_batch(SimpleNamespace(vocab_size=dims.vocab_size, image_size=dims.image_size), 2, 60, 500,
                                   seed=11, image_pos=5, ragged=ragged)
    _shared_step_matches_padded(LlavaDPOPolicy(dims, "cuda", seed=3), batch, shared_layouts)
    # one engine step each way from the same weights: the 9 step metrics are the same bits
    batch.update(ref_win_logp=torch.tensor([-900.0, -950.0]), ref_rej_logp=torch.tensor([-905.0, -940.0]), beta=0.1)
    metrics = []
    for shared in (False, True):
        pol = LlavaDPOPolicy(dims, "cuda", seed=3)
        pol.pack_rows = pol.share_prefix = shared
        eng = DPOStepEngine(pol, lr=1e-5, total_steps=10, constant_lr=True)
        metrics.append(eng.train_step(batch).clone())
        del eng, pol
    assert torch.equal(metrics[0], metrics[1])


def test_7b_width_lora_shared_matches_padded_and_dropout_does_not_share(shared_layouts):
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    dims = LlavaDims(num_layers=2, clip_layers=3)
    batch = O.synthetic_pair_batch(SimpleNamespace(vocab_size=dims.vocab_size, image_size=dims.image_size), 2, 60, 500,
                                   seed=12, image_pos=5, ragged=True)
    pol = LlavaDPOPolicy(dims, "cuda", seed=3)
    pol.enable_lora(r=64, alpha=16, seed=7, init_b_zero=False, dropout=0.0)
    _shared_step_matches_padded(pol, batch, shared_layouts)
    # with dropout: the same packed layout as without the switch, and the same bits
    pol.lora.dropout = 0.05
    args = (batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"], True)
    pol.share_prefix = True
    on = PR._step(pol, *args)
    assert not shared_layouts[-1].shared
    pol.share_prefix = False
    off = PR._step(pol, *args)
    for k in on[0]:
        assert torch.equal(on[0][k], off[0][k]), k
    assert torch.equal(on[1], off[1])
    for k in on[2]:
        assert torch.equal(on[2][k], off[2][k]), k


@pytest.fixture
def sharing_policies(monkeypatch, shared_layouts):
    """Every LlavaDPOPolicy built in the test has share_prefix on."""
    from rlaifv_b200.model import LlavaDPOPolicy
    init = LlavaDPOPolicy.__init__

    def init_shared(self, *a, **kw):
        init(self, *a, **kw)
        self.share_prefix = True
    monkeypatch.setattr(LlavaDPOPolicy, "__init__", init_shared)
    L13._POL.clear()                          # the 13B tests cache their policy: build one with the switch on
    yield shared_layouts
    L13._POL.clear()


@pytest.mark.parametrize("name", L13.FULL_FT)
def test_13b_width_reference_fixtures_pass_with_shared_prefix(name, sharing_policies):
    L13.test_13b_width_forward_matches_reference_fixture(name)
    L13.test_13b_width_dpo_loss_and_grads_match_reference_fixture(name)
    assert any(pk is not None and pk.shared and int(pk.pos0_h.max()) == 512 for pk in sharing_policies)


def test_13b_width_lora_reference_fixture_passes_with_shared_prefix(sharing_policies):
    L13.test_13b_width_lora_matches_merged_weight_reference_fixture()
    assert any(pk is not None and pk.shared for pk in sharing_policies)
