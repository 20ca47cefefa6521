"""CPU tests of the FP8 frozen base: the oracle quantizer at its boundaries, exact dequantization, the fp64 error bound
accepting the rounded exact product and rejecting planted kernel errors, the parameter store without the base
matrices, the dry-run launch sequence of a LoRA step, and the --base_fp8 flag and its refusals."""
import ctypes
import math

import pytest
import torch

from oracle import fp8_oracle as F8
from oracle import llava_dpo_oracle as O

BF = torch.bfloat16


def _row(vals):
    x = torch.zeros(1, 128)
    x[0, :len(vals)] = torch.tensor(vals, dtype=torch.float64).float()
    return x.to(BF)


@pytest.mark.parametrize("e", [-20, 0, 7])
def test_scale_at_the_amax_boundaries(e):
    top = 448.0 * 2.0 ** e
    q, s = F8.quant_rows(_row([top, -1.0 * 2.0 ** e]))
    assert float(s[0, 0]) == 2.0 ** e and float(q[0, 0].float()) == 448.0          # exactly 448 * 2^e: scale 2^e
    up = float(torch.tensor(top).to(BF).float() * (1 + 2.0 ** -7))                  # one bf16 ulp above
    assert float(torch.tensor(up).to(BF)) > top
    q, s = F8.quant_rows(_row([up]))
    assert float(s[0, 0]) == 2.0 ** (e + 1) and float(q[0, 0].float()) == 224.0     # 225.75 rounds to 224


def test_zero_subnormal_and_clamped_tiles():
    q, s = F8.quant_rows(torch.zeros(2, 256, dtype=BF))
    assert torch.equal(s, torch.ones(2, 2)) and int(q.view(torch.uint8).count_nonzero()) == 0
    sub = 2.0 ** -130                                   # a bf16 subnormal: e clamps at -126
    q, s = F8.quant_rows(_row([sub, -sub / 2]))
    assert float(s[0, 0]) == 2.0 ** -126
    assert float(q[0, 0].float()) * 2.0 ** -126 == sub and float(q[0, 1].float()) * 2.0 ** -126 == -sub / 2
    assert int(F8.scale_exp(torch.tensor([3.0e38])).item()) == 120 and \
        int(F8.scale_exp(torch.tensor([1e-44])).item()) == -126


def test_codes_round_to_nearest_even_and_dequantize_exactly():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(64, 512, generator=g) * torch.exp2(torch.randint(-30, 30, (64, 1), generator=g).float())).to(BF)
    q, s = F8.quant_rows(x)
    d = F8.dequant_rows(q, s)
    # every dequantized value is an e4m3 value times a power of two: re-quantizing it gives the same codes
    q2, s2 = F8.quant_rows(d.to(BF))
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)
    # the rounding error is at most half an e4m3 ulp (3 mantissa bits: 2^-4 relative, 2^-9 * s absolute subnormal)
    err = (d - x.double()).abs()
    sc = s.t().repeat_interleave(128, 1).double()
    assert bool((err <= torch.maximum(x.double().abs() * 2.0 ** -4, sc * 2.0 ** -10)).all())
    w = (torch.randn(256, 384, generator=g) * 0.02).to(BF)
    qw, qt, sw = F8.quant_blocks(w)
    assert torch.equal(qt.view(torch.uint8), qw.view(torch.uint8).t())
    assert torch.equal(F8.quant_blocks(F8.dequant_blocks(qw, sw).to(BF))[0].view(torch.uint8), qw.view(torch.uint8))


# ------------------------------------------------------------------------------------- bound vs planted errors
def _case(M=96, N=256, K=512, r=16, n_sub=128, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * torch.exp2(torch.randint(-3, 4, (M, K // 128), generator=g).float()
                                                    ).repeat_interleave(128, 1)
    w = torch.randn(N, K, generator=g) * 0.02
    w *= torch.exp2(torch.randint(-3, 4, (N // 128, 1, K // 128, 1), generator=g).float()).repeat(
        1, 128, 1, 128).view(N, K)
    qa, sa = F8.quant_rows(x.to(BF))
    qw, _, sw = F8.quant_blocks(w.to(BF))
    a2 = torch.randn(M, (N // n_sub) * r, generator=g).to(BF).double()
    a2[::4] += 8
    b2 = (torch.randn(N, r, generator=g) * 0.05).to(BF).double()
    return qa, sa, qw, sw, a2, b2, r, n_sub


def _product(qa, sa, qw, sw, a2, b2, r, n_sub, koff_shift=0, drop2=None, sa_fn=None):
    """fp64 C with optional planted errors; also s1 and s2 of the bound."""
    a = F8.dequant_rows(qa, sa if sa_fn is None else sa_fn(sa))
    w = F8.dequant_blocks(qw, sw)
    c = a @ w.t()
    s1 = F8.dequant_rows(qa, sa).abs() @ w.abs().t()
    N = w.shape[0]
    parts, s2 = [], []
    for j in range(N // n_sub):
        k = (j + koff_shift) % (N // n_sub)
        a2j = a2[:, k * r:(k + 1) * r]
        parts.append(a2j @ b2[j * n_sub:(j + 1) * n_sub].t())
        s2.append(a2[:, j * r:(j + 1) * r].abs() @ b2[j * n_sub:(j + 1) * n_sub].abs().t())
    p2 = torch.cat(parts, 1)
    if drop2 is not None:
        p2[:, drop2] = 0
    return c + p2, s1, torch.cat(s2, 1)


def _fails(got, ref, s1, s2, K, r):
    bound = F8.epilogue_bound(ref, F8.acc_bound(s1, K, s2, r))
    return bool(((got - ref).abs() > bound).any())


def test_bound_accepts_the_rounded_exact_result_and_rejects_planted_errors():
    qa, sa, qw, sw, a2, b2, r, n_sub = _case()
    K = qa.shape[1]
    ref, s1, s2 = _product(qa, sa, qw, sw, a2, b2, r, n_sub)
    ok = ref.to(BF).double()
    assert not _fails(ok, ref, s1, s2, K, r)

    def planted(**kw):
        return _product(qa, sa, qw, sw, a2, b2, r, n_sub, **kw)[0].to(BF).double()

    # the scale of the neighbouring K-block
    assert _fails(planted(sa_fn=lambda s: torch.cat([s[1:2], s[1:]], 0)), ref, s1, s2, K, r)
    # one K-block's promotion dropped
    assert _fails(planted(sa_fn=lambda s: torch.cat([s[:2], s[2:3] * 0, s[3:]], 0)), ref, s1, s2, K, r)
    # second source dropped on the last 128-column tile, and koff one sub-linear off
    assert _fails(planted(drop2=slice(128, 256)), ref, s1, s2, K, r)
    assert _fails(planted(koff_shift=1), ref, s1, s2, K, r)
    # one bad row
    bad = ok.clone()
    bad[17] = (bad[17] * 1.01).to(BF).double()
    assert _fails(bad, ref, s1, s2, K, r)


def test_bound_rejects_one_operand_code_one_ulp_off():
    # a row whose product is dominated by one code at the top of its binade: one e4m3 ulp is 1/14 of it
    qa = torch.zeros(4, 128).to(F8.E4M3)
    qa[:, 5] = 448.0
    qa[:, 6:20] = 1.0
    sa = torch.ones(1, 4)
    qw = torch.ones(128, 128).to(F8.E4M3)
    sw = torch.ones(1, 1)
    ref, s1 = F8.gemm_ref(qa, sa, qw, sw)
    qa2 = qa.clone()
    qa2[2, 5] = 416.0                                   # 448 - one ulp (32)
    got = F8.gemm_ref(qa2, sa, qw, sw)[0].to(BF).double()
    bound = F8.epilogue_bound(ref, F8.acc_bound(s1, 128))
    assert bool(((got - ref).abs() > bound)[2].all()) and not bool(((got - ref).abs() > bound)[[0, 1, 3]].any())


def test_swiglu_bound_accepts_rounded_and_rejects_swapped_halves():
    g = torch.Generator().manual_seed(2)
    d = torch.randn(64, 128, generator=g, dtype=torch.float64) * 3
    gu = torch.randn(64, 256, generator=g).to(BF)
    gu[:, ::9] = -1.28
    ref, bound = F8.swiglu_bwd_ref(d, torch.zeros_like(d), gu)
    assert bool(((ref.to(BF).double() - ref).abs() <= bound).all())
    swapped = torch.cat([ref[:, 128:], ref[:, :128]], 1).to(BF).double()
    assert bool(((swapped - ref).abs() > bound).any())


# ------------------------------------------------------------------------------------- store, launches, flags
def _dims(c=O.TINY, **kw):
    from rlaifv_b200.model import LlavaDims
    return LlavaDims(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                     num_layers=c.num_layers, num_heads=c.num_heads, clip_hidden=c.clip_hidden,
                     clip_intermediate=c.clip_intermediate, clip_layers=c.clip_layers, clip_heads=c.clip_heads,
                     image_size=c.image_size, patch_size=c.patch_size, **kw)


def test_param_store_without_the_base_and_byte_counts():
    from rlaifv_b200.model import LlavaDims, ParamStore
    d = _dims()
    full, fp8 = ParamStore(d, "cpu"), ParamStore(d, "cpu", base=False)
    H, F = d.hidden_size, d.intermediate_size
    base = d.num_layers * (3 * H * H + H * H + 2 * F * H + H * F)
    assert full.numel - fp8.numel == base
    assert all(f"l{i}.{g}" not in fp8.p for i in range(d.num_layers) for g in ("qkv", "o", "gu", "down"))
    assert f"l1.ln2" in fp8.p and f"l1.ln2" in fp8.g
    hf = fp8.hf_views()
    assert "model.layers.0.input_layernorm.weight" in hf and "model.layers.0.self_attn.q_proj.weight" not in hf
    # 13B: the bf16 base and its gradient storage (2 x 2 B per element) against W + W^T codes and the block scales
    d13 = LlavaDims(hidden_size=5120, intermediate_size=13824, num_layers=40, num_heads=40)
    n = ParamStore.layout(d13)
    n_base = sum(math.prod(s) for _, dec, _ in n[1:41] for _, s in dec)
    fp8_bytes = 2 * n_base + 4 * n_base // (128 * 128)
    assert n_base == 40 * (4 * 5120 * 5120 + 3 * 13824 * 5120)
    print("13B base: bf16 W %.1f GB + grad %.1f GB; fp8 W + W^T + scales %.1f GB" %
          (2 * n_base / 1e9, 2 * n_base / 1e9, fp8_bytes / 1e9))


def _fake_lib(monkeypatch):
    from rlaifv_b200 import lib, ops
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(lib._SIGNATURES[name]), name
        calls.append((name, args))

    monkeypatch.setattr(lib, "call", fake_call)
    monkeypatch.setattr(lib, "stream_ptr", lambda: ctypes.c_void_p(0))
    monkeypatch.setattr(lib, "load", lambda: type("L", (), {"rlaifv_rmsnorm_bwd_partials": staticmethod(lambda: 4)})())
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=None: t)
    return calls


def _step(monkeypatch, base_fp8):
    from rlaifv_b200.model import LlavaDPOPolicy
    calls = _fake_lib(monkeypatch)
    c = O.TINY
    d = _dims()
    pol = LlavaDPOPolicy(d, "cpu", hf_state=O.make_params(c, seed=0), base_fp8=base_fp8)
    n_load = len(calls)
    pol.enable_lora(r=8, alpha=2.0)
    batch = O.synthetic_pair_batch(c, 2, 24, 30, seed=31, image_pos=7, ragged=True)
    T = 60
    monkeypatch.setattr(pol, "splice", lambda ids, labels, rows, nb, idx, T_hint=None: (
        torch.zeros(4 * T, d.hidden_size, dtype=BF), torch.full((4, T), -100), torch.zeros(4, T, dtype=torch.int32), T))
    pol.forward_logps(batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    pol.backward_logps(torch.zeros(4))
    return pol, calls[:n_load], calls[n_load:]


def test_lora_step_launch_sequence_sends_every_frozen_base_gemm_to_fp8(monkeypatch):
    _, load16, bf = _step(monkeypatch, False)
    pol, load8, f8 = _step(monkeypatch, True)
    L = pol.dims.num_layers
    # loading: 7 HF linears per layer through the block quantizer
    assert [n for n, _ in load8] == ["rlaifv_quant_fp8_blocks"] * 7 * L and not load16
    names8 = [n for n, _ in f8]
    assert names8.count("rlaifv_gemm_fp8") == 8 * L and names8.count("rlaifv_quant_fp8_rows") == 8 * L
    assert "rlaifv_gemm_bf16_dual" not in names8 and "rlaifv_gemm_bf16_swiglu_bwd" not in names8
    # nothing else changes: drop the quantizations and map the FP8 launches back to the bf16 forms
    names16 = [n for n, _ in bf]
    back = [n for n in names8 if n != "rlaifv_quant_fp8_rows"]
    fp8_as = iter(n for n in names16 if n in ("rlaifv_gemm_bf16_dual", "rlaifv_gemm_bf16_swiglu_bwd"))
    assert [next(fp8_as) if n == "rlaifv_gemm_fp8" else n for n in back] == names16
    # each FP8 GEMM consumes the quantization just before it; dgrad (b_t = 1) in the backward, forward before
    gi = [i for i, n in enumerate(names8) if n == "rlaifv_gemm_fp8"]
    assert all(names8[i - 1] == "rlaifv_quant_fp8_rows" for i in gi)
    b_t = [f8[i][1][7] for i in gi]
    assert b_t == [0] * 4 * L + [1] * 4 * L
    glu = [f8[i][1][22].value is not None for i in gi]
    assert sum(glu) == L


def test_base_fp8_flag_and_refusals(monkeypatch):
    from rlaifv_b200 import train_llava15 as TL
    from rlaifv_b200.model import Fp8BaseStore, LlavaDims, LlavaDPOPolicy
    assert TL.parse_args_into_dataclasses([])[2].base_fp8 is False
    ta = TL.parse_args_into_dataclasses(["--base_fp8", "True"])[2]
    assert ta.base_fp8 is True
    with pytest.raises(ValueError, match="--lora_enable True"):
        TL.check_base_fp8(ta)
    TL.check_base_fp8(TL.parse_args_into_dataclasses(["--base_fp8", "True", "--lora_enable", "True"])[2])
    with pytest.raises(ValueError, match="multiples of 128"):
        Fp8BaseStore.check_dims(LlavaDims(hidden_size=320, intermediate_size=512, num_heads=2))
    _fake_lib(monkeypatch)
    pol = LlavaDPOPolicy(_dims(), "cpu", hf_state=O.make_params(O.TINY, seed=0), base_fp8=True)
    with pytest.raises(ValueError, match="only with LoRA"):
        pol.trainable_buckets()
    reserve = pol.activation_reserve_bytes(2, 512)
    pol.base_fp8 = False
    assert reserve - pol.activation_reserve_bytes(2, 512) == 2 * 2 * 512 * 2 * O.TINY.intermediate_size * (1 + 4 / 128)
