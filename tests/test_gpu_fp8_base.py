"""GPU tests of the FP8 frozen base (DESIGN.md §3 "FP8 frozen base"): both quantizers bit for bit against
oracle/fp8_oracle.py, gemm_fp8 per element against the fp64 product of its dequantized operands (oracle bound: FP8
K-block accumulation, fp32 promotion, epilogue rounding) at every frozen-base launch of a recorded LoRA step and at
edge shapes, and the FP8 policy at model level and through train_llava15."""
import math
import os
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

from oracle import fp8_oracle as F8  # noqa: E402

pytestmark = pytest.mark.gpu

WIDTHS = {"7b": dict(hidden_size=4096, intermediate_size=11008, num_heads=32),
          "13b": dict(hidden_size=5120, intermediate_size=13824, num_heads=40)}
M_STEP = 9080
WORST = {}


def _dev():
    return torch.device("cuda", 0)


def _rows(M, K, ld, seed, scale_spread=True):
    """bf16 [M, K] view of a wider [M, ld] buffer; rows spread over many binades, with zero and subnormal tiles."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn((M, ld), generator=g, device="cuda")
    if scale_spread:
        buf *= torch.exp2(torch.randint(-20, 12, (M, 1), generator=g, device="cuda").float())
    x = buf.to(torch.bfloat16)[:, :K]
    x[3, :128] = 0
    x[5, 128:256] = torch.tensor(2.0 ** -130).to(torch.bfloat16)
    return x


@pytest.mark.parametrize("K", [4096, 11008, 5120, 13824, 3 * 4096, 2 * 13824])
def test_quant_rows_bit_exact(K):
    from rlaifv_b200 import ops
    x = _rows(M_STEP, K, K + 256, K)
    q, s = ops.quant_fp8_rows(x)
    qr, sr = F8.quant_rows(x.cpu())
    assert s.shape == (K // 128, ops.fp8_scale_rows(M_STEP))
    assert torch.equal(q.cpu().view(torch.uint8), qr.view(torch.uint8))
    assert torch.equal(s[:, :M_STEP].cpu(), sr)


@pytest.mark.parametrize("N,K", [(3 * 4096, 4096), (4096, 4096), (2 * 11008, 4096), (4096, 11008),
                                 (3 * 5120, 5120), (2 * 13824, 5120), (5120, 13824)])
def test_quant_blocks_bit_exact(N, K):
    from rlaifv_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = (torch.randn((N, K + 128), generator=g, device="cuda") * 0.02).to(torch.bfloat16)[:, :K]
    w[:128, :128] = 0
    fw = ops.Fp8Weight(N, K, _dev())
    # two halves quantized into one weight (the model streams q / k / v and gate / up this way)
    h = N // 2 // 128 * 128
    ops.quant_fp8_blocks(w[:h], *fw.rows(0, h))
    ops.quant_fp8_blocks(w[h:], *fw.rows(h, N - h))
    q, qt, s = F8.quant_blocks(w.cpu())
    assert torch.equal(fw.q.cpu().view(torch.uint8), q.view(torch.uint8))
    assert torch.equal(fw.qt.cpu().view(torch.uint8), qt.view(torch.uint8))
    assert torch.equal(fw.s.cpu(), s)


def test_entry_points_refuse_bad_shapes():
    from rlaifv_b200 import ops
    from rlaifv_b200.lib import B200Error
    x = torch.zeros((256, 1088), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(B200Error, match="multiple of 128"):
        ops.quant_fp8_rows(x, torch.empty((256, 1088), dtype=torch.float8_e4m3fn, device="cuda"),
                           torch.empty((8, 256), dtype=torch.float32, device="cuda"))
    with pytest.raises(AssertionError):
        ops.Fp8Weight(1216, 4096, _dev())       # SwiGLU widths F = 1088 / 1216 are not FP8 shapes
    w = ops.Fp8Weight(256, 256, _dev())
    a, sa = ops.quant_fp8_rows(torch.zeros((64, 256), dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(B200Error, match="residual and a SwiGLU"):
        ops.gemm_fp8(a, sa, w, torch.empty((64, 512), dtype=torch.bfloat16, device="cuda"),
                     residual=torch.zeros((64, 256), dtype=torch.bfloat16, device="cuda"),
                     glu=torch.zeros((64, 512), dtype=torch.bfloat16, device="cuda"))


# ---------------------------------------------------------------------------------------------- gemm_fp8 vs fp64
def _weight(N, K, seed):
    from rlaifv_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn((N, K), generator=g, device="cuda") * 0.02
    # blocks of different magnitude, so a scale read from the wrong block shows
    w *= torch.exp2(torch.randint(-3, 4, (N // 128, 1, K // 128, 1), generator=g, device="cuda").float()).repeat(
        1, 128, 1, 128).view(N, K)
    w = w.to(torch.bfloat16)
    fw = ops.Fp8Weight(N, K, _dev())
    ops.quant_fp8_blocks(w, fw.q, fw.qt, fw.s)
    return fw


def run_case(M, fw, dgrad, k2=0, r=0, n_sub=0, residual=False, glu=False, seed=0, col_block=False):
    """One gemm_fp8 launch with crafted operands, checked per element against fp64; returns the worst err/bound.
    col_block: the output is a column block of a wider buffer whose other columns must keep their bits."""
    from rlaifv_b200 import ops
    N = fw.K if dgrad else fw.N
    K = fw.N if dgrad else fw.K
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((M, K), generator=g, device="cuda")
    x *= torch.exp2(torch.randint(-4, 5, (M, K // 128), generator=g, device="cuda").float()).repeat_interleave(128, 1)
    aq, sa = ops.quant_fp8_rows(x.to(torch.bfloat16))
    a2 = b2 = None
    if k2:
        ncols = (N // n_sub) * r if n_sub else k2
        a2 = (torch.randn((M, ncols), generator=g, device="cuda") * 0.5)
        a2[::4] += 2.0 ** 3                                            # every fourth row: a large second source
        a2 = a2.to(torch.bfloat16)
        b2 = (torch.randn((k2, N) if dgrad else (N, k2), generator=g, device="cuda") * 0.05).to(torch.bfloat16)
    res = (torch.randn((M, N), generator=g, device="cuda") * 4).to(torch.bfloat16) if residual else None
    gu = None
    if glu:
        gu = torch.randn((M, 2 * N), generator=g, device="cuda").to(torch.bfloat16)
        gu[:, :N:7] = -1.28                                            # around the zero of silu'
    width = (2 * N if glu else N)
    pad = 128 if col_block else 0
    big = torch.randn((M, width + 2 * pad), generator=g, device="cuda").to(torch.bfloat16)
    before = big.clone()
    out = big[:, pad:pad + width]
    ops.gemm_fp8(aq, sa, fw, out, dgrad=dgrad, a2=a2, b2=b2, k2=k2, r=r, n_sub=n_sub, residual=res, glu=gu)
    torch.cuda.synchronize()
    if col_block:
        assert torch.equal(big[:, :pad], before[:, :pad]) and torch.equal(big[:, pad + width:], before[:, pad + width:])
    # fp64 reference on the device, in row chunks
    worst, excess = 0.0, 0.0
    wd = F8.dequant_blocks(fw.q, fw.s)
    bmat = wd.t() if dgrad else wd                                     # [N, K]
    for m0 in range(0, M, 2048):
        m1 = min(M, m0 + 2048)
        ad = F8.dequant_rows(aq[m0:m1], sa[:, m0:m1])
        ref = ad @ bmat.t()
        s1 = ad.abs() @ bmat.abs().t()
        s2 = None
        if k2:
            if n_sub:
                rows = []
                for j in range(N // n_sub):
                    a2j = a2[m0:m1, j * r:j * r + k2].double()
                    rows.append(a2j @ b2[j * n_sub:(j + 1) * n_sub].double().t())
                ref = ref + torch.cat(rows, 1)
                s2 = torch.cat([a2[m0:m1, j * r:j * r + k2].double().abs() @
                                b2[j * n_sub:(j + 1) * n_sub].double().abs().t() for j in range(N // n_sub)], 1)
            else:
                b2m = b2.double().t() if dgrad else b2.double()        # [N, k2]
                ref = ref + a2[m0:m1].double() @ b2m.t()
                s2 = a2[m0:m1].double().abs() @ b2m.abs().t()
        acc_err = F8.acc_bound(s1, K, s2, k2)
        got = out[m0:m1].double()
        if glu:
            d_err = F8.epilogue_bound(ref, acc_err)
            ref, bound = F8.swiglu_bwd_ref(ref, d_err, gu[m0:m1])
        else:
            bound = F8.epilogue_bound(ref, acc_err, None if res is None else res[m0:m1])
            if res is not None:
                ref = ref + res[m0:m1].double()
            excess = max(excess, float(((got - ref).abs() - (bound - F8.EPS_BLK * s1)).div(s1.clamp(min=1e-30)).max()))
        err = (got - ref).abs()
        ratio = err / bound.clamp(min=1e-30)
        worst = max(worst, float(ratio.max()))
        assert bool(torch.isfinite(got).all())
    return worst, excess


def _report(name, worst, excess):
    WORST[name] = (worst, excess)
    print("fp8 bound %-48s worst err/bound %.4f  accumulation excess / sum|ab| %.3g" % (name, worst, excess))


@pytest.fixture(scope="module")
def recorded():
    """gemm_fp8 launches of one LoRA-DPO step of a one-layer FP8 policy at both widths (bench's batch)."""
    import bench
    from rlaifv_b200 import ops
    from rlaifv_b200.engine import DPOStepEngine
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    out = {}
    for wname, w in WIDTHS.items():
        pol = LlavaDPOPolicy(LlavaDims(num_layers=1, **w), _dev(), seed=0, base_fp8=True)
        pol.enable_lora(r=64, alpha=16)
        eng = DPOStepEngine(pol, lr=1e-5, weight_decay=0.01, total_steps=10, micro_pairs=4)
        hb = bench.synthetic_batch(0, 0, 8)
        hb["ref_win_logp"], hb["ref_rej_logp"] = torch.zeros(8), torch.zeros(8)
        calls, orig = [], ops.gemm_fp8

        def rec(aq, sa, fw, o, **kw):
            calls.append(dict(N=fw.N, K=fw.K, dgrad=kw.get("dgrad", False), k2=kw.get("k2", 0) if
                              kw.get("a2") is not None else 0, r=kw.get("r", 0), n_sub=kw.get("n_sub", 0),
                              residual=kw.get("residual") is not None, glu=kw.get("glu") is not None))
            return orig(aq, sa, fw, o, **kw)
        ops.gemm_fp8 = rec
        try:
            eng.train_step(hb, optimizer_step=False)
            torch.cuda.synchronize()
        finally:
            ops.gemm_fp8 = orig
        uniq = []
        for c in calls:
            if c not in uniq:
                uniq.append(c)
        out[wname] = uniq
        del eng, pol
        torch.cuda.empty_cache()
    return out


def test_recorded_launches_cover_the_frozen_base(recorded):
    for wname, calls in recorded.items():
        # forward: qkv, o (+res), gu, down (+res); dgrad: down (SwiGLU), gu, o, qkv
        assert len(calls) == 8, (wname, calls)
        assert sum(c["dgrad"] for c in calls) == 4 and sum(c["glu"] for c in calls) == 1
        assert sum(c["residual"] for c in calls) == 2 and all(c["k2"] > 0 for c in calls)


@pytest.mark.parametrize("wname", list(WIDTHS))
def test_gemm_fp8_recorded_launches_within_fp64_bound(recorded, wname):
    for j, c in enumerate(recorded[wname]):
        fw = _weight(c["N"], c["K"], seed=100 + j)
        worst, excess = run_case(M_STEP, fw, c["dgrad"], k2=c["k2"], r=c["r"], n_sub=c["n_sub"],
                                 residual=c["residual"], glu=c["glu"], seed=j)
        _report("%s N=%d K=%d dgrad=%d k2=%d res=%d glu=%d" % (wname, c["N"], c["K"], c["dgrad"], c["k2"],
                                                                c["residual"], c["glu"]), worst, excess)
        assert worst <= 1.0, (wname, c, worst)


@pytest.mark.parametrize("r", [8, 16, 64, 128])
@pytest.mark.parametrize("residual", [False, True])
def test_gemm_fp8_dual_forward_edges(r, residual):
    fw = _weight(3 * 512, 1024, seed=r)
    worst, excess = run_case(1000, fw, False, k2=r, r=r, n_sub=512, residual=residual, seed=r, col_block=True)
    _report("dual fwd r=%d res=%d M=1000" % (r, residual), worst, excess)
    assert worst <= 1.0


@pytest.mark.parametrize("g", [1, 2, 3])
def test_gemm_fp8_dgrad_edges(g):
    fw = _weight(g * 640, 768, seed=g)
    worst, excess = run_case(777, fw, True, k2=g * 64, r=64, seed=g, col_block=True)
    _report("dgrad K2=%d M=777" % (g * 64), worst, excess)
    assert worst <= 1.0


@pytest.mark.parametrize("F", [1152, 1280])
@pytest.mark.parametrize("k2", [0, 64])
def test_gemm_fp8_swiglu_bwd_edges(F, k2):
    fw = _weight(640, F, seed=F)                 # W_down [H, F]; dgrad d(act) [M, F]
    worst, excess = run_case(1111, fw, True, k2=k2, r=64 if k2 else 0, glu=True, seed=F + k2, col_block=True)
    _report("swiglu_bwd F=%d k2=%d M=1111" % (F, k2), worst, excess)
    assert worst <= 1.0


def test_gemm_fp8_plain_no_second_source():
    fw = _weight(1024, 4096, seed=9)
    worst, excess = run_case(300, fw, False, seed=9, col_block=True)
    _report("plain fwd M=300 K=4096", worst, excess)
    assert worst <= 1.0


# ---------------------------------------------------------------------------------------------- model level
def _policy_pair(num_layers=2):
    from rlaifv_b200.model import LlavaDims, LlavaDPOPolicy
    dims = LlavaDims(num_layers=num_layers, clip_layers=3)
    return dims, LlavaDPOPolicy(dims, _dev(), seed=0, base_fp8=True)


def test_fp8_policy_forward_bits_on_every_layout_and_gap_to_bf16():
    from types import SimpleNamespace
    from oracle import llava_dpo_oracle as O
    from rlaifv_b200.model import LlavaDPOPolicy
    dims, pol = _policy_pair()
    pol.enable_lora(r=64, alpha=16, init_b_zero=False)
    batch = O.synthetic_pair_batch(SimpleNamespace(vocab_size=dims.vocab_size, image_size=dims.image_size), 2, 60, 500,
                                   seed=3, image_pos=5, ragged=True)
    args = (batch["concatenated_input_ids"], batch["concatenated_labels"], batch["images"])
    outs = {}
    for name, pack, share in (("padded", False, False), ("packed", True, False), ("shared", True, True)):
        pol.pack_rows, pol.share_prefix = pack, share
        outs[name] = pol.forward_logps(*args, keep_stash=True)["logp"].clone()
        pol._stash = None
    assert torch.equal(outs["padded"], outs["packed"]) and torch.equal(outs["padded"], outs["shared"])
    bf = LlavaDPOPolicy(dims, _dev(), seed=0)
    bf.enable_lora(r=64, alpha=16, init_b_zero=False)
    ref = bf.forward_logps(*args, keep_stash=False)["logp"]
    gap = (outs["padded"] - ref).abs()
    print("fp8 base vs bf16 base, summed log-prob: |gap| max %.4f mean %.4f (logp %s)" %
          (float(gap.max()), float(gap.mean()), [round(float(v), 2) for v in ref]))
    assert float(gap.max()) < 0.05 * float(ref.abs().max())


def test_fp8_policy_trains_from_ln2_and_lowers_the_loss():
    import bench
    from rlaifv_b200.engine import DPOStepEngine
    dims, pol = _policy_pair()
    pol.enable_lora(r=64, alpha=16)
    eng = DPOStepEngine(pol, lr=2e-4, weight_decay=0.0, total_steps=20, constant_lr=True, micro_pairs=2)
    hb = bench.synthetic_batch(0, 0, 2)
    out = pol.forward_logps(hb["concatenated_input_ids"], hb["concatenated_labels"], hb["images"], keep_stash=False)
    hb["ref_win_logp"], hb["ref_rej_logp"] = out["logp"][:2].float().cpu(), out["logp"][2:].float().cpu()
    losses = []
    for _ in range(10):
        m = eng.train_step(hb)
        losses.append(float(m[0]))
    print("fp8 base losses", [round(v, 4) for v in losses])
    assert abs(losses[0] - math.log(2)) < 1e-3
    assert losses[-1] < losses[0] - 0.01 and all(v == v for v in losses)


def test_fp8_policy_refuses_full_fine_tuning():
    from rlaifv_b200.engine import DPOStepEngine
    _, pol = _policy_pair(1)
    with pytest.raises(ValueError, match="only with LoRA"):
        DPOStepEngine(pol, lr=1e-5, total_steps=2)


def test_train_llava15_entry_with_base_fp8(tmp_path, monkeypatch):
    """train_llava15.train(--lora_enable True --base_fp8 True) on a tiny checkpoint: two steps from ln 2 and a
    peft-layout adapter."""
    import io
    import json
    from PIL import Image
    from oracle import llava_dpo_oracle as O
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
                        "--lora_enable", "True", "--lora_dropout", "0.0", "--base_fp8", "True"], source_rows=rows)
    torch.cuda.synchronize()
    pol = tr.model.policy
    assert pol.base_fp8 and pol.fp8 is not None and "l0.qkv" not in pol.store.p
    losses = [h["loss"] for h in tr.state["log_history"] if "loss" in h]
    assert len(losses) == 2 and abs(losses[0] - 0.693147) < 5e-3 and all(v == v for v in losses)
    ad = torch.load(out_dir / "adapter_model.bin")
    assert "base_model.model.model.layers.0.self_attn.q_proj.lora_A.weight" in ad
    assert json.loads((out_dir / "adapter_config.json").read_text())["peft_type"] == "LORA"
