"""CPU tests of the host-side training stack: flag parsing (every flag of the reference launch
script), the llava_v1 sample encoding with a toy tokenizer, the ZeRO-2 partition / collective
plumbing on world_size-2 gloo, and the parquet contract of the reference log-prob cache."""
import json
import os
import re
import subprocess
import sys
import textwrap

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def script_flags(name="llava15_train.sh"):
    """--flag value pairs of the bash arrays in the launch script."""
    txt = open(os.path.join(REPO, "script", "train", name)).read()
    body = "\n".join(re.findall(r"^[A-Z]+=\((.*?)\)$", txt, flags=re.M | re.S))
    toks = re.findall(r"(--[a-z_0-9]+)\s+('[^']*'|\"[^\"]*\"|[^\s]+)", body)
    argv = []
    for k, v in toks:
        argv += [k, v.strip("'\"")]
    return argv


def reference_script_flags(name):
    """Flag names of the reference's own launch scripts (fixture: every `--flag` token of
    /root/reference/script/train/<name>, extracted with re.findall(r"(--[a-z_0-9]+)") in the build container)."""
    with open(os.path.join(REPO, "tests", "golden_host", "reference_script_flags.json")) as f:
        return set(json.load(f)[name])


def test_every_reference_flag_parses():
    from rlaifv_b200.train_llava15 import parse_args_into_dataclasses, zero_stage
    argv = [a.replace("$CKPT", "x").replace("$exp_name", "x") for a in script_flags()]
    ref = reference_script_flags("llava15_train.sh")
    assert ref <= set(argv[0::2]), ref - set(argv[0::2])      # every flag of the reference recipe is present
    m, d, t = parse_args_into_dataclasses(argv)
    assert t.task == "DPO" and d.dpo_beta == 0.1 and t.dpo_use_average is False and t.max_steps == 2672
    assert t.learning_rate == 5e-7 and t.weight_decay == 0.01 and t.warmup_ratio == 0.05 and t.bf16 is True
    assert m.mm_vision_select_layer == -2 and m.mm_projector_type == "mlp2x_gelu" and t.model_max_length == 2048
    assert zero_stage(os.path.join(REPO, "script", "zero2.json")) == 2
    assert len(argv) // 2 >= 40


def test_every_reference_lora_flag_parses():
    """script/train/llava15_train_lora.sh (reference: same file name, :6-49) through the LoRA entry's argv path."""
    from rlaifv_b200.train_llava15 import parse_args_into_dataclasses
    argv = [a.replace("$CKPT", "x").replace("$exp_name", "x") for a in script_flags("llava15_train_lora.sh")]
    ref = reference_script_flags("llava15_train_lora.sh")
    assert ref <= set(argv[0::2]), ref - set(argv[0::2])
    assert "--lora_enable" in argv and "rlaifv_b200.train_llava15_lora" in open(
        os.path.join(REPO, "script", "train", "llava15_train_lora.sh")).read()
    m, d, t = parse_args_into_dataclasses(argv)
    assert t.lora_enable is True and t.lora_r == 64 and t.lora_alpha == 16 and t.lora_dropout == 0.05
    assert t.learning_rate == 1e-5 and t.fully_tune is False and t.task == "DPO" and t.lora_bias == "none"
    # the module the script launches exists and forces --lora_enable when the flag is absent
    import rlaifv_b200.train_llava15_lora as L
    assert callable(L.train)


def test_llava_v1_encoding_matches_reference_fixture():
    """ids and label masks of encode_multimodal_preference_sample / preprocess_v1 equal the unmodified
    reference's (fixture from oracle/gen_golden.py, same toy tokenizer)."""
    import numpy as np
    from oracle.toy_tokenizer import ToyTokenizer
    from rlaifv_b200.data import IMAGE_TOKEN_INDEX, encode_multimodal_preference_sample
    fx = np.load(os.path.join(REPO, "tests", "golden_host", "encode_case.npz"))
    tok = ToyTokenizer()
    cfg = {"image_processor": lambda im: torch.zeros(3, 4, 4), "is_multimodal": True, "image_token_len": 576,
           "use_im_start_end": False, "keep_image_tag": True}
    for i in range(int(fx["n"])):
        src = {"question": {"from": "human", "value": str(fx[f"s{i}_q"])},
               "chosen": {"from": "gpt", "value": str(fx[f"s{i}_c"])},
               "rejected": {"from": "gpt", "value": str(fx[f"s{i}_r"])}, "image": "IMG",
               "ref_win_logp": -1.0, "ref_rej_logp": -2.0, "ref_win_avg_logp": -0.1, "ref_rej_avg_logp": -0.2,
               "ref_win_per_token_logp": [0.0] * 9, "ref_rej_per_token_logp": [0.0] * 9}
        rej, win = encode_multimodal_preference_sample(src, tok, cfg)
        assert np.array_equal(win["input_ids"].numpy(), fx[f"s{i}_win_ids"])
        assert np.array_equal(win["labels"].numpy(), fx[f"s{i}_win_labels"])
        assert np.array_equal(rej["input_ids"].numpy(), fx[f"s{i}_rej_ids"])
        assert np.array_equal(rej["labels"].numpy(), fx[f"s{i}_rej_labels"])
        assert (win["input_ids"] == IMAGE_TOKEN_INDEX).sum() == 1 and win["labels"][0] == -100
        assert win["ref_win_logp"] == -1.0 and rej["ref_rej_logp"] == -2.0


def test_logp_parquet_contract_roundtrip(tmp_path):
    from rlaifv_b200.data import _load_parquet_dir, write_logp_to_preference_parquet
    rows = [{"question": f"q{i}", "chosen": "c", "rejected": "r", "idx": i, "image": {"bytes": b"x"}} for i in range(3)]
    logps = [(-1.0 * i, -0.1, [0.5, 0.25], -2.0, -0.2, [0.125]) for i in range(3)]
    write_logp_to_preference_parquet(rows, str(tmp_path), logps)
    files = os.listdir(tmp_path)
    assert files == ["RLAIF-V-Dataset-withlogp_000-3.parquet"]
    back = _load_parquet_dir(str(tmp_path))
    v = json.loads(back[2]["logps"])["logps"]
    assert v[0] == -2.0 and v[2] == [0.5, 0.25] and v[5] == [0.125] and len(v) == 6


GLOO_WORKER = textwrap.dedent('''
    import os, sys, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    rank, world = int(sys.argv[1]), 2
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = sys.argv[2]
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rlaifv_b200.model import LlavaDims, ParamStore
    from rlaifv_b200 import zero2, ops
    # test double for the CUDA AdamW kernel (this test covers partitioning + collectives on CPU only)
    def fake_adamw(master, m, v, grad, param, lr, b1, b2, eps, wd, step, grad_scale=1.0):
        master.mul_(1 - lr * wd).add_(grad.float(), alpha=-lr)
        param.copy_(master.to(param.dtype))
    ops.adamw_step = fake_adamw
    zero2.ops.adamw_step = fake_adamw
    class Ev:
        def record(self, *a): pass
    class St:
        cuda_stream = 0
        def wait_stream(self, *a): pass
        def wait_event(self, *a): pass
    import contextlib
    torch.cuda.Event = lambda *a, **k: Ev()
    torch.cuda.current_stream = lambda *a, **k: St()
    torch.cuda.Stream = lambda *a, **k: St()
    torch.cuda.stream = lambda s: contextlib.nullcontext()
    # gloo lacks reduce_scatter_tensor: emulate with all_reduce + slice (same semantics)
    def rs(out, inp, op=None, group=None):
        t = inp.float(); dist.all_reduce(t); n = inp.numel() // world
        out.copy_(t[rank * n:(rank + 1) * n].to(out.dtype))
    def ag(out, inp, group=None):
        parts = [torch.empty_like(inp) for _ in range(world)]
        dist.all_gather(parts, inp.clone()); out.copy_(torch.cat(parts))
    dist.reduce_scatter_tensor = rs; dist.all_gather_into_tensor = ag
    zero2.dist.reduce_scatter_tensor = rs; zero2.dist.all_gather_into_tensor = ag
    d = LlavaDims(vocab_size=64, hidden_size=64, intermediate_size=128, num_layers=2, num_heads=1,
                  clip_hidden=64, clip_intermediate=64, clip_layers=2, clip_heads=1, image_size=28)
    st = ParamStore(d, "cpu")
    torch.manual_seed(0)
    st.flat.copy_(torch.randn(st.numel).bfloat16())
    p0 = st.flat.clone().float()
    torch.manual_seed(100 + rank)
    st.grad.copy_((torch.randn(st.numel) * 0.5).bfloat16())        # rank-local grads (already 1/world scaled)
    gsum = st.grad.float().clone(); dist.all_reduce(gsum)
    # an extra trainable bucket outside the ParamStore (LoRA adapters / the OmniLMM resampler are passed like this)
    torch.manual_seed(7)
    xflat = torch.randn(2048).bfloat16(); xgrad = torch.zeros(2048, dtype=torch.bfloat16)
    x0 = xflat.clone().float()
    torch.manual_seed(200 + rank); xgrad.copy_((torch.randn(2048) * 0.5).bfloat16())
    xsum = xgrad.float().clone(); dist.all_reduce(xsum)
    buckets = st.opt_buckets() + [zero2.OptBucket("resampler", xflat, xgrad, 1024)]
    opt = zero2.Zero2AdamW(buckets, lr=0.1, weight_decay=0.0, rank=rank, world=world,
                           gather_order=["resampler", "embed", "layer0", "layer1", "head", "projector"])
    assert opt.owned * world == st.numel + 2048 and opt.index["resampler"] == len(buckets) - 1
    opt.reduce_all()
    opt.step(0.1)
    expect = (p0 - 0.1 * gsum.bfloat16().float()).bfloat16().float()
    err = (st.flat.float() - expect).abs().max().item()
    # every rank holds the full updated parameters after the all-gather
    chk = st.flat.float().clone(); dist.all_reduce(chk)
    same = (chk / world - st.flat.float()).abs().max().item()
    xerr = (xflat.float() - (x0 - 0.1 * xsum.bfloat16().float()).bfloat16().float()).abs().max().item()
    print("RESULT", rank, err, same, xerr)
    assert err <= 4e-2 and same == 0.0 and xerr <= 4e-2
    dist.destroy_process_group()
''')


def test_zero2_partition_and_collectives_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(GLOO_WORKER % REPO)
    port = str(29000 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), port], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o
        assert "RESULT" in o


def test_clip_image_processor_matches_hf_processor():
    """rlaifv_b200.image_processing.ClipImageProcessor against transformers' CLIPImageProcessor (what the reference
    binds as `vision_tower.image_processor`, clip_encoder.py:29) with the clip-vit-large-patch14-336 settings."""
    import numpy as np
    from PIL import Image
    from transformers import CLIPImageProcessor
    from rlaifv_b200.image_processing import ClipImageProcessor, PixelValues, SquareResizeProcessor
    hf = CLIPImageProcessor(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336}, do_resize=True,
                            do_center_crop=True, do_normalize=True, do_convert_rgb=True, resample=3)
    ours = ClipImageProcessor(336, 336)
    rng = np.random.RandomState(0)
    for (h, w) in ((500, 375), (336, 336), (200, 640), (1000, 900)):
        img = Image.fromarray(rng.randint(0, 256, (h, w, 3), dtype=np.uint8))
        want = np.asarray(hf(img)["pixel_values"][0])
        got = ours(img)["pixel_values"][0]
        assert got.shape == want.shape == (3, 336, 336) and got.dtype == np.float32
        # transformers 5.5 resizes through its own (torch) backend; the pinned 4.35.0 processor — and this one — call
        # PIL's bicubic resize. The two agree to fp32 rounding except for < 1 % of the pixels, which land on the other
        # side of a uint8 rounding boundary (one or two grey levels = 0.015 / 0.03 after normalisation).
        d = np.abs(got - want)
        assert float(d.max()) <= 0.032 and float((d > 1e-4).mean()) <= 0.01 and float(d.mean()) <= 2e-4, (h, w)
    pv = PixelValues(ours)
    t = pv(Image.fromarray(rng.randint(0, 256, (50, 70), dtype=np.uint8)))       # grayscale -> RGB
    assert tuple(t.shape) == (3, 336, 336) and pv.crop_size == {"height": 336, "width": 336}
    sq = SquareResizeProcessor(448)(Image.fromarray(rng.randint(0, 256, (300, 500, 3), dtype=np.uint8)))
    assert tuple(sq.shape) == (3, 448, 448) and sq.dtype == torch.float32


def test_dims_from_checkpoint_reads_config(tmp_path):
    import json
    from rlaifv_b200.train_llava15 import dims_from_checkpoint
    d = dims_from_checkpoint("liuhaotian/llava-v1.5-7b", "openai/clip-vit-large-patch14-336", -2, 2048)   # hub names: defaults
    assert (d.hidden_size, d.num_layers, d.clip_hidden, d.image_size, d.select_layer, d.max_len) == (4096, 32, 1024, 336, -2, 2048)
    (tmp_path / "config.json").write_text(json.dumps({"hidden_size": 256, "num_hidden_layers": 2, "num_attention_heads": 2,
                                                      "intermediate_size": 512, "vocab_size": 512}))
    d = dims_from_checkpoint(str(tmp_path), None, -2, 512)
    assert (d.hidden_size, d.num_layers, d.num_heads, d.vocab_size, d.clip_hidden) == (256, 2, 2, 512, 1024)
