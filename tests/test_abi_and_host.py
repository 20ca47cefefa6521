"""CPU tests: the C-ABI library loads and exports every symbol include/rlaifv_b200.h declares
(no compute without a GPU), plus host-side logic (parameter store layout, LR schedule, product
path isolation from the oracle)."""
import math
import os
import re
import subprocess

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(REPO, "include", "rlaifv_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rlaifv_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    from rlaifv_b200 import lib
    so = lib.LIB_PATH
    if not os.path.exists(so):
        import __graft_entry__
        __graft_entry__.build()
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r" T (rlaifv_[a-z0-9_]+)", out))
    declared = header_symbols()
    assert len(declared) >= 25
    missing = [s for s in declared if s not in exported]
    assert not missing, missing
    # the Python binding table and the header agree
    assert sorted(lib.exported_symbols()) == declared
    handle = lib.load()           # dlopen works on a CPU-only box (no libcuda link dependency)
    assert handle.rlaifv_last_error() is not None


def test_sass_is_hopper_native():
    so = os.path.join(REPO, "rlaif-v_b200", "librlaifv_b200.so")
    if not os.path.exists(so):
        pytest.skip("library not built")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "HGMMA" in sass            # wgmma.mma_async
    assert "UTMALDG" in sass          # TMA loads
    assert "SYNCS" in sass            # mbarrier
    assert "HMMA." not in sass        # no legacy mma.sync path


def test_param_store_layout_cpu():
    from rlaifv_b200.model import LlavaDims, ParamStore
    d = LlavaDims(vocab_size=512, hidden_size=256, intermediate_size=512, num_layers=2, num_heads=2,
                  clip_hidden=128, clip_intermediate=256, clip_layers=3, clip_heads=2, image_size=56)
    st = ParamStore(d, "cpu")
    assert [b.name for b in st.buckets] == ["embed", "layer0", "layer1", "head", "projector"]
    for b in st.buckets:
        assert b.size % ParamStore.PAD == 0 and b.start % 8 == 0 and b.decay_size % 8 == 0
        for s in b.segments:
            assert s.offset % 8 == 0
    views = st.hf_views()
    n_named = sum(v.numel() for v in views.values())
    assert n_named == sum(math.prod(s.shape) for b in st.buckets for s in b.segments)
    # fused views alias the flat storage
    views["model.layers.1.self_attn.k_proj.weight"].fill_(3.0)
    assert float(st.p["l1.qkv"][256:512].float().mean()) == 3.0
    assert float(st.p["l1.qkv"][:256].float().abs().sum()) == 0.0
    # no-decay tail holds exactly the norm weights / biases
    lb = st.buckets[1]
    assert [s.name for s in lb.segments if not s.decay] == ["l0.ln1", "l0.ln2"]


def test_cosine_schedule_matches_hf():
    from transformers import get_cosine_schedule_with_warmup
    from rlaifv_b200.zero2 import cosine_lr
    total, base = 200, 5e-7
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.SGD([p], lr=base)
    sch = get_cosine_schedule_with_warmup(opt, math.ceil(total * 0.05), total)
    for step in range(total):
        assert abs(opt.param_groups[0]["lr"] - cosine_lr(step, total, base, 0.05)) < 1e-15
        opt.step()
        sch.step()


def test_product_path_never_imports_the_oracle():
    pkg = os.path.join(REPO, "rlaif-v_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(root, f)).read()
                assert "oracle" not in src.replace("oracle/", ""), f


def test_missing_extension_fails_loudly(tmp_path, monkeypatch):
    from rlaifv_b200 import lib
    monkeypatch.setattr(lib, "_lib", None)
    monkeypatch.setattr(lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(lib.B200Error):
        lib.load()
