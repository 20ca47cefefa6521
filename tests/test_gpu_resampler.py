"""-m gpu: perceiver-resampler piece of BASELINE config (d) (SURVEY.md §8 a13) through the C ABI —
cross-attention fwd/bwd (wgmma, shared learned queries), LayerNorm backward, position add, and the whole
`Resampler` forward + backward against the oracle that is pinned to the unmodified reference class
(oracle/gen_golden_resampler.py). Tolerances: bf16 storage vs fp32 oracle => norm-relative errors of ~1e-2."""
import glob
import math
import os

import numpy as np
import pytest
import torch

from oracle import resampler_oracle as R

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "resampler", "*.npz")))


def nrel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("nseq,Sq,Skv,nh,D,shared", [(3, 16, 144, 2, 128, True), (2, 64, 1024, 4, 128, True),
                                                    (2, 200, 333, 2, 128, False), (2, 64, 300, 2, 64, True)])
def test_cross_attention_forward_backward(nseq, Sq, Skv, nh, D, shared):
    from rlaifv_b200 import ops
    g = torch.Generator().manual_seed(7)
    E = nh * D
    q = (torch.randn((1 if shared else nseq) * Sq, E, generator=g)).to(torch.bfloat16).cuda()
    k = torch.randn(nseq * Skv, E, generator=g).to(torch.bfloat16).cuda()
    v = torch.randn(nseq * Skv, E, generator=g).to(torch.bfloat16).cuda()
    do = (0.5 * torch.randn(nseq * Sq, E, generator=g)).to(torch.bfloat16).cuda()
    scale = 1.0 / math.sqrt(D)
    out, lse = ops.cross_attention_fwd(q, k, v, nseq, Sq, Skv, nh, D, scale, q_shared=shared)
    # fp32 reference
    qf = q.float().view(-1, Sq, nh, D).permute(0, 2, 1, 3).clone().requires_grad_(True)       # [1|nseq, nh, Sq, D]
    kf = k.float().view(nseq, Skv, nh, D).permute(0, 2, 1, 3).clone().requires_grad_(True)
    vf = v.float().view(nseq, Skv, nh, D).permute(0, 2, 1, 3).clone().requires_grad_(True)
    s = torch.matmul(qf * scale, kf.transpose(-1, -2))                                         # broadcasts shared q
    ref = torch.matmul(torch.softmax(s, -1), vf)                                               # [nseq, nh, Sq, D]
    ref_out = ref.permute(0, 2, 1, 3).reshape(nseq * Sq, E)
    assert nrel(out, ref_out) < 8e-3
    assert torch.allclose(lse, torch.logsumexp(s, -1).detach(), atol=2e-3, rtol=1e-4)
    if D != 128:
        return
    ref_out.backward(do.float())
    dq32 = torch.zeros_like(q, dtype=torch.float32)
    dk, dv = torch.empty_like(k), torch.empty_like(v)
    ops.cross_attention_bwd(q, k, v, out, do, lse, nseq, Sq, Skv, nh, D, scale, dq32, dk, dv, q_shared=shared)
    torch.cuda.synchronize()
    unperm = lambda t, S: t.permute(0, 2, 1, 3).reshape(-1, E)
    assert nrel(dq32, unperm(qf.grad, Sq)) < 1.5e-2          # shared: summed over the batch by the fp32 atomics
    assert nrel(dk, unperm(kf.grad, Skv)) < 1.5e-2
    assert nrel(dv, unperm(vf.grad, Skv)) < 1.5e-2


def test_layernorm_backward_and_row_broadcast_add():
    from rlaifv_b200 import ops
    g = torch.Generator().manual_seed(3)
    for M, H in ((300, 256), (70, 4096), (5, 512)):
        x = (torch.randn(M, H, generator=g) * 2 + 0.3).to(torch.bfloat16).cuda()
        w = (1 + 0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
        b = (0.1 * torch.randn(H, generator=g)).to(torch.bfloat16).cuda()
        dy = torch.randn(M, H, generator=g).to(torch.bfloat16).cuda()
        xf, wf, bf = x.float().requires_grad_(True), w.float().requires_grad_(True), b.float().requires_grad_(True)
        y = torch.nn.functional.layer_norm(xf, (H,), wf, bf, 1e-6)
        y.backward(dy.float())
        assert nrel(ops.layernorm_fwd(x, w, b, 1e-6), y) < 4e-3
        dx = torch.empty_like(x)
        dw = torch.zeros(H, dtype=torch.bfloat16, device="cuda")
        db = torch.zeros(H, dtype=torch.bfloat16, device="cuda")
        ops.layernorm_bwd(dy, x, w, 1e-6, dx, dw, db, accumulate=False)
        assert nrel(dx, xf.grad) < 5e-3 and nrel(dw, wf.grad) < 5e-3 and nrel(db, bf.grad) < 5e-3
        ops.layernorm_bwd(dy, x, w, 1e-6, dx, dw, db, accumulate=True)          # accumulate doubles dw / db
        assert nrel(dw, 2 * wf.grad) < 8e-3 and nrel(db, 2 * bf.grad) < 8e-3
    t = torch.randn(7, 64, generator=g).to(torch.bfloat16).cuda()
    x = torch.randn(21, 64, generator=g).to(torch.bfloat16).cuda()
    want = (x.float().view(3, 7, 64) + t.float()).view(21, 64).to(torch.bfloat16)
    assert torch.equal(ops.add_rows_bcast(x, t), want)                           # single rounding: bit-exact


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_resampler_module_matches_oracle_and_reference_fixture(path):
    from rlaifv_b200.resampler import Resampler
    fx = np.load(path)
    cfg = R.R_CONFIGS[str(fx["cfg_name"])]
    B, seed = int(fx["B"]), int(fx["seed"])
    p32 = R.make_resampler_params(cfg, seed=seed)
    m = Resampler(cfg.grid_size, cfg.embed_dim, cfg.num_heads, cfg.kv_dim, "cuda", state=p32)
    x, d_out = R.synthetic_vision_tokens(cfg, B, seed + 100)
    xb, db = x.to(torch.bfloat16), d_out.to(torch.bfloat16)
    y = m(xb.cuda())
    dx = m.backward(db.cuda())
    torch.cuda.synchronize()
    # oracle on the SAME bf16-rounded weights / inputs, fp32 arithmetic
    po = {k: v.to(torch.bfloat16).float().requires_grad_(k != "pos_embed") for k, v in p32.items()}
    xo = xb.float().requires_grad_(True)
    yo = R.resampler_forward(po, xo, cfg)
    yo.backward(db.float())
    assert nrel(y, yo) < 1.2e-2, nrel(y, yo)
    assert nrel(dx, xo.grad) < 2.5e-2, nrel(dx, xo.grad)
    for name in R.PARAM_SHAPES(cfg):
        e = nrel(m.g[name], po[name].grad)
        print(f"{name}: grad norm-relative error {e:.3e}")
        assert e < 2.5e-2, (name, e)
    # and against the fixture written by the unmodified reference class (fp32 weights): same numbers up to bf16
    f = y.float().flatten().cpu()
    got = f[torch.linspace(0, f.numel() - 1, 256).long()].numpy()
    assert np.abs(got - fx["out_sample"]).max() <= 4e-2 * np.abs(fx["out_sample"]).max()
    assert abs(float(y.float().norm()) - float(fx["out_norm"])) <= 1e-2 * float(fx["out_norm"])
    assert abs(float(dx.float().norm()) - float(fx["dx_norm"])) <= 2e-2 * float(fx["dx_norm"])
    for key in fx.files:
        if key.startswith("gradnorm:"):
            name = key.split(":", 1)[1]
            assert abs(float(m.g[name].float().norm()) - float(fx[key])) <= 3e-2 * float(fx[key]), name
    # gradients accumulate: a second forward/backward doubles them
    before = m.grad.float().clone()
    m(xb.cuda())
    m.backward(db.cuda())
    assert nrel(m.grad.float(), 2 * before) < 1e-2
