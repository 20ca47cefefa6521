"""-m gpu bit identity of the GEMM's specialised epilogue forms (gemm.cu: EpiKind).

Plain, residual and SwiGLU-backward launches run their own kernel instantiations. Their results must not depend on
the tile form, the raster or the L2 hints, the residual form must give exactly bf16(bf16(A B^T) + residual), the
rounding points of the general epilogue, and the SwiGLU form must agree with the unfused path on the cluster tile the
real down-projection dgrad runs on."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16

# rows not a multiple of the 256-row cluster tile, N not a multiple of 256: the ragged tile edges take part
M, N, K = 2100, 1088, 520


def _operands(b_mn, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(BF).to(DEV)
    b = (torch.randn(K, N, generator=g) if b_mn else torch.randn(N, K, generator=g)).to(BF).to(DEV)
    res = torch.randn(M, N, generator=g).to(BF).to(DEV)
    return a, b, res


@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_gemm_residual_form_is_plain_gemm_plus_bf16_add(b_mn):
    from rlaifv_b200 import ops
    a, b, res = _operands(b_mn, 1)
    plain = ops.gemm(a, b, b_mn=b_mn, tile_n=512)
    fused = ops.gemm(a, b, b_mn=b_mn, residual=res, tile_n=512)
    assert torch.equal(fused, (plain.float() + res.float()).to(BF))


@pytest.mark.parametrize("epi", ["plain", "residual", "swiglu_bwd"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_gemm_epilogue_forms_bit_identical_across_tiles_and_rasters(epi, b_mn):
    from rlaifv_b200 import lib, ops
    L = lib.load()
    a, b, res = _operands(b_mn, 2)
    gen = torch.Generator(device="cpu").manual_seed(3)
    gu = torch.randn(M, 2 * N, generator=gen).to(BF).to(DEV)

    def run(tile_n):
        if epi == "swiglu_bwd":
            # automatic tile choice only (tile 128 at this shape; the cluster tile has its own test below); the raster
            # settings still vary
            return ops.gemm_swiglu_bwd(a, b, gu, torch.empty(M, 2 * N, dtype=BF, device=DEV), b_mn=b_mn).clone()
        return ops.gemm(a, b, b_mn=b_mn, residual=res if epi == "residual" else None, tile_n=tile_n).clone()

    outs = []
    try:
        for tile_n in (512, 256, 128):
            outs.append(run(tile_n))
        for group, l2 in ((4, 0), (8, 0x40 | 1 | (2 << 2)), (2, 2 | (1 << 2))):
            L.rlaifv_gemm_set_tuning(group, 0)
            L.rlaifv_gemm_set_l2(l2)
            outs.append(run(512))
    finally:
        L.rlaifv_gemm_set_tuning(16, 0)
        L.rlaifv_gemm_set_l2(-1)
    assert bool(torch.isfinite(outs[0].float()).all())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


@pytest.mark.parametrize("k2", [0, 64])
def test_gemm_swiglu_bwd_form_on_the_cluster_tile(k2):
    """The SwiGLU-backward form at the 2-CTA 256 x 256 tile, which the automatic choice takes for the real down-projection
    dgrad: each row of a thread's accumulators is read in two groups of 16 gate|up pairs. F = 2048 at M = 2100 is 72
    cluster tiles, enough for that choice. Against the unfused path (GEMM, then swiglu_bwd), which differs only by an
    approximate reciprocal (at most one bf16 ulp), and bitwise across rasters."""
    from rlaifv_b200 import lib, ops
    L = lib.load()
    Mg, F, Kg = 2100, 2048, 520
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert -(-Mg // 256) * (F // 256) >= sms // 2          # gemm_impl's rule for the cluster tile
    gen = torch.Generator(device="cpu").manual_seed(5)
    dy = (torch.randn(Mg, Kg, generator=gen) * 0.5).to(BF).to(DEV)
    w = (torch.randn(Kg, F, generator=gen) * 0.1).to(BF).to(DEV)       # W_down stored [H, F]: MN-major B operand
    gu = torch.randn(Mg, 2 * F, generator=gen).to(BF).to(DEV)
    a2 = b2 = None
    if k2:
        a2 = (torch.randn(Mg, k2, generator=gen) * 0.5).to(BF).to(DEV)
        b2 = (torch.randn(k2, F, generator=gen) * 0.1).to(BF).to(DEV)

    def fused():
        return ops.gemm_swiglu_bwd(dy, w, gu, torch.empty(Mg, 2 * F, dtype=BF, device=DEV), a2=a2, b2=b2).clone()

    outs = []
    try:
        outs.append(fused())
        for group, l2 in ((4, 0), (8, 0x40 | 1 | (2 << 2))):
            L.rlaifv_gemm_set_tuning(group, 0)
            L.rlaifv_gemm_set_l2(l2)
            outs.append(fused())
    finally:
        L.rlaifv_gemm_set_tuning(16, 0)
        L.rlaifv_gemm_set_l2(-1)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    if k2:
        dact = torch.empty(Mg, F, dtype=BF, device=DEV)
        ops.gemm_dual(dy, w, a2, b2, dact, k2=k2, r=k2, n_sub=0, b_mn=True)
    else:
        dact = ops.gemm(dy, w, b_mn=True)
    two_step = ops.swiglu_bwd(gu, dact).float()
    err = (outs[0].float() - two_step).abs()
    ulp = two_step.abs() * 2.0 ** -7 + 1e-30                          # one bf16 ulp of the unfused result, at most
    assert bool((err <= ulp).all()), float((err / ulp).max())


def test_gemm_resident_cluster_query():
    import ctypes
    from rlaifv_b200 import lib
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for tile_n, cl in ((512, 2), (256, 1), (128, 1)):
        n = ctypes.c_int(0)
        lib.call("rlaifv_gemm_max_active_clusters", tile_n, ctypes.byref(n))
        assert 1 <= n.value <= sms // cl
