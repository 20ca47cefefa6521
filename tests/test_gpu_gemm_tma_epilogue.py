"""-m gpu: the staged epilogue of the GEMM's plain, residual and SwiGLU-backward forms (gemm.cu: epilogue_staged, C
written through shared memory by TMA stores) against the register epilogue of the same forms, which
rlaifv_gemm_set_tuning's debug bit 1 forces. The two must give the same bits, and a second staged run the same bits
again.

The cases cover the tiles 128, 256 and 512 (the 2-CTA pair), the LoRA second source, M tails (including 64-row halves
and CTAs of a pair whose rows all lie past M), N tails, column-block views whose neighbouring columns must stay
untouched, a C that is its own residual, a 4-byte-aligned residual (register epilogue) and persistent walks of at
least three tiles per CTA, which reuse the staging buffers across tiles."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16

# "walk": at least 3 tiles per CTA (or 2-CTA cluster) on a 132-SM H100 at every tile size:
#   tile 128: 33 x 32 = 1056 tiles, 256: 33 x 16 = 528, 512: 17 x 16 = 272 (66 clusters)
# "tails": M = 2100 = 16 * 128 + 52 (the last 256-row block has a 52-row warpgroup, an empty warpgroup and, on the
#   pair, an empty CTA), N = 1000 = 15 * 64 + 40
SHAPES = {"walk": (4200, 4096, 256), "tails": (2100, 1000, 200)}


def _rand(shape, g):
    return torch.randn(*shape, generator=g).to(BF).to(DEV)


@contextlib.contextmanager
def _register_epilogue():
    from rlaifv_b200 import lib
    L = lib.load()
    L.rlaifv_gemm_set_tuning(0, 2)
    try:
        yield
    finally:
        L.rlaifv_gemm_set_tuning(0, 0)


def _staged_matches_register(fn):
    """fn() -> tensor; staged, register, staged again: all bit-identical. Returns the staged result."""
    first = fn().clone()
    with _register_epilogue():
        reg = fn().clone()
    again = fn().clone()
    assert torch.equal(first, reg)
    assert torch.equal(first, again)
    return first


def _operands(shape, b_mn, seed):
    M, N, K = SHAPES[shape]
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = _rand((M, K), g)
    b = _rand((K, N) if b_mn else (N, K), g)
    res = _rand((M, N), g)
    return a, b, res


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("tile_n", [128, 256, 512])
@pytest.mark.parametrize("epi", ["plain", "residual"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_staged_plain_residual_match_register_epilogue(shape, tile_n, epi, b_mn):
    from rlaifv_b200 import ops
    a, b, res = _operands(shape, b_mn, 1)
    out = _staged_matches_register(
        lambda: ops.gemm(a, b, b_mn=b_mn, residual=res if epi == "residual" else None, tile_n=tile_n))
    assert bool(torch.isfinite(out.float()).all())


@pytest.mark.parametrize("tile_n", [128, 256, 512])
def test_staged_wgrad_plain_matches_register_epilogue(tile_n):
    from rlaifv_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(2)
    dy, x = _rand((1000, 2104), g), _rand((1000, 520), g)     # dW [2104, 520] = dy^T x, K = 1000
    _staged_matches_register(lambda: ops.gemm(dy, x, a_mn=True, b_mn=True, tile_n=tile_n))


@pytest.mark.parametrize("shape", sorted(SHAPES))      # automatic tile: 512 for "walk", 128 for "tails"
@pytest.mark.parametrize("epi", ["plain", "residual"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_staged_lora_second_source_matches_register_epilogue(shape, epi, b_mn):
    from rlaifv_b200 import ops
    M, N, K = SHAPES[shape]
    a, b, res = _operands(shape, b_mn, 3)
    g = torch.Generator(device="cpu").manual_seed(4)
    a2 = _rand((M, 64), g)
    b2 = _rand((64, N) if b_mn else (N, 64), g)
    _staged_matches_register(lambda: ops.gemm_dual(a, b, a2, b2, torch.empty(M, N, dtype=BF, device=DEV), k2=64, r=64,
                                                   b_mn=b_mn, residual=res if epi == "residual" else None))


# automatic tile: 512 with 4+ tiles per cluster for (4200, 4096), 128 for (1000, 1024)
@pytest.mark.parametrize("mf", [(4200, 4096), (1000, 1024)], ids=["pair_walk", "tile128"])
@pytest.mark.parametrize("lora", [False, True], ids=["base", "lora"])
@pytest.mark.parametrize("b_mn", [False, True], ids=["w_kmajor", "w_mnmajor"])
def test_staged_swiglu_bwd_matches_register_epilogue(mf, lora, b_mn):
    from rlaifv_b200 import ops
    M, F = mf
    K = 320
    g = torch.Generator(device="cpu").manual_seed(5)
    dy = _rand((M, K), g)
    w = _rand((K, F) if b_mn else (F, K), g)
    gu = _rand((M, 2 * F), g)
    a2 = _rand((M, 64), g) if lora else None
    b2 = (_rand((64, F) if b_mn else (F, 64), g)) if lora else None
    out = _staged_matches_register(
        lambda: ops.gemm_swiglu_bwd(dy, w, gu, torch.empty(M, 2 * F, dtype=BF, device=DEV), b_mn=b_mn, a2=a2, b2=b2))
    assert bool(torch.isfinite(out.float()).all())


@pytest.mark.parametrize("tile_n", [128, 256, 512])
@pytest.mark.parametrize("epi", ["plain", "residual", "swiglu_bwd"])
def test_staged_column_block_view_leaves_neighbours_untouched(tile_n, epi):
    """C is columns [8, 8 + width) of a wider buffer; the columns around it keep their bits."""
    from rlaifv_b200 import ops
    M, N, K = SHAPES["tails"]
    if epi == "swiglu_bwd":
        N = 1024                                  # F % 64 == 0; C is [M, 2F]
    width = 2 * N if epi == "swiglu_bwd" else N
    g = torch.Generator(device="cpu").manual_seed(6)
    a, b = _rand((M, K), g), _rand((N, K), g)
    res, gu = _rand((M, N), g), _rand((M, 2 * N), g)
    fill = _rand((M, width + 24), g)

    def run():
        buf = fill.clone()
        c = buf[:, 8:8 + width]
        if epi == "swiglu_bwd":
            ops.gemm_swiglu_bwd(a, b, gu, c, b_mn=False)
        else:
            ops.gemm(a, b, out=c, residual=res if epi == "residual" else None, tile_n=tile_n)
        return buf

    buf = _staged_matches_register(run)
    assert torch.equal(buf[:, :8], fill[:, :8])
    assert torch.equal(buf[:, 8 + width:], fill[:, 8 + width:])


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("tile_n", [128, 256, 512])
def test_staged_residual_aliasing_c(shape, tile_n):
    """out is its own residual: every element must still be bf16(bf16(acc) + old value)."""
    from rlaifv_b200 import ops
    a, b, res = _operands(shape, False, 7)
    want = ops.gemm(a, b, residual=res, tile_n=tile_n).clone()

    def run():
        buf = res.clone()
        return ops.gemm(a, b, out=buf, residual=buf, tile_n=tile_n)

    assert torch.equal(_staged_matches_register(run), want)


@pytest.mark.parametrize("tile_n", [128, 512])
def test_4byte_aligned_residual_takes_register_epilogue(tile_n):
    """A residual view 4 bytes into its row (ldr % 8 != 0) cannot be a tensor map: the register epilogue runs it, with
    the same bits as the staged epilogue on a 16-byte-aligned copy."""
    from rlaifv_b200 import ops
    a, b, res = _operands("tails", False, 8)
    M, N, _ = SHAPES["tails"]
    wide = torch.zeros(M, N + 2, dtype=BF, device=DEV)
    wide[:, 2:] = res
    view = wide[:, 2:]
    assert view.data_ptr() % 16 == 4 and view.stride(0) % 8 != 0
    got = _staged_matches_register(lambda: ops.gemm(a, b, residual=view, tile_n=tile_n))
    assert torch.equal(got, ops.gemm(a, b, residual=res, tile_n=tile_n))
