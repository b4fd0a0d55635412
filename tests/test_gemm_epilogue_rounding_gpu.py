"""The GEMM epilogues are exact roundings of one fp32 accumulator.  On the same operands the f32 epilogue returns the
accumulator acc itself, and then, bit for bit:

  * the bf16 epilogue returns RN_bf16(acc);
  * the gated residual turns x0 into RN(x0 + RN(gate * acc)): the product is rounded to fp32 before TMA adds it into x
    in L2, so the expectation is two separate fp32 operations (not a fused multiply-add).

Covered for bf16 tiles of 64 / 128 / 256 columns and fp8 tiles of 64 / 128, at M / N / K tails (including a last row
block whose second 64-row half lies past M), at tile counts above twice the SM count (each consumer warpgroup reuses
its staging buffer across tiles), and at one engine shape."""
import pytest
import torch

from gen3c_b200 import ops

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def _check(M, N, K, block_n, fp8, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    b = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    gate = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(M, N, device="cuda", generator=g)
    if fp8:
        a8, sa = ops.quantize_rows_fp8(a)
        b8, sb = ops.quantize_rows_fp8(b)

        def run(epi, out=None, gate=None):
            return ops.gemm_fp8(a8, sa, b8, sb, epi, out=out, gate=gate, block_n=block_n)
    else:
        def run(epi, out=None, gate=None):
            return ops.gemm(a, b, epi, out=out, gate=gate, block_n=block_n)

    acc = run(ops.EPI_F32)
    bf = run(ops.EPI_BF16)
    x = x0.clone()
    run(ops.EPI_GATED_RESIDUAL_F32, out=x, gate=gate)
    torch.cuda.synchronize()
    assert torch.isfinite(acc).all()
    want_bf = acc.to(torch.bfloat16)
    assert torch.equal(_bits(bf), _bits(want_bf)), f"bf16 epilogue: {int((bf != want_bf).sum())} elements differ"
    prod = gate[None, :] * acc
    want_x = x0 + prod
    assert torch.equal(_bits(x), _bits(want_x)), f"gated residual: {int((x != want_x).sum())} elements differ"


# (M, N, K): tails in every dimension, M % 128 below and above 64 (the second warpgroup's rows past M, or partly)
TAILS = [(300, 200, 264), (1000, 456, 136)]
# more than 2 x 132 tiles for every tile width: 65 x 5 = 325 tiles at 256 columns
MANY_TILES = [(8264, 1048, 256)]


@pytest.mark.parametrize("block_n", [64, 128, 256])
@pytest.mark.parametrize("shape", TAILS + MANY_TILES)
def test_bf16_epilogues_round_the_accumulator(shape, block_n):
    _check(*shape, block_n=block_n, fp8=False, seed=block_n)


@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("shape", [(300, 200, 272), (1000, 456, 144)] + MANY_TILES)
def test_fp8_epilogues_round_the_accumulator(shape, block_n):
    _check(*shape, block_n=block_n, fp8=True, seed=block_n + 1)


def test_engine_shape_epilogues_round_the_accumulator():
    # to_out of the benchmark's latent: 56 320 tokens x 4096 x 4096, the automatic (256-column) tile
    _check(56320, 4096, 4096, block_n=0, fp8=False, seed=7)
