"""The fp8 Linear mode without a GPU: the reference row quantiser on edge rows, the fp8 reference forward against the
oracle, and the argument checks of the fp8 C entry points (they return G3C_EINVAL before touching memory)."""
import pytest
import torch

from oracle import cases, dit_oracle
from tests import fp8_oracle

E4M3_VALUES = None


def e4m3_grid() -> torch.Tensor:
    """Every finite non-negative e4m3fn value (the 127 bit patterns below 0x7f)."""
    global E4M3_VALUES
    if E4M3_VALUES is None:
        E4M3_VALUES = torch.arange(127, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
    return E4M3_VALUES


def test_quantiser_edge_rows():
    q = fp8_oracle.quantize_rows_e4m3
    # zero row: codes 0, scale 1
    c, s = q(torch.zeros(2, 32))
    assert torch.equal(c.float(), torch.zeros(2, 32)) and torch.equal(s, torch.ones(2))
    # values at +-448 with amax 448: inv = 1, every e4m3 value (subnormals included) is reproduced exactly, with sign
    g = e4m3_grid()
    row = torch.cat([g, -g])[None]
    c, s = q(row)
    assert float(s[0]) == 1.0 and torch.equal(c.float(), row)
    # values in e4m3's subnormal range (below 2^-6) round to the nearest multiple of 2^-9, ties to even
    row = torch.tensor([[448.0, 2.0 ** -9, 1.5 * 2.0 ** -9, 2.5 * 2.0 ** -9, 2.0 ** -11, -3 * 2.0 ** -9]])
    c, _ = q(row)
    assert c.float()[0, 1:].tolist() == [2.0 ** -9, 2 * 2.0 ** -9, 2 * 2.0 ** -9, 0.0, -3 * 2.0 ** -9]
    # a single outlier takes code 448 and squeezes the rest of its row
    row = torch.full((1, 64), 0.01)
    row[0, 5] = -1000.0
    c, s = q(row)
    assert float(c.float()[0, 5]) == -448.0 and float(s[0]) == pytest.approx(1000.0 / 448.0, rel=1e-7)
    # 0.01 * 448 / 1000 = 0.00448 = 2.29 * 2^-9: pushed into the subnormal range, code 2 * 2^-9
    assert torch.all(c.float()[0, torch.arange(64) != 5] == 2 * 2.0 ** -9)
    # random rows: dequantised error within half an e4m3 step (2^-4 relative for normal codes), negatives symmetric
    x = torch.randn(16, 256, generator=torch.Generator().manual_seed(0)) * torch.logspace(-3, 3, 16)[:, None]
    c, s = q(x)
    cn, sn = q(-x)
    assert torch.equal(cn.float(), -c.float()) and torch.equal(sn, s)
    deq = c.float() * s[:, None]
    assert torch.all((deq - x).abs() <= x.abs() * 2 ** -4 + s[:, None] * 2 ** -10)
    # the IEEE arithmetic of the contract: scale = amax / 448, codes = rn(x * (448 / amax))
    amax = x.abs().amax(1)
    assert torch.equal(s, amax / torch.full_like(amax, 448.0))


def _tiny(fn):
    cfg, shp = cases.TINY, cases.TINY_SHAPE
    sd = dit_oracle.random_state_dict(cfg, seed=0)
    inp = cases.dit_inputs(cfg, **shp)
    return fn(sd, cfg, inp["x"], inp["cond_mask"], inp["pose"], inp["padding"], inp["timestep"], inp["ctx_c"])


def test_fp8_oracle_is_the_oracle_with_quantised_linears(monkeypatch):
    """With the quantisation taken out, the fp8 reference is dit_oracle.forward bit for bit (it restates the same graph op
    for op); with it, the tiny net's output moves measurably (4.2e-4 rel-L2 on this case), not by 0 and not by more than
    the bf16 bar (5e-3)."""
    base = _tiny(dit_oracle.forward)
    f8 = _tiny(fp8_oracle.forward)
    err = float((f8 - base).norm() / base.norm())
    print(f"oracle fp8 vs fp32 rel-L2 {err:.3e}")
    assert 1e-4 < err < 5e-3, err
    monkeypatch.setattr(fp8_oracle, "linear_fp8", lambda a, w: a @ w.T)
    assert torch.equal(_tiny(fp8_oracle.forward), base)


def test_linear_fp8_is_the_scaled_code_product():
    g = torch.Generator().manual_seed(3)
    a, w = torch.randn(5, 48, generator=g), torch.randn(7, 48, generator=g)
    ca, sa = fp8_oracle.quantize_rows_e4m3(a)
    cw, sw = fp8_oracle.quantize_rows_e4m3(w)
    want = (ca.double() @ cw.double().T) * sa.double()[:, None] * sw.double()[None, :]
    got = fp8_oracle.linear_fp8(a, w)
    assert torch.allclose(got.double(), want, rtol=1e-6, atol=1e-6)
    assert float((got - a @ w.T).norm() / (a @ w.T).norm()) < 0.05


P = 1 << 20  # aligned, never dereferenced: the checks come first
BAD_GEMM = [
    (dict(K=40, lda=40, ldb=40), "multiples of 16"),
    (dict(lda=72), "multiples of 16"),
    (dict(sa=0), "null scale"),
    (dict(sb=P + 4), "16-byte aligned"),
    (dict(M=0), "bad shape"),
    (dict(ldd=8), "leading dimension"),
    (dict(block_n=96), "block_n"),
]


@pytest.mark.parametrize("over,what", BAD_GEMM)
def test_gemm_fp8_argument_checks(over, what):
    from gen3c_b200 import _lib

    lib = _lib.load()
    a = dict(M=128, N=128, K=64, lda=64, ldb=64, ldd=128, epi=0, sa=P, sb=P, block_n=0)
    a.update(over)
    rc = lib.g3c_gemm_fp8(P, a["sa"] or None, P, a["sb"], P, a["M"], a["N"], a["K"], a["lda"], a["ldb"], a["ldd"],
                          a["epi"], None, a["block_n"], None)
    msg = lib.g3c_last_error().decode()
    assert rc == -1 and what in msg, msg


def test_norm_rope_fp8_and_quantiser_argument_checks():
    from gen3c_b200 import _lib

    lib = _lib.load()
    assert lib.g3c_gemm_norm_rope_fp8(P, P, P, P, P, 128, 96, 64, 64, 64, 96, P, None, 1e-6, None) == -1
    assert "N % 128" in lib.g3c_last_error().decode()
    assert lib.g3c_gemm_norm_rope_fp8(P, P, P, None, P, 128, 128, 64, 64, 64, 128, P, None, 1e-6, None) == -1
    assert "null scale" in lib.g3c_last_error().decode()
    for args, what in (((P, 64, 4, 24, P, 32, P), "multiple of 16"),
                       ((P, 60, 4, 48, P, 48, P), "leading dimensions"),
                       ((P, 64, 4, 64, P, 56, P), "leading dimensions"),
                       ((P + 8, 64, 4, 64, P, 64, P), "aligned"),
                       ((P, 64, 4, 64, P, 64, P + 4), "aligned"),
                       ((P, 64, 0, 64, P, 64, P), "positive")):
        assert lib.g3c_quantize_rows_fp8(*args, None) == -1
        assert what in lib.g3c_last_error().decode(), (args, lib.g3c_last_error())
    assert lib.g3c_ln_modulate_fp8(P, None, P, P, P + 8, P, 4, 64, 1e-6, None) == -1
    assert "aligned" in lib.g3c_last_error().decode()
    assert lib.g3c_ln_modulate_fp8(P, None, P, P, P, P, 4, 72, 1e-6, None) == -1
    assert "unsupported" in lib.g3c_last_error().decode()
    assert lib.g3c_dit_set_linear_fp8(None, 1) == -1


def test_fp8_entry_points_refuse_malformed_tensors():
    from gen3c_b200 import ops

    with pytest.raises(ValueError):
        ops.quantize_rows_fp8(torch.zeros(4, 64, dtype=torch.bfloat16))  # not on the GPU
    with pytest.raises(ValueError):
        ops.gemm_fp8(torch.zeros(4, 64).to(torch.float8_e4m3fn), torch.ones(4), torch.zeros(4, 64).to(torch.float8_e4m3fn),
                     torch.ones(4))


def test_fp8_flag_and_module_surface():
    from gen3c_b200.dit import VideoExtendGeneralDIT
    from gen3c_b200.inference import gen3c_single_image as m

    p = m.create_parser()
    assert p.parse_args([]).fp8_linear is False and p.parse_args(["--fp8_linear"]).fp8_linear is True
    net = VideoExtendGeneralDIT(model_channels=256, num_blocks=1, num_heads=2, adaln_lora_dim=32, device="cpu")
    assert net.is_fp8_linear_enabled is False
    assert not any("fp8" in k for k in net.state_dict())
