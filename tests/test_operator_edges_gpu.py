"""The edges of the C ABI's operators, called directly (not through `ops`, which always passes packed leading
dimensions): the GEMM in bf16 and fp8 at K / N / M tails, with strided operands whose padding holds NaN, strided outputs
inside guard bands, persistent tile counts around the SM count and a narrower last super-column; the row kernels and
the attention output with strided outputs; and the documented argument errors, which must not launch anything.

Every output is a view into a larger buffer filled with a NaN bit pattern no kernel produces by accident.  The bands
are at least one tile (128 rows after the end, 256 columns of row gap where the ABI allows it), so a kernel that
ignores its bounds writes into the band, where the check sees it, and never past the allocation.

References are float64 on the GPU, from the operands' exact values.  Besides one relative L2 error per output, every
GEMM element is held to a bound scaled by its own conditioning S = |A| . |B|^T: one wrong element of a large output
moves the relative L2 error by far less than its tolerance, but it breaks its own bound."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from tests import fp8_oracle

pytestmark = pytest.mark.gpu

BF16, GELU, GATED, F32 = 0, 1, 2, 3
EINVAL = -1
E4M3 = torch.float8_e4m3fn

# The per-element constants below are set to about 4x the largest ratio observed over the cases of this file on one
# H100 80GB HBM3 (132 SMs, 700 W power limit).
# bf16 operands, fp32 wgmma sums: |error| / S reached 1.20e-6 (about 20 * 2^-24).  S grows with K, and the ratio stays
# at a few roundings of the tensor core's sum rather than growing like sqrt(K) * 2^-24 (7.6e-6 at K = 16384).  It is not
# quite flat: at the engine's shapes (test_engine_shapes_gpu.py) it went from 2.8e-7 at K = 384 to 7.6e-7 at K = 4096
# and 1.5e-6 at K = 16384, the largest K the engine runs.
C32 = 4.5e-6
# fp8 operands: 3.6e-4 (about 2^-11.5; 2.0e-4 over the shape matrix).  The e4m3 instruction keeps only about 14 bits of
# its own k32 sum (the DeepSeek-V3 report measured the same on Hopper), so every element carries that much of its S.
# The kernel adds each k-block's partial sum in fp32, so the ratio does not grow with K either.
C8 = 1.4e-3
# attention: |o - ref| <= 2^-8 |ref| + C_ATT * (P . |V|).  P is rounded to bf16 for the P.V product (up to 2^-8 of each
# term), and most of that cancels: 8.9e-4 observed.
C_ATT = 3.5e-3
# LayerNorm statistics in fp32: |y - ref| <= 2^-8 |ref| + C_LN * 2^-24 sqrt(D) mean|x| rstd |1 + scale|.  Observed 0.33,
# on rows offset by 1e4 (the fp32 mean's rounding); 0.004 without the offset.
C_LN = 1.3

OBSERVED: dict = {}  # largest ratio per check, for re-deriving the constants above


def _note(key, value):
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), float(value))


def lib():
    from gen3c_b200 import _lib

    return _lib.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def sm_count():
    sm, ma, mi = C.c_int(), C.c_int(), C.c_int()
    assert lib().g3c_device_info(C.byref(sm), C.byref(ma), C.byref(mi)) == 0
    return sm.value


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rup(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------------------------
# guard-banded outputs and poisoned inputs
# ------------------------------------------------------------------------------------------------------------------
_BITS = {torch.float32: (torch.int32, 0x7FC01234), torch.bfloat16: (torch.int16, 0x7FA1), torch.uint8: (torch.uint8, 0x7F)}
LEAD = 4096  # elements before the view: a multiple of 16 bytes at every element size
GAP = 256  # columns of row gap where the ABI allows it: one widest tile


class Guarded:
    """A [rows, cols] view with leading dimension `ld` inside one flat buffer: LEAD elements, the view's rows (each with
    its ld - cols gap), then `after_rows` whole rows and GAP more elements.  Everything outside the view holds a NaN
    with a payload; the view holds `init`, or the same pattern."""

    def __init__(self, rows, cols, ld, dtype, init=None, after_rows=128):
        ity, pattern = _BITS[dtype]
        self.ld = ld
        after = rup(after_rows * ld + GAP, 16)
        n = LEAD + rows * ld + after
        self.buf = torch.empty(n, dtype=dtype, device="cuda")
        self.bits = self.buf.view(ity)
        self.bits.fill_(pattern)
        body = slice(LEAD, LEAD + rows * ld)
        self.view = self.buf[body].view(rows, ld)[:, :cols]
        if init is not None:
            self.view.copy_(init)
        self.inside = torch.zeros(n, dtype=torch.bool, device="cuda")
        self.inside[body].view(rows, ld)[:, :cols] = True
        self.before = self.bits.clone()

    @property
    def ptr(self):
        return self.view.data_ptr()

    def assert_outside_untouched(self):
        torch.cuda.synchronize()
        changed = (self.bits != self.before) & ~self.inside
        n = int(changed.sum())
        if n:
            first = int(changed.nonzero()[0, 0]) - LEAD
            where = f"row {first // self.ld} column {first % self.ld}" if first >= 0 else f"{-first} before the view"
            raise AssertionError(f"{n} elements written outside the output (first: {where}, ld {self.ld})")

    def assert_untouched(self):
        torch.cuda.synchronize()
        assert torch.equal(self.bits, self.before), "an erroring call wrote to its output"


def strided(values, ld, fill):
    """values [rows, cols] as a view of a [rows, ld] buffer whose columns past `cols` hold `fill` (raw bits for bf16 /
    uint8 buffers: NaN; or a float tensor broadcast to the gap)."""
    rows, cols = values.shape
    buf = torch.empty(rows, ld, dtype=values.dtype, device="cuda")
    if isinstance(fill, int):
        buf.view(_BITS[values.dtype][0]).fill_(fill)
    else:
        buf[:, cols:] = fill
    buf[:, :cols] = values
    return buf[:, :cols]


BF16_NAN, E4M3_NAN = 0x7FC0, 0x7F


def gate_vector(N, seed):
    """A random gate in [0.5, 1.5) followed by NaN: a kernel that reads the gate past N writes NaN."""
    buf = torch.full((N + GAP,), float("nan"), device="cuda")
    buf[:N] = torch.rand(N, device="cuda", generator=gen(seed)) + 0.5
    return buf[:N]


# ------------------------------------------------------------------------------------------------------------------
# GEMM: operands, calls, references and the per-element bound
# ------------------------------------------------------------------------------------------------------------------
def bf16_operands(M, N, K, lda, ldb, seed, spread=1.0):
    """Random bf16 operands in NaN-padded [., ld] buffers, their rows' magnitudes spread over 10^(+-spread)."""
    g = gen(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.logspace(-spread, spread, M, device="cuda")[:, None]
    b = torch.randn(N, K, device="cuda", generator=g) * (0.2 * torch.logspace(spread, -spread, N, device="cuda"))[:, None]
    a = strided(a.to(torch.bfloat16), lda, BF16_NAN)
    b = strided(b.to(torch.bfloat16), ldb, BF16_NAN)
    return a, b, None, None


def fp8_operands(M, N, K, lda, ldb, seed, spread=2.0):
    """Row-quantised codes (the quantiser's contract, restated in torch) in NaN-padded [., ld] buffers, and the row
    scales; a magnitude spread over the rows so that the scales matter."""
    g = gen(seed)
    a = torch.randn(M, K, device="cuda", generator=g) * torch.logspace(-spread, spread, M, device="cuda")[:, None]
    b = torch.randn(N, K, device="cuda", generator=g) * torch.logspace(spread, -spread, N, device="cuda")[:, None]
    ca, sa = fp8_oracle.quantize_rows_e4m3(a.to(torch.bfloat16))
    cb, sb = fp8_oracle.quantize_rows_e4m3(b.to(torch.bfloat16))
    return (strided(ca.view(torch.uint8), lda, E4M3_NAN), strided(cb.view(torch.uint8), ldb, E4M3_NAN),
            sa.contiguous(), sb.contiguous())


def dequant(codes, scale):
    return codes.view(E4M3).double() * scale.double()[:, None]


def reference(a, b, sa, sb):
    """fp64 product and its conditioning S = |A| . |B|^T, from the exact operand values."""
    if sa is None:
        ad, bd = a.double(), b.double()
    else:
        ad, bd = dequant(a, sa), dequant(b, sb)
    return ad @ bd.T, ad.abs() @ bd.abs().T


def call_gemm(a, b, sa, sb, out, epi, gate=None, bn=0):
    M, K = a.shape
    N = b.shape[0]
    gp = None if gate is None else gate.data_ptr()
    if sa is None:
        return lib().g3c_gemm_bf16(a.data_ptr(), b.data_ptr(), out.ptr, M, N, K, a.stride(0), b.stride(0), out.ld, epi,
                                   gp, bn, stream())
    return lib().g3c_gemm_fp8(a.data_ptr(), sa.data_ptr(), b.data_ptr(), sb.data_ptr(), out.ptr, M, N, K, a.stride(0),
                              b.stride(0), out.ld, epi, gp, bn, stream())


def out_ld(N, epi, pad_kind):
    q = 8 if epi in (BF16, GELU) else 4  # the ABI's ldd rule for bf16 / f32 outputs
    return rup(N, q) + (0, q, GAP)[pad_kind]


def run_gemm(a, b, sa, sb, epi, bn, ld, seed=0):
    """One guard-banded call; returns (output, x before the call, gate) after checking the bands."""
    M, N = a.shape[0], b.shape[0]
    dt = torch.bfloat16 if epi in (BF16, GELU) else torch.float32
    x0 = gate = None
    if epi == GATED:
        x0 = torch.randn(M, N, device="cuda", generator=gen(seed + 1)) * 8
        gate = gate_vector(N, seed + 2)
    out = Guarded(M, N, ld, dt, init=x0)
    assert call_gemm(a, b, sa, sb, out, epi, gate, bn) == 0, lib().g3c_last_error()
    out.assert_outside_untouched()
    return out.view, x0, gate


REL_TOL = {False: {BF16: 3e-3, GELU: 3e-3, GATED: 1e-5, F32: 1e-5},  # bf16 operands (test_dit_ops_gpu.py's bars)
           True: {BF16: 3e-3, GELU: 3e-3, GATED: 3e-4, F32: 3e-4}}  # fp8 (test_fp8_linear_gpu.py's bars)


def rel_tol(fp8, epi, K):
    """The bars above were set at K <= 4096.  The fp32 outputs of bf16 operands get 1e-5 * sqrt(K / 1024) past
    K = 1024: their error grows as sqrt(K) (1.9e-5 measured at K = 16384, against a bar of 4e-5)."""
    t = REL_TOL[fp8][epi]
    return t * max(1.0, math.sqrt(K / 1024)) if not fp8 and epi in (GATED, F32) else t


def check_gemm(tag, got, epi, acc, S, c, x0=None, gate=None, fp8=False, K=0):
    """Per element: fp32 outputs |got - ref| <= c S (gated: c |gate| S plus the fma's rounding); bf16 outputs
    2^-8 |ref| + c S; GELU propagates the bound through gelu (|gelu'| < 1.13, plus erff's few ulp).  The relative L2
    error is an average and is not checked on outputs of fewer than 64 elements (one bf16 rounding is 2^-8 of a lone
    element, and a GELU of a large negative product is ~1e-88): the per-element bound covers those."""
    g = got.double()
    assert torch.isfinite(g).all(), f"{tag}: non-finite output"
    if epi == GELU:
        ref = F.gelu(acc)
        rnd, cond = 2.0 ** -8 * ref.abs() + 2.0 ** -20 * acc.abs(), 1.2 * S
    elif epi == BF16:
        ref = acc
        rnd, cond = 2.0 ** -8 * ref.abs(), S
    elif epi == GATED:
        ref = x0.double() + gate.double()[None] * acc
        rnd, cond = 2.0 ** -24 * ref.abs(), gate.double().abs()[None] * S
    else:
        ref, rnd, cond = acc, 0.0, S
    excess = ((g - ref).abs() - rnd).clamp_min(0)
    ratio = excess / cond
    worst = float(torch.where(excess > 0, ratio, torch.zeros_like(ratio)).max())
    _note(("c8" if fp8 else "c32", epi, K), worst)
    if worst > c:
        i = int(torch.argmax(torch.where(excess > 0, ratio, torch.zeros_like(ratio))))
        r, col = divmod(i, ref.shape[1])
        raise AssertionError(f"{tag}: element ({r}, {col}) of {tuple(ref.shape)} is off by {float(excess.view(-1)[i]):.3e} "
                             f"beyond rounding, {worst:.3e} x S > {c:.1e} (got {float(g[r, col])}, ref {float(ref[r, col])})")
    if ref.numel() >= 64:
        e = rel(g, ref)
        assert e < rel_tol(fp8, epi, K), f"{tag}: rel-L2 {e:.3e}"
    return ref


def norm_rope_reference(acc, S, c, gamma, cs, eps=1e-6):
    """fp64 RMSNorm(head) * gamma (+ rotate-half RoPE) of the exact product, and a per-element bound propagated from
    |acc error| <= c S: through the norm (first order: |d rstd / rstd| <= sum |a| e / (128 ms), plus 2^-18 for the fp32
    sum of squares and rsqrtf), the gain and the rotation (2^-22 per fp32 product)."""
    M, N = acc.shape
    a = acc.view(M, N // 128, 128)
    e = (c * S).view(M, N // 128, 128)
    g = gamma.double()
    ms = a.pow(2).mean(-1, keepdim=True) + eps
    r = ms.rsqrt()
    z = a * r * g
    rel_r = (a.abs() * e).sum(-1, keepdim=True) / (128 * ms) + 2.0 ** -18
    ez = r * g.abs() * (e + a.abs() * rel_r) + 2.0 ** -22 * z.abs()
    if cs is None:
        return z.reshape(M, N), ez.reshape(M, N)
    co, si = cs[:, None, :64].double(), cs[:, None, 64:].double()
    za, zb, ea, eb = z[..., :64], z[..., 64:], ez[..., :64], ez[..., 64:]
    y = torch.cat([za * co - zb * si, zb * co + za * si], -1)
    ey = torch.cat([ea * co.abs() + eb * si.abs() + 2.0 ** -22 * ((za * co).abs() + (zb * si).abs()),
                    eb * co.abs() + ea * si.abs() + 2.0 ** -22 * ((zb * co).abs() + (za * si).abs())], -1)
    return y.reshape(M, N), ey.reshape(M, N)


# ------------------------------------------------------------------------------------------------------------------
# the shape matrix: every K with every N, M and the leading dimensions cycling
# ------------------------------------------------------------------------------------------------------------------
N_EDGE = (1, 7, 8, 63, 65, 1001)
M_EDGE = (1, 127, 129)
K_BF16 = (8, 16, 40, 72, 328, 4104)  # K < one k-block (64), and partial last k-blocks
K_FP8 = (16, 48, 144, 1040)  # the same against 128-code k-blocks, K % 16 == 0


def matrix(Ks, step):
    """(M, N, K, lda, ldb, pad_kind, seed): lda = K + step * {0, 1, 2}, ldb = K + step * {1, 2, 3, 0}, and the output's
    row gap none, one ABI step or GAP columns."""
    cases = []
    for i, K in enumerate(Ks):
        for j, N in enumerate(N_EDGE):
            t = i * len(N_EDGE) + j
            cases.append((M_EDGE[t % 3], N, K, K + step * (t % 3), K + step * ((t + 1) % 4), (t // 3) % 3, t))
    return cases


def _matrix(fp8, epi, bn):
    make = fp8_operands if fp8 else bf16_operands
    c = C8 if fp8 else C32
    for M, N, K, lda, ldb, pad_kind, seed in matrix(K_FP8 if fp8 else K_BF16, 16 if fp8 else 8):
        a, b, sa, sb = make(M, N, K, lda, ldb, seed)
        tag = f"M={M} N={N} K={K} lda={lda} ldb={ldb} epi={epi} bn={bn}"
        got, x0, gate = run_gemm(a, b, sa, sb, epi, bn, out_ld(N, epi, pad_kind), seed)
        acc, S = reference(a, b, sa, sb)
        check_gemm(tag, got, epi, acc, S, c, x0, gate, fp8, K)


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("epi", [BF16, GELU, GATED, F32])
def test_gemm_bf16_matrix(epi, bn):
    _matrix(False, epi, bn)


@pytest.mark.parametrize("bn", [64, 128, 256])  # 256 runs the 128-column fp8 tile
@pytest.mark.parametrize("epi", [BF16, GELU, GATED, F32])
def test_gemm_fp8_matrix(epi, bn):
    _matrix(True, epi, bn)


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("N", [128, 384, 512, 1152])  # 512: the 256-column tile of the bf16 entry
@pytest.mark.parametrize("with_rope", [True, False])
def test_gemm_norm_rope(with_rope, N, fp8):
    """The fused RMSNorm/RoPE epilogue through its own entry point (which chooses the tile) at K, M and lda/ldb/ldd
    edges, against fp64 with the propagated per-element bound."""
    step = 16 if fp8 else 8
    Ks = K_FP8 if fp8 else K_BF16
    make = fp8_operands if fp8 else bf16_operands
    c = C8 if fp8 else C32
    gamma = 1 + 0.2 * torch.randn(128, device="cuda", generator=gen(N))
    for t, K in enumerate(Ks):
        M = M_EDGE[t % 3]
        lda, ldb, ld = K + step * (t % 3), K + step * ((t + 1) % 3), N + (0, 8, GAP)[(t + N // 128) % 3]
        a, b, sa, sb = make(M, N, K, lda, ldb, seed=100 + t)
        cs = None
        if with_rope:
            ang = torch.rand(M, 64, device="cuda", generator=gen(t)) * 6.0
            cs = torch.cat([ang.cos(), ang.sin()], 1).contiguous()
        out = Guarded(M, N, ld, torch.bfloat16)
        cp = None if cs is None else cs.data_ptr()
        if fp8:
            rc = lib().g3c_gemm_norm_rope_fp8(a.data_ptr(), sa.data_ptr(), b.data_ptr(), sb.data_ptr(), out.ptr, M, N, K,
                                              lda, ldb, ld, gamma.data_ptr(), cp, 1e-6, stream())
        else:
            rc = lib().g3c_gemm_norm_rope_bf16(a.data_ptr(), b.data_ptr(), out.ptr, M, N, K, lda, ldb, ld,
                                               gamma.data_ptr(), cp, 1e-6, stream())
        assert rc == 0, lib().g3c_last_error()
        out.assert_outside_untouched()
        acc, S = reference(a, b, sa, sb)
        y, ey = norm_rope_reference(acc, S, c, gamma, cs)
        got = out.view.double()
        assert torch.isfinite(got).all()
        excess = (got - y).abs() - 2.0 ** -8 * y.abs()
        worst = float((excess / ey).max())
        _note(("norm_rope", fp8), worst)
        assert worst <= 1.0, f"M={M} N={N} K={K}: {worst:.3f} x the propagated bound"
        assert rel(got, y) < 3e-3


# ------------------------------------------------------------------------------------------------------------------
# tile counts around the persistent grid, and the narrower last super-column
# ------------------------------------------------------------------------------------------------------------------
def run_bn(bn, N, fp8):
    """The tile width the host runs for a block_n request (mirrors gemm_any)."""
    if bn == 512:
        bn = 256
    if bn == 0:
        bn = 256 if (N >= 256 and N % 256 == 0) else (128 if N > 64 else 64)
    return 128 if fp8 and bn == 256 else bn


def super_n(bn, K, esize, num_n_blk):
    """n-blocks per super-column (mirrors gemm_any: 16 MiB of B per super-column)."""
    return max(1, min((16 << 20) // (bn * K * esize), num_n_blk))


def tile_coords(tile, num_m_blk, num_n_blk, sn):
    """(m_blk, n_blk) of a linear tile index (mirrors tile_coords in gemm_wgmma.cu)."""
    per_super = num_m_blk * sn
    sc, rem = divmod(tile, per_super)
    n0 = sc * sn
    width = min(num_n_blk - n0, sn)
    return rem // width, n0 + rem % width


def odd_split(tiles):
    """tiles = m * n with m odd, m as close to sqrt(tiles) as the odd divisors allow."""
    m = min((d for d in range(1, tiles + 1, 2) if tiles % d == 0), key=lambda d: abs(math.log(d / math.sqrt(tiles))))
    return m, tiles // m


def tile_count_cases(fp8):
    sm = sm_count()
    return [(t, bn) for t in (1, sm - 1, sm, sm + 1, 2 * sm + 1) for bn in ((64, 128) if fp8 else (64, 128, 256))]


@pytest.mark.parametrize("fp8", [False, True])
def test_gemm_tile_counts_around_the_grid(fp8):
    """tiles in {1, sm - 1, sm, sm + 1, 2 sm + 1} (the grid is min(tiles, sm)) with an odd number of row blocks, each
    tile ragged in M and N, on the gated residual from a non-zero x: a tile that runs twice adds its term twice and a
    skipped tile adds nothing.  The operands have no magnitude spread, so that every tile weighs alike.  Negative
    controls: either fault in one tile misses the relative L2 tolerance, and the per-element bound, by >= 10x."""
    sm = sm_count()
    K = 80 if fp8 else 72
    for tiles, bn in tile_count_cases(fp8):
        bnr = run_bn(bn, 0, fp8)
        mb, nb = odd_split(tiles)
        M, N = 128 * mb - 5, bnr * nb - 3
        make = fp8_operands if fp8 else bf16_operands
        a, b, sa, sb = make(M, N, K, K + 16, K, seed=tiles + bn, spread=0.0)
        got, x0, gate = run_gemm(a, b, sa, sb, GATED, bn, rup(N, 4) + 4, seed=tiles)
        acc, S = reference(a, b, sa, sb)
        tag = f"tiles={tiles} ({mb} x {nb}) bn={bn} M={M} N={N}"
        ref = check_gemm(tag, got, GATED, acc, S, C8 if fp8 else C32, x0, gate, fp8, K)
        # the tile the last CTA runs first, added twice or not at all
        grid = min(tiles, sm)
        m_blk, n_blk = tile_coords(grid - 1, mb, nb, super_n(bnr, K, 1 if fp8 else 2, nb))
        rows, cols = slice(128 * m_blk, 128 * m_blk + 128), slice(bnr * n_blk, bnr * n_blk + bnr)
        term = torch.zeros_like(ref)
        term[rows, cols] = gate.double()[None, cols] * acc[rows, cols]
        tol = rel_tol(fp8, GATED, K)
        assert rel(ref + term, ref) > 10 * tol and rel(ref - term, ref) > 10 * tol, tag
        assert float((term.abs() / (gate.double().abs()[None] * S)).max()) > 10 * (C8 if fp8 else C32), tag


SUPER_COLUMN_CASES = [(False, 256, 8192, 1536), (False, 64, 16384, 704), (True, 128, 16384, 1280)]


@pytest.mark.parametrize("fp8,bn,K,N", SUPER_COLUMN_CASES)
def test_gemm_last_super_column_is_narrower(fp8, bn, K, N):
    """B is walked in super-columns of super_n n-blocks; here the last one is narrower than the rest."""
    nb = -(-N // bn)
    sn = super_n(bn, K, 1 if fp8 else 2, nb)
    assert sn < nb and nb % sn != 0, (sn, nb)  # the case still covers a remainder
    M = 300  # three row blocks
    make = fp8_operands if fp8 else bf16_operands
    a, b, sa, sb = make(M, N, K, K + (16 if fp8 else 8), K, seed=K + N)
    acc, S = reference(a, b, sa, sb)
    for epi in (F32, BF16):
        got, _, _ = run_gemm(a, b, sa, sb, epi, bn, out_ld(N, epi, 2))
        check_gemm(f"K={K} N={N} bn={bn} super_n={sn}", got, epi, acc, S, C8 if fp8 else C32, fp8=fp8, K=K)


# ------------------------------------------------------------------------------------------------------------------
# bitwise properties: row slices and repeats
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fp8,bn", [(False, 64), (False, 128), (False, 256), (True, 64), (True, 128)])
def test_gemm_row_slices_are_bitwise(fp8, bn):
    """Each output row depends on its A row only, in a fixed k order: A[r0:r1] (a view starting inside the buffer) gives
    rows r0:r1 of the full output bit for bit, across 128-row tile boundaries.  A repeat is bitwise as well."""
    M, N, K = 300, 200, 1040 if fp8 else 392
    make = fp8_operands if fp8 else bf16_operands
    a, b, sa, sb = make(M, N, K, K + 16, K + 16, seed=bn)
    full, _, _ = run_gemm(a, b, sa, sb, F32, bn, N + 4)
    again, _, _ = run_gemm(a, b, sa, sb, F32, bn, N + 4)
    assert torch.equal(full.view(torch.int32), again.view(torch.int32))
    for r0, r1 in [(0, 1), (4, 132), (100, 200), (124, 129), (128, 300), (296, 300)]:
        part, _, _ = run_gemm(a[r0:r1], b, None if sa is None else sa[r0:r1], sb, F32, bn, N + GAP)
        assert torch.equal(part.view(torch.int32), full[r0:r1].view(torch.int32)), (r0, r1)


# ------------------------------------------------------------------------------------------------------------------
# the argument errors of the GEMM entry points: an error code, nothing written
# ------------------------------------------------------------------------------------------------------------------
def _error_call(case):
    M, N, K = 129, 64, 64
    kw = dict(M=M, N=N, K=K, lda=K, ldb=K, ld=None, epi=BF16, bn=0, gate=True, a_off=0, b_off=0, d_off=0, g_off=0,
              fp8=False, nr=False, gamma=True, cs_off=0, sa=True, s_off=0)
    kw.update(case)
    if kw["ld"] is None:
        kw["ld"] = kw["N"] + GAP
    fp8, epi = kw["fp8"], kw["epi"]
    dt = torch.bfloat16 if epi in (BF16, GELU, 4, 5, -1) else torch.float32
    esz = 1 if fp8 else 2
    a = torch.zeros(M, max(kw["lda"], kw["K"]) + 16, dtype=torch.uint8 if fp8 else torch.bfloat16, device="cuda")
    b = torch.zeros(max(kw["N"], N), max(kw["ldb"], kw["K"]) + 16, dtype=a.dtype, device="cuda")
    out = Guarded(M, kw["N"], max(kw["ld"], 8), dt)
    gate = torch.ones(kw["N"] + 8, device="cuda")
    scales = torch.ones(max(M, kw["N"]) + 8, device="cuda")
    gamma = torch.ones(132, device="cuda")
    cs = torch.zeros(M * 128 + 8, device="cuda")
    ap, bp = a.data_ptr() + kw["a_off"] * esz, b.data_ptr() + kw["b_off"] * esz
    dp = out.ptr + kw["d_off"]
    gp = gate.data_ptr() + kw["g_off"] if kw["gate"] else None
    sp = scales.data_ptr() + kw["s_off"] if kw["sa"] else None
    args = (kw["M"], kw["N"], kw["K"], kw["lda"], kw["ldb"], kw["ld"])
    L = lib()
    if kw["nr"]:
        gm = gamma.data_ptr() if kw["gamma"] else None
        cp = cs.data_ptr() + kw["cs_off"]
        if fp8:
            rc = L.g3c_gemm_norm_rope_fp8(ap, sp, bp, scales.data_ptr(), dp, *args, gm, cp, 1e-6, stream())
        else:
            rc = L.g3c_gemm_norm_rope_bf16(ap, bp, dp, *args, gm, cp, 1e-6, stream())
    elif fp8:
        rc = L.g3c_gemm_fp8(ap, sp, bp, scales.data_ptr(), dp, *args, epi, gp, kw["bn"], stream())
    else:
        rc = L.g3c_gemm_bf16(ap, bp, dp, *args, epi, gp, kw["bn"], stream())
    return rc, out


ERROR_CASES = {
    "k_not_multiple_of_8": dict(K=60),
    "lda_not_multiple_of_8": dict(lda=68),
    "lda_below_k": dict(lda=56),
    "ldb_below_k": dict(ldb=56),
    "ldd_below_n": dict(ld=56),
    "bf16_ldd_not_multiple_of_8": dict(ld=68),
    "f32_ldd_not_multiple_of_4": dict(epi=F32, ld=66),
    "bf16_d_misaligned": dict(d_off=2),
    "f32_d_misaligned": dict(epi=F32, d_off=4),
    "gate_misaligned": dict(epi=GATED, g_off=4),
    "gate_null": dict(epi=GATED, gate=False),
    "block_n_512_with_n_not_multiple_of_256": dict(N=384, bn=512),
    "block_n_96": dict(bn=96),
    "epilogue_negative": dict(epi=-1, bn=128),
    "epilogue_4_is_internal": dict(epi=4, bn=128),
    "epilogue_5": dict(epi=5, bn=256),
    "norm_rope_n_not_multiple_of_128": dict(nr=True, N=192),
    "norm_rope_null_gain": dict(nr=True, N=128, gamma=False),
    "norm_rope_table_misaligned": dict(nr=True, N=128, cs_off=8),
    "a_base_misaligned": dict(a_off=1),
    "b_base_misaligned": dict(b_off=4),
    "fp8_k_not_multiple_of_16": dict(fp8=True, K=56, lda=64, ldb=64),
    "fp8_lda_not_multiple_of_16": dict(fp8=True, lda=72),
    "fp8_ldb_not_multiple_of_16": dict(fp8=True, ldb=72),
    "fp8_null_scale": dict(fp8=True, sa=False),
    "fp8_scale_misaligned": dict(fp8=True, s_off=4),
    "fp8_epilogue_4_is_internal": dict(fp8=True, epi=4, bn=128),
    "fp8_norm_rope_n_not_multiple_of_128": dict(fp8=True, nr=True, N=192),
    "fp8_a_base_misaligned": dict(fp8=True, a_off=8),
}


@pytest.mark.parametrize("name", list(ERROR_CASES))
def test_gemm_errors_launch_nothing(name):
    rc, out = _error_call(ERROR_CASES[name])
    assert rc == EINVAL, (rc, lib().g3c_last_error())
    assert lib().g3c_last_error()
    out.assert_untouched()


def test_gemm_error_cases_are_otherwise_valid():
    """The base call of the error cases succeeds: each error above comes from its one changed argument."""
    for case in (dict(), dict(epi=F32), dict(epi=GATED), dict(nr=True, N=128), dict(fp8=True),
                 dict(fp8=True, nr=True, N=128)):
        rc, out = _error_call(case)
        assert rc == 0, (case, lib().g3c_last_error())
        out.assert_outside_untouched()


# ------------------------------------------------------------------------------------------------------------------
# row kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_rope", [True, False])
@pytest.mark.parametrize("heads", [1, 3])
def test_rmsnorm_rope_strided(heads, with_rope):
    """In place on [L, heads*128] with ld = heads*128 + 64 and L*heads not a multiple of the 8 warps of a CTA: the gap
    columns and the bands stay as they were.  Bound: bf16 rounding plus 2^-16 r |gamma| (|a| + |b|) for the fp32 sum
    of squares, rsqrtf and the rotation (each a few 2^-24)."""
    L = 77
    D = heads * 128
    x = torch.randn(L, D, device="cuda", generator=gen(heads)).mul(3).to(torch.bfloat16)
    gamma = 1 + 0.2 * torch.randn(128, device="cuda", generator=gen(7))
    ang = torch.rand(L, 64, device="cuda", generator=gen(8)) * 6.0
    cs = torch.cat([ang.cos(), ang.sin()], 1).contiguous()
    buf = Guarded(L, D, D + 64, torch.bfloat16, init=x)
    rc = lib().g3c_rmsnorm_rope(buf.ptr, D + 64, L, heads, gamma.data_ptr(), cs.data_ptr() if with_rope else None,
                                1e-6, stream())
    assert rc == 0, lib().g3c_last_error()
    buf.assert_outside_untouched()
    a = x.double().view(L, heads, 128)
    r = (a.pow(2).mean(-1, keepdim=True) + 1e-6).rsqrt()
    z = a * r * gamma.double()
    mag = r * gamma.double().abs() * (a.abs() + torch.cat([a[..., 64:], a[..., :64]], -1).abs())
    if with_rope:
        from oracle import dit_oracle

        z = dit_oracle.apply_rope(z, torch.cat([ang, ang], 1).double())
    y = z.reshape(L, D)
    err = (buf.view.double() - y).abs() - 2.0 ** -8 * y.abs()
    ratio = float((err / mag.reshape(L, D)).max())
    _note("rmsnorm_rope", ratio)
    assert ratio <= 2.0 ** -16, ratio


@pytest.mark.parametrize("R,C", [(1, 16), (5, 272), (129, 4112)])
def test_quantize_rows_strided(R, C):
    """x [R, C] in a [R, C + 24] buffer whose gap holds +-3e38 (a NaN would vanish in the kernel's fmaxf amax), codes
    into [R, C] with ldq = C + 32 inside guard bands, the scales inside bands: byte-exact against the oracle."""
    g = gen(R)
    x = torch.randn(R, C, device="cuda", generator=g) * torch.logspace(-3, 3, R, device="cuda")[:, None]
    x[0, C // 2] = -500.0
    huge = torch.tensor([3e38, -3e38], device="cuda").repeat(12)
    xs = strided(x.to(torch.bfloat16), C + 24, huge.to(torch.bfloat16))
    codes = Guarded(R, C, C + 32, torch.uint8)
    scales = Guarded(1, R, rup(R, 4), torch.float32)
    rc = lib().g3c_quantize_rows_fp8(xs.data_ptr(), C + 24, R, C, codes.ptr, C + 32, scales.ptr, stream())
    assert rc == 0, lib().g3c_last_error()
    codes.assert_outside_untouched()
    scales.assert_outside_untouched()
    want_c, want_s = fp8_oracle.quantize_rows_e4m3(xs.float().cpu())
    assert torch.equal(codes.view.cpu(), want_c.view(torch.uint8))
    assert torch.equal(scales.view[0].cpu().view(torch.int32), want_s.view(torch.int32))


def ln_reference(x, shift, scale, eps=1e-6):
    """fp64 LayerNorm * (1 + scale) + shift of the fp32 rows, and the scale of the error of fp32 statistics:
    2^-24 sqrt(D) mean|x| rstd |1 + scale|."""
    xd = x.double()
    D = x.shape[1]
    mean = xd.mean(1, keepdim=True)
    var = (xd - mean).pow(2).mean(1, keepdim=True)
    rstd = (var + eps).rsqrt()
    y = (xd - mean) * rstd * (1 + scale.double()) + shift.double()
    stat = 2.0 ** -24 * math.sqrt(D) * xd.abs().mean(1, keepdim=True) * rstd * (1 + scale.double()).abs()
    return y, stat


def _ln_inputs(L, D, seed, offset):
    g = gen(seed)
    x = torch.randn(L, D, device="cuda", generator=g) * 2 + offset
    pos = torch.randn(L, D, device="cuda", generator=g).to(torch.bfloat16)
    shift = 0.3 * torch.randn(D, device="cuda", generator=g)
    scale = 0.3 * torch.randn(D, device="cuda", generator=g)
    return x, pos, shift, scale


LN_D = [16, 260, 4100, 24576]  # 24576 * 4 B = 96 KiB: the row cache's limit


@pytest.mark.parametrize("with_pos", [True, False])
@pytest.mark.parametrize("offset", [0.0, 1e4])
@pytest.mark.parametrize("D", LN_D)
def test_ln_modulate_edges(D, offset, with_pos):
    """D not a multiple of the CTA's 1024-element stride, up to the shared-memory limit; rows offset by 1e4 (a one-pass
    variance E[x^2] - E[x]^2 would lose every bit of it); x += pos exactly in fp32, or x bit-unchanged without pos."""
    L = 7
    x, pos, shift, scale = _ln_inputs(L, D, D, offset)
    xg = Guarded(L, D, D, torch.float32, init=x)
    y = Guarded(L, D, D, torch.bfloat16)
    rc = lib().g3c_ln_modulate(xg.ptr, pos.data_ptr() if with_pos else None, shift.data_ptr(), scale.data_ptr(), y.ptr,
                               L, D, 1e-6, stream())
    assert rc == 0, lib().g3c_last_error()
    xg.assert_outside_untouched()
    y.assert_outside_untouched()
    xr = x + pos.float() if with_pos else x
    assert torch.equal(xg.view.view(torch.int32), xr.view(torch.int32))
    ref, stat = ln_reference(xr, shift, scale)
    excess = (y.view.double() - ref).abs() - 2.0 ** -8 * ref.abs()
    ratio = float((excess / stat).max())
    _note(("ln", D, offset), ratio)
    assert ratio <= C_LN, ratio


@pytest.mark.parametrize("with_pos", [True, False])
@pytest.mark.parametrize("offset", [0.0, 1e4])
@pytest.mark.parametrize("D", [d for d in LN_D if d % 16 == 0])
def test_ln_modulate_fp8_edges(D, offset, with_pos):
    """The e4m3 variant at the same edges: codes * scale within e4m3 rounding (2^-4 relative, 2^-10 scale in the
    subnormals) of the fp64 result plus the statistics' error, the scale within the same of amax / 448."""
    L = 7
    x, pos, shift, scale = _ln_inputs(L, D, D + 1, offset)
    xg = Guarded(L, D, D, torch.float32, init=x)
    codes = Guarded(L, D, D, torch.uint8)
    scales = Guarded(1, L, 8, torch.float32)
    rc = lib().g3c_ln_modulate_fp8(xg.ptr, pos.data_ptr() if with_pos else None, shift.data_ptr(), scale.data_ptr(),
                                   codes.ptr, scales.ptr, L, D, 1e-6, stream())
    assert rc == 0, lib().g3c_last_error()
    for gb in (xg, codes, scales):
        gb.assert_outside_untouched()
    xr = x + pos.float() if with_pos else x
    assert torch.equal(xg.view.view(torch.int32), xr.view(torch.int32))
    ref, stat = ln_reference(xr, shift, scale)
    s = scales.view[0].double()
    amax = ref.abs().amax(1)
    assert ((s * 448 - amax).abs() <= C_LN * stat.amax(1) + 1e-6 * amax).all()
    deq = codes.view.view(E4M3).double() * s[:, None]
    excess = (deq - ref).abs() - 2.0 ** -4 * ref.abs() - 2.0 ** -10 * s[:, None]
    ratio = float((excess / stat).max())
    _note(("ln_fp8", D, offset), ratio)
    assert ratio <= 1.1 * C_LN, ratio


def test_ln_modulate_rejects_rows_past_the_row_cache():
    """D = 24580 (bf16) / 24592 (fp8) rows do not fit the 96 KiB row cache: an error, and neither x nor y written."""
    for D, fp8 in ((24580, False), (24592, True)):
        L = 3
        x, pos, shift, scale = _ln_inputs(L, D, 5, 0.0)
        xg = Guarded(L, D, D, torch.float32, init=x)
        y = Guarded(L, D, D, torch.uint8 if fp8 else torch.bfloat16)
        if fp8:
            s = Guarded(1, L, 4, torch.float32)
            rc = lib().g3c_ln_modulate_fp8(xg.ptr, pos.data_ptr(), shift.data_ptr(), scale.data_ptr(), y.ptr, s.ptr, L,
                                           D, 1e-6, stream())
            s.assert_untouched()
        else:
            rc = lib().g3c_ln_modulate(xg.ptr, pos.data_ptr(), shift.data_ptr(), scale.data_ptr(), y.ptr, L, D, 1e-6,
                                       stream())
        assert rc == EINVAL
        xg.assert_untouched()
        y.assert_untouched()


# ------------------------------------------------------------------------------------------------------------------
# attention: the output side
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,h", [(1, 1), (2, 3)])
@pytest.mark.parametrize("Lq", [1, 77, 129])
def test_attention_sbhd_strided_output(Lq, b, h):
    """o [Lq, b*h*128] with ldo = b*h*128 + 64 and 128 rows of band after it: rows past Lq in the last query tile and
    the row gaps stay untouched.  Per element: 2^-8 |ref| + C_ATT * (P . |V|), P from fp64 softmax."""
    Lk = 200
    bh = b * h
    D = bh * 128
    g = gen(Lq + bh)
    q, k, v = (torch.randn(n, D, device="cuda", generator=g).to(torch.bfloat16) for n in (Lq, Lk, Lk))
    o = Guarded(Lq, D, D + 64, torch.bfloat16)
    scale = 128 ** -0.5
    rc = lib().g3c_attn_fwd_sbhd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.ptr, Lq, Lk, b, h, D, D, D, D + 64, scale,
                                 stream())
    assert rc == 0, lib().g3c_last_error()
    o.assert_outside_untouched()
    qh, kh, vh = (t.double().view(-1, bh, 128).transpose(0, 1) for t in (q, k, v))
    p = torch.softmax(qh @ kh.transpose(1, 2) * scale, -1)
    ref = (p @ vh).transpose(0, 1).reshape(Lq, D)
    pv = (p @ vh.abs()).transpose(0, 1).reshape(Lq, D)
    got = o.view.double()
    assert torch.isfinite(got).all()
    excess = (got - ref).abs() - 2.0 ** -8 * ref.abs()
    ratio = float((excess / pv).max())
    _note("attn", ratio)
    assert ratio <= C_ATT, ratio
    assert rel(got, ref) < 5e-3
