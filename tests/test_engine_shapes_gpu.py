"""The GEMM and the attention at the shapes `dit_engine.cu::forward` launches them, checked element by element.

The small-shape files (test_operator_edges_gpu.py, test_gemm_epilogue_rounding_gpu.py) cannot see a fault that only
shows after a persistent CTA has run many tiles: a wrong stage of the ring, a staging buffer reused too early, a tile
of the last super-column.  Such a fault spoils one 64-row output box, which a sampled-row or rel-L2 check over a
56 320-row product misses most of the time.  This file

1. runs every Linear of a DiT block (7B width: D = 4096, ffn 16 384, context 512 x 1024, patch K 384, 64 output
   columns) at its exact launch (M, N, K, leading dimensions, block_n, epilogue, operands swapped for V^T, real RoPE
   table, folded query gain, gated residual from a non-zero x with a gate of both signs), bf16 and fp8, at 56 320 tokens
   (one GPU) and on subsets at 7 040 (cp = 8 per rank) and 14 080 (CFG x CP on 8 GPUs).  Every output starts as NaN,
   and every element is held to the per-element bounds of test_operator_edges_gpu.py against float64 products of the
   operands' exact values, computed on the GPU in row chunks;
2. launches 128-row blocks of those products alone (one or two tiles per CTA) and requires them bit for bit equal to
   the full launch's rows: blocks from the first wave, the last wave and the last tile of the last CTA;
3. runs the attention at the engine's shapes with all 32 heads and the engine's scale (ln 2, the query carrying
   1/sqrt(128) log2 e): self-attention 56 320 x 56 320 on two rows of every query tile, one per consumer warpgroup,
   and cross-attention 56 320 x 512 on every row, both against tests/attn_ref64.py;
4. applies negative controls in torch to real outputs: each must miss its check by >= 10x.

The largest ratio to each bound is printed per shape and mode (run with -s)."""
import math
import time

import pytest
import torch

from oracle import dit_oracle
from tests import attn_ref64
from tests.test_engine_signal_gpu import rope_angles64
from tests.test_operator_edges_gpu import (BF16, C8, C32, E4M3, F32, GATED, GELU, OBSERVED, check_gemm, gen, lib,
                                           norm_rope_reference, rel, run_bn, sm_count, stream, super_n, tile_coords)

pytestmark = pytest.mark.gpu

D, FFN, HEADS, CTX_LEN, CTX_DIM, KPAD, NO = 4096, 16384, 32, 512, 1024, 384, 64
HP, WP = 44, 80  # latent patches per frame of the benchmark's 704 x 1280 video: L = T * 3520
L_FULL = 56320
# the engine folds the softmax scale and log2(e) into the query gain (dit_engine.cu kQScale, an fp32 product)
KQ_SCALE = float(torch.tensor(0.08838834764831845, dtype=torch.float32) * torch.tensor(1.4426950408889634,
                                                                                    dtype=torch.float32))
LN2 = 0.6931471805599453
CHUNK = 1 << 26  # float64 elements per reference chunk (512 MB per tensor)

# name: (activation, N, K, epilogue, fused norm, swapped, block_n, e4m3 in the fp8 Linear mode), as forward() launches
# them: activation rows [M, K] are the block's tokens ("L") or the T5 context ("ctx"); "rope" / "norm" is the fused
# per-head RMSNorm with / without rotation (q_gain: the query gain with the folded scale); swapped is V^T = W . x^T.
LINEARS = {
    "patch_embed": ("L", D, KPAD, F32, None, False, 0, False),
    "fa_to_k": ("L", D, D, BF16, "rope", False, 0, True),
    "fa_to_q": ("L", D, D, BF16, "rope_q", False, 0, True),
    "fa_vt": ("L", D, D, BF16, None, True, 0, True),
    "fa_to_out": ("L", D, D, GATED, None, False, 0, True),
    "ca_to_k": ("ctx", D, CTX_DIM, BF16, "norm", False, 0, False),
    "ca_vt": ("ctx", D, CTX_DIM, BF16, None, True, 0, False),
    "ca_to_q": ("L", D, D, BF16, "norm_q", False, 0, True),
    "ca_to_out": ("L", D, D, GATED, None, False, 0, True),
    "layer1": ("L", FFN, D, GELU, None, False, 0, True),
    "layer2": ("L", D, FFN, GATED, None, False, 0, True),
    "final": ("L", NO, D, F32, None, False, 64, False),
}
# the 7 040 / 14 080 subsets: the V^T tile changes to 128 columns at 7 040 (7 040 % 256 != 0)
SUBSETS = {L_FULL: list(LINEARS), 7040: ["fa_to_k", "fa_vt", "fa_to_out", "layer1", "layer2"],
           14080: ["fa_to_q", "fa_vt", "ca_to_out", "layer2"]}
FIRST_FRAME = {L_FULL: 0, 7040: 14, 14080: 12}  # the last context-parallel rank's frames

def report(key, value):
    """Print the largest ratio of a check (L, mode, what) to its bound."""
    print(f"engine shapes {key}: {value:.3g} of the bound")


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def rows_bf16(R, C, seed, scale=1.0, spread=1.0):
    """Random bf16 rows [R, C], the rows' magnitudes spread over scale * 10^(+-spread), generated in chunks."""
    out = torch.empty(R, C, dtype=torch.bfloat16, device="cuda")
    g = gen(seed)
    mags = scale * torch.logspace(-spread, spread, R, device="cuda")
    step = max(1, (1 << 25) // C)
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        out[r0:r1] = torch.randn(r1 - r0, C, device="cuda", generator=g).mul_(mags[r0:r1, None])
    return out


def quantize(x):
    """e4m3 codes and row scales of bf16 rows through g3c_quantize_rows_fp8 (the engine's quantiser)."""
    R, C = x.shape
    codes = torch.empty(R, C, dtype=torch.uint8, device="cuda")
    scales = torch.empty(R, dtype=torch.float32, device="cuda")
    rc = lib().g3c_quantize_rows_fp8(x.data_ptr(), C, R, C, codes.data_ptr(), C, scales.data_ptr(), stream())
    assert rc == 0, lib().g3c_last_error()
    return codes, scales


def exact(t, s):
    """The float64 values an operand stands for: bf16 as is, e4m3 codes times their row scales."""
    return t.double() if s is None else t.view(E4M3).double() * s.double()[:, None]


def rope_table(L):
    """The engine's cos|sin table [L, 128] for the frames of a rank that starts at FIRST_FRAME[L] (24 fps)."""
    ang = torch.from_numpy(rope_angles64(dit_oracle.DitCfg(), L // (HP * WP), HP, WP, 24.0, FIRST_FRAME[L]))
    return torch.cat([ang[:, :64].cos(), ang[:, 64:].sin()], 1).float().contiguous().cuda()


class Operands:
    """Activations shared by the Linears of one token count (as in a block, where several Linears read xn), and each
    Linear's own weight."""

    def __init__(self, L):
        self.L = L
        self.act = {}

    def activation(self, kind, K):
        key = (kind, K)
        if key not in self.act:
            R = self.L if kind == "L" else CTX_LEN
            self.act[key] = rows_bf16(R, K, seed=K + (1 if kind == "L" else 2))
        return self.act[key]


def weight(name, N, K):
    w = rows_bf16(N, K, seed=sum(map(ord, name)) * 131 + N + K, scale=0.02, spread=0.5)
    if name == "patch_embed":
        w[:, 328:] = 0  # the engine zero-pads the 328 patch inputs to Kpad = 384
    return w


class Launch:
    """One Linear of the engine at L tokens: operands (codes in fp8 mode), the GEMM's M / N / K after the swap, the
    epilogue inputs, and the NaN-filled output of a full launch."""

    def __init__(self, ops, name, fp8):
        kind, N, K, epi, fused, swapped, bn, e4m3 = LINEARS[name]
        self.name, self.epi, self.fused, self.bn, self.K = name, epi, fused, bn, K
        self.fp8 = fp8 and e4m3
        x = ops.activation(kind, K)
        w = weight(name, N, K)
        if self.fp8:
            (xa, xs), (wa, ws) = quantize(x), quantize(w)
        else:
            (xa, xs), (wa, ws) = (x, None), (w, None)
        self.A, self.sa, self.B, self.sb = (wa, ws, xa, xs) if swapped else (xa, xs, wa, ws)
        self.M, self.N = self.A.shape[0], self.B.shape[0]
        self.gate = self.x0 = self.gamma = self.cs = None
        if epi == GATED:
            self.gate = torch.randn(self.N, device="cuda", generator=gen(N + 7)) * 0.6  # both signs
            self.x0 = torch.randn(self.M, self.N, device="cuda", generator=gen(N + 8)) * 4
        if fused:
            g = (1 + 0.2 * torch.randn(128, device="cuda", generator=gen(K + 9))).to(torch.bfloat16).float()
            self.gamma = g * KQ_SCALE if fused.endswith("_q") else g
            if fused.startswith("rope"):
                self.cs = rope_table(self.M)
        self.c = C8 if self.fp8 else C32

    def run(self, r0=0, r1=None):
        """Launch rows [r0, r1) of A (all by default) as one GEMM; returns its output."""
        r1 = self.M if r1 is None else r1
        M = r1 - r0
        dt = torch.float32 if self.epi in (F32, GATED) else torch.bfloat16
        if self.epi == GATED:
            out = self.x0[r0:r1].clone()
        else:
            out = torch.empty(M, self.N, dtype=dt, device="cuda")
            out.view(torch.int16 if dt == torch.bfloat16 else torch.int32).fill_(0x7FA1 if dt == torch.bfloat16
                                                                                 else 0x7FC01234)
        A = self.A[r0:r1]
        sa = None if self.sa is None else self.sa[r0:r1]
        K, N, L = self.K, self.N, lib()
        if self.fused:
            cs = None if self.cs is None else self.cs[r0:r1].data_ptr()
            if self.fp8:
                rc = L.g3c_gemm_norm_rope_fp8(A.data_ptr(), sa.data_ptr(), self.B.data_ptr(), self.sb.data_ptr(),
                                              out.data_ptr(), M, N, K, K, K, N, self.gamma.data_ptr(), cs, 1e-6,
                                              stream())
            else:
                rc = L.g3c_gemm_norm_rope_bf16(A.data_ptr(), self.B.data_ptr(), out.data_ptr(), M, N, K, K, K, N,
                                               self.gamma.data_ptr(), cs, 1e-6, stream())
        else:
            gp = None if self.gate is None else self.gate.data_ptr()
            if self.fp8:
                rc = L.g3c_gemm_fp8(A.data_ptr(), sa.data_ptr(), self.B.data_ptr(), self.sb.data_ptr(), out.data_ptr(),
                                    M, N, K, K, K, N, self.epi, gp, self.bn, stream())
            else:
                rc = L.g3c_gemm_bf16(A.data_ptr(), self.B.data_ptr(), out.data_ptr(), M, N, K, K, K, N, self.epi, gp,
                                     self.bn, stream())
        assert rc == 0, L.g3c_last_error()
        return out

    # --------------------------------------------------------------------------------------------------------------
    def chunks(self):
        step = max(128, CHUNK // max(self.N, self.K) // 128 * 128)
        return [(r0, min(self.M, r0 + step)) for r0 in range(0, self.M, step)]

    def reference(self, r0, r1, Bd=None):
        """float64 product of rows [r0, r1) and its conditioning S = |A| . |B|^T."""
        if Bd is None:
            Bd = exact(self.B, self.sb)
            Bd = (Bd, Bd.abs())
        ad = exact(self.A[r0:r1], None if self.sa is None else self.sa[r0:r1])
        return ad @ Bd[0].T, ad.abs() @ Bd[1].T

    def check(self, got, r0, r1, acc, S, tag):
        """The per-element check of rows [r0, r1) of an output; returns the largest ratio to the bound (raises past 1)."""
        if self.fused:
            cs = None if self.cs is None else self.cs[r0:r1]
            y, ey = norm_rope_reference(acc, S, self.c, self.gamma, cs)
            g = got[r0:r1].double()
            assert torch.isfinite(g).all(), f"{tag}: non-finite output"
            ratio = ((g - y).abs() - 2.0 ** -8 * y.abs()) / ey
            worst = float(ratio.max())
            if worst > 1.0:
                r, col = divmod(int(ratio.argmax()), self.N)
                raise AssertionError(f"{tag}: element ({r0 + r}, {col}) is {worst:.3f} x the propagated bound")
            assert rel(g, y) < 3e-3, tag
            return worst
        key = ("c8" if self.fp8 else "c32", self.epi, self.K)
        OBSERVED.pop(key, None)
        x0 = None if self.x0 is None else self.x0[r0:r1]
        check_gemm(f"{tag} rows {r0}:{r1}", got[r0:r1], self.epi, acc, S, self.c, x0, self.gate, self.fp8, self.K)
        return OBSERVED.get(key, 0.0) / self.c

    def schedule_blocks(self):
        """Row blocks of the tiles a persistent CTA runs first and last: (label, m_blk)."""
        bnr = run_bn(self.bn, self.N, self.fp8)
        mb, nb = -(-self.M // 128), -(-self.N // bnr)
        sn = super_n(bnr, self.K, 1 if self.fp8 else 2, nb)
        tiles = mb * nb
        grid = min(tiles, sm_count())
        picks = {"first wave": grid // 2, "last wave": tiles - 1,
                 "last tile of the last CTA": grid - 1 + grid * ((tiles - grid) // grid)}
        return [(label, tile_coords(t, mb, nb, sn)[0], t // grid) for label, t in picks.items()]


# ------------------------------------------------------------------------------------------------------------------
# 1 + 2: every Linear per element, and row blocks launched alone
# ------------------------------------------------------------------------------------------------------------------
def run_linear(ops, name, fp8):
    t0 = time.time()
    lin = Launch(ops, name, fp8)
    mode = "fp8" if lin.fp8 else "bf16"
    tag = f"L={ops.L} {mode} {name} ({lin.M} x {lin.N} x {lin.K})"
    full = lin.run()
    torch.cuda.synchronize()
    Bd = exact(lin.B, lin.sb)
    Bd = (Bd, Bd.abs())
    worst = 0.0
    for r0, r1 in lin.chunks():
        acc, S = lin.reference(r0, r1, Bd)
        worst = max(worst, lin.check(full, r0, r1, acc, S, tag))
        del acc, S
    del Bd
    report((ops.L, mode, name), worst)
    bits = torch.int32 if full.dtype == torch.float32 else torch.int16
    for label, m_blk, wave in lin.schedule_blocks():
        r0, r1 = 128 * m_blk, min(lin.M, 128 * m_blk + 128)
        part = lin.run(r0, r1)
        assert torch.equal(part.view(bits), full[r0:r1].view(bits)), \
            f"{tag}: rows {r0}:{r1} ({label}, wave {wave}) launched alone differ from the full launch"
    print(f"engine shapes {tag}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


SHAPE_CASES = [(L, fp8) for L in (L_FULL, 7040, 14080) for fp8 in (False, True)]


@pytest.mark.parametrize("L,fp8", SHAPE_CASES, ids=[f"L{L}-{'fp8' if f else 'bf16'}" for L, f in SHAPE_CASES])
def test_every_linear_per_element_and_row_blocks_bitwise(L, fp8):
    """Each Linear of the case's subset (the e4m3 ones in fp8 mode): every element within its bound of the float64
    product, and the row blocks of the first wave, the last wave and the last CTA's last tile, launched alone, bit for
    bit equal to the full launch's rows."""
    torch.cuda.reset_peak_memory_stats()
    ops = Operands(L)
    for name in SUBSETS[L]:
        if fp8 and not LINEARS[name][7]:
            continue
        run_linear(ops, name, fp8)
        torch.cuda.empty_cache()


@pytest.mark.parametrize("fp8", [False, True])
def test_tile_width_does_not_change_the_accumulators(fp8):
    """FA to_out's operands at 56 320 tokens in the f32 epilogue: the 64-, 128- and (bf16) 256-column tiles give the
    same fp32 accumulators bit for bit (each element is the same k-ordered chain of wgmma k-steps, whatever the
    instruction's N)."""
    lin = Launch(Operands(L_FULL), "fa_to_out", fp8)
    lin.epi, lin.gate, lin.x0 = F32, None, None
    outs = {}
    for bn in ((64, 128) if fp8 else (64, 128, 256)):
        lin.bn = bn
        outs[bn] = lin.run().view(torch.int32)
    first = outs.pop(64)
    for bn, o in outs.items():
        same = torch.equal(o, first)
        print(f"engine shapes {'fp8' if fp8 else 'bf16'} f32 accumulators block_n 64 vs {bn}: "
              f"{'bitwise equal' if same else f'{int((o != first).sum())} elements differ'}")
        assert same, f"block_n {bn} differs from block_n 64"


# ------------------------------------------------------------------------------------------------------------------
# 3: attention at the engine's shapes
# ------------------------------------------------------------------------------------------------------------------
def attention_inputs(Lq, Lk, seed):
    """q as the engine's fused to_q leaves it (unit-RMS rows times the gain with the folded scale; the rows' magnitudes
    spread 0.5x-4x so that softmaxes range from diffuse to peaked), k, token-major v and its transpose."""
    q = rows_bf16(Lq, D, seed, scale=KQ_SCALE * math.sqrt(2.0), spread=math.log10(2.828))
    k = rows_bf16(Lk, D, seed + 1, spread=0.0)
    v = rows_bf16(Lk, D, seed + 2, spread=0.0)
    return q, k, v, v.T.contiguous()


def attend(q, k, vt, Lk):
    Lq = q.shape[0]
    o = torch.full_like(q, float("nan"))
    rc = lib().g3c_attn_fwd(q.data_ptr(), k.data_ptr(), vt.data_ptr(), o.data_ptr(), Lq, Lk, HEADS, D, D, D, Lk, LN2,
                            stream())
    assert rc == 0, lib().g3c_last_error()
    return o


def sampled_rows(L):
    """Two rows of every 128-row query tile, one per consumer warpgroup (rows 0-63 / 64-127); the warp (16 rows) and
    the accumulator fragment row inside it rotate with the tile index."""
    t = torch.arange(L // 128, device="cuda")
    r_a = 16 * (t % 4) + (t // 4) % 16
    r_b = 64 + 16 * ((t + 1) % 4) + (t // 4 + 5) % 16
    return torch.stack([128 * t + r_a, 128 * t + r_b], 1).reshape(-1)


def neighbour_tile(o, tile, head):
    """o with the (query tile, head) block replaced by the next tile's."""
    bad = o.clone()
    hs = slice(head * 128, head * 128 + 128)
    nxt = tile + 1 if 128 * (tile + 2) <= o.shape[0] else tile - 1
    bad[128 * tile:128 * tile + 128, hs] = o[128 * nxt:128 * nxt + 128, hs]
    return bad


def test_self_attention_engine_shape_every_tile_and_head():
    """Self-attention 56 320 x 56 320, 32 heads, V^T with vt_chunk_len = L: two rows of every query tile of every head
    against both float64 checks.  Control: one (query tile, head) taken from its neighbour misses by >= 10x."""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    q, k, v, vt = attention_inputs(L_FULL, L_FULL, 21)
    o = attend(q, k, vt, L_FULL)
    rows = sampled_rows(L_FULL)
    ref = attn_ref64.Reference(q, k, v, HEADS, LN2, rows)
    e, s = ref.check(o[rows], "self-attention 56320 x 56320")
    report((L_FULL, "bf16", "self_attention element"), e)
    report((L_FULL, "bf16", "self_attention norm"), s)
    be, bs, _ = ref.ratios(neighbour_tile(o, 301, 17)[rows])
    print(f"engine shapes self-attention control: element {be:.3g}, norm {bs:.3g}")
    assert max(be, bs) >= 10, (be, bs)
    print(f"engine shapes self-attention: {time.time() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


def test_cross_attention_engine_shape_every_row():
    """Cross-attention 56 320 queries x 512 context keys, 32 heads: every row against both float64 checks.  Control:
    one (query tile, head) taken from its neighbour misses by >= 10x."""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    q, k, v, vt = attention_inputs(L_FULL, CTX_LEN, 31)
    o = attend(q, k, vt, CTX_LEN)
    ref = attn_ref64.Reference(q, k, v, HEADS, LN2, None, block=8192)
    e, s = ref.check(o, "cross-attention 56320 x 512")
    report((L_FULL, "bf16", "cross_attention element"), e)
    report((L_FULL, "bf16", "cross_attention norm"), s)
    be, bs, _ = ref.ratios(neighbour_tile(o, 439, 31))
    print(f"engine shapes cross-attention control: element {be:.3g}, norm {bs:.3g}")
    assert max(be, bs) >= 10, (be, bs)
    print(f"engine shapes cross-attention: {time.time() - t0:.1f} s, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------------------------------------------
# 4: GEMM negative controls on real outputs
# ------------------------------------------------------------------------------------------------------------------
def miss(lin, bad, r0, tag):
    """The ratio of the per-element check of rows [r0, r0 + 128) of `bad` to its bound (the check must fail)."""
    acc, S = lin.reference(r0, r0 + 128)
    try:
        ratio = lin.check(bad, r0, r0 + 128, acc, S, tag)
    except AssertionError:
        key = ("c8" if lin.fp8 else "c32", lin.epi, lin.K)
        ratio = OBSERVED[key] / lin.c
    else:
        raise AssertionError(f"{tag}: the check passed")
    print(f"engine shapes control {tag}: {ratio:.3g} of the bound")
    return ratio


def last_tile(lin):
    """(m_blk, n_blk, tile width) of the last tile the last CTA runs."""
    bnr = run_bn(lin.bn, lin.N, lin.fp8)
    mb, nb = -(-lin.M // 128), -(-lin.N // bnr)
    tiles = mb * nb
    grid = min(tiles, sm_count())
    m_blk, n_blk = tile_coords(grid - 1 + grid * ((tiles - grid) // grid), mb, nb,
                               super_n(bnr, lin.K, 1 if lin.fp8 else 2, nb))
    return m_blk, n_blk, bnr


def test_gemm_controls_miss_by_10x():
    """On FA to_out's and layer2's operands at 56 320 tokens (bf16), each in the last tile the last CTA runs:
    - one 64-row x 128-byte box of the f32 output replaced by the neighbouring tile's box;
    - the gated output with its term added twice;
    - layer2's gated output missing one k-block's float64 contribution (K = 16 384: 1 of 256 k-blocks).
    Each misses the per-element bound by >= 10x.  Also printed: whether test_fullsize_properties_gpu.py's sampled-row
    check (rows 0, 877, ...; rel-L2 1e-5) sees the first control."""
    ops = Operands(L_FULL)
    lin = Launch(ops, "fa_to_out", False)
    m_blk, n_blk, bnr = last_tile(lin)
    r0 = 128 * m_blk
    # 1. a box from the neighbouring tile, in the f32 epilogue (the sampled-row test's own shape and epilogue)
    lin.epi, gate, x0 = F32, lin.gate, lin.x0
    lin.gate = lin.x0 = None
    out = lin.run()
    rows, cols = slice(r0 + 64, r0 + 128), slice(n_blk * bnr + 32, n_blk * bnr + 64)
    shift = bnr if (n_blk + 1) * bnr < lin.N else -bnr
    bad = out.clone()
    bad[rows, cols] = out[rows, cols.start + shift:cols.stop + shift]
    assert miss(lin, bad, r0, "box from the neighbouring tile") >= 10
    sampled = torch.arange(0, L_FULL, 877, device="cuda")
    a = lin.A[sampled].double()
    sampled_ref = a @ lin.B.double().T
    seen = rel(bad[sampled], sampled_ref) >= 1e-5
    hit = bool(((sampled >= rows.start) & (sampled < rows.stop)).any())
    print(f"engine shapes control: the sampled-row check {'sees' if seen else 'misses'} the swapped box "
          f"(a sampled row {'lies' if hit else 'does not lie'} in it)")
    del out, bad
    # 2. the gated term of one tile added twice
    lin.epi, lin.gate, lin.x0 = GATED, gate, x0
    out = lin.run()
    acc, _ = lin.reference(r0, r0 + 128)
    cs = slice(n_blk * bnr, n_blk * bnr + bnr)
    bad = out.clone()
    bad[r0:r0 + 128, cs] = (out[r0:r0 + 128, cs].double() + gate.double()[None, cs] * acc[:, cs]).float()
    assert miss(lin, bad, r0, "gated term added twice") >= 10
    del out, bad, lin
    # 3. one k-block missing from one tile of layer2
    lin = Launch(ops, "layer2", False)
    m_blk, n_blk, bnr = last_tile(lin)
    r0, cs, ks = 128 * m_blk, slice(n_blk * bnr, n_blk * bnr + bnr), slice(64 * 100, 64 * 101)
    out = lin.run()
    part = lin.A[r0:r0 + 128, ks].double() @ lin.B[cs, ks].double().T
    bad = out.clone()
    bad[r0:r0 + 128, cs] = (out[r0:r0 + 128, cs].double() - lin.gate.double()[None, cs] * part).float()
    assert miss(lin, bad, r0, "one k-block missing (K = 16384)") >= 10
