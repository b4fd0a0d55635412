"""Thin torch-tensor wrappers over the per-operator C ABI entry points of Path D (used by the tests,
and usable as drop-in operators, e.g. ``attention_sbhd`` behind ``attention_op.DotProductAttention``, the
``attn_op`` of the reference's ``Attention(attn_op=...)`` seam, module/attention.py:136-139).  CUDA only; no
fallback."""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib

EPI_BF16, EPI_GELU_BF16, EPI_GATED_RESIDUAL_F32, EPI_F32 = 0, 1, 2, 3


def _chk(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous CUDA tensor of dtype {dtype}")


def gemm(a: torch.Tensor, b: torch.Tensor, epilogue: int = EPI_BF16, out: Optional[torch.Tensor] = None,
         gate: Optional[torch.Tensor] = None, block_n: int = 0) -> torch.Tensor:
    """out[M,N] = a[M,K] @ b[N,K]^T on wgmma (bf16 in, fp32 accumulate).
    epilogue: EPI_BF16 | EPI_GELU_BF16 (bf16 out) | EPI_F32 (f32 out) | EPI_GATED_RESIDUAL_F32 (out f32 += gate*acc)."""
    _chk(a, torch.bfloat16, "a")
    _chk(b, torch.bfloat16, "b")
    M, K = a.shape
    N, K2 = b.shape
    assert K == K2, "inner dimensions differ"
    odt = torch.bfloat16 if epilogue in (EPI_BF16, EPI_GELU_BF16) else torch.float32
    if out is None:
        if epilogue == EPI_GATED_RESIDUAL_F32:
            raise ValueError("gated-residual epilogue accumulates into `out`")
        out = torch.empty((M, N), device=a.device, dtype=odt)
    _chk(out, odt, "out")
    if gate is not None:
        _chk(gate, torch.float32, "gate")
    lib = _lib.load()
    with torch.cuda.device(a.device):
        _lib.check(lib.g3c_gemm_bf16(_lib.ptr(a), _lib.ptr(b), _lib.ptr(out), M, N, K, K, K, N, epilogue,
                                     _lib.ptr(gate), block_n, _lib.stream_ptr()), "g3c_gemm_bf16")
    return out


def gemm_norm_rope(a: torch.Tensor, b: torch.Tensor, gamma: torch.Tensor, cos_sin: Optional[torch.Tensor] = None,
                   eps: float = 1e-6) -> torch.Tensor:
    """out[M,N] (bf16) = RoPE(RMSNorm_head(a @ b^T) * gamma): projection + per-head (128) RMSNorm + rotate-half RoPE in
    one kernel (reference: to_q / to_k = Sequential(Linear, RMSNorm) + apply_rotary_pos_emb, module/attention.py:263-283).
    gamma f32 [128]; cos_sin f32 [M, 128] (cos | sin of the 64 angles) or None."""
    _chk(a, torch.bfloat16, "a")
    _chk(b, torch.bfloat16, "b")
    _chk(gamma, torch.float32, "gamma")
    M, K = a.shape
    N = b.shape[0]
    assert b.shape[1] == K and N % 128 == 0 and gamma.numel() == 128
    if cos_sin is not None:
        _chk(cos_sin, torch.float32, "cos_sin")
        assert tuple(cos_sin.shape) == (M, 128)
    out = torch.empty((M, N), device=a.device, dtype=torch.bfloat16)
    lib = _lib.load()
    with torch.cuda.device(a.device):
        _lib.check(lib.g3c_gemm_norm_rope_bf16(_lib.ptr(a), _lib.ptr(b), _lib.ptr(out), M, N, K, K, K, N, _lib.ptr(gamma),
                                               _lib.ptr(cos_sin), eps, _lib.stream_ptr()), "g3c_gemm_norm_rope_bf16")
    return out


def _rows_ld(t: torch.Tensor, dtype, name: str) -> int:
    """Leading dimension of a 2-D CUDA tensor with contiguous rows; ValueError unless the fp8 kernels can read it."""
    if not t.is_cuda or t.dtype != dtype:
        raise ValueError(f"{name} must be a CUDA tensor of dtype {dtype}, got {t.dtype} on {t.device}")
    if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
        raise ValueError(f"{name} must be a non-empty 2-D tensor, got shape {tuple(t.shape)}")
    if t.stride(1) != 1:
        raise ValueError(f"the rows of {name} must be contiguous, got strides {t.stride()}")
    if t.data_ptr() % 16 != 0:
        raise ValueError(f"{name} must start on a 16-byte boundary")
    return t.stride(0) if t.shape[0] > 1 else t.shape[1]


def quantize_rows_fp8(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Per-row e4m3 quantisation of bf16 x [R, C] (rows contiguous, any row stride that is a multiple of 8; C a
    multiple of 16): codes [R, C] torch.float8_e4m3fn = e4m3_rn_satfinite(x * (448 / amax_r)), scales [R] float32 =
    amax_r / 448 (1 for an all-zero row), so x ~= codes * scales[:, None]."""
    ld = _rows_ld(x, torch.bfloat16, "x")
    R, Cn = x.shape
    if Cn % 16 != 0 or ld % 8 != 0:
        raise ValueError(f"x: columns ({Cn}) must be a multiple of 16 and the row stride ({ld}) of 8")
    codes = torch.empty((R, Cn), device=x.device, dtype=torch.float8_e4m3fn)
    scales = torch.empty(R, device=x.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.g3c_quantize_rows_fp8(x.data_ptr(), ld, R, Cn, codes.data_ptr(), Cn, scales.data_ptr(),
                                             _lib.stream_ptr()), "g3c_quantize_rows_fp8")
    return codes, scales


def _fp8_operands(a, scale_a, b, scale_b):
    lda, ldb = _rows_ld(a, torch.float8_e4m3fn, "a"), _rows_ld(b, torch.float8_e4m3fn, "b")
    M, K = a.shape
    N, K2 = b.shape
    if K != K2:
        raise ValueError(f"inner dimensions differ: a {tuple(a.shape)}, b {tuple(b.shape)}")
    for t, n, want in ((scale_a, "scale_a", M), (scale_b, "scale_b", N)):
        _chk(t, torch.float32, n)
        if t.numel() != want or t.data_ptr() % 16 != 0:
            raise ValueError(f"{n} must hold {want} float32 values and start on a 16-byte boundary")
    if K % 16 != 0 or lda % 16 != 0 or ldb % 16 != 0:
        raise ValueError(f"K ({K}) and the row strides of a ({lda}) and b ({ldb}) must be multiples of 16")
    return M, N, K, lda, ldb


def gemm_fp8(a: torch.Tensor, scale_a: torch.Tensor, b: torch.Tensor, scale_b: torch.Tensor, epilogue: int = EPI_BF16,
             out: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None, block_n: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue((a[M,K] @ b[N,K]^T) * scale_a[:, None] * scale_b[None, :]) on the fp8 wgmma: a, b
    torch.float8_e4m3fn codes (e.g. from quantize_rows_fp8), fp32 accumulation; epilogues as in `gemm`."""
    M, N, K, lda, ldb = _fp8_operands(a, scale_a, b, scale_b)
    odt = torch.bfloat16 if epilogue in (EPI_BF16, EPI_GELU_BF16) else torch.float32
    if out is None:
        if epilogue == EPI_GATED_RESIDUAL_F32:
            raise ValueError("gated-residual epilogue accumulates into `out`")
        out = torch.empty((M, N), device=a.device, dtype=odt)
    _chk(out, odt, "out")
    if tuple(out.shape) != (M, N):
        raise ValueError(f"out must have shape {(M, N)}, got {tuple(out.shape)}")
    if gate is not None:
        _chk(gate, torch.float32, "gate")
    lib = _lib.load()
    with torch.cuda.device(a.device):
        _lib.check(lib.g3c_gemm_fp8(a.data_ptr(), scale_a.data_ptr(), b.data_ptr(), scale_b.data_ptr(), out.data_ptr(),
                                    M, N, K, lda, ldb, N, epilogue, _lib.ptr(gate), block_n, _lib.stream_ptr()),
                   "g3c_gemm_fp8")
    return out


def gemm_norm_rope_fp8(a: torch.Tensor, scale_a: torch.Tensor, b: torch.Tensor, scale_b: torch.Tensor,
                       gamma: torch.Tensor, cos_sin: Optional[torch.Tensor] = None, eps: float = 1e-6) -> torch.Tensor:
    """`gemm_norm_rope` on e4m3 operands: the RMSNorm sees the dequantised accumulators."""
    M, N, K, lda, ldb = _fp8_operands(a, scale_a, b, scale_b)
    _chk(gamma, torch.float32, "gamma")
    if N % 128 != 0 or gamma.numel() != 128:
        raise ValueError("N must be a multiple of 128 and gamma hold 128 values")
    if cos_sin is not None:
        _chk(cos_sin, torch.float32, "cos_sin")
        if tuple(cos_sin.shape) != (M, 128):
            raise ValueError(f"cos_sin must have shape {(M, 128)}")
    out = torch.empty((M, N), device=a.device, dtype=torch.bfloat16)
    lib = _lib.load()
    with torch.cuda.device(a.device):
        _lib.check(lib.g3c_gemm_norm_rope_fp8(a.data_ptr(), scale_a.data_ptr(), b.data_ptr(), scale_b.data_ptr(),
                                              out.data_ptr(), M, N, K, lda, ldb, N, gamma.data_ptr(), _lib.ptr(cos_sin),
                                              eps, _lib.stream_ptr()), "g3c_gemm_norm_rope_fp8")
    return out


def attention(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, heads: int, scale: Optional[float] = None,
              vt_chunk_len: int = 0) -> torch.Tensor:
    """q [Lq, heads*128], k [Lk, heads*128], vt [chunks, heads*128, chunk_len] or [heads*128, Lk] (V transposed).
    Returns o [Lq, heads*128] = softmax(q k^T * scale) v per head."""
    for t, n in ((q, "q"), (k, "k"), (vt, "vt")):
        _chk(t, torch.bfloat16, n)
    Lq, Dq = q.shape
    Lk = k.shape[0]
    assert Dq == heads * 128 and k.shape[1] == heads * 128
    o = torch.empty_like(q)
    if scale is None:
        scale = 128 ** -0.5
    lib = _lib.load()
    with torch.cuda.device(q.device):
        _lib.check(lib.g3c_attn_fwd(_lib.ptr(q), _lib.ptr(k), _lib.ptr(vt), _lib.ptr(o), Lq, Lk, heads, Dq, Dq, Dq,
                                    vt_chunk_len, scale, _lib.stream_ptr()), "g3c_attn_fwd")
    return o


def _token_stride(t: torch.Tensor, name: str) -> int:
    """Leading dimension (elements) of an sbhd tensor viewed as [s, b*h*d]; ValueError unless the kernel can read it."""
    if not t.is_cuda or t.dtype != torch.bfloat16:
        raise ValueError(f"{name} must be a bf16 CUDA tensor, got {t.dtype} on {t.device}")
    if t.dim() != 4 or t.shape[0] < 1 or t[0].numel() == 0:
        raise ValueError(f"{name} must be a non-empty [s, b, h, d] tensor, got shape {tuple(t.shape)}")
    if not t[0].is_contiguous():
        raise ValueError(f"the (b, h, d) block of {name} must be contiguous, got strides {t.stride()}")
    row = t[0].numel()
    ld = t.stride(0) if t.shape[0] > 1 else row
    if ld < row or ld % 8 != 0:
        raise ValueError(f"the token stride of {name} ({ld}) must be a multiple of 8 and >= b*h*d = {row}")
    if t.data_ptr() % 16 != 0:
        raise ValueError(f"{name} must start on a 16-byte boundary")
    return ld


def _sbhd_operands(q, k, v):
    """Checks of attention_sbhd; returns the token strides of q, k and v."""
    if q.dim() == 4 and q.shape[-1] != 128:
        raise NotImplementedError(f"head_dim {q.shape[-1]}: only 128 is implemented")
    if q.dim() == 4 and k.dim() == 4 and k.shape[2] != q.shape[2]:
        raise NotImplementedError(f"{k.shape[2]} key heads for {q.shape[2]} query heads: GQA is not implemented")
    ldq, ldk, ldv = _token_stride(q, "q"), _token_stride(k, "k"), _token_stride(v, "v")
    if k.shape != v.shape or k.shape[1:] != q.shape[1:]:
        raise ValueError(f"q {tuple(q.shape)}, k {tuple(k.shape)} and v {tuple(v.shape)} must agree in (b, h, d) "
                         "and k, v in s")
    if not (q.device == k.device == v.device):
        raise ValueError("q, k and v must be on one device")
    return ldq, ldk, ldv


def _attention_sbhd_fwd(q, k, v, scale, with_lse):
    """o [sq, b, h*128] of g3c_attn_fwd_sbhd, or (o, lse) of g3c_attn_fwd_sbhd_lse."""
    ldq, ldk, ldv = _sbhd_operands(q, k, v)
    sq, b, h, d = q.shape
    o = torch.empty((sq, b, h * d), device=q.device, dtype=torch.bfloat16)
    lse = torch.empty((b * h, sq), device=q.device, dtype=torch.float32) if with_lse else None
    if scale is None:
        scale = 128 ** -0.5
    lib = _lib.load()
    with torch.cuda.device(q.device):
        args = (sq, k.shape[0], b, h, ldq, ldk, ldv, b * h * d, scale, _lib.stream_ptr())
        if with_lse:
            _lib.check(lib.g3c_attn_fwd_sbhd_lse(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                                 *args), "g3c_attn_fwd_sbhd_lse")
            return o, lse
        _lib.check(lib.g3c_attn_fwd_sbhd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), *args),
                   "g3c_attn_fwd_sbhd")
    return o


def attention_sbhd_lse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
                       scale: Optional[float] = None) -> tuple[torch.Tensor, torch.Tensor]:
    """attention_sbhd that also returns lse f32 [b*h, sq], each query row's log-sum-exp in log2 units of
    q.k * scale * log2(e) (g3c_attn_fwd_sbhd_lse), for attention_sbhd_backward.  o equals attention_sbhd's bit for bit."""
    return _attention_sbhd_fwd(q, k, v, scale, True)


def attention_sbhd_backward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, lse: torch.Tensor,
                            dout: torch.Tensor, scale: Optional[float] = None
                            ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(dq, dk, dv) of attention_sbhd_lse's (o, lse) for dout = dL/do (g3c_attn_bwd_sbhd): bf16, contiguous, in the
    shapes of q, k and v.  o and dout [sq, b, h*128] (or [sq, b, h, 128]); bitwise reproducible."""
    ldq, ldk, ldv = _sbhd_operands(q, k, v)
    sq, b, h, d = q.shape
    o4, do4 = o.view(sq, b, h, d), dout.reshape(sq, b, h, d)
    ldo, lddo = _token_stride(o4, "o"), _token_stride(do4, "dout")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (b * h, sq) or not lse.is_contiguous():
        raise ValueError(f"lse must be a contiguous float32 [{b * h}, {sq}] tensor")
    if not (o.device == dout.device == lse.device == q.device):
        raise ValueError("o, dout and lse must be on the device of q, k and v")
    if scale is None:
        scale = 128 ** -0.5
    dq, dk, dv = (torch.empty(t.shape, device=q.device, dtype=torch.bfloat16) for t in (q, k, v))
    delta = torch.empty((b * h, sq), device=q.device, dtype=torch.float32)
    row = b * h * d
    lib = _lib.load()
    with torch.cuda.device(q.device):
        _lib.check(lib.g3c_attn_bwd_sbhd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o4.data_ptr(), do4.data_ptr(),
                                         lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                         sq, k.shape[0], b, h, ldq, ldk, ldv, ldo, lddo, row, row, row, scale,
                                         _lib.stream_ptr()), "g3c_attn_bwd_sbhd")
    return dq, dk, dv


class _AttentionSbhd(torch.autograd.Function):
    """attention_sbhd inside an autograd graph: the LSE-saving forward, the native backward."""

    @staticmethod
    def forward(ctx, q, k, v, scale):
        o, lse = attention_sbhd_lse(q, k, v, scale)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.scale = scale
        return o

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dout):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = attention_sbhd_backward(q, k, v, o, lse, dout.to(torch.bfloat16).contiguous(), ctx.scale)
        return dq, dk, dv, None


def attention_sbhd(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: Optional[float] = None) -> torch.Tensor:
    """TE DotProductAttention(qkv_format="sbhd") semantics on the native kernel: q [sq, b, h, 128], k and v
    [sk, b, h, 128] (V as given, any sq, sk >= 1) -> o [sq, b, h*128] = softmax(q k^T * scale) v per (batch, head).
    scale defaults to 1/sqrt(128).  Unsupported shapes raise NotImplementedError, malformed tensors ValueError.
    Differentiable: when grad mode is on and q, k or v requires grad, the forward also keeps each row's log-sum-exp and
    the backward runs the native kernels of attention_sbhd_backward (bf16 gradients)."""
    if scale is None:
        scale = 128 ** -0.5
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        _sbhd_operands(q, k, v)
        return _AttentionSbhd.apply(q, k, v, scale)
    return _attention_sbhd_fwd(q, k, v, scale, False)


def ln_modulate(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, pos: Optional[torch.Tensor] = None,
                eps: float = 1e-6) -> torch.Tensor:
    """x (f32 [L,D], updated in place when pos is given: x += pos) ; returns bf16 LN(x)*(1+scale)+shift."""
    _chk(x, torch.float32, "x")
    L, D = x.shape
    y = torch.empty((L, D), device=x.device, dtype=torch.bfloat16)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.g3c_ln_modulate(_lib.ptr(x), _lib.ptr(pos), _lib.ptr(shift), _lib.ptr(scale), _lib.ptr(y), L, D,
                                       eps, _lib.stream_ptr()), "g3c_ln_modulate")
    return y


def ln_modulate_fp8(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, pos: Optional[torch.Tensor] = None,
                    eps: float = 1e-6) -> tuple[torch.Tensor, torch.Tensor]:
    """`ln_modulate` with the fp32 result quantised per row as by quantize_rows_fp8 (never rounded to bf16):
    returns (codes [L, D] torch.float8_e4m3fn, scales [L] float32)."""
    _chk(x, torch.float32, "x")
    L, D = x.shape
    codes = torch.empty((L, D), device=x.device, dtype=torch.float8_e4m3fn)
    scales = torch.empty(L, device=x.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        _lib.check(lib.g3c_ln_modulate_fp8(_lib.ptr(x), _lib.ptr(pos), _lib.ptr(shift), _lib.ptr(scale), codes.data_ptr(),
                                           scales.data_ptr(), L, D, eps, _lib.stream_ptr()), "g3c_ln_modulate_fp8")
    return codes, scales


def rmsnorm_rope_(qk: torch.Tensor, heads: int, gamma: torch.Tensor, cos_sin: Optional[torch.Tensor] = None,
                  eps: float = 1e-6) -> torch.Tensor:
    """In place: per-head RMSNorm (+ rotate-half RoPE with cos_sin [L,128] = cos|sin of the 64 angles)."""
    _chk(qk, torch.bfloat16, "qk")
    _chk(gamma, torch.float32, "gamma")
    L, ld = qk.shape
    lib = _lib.load()
    with torch.cuda.device(qk.device):
        _lib.check(lib.g3c_rmsnorm_rope(_lib.ptr(qk), ld, L, heads, _lib.ptr(gamma), _lib.ptr(cos_sin), eps,
                                        _lib.stream_ptr()), "g3c_rmsnorm_rope")
    return qk
