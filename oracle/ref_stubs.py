"""ORACLE (test infrastructure only) — import the *reference's own* modules from /root/reference on
CPU by faking the third-party packages that are absent from this container (SURVEY.md Appendix A).

Only used by ``oracle/make_golden.py`` (in the build container, where /root/reference exists) to mint
the golden vectors under ``tests/golden/``.  Nothing here runs on the GPU.

Restated third-party semantics (not in /root/reference; pins from the reference's INSTALL.md /
requirements.txt): transformer-engine 1.12.0 RMSNorm / apply_rotary_pos_emb / DotProductAttention,
megatron-core 0.10.0 parallel_state (only ``is_initialized``), warp-lang (import only).
"""
from __future__ import annotations

import os
import sys
import types

import torch

REFERENCE_ROOT = os.environ.get("GEN3C_REFERENCE_ROOT", "/root/reference")


def _mod(name: str, **attrs) -> types.ModuleType:
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


class _TERMSNorm(torch.nn.Module):
    """te.pytorch.RMSNorm(dim, eps): y = x * rsqrt(mean(x^2) + eps) * weight, computed in fp32."""

    def __init__(self, dim, eps=1e-6, **_):
        super().__init__()
        self.eps = eps
        self.weight = torch.nn.Parameter(torch.ones(dim))

    def forward(self, x):
        xf = x.float()
        y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + self.eps) * self.weight.float()
        return y.to(x.dtype)


def _rotate_half(x):
    d = x.shape[-1] // 2
    return torch.cat((-x[..., d:], x[..., :d]), dim=-1)


def _apply_rotary_pos_emb(t, freqs, tensor_format="sbhd", fused=False, **_):
    """TE apply_rotary_pos_emb, sbhd: t [s,b,h,d], freqs [s,1,1,d] fp32; rotate-half (NeoX) form."""
    assert tensor_format == "sbhd"
    cos = torch.cos(freqs).to(t.dtype)
    sin = torch.sin(freqs).to(t.dtype)
    return t * cos + _rotate_half(t) * sin


class _TEDotProductAttention(torch.nn.Module):
    def __init__(self, heads, dim_head, num_gqa_groups=None, attention_dropout=0, qkv_format="sbhd",
                 attn_mask_type="no_mask", tp_size=1, tp_group=None, sequence_parallel=False, **_):
        super().__init__()
        assert qkv_format == "sbhd" and attn_mask_type == "no_mask"
        self.cp_group = None
        self.cp_ranks = None
        self.cp_stream = None

    def set_context_parallel_group(self, cp_group, cp_ranks, cp_stream, *a, **k):
        self.cp_group, self.cp_ranks, self.cp_stream = cp_group, cp_ranks, cp_stream

    def forward(self, q, k, v, core_attention_bias_type="no_bias", core_attention_bias=None, **_):
        s, b, h, d = q.shape
        qq, kk, vv = (x.permute(1, 2, 0, 3) for x in (q, k, v))
        o = torch.nn.functional.scaled_dot_product_attention(qq, kk, vv)  # scale 1/sqrt(d)
        return o.permute(2, 0, 1, 3).reshape(s, b, h * d)


def install() -> None:
    """Insert the fakes into sys.modules and put the reference on sys.path (idempotent)."""
    if "cosmos_predict1" in sys.modules or getattr(install, "_done", False):
        return
    if not os.path.isdir(REFERENCE_ROOT):
        raise RuntimeError(f"{REFERENCE_ROOT} not present: golden vectors can only be minted in the build container")
    sys.path.insert(0, REFERENCE_ROOT)
    _mod("warp")

    class _Any:
        def __init__(self, *a, **k):
            pass

        def __getattr__(self, name):  # inert placeholder: any method is a no-op
            return lambda *a, **k: None

    oc = _mod("omegaconf", DictConfig=_Any, ListConfig=_Any, OmegaConf=_Any, SCMode=_Any)
    _mod("omegaconf.base", DictKeyType=_Any, SCMode=_Any)
    _mod("omegaconf.dictconfig", DictConfig=_Any)
    _mod("omegaconf.errors", ConfigAttributeError=Exception)
    oc.base = sys.modules["omegaconf.base"]
    _mod("iopath")
    _mod("iopath.common")
    _mod("iopath.common.file_io", HTTPURLHandler=_Any, OneDrivePathHandler=_Any, PathHandler=_Any, PathManager=_Any)

    class _ParallelState:
        @staticmethod
        def is_initialized():
            return False

    mc = _mod("megatron.core", parallel_state=_ParallelState, ModelParallelConfig=object)
    _mod("megatron", core=mc)
    _mod("megatron.core.parallel_state", is_initialized=_ParallelState.is_initialized)
    te_pt = _mod("transformer_engine.pytorch", RMSNorm=_TERMSNorm)
    te_attn = _mod("transformer_engine.pytorch.attention", apply_rotary_pos_emb=_apply_rotary_pos_emb,
                   DotProductAttention=_TEDotProductAttention)
    te_pt.attention = te_attn
    _mod("transformer_engine", pytorch=te_pt)
    # position_embedding.py:113,118 call .cuda() inside __init__
    torch.Tensor.cuda = lambda self, *a, **k: self
    install._done = True


def reference_warp_module():
    install()
    import cosmos_predict1.diffusion.inference.forward_warp_utils_pytorch as m

    return m


def reference_cache_module():
    install()
    import cosmos_predict1.diffusion.inference.cache_3d as m

    return m


def reference_dit_class():
    install()
    from cosmos_predict1.diffusion.networks.general_dit_video_conditioned import VideoExtendGeneralDIT

    return VideoExtendGeneralDIT
