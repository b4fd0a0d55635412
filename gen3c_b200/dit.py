"""Host-side mirror of the reference network ``VideoExtendGeneralDIT`` (Path D), backed by the native
engine in libgen3c_b200.so.

Drop-in at the reference's network seam (SURVEY.md §8b-2): same constructor keywords, same
``state_dict`` key layout (so ``checkpoints/Gen3C-Cosmos-7B/model.pt`` loads unchanged under the
``net.`` prefix), same ``forward`` keyword arguments, ``enable_context_parallel`` /
``disable_context_parallel`` / ``is_context_parallel_enabled``.  Opt-in extension: ``enable_fp8_linear`` /
``disable_fp8_linear`` / ``is_fp8_linear_enabled`` (e4m3 Linear layers, DESIGN.md §3.1).
reference: cosmos_predict1/diffusion/networks/general_dit_video_conditioned.py:30-217,
           cosmos_predict1/diffusion/networks/general_dit.py:57-569
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib


class _Node(nn.Module):
    """Anonymous container so that parameters can live under the reference's dotted key names."""


def _register(root: nn.Module, dotted: str, value: torch.Tensor, buffer: bool = False) -> None:
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Node())
        mod = mod._modules[p]
    if buffer:
        mod.register_buffer(parts[-1], value, persistent=True)
    else:
        mod.register_parameter(parts[-1], nn.Parameter(value, requires_grad=False))


class VideoExtendGeneralDIT(nn.Module):
    def __init__(
        self,
        max_img_h: int = 240,
        max_img_w: int = 240,
        max_frames: int = 128,
        in_channels: int = 16 + 16 * 4 + 1,
        out_channels: int = 16,
        patch_spatial: int = 2,
        patch_temporal: int = 1,
        concat_padding_mask: bool = True,
        block_config: str = "FA-CA-MLP",
        model_channels: int = 4096,
        num_blocks: int = 28,
        num_heads: int = 32,
        mlp_ratio: float = 4.0,
        block_x_format: str = "THWBD",
        crossattn_emb_channels: int = 1024,
        use_cross_attn_mask: bool = False,
        pos_emb_cls: str = "rope3d",
        pos_emb_learnable: bool = False,
        pos_emb_interpolation: str = "crop",
        affline_emb_norm: bool = True,
        use_adaln_lora: bool = True,
        adaln_lora_dim: int = 256,
        rope_h_extrapolation_ratio: float = 1.0,
        rope_w_extrapolation_ratio: float = 1.0,
        rope_t_extrapolation_ratio: float = 2.0,
        extra_per_block_abs_pos_emb: bool = True,
        extra_per_block_abs_pos_emb_type: str = "learnable",
        add_augment_sigma_embedding: bool = False,
        base_fps: int = 24,
        device: str | torch.device = "cuda",
        **kwargs,
    ) -> None:
        super().__init__()
        # The engine hard-codes the one experiment GEN3C runs (config/inference/cosmos-1-diffusion-gen3c.py:22-46
        # over config/base/net.py:23-43); anything else is an explicit error, not a silent fallback.
        if (patch_spatial, patch_temporal) != (2, 1):
            raise NotImplementedError("only patch_spatial=2, patch_temporal=1")
        if block_config.upper() != "FA-CA-MLP" or block_x_format != "THWBD":
            raise NotImplementedError("only block_config='FA-CA-MLP', block_x_format='THWBD'")
        if pos_emb_cls != "rope3d" or not extra_per_block_abs_pos_emb or not use_adaln_lora or not affline_emb_norm:
            raise NotImplementedError("only rope3d + learnable per-block abs-pos + adaLN-LoRA + affine emb norm")
        if use_cross_attn_mask or add_augment_sigma_embedding:
            raise NotImplementedError("cross-attention mask / augment-sigma embedding are off in GEN3C_Cosmos_7B")
        if model_channels != num_heads * 128:
            raise NotImplementedError("head_dim must be 128")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.model_channels, self.num_blocks, self.num_heads = model_channels, num_blocks, num_heads
        self.ffn_dim = int(model_channels * mlp_ratio)
        self.context_dim, self.adaln_lora_dim = crossattn_emb_channels, adaln_lora_dim
        self.concat_padding_mask = concat_padding_mask
        self.max_frames, self.max_h, self.max_w = max_frames, max_img_h // patch_spatial, max_img_w // patch_spatial
        self.rope_ratios = (rope_h_extrapolation_ratio, rope_w_extrapolation_ratio, rope_t_extrapolation_ratio)
        self.base_fps = base_fps
        self.patch_spatial, self.patch_temporal = patch_spatial, patch_temporal
        self.cp_group = None
        self.cfg_group = None
        self._fp8_linear = False
        self._handle = None
        self._registered_ptrs = None
        self._shape_key = None

        dev, dt = torch.device(device), torch.bfloat16
        D, R, Fd, Cx = model_channels, adaln_lora_dim, self.ffn_dim, crossattn_emb_channels
        kin = (in_channels + (1 if concat_padding_mask else 0)) * 4

        def z(*shape):
            return torch.zeros(*shape, device=dev, dtype=dt)

        _register(self, "x_embedder.proj.1.weight", z(D, kin))
        _register(self, "pos_embedder.seq", torch.arange(max(self.max_h, self.max_w, max_frames), device=dev,
                                                          dtype=torch.float32), buffer=True)
        _register(self, "extra_pos_embedder.pos_emb_h", z(self.max_h, D))
        _register(self, "extra_pos_embedder.pos_emb_w", z(self.max_w, D))
        _register(self, "extra_pos_embedder.pos_emb_t", z(max_frames, D))
        _register(self, "t_embedder.1.linear_1.weight", z(D, D))
        _register(self, "t_embedder.1.linear_2.weight", z(3 * D, D))
        for i in range(num_blocks):
            for j in range(3):
                p = f"blocks.block{i}.blocks.{j}."
                if j < 2:
                    k_in = D if j == 0 else Cx
                    _register(self, p + "block.attn.to_q.0.weight", z(D, D))
                    _register(self, p + "block.attn.to_q.1.weight", torch.ones(128, device=dev, dtype=dt))
                    _register(self, p + "block.attn.to_k.0.weight", z(D, k_in))
                    _register(self, p + "block.attn.to_k.1.weight", torch.ones(128, device=dev, dtype=dt))
                    _register(self, p + "block.attn.to_v.0.weight", z(D, k_in))
                    _register(self, p + "block.attn.to_out.0.weight", z(D, D))
                else:
                    _register(self, p + "block.layer1.weight", z(Fd, D))
                    _register(self, p + "block.layer2.weight", z(D, Fd))
                _register(self, p + "adaLN_modulation.1.weight", z(R, D))
                _register(self, p + "adaLN_modulation.2.weight", z(3 * D, R))
        _register(self, "final_layer.linear.weight", z(out_channels * 4, D))
        _register(self, "final_layer.adaLN_modulation.1.weight", z(R, D))
        _register(self, "final_layer.adaLN_modulation.2.weight", z(2 * D, R))
        _register(self, "affline_norm.weight", torch.ones(D, device=dev, dtype=dt))

    # ------------------------------------------------------------------------------------------
    # engine plumbing
    # ------------------------------------------------------------------------------------------
    def _engine(self):
        if self._handle is None:
            lib = _lib.load()
            cfg = _lib.DitConfig(self.model_channels, self.num_blocks, self.num_heads, self.ffn_dim, self.context_dim,
                                 self.adaln_lora_dim, self.in_channels, self.out_channels,
                                 1 if self.concat_padding_mask else 0, self.max_frames, self.max_h, self.max_w,
                                 self.rope_ratios[0], self.rope_ratios[1], self.rope_ratios[2], self.base_fps)
            h = C.c_void_p()
            _lib.check(lib.g3c_dit_create(C.byref(cfg), C.byref(h)), "g3c_dit_create")
            self._handle = h
        return self._handle

    def _sync_weights(self):
        lib = _lib.load()
        h = self._engine()
        params = [(k, v) for k, v in self.state_dict(keep_vars=True).items() if k != "pos_embedder.seq"]
        # (address, version counter): an in-place update (load_state_dict, param.copy_) keeps the address but bumps
        # the version; the engine caches derived copies (padded patch-embed weight, fp32 RMSNorm gains, abs-pos table,
        # modulation vectors) that g3c_dit_load invalidates
        ptrs = tuple((v.data_ptr(), v._version) for _, v in params)
        if ptrs == self._registered_ptrs:
            return
        for k, v in params:
            if not v.is_cuda or v.dtype != torch.bfloat16 or not v.is_contiguous():
                raise _lib.G3CError(f"weight {k} must be a contiguous CUDA bf16 tensor (got {v.dtype} on {v.device})")
            shape = (C.c_int64 * v.dim())(*v.shape)
            _lib.check(lib.g3c_dit_load(h, k.encode(), v.data_ptr(), shape, v.dim(), 0), f"g3c_dit_load({k})")
        self._registered_ptrs = ptrs

    def _set_shape(self, T: int, H: int, W: int, ctx_len: int, fps: float):
        key = (T, H, W, ctx_len, fps)
        if key != self._shape_key:
            lib = _lib.load()
            if self._shape_key is not None:
                self._teardown_barrier()  # a live peer-mapped region is about to be freed
            _lib.check(lib.g3c_dit_set_shape(self._engine(), T, H, W, ctx_len, fps), "g3c_dit_set_shape")
            if self.cp_group is not None and lib.g3c_dit_cp_mode(self._engine()) == 1:
                # fused peer-memory mode: exchange the IPC handles of the per-rank K / V^T regions (collective; plain
                # python objects, so any torch.distributed backend will do)
                import torch.distributed as dist

                buf = (C.c_uint8 * 64)()
                _lib.check(lib.g3c_dit_cp_export(self._engine(), buf), "g3c_dit_cp_export")
                allh = [None] * self._cp_size
                dist.all_gather_object(allh, bytes(buf), group=self.cp_group)
                _lib.check(lib.g3c_dit_cp_import(self._engine(), b"".join(allh), self._cp_size), "g3c_dit_cp_import")
                # every rank has resolved, allocated and mapped before anyone launches a kernel that polls a peer flag
                dist.barrier(group=self.cp_group)
            if self.cfg_group is not None:
                import torch.distributed as dist

                buf = (C.c_uint8 * 64)()
                _lib.check(lib.g3c_dit_cfg_export(self._engine(), buf), "g3c_dit_cfg_export")
                both = [None, None]
                dist.all_gather_object(both, bytes(buf), group=self.cfg_group)
                _lib.check(lib.g3c_dit_cfg_import(self._engine(), both[1 - self._cfg_role]), "g3c_dit_cfg_import")
                dist.barrier(group=self.cfg_group)
            self._shape_key = key

    def __del__(self):
        try:
            if self._handle is not None:
                _lib.load().g3c_dit_destroy(self._handle)
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------
    # context parallelism (reference: general_dit.py:524-569)
    # ------------------------------------------------------------------------------------------
    @property
    def is_context_parallel_enabled(self) -> bool:
        return self.cp_group is not None

    def enable_context_parallel(self, cp_group, mode: Optional[str] = None):
        """mode "p2p" (default; env G3C_CP_MODE): K / V^T projections store straight into every rank's buffers over
        NVLink peer memory; "nccl": one ncclAllGather of K and of V^T per layer (the baseline)."""
        import os

        import torch.distributed as dist

        mode = mode or os.environ.get("G3C_CP_MODE", "p2p")
        self._teardown_barrier()
        rank, size = dist.get_rank(cp_group), dist.get_world_size(cp_group)
        lib = _lib.load()
        raw = None
        if mode == "nccl":
            uid = torch.zeros(128, dtype=torch.uint8)
            if rank == 0:
                buf = (C.c_uint8 * 128)()
                _lib.check(lib.g3c_nccl_unique_id(buf), "g3c_nccl_unique_id")
                uid = torch.tensor(list(buf), dtype=torch.uint8)
            uid = uid.cuda()
            dist.broadcast(uid, src=dist.get_global_rank(cp_group, 0), group=cp_group)
            raw = bytes(uid.cpu().tolist())
        elif mode != "p2p":
            raise ValueError(f"unknown context-parallel mode {mode!r}")
        _lib.check(lib.g3c_dit_enable_cp(self._engine(), raw, rank, size), "g3c_dit_enable_cp")
        self.cp_group, self._cp_rank, self._cp_size = cp_group, rank, size
        self._shape_key = None

    def disable_context_parallel(self):
        self._teardown_barrier()
        if self._handle is not None:
            _lib.check(_lib.load().g3c_dit_disable_cp(self._handle), "g3c_dit_disable_cp")
        self.cp_group = None
        self._shape_key = None

    def _teardown_barrier(self):
        """Before peer-mapped regions are unmapped / freed: this rank's queued work is done and so is every peer's
        (they may still be pushing K / V^T or CFG outputs into the region this rank is about to free)."""
        if self._shape_key is None or (self.cp_group is None and self.cfg_group is None):
            return
        import torch.distributed as dist

        torch.cuda.synchronize()
        for g in (self.cp_group, self.cfg_group):
            if g is not None:
                dist.barrier(group=g)

    # ------------------------------------------------------------------------------------------
    # FP8 Linear mode (extension; DESIGN.md §3.1)
    # ------------------------------------------------------------------------------------------
    @property
    def is_fp8_linear_enabled(self) -> bool:
        return self._fp8_linear

    def enable_fp8_linear(self):
        """Run the eight large Linears of every block (self-attention to_q/to_k/to_v/to_out, cross-attention to_q/to_out,
        MLP layer1/layer2) on e4m3 codes with per-row scales: weights per output channel, activations per token.  The
        engine keeps its own e4m3 copy of those weights (6.6 GB for the 7B net), re-quantised after every weight update.
        The state_dict is unchanged."""
        self._set_linear_fp8(True)

    def disable_fp8_linear(self):
        """Back to the bf16 forward; frees the e4m3 weight copies and activation buffers."""
        self._set_linear_fp8(False)

    def _set_linear_fp8(self, on: bool):
        if on == self._fp8_linear:
            return
        self._teardown_barrier()  # the engine frees the shape's workspace, peer-mapped regions included
        _lib.check(_lib.load().g3c_dit_set_linear_fp8(self._engine(), 1 if on else 0), "g3c_dit_set_linear_fp8")
        self._fp8_linear = on
        self._shape_key = None

    # ------------------------------------------------------------------------------------------
    # classifier-free-guidance parallelism (extension; SURVEY.md §8e "CFG x CP hybrid")
    # ------------------------------------------------------------------------------------------
    @property
    def is_cfg_parallel_enabled(self) -> bool:
        return self.cfg_group is not None

    def enable_cfg_parallel(self, cfg_group):
        """`cfg_group`: a 2-rank process group; group rank 0 evaluates the conditional forward of every denoise step,
        rank 1 the unconditional one, and `sampler.denoise_step` swaps the two network outputs over NVLink peer memory.
        Both ranks must hold the same latent slice (same context-parallel rank in their respective cp groups)."""
        import torch.distributed as dist

        assert dist.get_world_size(cfg_group) == 2, "a CFG pair has exactly two ranks"
        self._teardown_barrier()
        self._cfg_role = dist.get_rank(cfg_group)
        _lib.check(_lib.load().g3c_dit_enable_cfg_parallel(self._engine(), self._cfg_role), "g3c_dit_enable_cfg_parallel")
        self.cfg_group = cfg_group
        self._shape_key = None

    def disable_cfg_parallel(self):
        self._teardown_barrier()
        if self._handle is not None:
            _lib.check(_lib.load().g3c_dit_enable_cfg_parallel(self._handle, -1), "g3c_dit_enable_cfg_parallel")
        self.cfg_group = None
        self._shape_key = None

    def _cp_slice(self, t: Optional[torch.Tensor], dim: int = 2) -> Optional[torch.Tensor]:
        """split_inputs_cp (module/parallel.py:25-53): contiguous chunk of this rank along `dim`."""
        if t is None or self.cp_group is None:
            return t
        n = t.shape[dim]
        assert n % self._cp_size == 0, f"sequence length {n} not divisible by cp size {self._cp_size}"
        c = n // self._cp_size
        return t.narrow(dim, self._cp_rank * c, c)

    # ------------------------------------------------------------------------------------------
    def _prep(self, t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
        return None if t is None else t.to(torch.bfloat16).contiguous()

    def forward(
        self,
        x: torch.Tensor,
        timesteps: torch.Tensor,
        crossattn_emb: torch.Tensor,
        crossattn_mask: Optional[torch.Tensor] = None,
        fps: Optional[torch.Tensor] = None,
        image_size: Optional[torch.Tensor] = None,
        padding_mask: Optional[torch.Tensor] = None,
        scalar_feature: Optional[torch.Tensor] = None,
        data_type=None,
        video_cond_bool: Optional[torch.Tensor] = None,
        condition_video_indicator: Optional[torch.Tensor] = None,
        condition_video_input_mask: Optional[torch.Tensor] = None,
        condition_video_augment_sigma: Optional[torch.Tensor] = None,
        condition_video_pose: Optional[torch.Tensor] = None,
        **kwargs,
    ) -> torch.Tensor:
        """x (B,16,T,H,W) [this rank's T slice under CP]; condition tensors at full T (sliced here, as the
        reference does: general_dit_video_conditioned.py:102-110).  Returns (B,16,T,H,W) bf16."""
        if scalar_feature is not None:
            raise NotImplementedError("Scalar feature is not implemented yet.")
        assert condition_video_input_mask is not None, "condition_video_input_mask is required for video data type"
        B, _, T, H, W = x.shape
        self._sync_weights()
        fps_v = float(fps.flatten()[0]) if fps is not None else float(self.base_fps)
        self._set_shape(T, H, W, crossattn_emb.shape[1], fps_v)
        mask = self._cp_slice(condition_video_input_mask)
        pose = self._cp_slice(condition_video_pose)
        if self.concat_padding_mask:
            assert padding_mask is not None
            pm = F.interpolate(padding_mask.float(), size=(H, W), mode="nearest")  # transforms resize NEAREST
        lib = _lib.load()
        out = torch.empty((B, self.out_channels, T, H, W), device=x.device, dtype=torch.bfloat16)
        ts = timesteps.flatten().float().tolist()
        with torch.cuda.device(x.device):
            for b in range(B):
                xb, mb = self._prep(x[b]), self._prep(mask[b])
                pb = self._prep(pose[b]) if pose is not None else None
                cb = self._prep(crossattn_emb[b])
                pmb = self._prep(pm[b, 0]) if self.concat_padding_mask else None
                _lib.check(lib.g3c_dit_forward(self._engine(), _lib.ptr(xb), _lib.ptr(mb), _lib.ptr(pb), _lib.ptr(pmb),
                                               ts[b if len(ts) > 1 else 0], _lib.ptr(cb), out[b].data_ptr(),
                                               _lib.stream_ptr()), "g3c_dit_forward")
        return out

    def last_launch_count(self) -> int:
        return _lib.load().g3c_dit_last_launch_count(self._engine())

    def workspace_bytes(self) -> int:
        return _lib.load().g3c_dit_workspace_bytes(self._engine())
