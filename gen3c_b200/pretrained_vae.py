"""Host-side mirror of the reference's pretrained video tokenizer wrapper (SURVEY.md §8f rank 2; the caller either side
of Path D: `model.encode` / `model.decode`, model_gen3c.py:42-51, inference_utils.py:696-757).

reference: cosmos_predict1/diffusion/module/pretrained_vae.py — BasePretrainedImageVAE :96-165 (dtype handling, latent
mean / std), JITVAE :168-217 (encoder.jit / decoder.jit), BasePretrainedVideoTokenizer :314-466 (temporal chunking:
121 pixel frames <-> 16 latent frames per chunk), VideoJITTokenizer :469-509.  Same constructor keywords, properties
and `encode` / `decode` / `get_latent_num_frames` / `get_pixel_num_frames` behaviour.

As in the reference the convolutional encoder / decoder themselves are the TorchScript modules shipped in
`checkpoints/Cosmos-Tokenize1-CV8x8x8-720p/{encoder,decoder}.jit` and executed by torch — they are data, not code of
either repository.  A native sm_90a VAE is outside this round's scope (DESIGN.md §6); this wrapper is what lets the
entry point (`gen3c_b200/inference/gen3c_single_image.py`) run the real tokenizer when the checkpoint directory exists.
`SyntheticVideoTokenizer` is a weight-free stand-in with the same interface and compression factors for tests and the
synthetic end-to-end run; it is only used when the caller asks for it by name.
"""
from __future__ import annotations

import os

import torch


class VideoJITTokenizer(torch.nn.Module):
    def __init__(self, name: str = "cosmos_diffusion_tokenizer_comp8x8x8", latent_ch: int = 16, is_bf16: bool = True,
                 spatial_compression_factor: int = 8, temporal_compression_factor: int = 8, pixel_chunk_duration: int = 121,
                 max_enc_batch_size: int = 8, max_dec_batch_size: int = 4, spatial_resolution: str = "720"):
        super().__init__()
        self.name = name
        self.channel = latent_ch
        self.dtype = torch.bfloat16 if is_bf16 else torch.float32
        self._spatial_compression_factor = spatial_compression_factor
        self._temporal_compress_factor = temporal_compression_factor
        self._pixel_chunk_duration = pixel_chunk_duration
        self._spatial_resolution = spatial_resolution
        self.max_enc_batch_size, self.max_dec_batch_size = max_enc_batch_size, max_dec_batch_size
        self.encoder = self.decoder = None

    # ---- properties of the reference interface -------------------------------------------------------------
    @property
    def latent_ch(self) -> int:
        return self.channel

    @property
    def spatial_compression_factor(self) -> int:
        return self._spatial_compression_factor

    @property
    def temporal_compression_factor(self) -> int:
        return self._temporal_compress_factor

    @property
    def spatial_resolution(self) -> str:
        return self._spatial_resolution

    @property
    def pixel_chunk_duration(self) -> int:
        return self._pixel_chunk_duration

    @property
    def latent_chunk_duration(self) -> int:
        assert (self.pixel_chunk_duration - 1) % self.temporal_compression_factor == 0, (
            f"Pixel chunk duration {self.pixel_chunk_duration} minus one is not divisible by the temporal compression "
            f"factor {self.temporal_compression_factor}")
        return (self.pixel_chunk_duration - 1) // self.temporal_compression_factor + 1

    def get_latent_num_frames(self, num_pixel_frames: int) -> int:
        if num_pixel_frames == 1:
            return 1
        assert num_pixel_frames % self.pixel_chunk_duration == 0, (
            f"Temporal dimension {num_pixel_frames} is not divisible by chunk_length {self.pixel_chunk_duration}")
        return num_pixel_frames // self.pixel_chunk_duration * self.latent_chunk_duration

    def get_pixel_num_frames(self, num_latent_frames: int) -> int:
        if num_latent_frames == 1:
            return 1
        assert num_latent_frames % self.latent_chunk_duration == 0, (
            f"Temporal dimension {num_latent_frames} is not divisible by chunk_length {self.latent_chunk_duration}")
        return num_latent_frames // self.latent_chunk_duration * self.pixel_chunk_duration

    # ---- weights ------------------------------------------------------------------------------------------------
    def register_mean_std(self, vae_dir: str) -> None:
        """reference :346-364 — per-channel, per-latent-frame statistics; the first latent_chunk_duration frames are used."""
        mean, std = torch.load(os.path.join(vae_dir, "mean_std.pt"), weights_only=True)
        shape = [1, self.latent_ch, self.latent_chunk_duration, 1, 1]
        for key, val in (("latent_mean", mean), ("latent_std", std)):
            val = val.view(self.latent_ch, -1)[:, : self.latent_chunk_duration]
            self.register_buffer(key, val.to(self.dtype).reshape(*shape), persistent=False)

    def _load_jit(self, path: str):
        m = torch.jit.load(path)
        m.eval()
        for p in m.parameters():
            p.requires_grad = False
        return m.to(self.dtype)

    def load_encoder(self, vae_dir: str) -> None:
        self.encoder = self._load_jit(os.path.join(vae_dir, "encoder.jit"))

    def load_decoder(self, vae_dir: str) -> None:
        self.decoder = self._load_jit(os.path.join(vae_dir, "decoder.jit"))

    def load_weights(self, vae_dir: str) -> None:
        self.register_mean_std(vae_dir)
        self.load_decoder(vae_dir)
        self.load_encoder(vae_dir)

    def reset_dtype(self, *args, **kwargs):
        self.decoder.to(self.dtype)
        self.encoder.to(self.dtype)

    # ---- one chunk (reference JITVAE.encode / decode :124-152) ------------------------------------------------
    def _encode_chunks(self, state: torch.Tensor) -> torch.Tensor:
        in_dtype = state.dtype
        z = self.encoder(state.to(self.dtype))
        if isinstance(z, tuple):
            assert isinstance(z[0], torch.Tensor)
            z = z[0]
        elif not isinstance(z, torch.Tensor):
            raise ValueError("Invalid type of encoded state")
        return (z.to(in_dtype) - self.latent_mean.to(in_dtype)) / self.latent_std.to(in_dtype)

    def _decode_chunks(self, latent: torch.Tensor) -> torch.Tensor:
        in_dtype = latent.dtype
        latent = latent * self.latent_std.to(in_dtype) + self.latent_mean.to(in_dtype)
        return self.decoder(latent.to(self.dtype)).to(in_dtype)

    @staticmethod
    def _batched(fn, x: torch.Tensor, limit: int) -> torch.Tensor:
        if x.shape[0] <= limit:
            return fn(x)
        return torch.cat([fn(x[i:i + limit]) for i in range(0, x.shape[0], limit)], dim=0)

    # ---- public: temporal chunking (reference :384-440) ----------------------------------------------------------
    @torch.no_grad()
    def encode(self, state: torch.Tensor) -> torch.Tensor:
        """state [B, 3, T, H, W] in [-1, 1], T a multiple of pixel_chunk_duration -> latent [B, 16, T_latent, H/8, W/8]."""
        per_frame = self.temporal_compression_factor == 1
        if per_frame:
            t0 = state.shape[2]
            state = state.permute(0, 2, 1, 3, 4).reshape(-1, state.shape[1], 1, *state.shape[3:])
        B, C, T, H, W = state.shape
        n = self.pixel_chunk_duration
        assert T % n == 0, f"Temporal dimension {T} is not divisible by chunk_length {n}"
        chunks = state.reshape(B, C, T // n, n, H, W).permute(0, 2, 1, 3, 4, 5).reshape(B * (T // n), C, n, H, W)
        z = self._batched(self._encode_chunks, chunks, self.max_enc_batch_size)
        z = z.reshape(B, T // n, *z.shape[1:]).permute(0, 2, 1, 3, 4, 5).reshape(B, z.shape[1], -1, *z.shape[3:])
        if per_frame:
            z = z.reshape(-1, t0, z.shape[1], *z.shape[3:]).permute(0, 2, 1, 3, 4)
        return z

    @torch.no_grad()
    def decode(self, latent: torch.Tensor) -> torch.Tensor:
        per_frame = self.temporal_compression_factor == 1
        if per_frame:
            t0 = latent.shape[2]
            latent = latent.permute(0, 2, 1, 3, 4).reshape(-1, latent.shape[1], 1, *latent.shape[3:])
        B, C, T, H, W = latent.shape
        n = self.latent_chunk_duration
        assert T % n == 0, f"Temporal dimension {T} is not divisible by chunk_length {n}"
        chunks = latent.reshape(B, C, T // n, n, H, W).permute(0, 2, 1, 3, 4, 5).reshape(B * (T // n), C, n, H, W)
        x = self._batched(self._decode_chunks, chunks, self.max_dec_batch_size)
        assert x.shape[2] == self.pixel_chunk_duration
        x = x.reshape(B, T // n, *x.shape[1:]).permute(0, 2, 1, 3, 4, 5).reshape(B, x.shape[1], -1, *x.shape[3:])
        if per_frame:
            x = x.reshape(-1, t0, x.shape[1], *x.shape[3:]).permute(0, 2, 1, 3, 4)
        return x


class SyntheticVideoTokenizer(VideoJITTokenizer):
    """Weight-free stand-in with the tokenizer's interface and 8x8x8 compression (1 + 8k pixel frames <-> 1 + k latent
    frames per chunk): encode = causal temporal mean + 8x8 spatial mean of fixed channel mixes, decode = nearest
    up-sampling of the first 3 channels.  For tests and `--synthetic` runs only; not a model of the real VAE."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        g = torch.Generator().manual_seed(1234)
        self.register_buffer("mix", torch.randn(self.latent_ch, 3, generator=g) * 0.5, persistent=False)
        self.mix[:3] = torch.eye(3)
        shape = [1, self.latent_ch, self.latent_chunk_duration, 1, 1]
        self.register_buffer("latent_mean", torch.zeros(shape, dtype=self.dtype), persistent=False)
        self.register_buffer("latent_std", torch.ones(shape, dtype=self.dtype), persistent=False)
        self.encoder, self.decoder = self._enc, self._dec

    def load_weights(self, vae_dir: str) -> None:  # nothing to load
        return None

    def reset_dtype(self, *args, **kwargs):
        return None

    def _enc(self, x: torch.Tensor) -> torch.Tensor:
        s, f = self.spatial_compression_factor, self.temporal_compression_factor
        xs = torch.nn.functional.avg_pool3d(x.float(), (1, s, s))
        first, rest = xs[:, :, :1], xs[:, :, 1:]
        if rest.shape[2]:
            rest = rest.reshape(*rest.shape[:2], -1, f, *rest.shape[3:]).mean(dim=3)
        xt = torch.cat([first, rest], dim=2)
        return torch.einsum("oc,bcthw->bothw", self.mix.to(xt), xt).to(x.dtype)

    def _dec(self, z: torch.Tensor) -> torch.Tensor:
        s, f = self.spatial_compression_factor, self.temporal_compression_factor
        rgb = z[:, :3].float()
        t = torch.cat([rgb[:, :, :1], rgb[:, :, 1:].repeat_interleave(f, dim=2)], dim=2)
        return torch.nn.functional.interpolate(t, scale_factor=(1, s, s), mode="nearest").clamp(-1, 1).to(z.dtype)
