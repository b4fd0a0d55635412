"""Host-side mirror of the reference's generation pipeline (SURVEY.md §8 row ★: the entry points north_star names).

reference: cosmos_predict1/diffusion/inference/gen3c_pipeline.py — Gen3cPipeline.__init__ :29-100, generate :108-184,
_run_model_with_offload :186-225, _run_model :227-260; world_generation_pipeline.py (_run_tokenizer_encoding :559-576,
_run_tokenizer_decoding :233-247); utils/base_world_generation_pipeline.py (text embedding :287-337);
auxiliary/t5_text_encoder.py.  Same constructor keywords and `generate` signature / return value.

What each reference sub-model maps to here:
  diffusion transformer  -> gen3c_b200.dit.VideoExtendGeneralDIT (native engine), weights from
                            <checkpoint_dir>/<checkpoint_name>/model.pt under the `net.` prefix (load_network_model)
  tokenizer              -> gen3c_b200.pretrained_vae.VideoJITTokenizer on <checkpoint_dir>/<tokenizer_dir> (the
                            TorchScript encoder / decoder shipped with the checkpoint, as in the reference)
  T5 text encoder        -> transformers' T5EncoderModel from <checkpoint_dir>/google-t5/t5-11b, or the reference's
                            dummy zero embeddings with disable_prompt_encoder (t5_text_encoder.py:111-132)
  prompt upsampler, guardrails -> outside the scope of this tier (DESIGN.md §6): they must be disabled explicitly,
                            enabling them raises instead of being skipped silently.
`synthetic=True` (an extension for machines without the 50 GB of checkpoints, e.g. the test box): random-init network
weights in the checkpoint layout and the weight-free SyntheticVideoTokenizer; everything else is the same code path.
"""
from __future__ import annotations

import os
from typing import Any, Optional

import numpy as np
import torch

from . import inference_utils as iu
from .dit import VideoExtendGeneralDIT
from .model_gen3c import DiffusionGen3CModel
from .pretrained_vae import SyntheticVideoTokenizer, VideoJITTokenizer


class DummyT5TextEncoder:
    """reference auxiliary/t5_text_encoder.py:111-132."""

    def __init__(self, device="cuda"):
        self.device = device

    @torch.inference_mode()
    def encode_prompts(self, prompts, max_length: int = 512):
        if isinstance(prompts, str):
            prompts = [prompts]
        if not prompts:
            raise ValueError("The input prompt list is empty.")
        emb = torch.zeros(len(prompts), max_length, 1024, device=self.device)
        mask = torch.zeros(len(prompts), max_length, device=self.device, dtype=torch.bool)
        mask[0] = True
        return emb, mask


class CosmosT5TextEncoder:
    """reference auxiliary/t5_text_encoder.py:27-108 (T5-11B encoder through transformers; no network access here, so
    the weights must already be under `cache_dir`)."""

    def __init__(self, cache_dir: str, device="cuda"):
        from transformers import T5EncoderModel, T5TokenizerFast

        self.tokenizer = T5TokenizerFast.from_pretrained(cache_dir)
        self.text_encoder = T5EncoderModel.from_pretrained(cache_dir).to(device).eval()
        self.device = device

    @torch.inference_mode()
    def encode_prompts(self, prompts, max_length: int = 512):
        if isinstance(prompts, str):
            prompts = [prompts]
        if not prompts:
            raise ValueError("The input prompt list is empty.")
        enc = self.tokenizer(prompts, return_tensors="pt", truncation=True, padding="max_length", max_length=max_length)
        ids, mask = enc.input_ids.to(self.device), enc.attention_mask.to(self.device)
        out = self.text_encoder(input_ids=ids, attention_mask=mask).last_hidden_state
        for b, n in enumerate(mask.sum(dim=1).tolist()):
            out[b][n:] = 0
        return out, mask


class Gen3cPipeline:
    def __init__(self, inference_type: str, checkpoint_dir: str, checkpoint_name: str,
                 prompt_upsampler_dir: Optional[str] = None, enable_prompt_upsampler: bool = True,
                 has_text_input: bool = True, offload_network: bool = False, offload_tokenizer: bool = False,
                 offload_text_encoder_model: bool = False, offload_prompt_upsampler: bool = False,
                 offload_guardrail_models: bool = False, disable_guardrail: bool = False,
                 disable_prompt_encoder: bool = False, guidance: float = 7.0, num_steps: int = 35, height: int = 704,
                 width: int = 1280, fps: int = 24, num_video_frames: int = 121, seed: int = 0,
                 tokenizer_dir: str = "Cosmos-Tokenize1-CV8x8x8-720p", synthetic: bool = False, device="cuda",
                 net_kwargs: Optional[dict] = None):
        assert inference_type in ("text2world", "video2world", "world_interpolator"), \
            "Invalid inference_type, must be 'text2world' or 'video2world'"
        if enable_prompt_upsampler:
            raise NotImplementedError("the Pixtral prompt upsampler is outside this engine's scope: pass "
                                      "--disable_prompt_upsampler (the reference's README commands do)")
        if not disable_guardrail:
            raise NotImplementedError("the guardrail models are outside this engine's scope: pass --disable_guardrail")
        if offload_network or offload_tokenizer or offload_text_encoder_model:
            raise NotImplementedError("model offloading is not implemented (the 7B DiT and its workspace fit one 80 GB H100)")
        self.inference_type, self.checkpoint_dir, self.checkpoint_name = inference_type, checkpoint_dir, checkpoint_name
        self.model_name = checkpoint_name
        self.enable_prompt_upsampler, self.disable_guardrail = enable_prompt_upsampler, disable_guardrail
        self.disable_prompt_encoder = disable_prompt_encoder
        self.guidance, self.num_steps, self.height, self.width = guidance, num_steps, height, width
        self.fps, self.num_video_frames, self.seed = fps, num_video_frames, seed
        self.num_input_frames = 1
        self.synthetic = synthetic
        self.device = torch.device(device)
        self.tokenizer_dir = tokenizer_dir
        self._net_kwargs = dict(net_kwargs or {})
        self._load_model()
        self._load_network()
        self._load_tokenizer()
        self._load_text_encoder_model()

    # ---- loading (reference base pipeline: _load_model / _load_network / _load_tokenizer / _load_text_encoder_model)
    def _load_model(self):
        self.model = DiffusionGen3CModel(
            state_shape=(16, 16, self.height // 8, self.width // 8), device=self.device)

    def _load_network(self):
        net = VideoExtendGeneralDIT(device=self.device, **self._net_kwargs)   # GEN3C_Cosmos_7B defaults
        self.model.net = net
        if self.synthetic:
            g = torch.Generator(device=self.device).manual_seed(1234)
            with torch.no_grad():
                for k, p in net.state_dict(keep_vars=True).items():
                    if k == "pos_embedder.seq":
                        continue
                    if p.dim() == 1:
                        p.copy_((1.0 + 0.05 * torch.randn(p.shape, device=self.device, generator=g)).to(p.dtype))
                    else:
                        p.copy_((0.02 * torch.randn(p.shape, device=self.device, generator=g)).to(p.dtype))
            return
        path = os.path.join(self.checkpoint_dir, self.checkpoint_name, "model.pt")
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} not found (download Gen3C-Cosmos-7B, or run with synthetic=True)")
        res = iu.load_network_model(self.model, path)
        if res.missing_keys or res.incorrect_shapes:
            raise RuntimeError(f"checkpoint {path} does not fit the network: missing {res.missing_keys[:5]}..., "
                               f"incorrect shapes {res.incorrect_shapes[:5]}")

    def _load_tokenizer(self):
        if self.synthetic:
            self.model.tokenizer = SyntheticVideoTokenizer().to(self.device)
            return
        tok = VideoJITTokenizer(name="cosmos_predict1_tokenizer", latent_ch=16, is_bf16=True, pixel_chunk_duration=121,
                                temporal_compression_factor=8, spatial_compression_factor=8, spatial_resolution="720")
        tok.load_weights(os.path.join(self.checkpoint_dir, self.tokenizer_dir))
        self.model.tokenizer = tok.to(self.device)

    def _load_text_encoder_model(self):
        if self.disable_prompt_encoder:
            self.text_encoder = DummyT5TextEncoder(device=self.device)
        else:
            self.text_encoder = CosmosT5TextEncoder(os.path.join(self.checkpoint_dir, "google-t5/t5-11b"), self.device)

    # ---- generation ---------------------------------------------------------------------------------------------
    def _run_text_embedding_on_prompt(self, prompts):
        embs, masks = [], []
        for p in prompts:
            e, m = self.text_encoder.encode_prompts([p])
            embs.append(e)
            masks.append(m)
        return embs, masks

    def _run_tokenizer_encoding(self, image_or_video_path) -> torch.Tensor:
        return iu.get_condition_latent(self.model, image_or_video_path, num_input_frames=self.num_input_frames,
                                       state_shape=self.model.state_shape)

    def _run_tokenizer_decoding(self, sample: torch.Tensor) -> np.ndarray:
        video = (1.0 + self.model.decode(sample.float())).clamp(0, 2) / 2
        return (video[0].permute(1, 2, 3, 0) * 255).to(torch.uint8).cpu().numpy()

    def _run_model(self, embedding, condition_latent, rendered_warp_images, rendered_warp_masks,
                   negative_prompt_embedding=None):
        batch, _state_shape = iu.get_video_batch(self.model, embedding, negative_prompt_embedding, self.height, self.width,
                                                 self.fps, self.num_video_frames)
        batch["condition_state"] = rendered_warp_images
        batch["condition_state_mask"] = rendered_warp_masks
        # the reference always takes the negative-prompt branch here (:248); without a negative prompt the
        # unconditional branch then sees the prompt's own embedding
        return iu.generate_world_from_video(self.model, self.model.state_shape, True, batch,
                                            self.guidance, self.num_steps, self.seed, condition_latent,
                                            self.num_input_frames)

    def generate(self, prompt: str, image_path, rendered_warp_images: torch.Tensor, rendered_warp_masks: torch.Tensor,
                 negative_prompt: Optional[str] = None) -> Any:
        """-> (uint8 video [T, H, W, 3], prompt)   (reference :108-184)."""
        prompts = [prompt, negative_prompt] if negative_prompt else [prompt]
        embs, _ = self._run_text_embedding_on_prompt(prompts)
        condition_latent = self._run_tokenizer_encoding(image_path)
        sample = self._run_model(embs[0], condition_latent, rendered_warp_images, rendered_warp_masks,
                                 embs[1] if negative_prompt else None)
        return self._run_tokenizer_decoding(sample), prompt
