"""Host-side mirror of the reference's inference helpers that surround the two hot paths (SURVEY.md §8 row ★).

reference: cosmos_predict1/diffusion/inference/inference_utils.py — add_common_arguments :53-171,
non_strict_load_model :217-293, load_network_model :327-347, prepare_data_batch :356-406, get_video_batch :409-455,
generate_world_from_video :542-595, compute_num_latent_frames :667-693, create_condition_latent_from_input_frames
:696-756, get_condition_latent :787-843, check_input_frames :886-913.  Same names and argument meaning; Hydra / LazyConfig
is replaced by the one hard-coded experiment (GEN3C_Cosmos_7B, config/inference/cosmos-1-diffusion-gen3c.py:22-46).
"""
from __future__ import annotations

import argparse
import os
from collections import namedtuple
from typing import Optional

import numpy as np
import torch

DEFAULT_AUGMENT_SIGMA = 0.001
NEGATIVE_PROMPT = (
    "The video captures a series of frames showing ugly scenes, static with no motion, motion blur, "
    "over-saturation, shaky footage, low resolution, grainy texture, pixelated images, poorly lit areas, "
    "underexposed and overexposed scenes, poor color balance, washed out colors, choppy sequences, "
    "jerky movements, low frame rate, artifacting, color banding, unnatural transitions, outdated special "
    "effects, fake elements, unconvincing visuals, poorly edited content, jump cuts, visual noise, and "
    "flickering. Overall, the video is of poor quality.")


def add_common_arguments(parser: argparse.ArgumentParser) -> None:
    """The reference's common command-line surface (:53-171), option for option."""
    a = parser.add_argument
    a("--checkpoint_dir", type=str, default="checkpoints", help="Base directory containing model checkpoints")
    a("--tokenizer_dir", type=str, default="Cosmos-Tokenize1-CV8x8x8-720p",
      help="Tokenizer weights directory relative to checkpoint_dir")
    a("--video_save_name", type=str, default="output", help="Output filename for generating a single video")
    a("--video_save_folder", type=str, default="outputs/", help="Output folder for generating a batch of videos")
    a("--prompt", type=str, help="Text prompt for generating a single video")
    a("--batch_input_path", type=str, help="Path to a JSONL file of input prompts for generating a batch of videos")
    a("--negative_prompt", type=str, default=NEGATIVE_PROMPT, help="Negative prompt for the video")
    a("--num_steps", type=int, default=35, help="Number of diffusion sampling steps")
    a("--guidance", type=float, default=1, help="Guidance scale value")
    a("--num_video_frames", type=int, default=121, help="Number of video frames to sample")
    a("--height", type=int, default=704, help="Height of video to sample")
    a("--width", type=int, default=1280, help="Width of video to sample")
    a("--fps", type=int, default=24, help="FPS of the sampled video")
    a("--seed", type=int, default=1, help="Random seed")
    a("--num_gpus", type=int, default=1, help="Number of GPUs used to run inference in parallel.")
    for flag, text in (("--disable_prompt_upsampler", "Disable prompt upsampling"),
                       ("--offload_diffusion_transformer", "Offload DiT after inference"),
                       ("--offload_tokenizer", "Offload tokenizer after inference"),
                       ("--offload_text_encoder_model", "Offload text encoder model after inference"),
                       ("--offload_prompt_upsampler", "Offload prompt upsampler after inference"),
                       ("--offload_guardrail_models", "Offload guardrail models after inference"),
                       ("--disable_guardrail", "Disable guardrail models"),
                       ("--disable_prompt_encoder",
                        "Disable prompt encoder to save memory, returns dummy embeddings instead")):
        a(flag, action="store_true", help=text)
    # not in the reference: an opt-in of this implementation
    a("--fp8_linear", action="store_true",
      help="Run the DiT's large Linear layers on FP8 (e4m3) tensor cores with per-row scales (off by default)")


_IncompatibleKeys = namedtuple("IncompatibleKeys", ["missing_keys", "unexpected_keys", "incorrect_shapes"])


def non_strict_load_model(model: torch.nn.Module, checkpoint_state_dict: dict) -> _IncompatibleKeys:
    """reference :217-293: drop entries whose shape disagrees with the model (reported, not fatal), ignore
    TransformerEngine's `_extra_state` blobs, load the rest non-strictly."""
    own = model.state_dict()
    incorrect = []
    for k in list(checkpoint_state_dict.keys()):
        if k not in own or "_extra_state" in k:
            continue
        if not isinstance(own[k], torch.Tensor):
            raise ValueError(f"Find non-tensor parameter {k} in the model. type: {type(own[k])} "
                             f"{type(checkpoint_state_dict[k])}, please check if this key is safe to skip or not.")
        have, want = tuple(checkpoint_state_dict[k].shape), tuple(own[k].shape)
        if have != want:
            incorrect.append((k, have, want))
            checkpoint_state_dict.pop(k)
    usable = {k: v for k, v in checkpoint_state_dict.items() if "_extra_state" not in k}
    res = model.load_state_dict(usable, strict=False)
    return _IncompatibleKeys(missing_keys=[k for k in res.missing_keys if "_extra_state" not in k],
                             unexpected_keys=[k for k in res.unexpected_keys if "_extra_state" not in k],
                             incorrect_shapes=incorrect)


def load_network_model(model, ckpt_path: str) -> _IncompatibleKeys:
    """reference :327-347.  `model.pt` of Gen3C-Cosmos-7B holds the diffusion model's state dict (optionally under a
    "model" key) with the network under the `net.` prefix; everything else in it (conditioner, logvar) has no
    counterpart here and is reported as unexpected."""
    try:
        sd = torch.load(ckpt_path, map_location="cpu", weights_only=True)
    except Exception:  # noqa: BLE001 - post-trained checkpoints pickle extra objects (reference :331-334)
        sd = torch.load(ckpt_path, map_location="cpu", weights_only=False)
    if "model" in sd:
        sd = sd["model"]
    net_sd = {k[len("net."):]: v for k, v in sd.items() if k.startswith("net.")}
    other = [k for k in sd if not k.startswith("net.")]
    res = non_strict_load_model(model.net, net_sd)
    return _IncompatibleKeys(res.missing_keys, res.unexpected_keys + other, res.incorrect_shapes)


def prepare_data_batch(height: int, width: int, num_frames: int, fps: int, prompt_embedding: torch.Tensor,
                       negative_prompt_embedding: Optional[torch.Tensor] = None, device="cuda") -> dict:
    """reference :356-406."""
    bf = torch.bfloat16
    batch = {
        "video": torch.zeros((1, 3, num_frames, height, width), dtype=torch.uint8, device=device),
        "t5_text_mask": torch.ones(1, 512, dtype=bf, device=device),
        "image_size": torch.tensor([[height, width, height, width]], dtype=bf, device=device),
        "fps": torch.tensor([fps], dtype=bf, device=device),
        "num_frames": torch.tensor([num_frames], dtype=bf, device=device),
        "padding_mask": torch.zeros((1, 1, height, width), dtype=bf, device=device),
        "t5_text_embeddings": prompt_embedding.to(device=device, dtype=bf),
    }
    if negative_prompt_embedding is not None:
        batch["neg_t5_text_embeddings"] = negative_prompt_embedding.to(device=device, dtype=bf)
        batch["neg_t5_text_mask"] = torch.ones(1, 512, dtype=bf, device=device)
    return batch


def get_video_batch(model, prompt_embedding, negative_prompt_embedding, height, width, fps, num_video_frames):
    """reference :409-455 (condition_location = "first_n" for GEN3C) -> (data_batch, state_shape [C, T, H, W])."""
    batch = prepare_data_batch(height, width, num_video_frames, fps, prompt_embedding, negative_prompt_embedding,
                               device=model.device)
    tok = model.tokenizer
    state_shape = [tok.channel, tok.get_latent_num_frames(num_video_frames), height // tok.spatial_compression_factor,
                   width // tok.spatial_compression_factor]
    return batch, state_shape


def compute_num_latent_frames(model, num_input_frames: int, downsample_factor: int = 8) -> int:
    """reference :667-693."""
    vae = model.tokenizer
    n = num_input_frames // vae.pixel_chunk_duration * vae.latent_chunk_duration
    rem = num_input_frames % vae.latent_chunk_duration
    if rem == 1:
        n += 1
    elif rem > 1:
        r = num_input_frames % vae.pixel_chunk_duration - 1
        assert r % downsample_factor == 0, (
            f"num_input_frames % model.tokenizer.video_vae.pixel_chunk_duration - 1 must be divisible by {downsample_factor}")
        n += 1 + r // downsample_factor
    return n


def create_condition_latent_from_input_frames(model, input_frames: torch.Tensor, num_frames_condition: int = 25):
    """reference :696-756 ("first_n"): the last num_frames_condition frames open a pixel chunk that is zero-padded to
    the tokenizer's chunk length and encoded."""
    B, C, T, H, W = input_frames.shape
    n_enc = model.tokenizer.pixel_chunk_duration
    assert T >= num_frames_condition, (f"input_frames not enough for condition, require at least "
                                       f"{num_frames_condition}, get {T}, {input_frames.shape}")
    assert n_enc >= num_frames_condition, (f"num_frames_encode should be larger than num_frames_condition, get "
                                           f"{n_enc}, {num_frames_condition}")
    cond = input_frames[:, :, -num_frames_condition:]
    enc_in = torch.cat([cond, cond.new_zeros(B, C, n_enc - num_frames_condition, H, W)], dim=2)
    return model.encode(enc_in), enc_in


def get_condition_latent(model, input_image_or_video_path, num_input_frames: int = 1, state_shape=None):
    """reference :787-843 for tensor input [B, C, T, H, W] in [-1, 1] or an image file (read with OpenCV, resized to the
    model resolution)."""
    if state_shape is None:
        state_shape = model.state_shape
    assert num_input_frames > 0, "num_input_frames must be greater than 0"
    H = state_shape[-2] * model.tokenizer.spatial_compression_factor
    W = state_shape[-1] * model.tokenizer.spatial_compression_factor
    if isinstance(input_image_or_video_path, str):
        import cv2

        bgr = cv2.imread(input_image_or_video_path)
        if bgr is None:
            raise FileNotFoundError(f"Input image not found: {input_image_or_video_path}")
        rgb = cv2.resize(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB), (W, H))
        frames = torch.from_numpy(rgb).permute(2, 0, 1)[None, :, None].float() / 127.5 - 1.0
        frames = frames.to(model.device)
    else:
        frames = input_image_or_video_path
    latent, _ = create_condition_latent_from_input_frames(model, frames, num_input_frames)
    return latent.to(torch.bfloat16)


def generate_world_from_video(model, state_shape, is_negative_prompt: bool, data_batch: dict, guidance: float,
                              num_steps: int, seed: int, condition_latent: torch.Tensor, num_input_frames: int):
    """reference :542-595."""
    if condition_latent.shape[2] < state_shape[1]:
        b, c, t, h, w = condition_latent.shape
        condition_latent = torch.cat([condition_latent, condition_latent.new_zeros(b, c, state_shape[1] - t, h, w)],
                                     dim=2).contiguous()
    return model.generate_samples_from_batch(
        data_batch, guidance=guidance, state_shape=state_shape, num_steps=num_steps, is_negative_prompt=is_negative_prompt,
        seed=seed, condition_latent=condition_latent, num_condition_t=compute_num_latent_frames(model, num_input_frames),
        condition_augment_sigma=DEFAULT_AUGMENT_SIGMA)


def check_input_frames(input_path, required_frames: int) -> bool:
    """reference :886-913 for images: any readable image holds one frame."""
    if not isinstance(input_path, str):
        return True
    if input_path.lower().endswith((".jpg", ".jpeg", ".png")):
        if required_frames > 1:
            return False
        return os.path.exists(input_path)
    return False


def save_video(video: np.ndarray, fps: int, H: int, W: int, video_save_quality: int, video_save_path: str) -> None:
    """utils/io.py save_video: uint8 [T, H, W, 3] -> mp4 through OpenCV (imageio / mediapy are not in this image)."""
    import cv2

    os.makedirs(os.path.dirname(os.path.abspath(video_save_path)), exist_ok=True)
    wr = cv2.VideoWriter(video_save_path, cv2.VideoWriter_fourcc(*"mp4v"), float(fps), (W, H))
    if not wr.isOpened():
        np.save(os.path.splitext(video_save_path)[0] + ".npy", video)
        return
    for frame in video:
        wr.write(cv2.cvtColor(np.ascontiguousarray(frame), cv2.COLOR_RGB2BGR))
    wr.release()
