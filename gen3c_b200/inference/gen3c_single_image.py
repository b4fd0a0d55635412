"""Single-image GEN3C generation — the reference's command-line entry point on the H100-native engine.

reference: cosmos_predict1/diffusion/inference/gen3c_single_image.py — create_parser :35-99, validate_args :106-108,
_predict_moge_depth :110-203, _predict_moge_depth_from_tensor :205-221, demo :223-477.  Same argparse surface (plus
`--synthetic`, `--depth_npy`), same control flow: depth -> Cache3D_Buffer -> camera trajectory -> render_cache ->
Gen3cPipeline.generate, then per 120-frame extension: depth of the last frame -> update_cache (depth alignment) ->
render_cache -> generate.

The monocular depth model (MoGe, a third-party package that is not in this image) enters through `depth_predictor`:
a callable image [3,H,W] in [0,1] -> dict(depth [H,W], mask [H,W], intrinsics [3,3] normalised) with MoGe's `infer`
contract.  Without the package: `--depth_npy file.npy` (a precomputed depth map) or `--synthetic` (a smooth synthetic
depth; random-init network weights; weight-free tokenizer) — so the whole pipeline can be exercised on a machine that
has neither checkpoints nor network access.
"""
from __future__ import annotations

import argparse
import os
from typing import Callable, Optional

import numpy as np
import torch
import torch.nn.functional as F

from ..cache_3d import Cache3D_Buffer
from ..camera_utils import generate_camera_trajectory
from ..gen3c_pipeline import Gen3cPipeline
from ..inference_utils import add_common_arguments, check_input_frames, save_video

TRAJECTORIES = ["left", "right", "up", "down", "zoom_in", "zoom_out", "clockwise", "counterclockwise", "none"]


def create_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="Video to world generation demo script")
    add_common_arguments(parser)
    a = parser.add_argument
    a("--prompt_upsampler_dir", type=str, default="Pixtral-12B",
      help="Prompt upsampler weights directory relative to checkpoint_dir")
    a("--input_image_path", type=str, help="Input image path for generating a single video")
    a("--trajectory", type=str, choices=TRAJECTORIES, default="left",
      help="Select a trajectory type from the available options (default: original)")
    a("--camera_rotation", type=str, choices=["center_facing", "no_rotation", "trajectory_aligned"],
      default="center_facing", help="Controls camera rotation during movement")
    a("--movement_distance", type=float, default=0.3, help="Distance of the camera from the center of the scene")
    a("--noise_aug_strength", type=float, default=0.0, help="Strength of noise augmentation on warped frames")
    a("--save_buffer", action="store_true",
      help="If set, save the warped images (buffer) side by side with the output video.")
    a("--filter_points_threshold", type=float, default=0.05,
      help="If set, filter the points continuity of the warped images.")
    a("--foreground_masking", action="store_true", help="If set, use foreground masking for the warped images.")
    # extensions of this repo
    a("--synthetic", action="store_true",
      help="No checkpoints: random-init 7B weights in the checkpoint layout, weight-free tokenizer, synthetic depth")
    a("--depth_npy", type=str, default=None, help="Precomputed depth map (.npy, HxW, metres) instead of MoGe")
    return parser


def parse_arguments() -> argparse.Namespace:
    return create_parser().parse_args()


def validate_args(args):
    assert args.num_video_frames is not None, "num_video_frames must be provided"
    assert (args.num_video_frames - 1) % 120 == 0, "num_video_frames must be 121, 241, 361, ... (N*120+1)"


def synthetic_depth_predictor(image_chw_0_1: torch.Tensor) -> dict:
    """MoGe-shaped output for tests: a smooth depth field (2..4.5 m) modulated by the image luminance, full mask,
    normalised pinhole intrinsics with a 60-degree horizontal field of view."""
    _, h, w = image_chw_0_1.shape
    dev = image_chw_0_1.device
    y, x = torch.meshgrid(torch.linspace(0, 1, h, device=dev), torch.linspace(0, 1, w, device=dev), indexing="ij")
    lum = F.avg_pool2d(image_chw_0_1.mean(0)[None, None], 31, 1, 15)[0, 0]
    depth = 3.0 + torch.sin(3 * x) + 0.5 * torch.cos(4 * y) + 0.3 * lum
    fx = 0.5 / np.tan(np.radians(30.0))
    K = torch.tensor([[fx, 0, 0.5], [0, fx * w / h, 0.5], [0, 0, 1]], device=dev, dtype=torch.float32)
    return {"depth": depth, "mask": torch.ones(h, w, dtype=torch.bool, device=dev), "intrinsics": K}


def load_moge(device):
    """MoGeModel.from_pretrained("Ruicheng/moge-vitl") of the reference (:286); raises when the package is absent."""
    try:
        from moge.model.v1 import MoGeModel
    except ImportError as e:  # not in this image and no network to fetch it
        raise RuntimeError("the `moge` package is not installed: pass a depth_predictor, --depth_npy or --synthetic") from e
    model = MoGeModel.from_pretrained("Ruicheng/moge-vitl").to(device)
    return model.infer


def _read_rgb(path_or_array, size_wh=None) -> np.ndarray:
    import cv2

    if isinstance(path_or_array, str):
        bgr = cv2.imread(path_or_array)
        if bgr is None:
            raise FileNotFoundError(f"Input image not found: {path_or_array}")
        rgb = cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB)
    else:
        rgb = path_or_array
    return cv2.resize(rgb, size_wh) if size_wh is not None else rgb


def _predict_moge_depth(current_image_path, target_h: int, target_w: int, device, depth_predictor: Callable):
    """reference :110-203 -> (image [1,1,3,H,W] in [-1,1], depth [1,1,1,H,W], mask [1,1,1,H,W], w2c [1,1,4,4],
    intrinsics [1,1,3,3] in pixels of the target resolution)."""
    ph, pw = 720, 1280
    rgb = _read_rgb(current_image_path, (pw, ph))
    img = torch.tensor(rgb / 255.0, dtype=torch.float32, device=device).permute(2, 0, 1)
    out = depth_predictor(img)
    depth_full, K_norm, mask_full = out["depth"], out["intrinsics"], out["mask"]
    depth_full = torch.where(mask_full == 0, torch.tensor(1000.0, device=depth_full.device), depth_full)
    K = K_norm.clone()
    K[0, 0] *= pw
    K[1, 1] *= ph
    K[0, 2] *= pw
    K[1, 2] *= ph
    depth = F.interpolate(depth_full[None, None], size=(target_h, target_w), mode="bilinear", align_corners=False)[0, 0]
    mask = F.interpolate(mask_full[None, None].float(), size=(target_h, target_w), mode="nearest")[0, 0].bool()
    image = F.interpolate(img[None], size=(target_h, target_w), mode="bilinear", align_corners=False)[0]
    K[1, 1] *= target_h / ph
    K[1, 2] *= target_h / ph
    K[0, 0] *= target_w / pw
    K[0, 2] *= target_w / pw
    depth = torch.clamp(torch.nan_to_num(depth[None, None, None], nan=1e4), min=0, max=1e4)
    w2c = torch.eye(4, dtype=torch.float32, device=device)[None, None]
    return image[None, None] * 2 - 1, depth, mask[None, None, None], w2c, K[None, None]


def _predict_moge_depth_from_tensor(image_tensor_chw_0_1: torch.Tensor, depth_predictor: Callable):
    """reference :205-221 -> (depth [1,1,H,W], mask [1,1,H,W])."""
    out = depth_predictor(image_tensor_chw_0_1)
    depth = torch.clamp(torch.nan_to_num(out["depth"][None, None], nan=1e4), min=0, max=1e4)
    mask = out["mask"][None, None]
    return torch.where(mask == 0, torch.tensor(1000.0, device=depth.device), depth), mask


def demo(args, depth_predictor: Optional[Callable] = None, pipeline: Optional[Gen3cPipeline] = None):
    """reference :223-477.  Returns the list of saved video paths (the reference returns None)."""
    torch.manual_seed(args.seed)
    np.random.seed(args.seed)
    validate_args(args)
    device = torch.device("cuda")
    process_group = None
    if args.num_gpus > 1:
        import torch.distributed as dist

        if not dist.is_initialized():
            dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
        process_group = dist.group.WORLD
    if pipeline is None:
        pipeline = Gen3cPipeline(
            inference_type="video2world", checkpoint_dir=args.checkpoint_dir, checkpoint_name="Gen3C-Cosmos-7B",
            prompt_upsampler_dir=args.prompt_upsampler_dir, enable_prompt_upsampler=not args.disable_prompt_upsampler,
            offload_network=args.offload_diffusion_transformer, offload_tokenizer=args.offload_tokenizer,
            offload_text_encoder_model=args.offload_text_encoder_model,
            offload_prompt_upsampler=args.offload_prompt_upsampler, offload_guardrail_models=args.offload_guardrail_models,
            disable_guardrail=args.disable_guardrail, disable_prompt_encoder=args.disable_prompt_encoder,
            guidance=args.guidance, num_steps=args.num_steps, height=args.height, width=args.width, fps=args.fps,
            num_video_frames=121, seed=args.seed, tokenizer_dir=args.tokenizer_dir, synthetic=args.synthetic)
    frame_buffer_max = pipeline.model.frame_buffer_max
    generator = torch.Generator(device=device).manual_seed(args.seed)
    sample_n_frames = pipeline.model.chunk_size
    if depth_predictor is None:
        if args.synthetic:
            depth_predictor = synthetic_depth_predictor
        elif args.depth_npy:
            fixed = torch.from_numpy(np.load(args.depth_npy).astype(np.float32))

            def depth_predictor(img, _d=fixed):
                d = F.interpolate(_d[None, None].to(img.device), size=img.shape[1:], mode="bilinear", align_corners=False)[0, 0]
                out = synthetic_depth_predictor(img)
                out["depth"] = d
                return out
        else:
            depth_predictor = load_moge(device)
    if process_group is not None:
        pipeline.model.net.enable_context_parallel(process_group)
    if getattr(args, "fp8_linear", False):
        pipeline.model.net.enable_fp8_linear()

    if args.batch_input_path:
        import json

        with open(args.batch_input_path) as f:
            prompts = [json.loads(line) for line in f if line.strip()]
    else:
        prompts = [{"prompt": args.prompt, "visual_input": args.input_image_path}]
    os.makedirs(os.path.dirname(os.path.abspath(args.video_save_folder)), exist_ok=True)
    saved = []
    for i, input_dict in enumerate(prompts):
        current_prompt = input_dict.get("prompt", None)
        if current_prompt is None and args.disable_prompt_upsampler:
            print("Prompt is missing, skipping world generation.")
            continue
        current_image_path = input_dict.get("visual_input", None)
        if current_image_path is None:
            print("Visual input is missing, skipping world generation.")
            continue
        if not check_input_frames(current_image_path, 1):
            print(f"Input image {current_image_path} is not valid, skipping.")
            continue
        image_b1chw, depth_b11hw, _mask, w2c_b144, K_b133 = _predict_moge_depth(
            current_image_path, args.height, args.width, device, depth_predictor)
        cache = Cache3D_Buffer(
            frame_buffer_max=frame_buffer_max, generator=generator, noise_aug_strength=args.noise_aug_strength,
            input_image=image_b1chw[:, 0].clone(), input_depth=depth_b11hw[:, 0], input_w2c=w2c_b144[:, 0],
            input_intrinsics=K_b133[:, 0], filter_points_threshold=args.filter_points_threshold,
            foreground_masking=args.foreground_masking, device=device)
        try:
            w2cs, Ks = generate_camera_trajectory(
                trajectory_type=args.trajectory, initial_w2c=w2c_b144[0, 0], initial_intrinsics=K_b133[0, 0],
                num_frames=args.num_video_frames, movement_distance=args.movement_distance,
                camera_rotation=args.camera_rotation, center_depth=1.0, device=device.type)
        except (ValueError, NotImplementedError) as e:
            print(f"Failed to generate trajectory: {e}")
            continue
        warp_images, warp_masks = cache.render_cache(w2cs[:, 0:sample_n_frames], Ks[:, 0:sample_n_frames])
        all_warps = [warp_images.clone().cpu()] if args.save_buffer else []
        video, prompt = pipeline.generate(prompt=current_prompt, image_path=current_image_path,
                                          negative_prompt=args.negative_prompt, rendered_warp_images=warp_images,
                                          rendered_warp_masks=warp_masks)
        num_ar_iterations = (w2cs.shape[1] - 1) // (sample_n_frames - 1)
        for num_iter in range(1, num_ar_iterations):
            start = num_iter * (sample_n_frames - 1)  # overlap by one frame
            end = start + sample_n_frames
            last_chw = torch.tensor(video[-1], device=device).permute(2, 0, 1) / 255.0
            pred_depth, _pred_mask = _predict_moge_depth_from_tensor(last_chw, depth_predictor)
            cache.update_cache(new_image=last_chw.unsqueeze(0) * 2 - 1, new_depth=pred_depth, new_w2c=w2cs[:, start],
                               new_intrinsics=Ks[:, start])
            warp_images, warp_masks = cache.render_cache(w2cs[:, start:end], Ks[:, start:end])
            if args.save_buffer:
                all_warps.append(warp_images[:, 1:].clone().cpu())
            video_new, prompt = pipeline.generate(prompt=current_prompt, image_path=last_chw[None, :, None] * 2 - 1,
                                                  negative_prompt=args.negative_prompt,
                                                  rendered_warp_images=warp_images, rendered_warp_masks=warp_masks)
            video = np.concatenate([video, video_new[1:]], axis=0)
        final_video, final_width = video, args.width
        if args.save_buffer and all_warps:
            sq = [t.squeeze(0) for t in all_warps]                     # (T_chunk, n_i, C, H, W)
            n_max = max(t.shape[1] for t in sq)
            full = torch.cat([F.pad(t, (0, 0, 0, 0, 0, 0, 0, n_max - t.shape[1], 0, 0), value=-1.0) for t in sq], dim=0)
            T_total, _, C_dim, H_dim, W_dim = full.shape
            strip = full.permute(0, 2, 3, 1, 4).contiguous().view(T_total, C_dim, H_dim, n_max * W_dim)
            strip = ((strip * 0.5 + 0.5) * 255.0).numpy().astype(np.uint8).transpose(0, 2, 3, 1)
            final_video = np.concatenate([strip, final_video], axis=2)
            final_width = args.width * (1 + n_max)
        path = os.path.join(args.video_save_folder, f"{i if args.batch_input_path else args.video_save_name}.mp4")
        if int(os.environ.get("RANK", "0")) == 0:
            save_video(video=final_video, fps=args.fps, H=args.height, W=final_width, video_save_quality=5,
                       video_save_path=path)
        saved.append((path, final_video))
    if args.num_gpus > 1:
        import torch.distributed as dist

        pipeline.model.net._teardown_barrier()
        dist.destroy_process_group()
    return saved


if __name__ == "__main__":
    demo(parse_arguments())
