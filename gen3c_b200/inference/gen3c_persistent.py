"""Persistent GEN3C model — load once, serve many requests (SURVEY.md §8f rank 4: the server-side caller of both paths).

reference: cosmos_predict1/diffusion/inference/gen3c_persistent.py — validate_args :26-32, resize_intrinsics :35-52,
Gen3cPersistentModel.__init__ :80-135, seed_model_from_values :138-268, inference_on_cameras :272-515,
prepare_camera_for_inference :518-534, get_cache_input_depths / W / H / clear_cache / cleanup :537-569.  Same class,
method names, arguments and return dictionaries; the HTTP layer on top of it (gui/api/server.py) is outside this tier
(DESIGN.md §6).  As in `gen3c_single_image.py` the MoGe depth model is a `depth_predictor` callable and `args.synthetic`
runs without checkpoints.
"""
from __future__ import annotations

import argparse
import os
import time
from typing import Callable, Optional

import numpy as np
import torch
import torch.nn.functional as F

from ..cache_3d import Cache3D_Buffer, Cache4D
from ..gen3c_pipeline import Gen3cPipeline
from ..inference_utils import save_video
from . import gen3c_single_image as single


def create_parser() -> argparse.ArgumentParser:
    return single.create_parser()


def validate_args(args: argparse.Namespace):
    single.validate_args(args)
    assert args.batch_input_path is None, "Unsupported in persistent mode"
    assert args.prompt is not None, "Prompt is required in persistent mode (but it can be the empty string)"
    assert args.input_image_path is None, "Image should be provided directly by value in persistent mode"
    assert args.trajectory in (None, "none"), \
        "Trajectory should be provided directly by value in persistent mode, set --trajectory=none"
    assert not args.video_save_name, ("Video saving name will be set automatically for each inference request. "
                                      f"Found string: \"{args.video_save_name}\"")


def resize_intrinsics(intrinsics, old_size, new_size, crop_size=None):
    """[n,3,3] intrinsics of (h1, w1) images -> of (h2, w2) images (optionally centre-cropped)."""
    if isinstance(intrinsics, np.ndarray):
        out = np.copy(intrinsics)
    elif isinstance(intrinsics, torch.Tensor):
        out = intrinsics.clone()
    else:
        raise ValueError(f"Invalid intrinsics type: {type(intrinsics)}")
    out[:, 0, :] *= new_size[1] / old_size[1]
    out[:, 1, :] *= new_size[0] / old_size[0]
    if crop_size is not None:
        out[:, 0, -1] = out[:, 0, -1] - (new_size[1] - crop_size[1]) / 2
        out[:, 1, -1] = out[:, 1, -1] - (new_size[0] - crop_size[0]) / 2
    return out


def _resize_bicubic(x: torch.Tensor, size) -> torch.Tensor:
    return F.interpolate(x, size=size, mode="bicubic", align_corners=False, antialias=True)


class Gen3cPersistentModel:
    @torch.no_grad()
    def __init__(self, args: argparse.Namespace, depth_predictor: Optional[Callable] = None,
                 pipeline: Optional[Gen3cPipeline] = None):
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
        self.frames_per_batch = 121
        self.inference_overlap_frames = 1
        if pipeline is None:
            pipeline = Gen3cPipeline(
                inference_type="video2world", checkpoint_dir=args.checkpoint_dir, checkpoint_name="Gen3C-Cosmos-7B",
                prompt_upsampler_dir=args.prompt_upsampler_dir, enable_prompt_upsampler=not args.disable_prompt_upsampler,
                offload_network=args.offload_diffusion_transformer, offload_tokenizer=args.offload_tokenizer,
                offload_text_encoder_model=args.offload_text_encoder_model,
                offload_prompt_upsampler=args.offload_prompt_upsampler,
                offload_guardrail_models=args.offload_guardrail_models, disable_guardrail=args.disable_guardrail,
                disable_prompt_encoder=getattr(args, "disable_prompt_encoder", False), guidance=args.guidance,
                num_steps=args.num_steps, height=args.height, width=args.width, fps=args.fps,
                num_video_frames=self.frames_per_batch, seed=args.seed, tokenizer_dir=args.tokenizer_dir,
                synthetic=getattr(args, "synthetic", False))
        if process_group is not None:
            pipeline.model.net.enable_context_parallel(process_group)
        if getattr(args, "fp8_linear", False):
            pipeline.model.net.enable_fp8_linear()
        self.args = args
        self.frame_buffer_max = pipeline.model.frame_buffer_max
        self.generator = torch.Generator(device=device).manual_seed(args.seed)
        self.sample_n_frames = pipeline.model.chunk_size
        if depth_predictor is None:
            depth_predictor = single.synthetic_depth_predictor if getattr(args, "synthetic", False) else single.load_moge(device)
        self.depth_predictor = depth_predictor
        self.pipeline = pipeline
        self.device = device
        self.device_with_rank = device
        self.cache = None
        self.model_was_seeded = False
        self.seeding_image: Optional[torch.Tensor] = None   # [B, C, T, H, W] in [-1, 1]

    # ------------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def seed_model_from_values(self, images_np: np.ndarray, depths_np: Optional[np.ndarray], world_to_cameras_np: np.ndarray,
                               focal_lengths_np: np.ndarray, principal_point_rel_np: np.ndarray, resolutions: np.ndarray,
                               masks_np: Optional[np.ndarray] = None):
        n = images_np.shape[0]
        assert images_np.shape[-1] == 3
        assert world_to_cameras_np.shape == (n, 4, 4)
        assert focal_lengths_np.shape == (n, 2)
        assert principal_point_rel_np.shape == (n, 2)
        assert resolutions.shape == (n, 2)
        assert (depths_np is None) or (depths_np.shape == images_np.shape[:-1])
        assert (masks_np is None) or (masks_np.shape == images_np.shape[:-1])
        dev = self.device_with_rank
        if n == 1:
            assert depths_np is None, ("Not supported yet: directly providing pre-estimated depth values along with a "
                                       "single image.")
            image_np = images_np[0] * 255.0     # received as 0..1 floats, the depth stage expects 0..255
            image_b1chw, depth_b11hw, _mask, w2c_b144, K_b133 = single._predict_moge_depth(
                image_np.astype(np.float32), self.args.height, self.args.width, dev, self.depth_predictor)
            input_image = image_b1chw[:, 0].clone()
            self.cache = Cache3D_Buffer(
                frame_buffer_max=self.frame_buffer_max, generator=self.generator,
                noise_aug_strength=self.args.noise_aug_strength, input_image=input_image, input_depth=depth_b11hw[:, 0],
                input_w2c=w2c_b144[:, 0], input_intrinsics=K_b133[:, 0],
                filter_points_threshold=self.args.filter_points_threshold,
                foreground_masking=self.args.foreground_masking, device=dev)
            seeding_image = torch.from_numpy(image_np.transpose(2, 0, 1)[None] / 128.0 - 1.0).float().to(dev)
            est_w2c = w2c_b144.cpu().numpy()[:, 0]
            Knp = K_b133.cpu().numpy()
            est_focal = np.stack([Knp[:, 0, 0, 0], Knp[:, 0, 1, 1]], axis=1)
            est_pp = Knp[:, 0, :2, 2]
        else:
            if depths_np is None:
                raise NotImplementedError("Seeding from multiple frames requires providing depth values.")
            if masks_np is None:
                raise NotImplementedError("Seeding from multiple frames requires providing mask values.")
            image = torch.from_numpy(images_np.transpose(0, 3, 1, 2).astype(np.float32)).to(dev) * 2.0 - 1.0
            depth = torch.from_numpy(depths_np[:, None].astype(np.float32)).to(dev)
            mask = torch.from_numpy(masks_np[:, None].astype(np.float32)).to(dev)
            w2c = torch.from_numpy(world_to_cameras_np).float().to(dev)
            K = np.zeros((n, 3, 3), dtype=np.float32)
            K[:, 0, 0], K[:, 1, 1] = focal_lengths_np[:, 0], focal_lengths_np[:, 1]
            K[:, 0, 2] = principal_point_rel_np[:, 0] * self.args.width
            K[:, 1, 2] = principal_point_rel_np[:, 1] * self.args.height
            K[:, 2, 2] = 1.0
            self.cache = Cache4D(input_image=image.clone(), input_depth=depth, input_mask=mask, input_w2c=w2c,
                                 input_intrinsics=torch.from_numpy(K).to(dev),
                                 filter_points_threshold=self.args.filter_points_threshold,
                                 foreground_masking=self.args.foreground_masking, input_format=["F", "C", "H", "W"],
                                 device=dev)
            seeding_image = image
            est_w2c, est_focal, est_pp = world_to_cameras_np, focal_lengths_np, principal_point_rel_np
        if seeding_image.shape[2] != self.H or seeding_image.shape[3] != self.W:
            seeding_image = _resize_bicubic(seeding_image, (self.H, self.W))
        self.seeding_image = seeding_image[:, :, None]
        self.model_was_seeded = True
        return est_w2c, est_focal, est_pp, np.tile([[self.args.width, self.args.height]], (n, 1))

    # ------------------------------------------------------------------------------------------------------------------
    def _depth_for_frame(self, frame):
        chw = torch.tensor(frame, device=self.device_with_rank).permute(2, 0, 1) / 255.0
        depth, mask = single._predict_moge_depth_from_tensor(chw, self.depth_predictor)
        return depth, mask, chw

    @torch.no_grad()
    def inference_on_cameras(self, view_cameras_w2cs: np.ndarray, view_camera_intrinsics: np.ndarray, fps,
                             overlap_frames: int = 1, return_estimated_depths: bool = False, video_save_quality: int = 5,
                             save_buffer: Optional[bool] = None) -> Optional[dict]:
        self.pipeline.fps = int(fps)
        save_buffer = save_buffer if save_buffer is not None else self.args.save_buffer
        name = self.args.video_save_name or f"video_{time.strftime('%Y-%m-%d_%H-%M-%S')}"
        video_save_path = os.path.join(self.args.video_save_folder, f"{name}.mp4")
        os.makedirs(self.args.video_save_folder, exist_ok=True)
        multiframe = isinstance(self.cache, Cache4D)
        w2cs, Ks = self.prepare_camera_for_inference(view_cameras_w2cs, view_camera_intrinsics, old_size=(self.H, self.W),
                                                     new_size=(self.H, self.W))
        n_total = w2cs.shape[1]
        S = self.sample_n_frames
        num_ar_iterations = (n_total - overlap_frames) // (S - overlap_frames)
        warp_images, warp_masks = self.cache.render_cache(w2cs[:, 0:S], Ks[:, 0:S], start_frame_idx=0)
        all_warps = [warp_images.clone().cpu()] if save_buffer else []
        all_depth = []
        prompt = self.args.prompt
        if prompt is None and self.args.disable_prompt_upsampler:
            return None
        start = self.seeding_image[0].unsqueeze(0) if multiframe else self.seeding_image
        out = self.pipeline.generate(prompt=prompt, image_path=start, negative_prompt=self.args.negative_prompt,
                                     rendered_warp_images=warp_images, rendered_warp_masks=warp_masks)
        if out is None:
            return None
        video, _ = out
        pred_depth = last_chw = None
        if return_estimated_depths or (num_ar_iterations > 1 and not multiframe):
            pred_depth, _, last_chw = self._depth_for_frame(video[-1])
            if return_estimated_depths:
                d0 = np.full((video.shape[0], 1, self.H, self.W), np.nan, dtype=np.float32)
                d0[-1] = pred_depth.cpu().numpy()
                all_depth.append(d0)
        for it in range(1, num_ar_iterations):
            s0 = it * (S - overlap_frames)
            s1 = s0 + S
            if multiframe:
                last_chw = torch.tensor(video[-1], device=self.device_with_rank).permute(2, 0, 1) / 255.0
            else:
                self.cache.update_cache(new_image=last_chw.unsqueeze(0) * 2 - 1, new_depth=pred_depth, new_w2c=w2cs[:, s0],
                                        new_intrinsics=Ks[:, s0])
            cache_start = 0
            if multiframe:  # hold on the last batch of cache frames when the request outruns the cache
                cache_start = min(s0, self.cache.input_frame_count() - (s1 - s0))
            warp_images, warp_masks = self.cache.render_cache(w2cs[:, s0:s1], Ks[:, s0:s1], start_frame_idx=cache_start)
            if save_buffer:
                all_warps.append(warp_images[:, overlap_frames:].clone().cpu())
            video_new, _ = self.pipeline.generate(prompt=prompt, image_path=last_chw[None, :, None] * 2 - 1,
                                                  negative_prompt=self.args.negative_prompt,
                                                  rendered_warp_images=warp_images, rendered_warp_masks=warp_masks)
            video = np.concatenate([video, video_new[overlap_frames:]], axis=0)
            if return_estimated_depths or ((it < num_ar_iterations - 1) and not multiframe):
                pred_depth, _, last_chw = self._depth_for_frame(video_new[-1])
            if return_estimated_depths:
                di = np.full((video_new.shape[0] - overlap_frames, 1, self.H, self.W), np.nan, dtype=np.float32)
                di[-1] = pred_depth.cpu().numpy()
                all_depth.append(di)
        if int(os.environ.get("RANK", "0")) == 0:
            final, final_w = video, self.args.width
            if save_buffer and all_warps:
                sq = [t.squeeze(0) for t in all_warps]
                n_max = max(t.shape[1] for t in sq)
                full = torch.cat([F.pad(t, (0, 0, 0, 0, 0, 0, 0, n_max - t.shape[1], 0, 0), value=-1.0) for t in sq], dim=0)
                T_total, _, C_dim, H_dim, W_dim = full.shape
                strip = full.permute(0, 2, 3, 1, 4).contiguous().view(T_total, C_dim, H_dim, n_max * W_dim)
                strip = ((strip * 0.5 + 0.5) * 255.0).numpy().astype(np.uint8).transpose(0, 2, 3, 1)
                final = np.concatenate([strip, final], axis=2)
                final_w = self.args.width * (1 + n_max)
            save_video(video=final, fps=self.pipeline.fps, H=self.args.height, W=final_w,
                       video_save_quality=video_save_quality, video_save_path=video_save_path)
        video_bfchw = video.transpose(0, 3, 1, 2)[None]
        return {"rendered_warp_images": warp_images, "video": video_bfchw,
                "rendered_warp_images_no_overlap": warp_images, "video_no_overlap": video_bfchw,
                "predicted_depth": np.concatenate(all_depth, axis=0) if return_estimated_depths else None,
                "video_save_path": video_save_path}

    # ------------------------------------------------------------------------------------------------------------------
    def prepare_camera_for_inference(self, view_cameras, view_camera_intrinsics, old_size, new_size):
        """Old and new sizes are (height, width).  -> ([1, F, 4, 4], [1, F, 3, 3]) on the device."""
        if isinstance(view_cameras, np.ndarray):
            view_cameras = torch.from_numpy(view_cameras).float().contiguous()
        if view_cameras.ndim == 3:
            view_cameras = view_cameras.unsqueeze(dim=0)
        if isinstance(view_camera_intrinsics, np.ndarray):
            view_camera_intrinsics = torch.from_numpy(view_camera_intrinsics).float().contiguous()
        view_camera_intrinsics = resize_intrinsics(view_camera_intrinsics, old_size, new_size).unsqueeze(dim=0)
        assert view_camera_intrinsics.ndim == 4
        return view_cameras.to(self.device_with_rank), view_camera_intrinsics.to(self.device_with_rank)

    def get_cache_input_depths(self):
        return None if self.cache is None else self.cache.input_depth

    @property
    def W(self) -> int:
        return self.args.width

    @property
    def H(self) -> int:
        return self.args.height

    def clear_cache(self) -> None:
        self.cache = None
        self.model_was_seeded = False

    def cleanup(self) -> None:
        if self.args.num_gpus > 1:
            import torch.distributed as dist

            self.pipeline.model.net._teardown_barrier()
            dist.destroy_process_group()
